"""In-tree build of the native extension ``oktopk_b200/_C*.so`` for sm_90a (H100).

``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` for every ``.cu`` (no torch headers in
the kernels: each file compiles in seconds), ``g++`` + pybind11 for the bindings, one shared
object next to the package, so that the source tree is importable in place.
"""
from __future__ import annotations

import os
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG = Path(__file__).resolve().parent.parent
CSRC = PKG / "csrc"
BUILD = CSRC / "build"
CU_SOURCES = ["oktopk.cu", "gather.cu", "gtopk.cu", "dense.cu", "optim.cu", "bnrelu.cu", "scale.cu", "layernorm.cu",
              "xent.cu", "lstm.cu", "mlm_gather.cu", "attention.cu", "ctc.cu", "embedding.cu",
              "frame_bn.cu", "lookahead.cu"]
CPP_SOURCES = ["bindings.cpp"]
HEADERS = ["common.cuh", "oktopk.cuh", "devlib.cuh", "elem.cuh"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def so_path() -> Path:
    return PKG / ("_C" + sysconfig.get_config_var("EXT_SUFFIX"))


def _nvcc() -> str:
    for c in (os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/bin/nvcc", "/usr/local/cuda/bin/nvcc", "nvcc"):
        if os.path.exists(c) or c == "nvcc":
            return c
    return "nvcc"


def needs_build() -> bool:
    so = so_path()
    if not so.exists():
        return True
    t = so.stat().st_mtime
    return any((CSRC / f).stat().st_mtime > t for f in CU_SOURCES + CPP_SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> Path:
    so = so_path()
    if not force and not needs_build():
        return so
    import pybind11
    BUILD.mkdir(exist_ok=True)
    nvcc = _nvcc()
    cuda_home = str(Path(nvcc).resolve().parent.parent) if os.path.sep in nvcc else "/usr/local/cuda"
    py_inc = sysconfig.get_paths()["include"]
    cmds, objs = [], []
    for f in CU_SOURCES:
        o = BUILD / (f + ".o")
        objs.append(str(o))
        cmds.append([nvcc, *ARCH, "-lineinfo", "-O3", "-std=c++17", "-Xptxas", "-v", "-Xcompiler", "-fPIC",
                     "-c", str(CSRC / f), "-o", str(o)])
    for f in CPP_SOURCES:
        o = BUILD / (f + ".o")
        objs.append(str(o))
        cmds.append(["g++", "-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-I", pybind11.get_include(), "-I", py_inc,
                     "-I", cuda_home + "/include", "-c", str(CSRC / f), "-o", str(o)])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    with ThreadPoolExecutor(max_workers=len(cmds)) as ex:
        logs = list(ex.map(run, cmds))
    (BUILD / "ptxas.log").write_text("\n".join(logs))
    if verbose:
        print("\n".join(logs))
    link = [nvcc, *ARCH, "-shared", "-o", str(so), *objs, "-cudart", "static"]
    run(link)
    return so


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
