"""Loader of the native extension.  On a GPU box a missing/unloadable extension is a hard error
(no silent eager fallback: the CUDA path is the product); on a CPU-only box ``available()`` is
simply False and the torch.distributed ("dist") backend is used."""
from __future__ import annotations

import importlib
import os
from typing import Optional

import torch

_C = None
_ERR: Optional[BaseException] = None

# kernels launched by this package since import (the bench reports the delta over its timed region)
LAUNCH_COUNT = {"total": 0}
_LAUNCHERS = {"oktopk_run": 1, "gather_run": 1, "gtopk_run": 1, "dense_run": 1, "kth_abs": 1, "fused_sgd": 1,
              "sgd_ahead": 1, "fused_sgd_tail": 1, "fused_bert_adam": 1, "fused_adam": 1, "momentum_correct": 1, "clip_by_norm": 2, "land_grads": 1, "bn_forward": 1, "bn_backward": 1,
              "maxpool2_fwd": 1, "maxpool2_bwd": 1, "unscale_check": 1, "ln_forward": 1, "ln_backward": 2,
              "xent_forward": 2, "xent_backward": 1, "lstm_forward": 1, "lstm_backward": 1, "mlm_select": 1,
              "mlm_gather": 1, "mlm_scatter": 1, "attn_forward": 1, "attn_backward": 2, "lstm_seq_forward": 1,
              "lstm_seq_backward": 1, "ctc_forward": 2, "ctc_backward": 1, "emb_forward": 1, "emb_backward": 3,
              "frame_bn_forward": 1, "frame_bn_backward": 1}


class _CountingModule:
    """Thin proxy over the native module that counts kernel launches per entry point."""

    def __init__(self, mod):
        self._mod = mod
        for name, per_call in _LAUNCHERS.items():
            setattr(self, name, self._wrap(getattr(mod, name), name, per_call))

    def _wrap(self, fn, name, per_call):
        def call(*a, **kw):
            n = per_call
            if name == "oktopk_run" and isinstance(a[9], dict) and a[9].get("split_phases"):
                n = 7
            if name == "land_grads":
                n = max(1, (len(a[0]) + 95) // 96)
            LAUNCH_COUNT["total"] += n
            LAUNCH_COUNT[name] = LAUNCH_COUNT.get(name, 0) + n
            return fn(*a, **kw)
        return call

    def __getattr__(self, name):
        return getattr(self._mod, name)


def load(build_if_missing: bool = True):
    """Import ``oktopk_b200._C`` (building it in-tree first if nvcc is around and it is stale)."""
    global _C, _ERR
    if _C is not None:
        return _C
    try:
        from . import build as _b
        if build_if_missing and _b.needs_build() and os.environ.get("OKTOPK_NO_BUILD", "0") != "1":
            _b.build()
        _C = _CountingModule(importlib.import_module("oktopk_b200._C"))
        _ERR = None
    except Exception as e:  # noqa: BLE001
        _ERR = e
        _C = None
    return _C


# The kernels' storage-type code of an fp32 / bf16 / fp16 tensor (csrc/oktopk.cuh Dtype; bindings reject other codes).
DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}


def dense16(t: torch.Tensor) -> torch.Tensor:
    """Contiguous and 16-byte aligned (the kernels move 128-bit vectors), copied once if it is not."""
    t = t.contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def available() -> bool:
    return load() is not None


def require():
    c = load()
    if c is None:
        raise RuntimeError("oktopk_b200 native extension (_C) is not available: %r" % (_ERR,))
    return c


class DevPtr:
    """A raw device allocation exposed through ``__cuda_array_interface__`` so that
    ``torch.as_tensor(DevPtr(...), device='cuda')`` aliases it without a copy."""

    def __init__(self, ptr: int, numel: int, typestr: str = "<f4"):
        self.ptr, self.numel, self.typestr = int(ptr), int(numel), typestr

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.numel,), "typestr": self.typestr, "data": (self.ptr, False), "version": 3,
                "strides": None}


def tensor_from_ptr(ptr: int, numel: int, dtype="float32", device=None):
    ts = {"float32": "<f4", "int32": "<i4", "uint8": "|u1", "int64": "<i8"}[dtype]
    dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
    return torch.as_tensor(DevPtr(ptr, numel, ts), device=dev)
