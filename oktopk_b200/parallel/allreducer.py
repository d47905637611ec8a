"""``AllReducer``: the sparse-allreduce engine front end (L4 of the reference's layer map).

Two faces, like the reference:
  * synchronous functional form (BERT flavour, ``BERT/bert/allreducer.py:182,347``):
    ``AllReducer(compression, sparse, density).run(flat_grad) -> flat_grad``;
  * named buckets for the optimizer wrapper (CNN/LSTM flavour, ``VGG/allreducer.py:191-473``:
    ``add_tensor`` / ``get_result`` / ``train_epoch`` / ``get_current_density`` / ``stop``) -- but
    without the consumer thread, the queues and the per-hook ``torch.cuda.synchronize()``: a
    bucket's reduction is enqueued on a CUDA stream the moment its last gradient lands.

Backends: ``cuda`` = fused sm_90a kernels over peer memory (``gpu_engine.py``); ``dist`` = the
same schemes on ``torch.distributed`` collectives (``algorithms.py``; CPU/gloo plumbing and the
NCCL baseline).
"""
from __future__ import annotations

import time
from typing import Dict, Optional

import torch

from ..compression import Compressor, resolve_compressor
from ..config import OkTopkConfig
from ..ops import ext
from . import algorithms
from .state import SparseState
from .world import World, world as _world


def _capturing() -> bool:
    return torch.cuda.is_available() and torch.cuda.is_current_stream_capturing()


class AllReducer:
    def __init__(self, compression="oktopk", sparse: bool = True, density: float = 0.01, train_epoch: int = 0,
                 cfg: Optional[OkTopkConfig] = None, world: Optional[World] = None, backend: Optional[str] = None,
                 named_parameters=None, err_callback=None, layerwise_times=None, sigma_scale: float = 2.5,
                 norm_clip: Optional[float] = None, writer=None, **_ignored):
        base = cfg if cfg is not None else OkTopkConfig()
        self.compressor: Compressor = resolve_compressor(compression, base)
        over = {"sparse": bool(sparse) and self.compressor.name != "none", "compressor": self.compressor.name}
        if cfg is None:
            over.update(density=density, sigma_scale=sigma_scale, norm_clip=norm_clip)
        self.cfg = base.replace(**over)
        if backend is not None:
            self.cfg = self.cfg.replace(backend=backend)
        self.compressor.cfg = self.cfg
        self.world = world if world is not None else _world()
        self.train_epoch = train_epoch
        self.err_callback = err_callback           # kept for API parity; see utils/elastic.py
        self.writer = writer
        self._dist_states: Dict[str, SparseState] = {}
        self._engines: Dict[str, "object"] = {}
        self._timers: Dict[str, list] = {}
        self._running = True
        self.profile_records: list = []              # filled when settings.PROFILING_NORM is on
        self._profiling_norms: list = []             # (gtopk_norm, randk_norm, upbound, xnorm, dense_std), VGG/allreducer.py:1418
        self._prof_calls: Dict[str, int] = {}

    # ------------------------------------------------------------------ density schedule
    def get_current_density(self) -> float:
        """``VGG/allreducer.py:451-458``: optional per-epoch density schedule."""
        dd = self.cfg.dynamic_densities
        if dd:
            return float(dd[min(self.train_epoch, len(dd) - 1)])
        return float(self.cfg.density)

    # ------------------------------------------------------------------ backend choice
    def _use_cuda(self, device: torch.device) -> bool:
        if device.type != "cuda" or self.cfg.backend == "dist":
            return False
        if not ext.available():
            if self.cfg.backend == "cuda" or device.type == "cuda":
                ext.require()       # GPU box without the extension: fail loudly, no silent fallback
            return False
        return True

    # ------------------------------------------------------------------ bucket registration (optimizer path)
    def register_bucket(self, name: str, numel: int, device: torch.device) -> torch.Tensor:
        """Create the bucket's engine/state and return the flat fp32 gradient buffer to alias."""
        if self._use_cuda(device):
            from .gpu_engine import CudaBucketEngine
            eng = CudaBucketEngine(numel, self.cfg, self.world, name=name)
            self._engines[name] = eng
            return eng.grad
        self._dist_states[name] = SparseState(numel, self.world.size)
        return torch.zeros(numel, dtype=torch.float32, device=device)

    def reads_sources(self, name: str) -> bool:
        """True if the next reduction of bucket ``name`` can read the gradient straight from autograd's tensors
        (``reduce_bucket(srcs=...)``) instead of from the bucket.  Not in the diagnostic modes, which read the bucket."""
        from ..utils import settings
        eng = self._engines.get(name)
        if eng is None or settings.PROFILING_GRAD or settings.PROFILING_NORM:
            return False
        return eng.reads_sources(self.compressor.name, self.get_current_density())

    def packs_early(self, name: str) -> bool:
        """True if the next reduction of bucket ``name`` may pack ready gradients during backward (``pack_segment``);
        the caller reads the gradient from its sources and runs without loss scaling."""
        from ..utils import settings
        eng = self._engines.get(name)
        if eng is None or settings.PROFILING or settings.PROFILING_GRAD or settings.PROFILING_NORM:
            return False
        return eng.packs_early(self.compressor.name, self.get_current_density())

    def pack_segment(self, name: str, ranges, srcs, stream=None) -> None:
        self._engines[name].pack_segment(self.compressor.name, ranges, srcs, self.get_current_density(), stream)

    def reduce_bucket(self, name: str, flat: torch.Tensor, stream=None, srcs=None, scale=None,
                      pack_ranges=None) -> torch.Tensor:
        """Reduce bucket ``name`` in place.  ``srcs = (pointers, offsets, lengths)``: the gradient is in these fp32
        tensors rather than in ``flat``, which must then be all-zero (only where ``reads_sources(name)``).

        ``scale``: the optimizer's loss-scale state (``optimizer._ScaleState``).  The gradient is unscaled first, and the
        reduction is skipped on every rank when any rank's bucket holds a non-finite value (``config.LossScale``)."""
        skip = 0
        if scale is not None:
            eng = self._engines.get(name)
            if eng is not None:                   # on the device: no host synchronisation, graph-replayable
                eng.unscale_check(scale.ptr, stream, srcs)
                skip = eng.verdict_ptr
            elif scale.check_host(flat, self.world):
                st = self._dist_states.get(name)
                if st is None:
                    st = self._dist_states[name] = SparseState(flat.numel(), self.world.size)
                st.counter += 1
                return flat
        density = self.get_current_density()
        from ..utils import settings
        if settings.PROFILING_GRAD and self.cfg.sparse:
            self._dump_grad(name, flat, density)
        if settings.PROFILING_NORM and self.cfg.sparse:
            return self._reduce_profiled(name, flat, stream, density, skip)
        if name in self._engines:
            out = self._engines[name].reduce(self.compressor.name, density, stream=stream, g=flat, srcs=srcs,
                                             skip=skip, pack_ranges=pack_ranges)
            if settings.PROFILING:
                self._profile_iteration(name)
            return out
        st = self._dist_states.get(name)
        if st is None:
            st = self._dist_states[name] = SparseState(flat.numel(), self.world.size)
        t0 = time.perf_counter()
        out = algorithms.sparse_allreduce(self.compressor.name, flat, st, self.cfg, self.world, density)
        self._timers.setdefault(name, []).append(time.perf_counter() - t0)
        return out

    # ------------------------------------------------------------------ settings.PROFILING / PROFILING_GRAD
    def _profile_iteration(self, name: str) -> None:
        """``settings.PROFILING`` (``VGG/allreducer.py:608-623,702-703,848-849``): rank 0 prints the selected counts and
        thresholds of every call, and every 50 calls the mean per-phase times (``_print_profiling``, :379-443) -- here
        the phases are the device-side stamps of the fused kernel, not host wall-clock.  Synchronous (diagnostic mode)."""
        eng = self._engines[name]
        if _capturing():
            return
        st = eng.stats()
        c = self._prof_calls[name] = self._prof_calls.get(name, 0) + 1
        if self.world.rank == 0:
            print("counter: %d rank: %d mode: %s local topk elements: %d localtopk threshold: %.6g global topk elements: %d "
                  "globaltopk threshold: %.6g overflow: %d/%d redo: %d" % (
                      st["counter"], self.world.rank, st["mode"], st["local_count"], st["local_thr_used"], st["global_count"],
                      st["global_thr"], st["overflow_send"], st["overflow_gather"], st.get("redo", 0)), flush=True)
        if c % 50 == 0:
            self._print_profiling(name)

    def _print_profiling(self, name: Optional[str] = None) -> Dict[str, Dict[str, float]]:
        """Mean device-side phase durations (microseconds) over the last <= 50 fused calls of each bucket."""
        out = {}
        for nm, eng in self._engines.items():
            if name is not None and nm != name:
                continue
            recs = eng.trace()[-50:]
            if not recs:
                continue
            keys = [k for k in recs[0] if k.startswith("us_")]
            means = {k: sum(r[k] for r in recs) / len(recs) for k in keys}
            out[nm] = means
            if self.world.rank == 0:
                print("[rank:%d]%s[%d]: " % (self.world.rank, nm[:24], eng.n) +
                      ", ".join("%s %.1f" % (k[3:], v) for k, v in means.items()) + " (us, mean of %d calls)" % len(recs),
                      flush=True)
        return out

    def _dump_grad(self, name: str, flat: torch.Tensor, density: float) -> None:
        """``settings.PROFILING_GRAD`` (``VGG/allreducer.py:854-888``): snapshots of the error-compensated local gradient
        and of the Ok-Topk / Gaussian-estimate thresholds at chosen iterations (``OKTOPK_GRAD_DUMP_ITERS``, default the
        reference's 3991-3995,12991-12995), written as .npy next to the logs by rank 0."""
        import os
        import numpy as np
        from ..compression import gen_threshold_from_normal_distribution
        from ..utils import settings
        if _capturing():
            return
        eng = self._engines.get(name)
        st = self._dist_states.get(name)
        counter = eng.host.counter if eng is not None else (st.counter if st is not None else 0)
        spec = os.environ.get("OKTOPK_GRAD_DUMP_ITERS", "3991-3995,12991-12995")
        hit = False
        for part in spec.split(","):
            lo, _, hi = part.partition("-")
            if lo.strip() and int(lo) <= counter <= int(hi or lo):
                hit = True
        res = eng.residual if eng is not None else (st.residual if st is not None else None)
        with torch.no_grad():
            acc = flat.detach().clone()
            if res is not None and res.numel() == acc.numel():
                acc += res
            k = max(int(acc.numel() * density), 1)
            gk_thr = float(gen_threshold_from_normal_distribution(1.0 - density, float(acc.mean()), float(acc.std()))[1])
            gk_topk = int((acc.abs() > gk_thr).sum())
            ok_thr = float(eng.stats()["local_thr"]) if eng is not None else float(getattr(st, "local_thr", 0.0))
        if self.world.rank == 0:
            print("counter: %d rank: %d ok_gk_local_thrds: [%.6g %.6g] gk_localtopk_value: %d" %
                  (counter, self.world.rank, ok_thr, gk_thr, gk_topk), flush=True)
            if hit:
                d = settings.PREFIX or "."
                os.makedirs(d, exist_ok=True)
                np.save(os.path.join(d, "localgrad%d_k%d.npy" % (counter, k)), acc.cpu().numpy())
                np.save(os.path.join(d, "localthrds%d_k%d.npy" % (counter, k)), np.asarray([ok_thr, gk_thr], dtype="float32"))

    def save_profiling_norms(self, directory: str, epoch: int) -> None:
        """Per-epoch ``gtopknorm/randknorm/upbound/densestd-rank%d-epoch%d.npy`` (``VGG/main_trainer.py:107-139``)."""
        import os
        import numpy as np
        if not self._profiling_norms:
            return
        os.makedirs(directory, exist_ok=True)
        cols = list(zip(*self._profiling_norms))
        for nm, col in zip(("gtopknorm", "randknorm", "upbound", "xnorm", "densestd"), cols):
            np.save(os.path.join(directory, "%s-rank%d-epoch%d.npy" % (nm, self.world.rank, epoch)), np.asarray(col))
        self._profiling_norms = []

    def _reduce_profiled(self, name: str, flat: torch.Tensor, stream, density: float, skip: int = 0) -> torch.Tensor:
        """``settings.PROFILING_NORM`` (``VGG/allreducer.py:584-606,1072-1080``): one extra dense allreduce of the
        error-compensated gradient per step gives the true global top-k, against which the sparse result's relative
        error (the paper's xi) and the selected counts are recorded.  Diagnostic mode: synchronous and slow."""
        from ..utils.metrics import sparsification_error
        eng = self._engines.get(name)
        st = self._dist_states.get(name)
        res = eng.residual if eng is not None else (st.residual if st is not None else None)
        with torch.no_grad():
            acc = flat.detach().clone()
            if res is not None and res.numel() == acc.numel():
                acc += res
            if self.world.size > 1:
                self.world.all_reduce_sum(acc)
            acc /= self.world.size
        if eng is not None:
            out = eng.reduce(self.compressor.name, density, stream=stream, g=flat, skip=skip)
            if flat.is_cuda:
                torch.cuda.synchronize()
        else:
            if st is None:
                st = self._dist_states[name] = SparseState(flat.numel(), self.world.size)
            out = algorithms.sparse_allreduce(self.compressor.name, flat, st, self.cfg, self.world, density)
        k = max(int(flat.numel() * density), 1)
        rec = sparsification_error(acc, out, k)
        rec["bucket"], rec["density"] = name, density
        self.profile_records.append(rec)
        # the reference's tuple for the gather/tree schemes (VGG/allreducer.py:1361-1418): error of the sparse result,
        # error of a random-k selection of the same size, the (n-k)/n * ||x|| bound, ||x||, std(x)
        with torch.no_grad():
            n = acc.numel()
            rk = torch.randperm(n, device=acc.device)[:k]
            randk = torch.zeros_like(acc)
            randk[rk] = acc[rk]
            xnorm = float(acc.norm())
            self._profiling_norms.append((float((acc - out).norm()), float((acc - randk).norm()),
                                          1.0 * (n - k) / n * xnorm, xnorm, float(acc.std())))
        if self.writer is not None and hasattr(self.writer, "add_scalars"):
            self.writer.add_scalars("profiling_norm/" + name, {k2: v for k2, v in rec.items() if isinstance(v, (int, float))},
                                    len(self.profile_records))
        return out

    # ------------------------------------------------------------------ functional form
    def run(self, flat_tensor: torch.Tensor, name: str = "flat") -> torch.Tensor:
        """Reduce one flat fp32 tensor in place and return it (``BERT/bert/allreducer.py:347``)."""
        assert flat_tensor.dim() == 1 and flat_tensor.dtype == torch.float32
        if name not in self._engines and name not in self._dist_states and self._use_cuda(flat_tensor.device):
            from .gpu_engine import CudaBucketEngine
            self._engines[name] = CudaBucketEngine(flat_tensor.numel(), self.cfg, self.world, name=name)
        return self.reduce_bucket(name, flat_tensor)

    # ------------------------------------------------------------------ reference-compatible odds and ends
    def add_tensor(self, name: str, tensor: torch.Tensor):
        return name

    def get_result(self, name: str):
        raise RuntimeError("results are written in place into the gradient bucket")

    def stop(self) -> None:
        self._running = False

    def stats(self, name: Optional[str] = None) -> Dict:
        out = {}
        for nm, eng in self._engines.items():
            out[nm] = eng.stats()
        for nm, st in self._dist_states.items():
            out[nm] = {"counter": st.counter, "local_thr": st.local_thr, "global_thr": st.global_thr,
                       "local_count": st.last_local_count, "global_count": st.last_global_count,
                       "volume_elems": st.last_volume_elems, "mode": st.last_mode,
                       "edges": st.region_offsets + [st.numel]}
        return out if name is None else out[name]

    def enable_loss_scaling(self) -> None:
        for eng in self._engines.values():
            eng.enable_loss_scaling()

    def fault_ptr(self, name: str) -> int:
        """Device address of the bucket's fault word (the fused optimizer kernels skip the update when it is set)."""
        eng = self._engines.get(name)
        return int(eng.fault_ptr) if eng is not None else 0

    def poll_faults(self) -> None:
        """Called at every optimizer step: reads the pinned host mirrors of the device fault words (no sync).  A fault
        means a peer did not reach a handshake in time; the partial reduction was NOT applied (the update kernels skipped
        it).  With an ``err_callback`` the replicas are re-synchronised and training continues, otherwise
        ``PeerTimeoutError`` is raised."""
        if not self._engines:
            return
        if _capturing():
            return
        for eng in self._engines.values():
            if eng.poll_fault():
                self.check_faults()
                return

    def trace(self) -> Dict[str, list]:
        return {nm: eng.trace() for nm, eng in self._engines.items()}

    def resync_hooks(self) -> list:
        return getattr(self, "_resync_hooks", [])

    def add_resync_hook(self, fn) -> None:
        """``fn()`` is called (collectively) after a fault was handled through ``err_callback``: the optimizer registers a
        parameter re-broadcast here."""
        self._resync_hooks = self.resync_hooks() + [fn]

    def check_faults(self) -> None:
        """Failure detection (SURVEY 5.3): surfaces device-side peer timeouts.  If an ``err_callback`` was given
        (``DistributedOptimizer(err_handler=...)``) it is invoked as ``cb(new_num_workers, new_rank)`` with the
        current world (the caller decides how to shrink); otherwise ``PeerTimeoutError`` propagates."""
        for eng in self._engines.values():
            try:
                eng.check_fault()
            except RuntimeError:
                if self.err_callback is None:
                    raise
                # recovery path: tell the application, then bring every replica back to a common state -- the residual /
                # thresholds of the faulted call are dropped, parameters re-broadcast (resync hooks), flags cleared
                self.err_callback(self.world.size, self.world.rank)
                for e2 in self._engines.values():
                    e2.reset_sparse_state()
                    e2.clear_fault()
                for fn in self.resync_hooks():
                    fn()
                return

    def state_dict(self) -> Dict:
        sd = {"train_epoch": self.train_epoch, "buckets": {}}
        for nm, eng in self._engines.items():
            sd["buckets"][nm] = eng.state_dict()
        for nm, st in self._dist_states.items():
            sd["buckets"][nm] = st.state_dict()
        return sd

    def load_state_dict(self, sd: Dict) -> None:
        self.train_epoch = sd.get("train_epoch", 0)
        for nm, b in sd.get("buckets", {}).items():
            if nm in self._engines:
                self._engines[nm].load_state_dict(b)
            elif nm in self._dist_states:
                dev = self._dist_states[nm].residual.device if self._dist_states[nm].residual is not None else None
                self._dist_states[nm].load_state_dict(b, dev)
            else:
                import warnings
                warnings.warn("checkpoint holds sparse state for bucket %r which is not registered (yet): ignored" % nm)

    def close(self) -> None:
        for eng in self._engines.values():
            eng.close()
        self._engines.clear()


# free functions of the reference module (VGG/allreducer.py:34,76,175) -------------------------------
def dense_allreduce(tensor: torch.Tensor, world: Optional[World] = None) -> torch.Tensor:
    return algorithms.dense_allreduce(tensor, world or _world())


def topk_sparse_allreduce(tensor: torch.Tensor, density: float, world: Optional[World] = None, state=None):
    w = world or _world()
    st = state or SparseState(tensor.numel(), w.size)
    return algorithms.topka_allreduce(tensor, st, OkTopkConfig(density=density), w, density)


def gtopk_sparse_allreduce(tensor: torch.Tensor, density: float, world: Optional[World] = None, state=None):
    w = world or _world()
    st = state or SparseState(tensor.numel(), w.size)
    return algorithms.gtopk_allreduce(tensor, st, OkTopkConfig(density=density), w, density)
