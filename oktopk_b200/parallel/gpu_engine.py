"""The CUDA engine: one ``CudaBucketEngine`` per gradient bucket drives the fused sm_90a kernels.

Host-side role is *scheduling only*: it knows the iteration counter (which iterations recompute
exact thresholds / re-partition regions, SURVEY 3.3) and enqueues ONE persistent cooperative
kernel per bucket per step on the communication stream.  Thresholds, region edges, slot cursors,
flag epochs and statistics are device resident; there is no host synchronisation, no NCCL call
and no count handshake on the host (the reference needs >= 3P+6 staging copies and 4-6 blocking
MPI calls per step, SURVEY 3.3 notes).

Memory per bucket (one IPC allocation, mapped by every peer):
    [ flat fp32 gradient bucket | mailboxes + send slots + gather slots | dense-allreduce flags ]
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional

import torch

from ..config import OkTopkConfig
from ..ops import ext
from .state import CallPlan, SparseState, plan_call, uniform_boundaries, offsets_of
from .symm import SymmBlock, make_symm_block
from .world import World

RES_OKTOPK, RES_LOCAL_GT, RES_LOCAL_GE = 0, 1, 2
GLB_THRESHOLD, GLB_EXACT_TOPK, GLB_ALL_NONZERO = 0, 1, 2
GS_THRESHOLD_REUSE, GS_GAUSSIAN, GS_EXACT_TOPK = 0, 1, 2

_CLASSIC_RESIDUAL = {"topkSA", "topkDSA", "gaussiankSA"}   # residual zeroed at selection: the gather must be lossless


def _round_up(x: int, m: int) -> int:
    return (int(x) + m - 1) // m * m


class PeerTimeoutError(RuntimeError):
    """A rank of the peer group did not reach a handshake in time (device-side failure detection)."""


class CudaBucketEngine:
    def __init__(self, numel: int, cfg: OkTopkConfig, world: World, name: str = "bucket",
                 max_density: Optional[float] = None, dense_grid: int = 0):
        self.C = ext.require()
        C = self.C
        self.cfg = cfg
        self.world = world
        self.name = name
        self.P = world.size
        self.rank = world.rank
        if self.P > C.MAXP:
            raise ValueError("world size %d exceeds OKT_MAXP=%d" % (self.P, C.MAXP))
        self.n = int(numel)
        self.device = torch.device("cuda", torch.cuda.current_device())
        dmax = max_density if max_density is not None else cfg.density
        if cfg.dynamic_densities:
            dmax = max(dmax, max(cfg.dynamic_densities))
        kmax = max(int(self.n * dmax), 1)
        self.kmax = kmax
        chunk = C.CHUNK
        # Slot capacities (config.py: slot_factor / gather_factor).  Default = LOSSLESS layout: the send slot of a
        # destination is as long as its region, the gather slot as long as the bucket -- nothing selected can be dropped,
        # however stale the threshold (HBM is 80 GB: 24 B/element of symmetric memory per bucket).  Bounded slots rely on
        # the in-kernel overflow policy (raise threshold + redo the pack; classic-residual schemes keep unsent entries).
        nmax = _round_up(self.n, chunk)
        if cfg.slot_factor > 0:
            self.cap = min(nmax, _round_up(max(cfg.slot_factor * kmax / self.P, chunk), chunk)) + chunk
        else:
            self.cap = 0                                   # lossless layout (oktopk.cuh)
        if cfg.gather_factor > 0 and cfg.compressor not in _CLASSIC_RESIDUAL:
            self.gcap = min(nmax, _round_up(max(cfg.gather_factor * kmax / self.P, 2 * kmax, chunk), chunk)) + chunk
        else:
            self.gcap = nmax + chunk
        info = C.layout_info(self.P, self.n, self.cap, self.gcap)
        self.layout = info
        self.grid = C.max_coop_grid(self.device.index)
        self.gather_grid = C.gather_max_coop_grid(self.device.index)
        self.tree_grid = C.gtopk_max_coop_grid(self.device.index)
        if cfg.comm_ctas > 0:
            self.grid = min(self.grid, cfg.comm_ctas)
            self.gather_grid = min(self.gather_grid, cfg.comm_ctas)
            self.tree_grid = min(self.tree_grid, cfg.comm_ctas)
        # dense two-shot kernel: one CTA per SM, cooperative launch (its per-CTA cross-GPU barrier needs co-residency)
        sms = torch.cuda.get_device_properties(self.device).multi_processor_count
        self.dense_grid = dense_grid or (min(sms, cfg.comm_ctas) if cfg.comm_ctas > 0 else sms)
        # ---- one symmetric allocation: [grad | comm block | dense flags] -------------------
        self.grad_bytes = _round_up(self.n * 4, 4096)
        self.comm_off = self.grad_bytes
        self.flags_off = self.comm_off + _round_up(info["total"], 4096)
        flags_bytes = 8 * 2 * self.dense_grid * C.MAXP
        self.block = make_symm_block(self.flags_off + _round_up(flags_bytes, 4096), world, cfg.nvls)
        self.grad = self.block.tensor(0, self.n, "float32")
        self.peer_comm = [p + self.comm_off for p in self.block.ptrs]
        self.peer_grad = [p for p in self.block.ptrs]
        self.peer_flags = [p + self.flags_off for p in self.block.ptrs]
        self.mc_grad = int(getattr(self.block, "mc_ptr", 0) or 0)      # multicast mapping of the bucket (NVLS), 0 if none
        # ---- local device state -------------------------------------------------------------
        self.state_ptr = C.dev_alloc_zero(C.state_bytes())
        self.fault_ptr = C.fault_ptr(self.state_ptr)
        self.host_flag, self.host_flag_dev = C.host_flag_alloc()      # fault code mirrored to pinned host memory
        self.dense_epoch_ptr = C.dev_alloc_zero(8 * self.dense_grid)
        self.scale_sync_ptr = 0                  # loss scaling: check ticket, epoch, bucket verdict (enable_loss_scaling)
        self.residual = torch.zeros(self.n, dtype=torch.float32, device=self.device)
        # first-touch candidate list of the reduce phase: at most one entry per distinct index of my region
        # (also: pre-filtered candidates of the exact-threshold radix select, union lists of TopkA2 / gTopk)
        if self.cap == 0:
            self.ccap = _round_up(self.n, 32)
        else:
            self.ccap = int(min(_round_up(self.n, 32), max(self.P * self.cap, 32 * kmax + chunk)))
        self.cand = torch.zeros(self.ccap, dtype=torch.int32, device=self.device)
        self._bitmap: Optional[torch.Tensor] = None          # TopkA2 / gTopk: exact first-touch detection
        self._sel: Optional[tuple] = None                    # gTopk: private copy of my picks for the put-back
        self.host = SparseState(self.n, self.P)          # counter + (lazily refreshed) mirrors
        self._write_edges(self.host.region_offsets + [self.n])
        self.last_mode = ""
        self._res_clean = False                  # True while the residual is known to be all-zero (dense-switch calls)
        self._skip = 0                           # bucket verdict address of the running call (loss scaling), 0 = off
        self.early_pack = bool(cfg.early_pack) and os.environ.get("OKTOPK_EARLY_PACK", "1") != "0"

    # ------------------------------------------------------------------ helpers
    def _stream(self, stream: Optional[torch.cuda.Stream]) -> int:
        return (stream or torch.cuda.current_stream()).cuda_stream

    def _write_edges(self, edges: List[int], local_thr: float = 0.0, global_thr: float = 0.0) -> None:
        self.C.write_state(self.state_ptr, float(local_thr), float(global_thr), [int(e) for e in edges],
                           torch.cuda.current_stream().cuda_stream)

    def k_now(self, density: Optional[float] = None) -> int:
        d = self.cfg.density if density is None else density
        return max(int(self.n * d), 1)

    # ------------------------------------------------------------------ the step
    def _plan(self, compressor: str, density: Optional[float]) -> CallPlan:
        return plan_call(self.cfg, compressor, self.host.counter, density, self.P)

    def reads_sources(self, compressor: str, density: Optional[float] = None) -> bool:
        """True if the next ``reduce`` call can read the gradient from its source tensors (``reduce(srcs=...)``) instead of
        the bucket: an Ok-Topk call of the fused kernel, whose pack pass then reads every source once and leaves the bucket
        alone.  The bucket must be all-zero when such a call starts."""
        return compressor == "oktopk" and self._plan(compressor, density).kind == "fused"

    def packs_early(self, compressor: str, density: Optional[float] = None) -> bool:
        """True if the next ``reduce`` call may be preceded by ``pack_segment`` launches (parallel/early_pack.py): an
        Ok-Topk threshold-reuse call of the fused kernel in the lossless slot layout.  The caller also makes sure that it
        reads the gradient from its sources and that loss scaling is off."""
        if not (self.early_pack and compressor == "oktopk" and self.cap == 0 and self.cfg.fused):
            return False
        plan = self._plan(compressor, density)
        return plan.kind == "fused" and not plan.exact_local and not plan.repartition

    def pack_segment(self, compressor: str, ranges, srcs: tuple, density: Optional[float] = None,
                     stream: Optional[torch.cuda.Stream] = None) -> None:
        """Pack the bucket ranges ``ranges = [(lo, hi), ...]`` of the next call now, from the gradient sources ``srcs``
        that cover them (only where ``packs_early``).  Enqueue it behind the previous call and ahead of the next one on
        the same stream."""
        self._fused(compressor, self._plan(compressor, density), density, self._stream(stream), self.grad, srcs,
                    pack_ranges=list(ranges), segment=True)

    def enable_loss_scaling(self) -> None:
        """Allocate the device words of ``unscale_check`` (before any graph capture; a no-op when already done)."""
        if not self.scale_sync_ptr:
            self.scale_sync_ptr = self.C.dev_alloc_zero(self.C.SCALE_SYNC_BYTES)

    @property
    def verdict_ptr(self) -> int:
        """Device address of the bucket verdict that ``unscale_check`` writes and ``reduce(skip=...)`` reads."""
        self.enable_loss_scaling()
        return self.scale_sync_ptr + self.C.VERDICT_OFFSET

    def unscale_check(self, loss_scale_ptr: int, stream: Optional[torch.cuda.Stream] = None,
                      srcs: Optional[tuple] = None) -> None:
        """Loss scaling, before ``reduce(skip=self.verdict_ptr)``: multiply the gradient (the ``srcs`` tensors, else the
        bucket) by the optimizer's inv_scale in place and agree with every peer on the bucket verdict (set if any rank
        saw a non-finite value; ORed into the step verdict)."""
        self.enable_loss_scaling()
        if srcs is not None and len(srcs[0]):
            ptrs, lens = list(srcs[0]), list(srcs[2])
        else:                                      # the landed bucket (or, with no gradient at all, the all-zero one)
            ptrs, lens = [self.grad.data_ptr()], [self.n]
        self.C.unscale_check(ptrs, lens, loss_scale_ptr, self.scale_sync_ptr, self.state_ptr, self.host_flag_dev,
                             self.peer_comm, self.layout["scale_mbox"], self.rank, float(self.cfg.peer_timeout_s),
                             self._stream(stream))

    def reduce(self, compressor: str, density: Optional[float] = None,
               stream: Optional[torch.cuda.Stream] = None, g: Optional[torch.Tensor] = None,
               srcs: Optional[tuple] = None, skip: int = 0, pack_ranges: Optional[list] = None) -> torch.Tensor:
        """Allreduce this bucket in place (``self.grad`` unless an external ``g`` is given).

        ``srcs = (pointers, offsets, lengths)``: the gradient is not in the bucket but in these fp32 tensors, at these
        element offsets of the bucket (Ok-Topk only, see ``reads_sources``); the result is written into the bucket.
        ``skip``: device address of the bucket verdict of loss scaling (0 = off); when set the kernels return at entry.
        ``pack_ranges``: after ``pack_segment`` launches, the element ranges they left for this call to pack."""
        ext_g = g is not None and g.data_ptr() != self.grad.data_ptr()
        plan = self._plan(compressor, density)
        if srcs is not None and (ext_g or compressor != "oktopk" or plan.kind != "fused"):
            raise ValueError("gradient sources are only read by an Ok-Topk call on the engine's own bucket")
        s = self._stream(stream)
        self._skip = int(skip)
        out = g if ext_g else self.grad
        if plan.kind in ("dense", "dense_switch"):
            if ext_g:
                self.grad.copy_(g)
            if plan.kind == "dense_switch":
                # reduce the error-compensated gradient densely (nothing is left behind, so the residual is cleared)
                if self._skip:                     # under loss scaling a skipped call keeps its residual: always carry
                    self.C.carry_residual(self.grad.data_ptr(), self.residual.data_ptr(), self.n, self._skip, s)
                elif not self._res_clean:          # a dense call leaves nothing behind: after the first switched call
                    self.grad.add_(self.residual)  # the residual is known to be all-zero and the carry-over is skipped
                    self.residual.zero_()
                    self._res_clean = True
            self._dense(s)
            if ext_g:
                g.copy_(self.grad)
            self.last_mode = "dense" if plan.kind == "dense" else "dense(auto)"
        else:
            self._res_clean = False
            if plan.kind == "fused":
                self._fused(compressor, plan, density, s, out, srcs, pack_ranges)
            elif plan.kind == "gather":
                self._gather(compressor, plan, density, s, out)
            else:
                self._tree(compressor, density, s, out)
        self.host.counter += 1
        return out

    def _dense(self, s: int) -> None:
        if self.P == 1:
            return
        self.C.dense_run(self.peer_grad, self.peer_flags, self.dense_epoch_ptr, self.n, self.rank,
                         self.dense_grid, s, self.state_ptr, float(self.cfg.peer_timeout_s), self.mc_grad,
                         self.host_flag_dev, self._skip)

    def _fused(self, compressor: str, plan: CallPlan, density: Optional[float], s: int, g: torch.Tensor,
               srcs: Optional[tuple] = None, pack_ranges: Optional[list] = None, segment: bool = False) -> None:
        cfg = self.cfg
        k = self.k_now(density)
        o: Dict = {"pull_tma": 1 if cfg.pull_mode == "tma" else 0, "deterministic": int(cfg.deterministic),
                   "split_phases": 0 if cfg.fused else 1, "timeout_s": float(cfg.peer_timeout_s),
                   "cand": self.cand.data_ptr(), "ccap": self.ccap, "host_fault": self.host_flag_dev,
                   "max_redo": int(cfg.max_redo), "redo_factor": float(cfg.redo_factor),
                   # global selection: candidate list when few entries land in a region (O(#entries) with atomics that
                   # return), region scan when a large fraction of it is non-zero (O(n/P) streaming)
                   "cand_mode": int(cfg.gselect_mode == "list" or (cfg.gselect_mode == "auto" and k * 200 <= self.n))}
        if compressor == "oktopk":
            o.update(
                exact_local=int(plan.exact_local),
                repartition=int(plan.repartition),
                residual_mode=RES_OKTOPK,
                global_mode=GLB_EXACT_TOPK if plan.exact_global else GLB_THRESHOLD,
                guard_loops=cfg.overselect_guard_loops,
                guard_limit=cfg.overselect_guard_num * k // cfg.overselect_guard_den,
                guard_factor=cfg.overselect_guard_factor,
                cap_limit=int(cfg.overselect_cap * k) if cfg.overselect_cap > 0 else 0,
                cap_rungs=int(cfg.overselect_cap_rungs), cap_factor=float(cfg.overselect_cap_factor),
                l_low_cnt=cfg.local_adapt_low * k, l_high_cnt=cfg.local_adapt_high * k, l_factor=cfg.local_adapt_factor,
                g_low_cnt=cfg.global_adapt_low * k, g_high_cnt=cfg.global_adapt_high * k,
                g_inc=cfg.global_adapt_inc, g_dec=cfg.global_adapt_dec,
            )
        else:  # TopkDSA / gaussiankSA: exact threshold every call, uniform regions, all non-zeros gathered
            o.update(exact_local=1, repartition=0,
                     residual_mode=RES_LOCAL_GT if compressor == "gaussiankSA" else RES_LOCAL_GE,
                     global_mode=GLB_ALL_NONZERO, guard_loops=0, guard_limit=0)
            # dynamic dense fallback (VGG/allreducer.py:1311-1353): when the reduced regions hold >= frac*n non-zeros
            # the kernel's final phase copies the peers' regions instead of their (idx,val) lists.  Needs the bucket to
            # be the symmetric one (peers read it directly).
            if compressor in ("topkDSA", "topkSA") and g.data_ptr() == self.grad.data_ptr() and self.P > 1 \
                    and cfg.dsa_dense_fallback_frac > 0:
                o["dense_nnz_limit"] = max(int(self.n * cfg.dsa_dense_fallback_frac), 1)
                o["peer_g"] = self.peer_grad
        if srcs is not None:
            o["srcs"] = srcs
        if self._skip:
            o["skip"] = self._skip
        if pack_ranges is not None:
            o["pack_ranges"] = [(int(a), int(b)) for a, b in pack_ranges]
            o["segment"] = int(segment)
            o["seg_ctas"] = int(cfg.early_pack_ctas)
        self.C.oktopk_run(g.data_ptr(), self.residual.data_ptr(), self.state_ptr, self.peer_comm, self.n,
                          self.rank, k, self.cap, self.gcap, o, self.grid, s)
        if not segment:
            self.last_mode = compressor

    def _gather(self, compressor: str, plan: CallPlan, density: Optional[float], s: int, g: torch.Tensor) -> None:
        cfg = self.cfg
        d = cfg.density if density is None else density
        k = self.k_now(density)
        o: Dict = {"density": d, "pull_tma": 1 if cfg.pull_mode == "tma" else 0, "timeout_s": float(cfg.peer_timeout_s),
                   "host_fault": self.host_flag_dev}
        if cfg.norm_clip is not None and compressor in ("topkA", "topkA2"):       # VGG/allreducer.py:1372-1379
            o["clip_max_norm"] = float((1.0 / self.P) ** 0.5 * cfg.norm_clip)
        if compressor in ("topkA", "topkA2"):
            o["select_mode"] = GS_EXACT_TOPK
            if compressor == "topkA2":
                o.update(reselect=1, bitmap=self._bitmap_ptr(), cand=self.cand.data_ptr(), ccap=self.ccap)
        elif compressor == "topkAopt":
            o["select_mode"] = GS_THRESHOLD_REUSE
            o["exact_now"] = int(plan.exact_local)
        else:
            o["select_mode"] = GS_GAUSSIAN
            o["gauss_mode"] = {"vgg": 0, "lstm": 1, "bert": 2}[cfg.gaussian_mode]
            o["gauss_loops"] = cfg.gaussian_loops
            o["gauss_factor"] = cfg.gaussian_factor
        if self._skip:
            o["skip"] = self._skip
        self.C.gather_run(g.data_ptr(), self.residual.data_ptr(), self.state_ptr, self.peer_comm, self.n,
                          self.rank, k, self.cap, self.gcap, o, self.gather_grid, s)
        self.last_mode = compressor

    def _bitmap_ptr(self) -> int:
        if self._bitmap is None:
            self._bitmap = torch.zeros((self.n + 31) // 32 + 32, dtype=torch.int32, device=self.device)
        return self._bitmap.data_ptr()

    def _tree(self, compressor: str, density: Optional[float], s: int, g: torch.Tensor) -> None:
        """gTopk on the native tree kernel (csrc/gtopk.cu)."""
        cfg = self.cfg
        k = self.k_now(density)
        if self._sel is None:
            selcap = int(min(_round_up(self.n, 32), 2 * self.kmax + self.C.CHUNK))
            self._sel = (torch.zeros(selcap, dtype=torch.int32, device=self.device),
                         torch.zeros(selcap, dtype=torch.float32, device=self.device), selcap)
        o: Dict = {"pull_tma": 1 if cfg.pull_mode == "tma" else 0, "timeout_s": float(cfg.peer_timeout_s),
                   "host_fault": self.host_flag_dev, "bitmap": self._bitmap_ptr(), "cand": self.cand.data_ptr(),
                   "ccap": self.ccap, "sel_idx": self._sel[0].data_ptr(), "sel_val": self._sel[1].data_ptr(),
                   "selcap": self._sel[2]}
        if cfg.norm_clip is not None:
            o["clip_max_norm"] = float((1.0 / self.P) ** 0.5 * cfg.norm_clip)
        if self._skip:
            o["skip"] = self._skip
        self.C.gtopk_run(g.data_ptr(), self.residual.data_ptr(), self.state_ptr, self.peer_comm, self.n,
                         self.rank, k, self.cap, self.gcap, o, self.tree_grid, s)
        self.last_mode = compressor

    # ------------------------------------------------------------------ observability / checkpoint
    def stats(self) -> Dict:
        """Synchronous read of the device-resident state (never called on the hot path)."""
        d = self.C.read_state(self.state_ptr, self.P, torch.cuda.current_stream().cuda_stream)
        d["counter"] = self.host.counter
        d["mode"] = self.last_mode
        d["cap"], d["gcap"], d["grid"] = self.cap, self.gcap, self.grid
        d["lossless"] = self.cap == 0
        d["nvls"] = bool(self.mc_grad)
        # scalars moved by this rank in the last call (idx + val per entry), cf. the 6k(P-1)/P bound
        d["volume_elems"] = 2 * (d["recv_total"] + d["gather_total"])
        return d

    def trace(self) -> List[Dict]:
        """The device-side per-call history ring (newest TRACE_LEN fused calls), oldest first.  Synchronous."""
        recs = list(self.C.read_trace(self.state_ptr, torch.cuda.current_stream().cuda_stream))
        recs.sort(key=lambda r: r["epoch"])
        return recs

    def poll_fault(self) -> int:
        """The fault code mirrored into pinned host memory by the kernels: a plain host read, no synchronisation,
        cheap enough for every step()."""
        return int(self.C.host_flag_read(self.host_flag))

    def check_fault(self) -> None:
        """Raise if a bounded cross-GPU wait timed out inside a kernel (a peer died or wedged).  Synchronous."""
        code = int(self.stats().get("fault", 0))
        if code:
            names = {1: "reduce-scatter mailbox", 2: "allgather mailbox", 3: "region-cut mailbox", 4: "dense barrier",
                     5: "gTopk tree mailbox", 6: "dense-fallback done flags",
                     7: "loss-scale verdict mailbox"}
            raise PeerTimeoutError("bucket %s: peer wait timed out in the %s (fault %d, timeout %.1fs)"
                                   % (self.name, names.get(code, "?"), code, self.cfg.peer_timeout_s))

    def clear_fault(self) -> None:
        self.C.clear_fault(self.state_ptr, torch.cuda.current_stream().cuda_stream)
        self.C.host_flag_clear(self.host_flag)

    def reset_sparse_state(self) -> None:
        """After a fault: drop the (possibly half-consumed) residual and thresholds, restore uniform regions, so that
        all replicas restart the sparse scheme from the same state (the next call recomputes exact thresholds).  The
        bucket is cleared too: the update that would have cleared it was skipped, and a call that reads the gradient from
        its sources expects an all-zero bucket."""
        self.residual.zero_()
        self.grad.zero_()
        self.host.counter = self.cfg.warmup_iters if self.host.counter >= self.cfg.warmup_iters else self.host.counter
        self._write_edges(offsets_of(uniform_boundaries(self.n, self.P)) + [self.n], 0.0, 0.0)

    def state_dict(self) -> Dict:
        d = self.stats()
        return {"numel": self.n, "world": self.P, "counter": self.host.counter, "local_thr": d["local_thr"],
                "global_thr": d["global_thr"], "boundaries": [d["edges"][i + 1] - d["edges"][i] for i in range(self.P)],
                "region_offsets": d["edges"][:-1], "residual": self.residual.detach().cpu().clone()}

    def load_state_dict(self, sd: Dict) -> None:
        assert sd["numel"] == self.n
        self.host.counter = int(sd["counter"])
        if sd.get("residual") is not None:
            self.residual.copy_(sd["residual"].to(self.device))
            self._res_clean = False
        if sd["world"] == self.P:
            edges = list(sd["region_offsets"]) + [self.n]
        else:
            edges = offsets_of(uniform_boundaries(self.n, self.P)) + [self.n]
        self._write_edges(edges, sd["local_thr"], sd["global_thr"])

    def close(self) -> None:
        """Release the symmetric block (collective: every rank must call it) and the local device state."""
        if getattr(self, "_closed", False):
            return
        self._closed = True
        self.block.close()                       # synchronises the device and the peer group first
        try:
            self.C.host_flag_free(self.host_flag)
        except Exception:  # noqa: BLE001
            pass
        self.host_flag = 0
        for attr in ("state_ptr", "dense_epoch_ptr", "scale_sync_ptr"):
            ptr = getattr(self, attr, 0)
            if ptr:
                try:
                    self.C.dev_free(ptr)
                except Exception:  # noqa: BLE001 - teardown must not raise
                    pass
                setattr(self, attr, 0)
