"""Single-process oracle of every sparse-allreduce scheme.

Simulates P ranks over a list of P fp32 tensors with plain torch ops and no communication,
encoding SURVEY 3.3 / Appendix B step by step.  It is the ground truth that the
torch.distributed path (``algorithms.py``) and the fused sm_90a kernels are tested against
(the reference has no such thing: its only correctness signal is the convergence curve,
SURVEY 4).

All functions take ``grads`` (list of P 1-D tensors, rank-major), ``states`` (list of P
``SparseState``) and an ``OkTopkConfig``; they return the list of P results (what each rank's
gradient bucket holds afterwards) and update the states (counter NOT incremented: the engine
does that).
"""
from __future__ import annotations

from typing import List, Sequence, Tuple

import torch

from ..compression import gaussian_correct_threshold, gen_threshold_from_normal_distribution
from ..config import OkTopkConfig
from .state import SparseState, offsets_of, plan_call, uniform_boundaries


# --------------------------------------------------------------------------- helpers
import numpy as _np


def f32_mul(a: float, b: float) -> float:
    """Thresholds live in fp32 on the device: mirror the kernel's arithmetic exactly."""
    return float(_np.float32(a) * _np.float32(b))


def f32_div(a: float, b: float) -> float:
    return float(_np.float32(a) / _np.float32(b))


def kth_largest_abs(x: torch.Tensor, k: int) -> float:
    k = max(min(k, x.numel()), 1)
    return float(torch.topk(x.abs().view(-1), k=k).values[-1])


def ftz(x: torch.Tensor) -> torch.Tensor:
    """Subnormals flushed to zero.  The reduce phase of the fused kernel sums with fp32 global atomics, which flush
    subnormal inputs and results to zero (PTX ``atom/red.add.f32``): a selected entry whose value or sum is subnormal
    reaches the owner as 0, is not gathered, and stays in the sender's residual."""
    return torch.where(x.abs() < torch.finfo(x.dtype).tiny, torch.zeros_like(x), x)


def topk_tie_inclusive(x: torch.Tensor, k: int) -> torch.Tensor:
    """Ascending indices of the exact top-k by magnitude, every element tied at the k-th magnitude included and zeros
    excluded (``|x| >= kth && |x| > 0``): more than k indices on a tie, fewer when x has fewer than k non-zeros.  The
    local picks of TopkA / TopkA2 / gTopk and their merge rounds select this way on the device; ``torch.topk`` returns
    exactly k but leaves unspecified which tied elements, so it cannot be the reference on tied data."""
    ax = x.abs()
    return ((ax >= kth_largest_abs(x, k)) & (ax > 0)).nonzero().view(-1)


def guard_threshold(absx: torch.Tensor, thr: float, k: int, cfg: OkTopkConfig) -> float:
    """``add2residual`` over-selection guard (``VGG/compression.py:392-404``) + the optional hard cap
    (``OkTopkConfig.overselect_cap``): one geometric ladder ``T_0 = thr, T_j = T_{j-1} * f`` (``f`` = guard factor on the
    first ``guard_loops`` rungs, cap factor on the coarse rungs after them), climbed while the count is above the guard
    limit (fine rungs only) and then while it is above the cap.  Mirrors ``ladder_pick`` in ``csrc/devlib.cuh`` with the
    same fp32 arithmetic."""
    n_fine = min(max(cfg.overselect_guard_loops, 0), 15)
    cap_limit = int(cfg.overselect_cap * k) if cfg.overselect_cap > 0 else 0
    n_coarse = min(cfg.overselect_cap_rungs, 63 - n_fine) if cap_limit > 0 else 0
    n_total = 1 + n_fine + n_coarse
    if n_total == 1:
        return thr
    limit = cfg.overselect_guard_num * k // cfg.overselect_guard_den

    def count(t: float) -> int:
        return int((absx > t).sum())
    j, t = 0, thr
    while j < n_fine and count(t) > limit:
        j += 1
        t = f32_mul(t, cfg.overselect_guard_factor)
    if cap_limit > 0:
        while j < n_total - 1 and count(t) > cap_limit:
            j += 1
            t = f32_mul(t, cfg.overselect_guard_factor if j <= n_fine else cfg.overselect_cap_factor)
    return t


def quantile_cuts(sel_idx: torch.Tensor, P: int, n: int) -> List[int]:
    """Local cut points ``I[j*(|I|//P)]`` (``VGG/allreducer.py:632-636``); uniform if nothing selected."""
    m = sel_idx.numel()
    if m == 0:
        return [(n // P) * j for j in range(1, P)]
    chunk = m // P
    return [int(sel_idx[chunk * j]) for j in range(1, P)]


def boundaries_from_cuts(avg_cuts: Sequence[int], n: int) -> Tuple[List[int], List[int]]:
    """``VGG/allreducer.py:641-654`` with monotonicity enforced (reference asserts, A.4-5)."""
    cuts, prev = [], 0
    for c in avg_cuts:
        c = min(max(int(c), prev), n)
        cuts.append(c)
        prev = c
    edges = [0] + cuts + [n]
    b = [edges[i + 1] - edges[i] for i in range(len(edges) - 1)]
    return b, edges[:-1]


def adapt_local(thr: float, count: int, k: int, cfg: OkTopkConfig) -> float:
    if count < cfg.local_adapt_low * k:
        return f32_div(thr, cfg.local_adapt_factor)
    if count > cfg.local_adapt_high * k:
        return f32_mul(thr, cfg.local_adapt_factor)
    return thr


def adapt_global(thr: float, total: int, k: int, cfg: OkTopkConfig) -> float:
    if total < cfg.global_adapt_low * k:
        return f32_div(thr, cfg.global_adapt_inc)
    if total > cfg.global_adapt_high * k:
        return f32_mul(thr, cfg.global_adapt_dec)
    return thr


def _k(n: int, density: float) -> int:
    return max(int(n * density), 1)


# --------------------------------------------------------------------------- dense
def dense_oracle(grads: List[torch.Tensor], states=None, cfg=None) -> List[torch.Tensor]:
    P = len(grads)
    s = torch.stack(grads).sum(0) / P
    for g in grads:
        g.copy_(s)
    return grads


# --------------------------------------------------------------------------- Ok-Topk
def oktopk_oracle(grads: List[torch.Tensor], states: List[SparseState], cfg: OkTopkConfig,
                  density: float = None) -> List[torch.Tensor]:
    """SURVEY 3.3 steps (1)-(7), with the exact-threshold and re-partition iterations of ``plan_call``."""
    P = len(grads)
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    plan = plan_call(cfg, "oktopk", states[0].counter, density, P)

    accs, thrs = [], []
    # (1) error feedback + local threshold; a carried threshold of 0 (the last exact call saw fewer than k non-zeros) is
    #     recomputed exactly: at 0 every non-zero would be selected and no ladder rung (0 * f) could cap the volume
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        acc = grads[r] + res
        res.copy_(acc)
        if plan.exact_local or st.local_thr == 0.0:
            thr = kth_largest_abs(acc, k)
        else:
            thr = guard_threshold(acc.abs(), st.local_thr, k, cfg)
        st.local_thr = thr
        accs.append(acc)
        thrs.append(thr)

    # (2) balanced region re-partition
    if plan.repartition:
        cuts = torch.zeros(P - 1, dtype=torch.int64)
        for r in range(P):
            sel = (accs[r].abs() > thrs[r]).nonzero().view(-1)
            cuts += torch.tensor(quantile_cuts(sel, P, n), dtype=torch.int64)
        avg = (cuts // P).tolist()
        b, off = boundaries_from_cuts(avg, n)
        for st in states:
            st.boundaries, st.region_offsets = list(b), list(off)
    b, off = states[0].boundaries, states[0].region_offsets
    edges = off + [n]

    # (3) select by the local threshold, (4) reduce every region on its owner
    reduced = torch.zeros(n, dtype=grads[0].dtype, device=grads[0].device)  # region r lives at off[r]..
    local_masks = []
    vol = [0] * P
    for r in range(P):
        mask = accs[r].abs() > thrs[r]
        local_masks.append(mask)
        cnt = int(mask.sum())
        states[r].last_local_count = cnt
        states[r].last_thr_used = thrs[r]
        reduced = ftz(reduced + ftz(torch.where(mask, accs[r], torch.zeros_like(accs[r]))))
        for d in range(P):
            if d != r:
                c = int(mask[edges[d]:edges[d + 1]].sum())
                vol[r] += 2 * c          # sent (idx, val)
                vol[d] += 2 * c          # received
        states[r].local_thr = adapt_local(thrs[r], cnt, k, cfg)

    # (5) global selection
    if plan.exact_global:
        nz = reduced.nonzero().view(-1)
        vals = reduced[nz]
        kk = min(nz.numel(), k)
        if kk > 0:
            gthr = float(torch.topk(vals.abs(), k=kk).values[-1])
            keep = vals.abs() >= gthr          # tie-inclusive exact top-k (see DESIGN.md)
            gidx = nz[keep]
        else:
            gthr, gidx = 0.0, nz
        for st in states:
            st.global_thr = gthr
        cand_per_region = [int((reduced[edges[d]:edges[d + 1]] != 0).sum()) for d in range(P)]
    else:
        gthr = states[0].global_thr
        gmask = reduced.abs() > gthr
        gidx = gmask.nonzero().view(-1)
        T = gidx.numel()
        for st in states:
            st.global_thr = adapt_global(gthr, T, k, cfg)
        cand_per_region = [int(gmask[edges[d]:edges[d + 1]].sum()) for d in range(P)]
    total_c = sum(cand_per_region)
    for r in range(P):
        vol[r] += 2 * (total_c - cand_per_region[r])      # allgatherv receive
        vol[r] += 2 * cand_per_region[r] * (1 if P > 1 else 0)  # my slot leaves once (bus view)
        states[r].last_volume_elems = vol[r]
        states[r].last_global_count = int(gidx.numel())
        states[r].last_mode = "oktopk"

    # (6) result, (7) residual cleared on local ∩ global
    gmask_full = torch.zeros(n, dtype=torch.bool, device=grads[0].device)
    gmask_full[gidx] = True
    result = torch.where(gmask_full, reduced / P, torch.zeros_like(reduced))
    for r in range(P):
        grads[r].copy_(result)
        states[r].residual[gmask_full & local_masks[r]] = 0.0
    return grads


# --------------------------------------------------------------------------- TopkA / TopkA2
def topka_oracle(grads, states, cfg: OkTopkConfig, density=None, reselect: bool = False):
    """Appendix B.1.  ``reselect=True`` is TopkA2 (global top-k of the sum + put-back).  Both selections are
    tie-inclusive (``topk_tie_inclusive``; the re-selection keeps every union entry at or above the k-th magnitude of
    the union, and the whole union when it has at most k entries)."""
    P = len(grads)
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    total = torch.zeros_like(grads[0])
    picked = torch.zeros(n, dtype=torch.bool, device=total.device)
    picks = []
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        g = grads[r]
        if cfg.norm_clip is not None:
            _clip(g, (1.0 / P) ** 0.5 * cfg.norm_clip)
        acc = g + res
        idx = topk_tie_inclusive(acc, k)
        vals = acc[idx]
        res.copy_(acc)
        res[idx] = 0.0
        total[idx] += vals
        picked[idx] = True
        picks.append((idx, vals))
        st.local_thr = kth_largest_abs(acc, k)
        st.last_local_count = int(idx.numel())
        st.last_volume_elems = 2 * int(idx.numel()) * (P - 1) * 2 if P > 1 else 0
        st.last_mode = "topkA2" if reselect else "topkA"
    if reselect:
        U = picked.nonzero().view(-1)
        keep = torch.zeros(n, dtype=torch.bool, device=total.device)
        if U.numel() > k:
            keep[U] = total[U].abs() >= float(torch.topk(total[U].abs(), k=k).values[-1])
        else:
            keep[U] = True
        total = torch.where(keep, total, torch.zeros_like(total))
        for r in range(P):
            idx, vals = picks[r]
            lost = ~keep[idx]
            states[r].residual[idx[lost]] += vals[lost]
    total /= P
    for r in range(P):
        grads[r].copy_(total)
        states[r].last_global_count = int((total != 0).sum())
    return grads


def _clip(g: torch.Tensor, max_norm: float) -> None:
    nrm = float(g.norm())
    if nrm > max_norm and nrm > 0:
        g.mul_(max_norm / nrm)


# --------------------------------------------------------------------------- TopkAopt
def topkaopt_oracle(grads, states, cfg: OkTopkConfig, density=None):
    """B.6: threshold reuse + residual zeroed at selection + allgatherv + scatter-add."""
    P = len(grads)
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    exact = plan_call(cfg, "topkAopt", states[0].counter, density, P).exact_local
    total = torch.zeros_like(grads[0])
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        acc = grads[r] + res
        res.copy_(acc)
        if exact:
            st.local_thr = kth_largest_abs(acc, k)
        mask = acc.abs() > st.local_thr
        res[mask] = 0.0
        total += torch.where(mask, acc, torch.zeros_like(acc))
        st.last_local_count = int(mask.sum())
        st.last_mode = "topkAopt"
    total /= P
    for r in range(P):
        grads[r].copy_(total)
    return grads


# --------------------------------------------------------------------------- gTopk
def gtopk_oracle(grads, states, cfg: OkTopkConfig, density=None):
    """Appendix B.2: tree merge of local top-k lists, re-selecting top-k of each union."""
    P = len(grads)
    assert P & (P - 1) == 0, "gTopk needs a power-of-two world (VGG/allreducer.py:113)"
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    lists, picks = [], []
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        g = grads[r]
        if cfg.norm_clip is not None:
            _clip(g, (1.0 / P) ** 0.5 * cfg.norm_clip)
        acc = g + res
        idx = topk_tie_inclusive(acc, k)
        vals = acc[idx]
        res.copy_(acc)
        res[idx] = 0.0
        lists.append((idx, vals))
        picks.append((idx, vals))
        st.last_local_count = int(idx.numel())
        st.last_mode = "gtopk"
    step = 1
    while step < P:
        for r in range(0, P, 2 * step):
            lists[r] = merge_topk(lists[r], lists[r + step], k, n)
        step *= 2
    fidx, fvals = lists[0]
    out = torch.zeros_like(grads[0])
    out[fidx] = fvals / P
    keep = torch.zeros(n, dtype=torch.bool, device=out.device)
    keep[fidx] = True
    for r in range(P):
        idx, vals = picks[r]
        lost = ~keep[idx]
        states[r].residual[idx[lost]] += vals[lost]
        grads[r].copy_(out)
        states[r].last_global_count = int(fidx.numel())
    return grads


def merge_topk(a, b, k: int, n: int):
    """Sum coincident indices, keep the top-k of the union by magnitude (``VGG/allreducer.py:129-138``): tie-inclusive,
    and a sum that cancelled to exactly 0 is dropped (its picks go back to their residuals), as on the device."""
    ia, va = a
    ib, vb = b
    idx = torch.cat([ia, ib])
    val = torch.cat([va, vb])
    uniq, inv = torch.unique(idx, return_inverse=True)   # sorted
    summed = torch.zeros(uniq.numel(), dtype=val.dtype, device=val.device)
    summed.index_add_(0, inv, val)
    keep = summed != 0
    if uniq.numel() > k:
        keep &= summed.abs() >= float(torch.topk(summed.abs(), k=k).values[-1])
    return uniq[keep], summed[keep]


# --------------------------------------------------------------------------- Gaussiank
def gaussiank_oracle(grads, states, cfg: OkTopkConfig, density=None):
    """Appendix B.3."""
    P = len(grads)
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    total = torch.zeros_like(grads[0])
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        acc = grads[r] + res
        std = float(torch.std(acc)) if n > 1 else 0.0
        mean = float(torch.mean(acc))
        _, thr = gen_threshold_from_normal_distribution(1.0 - density, mean, std)
        thr = gaussian_correct_threshold(acc.abs(), thr, k, cfg)
        mask = acc.abs() > thr
        res.copy_(acc)
        res[mask] = 0.0
        total += torch.where(mask, acc, torch.zeros_like(acc))
        st.local_thr = thr
        st.last_local_count = int(mask.sum())
        st.last_mode = "gaussiank"
    total /= P
    for r in range(P):
        grads[r].copy_(total)
    return grads


# --------------------------------------------------------------------------- TopkDSA / gaussiankSA
def topkdsa_oracle(grads, states, cfg: OkTopkConfig, density=None, gaussian_sa: bool = False):
    """Appendix B.4 (and the gaussiankSA variant of B.6: same data flow, no dense fallback).

    Exact local threshold every iteration, uniform regions, sparse reduce-scatter, allgather
    of all non-zeros of the reduced regions, dense fallback when the result is not sparse.
    Error feedback is the classic local one (residual zeroed at the exact local top-k for
    TopkDSA; at the strict ``>thr`` selection for gaussiankSA).  TopkDSA's top-k holds exactly
    ``k - #(|acc| > thr)`` of the elements tied at the k-th magnitude; which of them ``torch.topk``
    (or the device) picks is unspecified, so only that count is part of the specification.
    """
    P = len(grads)
    n = grads[0].numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    reduced = torch.zeros_like(grads[0])
    for r in range(P):
        st = states[r]
        res = st.ensure_residual(grads[r])
        acc = grads[r] + res
        top = torch.topk(acc.abs(), k=k)
        thr = float(top.values[-1])
        res.copy_(acc)
        mask = acc.abs() > thr
        if gaussian_sa:
            res[mask] = 0.0
        else:
            res[top.indices] = 0.0
        reduced = ftz(reduced + ftz(torch.where(mask, acc, torch.zeros_like(acc))))
        st.local_thr = thr
        st.last_local_count = int(mask.sum())
        st.last_mode = "gaussiankSA" if gaussian_sa else "topkSA"
    # the result is the same whichever branch (sparse lists vs dense regions) moves it
    nnz = int((reduced != 0).sum())
    dense_fallback = (not gaussian_sa) and nnz >= cfg.dsa_dense_fallback_frac * n
    out = reduced / P
    for r in range(P):
        grads[r].copy_(out)
        states[r].last_global_count = nnz
        states[r].last_mode += ":dense" if dense_fallback else ""
    return grads


ORACLES = {
    "none": lambda g, s, c, density=None: dense_oracle(g, s, c),
    "oktopk": oktopk_oracle,
    "topkA": topka_oracle,
    "topkA2": lambda g, s, c, density=None: topka_oracle(g, s, c, density, reselect=True),
    "topkAopt": topkaopt_oracle,
    "topkSA": topkdsa_oracle,
    "topkDSA": topkdsa_oracle,
    "gtopk": gtopk_oracle,
    "gaussiank": gaussiank_oracle,
    "gaussiankconcat": gaussiank_oracle,
    "gaussiankSA": lambda g, s, c, density=None: topkdsa_oracle(g, s, c, density, gaussian_sa=True),
}


def run_oracle(name: str, grads, states, cfg: OkTopkConfig, density=None):
    """One reduction of every rank's bucket, dense as ``plan_call`` says (warm-up, ``none``, the dense switch),
    counters advanced."""
    kind = plan_call(cfg, name, states[0].counter, density, len(grads)).kind
    if kind in ("dense", "dense_switch"):
        for g, st in zip(grads, states):
            if kind == "dense_switch":            # the error-compensated gradient is reduced densely, nothing left behind
                res = st.ensure_residual(g)
                g.add_(res)
                res.zero_()
            st.last_mode = "dense" if kind == "dense" else "dense(auto)"
        out = dense_oracle(grads)
    else:
        out = ORACLES[name](grads, states, cfg, density)
    for st in states:
        st.counter += 1
    return out


# --------------------------------------------------------------------------- dynamic loss scaling (config.LossScale)
def inv_scale_of(scale: float) -> float:
    """``torch.amp.GradScaler``'s inverse scale: the fp32 reciprocal of the scale computed in double."""
    return float(_np.float32(1.0 / float(_np.float32(scale))))


def update_scale(scale: float, growth_tracker: int, found_inf: bool, ls) -> Tuple[float, int]:
    """``torch._amp_update_scale_``: back off on a skipped step, grow after ``growth_interval`` clean steps (fp32 scale,
    products in double)."""
    if found_inf:
        return float(_np.float32(float(scale) * ls.backoff_factor)), 0
    successful = growth_tracker + 1
    if successful == ls.growth_interval:
        with _np.errstate(over="ignore"):
            grown = _np.float32(float(scale) * ls.growth_factor)
        return (float(grown) if _np.isfinite(grown) else scale), 0
    return scale, successful


def unscale_check_oracle(grads: List[torch.Tensor], inv_scale: float) -> bool:
    """Every rank's bucket is multiplied by ``inv_scale`` in place; returns the verdict all ranks agree on: True if any
    rank's bucket held a non-finite value (checked on the incoming values)."""
    bad = False
    for g in grads:
        bad |= bool((~torch.isfinite(g)).any())
        g.mul_(torch.tensor(inv_scale, dtype=torch.float32))
    return bad


def run_oracle_scaled(name: str, grads, states, cfg: OkTopkConfig, inv_scale: float, density=None):
    """One reduction under loss scaling: unscale, agree, and either skip -- residuals, thresholds and region edges
    untouched, counters advanced -- or reduce the unscaled gradients.  Returns (results or None, skipped)."""
    if unscale_check_oracle(grads, inv_scale):
        for st in states:
            st.counter += 1
        return None, True
    return run_oracle(name, grads, states, cfg, density), False
