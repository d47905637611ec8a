"""The sparse-allreduce schemes on library collectives (the "dist" backend).

Same state machine as the fused CUDA engine and the oracle, expressed with torch ops and
``torch.distributed`` collectives.  Runs on CPU/gloo (BASELINE config #1, the plumbing
configuration) and on GPU/NCCL, where it is the honest *strong baseline* the fused
peer-memory kernels are measured against (SURVEY 7.5-9).  Reference: the per-algorithm
branches of ``AllReducer.run`` (``VGG/allreducer.py:575-1622``) and the free functions
``topk_sparse_allreduce`` :34-69, ``gtopk_sparse_allreduce`` :76-172, ``dense_allreduce``
:175-180.  No host staging, no float-cast index packing (A.4-1), int32 indices.

Every function reduces ``g`` (1-D fp32 bucket) in place and returns it.
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch

from ..compression import gaussian_correct_threshold, gen_threshold_from_normal_distribution
from ..config import OkTopkConfig
from .oracle import (adapt_global, adapt_local, boundaries_from_cuts, ftz, guard_threshold,
                     kth_largest_abs, quantile_cuts, topk_tie_inclusive)
from .state import SparseState, offsets_of, plan_call, uniform_boundaries
from .world import World


def _k(n: int, density: float) -> int:
    return max(int(n * density), 1)


# --------------------------------------------------------------------------- dense (C11, B3)
def dense_allreduce(g: torch.Tensor, world: World) -> torch.Tensor:
    world.all_reduce_sum(g)
    if world.size > 1:
        g.div_(world.size)
    return g


# --------------------------------------------------------------------------- shared phases
def _select_regions(acc: torch.Tensor, thr: float, edges: List[int]):
    """Per-region strict ``|x| > thr`` select (A5): region-local int32 idx + fp32 val per destination."""
    mask = acc.abs() > thr
    sel = mask.nonzero(as_tuple=False).view(-1)                 # ascending global indices
    vals = acc[sel]
    cuts = torch.searchsorted(sel, torch.tensor(edges, dtype=sel.dtype, device=sel.device))
    cuts = cuts.tolist()
    send = []
    for d in range(len(edges) - 1):
        a, b = cuts[d], cuts[d + 1]
        send.append([(sel[a:b] - edges[d]).to(torch.int32), vals[a:b]])
    return send, sel, mask


def _sparse_reduce_scatter(send, world: World, cfg: OkTopkConfig, region_len: int, like: torch.Tensor,
                           st: SparseState) -> torch.Tensor:
    """Phase 4 / B5+B6+A7: count handshake, throttled pairwise exchange, scatter-add per source."""
    P = world.size
    ssizes = [s[0].numel() for s in send]
    rsizes = world.all_to_all_counts(ssizes, like.device)
    reduced = torch.zeros(region_len, dtype=like.dtype, device=like.device)

    def reduce_chunk(chunk):
        for _src, (idx, val) in chunk:
            if idx.numel():
                # indices are unique within one source -> plain indexed add is exact; subnormals flushed as the
                # device's atomics do (oracle.ftz)
                i = idx.long()
                reduced[i] = ftz(reduced[i] + ftz(val))

    world.exchange_pairwise(send, rsizes, throttle=min(cfg.throttle, P), on_chunk=reduce_chunk)
    st.last_volume_elems += 2 * (sum(ssizes) - ssizes[world.rank]) + 2 * (sum(rsizes) - rsizes[world.rank])
    return reduced


def _balanced_slices(counts: List[int], P: int):
    """B13: who must hand which contiguous slice of the rank-ordered global list to whom so that
    every rank holds ceil(T/P) entries (``BERT/bert/allreducer.py:615-710``)."""
    T = sum(counts)
    per = -(-T // P) if T else 0
    starts = offsets_of(counts)
    moves = []  # (src, dst, a, b) in global-list coordinates
    for d in range(P):
        lo, hi = min(d * per, T), min((d + 1) * per, T)
        for s in range(P):
            a, b = max(lo, starts[s]), min(hi, starts[s] + counts[s])
            if a < b:
                moves.append((s, d, a, b))
    return moves, per


def _allgather_sparse(gidx: torch.Tensor, gval: torch.Tensor, world: World, cfg: OkTopkConfig,
                      st: SparseState):
    """Phase 5 tail / B7+B8(+B13): allgatherv of (global int32 idx, fp32 val)."""
    P = world.size
    counts = world.all_gather_counts(gidx.numel(), gidx.device)
    if cfg.balanced_allgather and P > 1 and sum(counts) > 0:
        import torch.distributed as dist
        moves, per = _balanced_slices(counts, P)
        starts = offsets_of(counts)
        my_i, my_v, ops, landed = [], [], [], []
        for (s, d, a, b) in moves:
            if s == world.rank and d == world.rank:
                my_i.append((a, gidx[a - starts[s]:b - starts[s]]))
                my_v.append((a, gval[a - starts[s]:b - starts[s]]))
            elif s == world.rank:
                ops.append(dist.P2POp(dist.isend, gidx[a - starts[s]:b - starts[s]].contiguous(), world._global(d), group=world.group))
                ops.append(dist.P2POp(dist.isend, gval[a - starts[s]:b - starts[s]].contiguous(), world._global(d), group=world.group))
                st.last_volume_elems += 2 * (b - a)
            elif d == world.rank:
                bi = torch.empty(b - a, dtype=gidx.dtype, device=gidx.device)
                bv = torch.empty(b - a, dtype=gval.dtype, device=gval.device)
                ops.append(dist.P2POp(dist.irecv, bi, world._global(s), group=world.group))
                ops.append(dist.P2POp(dist.irecv, bv, world._global(s), group=world.group))
                landed.append((a, bi, bv))
                st.last_volume_elems += 2 * (b - a)
        for q in (dist.batch_isend_irecv(ops) if ops else []):
            q.wait()
        for a, bi, bv in landed:
            my_i.append((a, bi))
            my_v.append((a, bv))
        my_i.sort(key=lambda x: x[0])
        my_v.sort(key=lambda x: x[0])
        gidx = torch.cat([x[1] for x in my_i]) if my_i else gidx[:0]
        gval = torch.cat([x[1] for x in my_v]) if my_v else gval[:0]
        counts = world.all_gather_counts(gidx.numel(), gidx.device)
    (all_i, all_v), counts = world.all_gatherv([gidx, gval], counts)
    total = sum(counts)
    st.last_volume_elems += 2 * (total - counts[world.rank]) + (2 * counts[world.rank] if P > 1 else 0)
    return all_i, all_v, total


# --------------------------------------------------------------------------- Ok-Topk (C6)
def oktopk_allreduce(g: torch.Tensor, st: SparseState, cfg: OkTopkConfig, world: World,
                     density: Optional[float] = None) -> torch.Tensor:
    """SURVEY 3.3.  ``VGG/allreducer.py:575-1098`` / ``BERT/bert/allreducer.py:357-743``."""
    P, rank = world.size, world.rank
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    plan = plan_call(cfg, "oktopk", st.counter, density, P)
    st.last_volume_elems = 0
    with torch.no_grad():
        # (1) error feedback + local threshold
        res = st.ensure_residual(g)
        g.add_(res)
        res.copy_(g)
        if plan.exact_local or st.local_thr == 0.0:    # a carried 0 cannot be capped: recompute
            thr = kth_largest_abs(g, k)
        else:
            thr = guard_threshold(g.abs(), st.local_thr, k, cfg)
        st.local_thr = thr

        # (2) region re-partition: average the local quantile cut points (B4)
        if plan.repartition:
            sel = (g.abs() > thr).nonzero(as_tuple=False).view(-1)
            cuts = torch.tensor(quantile_cuts(sel, P, n), dtype=torch.int64, device=g.device)
            world.all_reduce_sum(cuts)
            st.boundaries, st.region_offsets = boundaries_from_cuts((cuts // P).tolist(), n)
        edges = st.region_offsets + [n]

        # (3) select + pack per destination
        send, sel_idx, lmask = _select_regions(g, thr, edges)
        cnt = int(sel_idx.numel())
        st.last_local_count = cnt
        st.local_thr = adapt_local(thr, cnt, k, cfg)

        # (4) sparse reduce-scatter onto the region owners
        reduced = _sparse_reduce_scatter(send, world, cfg, st.boundaries[rank], g, st)

        # (5) global selection on my region + sparse allgather
        off = st.region_offsets[rank]
        if plan.exact_global:
            ridx = reduced.nonzero(as_tuple=False).view(-1)
            all_i, all_v, total = _allgather_sparse((ridx + off).to(torch.int32), reduced[ridx], world,
                                                    cfg.replace(balanced_allgather=False), st)
            kk = min(total, k)
            if kk > 0:
                gthr = float(torch.topk(all_v.abs(), k=kk).values[-1])
                keep = all_v.abs() >= gthr
                all_i, all_v = all_i[keep], all_v[keep]
            else:
                gthr = 0.0
            st.global_thr = gthr
        else:
            ridx = (reduced.abs() > st.global_thr).nonzero(as_tuple=False).view(-1)
            all_i, all_v, total = _allgather_sparse((ridx + off).to(torch.int32), reduced[ridx], world, cfg, st)
            st.global_thr = adapt_global(st.global_thr, total, k, cfg)
        st.last_global_count = int(all_i.numel())

        # (6) result in place, (7) residual cleared where locally selected AND globally kept:
        #     "locally selected" <=> |residual| > thr  (SURVEY 3.3 note; no intersect1d needed)
        gi = all_i.long()
        g.zero_()
        g[gi] = all_v / P
        hit = res[gi].abs() > thr
        res[gi[hit]] = 0.0
        st.last_mode = "oktopk"
    return g


# --------------------------------------------------------------------------- TopkA / TopkA2 (C7)
def topka_allreduce(g, st: SparseState, cfg: OkTopkConfig, world: World, density=None,
                    reselect: bool = False):
    """Appendix B.1 (``VGG/allreducer.py:34-69,481-530,1359-1419``)."""
    P = world.size
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    with torch.no_grad():
        if cfg.norm_clip is not None:
            nrm = float(g.norm())
            mx = (1.0 / P) ** 0.5 * cfg.norm_clip
            if nrm > mx and nrm > 0:
                g.mul_(mx / nrm)
        res = st.ensure_residual(g)
        g.add_(res)
        st.local_thr = kth_largest_abs(g, k)
        idx = topk_tie_inclusive(g, k)                              # ties at the k-th magnitude: more than k entries
        vals = g[idx].clone()
        res.copy_(g)
        res[idx] = 0.0
        (all_i, all_v), counts = world.all_gatherv([idx.to(torch.int32), vals])
        g.zero_()
        for ri, rv in zip(all_i.split(counts), all_v.split(counts)):     # rank order, as the oracle adds them
            g[ri.long()] += rv
        if reselect:
            U = torch.unique(all_i.long())
            keep = torch.zeros(n, dtype=torch.bool, device=g.device)
            if U.numel() > k:
                keep[U] = g[U].abs() >= float(torch.topk(g[U].abs(), k=k).values[-1])
            else:
                keep[U] = True
            g.mul_(keep)
            lost = ~keep[idx]
            res[idx[lost]] += vals[lost]
        g.div_(P)
        st.last_local_count = int(idx.numel())
        st.last_global_count = int((g != 0).sum())
        st.last_volume_elems = 2 * (sum(counts) - counts[world.rank]) * 2
        st.last_mode = "topkA2" if reselect else "topkA"
    return g


# --------------------------------------------------------------------------- TopkAopt (C7b)
def topkaopt_allreduce(g, st: SparseState, cfg: OkTopkConfig, world: World, density=None):
    """``VGG/allreducer.py:1100-1150`` with the scatter-add on the device instead of NumPy."""
    P = world.size
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    exact = plan_call(cfg, "topkAopt", st.counter, density, P).exact_local
    with torch.no_grad():
        res = st.ensure_residual(g)
        g.add_(res)
        res.copy_(g)
        if exact:
            st.local_thr = kth_largest_abs(g, k)
        idx = (g.abs() > st.local_thr).nonzero(as_tuple=False).view(-1)
        vals = g[idx]
        res[idx] = 0.0
        (all_i, all_v), counts = world.all_gatherv([idx.to(torch.int32), vals])
        g.zero_()
        g.index_add_(0, all_i.long(), all_v)
        g.div_(P)
        st.last_local_count = int(idx.numel())
        st.last_global_count = int((g != 0).sum())
        st.last_volume_elems = 2 * (sum(counts) - counts[world.rank]) * 2
        st.last_mode = "topkAopt"
    return g


# --------------------------------------------------------------------------- gTopk (C9)
def gtopk_allreduce(g, st: SparseState, cfg: OkTopkConfig, world: World, density=None):
    """Appendix B.2 (``VGG/allreducer.py:76-172``): log2(P) rounds of pairwise merge toward rank 0,
    then a broadcast; the non-surviving local picks go back into the residual."""
    P, rank = world.size, world.rank
    assert P & (P - 1) == 0, "gTopk needs a power-of-two world size (VGG/allreducer.py:113)"
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    from .oracle import merge_topk
    with torch.no_grad():
        if cfg.norm_clip is not None:
            nrm = float(g.norm())
            mx = (1.0 / P) ** 0.5 * cfg.norm_clip
            if nrm > mx and nrm > 0:
                g.mul_(mx / nrm)
        res = st.ensure_residual(g)
        g.add_(res)
        idx0 = topk_tie_inclusive(g, k)
        val0 = g[idx0].clone()
        res.copy_(g)
        res[idx0] = 0.0
        idx, val = idx0, val0
        vol = 0
        step = 1
        while step < P:
            if rank % (2 * step) == 0:
                peer = rank + step
                hdr = torch.zeros(1, dtype=torch.int64, device=g.device)
                world.recv(hdr, peer)
                m = int(hdr.item())
                ri = torch.empty(m, dtype=torch.int32, device=g.device)
                rv = torch.empty(m, dtype=g.dtype, device=g.device)
                if m:
                    world.recv(ri, peer)
                    world.recv(rv, peer)
                idx, val = merge_topk((idx, val), (ri.long(), rv), k, n)
                vol += 2 * m
            elif rank % (2 * step) == step:
                peer = rank - step
                world.send(torch.tensor([idx.numel()], dtype=torch.int64, device=g.device), peer)
                if idx.numel():
                    world.send(idx.to(torch.int32), peer)
                    world.send(val, peer)
                vol += 2 * idx.numel()
            step *= 2
        hdr = torch.tensor([idx.numel() if rank == 0 else 0], dtype=torch.int64, device=g.device)
        world.broadcast(hdr, 0)
        m = int(hdr.item())
        bi = idx.to(torch.int32) if rank == 0 else torch.empty(m, dtype=torch.int32, device=g.device)
        bv = val if rank == 0 else torch.empty(m, dtype=g.dtype, device=g.device)
        if m:
            world.broadcast(bi, 0)
            world.broadcast(bv, 0)
        vol += 2 * m if P > 1 else 0
        g.zero_()
        g[bi.long()] = bv / P
        keep = torch.zeros(n, dtype=torch.bool, device=g.device)
        keep[bi.long()] = True
        lost = ~keep[idx0]
        res[idx0[lost]] += val0[lost]
        st.last_local_count = int(idx0.numel())
        st.last_global_count = m
        st.last_volume_elems = vol
        st.last_mode = "gtopk"
    return g


# --------------------------------------------------------------------------- Gaussiank (C10, C10b)
def gaussiank_allreduce(g, st: SparseState, cfg: OkTopkConfig, world: World, density=None):
    """Appendix B.3 (``VGG/allreducer.py:1420-1465``, ``VGG/compression.py:220-266``).
    ``gaussiankconcat`` (:1467-1501) differs only in wire packing, which does not exist here."""
    P = world.size
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    with torch.no_grad():
        res = st.ensure_residual(g)
        g.add_(res)
        std = float(torch.std(g)) if n > 1 else 0.0
        mean = float(torch.mean(g))
        _, thr = gen_threshold_from_normal_distribution(1.0 - density, mean, std)
        absx = g.abs()
        thr = gaussian_correct_threshold(absx, thr, k, cfg)
        idx = (absx > thr).nonzero(as_tuple=False).view(-1)
        vals = g[idx]
        res.copy_(g)
        res[idx] = 0.0
        (all_i, all_v), counts = world.all_gatherv([idx.to(torch.int32), vals])
        g.zero_()
        g.index_add_(0, all_i.long(), all_v)
        g.div_(P)
        st.local_thr = thr
        st.last_local_count = int(idx.numel())
        st.last_global_count = int((g != 0).sum())
        st.last_volume_elems = 2 * (sum(counts) - counts[world.rank]) * 2
        st.last_mode = "gaussiank"
    return g


# --------------------------------------------------------------------------- TopkDSA (C8) / gaussiankSA (C10c)
def topkdsa_allreduce(g, st: SparseState, cfg: OkTopkConfig, world: World, density=None,
                      gaussian_sa: bool = False):
    """Appendix B.4 (``VGG/allreducer.py:1153-1357``); ``gaussian_sa`` = B.6 (:1503-1620)."""
    P, rank = world.size, world.rank
    n = g.numel()
    density = cfg.density if density is None else density
    k = _k(n, density)
    st.last_volume_elems = 0
    with torch.no_grad():
        res = st.ensure_residual(g)
        g.add_(res)
        top = torch.topk(g.abs(), k=k)
        thr = float(top.values[-1])
        res.copy_(g)
        b = uniform_boundaries(n, P)
        off = offsets_of(b)
        edges = off + [n]
        send, sel_idx, _ = _select_regions(g, thr, edges)
        if gaussian_sa:
            res[sel_idx] = 0.0
        else:
            res[top.indices] = 0.0
        reduced = _sparse_reduce_scatter(send, world, cfg, b[rank], g, st)
        ridx = reduced.nonzero(as_tuple=False).view(-1)
        counts = world.all_gather_counts(ridx.numel(), g.device)
        total = sum(counts)
        if (not gaussian_sa) and total >= cfg.dsa_dense_fallback_frac * n:
            # B9: dense fallback -- allgatherv of the reduced regions
            mx = max(b)
            pad = torch.zeros(mx, dtype=g.dtype, device=g.device)
            pad[:b[rank]] = reduced
            allr = world.all_gather_fixed(pad)
            for r in range(P):
                g[off[r]:off[r] + b[r]] = allr[r, :b[r]]
            g.div_(P)
            st.last_volume_elems += 2 * (n - b[rank])
            st.last_mode = "topkSA:dense"
        else:
            (all_i, all_v), _ = world.all_gatherv([(ridx + off[rank]).to(torch.int32), reduced[ridx]], counts)
            g.zero_()
            g[all_i.long()] = all_v / P
            st.last_volume_elems += 2 * (total - counts[rank]) + (2 * counts[rank] if P > 1 else 0)
            st.last_mode = "gaussiankSA" if gaussian_sa else "topkSA"
        st.local_thr = thr
        st.last_local_count = int(sel_idx.numel())
        st.last_global_count = total
    return g


ALGORITHMS = {
    "oktopk": oktopk_allreduce,
    "topkA": topka_allreduce,
    "topkA2": lambda g, st, cfg, w, density=None: topka_allreduce(g, st, cfg, w, density, reselect=True),
    "topkAopt": topkaopt_allreduce,
    "topkSA": topkdsa_allreduce,
    "topkDSA": topkdsa_allreduce,
    "gtopk": gtopk_allreduce,
    "gaussiank": gaussiank_allreduce,
    "gaussiankconcat": gaussiank_allreduce,
    "gaussiankSA": lambda g, st, cfg, w, density=None: topkdsa_allreduce(g, st, cfg, w, density, gaussian_sa=True),
}


def sparse_allreduce(name: str, g: torch.Tensor, st: SparseState, cfg: OkTopkConfig, world: World,
                     density: Optional[float] = None) -> torch.Tensor:
    """Dispatch on the compressor name exactly like ``AllReducer.run`` (``VGG/allreducer.py:573-1622``):
    dense as ``plan_call`` says (warm-up, ``none``, the dense switch), else the named scheme.  Advances the bucket
    counter."""
    kind = plan_call(cfg, name, st.counter, density, world.size).kind
    if kind in ("dense", "dense_switch"):
        if kind == "dense_switch":
            with torch.no_grad():
                res = st.ensure_residual(g)
                g.add_(res)
                res.zero_()
        dense_allreduce(g, world)
        st.last_mode = "dense" if kind == "dense" else "dense(auto)"
        st.last_volume_elems = 2 * g.numel() * (world.size - 1) // max(world.size, 1)
    else:
        ALGORITHMS[name](g, st, cfg, world, density)
    st.counter += 1
    return g
