"""The magnitude-selection kernels on the inputs where selection goes wrong: ties at the k-th magnitude (bf16- and
fp16-valued gradients, one magnitude everywhere), zero-heavy and all-zero buckets, signed zeros, subnormals, a wide
dynamic range, and buckets from 1 element to just past one pack tile, one tile-row of the full grid and 1 M.

GPU cases (P = 1) compare the sm_90a kernels with the oracle bit for bit; CPU cases pin the tie and zero-threshold
rules of the oracle and of the torch.distributed path (gloo)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402

# ------------------------------------------------------------------------------------------------ gradient generators
GENS = ["bf16", "fp16", "one_mag", "zeros95", "zeros", "signed_zeros", "subnormal", "wide"]
TIED = ["bf16", "fp16", "one_mag"]
ZERO_HEAVY = ["zeros95", "zeros"]


def _sign(n, g):
    return torch.randint(0, 2, (n,), generator=g).float() * 2 - 1


def gen(kind, n, seed):
    """Seeded fp32 gradient of ``n`` elements (CPU)."""
    g = torch.Generator().manual_seed(seed)
    if kind == "bf16":                      # 8-bit mantissa: ties at the k-th magnitude are the normal case
        return torch.randn(n, generator=g).bfloat16().float()
    if kind == "fp16":
        return torch.randn(n, generator=g).half().float()
    if kind == "one_mag":                   # every element tied, mixed signs
        return _sign(n, g) * 0.375
    if kind == "zeros95":                   # ~95 % exact zeros
        x = torch.randn(n, generator=g)
        return torch.where(torch.rand(n, generator=g) < 0.05, x, torch.zeros(n))
    if kind == "zeros":
        return torch.zeros(n)
    if kind == "signed_zeros":              # -0.0 and +0.0 around a few normal values
        x = torch.randn(n, generator=g)
        z = torch.where(torch.rand(n, generator=g) < 0.5, torch.tensor(-0.0), torch.tensor(0.0))
        return torch.where(torch.rand(n, generator=g) < 0.3, x, z)
    if kind == "subnormal":                 # even elements subnormal (a 1-element bucket is one), odd ones normal
        sub = torch.rand(n, generator=g) * 2.0 ** -126 * _sign(n, g)
        return torch.where(torch.arange(n) % 2 == 0, sub, torch.randn(n, generator=g))
    if kind == "wide":                      # |x| log-uniform in [1e-30, 1e30]: no overflow once the residual is added
        e = torch.rand(n, generator=g, dtype=torch.float64) * 60.0 - 30.0
        return (_sign(n, g).double() * 10.0 ** e).float()
    raise KeyError(kind)


def test_generators_have_the_advertised_properties():
    n = 100_000
    x = gen("bf16", n, 0)
    assert torch.equal(x, x.bfloat16().float())
    k = n // 100
    t = torch.topk(x.abs(), k).values[-1]
    assert int((x.abs() == t).sum()) > 1                              # a tie at the k-th magnitude
    assert torch.equal(gen("fp16", n, 0), gen("fp16", n, 0).half().float())
    assert int((gen("one_mag", n, 0).abs() != 0.375).sum()) == 0
    z = gen("zeros95", n, 0)
    assert 0.04 * n < int((z != 0).sum()) < 0.06 * n
    s = gen("signed_zeros", n, 0)
    zero = s == 0
    assert bool((zero & torch.signbit(s)).any()) and bool((zero & ~torch.signbit(s)).any())
    u = gen("subnormal", n, 0)
    tiny = torch.finfo(torch.float32).tiny
    assert bool(((u.abs() < tiny) & (u != 0)).any()) and bool((u.abs() > 1e-3).any())
    w = gen("wide", n, 0).abs()
    assert float(w.min()) >= 1e-30 * 0.99 and float(w.max()) <= 1e30 * 1.01
    assert torch.isfinite(w + w).all()


# ------------------------------------------------------------------------------------------------ GPU helpers
def _C():
    from oktopk_b200.ops import ext
    return ext.require()


def _sizes():
    """Scalar tails only; around one pack tile (kTileV x 4 floats); one tile-row of the full grid +- 1; > 1 M, n % 4 != 0."""
    row = 4096 * _C().max_coop_grid(0)
    return [1, 2, 3, 5, 33, 4095, 4096, 4097, row - 1, row, row + 1, 1_048_579]


def _bits(t):
    return t.view(torch.int32)


# ------------------------------------------------------------------------------------------------ kth_abs
@pytest.mark.gpu
@pytest.mark.parametrize("kind", GENS)
def test_kth_abs_bitwise_on_edge_inputs(kind):
    """Radix select against torch.topk, bit for bit: k = 1, k = n, and k > nnz (the answer is +0.0)."""
    C = _C()
    st = C.dev_alloc_zero(C.state_bytes())
    out = torch.zeros(1, device="cuda")
    try:
        for n in _sizes():
            x = gen(kind, n, n)
            nnz = int((x != 0).sum())
            ks = {1, n} | ({nnz + 1} if nnz < n else set())
            xd = x.cuda()
            for k in sorted(ks):
                C.kth_abs(xd.data_ptr(), n, k, st, out.data_ptr(), C.max_coop_grid(0), torch.cuda.current_stream().cuda_stream)
                ref = torch.topk(x.abs(), k).values[-1:]
                got = out.cpu()
                assert torch.equal(_bits(got), _bits(ref)), (kind, n, k, float(got), float(ref))
    finally:
        torch.cuda.synchronize()
        C.dev_free(st)


# ------------------------------------------------------------------------------------------------ engine vs oracle
def _run_engine_vs_oracle(name, n, iters, cfg, data, tol_count=0, rtol=0.0, srcs_layout=None, reset_at=()):
    """``data(it, n)`` -> the CPU gradient of call ``it``.  After every call: result, residual, counts and thresholds
    equal the oracle's.  ``srcs_layout = (sizes, offsets)``: the engine reads the gradient from one tensor per segment
    (its bucket all-zero on entry); the oracle sees it landed at those offsets.  ``reset_at``: calls before which both
    residuals are cleared, so that the call sees only its own gradient.  Returns (engine stats, oracle local count) per
    call."""
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    from oktopk_b200.parallel.world import World
    eng = CudaBucketEngine(n, cfg, World(), name="t")
    states = [SparseState(n, 1)]
    ne = (lambda a, b: a != b) if rtol == 0.0 else (lambda a, b: ~torch.isclose(a, b, rtol=rtol, atol=5e-7))
    hist = []
    try:
        for it in range(iters):
            x = data(it, n)
            if it in reset_at:
                eng.residual.zero_()
                if states[0].residual is not None:
                    states[0].residual.zero_()
            if srcs_layout is None:
                eng.grad.copy_(x.cuda())
                eng.reduce(name)
            else:
                sizes, offs = srcs_layout
                parts = [x[o:o + s].cuda() for s, o in zip(sizes, offs)]
                eng.reduce(name, srcs=([t.data_ptr() for t in parts], list(offs), list(sizes)))
            torch.cuda.synchronize()
            ref = run_oracle(name, [x.clone()], states, cfg)[0]
            got = eng.grad.cpu()
            st = eng.stats()
            bad = int(ne(got, ref).sum())
            assert bad <= tol_count, "%s n %d it %d: %d mismatching elements (stats %s)" % (name, n, it, bad, st)
            rbad = int(ne(eng.residual.cpu(), states[0].residual).sum())
            assert rbad <= tol_count, "%s n %d it %d: residual mismatch %d" % (name, n, it, rbad)
            if tol_count == 0:
                assert st["local_count"] == states[0].last_local_count, (n, it, st, states[0].last_local_count)
                if name == "oktopk":
                    assert st["local_thr"] == states[0].local_thr, (n, it, st, states[0].local_thr)
                    assert st["local_thr_used"] == states[0].last_thr_used, (n, it, st, states[0].last_thr_used)
                    assert st["global_thr"] == states[0].global_thr, (n, it, st, states[0].global_thr)
                    assert st["global_count"] == states[0].last_global_count, (n, it, st, states[0].last_global_count)
                elif name == "topkAopt":
                    assert st["local_thr"] == states[0].local_thr, (n, it, st, states[0].local_thr)
            assert st["overflow_send"] == 0 and st["overflow_gather"] == 0, (n, it, st)
            assert st["fault"] == 0
            hist.append((st, states[0].last_local_count))
            if srcs_layout is not None:
                eng.grad.zero_()                     # what the fused update does before the next source-reading call
    finally:
        eng.close()
    return hist


# Ok-Topk schedule (exact calls at 0, 3, 6): (gradient scale, clear both residuals first).  x0.01 on a cleared exact
# call leaves no element above the prefilter cut (0.8 x the carried threshold) -> full radix select; the jump back
# (x100) on a cleared exact call puts almost every element above it, more than the bounded layout's candidate capacity
# -> full select.  (A stale threshold 100x too small would overflow a bounded send slot and run the redo policy, which
# the oracle does not model: tests/test_gpu_kernels.py covers that by conservation.)
_SCHEDULE = [(1.0, False), (1.0, False), (1.0, False), (0.01, True), (0.01, False), (0.01, False), (1.0, True),
             (1.0, False), (1.0, False)]
_LAYOUTS = {"lossless": dict(slot_factor=0.0, gather_factor=0.0), "bounded": dict(slot_factor=16.0, gather_factor=16.0)}


def _okt_cfg(mode, layout, **kw):
    from oktopk_b200.config import OkTopkConfig
    return OkTopkConfig(**dict(dict(density=0.01, local_recompute_interval=3, global_recompute_interval=3,
                                    repartition_interval=8, gselect_mode=mode, overselect_cap=2.0, **_LAYOUTS[layout]), **kw))


def _okt_vs_oracle(kind, n, cfg, srcs_layout=None, covered=None):
    def data(it, m):
        x = gen(kind, m, 31 * it + m) * _SCHEDULE[it][0]
        return x if covered is None else x * covered
    _run_engine_vs_oracle("oktopk", n, len(_SCHEDULE), cfg, data, srcs_layout=srcs_layout,
                          reset_at={i for i, (_, r) in enumerate(_SCHEDULE) if r})


def _okt_cases(kinds, combos):
    # every element tied: the reuse call after an exact one selects the whole bucket, which overflows any bounded send
    # slot by design (redo policy), so that generator runs on the lossless layout only
    return [(k, m, l) for k in kinds for m, l in combos if not (k == "one_mag" and l == "bounded")]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,mode,layout", _okt_cases(GENS + ["zeros95_nnz_below_k"], [
    ("list", "lossless"), ("scan", "lossless"), ("list", "bounded"), ("scan", "bounded")]))
def test_oktopk_edges_match_oracle(kind, mode, layout):
    """Landed bucket, every size, exact and threshold-reuse calls, prefilter fallbacks: bitwise the oracle's."""
    density = 0.1 if kind == "zeros95_nnz_below_k" else 0.01          # ~5 % non-zeros: nnz > k at 0.01, < k at 0.1
    kind = "zeros95" if kind == "zeros95_nnz_below_k" else kind
    for n in _sizes():
        _okt_vs_oracle(kind, n, _okt_cfg(mode, layout, density=density))


def _layout(sizes):
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 63) // 64 * 64
    return offs, o


@pytest.mark.gpu
@pytest.mark.parametrize("kind,mode,layout", _okt_cases(GENS, [("list", "lossless"), ("scan", "bounded")]))
def test_oktopk_edges_from_gradient_sources_match_oracle(kind, mode, layout):
    """The gradient read from its source tensors (tiny ones, ones around a tile, one > 1 M; padding between them)."""
    sizes = [1, 2, 3, 5, 33, 4095, 4096, 4097, 1_048_579]
    offs, n = _layout(sizes)
    covered = torch.zeros(n)
    for s, o in zip(sizes, offs):
        covered[o:o + s] = 1.0
    _okt_vs_oracle(kind, n, _okt_cfg(mode, layout), srcs_layout=(sizes, offs), covered=covered)


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("layout", ["lossless", "bounded"])
def test_overselect_cap_holds_after_a_zero_threshold(layout, fused):
    """An all-zero exact call leaves a carried threshold of 0; the threshold-reuse calls after it recompute the exact
    threshold instead of shipping every non-zero, so the volume stays within overselect_cap * k -- in the kernel
    (decided on the device, also when every phase is a launch of its own) and in the oracle."""
    n = 100_003
    k = int(n * 0.01)
    cfg = _okt_cfg("auto", layout, local_recompute_interval=4, global_recompute_interval=4, fused=fused)
    hist = _run_engine_vs_oracle("oktopk", n, 6, cfg,
                                 lambda it, m: torch.zeros(m) if it in (0, 4) else gen("bf16", m, it))
    assert [h[0]["local_count"] for h in hist] == [h[1] for h in hist]
    assert all(h[0]["local_count"] <= 2 * k for h in hist), [h[0]["local_count"] for h in hist]
    assert hist[1][0]["local_thr_used"] > 0.0


# ------------------------------------------------------------------------------------------------ gather / tree schemes
@pytest.mark.gpu
@pytest.mark.parametrize("kind", TIED + ZERO_HEAVY)
@pytest.mark.parametrize("name", ["topkA", "topkA2", "topkAopt", "gtopk", "gaussiank"])
def test_gather_and_tree_schemes_match_oracle_on_ties_and_zeros(name, kind):
    """Tie-inclusive local picks (TopkA / TopkA2 / gTopk), the re-selection of TopkA2, threshold reuse (TopkAopt) and
    the Gaussian threshold against the oracle.  Gaussiank keeps its tolerance for the rounding of the threshold."""
    from oktopk_b200.config import OkTopkConfig
    cfg = OkTopkConfig(density=0.01, topkaopt_recompute_interval=2)
    for n in _sizes():
        k = max(int(n * 0.01), 1)
        if name == "gtopk" and kind == "one_mag" and n > min((n + 31) // 32 * 32, 2 * k + 1024):
            continue        # more tied picks than gTopk's pick list holds: test_bounded_slots_keep_unsent_ties
        _run_engine_vs_oracle(name, n, 3, cfg, lambda it, m: gen(kind, m, 7 * it + m),
                              tol_count=40 if name == "gaussiank" else 0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["topkA", "topkA2", "gtopk"])
def test_bounded_slots_keep_unsent_ties_in_the_residual(name):
    """Every element tied: the tie-inclusive pick selects the whole bucket, far more than a bounded gather slot (or
    gTopk's pick list) holds.  What does not fit stays in the residual: acc == residual + result, exactly."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    n = 400_003
    eng = CudaBucketEngine(n, OkTopkConfig(density=0.01, gather_factor=1.0), World(), name="t")
    res_prev = torch.zeros(n)
    try:
        for it in range(3):
            x = gen("one_mag", n, it)
            acc = x + res_prev
            eng.grad.copy_(x.cuda())
            eng.reduce(name)
            torch.cuda.synchronize()
            out, res, st = eng.grad.cpu(), eng.residual.cpu(), eng.stats()
            assert int((acc != res + out).sum()) == 0, (it, st)
            assert st["overflow_gather"] > 0 and 0 < int((out != 0).sum()) < n, (it, st)
            assert st["fault"] == 0
            res_prev = res
    finally:
        eng.close()


# ------------------------------------------------------------------------------------------------ TopkDSA
@pytest.mark.gpu
@pytest.mark.parametrize("kind", TIED + ["zeros95"])
def test_topkdsa_clears_exactly_the_tied_top_k(kind):
    """TopkDSA sends |x| > thr and clears the residual of the exact top-k.  With a tie at the k-th magnitude that is
    every element above it plus exactly k - #(|x| > thr) of the tied ones (which ones is unspecified); every other
    element matches the oracle bit for bit and keeps its accumulated value."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    from oktopk_b200.parallel.world import World
    cfg = OkTopkConfig(density=0.01)
    for n in _sizes():
        k = max(int(n * 0.01), 1)
        eng = CudaBucketEngine(n, cfg, World(), name="t")
        states = [SparseState(n, 1)]
        res_prev = torch.zeros(n)
        try:
            for it in range(3):
                x = gen(kind, n, 5 * it + n)
                acc = x + res_prev
                eng.grad.copy_(x.cuda())
                eng.reduce("topkDSA")
                torch.cuda.synchronize()
                ref = run_oracle("topkDSA", [x.clone()], states, cfg)[0]
                out, res, st = eng.grad.cpu(), eng.residual.cpu(), eng.stats()
                thr = float(torch.topk(acc.abs(), k).values[-1])
                tie = (acc.abs() == thr) & (acc != 0)
                above = int((acc.abs() > thr).sum())
                assert int((out != ref).sum()) == 0, (kind, n, it, st)
                assert int((res != states[0].residual)[~tie].sum()) == 0, (kind, n, it)
                cleared = int((res[tie] == 0).sum())
                assert cleared == (k - above if thr > 0 else 0), (kind, n, it, cleared, k, above, int(tie.sum()))
                assert cleared == int((states[0].residual[tie] == 0).sum())               # the oracle's count
                kept = ~(tie & (res == 0))                                                  # conservation elsewhere
                assert int((acc != res + out)[kept].sum()) == 0, (kind, n, it)
                assert st["local_count"] == above and st["fault"] == 0
                res_prev = res
                states[0].residual.copy_(res)           # carry the device's choice of cleared ties into the next call
        finally:
            eng.close()


# ------------------------------------------------------------------------------------------------ CPU: oracle
def _oracle_run(name, xs, cfg, n):
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    states = [SparseState(n, 1)]
    outs = []
    for x in xs:
        outs.append(run_oracle(name, [x.clone()], states, cfg)[0].clone())
    return outs, states[0]


@pytest.mark.parametrize("kind", TIED + ZERO_HEAVY)
@pytest.mark.parametrize("name", ["topkA", "topkA2", "gtopk"])
def test_oracle_exact_topk_picks_are_tie_inclusive(name, kind):
    """TopkA / TopkA2 / gTopk pick |x| >= the k-th magnitude and |x| > 0: every tied element, no zero."""
    from oktopk_b200.config import OkTopkConfig
    n = 20_000
    k = int(n * 0.01)
    x = gen(kind, n, 3)
    outs, st = _oracle_run(name, [x], OkTopkConfig(density=0.01), n)
    thr = float(torch.topk(x.abs(), k).values[-1])
    pick = (x.abs() >= thr) & (x != 0)
    assert st.last_local_count == int(pick.sum())
    assert torch.equal(outs[0], torch.where(pick, x, torch.zeros(n)))          # P = 1: the picks are the result
    assert torch.equal(st.residual, torch.where(pick, torch.zeros(n), x))


def test_oracle_merge_is_tie_inclusive_and_drops_cancelled_sums():
    from oktopk_b200.parallel.oracle import merge_topk
    a = (torch.tensor([0, 1, 2, 3]), torch.tensor([1.0, -1.0, 2.0, 0.5]))
    b = (torch.tensor([1, 2, 4, 5]), torch.tensor([1.0, 1.0, -1.0, 1.0]))
    idx, val = merge_topk(a, b, 2, 8)          # sums: 0:1, 1:0 (cancelled), 2:3, 3:0.5, 4:-1, 5:1
    assert idx.tolist() == [0, 2, 4, 5] and val.tolist() == [1.0, 3.0, -1.0, 1.0]   # k-th magnitude 1.0: all ties kept
    idx, val = merge_topk(a, (torch.tensor([1]), torch.tensor([1.0])), 8, 8)
    assert idx.tolist() == [0, 2, 3] and val.tolist() == [1.0, 2.0, 0.5]


@pytest.mark.parametrize("kind", TIED)
def test_oracle_topkdsa_clears_k_minus_above_tied_residuals(kind):
    from oktopk_b200.config import OkTopkConfig
    n = 20_000
    k = int(n * 0.01)
    x = gen(kind, n, 4)
    _, st = _oracle_run("topkDSA", [x], OkTopkConfig(density=0.01), n)
    thr = float(torch.topk(x.abs(), k).values[-1])
    tie = (x.abs() == thr) & (x != 0)
    assert int((st.residual[tie] == 0).sum()) == k - int((x.abs() > thr).sum())
    assert torch.equal(st.residual[~tie], torch.where(x.abs() > thr, torch.zeros(n), x)[~tie])


@pytest.mark.parametrize("first", ["zeros", "zeros95"])
def test_oracle_cap_holds_after_a_zero_threshold(first):
    """An exact call that finds fewer than k non-zeros carries a threshold of 0; the reuse calls after it must still
    ship at most overselect_cap * k entries (DESIGN: whatever the staleness)."""
    from oktopk_b200.config import OkTopkConfig
    n = 100_000
    k = int(n * 0.1)
    cfg = OkTopkConfig(density=0.1, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=8,
                       overselect_cap=2.0)
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    states = [SparseState(n, 1)]
    counts = []
    for it in range(4):
        x = gen(first, n, 0) if it == 0 else gen("bf16", n, it)
        run_oracle("oktopk", [x], states, cfg)
        counts.append(states[0].last_local_count)
        if it == 0:
            assert states[0].local_thr == 0.0
    assert all(c <= 2 * k for c in counts), counts
    assert all(c > 0 for c in counts[1:]), counts


# ------------------------------------------------------------------------------------------------ CPU: dist path (gloo)
def _dist_worker(rank, P, name, kind, n, iters, cfg_kw):
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.algorithms import sparse_allreduce
    from oktopk_b200.parallel.state import SparseState
    from oktopk_b200.parallel.world import World
    w = World()
    cfg = OkTopkConfig(**cfg_kw)
    st = SparseState(n, P)
    outs, counts = [], []
    for it in range(iters):
        g = _dist_grad(kind, it, rank, n)
        sparse_allreduce(name, g, st, cfg, w)
        outs.append(g.clone())
        counts.append(st.last_local_count)
    return outs, st.residual.clone(), counts


def _dist_grad(kind, it, rank, n):
    if kind == "zero_first":                 # an all-zero exact call, then bf16-valued reuse calls
        return torch.zeros(n) if it == 0 else gen("bf16", n, 100 * it + rank)
    return gen(kind, n, 100 * it + rank)


@pytest.mark.parametrize("name,kind", [("topkA", "bf16"), ("topkA", "one_mag"), ("topkA2", "bf16"),
                                       ("topkA2", "zeros95"), ("gtopk", "bf16"), ("gtopk", "one_mag"),
                                       ("topkDSA", "bf16"), ("oktopk", "zero_first"), ("oktopk", "bf16")])
def test_dist_path_matches_oracle_on_ties_and_zero_thresholds(name, kind):
    """backend='dist' on gloo, P = 2: bitwise the oracle's result, residual and local counts, with the tie-inclusive
    picks, the TopkDSA clear count and the zero-threshold recompute."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    P, n, iters = 2, 6000, 4
    cfg_kw = dict(density=0.02, local_recompute_interval=4, global_recompute_interval=4, repartition_interval=4,
                  overselect_cap=2.0)
    got = run_distributed(_dist_worker, P, (name, kind, n, iters, cfg_kw), backend="gloo", timeout=240)
    cfg = OkTopkConfig(**cfg_kw)
    states = [SparseState(n, P) for _ in range(P)]
    k = int(n * 0.02)
    for it in range(iters):
        ref = run_oracle(name, [_dist_grad(kind, it, r, n) for r in range(P)], states, cfg)
        for r in range(P):
            assert torch.equal(got[r][0][it], ref[r]), "%s it %d rank %d differs from the oracle" % (name, it, r)
            assert got[r][2][it] == states[r].last_local_count, (it, r, got[r][2][it], states[r].last_local_count)
            if name == "oktopk":
                assert states[r].last_local_count <= 2 * k, (it, r, states[r].last_local_count)
    for r in range(P):
        assert torch.equal(got[r][1], states[r].residual), "residual of rank %d differs" % r


# ------------------------------------------------------------------------------------------------ two GPUs
def _mg_grad(kind, it, rank, n):
    """Rank 1 holds -(rank 0) on every third index, so those sums cancel to exactly 0.0; elsewhere independent."""
    base = gen(kind, n, 1000 * it)
    own = gen(kind, n, 1000 * it + 1 + rank)
    if rank == 0:
        return torch.where(torch.arange(n) % 3 == 0, base, own)
    return torch.where(torch.arange(n) % 3 == 0, -base, own)


def _mg_worker(rank, P, kind, n, iters, cfg_kw):
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    w = World()
    eng = CudaBucketEngine(n, OkTopkConfig(**cfg_kw), w, name="t")
    outs, stats = [], []
    for it in range(iters):
        eng.grad.copy_(_mg_grad(kind, it, rank, n).cuda())
        torch.cuda.synchronize()
        w.barrier()
        eng.reduce("oktopk")
        torch.cuda.synchronize()
        outs.append(eng.grad.cpu().clone())
        stats.append(eng.stats())
    res = eng.residual.cpu().clone()
    w.barrier()
    eng.close()
    return outs, res, stats


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.parametrize("mode", ["list", "scan"])
@pytest.mark.parametrize("kind", ["fp16", "bf16"])
def test_oktopk_two_gpus_cancelling_sums_match_oracle(kind, mode):
    """P = 2 with sums that cancel to exactly 0.0 (an index reaches the first-touch candidate list twice) and
    bf16 / fp16-valued gradients: bitwise the oracle's result and residual on both ranks."""
    from oktopk_b200.config import OkTopkConfig
    from oktopk_b200.parallel.oracle import run_oracle
    from oktopk_b200.parallel.state import SparseState
    P, n, iters = 2, 300_001, 6
    cfg_kw = dict(density=0.01, local_recompute_interval=3, global_recompute_interval=3, repartition_interval=3,
                  gselect_mode=mode, overselect_cap=2.0)
    got = run_distributed(_mg_worker, P, (kind, n, iters, cfg_kw), backend="nccl", timeout=600)
    cfg = OkTopkConfig(**cfg_kw)
    states = [SparseState(n, P) for _ in range(P)]
    for it in range(iters):
        ref = run_oracle("oktopk", [_mg_grad(kind, it, r, n) for r in range(P)], states, cfg)
        for r in range(P):
            bad = int((got[r][0][it] != ref[r]).sum())
            assert bad == 0, "it %d rank %d: %d mismatches, stats %s" % (it, r, bad, got[r][2][it])
            assert got[r][2][it]["local_count"] == states[r].last_local_count
    for r in range(P):
        assert int((got[r][1] != states[r].residual).sum()) == 0, "residual mismatch rank %d" % r
