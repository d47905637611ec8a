"""The fused softmax + CTC loss (``csrc/ctc.cu``, ``ops/fused_ctc.py``) on the GPU: loss and logits' gradient against
``F.ctc_loss`` in float64 on the CPU, no worse than the stock fp32 op on the GPU, with int32 and int64 targets, C from 1
to 128, Ln on either side of every warp boundary up to 2047, batches past 32 utterances and blank labels; a single
alignment against its closed form; the edge cases of the kernels' header (zero_infinity, frames past Tn, a bad label or
length, Ln = 0, Tn = 0, a -inf logit); the loss scale and an fp16 overflow; determinism; no host synchronisation and
CUDA-graph replay; launch counts; the whole DeepSpeech model; and Trainer steps against stock."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oktopk_b200.models import create_net
from oktopk_b200.ops import ext
from oktopk_b200.ops.fused_ctc import ctc_loss

pytestmark = pytest.mark.gpu

C = 29


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _launches():
    return ext.LAUNCH_COUNT.get("ctc_forward", 0), ext.LAUNCH_COUNT.get("ctc_backward", 0)


def _stock(x, targets, tn, ln, reduction="sum"):
    return F.ctc_loss(F.log_softmax(x, -1).float(), targets.long(), tn.long(), ln.long(), blank=0,
                      reduction=reduction, zero_infinity=True)


def _need(labels):
    """Frames the labels need: one each, plus a blank between equal neighbours."""
    return len(labels) + sum(1 for a, b in zip(labels, labels[1:]) if a == b)


def _path(labels):
    """The one alignment of `labels` in _need(labels) frames: each label once, a blank between equal neighbours."""
    out = []
    for j, c in enumerate(labels):
        if j and c == labels[j - 1]:
            out.append(0)
        out.append(c)
    return out


def _labels(L, g, nc=C, distinct=False):
    """L random labels in [1, nc), with equal neighbours unless `distinct`."""
    lab = torch.randint(1, nc, (L,), generator=g).tolist() if nc > 1 else []
    for j in range(1, L if distinct else 0):
        if lab[j] == lab[j - 1]:
            lab[j] = lab[j] % (nc - 1) + 1
    return lab


def _batch(N, T, seed, infeasible=False, nc=C, labels=None, tn=None, targets=torch.int64):
    """Logits [T, N, nc] and a batch: by default mixed Tn (the first utterance full length), Ln from 0 up to
    feasibility, runs of repeated labels, and with `infeasible` one utterance that cannot be aligned.  `labels` (one
    list per utterance; Tn defaults to T) and `tn` replace the drawn ones; `targets` is the targets' dtype."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(T, N, nc, generator=g) * 2
    if tn is None:
        tn = [T] * N if labels is not None else [T] + [int(torch.randint(1, T + 1, (1,), generator=g)) for _ in range(N - 1)]
    if labels is None:
        labels = []
        for n in range(N):
            cap = tn[n]
            L = int(torch.randint(0, cap + 1, (1,), generator=g)) if n else min(cap, 33)
            lab = _labels(L, g, nc)
            if L >= 4:
                lab[1] = lab[2] = lab[3] = lab[0]              # a run of repeats
            while lab and _need(lab) > cap:
                lab.pop()
            if infeasible and n == N - 1:                    # cap repeats need 2 cap - 1 > cap frames
                lab = [7] * cap if cap >= 2 else [3, 4]
            labels.append(lab)
    tgts = [c for lab in labels for c in lab]
    return (x, torch.tensor(tgts, dtype=targets), torch.tensor(tn, dtype=torch.int32),
            torch.tensor([len(lab) for lab in labels], dtype=torch.int32))


def _fused(x, targets, tn, ln, g=1.0):
    xi = x.detach().clone().requires_grad_(True)
    loss = ctc_loss(xi, targets, tn, ln)
    (dx,) = torch.autograd.grad(loss, xi, torch.tensor(g, device=loss.device))
    return loss.detach(), dx


def _ctc64(x, targets, tn, ln):
    """F.ctc_loss in float64 on the CPU, on log_softmax of the widened logits (no .float() in between)."""
    return F.ctc_loss(F.log_softmax(x.double().cpu(), -1), targets.cpu().long(), tn.cpu().long(), ln.cpu().long(),
                      blank=0, reduction="sum", zero_infinity=True)


def _ref(x, targets, tn, ln):
    xi = x.detach().double().cpu().requires_grad_(True)
    loss = _ctc64(xi, targets, tn, ln)
    (dx,) = torch.autograd.grad(loss, xi)
    return loss.detach(), dx


def _stock_gpu(x, targets, tn, ln):
    xi = x.detach().float().cuda().requires_grad_(True)
    loss = _stock(xi, targets.cuda(), tn.cuda(), ln.cuda())
    (dx,) = torch.autograd.grad(loss, xi)
    return loss.detach(), dx


DTYPES = [torch.float32, torch.bfloat16, torch.float16]
TARGETS = [torch.int32, torch.int64]
RND = {torch.float32: 0.0, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}   # dx's rounding to x's type


def _fused_fast(x, targets, tn, ln):
    """_fused, asserting that the kernels ran: two launches forward, one backward."""
    n0 = _launches()
    lf, df = _fused(x.cuda(), targets.cuda(), tn, ln)
    n1 = _launches()
    assert (n1[0] - n0[0], n1[1] - n0[1]) == (2, 1)
    assert df.dtype == x.dtype
    return lf, df


def _ref_alpha(x, targets, tn, ln):
    """The summed loss of feasible utterances by the plain α recursion in float64 on the CPU, without torch's CTC, and
    its gradient by autograd (-1e300 stands for log 0, so that no gradient is NaN)."""
    xi = x.detach().double().cpu().requires_grad_(True)
    lp = F.log_softmax(xi, -1)
    loss, off = 0.0, 0
    for n in range(x.shape[1]):
        lab = targets[off:off + int(ln[n])].tolist()
        off += len(lab)
        ext = [0] + [v for c in lab for v in (c, 0)]
        skip = torch.tensor([s >= 3 and s % 2 == 1 and ext[s] != ext[s - 2] for s in range(len(ext))])
        neg = torch.full((len(ext),), -1e300, dtype=torch.float64)
        a = torch.cat([torch.zeros(1, dtype=torch.float64), neg[1:]])       # before t = 0: the start state
        for t in range(int(tn[n])):
            a1 = torch.cat([neg[:1], a[:-1]])
            a2 = torch.where(skip, torch.cat([neg[:2], a[:-2]]), neg)
            a = torch.logsumexp(torch.stack([a, a1, a2]), 0) + lp[t, n, ext]
        loss = loss - torch.logsumexp(a[-2:], 0)
    (dx,) = torch.autograd.grad(loss, xi)
    return loss.detach(), dx


def _check_against_float64(x, targets, tn, ln, nan_frames=(), ref=_ref):
    """The fused loss and dx of x (on the host, in its own dtype) against float64 on the CPU (`ref`): the error is at
    most twice stock fp32 GPU's, plus dx's rounding to x's type and a 1e-5 floor.  On `nan_frames`, (t, n) pairs, dx is
    NaN in every class, as float64's is; frames past Tn get exactly 0.  Returns the fused loss and dx."""
    lf, df = _fused_fast(x, targets, tn, ln)
    lr, dr = ref(x, targets, tn, ln)
    ls, ds = _stock_gpu(x, targets, tn, ln)
    el, es_l = abs(lf.double().cpu() - lr).item(), abs(ls.double().cpu() - lr).item()
    assert el <= 2 * es_l + 1e-5 * max(1.0, abs(lr.item())), (el, es_l, lr.item())
    df64, ds = df.cpu().double(), ds.cpu().double()
    keep = torch.ones(x.shape[:2], dtype=torch.bool)
    for t, n in nan_frames:
        assert torch.isnan(df64[t, n]).all() and torch.isnan(dr[t, n]).all(), (t, n)
        keep[t, n] = False
    ef = (df64 - dr).abs()[keep]
    es = (ds - dr).abs()[keep].max().item()
    tol = RND[x.dtype] * dr.abs()[keep] + 2 * es + 1e-5
    assert bool((ef <= tol).all()), (ef.max().item(), es)
    for n in range(x.shape[1]):                               # frames past Tn: exactly 0
        assert torch.all(df[int(tn[n]):, n] == 0)
    return lf, df


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("N,T", [(1, 1), (2, 2), (2, 48), (5, 48), (1, 198), (2, 198), (5, 198), (2, 400), (5, 400)])
def test_loss_and_gradient_against_float64(N, T, dtype, targets):
    x, tg, tn, ln = _batch(N, T, seed=N * 1000 + T, infeasible=T >= 2 and N >= 2, targets=targets)
    _check_against_float64(x.to(dtype), tg, tn, ln)           # the reference sees the same (widened) values


def _multiwarp_batch(seed, targets=torch.int64):
    """Utterances of 1023, 64, 0 and 500 labels (S = 2047, 129, 1, 1001: 16, 2, 1 and 8 warps), T = 1200."""
    g = torch.Generator().manual_seed(seed)
    labels = [_labels(L, g) for L in (1023, 64, 0, 500)]
    return _batch(4, 1200, seed, labels=labels, tn=[1200, 300, 50, 1100], targets=targets)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("case", ["mixed", "multiwarp"])
def test_int32_and_int64_targets_are_bitwise_equal(case, dtype):
    out = []
    for targets in TARGETS:
        x, tg, tn, ln = _batch(5, 198, seed=16, targets=targets) if case == "mixed" else _multiwarp_batch(23, targets)
        out.append(_fused_fast(x.to(dtype), tg, tn, ln))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nc", [1, 2, 31, 32, 33, 64, 127, 128])
def test_class_counts_against_float64(nc, dtype):
    """C from 1 to kCtcMaxC, the labels reaching the top classes (96..127 at C = 128: the last 32-wide column of the
    backward's per-class rows).  C = 1 holds only the blank, so Ln = 0."""
    g = torch.Generator().manual_seed(100 + nc)
    top = list(range(max(1, nc - 32), nc))
    labels = [top[::-1], _labels(20, g, nc), [], top[-5:] + [1] + top[:5]] if nc > 1 else [[], [], [], []]
    x, tg, tn, ln = _batch(4, 70, seed=nc, nc=nc, labels=labels, tn=[70, 50, 30, 45])
    _check_against_float64(x.to(dtype), tg, tn, ln)


# Ln around the α / β warp boundaries: S = 2 Ln + 1 states, 128 per warp, so Ln = 63 / 64 is one warp / two, 127 / 128
# two / three, 191 / 192 two / four ... and 2047 = kCtcMaxTargets all 32 warps (S = 4095).
LN_EDGES = [63, 64, 127, 128, 191, 192, 1023, 1024, 2047]


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("Ln,dtype", [(L, dt) for L in LN_EDGES for dt in (DTYPES if L in (63, 64, 2047) else DTYPES[:1])])
def test_warp_boundaries_against_float64(Ln, dtype, targets):
    """One utterance of Ln labels.  At Ln = 2047 the labels have no equal neighbours, so that T = 2100 is feasible."""
    g = torch.Generator().manual_seed(Ln)
    lab = _labels(Ln, g, distinct=Ln == 2047)
    T = 2100 if Ln == 2047 else _need(lab) + 60
    x, tg, tn, ln = _batch(1, T, seed=Ln, labels=[lab], targets=targets)
    _check_against_float64(x.to(dtype), tg, tn, ln)


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_warp_boundaries_in_a_mixed_batch(dtype, targets):
    """Single- and multi-warp utterances side by side, each at its own target and α offset, Tn from need to need + 60."""
    g = torch.Generator().manual_seed(24)
    labels = [_labels(L, g) for L in (63, 1023, 0, 128, 192, 64, 127)]
    tn = [min(1200, _need(lab) + 10 * n) for n, lab in enumerate(labels)]
    x, tg, tn, ln = _batch(7, 1200, seed=24, labels=labels, tn=tn, targets=targets)
    _check_against_float64(x.to(dtype), tg, tn, ln)


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Ln,pair,equal", [(128, 63, True), (128, 63, False), (1100, 1023, True), (1100, 1023, False),
                                           (2047, None, None)])
def test_exactly_one_alignment(Ln, pair, equal, dtype, targets):
    """Tn = need: one alignment, so the posterior is one-hot along it, dx = softmax(x) - onehot(path) and the loss is
    -sum log softmax along the path, in float64 without torch's CTC.  Labels `pair` and `pair` + 1 sit in states 2 pair
    + 1 and 2 pair + 3 on either side of a warp boundary; equal, the α skip into the second and the β skip out of the
    first must be off.  Tn = need - 1 is infeasible: loss and dx exactly 0."""
    g = torch.Generator().manual_seed(Ln + 7 * bool(equal))
    lab = _labels(Ln, g)
    if pair is not None:
        lab[pair + 1] = lab[pair] if equal else lab[pair] % (C - 1) + 1
    path = _path(lab)
    T = len(path)
    assert T == _need(lab)
    x, tg, tn, ln = _batch(1, T, seed=Ln, labels=[lab], targets=targets)
    x = x.to(dtype)
    lf, df = _fused_fast(x, tg, tn, ln)
    lp = F.log_softmax(x[:, 0].double(), -1)
    at = torch.arange(T)
    lr = -lp[at, path].sum().item()
    dr = lp.exp()
    dr[at, path] -= 1
    assert abs(lf.item() - lr) <= (1e-5 + T * 2.0 ** -24) * max(1.0, abs(lr)), (lf.item(), lr)
    ef = (df[:, 0].cpu().double() - dr).abs()
    assert bool((ef <= RND[dtype] * dr.abs() + 2e-6).all()), ef.max().item()
    l0, d0 = _fused_fast(x[:-1], tg, tn - 1, ln)
    assert l0.item() == 0 and torch.all(d0 == 0)


@pytest.mark.parametrize("scale", [1, 8])
def test_max_targets_deterministic_and_against_float64(scale):
    """Ln = kCtcMaxTargets, T = 2100, fp32 logits, and x 8 (peaked): 2100 steps of the log-space recursion on all 32
    warps, bitwise the same twice."""
    g = torch.Generator().manual_seed(25)
    x, tg, tn, ln = _batch(1, 2100, seed=25, labels=[_labels(2047, g, distinct=True)], targets=torch.int32)
    x = x * scale
    lf, df = _check_against_float64(x, tg, tn, ln)
    l2, d2 = _fused_fast(x, tg, tn, ln)
    assert torch.equal(lf, l2) and torch.equal(df, d2)


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("N,T", [(32, 40), (33, 40), (64, 40), (257, 14)])
def test_large_batches_against_float64(N, T, targets):
    """More than 32 utterances: the loss's reduction adds several per lane."""
    x, tg, tn, ln = _batch(N, T, seed=N, targets=targets)
    _check_against_float64(x, tg, tn, ln)


def test_infeasible_utterance_past_32_leaves_the_others_unchanged():
    x, targets, tn, ln = _batch(64, 40, seed=26)
    labels = [lab.tolist() for lab in torch.split(targets, ln.tolist())]
    keep = [n for n in range(64) if n != 40]
    l63, d63 = _fused_fast(x[:, keep].contiguous(), torch.tensor([c for n in keep for c in labels[n]]), tn[keep],
                           ln[keep])
    labels[40] = [6] * (int(tn[40]) + 1)                     # more labels than frames
    tb = torch.tensor([c for lab in labels for c in lab])
    lnb = torch.tensor([len(lab) for lab in labels], dtype=torch.int32)
    l64, d64 = _fused_fast(x, tb, tn, lnb)
    assert torch.all(d64[:, 40] == 0)
    assert torch.equal(d64[:, keep], d63)
    assert l64.item() == pytest.approx(l63.item(), rel=1e-6)
    assert _stock(x.double(), tb, tn, lnb, reduction="none")[40].item() == 0 and torch.isfinite(l64)


@pytest.mark.parametrize("targets", TARGETS)
@pytest.mark.parametrize("dtype", DTYPES)
def test_blank_label_in_targets_against_float64(dtype, targets):
    """Label 0 among the targets, as torch accepts: class 0's posterior adds the blank states and those odd states.
    The reference is the plain α recursion: torch's CPU CTC backward sets class 0's posterior at an utterance's last
    frame, rather than adding to it, when the last label is 0.  Elsewhere the two references agree."""
    g = torch.Generator().manual_seed(27)
    lab = _labels(12, g)
    lab[2] = lab[5] = lab[6] = 0
    labels = [[3, 0, 5, 0, 0, 7, 0], [0], [0, 0, 0], lab]
    x, tg, tn, ln = _batch(4, 40, seed=27, labels=labels, tn=[40, 10, 25, 33], targets=targets)
    x = x.to(dtype)
    la, da = _ref_alpha(x, tg, tn, ln)
    lr, dr = _ref(x, tg, tn, ln)
    assert la.item() == pytest.approx(lr.item(), rel=1e-12)
    for n, lab in enumerate(labels):
        last = int(tn[n]) - (lab[-1] == 0)
        assert torch.allclose(da[:last, n], dr[:last, n], rtol=0, atol=1e-12), n
    _check_against_float64(x, tg, tn, ln, ref=_ref_alpha)


def test_zero_infinity_leaves_the_others_unchanged():
    x, targets, tn, ln = _batch(4, 60, seed=11)
    bad_t = torch.cat([targets, torch.tensor([6, 6, 6, 6])])   # 4 repeats need 7 frames; the extra utterance has 5
    bad_tn = torch.cat([tn, torch.tensor([5], dtype=torch.int32)])
    bad_ln = torch.cat([ln, torch.tensor([4], dtype=torch.int32)])
    xb = torch.cat([x, torch.randn(60, 1, C)], dim=1)
    l4, d4 = _fused(x.cuda(), targets.cuda(), tn, ln)
    l5, d5 = _fused(xb.cuda(), bad_t.cuda(), bad_tn, bad_ln)
    assert torch.all(d5[:, 4] == 0)
    assert torch.equal(d5[:, :4], d4)
    assert l5.item() == pytest.approx(l4.item(), rel=1e-6)
    per = _stock(xb.double(), bad_t, bad_tn, bad_ln, reduction="none")
    assert per[4].item() == 0 and torch.isfinite(l5)


def test_frames_past_tn_are_never_read():
    g = torch.Generator().manual_seed(12)
    x = torch.randn(80, 3, C, generator=g)
    tn = torch.tensor([80, 50, 70], dtype=torch.int32)
    ln = torch.tensor([10, 12, 8], dtype=torch.int32)
    targets = torch.randint(1, C, (30,), generator=g)
    l0, d0 = _fused(x.cuda(), targets.cuda(), tn, ln)
    xp = x.clone()
    xp[50:, 1] = float("nan")
    xp[60:, 1, 3] = float("inf")
    l1, d1 = _fused(xp.cuda(), targets.cuda(), tn, ln)
    assert torch.equal(l0, l1) and torch.equal(d0, d1)
    assert torch.all(d1[50:, 1] == 0) and torch.isfinite(d1).all()
    assert torch.all(d1[70:, 2] == 0) and d1[:50, 1].abs().max() > 0


def test_label_out_of_range_is_nan_for_that_utterance():
    x, targets, tn, ln = _batch(3, 40, seed=13)
    ln = torch.tensor([3, 4, 2], dtype=torch.int32)
    targets = torch.tensor([1, 2, 3, 4, C, 5, 6, 7, 8])         # the second utterance holds C
    tn = torch.tensor([40, 30, 20], dtype=torch.int32)
    loss, dx = _fused(x.cuda(), targets.cuda(), tn, ln)
    assert torch.isnan(loss)
    assert torch.isnan(dx[:30, 1]).all() and torch.all(dx[30:, 1] == 0)
    assert torch.isfinite(dx[:, 0]).all() and torch.isfinite(dx[:, 2]).all()
    ref = _fused(x[:, [0, 2]].contiguous().cuda(), torch.tensor([1, 2, 3, 7, 8]).cuda(), torch.tensor([40, 20], dtype=torch.int32),
                 torch.tensor([3, 2], dtype=torch.int32))[1]
    assert torch.equal(dx[:, 0], ref[:, 0]) and torch.equal(dx[:, 2], ref[:, 1])


@pytest.mark.parametrize("case", ["negative", "past_nt"])
def test_bad_target_length_is_nan_from_that_utterance_on(case):
    """A negative Ln at utterance m, or one that takes sum Ln past nt, leaves the target offsets of m and every later
    utterance undefined: they are NaN on their frames t < Tn; the ones before m are unchanged."""
    x, targets, tn, ln = _batch(5, 50, seed=28)
    m = 2
    bad = ln.clone()
    bad[m] = -1 if case == "negative" else int(ln[m]) + targets.numel()
    l0, d0 = _fused_fast(x, targets, tn, ln)
    lb, db = _fused_fast(x, targets, tn, bad)
    assert torch.isnan(lb)
    assert torch.equal(db[:, :m], d0[:, :m])
    for n in range(m, 5):
        assert torch.isnan(db[:int(tn[n]), n]).all() and torch.all(db[int(tn[n]):, n] == 0), n


def test_device_input_length_past_t_is_nan_for_that_utterance():
    x, targets, tn, ln = _batch(3, 50, seed=29)
    bad = tn.clone()
    bad[1] = 53
    l0, d0 = _fused_fast(x, targets, tn.cuda(), ln)
    lb, db = _fused_fast(x, targets, bad.cuda(), ln)
    assert torch.isnan(lb)
    assert torch.isnan(db[:, 1]).all()
    assert torch.equal(db[:, 0], d0[:, 0]) and torch.equal(db[:, 2], d0[:, 2])


@pytest.mark.parametrize("dtype", DTYPES)
def test_minus_inf_logit_keeps_the_loss_and_makes_its_frames_nan(dtype):
    """The frame's log-sum-exp skips a -inf logit, so the loss stays finite and equals float64; the gradient is NaN in
    every class of exactly the frames that hold one, as float64 torch's is.  One -inf at a class of the utterance's
    labels, one at another class."""
    x, targets, tn, ln = _batch(3, 60, seed=30, labels=[[1, 2, 3, 4], [5, 6, 5, 7, 8], [9]], tn=[60, 45, 30])
    x = x.to(dtype)
    x[10, 1, 6] = x[20, 1, 11] = float("-inf")
    lf, _ = _check_against_float64(x, targets, tn, ln, nan_frames=[(10, 1), (20, 1)])
    assert torch.isfinite(lf)


def test_empty_targets_and_zero_length_inputs():
    g = torch.Generator().manual_seed(14)
    x = torch.randn(30, 4, C, generator=g)
    targets = torch.tensor([4, 9], dtype=torch.int64)
    tn = torch.tensor([30, 0, 0, 17], dtype=torch.int32)
    ln = torch.tensor([0, 0, 2, 0], dtype=torch.int32)            # Ln = 0 twice, Tn = 0 with and without labels
    lf, df = _fused(x.cuda(), targets.cuda(), tn, ln)
    lr, dr = _ref(x, targets, tn, ln)
    assert lf.item() == pytest.approx(lr.item(), rel=1e-5)
    assert (df.cpu().double() - dr).abs().max().item() < 1e-5
    assert torch.all(df[:, 1] == 0) and torch.all(df[:, 2] == 0) and torch.all(df[17:, 3] == 0)
    lf0, df0 = _fused(x.cuda(), targets[:0].cuda(), tn, torch.zeros(4, dtype=torch.int32))   # no targets at all
    lr0, dr0 = _ref(x, targets[:0], tn, torch.zeros(4, dtype=torch.int32))
    assert lf0.item() == pytest.approx(lr0.item(), rel=1e-5) and (df0.cpu().double() - dr0).abs().max() < 1e-5


def test_loss_scale_and_fp16_overflow():
    x, targets, tn, ln = _batch(2, 100, seed=15)
    _, d1 = _fused(x.cuda(), targets.cuda(), tn, ln)
    _, d2 = _fused(x.cuda(), targets.cuda(), tn, ln, g=1024.0)
    assert torch.equal(d2, d1 * 1024)
    _, dh = _fused(x.half().cuda(), targets.cuda(), tn, ln, g=2.0 ** 17)
    assert torch.isinf(dh).any()
    assert not torch.isnan(dh).any()


def test_deterministic():
    x, targets, tn, ln = _batch(5, 198, seed=16)
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        outs = [_fused(x.cuda(), targets.cuda(), tn.cuda(), ln.cuda()) for _ in range(2)]
    finally:
        torch.use_deterministic_algorithms(old)
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_no_host_synchronisation():
    x, targets, tn, ln = _batch(2, 198, seed=17)
    xs = x.cuda().requires_grad_(True)
    ts, tns, lns = targets.cuda(), tn.cuda(), ln.cuda()
    torch.cuda.synchronize()
    old = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = ctc_loss(xs, ts, tns, lns)
        (dx,) = torch.autograd.grad(loss, xs)
    finally:
        torch.cuda.set_sync_debug_mode(old)
    assert torch.isfinite(dx).all()


def test_graph_replay_on_new_logits_and_lengths():
    x, targets, tn, ln = _batch(2, 198, seed=17)
    xs = x.cuda().requires_grad_(True)
    ts, tns, lns = targets.cuda(), tn.cuda(), ln.cuda()

    def run():
        loss = ctc_loss(xs, ts, tns, lns)
        (dx,) = torch.autograd.grad(loss, xs)
        return loss, dx

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss_s, dx_s = run()
    # new logits and lengths (the same total of targets), copied into the static inputs
    x2 = _batch(2, 198, seed=18)[0]
    tn2 = torch.tensor([150, 198], dtype=torch.int32)
    k = int(ln.sum()) // 2
    ln2 = torch.tensor([int(ln.sum()) - k, k], dtype=torch.int32)
    with torch.no_grad():
        xs.copy_(x2)
    tns.copy_(tn2)
    lns.copy_(ln2)
    graph.replay()
    le, de = _fused(x2.cuda(), targets.cuda(), tn2, ln2)
    assert torch.equal(loss_s, le) and torch.equal(dx_s, de)


def _an4_loss(out, targets, out_lens, tsizes, kind):
    if kind == "fused":
        return ctc_loss(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)
    if kind == "ref":
        return _ctc64(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)
    return _stock(out.transpose(0, 1), targets, out_lens, tsizes) / out.size(0)


@pytest.mark.parametrize("fuse_lstm", [False, True])
def test_whole_model_against_float64(fuse_lstm):
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4")
    ref = copy.deepcopy(net).double()
    stock = net.cuda()
    fused = copy.deepcopy(stock)
    fused.fuse_ctc = True
    stock.fuse_lstm = fused.fuse_lstm = fuse_lstm
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 400, generator=g)
    lens = torch.tensor([400, 290], dtype=torch.int32)
    tsizes = torch.tensor([20, 14])
    targets = torch.randint(1, 29, (int(tsizes.sum()),), generator=g)
    res = {}
    for name, m, dev, dt in (("ref", ref, "cpu", torch.float64), ("stock", stock, "cuda", torch.float32),
                             ("fused", fused, "cuda", torch.float32)):
        m.train()
        n0 = _launches()
        out, out_lens = m(x.to(dev, dt), lens)
        loss = _an4_loss(out, targets.to(dev), out_lens, tsizes.to(dev), name)
        loss.backward()
        assert (_launches() != n0) == (name == "fused"), name
        res[name] = [loss.detach().cpu().double()] + [p.grad.detach().cpu().double() for p in m.parameters()]
    assert torch.isfinite(res["fused"][0])
    names = ["ctc"] + [n for n, _ in net.named_parameters()]
    for i, name in enumerate(names):
        r = res["ref"][i]
        es = (res["stock"][i] - r).abs().max().item()
        ef = (res["fused"][i] - r).abs().max().item()
        floor = 1e-5 * max(1.0, r.abs().max().item())
        assert ef <= 2 * es + floor, (name, ef, es, floor)


@pytest.mark.parametrize("precision", ["fp32", "bf16", "fp16"])
def test_trainer_steps_follow_stock(precision):
    """Five steps on the bench's AN4 batches with the fused LSTM on in both arms, stock loss against fused loss (fp16
    with dynamic loss scaling)."""
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    autocast = None if precision == "fp32" else precision
    losses = {}
    for fuse in (False, True):
        cfg = okt.preset(preset, density=0.001, warmup_iters=2)
        tr = Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                     t_total=100000, warmup=0.1, seed=0, autocast=autocast,
                     loss_scale=okt.LossScale() if precision == "fp16" else None,
                     model_kwargs={"fuse_lstm": True, "fuse_lstm_autocast": autocast is not None, "fuse_ctc": fuse})
        assert tr.net.fuse_ctc is fuse
        seq = []
        n0 = _launches()
        for i in range(5):
            batch = tuple(t.to(tr.device) for t in bench.make_batch("lstman4", i, 0, bs, 128))
            tr.net.train()
            tr.optimizer.zero_grad()
            loss, _ = tr._forward_loss(batch)
            tr.backward(loss)
            tr.update_model()
            seq.append(float(loss))
        n1 = _launches()
        assert (n1[0] - n0[0], n1[1] - n0[1]) == ((10, 5) if fuse else (0, 0))
        assert all(torch.isfinite(p).all() for p in tr.net.parameters())
        assert all(torch.isfinite(torch.tensor(seq)))
        tr.close()
        losses[fuse] = seq
    rel = 2e-2 if precision == "fp32" else 5e-2
    for a, b in zip(losses[False], losses[True]):
        assert b == pytest.approx(a, rel=rel), losses


@pytest.mark.parametrize("case", ["fp64", "wide_c", "c129", "many_targets", "padded_targets", "at_limit"])
def test_fallbacks_on_the_gpu_are_the_stock_expression(case):
    """Past the gate's limits the op is the stock expression, bitwise; at them (C = 128, nt = 2047) the kernels run."""
    g = torch.Generator().manual_seed(19)
    T, N = 12, 3
    x = torch.randn(T, N, C, generator=g)
    tn = torch.tensor([12, 9, 5], dtype=torch.int32)
    ln = torch.tensor([4, 3, 2], dtype=torch.int32)
    t = torch.randint(1, C, (9,), generator=g)
    if case == "fp64":
        x = x.double()
    elif case == "wide_c":
        x = torch.randn(T, N, 200, generator=g)
    elif case == "c129":
        x = torch.randn(T, N, 129, generator=g)
        t[0] = 128
    elif case == "many_targets":                              # 2048 targets, though each utterance's are feasible
        ln = torch.tensor([4, 3, 2041], dtype=torch.int32)
        tn = torch.tensor([12, 9, 12], dtype=torch.int32)
        t = torch.randint(1, C, (2048,), generator=g)
    elif case == "at_limit":                                  # C = 128 and 2047 targets, the last utterance infeasible
        x = torch.randn(T, N, 128, generator=g)
        ln = torch.tensor([4, 3, 2040], dtype=torch.int32)
        tn = torch.tensor([12, 9, 12], dtype=torch.int32)
        t = torch.randint(1, 128, (2047,), generator=g)
    else:
        t = torch.randint(1, C, (N, 4), generator=g)
    if case == "at_limit":
        _check_against_float64(x, t, tn, ln)
        return
    x, t = x.cuda(), t.cuda()
    outs = []
    for fused in (True, False):
        xi = x.clone().requires_grad_(True)
        n0 = _launches()
        loss = ctc_loss(xi, t, tn, ln) if fused else _stock(xi, t, tn, ln)
        loss.backward()
        assert _launches() == n0
        outs.append((loss.detach(), xi.grad))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
