"""Fused self-attention (``ops/fused_attn.py``, ``csrc/attention.cu``) on the GPU: O and d(qkv) against a float64
reference of the formula (within twice stock SDPA's error plus a few ulps) at every 64-row tile edge, on skewed score
rows and at the masks' extremes, fully masked sequences, per-slice independence, the largest grid and unaligned
inputs; the Philox dropout mask against a NumPy Philox4x32-10, read off element by element at rates up to 0.99 and past
counter 2^32; determinism, checkpoint recompute and CUDA-graph replays, fp16 overflow, the whole BERT model, a graphed
Trainer step with every fused BERT op, and the fallbacks."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

D = 64
ULPS = 8
EPS = {torch.float32: 2.0 ** -23, torch.bfloat16: 2.0 ** -7, torch.float16: 2.0 ** -10}


def philox4x32_10(ctr, key):
    """``ctr``: [n, 4] uint32 counters, ``key``: (k0, k1).  Returns [n, 4] uint32 words (Random123's round order)."""
    c = [ctr[:, i].astype(np.uint64) for i in range(4)]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    m0, m1, mask = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0xFFFFFFFF)
    for r in range(10):
        if r > 0:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & mask, (k1 + np.uint64(0xBB67AE85)) & mask
        p0, p1 = m0 * c[0], m1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & mask]
    return np.stack(c, 1).astype(np.uint32)


def test_philox_reference_known_answers():
    z = philox4x32_10(np.zeros((1, 4), np.uint32), (0, 0))
    assert [int(v) for v in z[0]] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    o = philox4x32_10(np.full((1, 4), 0xFFFFFFFF, np.uint32), (0xFFFFFFFF, 0xFFFFFFFF))
    assert [int(v) for v in o[0]] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


def seed_of(s):
    """The seed the fused op draws as its first CUDA random call after ``torch.cuda.manual_seed(s)``."""
    torch.cuda.manual_seed(s)
    return int(torch.empty(1, dtype=torch.int64, device="cuda").random_().item())


def keep_mask(seed, B, H, S, p, b0=0):
    """[B, H, S, S] bool for the sequences b0 .. b0 + B - 1: element idx = ((b H + h) S + i) S + j is kept iff word
    idx % 4 at counter idx // 4 is below floor((1-p) 2^32)."""
    from oktopk_b200.ops.fused_ln import keep_threshold
    n, lo = B * H * S * S, b0 * H * S * S
    q = np.arange(lo // 4, (lo + n + 3) // 4, dtype=np.uint64)
    ctr = np.zeros((len(q), 4), np.uint32)
    ctr[:, 0] = (q & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    ctr[:, 1] = (q >> np.uint64(32)).astype(np.uint32)
    u = seed & ((1 << 64) - 1)
    words = philox4x32_10(ctr, (u & 0xFFFFFFFF, u >> 32)).reshape(-1)[lo % 4:lo % 4 + n]
    return torch.from_numpy(words.astype(np.int64) < keep_threshold(p)).view(B, H, S, S).cuda()


# ------------------------------------------------------------------------------------------ helpers
def _counts():
    from oktopk_b200.ops import ext
    return {k: ext.LAUNCH_COUNT.get(k, 0) for k in ("attn_forward", "attn_backward")}


def _delta(n0):
    return {k: v - n0[k] for k, v in _counts().items()}


def _inputs(B, S, H, dtype, seed, lengths=None):
    g = torch.Generator("cuda").manual_seed(seed)
    qkv = torch.randn(B, S, 3 * H * D, device="cuda", generator=g).to(dtype)
    dout = torch.randn(B, S, H * D, device="cuda", generator=g).to(dtype)
    mask = None
    if lengths is not None:
        valid = torch.arange(S, device="cuda")[None, :] < torch.tensor(lengths, device="cuda")[:, None]
        mask = ((1.0 - valid.float()) * -10000.0)[:, None, None, :]
    return qkv, dout, mask


def _formula(qkv, H, mask, keep, p):
    """The torch formula in qkv's dtype (mask as given, dropout by `keep`): returns (O, d(qkv)) as a function of dout."""
    B, S, _ = qkv.shape
    q, k, v = qkv.view(B, S, 3, H, D).permute(2, 0, 3, 1, 4)
    s = q @ k.transpose(-1, -2) / D ** 0.5
    if mask is not None:
        s = s + mask
    P = torch.softmax(s, -1)
    if keep is not None:
        P = P * keep / (1.0 - p)
    return (P @ v).transpose(1, 2).reshape(B, S, H * D)


def _run(fn, qkv, dout):
    x = qkv.detach().clone().requires_grad_(True)
    o = fn(x)
    o.backward(dout)
    return o.detach(), x.grad


def _fused(qkv, dout, H, mask, p, cuda_seed=None):
    from oktopk_b200.ops.fused_attn import self_attention
    if cuda_seed is not None:
        torch.cuda.manual_seed(cuda_seed)
    return _run(lambda x: self_attention(x, H, mask, p), qkv, dout)


def _stock(qkv, dout, H, mask):
    B, S, _ = qkv.shape
    m = None if mask is None else mask.to(qkv.dtype)

    def f(x):
        q, k, v = x.view(B, S, 3, H, D).permute(2, 0, 3, 1, 4)
        return F.scaled_dot_product_attention(q, k, v, attn_mask=m).transpose(1, 2).reshape(B, S, H * D)
    return _run(f, qkv, dout)


def _err(got, want):
    return float((got.double() - want).abs().max())


def _within(got, base, want, dtype, what):
    """|got - want| <= 2 |base - want| + ULPS ulps of dtype at want's scale."""
    e, eb = _err(got, want), _err(base, want)
    tol = 2 * eb + ULPS * EPS[dtype] * float(want.abs().max())
    assert e <= tol, (what, e, eb, tol)


def _reference(qkv, dout, H, mask):
    """(O, d(qkv)) of the float64 formula and of stock SDPA in qkv's dtype."""
    ref = _run(lambda x: _formula(x, H, mask.double() if mask is not None else None, None, 0.0), qkv.double(),
               dout.double())
    return ref, _stock(qkv, dout, H, mask)


def _check(o, g, qkv, dout, H, mask, what=""):
    """The fused (o, g) of (qkv, dout, mask) at p = 0 within the criterion of _within, O and d(qkv)."""
    (od, gd), (os_, gs) = _reference(qkv, dout, H, mask)
    _within(o, os_, od, qkv.dtype, what + "O")
    _within(g, gs, gd, qkv.dtype, what + "dqkv")


DTYPES = [torch.float32, torch.bfloat16, torch.float16]
# 64-row tiles: S = 64 k - 1, 64 k, 64 k + 1 around every boundary up to 512 (64 k + 1 leaves a final query and key
# tile with one valid row), one and three heads
TILE_EDGES = [63, 64, 65, 127, 191, 192, 193, 255, 256, 257, 383, 384, 385, 447, 448, 449, 511]
SHAPES = ([(8, 128, 12), (2, 512, 16), (3, 1, 2), (3, 7, 2), (2, 100, 3), (2, 129, 2), (2, 200, 2)]
          + [(2, S, H) for S in TILE_EDGES for H in (1, 3)] + [(4, 256, 2)])


# ------------------------------------------------------------------------------------------ 1. accuracy at p = 0
@pytest.mark.parametrize("masking", ["none", "padding", "single_key", "tiles"])
@pytest.mark.parametrize("B,S,H", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_matches_float64_reference(dtype, B, S, H, masking):
    lengths = None
    if masking == "padding":
        lengths = [max(1, S - (37 * b) % S) for b in range(B)]
    elif masking == "single_key":
        lengths = [S] * B
        lengths[-1] = 1
    elif masking == "tiles":                            # whole key tiles padded: lengths 1, 63, 64, 65
        lengths = [min(S, (1, 63, 64, 65)[b % 4]) for b in range(B)]
    qkv, dout, mask = _inputs(B, S, H, dtype, B * 1000 + S + H, lengths)
    n0 = _counts()
    o, g = _fused(qkv, dout, H, mask, 0.0)
    assert _delta(n0) == {"attn_forward": 1, "attn_backward": 2}
    assert o.dtype == g.dtype == dtype and o.shape == (B, S, H * D) and g.shape == qkv.shape
    _check(o, g, qkv, dout, H, mask)


def _skewed(case, B, S, H, dtype, seed):
    """Inputs whose score rows are far from N(0, 1): see test_skewed_score_rows_match_float64_reference."""
    gen = torch.Generator("cuda").manual_seed(seed)
    x = torch.randn(B, S, 3, H, D, device="cuda", generator=gen)
    mask = None
    if case in ("rising", "falling"):
        ramp = torch.linspace(-1.0, 1.0, S, device="cuda")
        x[:, :, :2] *= 0.1
        x[:, :, 0, :, 0] = 16.0                         # s_ij ~ 16 * 20 / 8 * ramp_j: -40 .. 40 along the keys
        x[:, :, 1, :, 0] = 20.0 * (ramp if case == "rising" else ramp.flip(0))[None, :, None]
    elif case == "wide":                                # score std ~ 12: P underflows for most keys of a row
        x[:, :, :2] *= 3.5
    elif case == "off_centre":                          # scores ~ 128 +- 6: the split and lse precision in fp32
        x[:, :, :2] += 4.0
    elif case == "constant":                            # q = 0: P uniform
        x[:, :, 0] = 0.0
    elif case == "first_tile_masked":                   # the row max jumps from ~ -14427 to ~ 0 in key block 1
        mask = torch.zeros(B, 1, 1, S, device="cuda")
        mask[..., :64] = -10000.0
    dout = torch.randn(B, S, H * D, device="cuda", generator=gen).to(dtype)
    return x.reshape(B, S, 3 * H * D).to(dtype), dout, mask


@pytest.mark.parametrize("case", ["rising", "falling", "wide", "off_centre", "constant", "first_tile_masked"])
@pytest.mark.parametrize("S", [65, 256, 512])
@pytest.mark.parametrize("dtype", DTYPES)
def test_skewed_score_rows_match_float64_reference(dtype, S, case):
    """Rows whose max arrives in a late key block (rising), sits in the first one (falling), or jumps out of a masked
    first tile, so that the running max's rescale factor is far from 1; rows where most of P underflows; scores far
    from 0; and uniform rows."""
    B, H = 2, 2
    qkv, dout, mask = _skewed(case, B, S, H, dtype, 300 + S)
    o, g = _fused(qkv, dout, H, mask, 0.0)
    _check(o, g, qkv, dout, H, mask)


def _fill(name, dtype):
    return {"-inf": float("-inf"), "-1e9": -1e9, "bert": -10000.0, "f32_min": torch.finfo(torch.float32).min,
            "dtype_min": torch.finfo(dtype).min}[name]


@pytest.mark.parametrize("fill", ["-inf", "-1e9", "f32_min", "dtype_min"])
@pytest.mark.parametrize("dtype", DTYPES)
def test_extreme_partial_masks_match_float64_reference(dtype, fill):
    """Sequence 0 masks its whole first key tile, 1 every third key, 2 its two middle tiles, all with `fill`; every row
    keeps finite keys.  Stock SDPA takes the mask in qkv's type, where f32_min and -1e9 (fp16) round to -inf."""
    B, S, H = 3, 200, 2
    qkv, dout, _ = _inputs(B, S, H, dtype, 70)
    j = torch.arange(S, device="cuda")
    masked = torch.stack([j < 64, j % 3 == 0, (j >= 64) & (j < 192)])
    mask = torch.where(masked, _fill(fill, dtype), 0.0)[:, None, None, :].float()
    o, g = _fused(qkv, dout, H, mask, 0.0)
    _check(o, g, qkv, dout, H, mask)


FULL = [(d, f) for d in DTYPES for f in ("bert", "f32_min", "dtype_min") if (d, f) != (torch.float32, "dtype_min")]


@pytest.mark.parametrize("dtype,fill", FULL, ids=["%s-%s" % (str(d)[6:], f) for d, f in FULL])
def test_fully_masked_sequence_matches_float64_reference(dtype, fill):
    """Sequence 1 masked at every key with a finite `fill`, between a full and a padded one.  Where fill * log2 e
    overflows fp32 (f32_min, bf16's minimum), float64 absorbs every score into the fill, so its softmax is uniform and
    O the plain average of V: the fused result must be that within ULPS ulps.  Stock SDPA is no yardstick there (it may
    give NaN).  Below that (-10000, fp16's -65504) fp32 holds a biased score only to 2^-24 of its magnitude, 2^-11 at
    -10000 log2 e, which float64's exact scores are beyond; the criterion is stock's, which is finite there."""
    B, S, H = 3, 200, 2
    qkv, dout, mask = _inputs(B, S, H, dtype, 80, [S, S, 150])
    v = _fill(fill, dtype)
    mask[1] = v
    o, g = _fused(qkv, dout, H, mask, 0.0)
    for b in (0, 2):
        _check(o[b:b + 1], g[b:b + 1], qkv[b:b + 1], dout[b:b + 1], H, mask[b:b + 1], "seq %d " % b)
    x, dy, m = qkv[1:2], dout[1:2], mask[1:2]
    if abs(v) * np.log2(np.e) > torch.finfo(torch.float32).max:
        (od, gd), _ = _reference(x, dy, H, m)
        mean_v = x.double().view(S, 3, H, D)[:, 2].mean(0).reshape(1, 1, H * D).expand(1, S, H * D)
        torch.testing.assert_close(od, mean_v, rtol=1e-12, atol=1e-12)
        for got, want, what in ((o[1:2], od, "O"), (g[1:2], gd, "dqkv")):
            tol = ULPS * EPS[dtype] * float(want.abs().max())
            assert _err(got, want) <= tol, (what, _err(got, want), tol)
    else:
        _check(o[1:2], g[1:2], x, dy, H, m, "seq 1 ")


@pytest.mark.parametrize("dtype", DTYPES)
def test_all_inf_sequence_is_nan_and_leaves_the_others_alone(dtype):
    B, S, H = 3, 200, 2
    qkv, dout, mask = _inputs(B, S, H, dtype, 90, [S, 150, 77])
    o0, g0 = _fused(qkv, dout, H, mask, 0.0)
    mask[1] = float("-inf")
    o, g = _fused(qkv, dout, H, mask, 0.0)
    assert torch.isnan(o[1]).all() and torch.isnan(g[1]).all()
    rest = [0, 2]
    assert torch.isfinite(o[rest]).all() and torch.isfinite(g[rest]).all()
    assert torch.equal(o[rest], o0[rest]) and torch.equal(g[rest], g0[rest])


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_16bit_mask_is_the_fp32_mask_of_its_values(dtype):
    B, S, H = 3, 130, 2
    qkv, dout, _ = _inputs(B, S, H, dtype, 95)
    gen = torch.Generator("cuda").manual_seed(96)
    mask = torch.randn(B, 1, 1, S, device="cuda", generator=gen) * 3
    mask[0, ..., 100:] = -10000.0                       # -9984 in bf16
    mask[2, ..., :70] = torch.finfo(dtype).min
    mask = mask.to(dtype)
    n0 = _counts()
    a = _fused(qkv, dout, H, mask, 0.0)
    b = _fused(qkv, dout, H, mask.float(), 0.0)
    assert _delta(n0) == {"attn_forward": 2, "attn_backward": 4}
    for u, v in zip(a, b):
        assert torch.equal(u, v)


@pytest.mark.parametrize("S", [65, 200, 512])
@pytest.mark.parametrize("dtype", DTYPES)
def test_every_sequence_and_head_is_its_own_launch(dtype, S):
    """Every sum's order depends on S alone, so each (b, h) slice of a batched launch is bit for bit a launch on that
    slice by itself: anything else is an indexing bug."""
    B, H = 3, 5
    qkv, dout, mask = _inputs(B, S, H, dtype, 600 + S, [S, S - 13, 1])
    o, g = _fused(qkv, dout, H, mask, 0.0)
    q5, d5, o5, g5 = qkv.view(B, S, 3, H, D), dout.view(B, S, H, D), o.view(B, S, H, D), g.view(B, S, 3, H, D)
    for b in range(B):
        for h in range(H):
            x = q5[b:b + 1, :, :, h].reshape(1, S, 3 * D)
            ob, gb = _fused(x, d5[b:b + 1, :, h].contiguous(), 1, mask[b:b + 1], 0.0)
            assert torch.equal(ob.view(1, S, D), o5[b:b + 1, :, h]), (b, h)
            assert torch.equal(gb.view(1, S, 3, D), g5[b:b + 1, :, :, h]), (b, h)


@pytest.mark.parametrize("dtype", DTYPES)
def test_largest_grid_matches_float64_reference(dtype):
    """65535 sequences, the most grid.z takes; by the test above a sample of sequences stands for all of them."""
    B, S, H = 65535, 64, 1
    qkv, dout, mask = _inputs(B, S, H, dtype, 65, [1 + (37 * b) % S for b in range(B)])
    n0 = _counts()
    o, g = _fused(qkv, dout, H, mask, 0.0)
    assert _delta(n0) == {"attn_forward": 1, "attn_backward": 2}
    for b in (0, 1, 40000, B - 2, B - 1):
        s = slice(b, b + 1)
        _check(o[s], g[s], qkv[s], dout[s], H, mask[s], "seq %d " % b)
    del qkv, dout, o, g
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", DTYPES)
def test_misaligned_qkv_strided_dout_and_mask_match_the_dense_result(dtype):
    """qkv 2 or 4 bytes past a 16-byte boundary, dout and the mask every other element of a wider tensor: the op copies
    them dense and aligned, and the result is bit for bit that of the dense inputs."""
    from oktopk_b200.ops.fused_attn import self_attention
    B, S, H = 2, 100, 3
    qkv, dout, mask = _inputs(B, S, H, dtype, 45, [S, 61])
    o0, g0 = _fused(qkv, dout, H, mask, 0.0)
    buf = torch.zeros(qkv.numel() + 1, dtype=dtype, device="cuda")
    buf[1:] = qkv.reshape(-1)
    buf.requires_grad_(True)
    x = buf[1:].view(qkv.shape)
    wide = torch.zeros(B, S, 2 * H * D, dtype=dtype, device="cuda")
    wide[..., ::2] = dout
    wmask = torch.zeros(B, 1, 1, 2 * S, device="cuda")
    wmask[..., ::2] = mask
    dy, m = wide[..., ::2], wmask[..., ::2]
    assert x.data_ptr() % 16 != 0 and not dy.is_contiguous() and not m.is_contiguous()
    n0 = _counts()
    o = self_attention(x, H, m, 0.0)
    o.backward(dy)
    assert _delta(n0) == {"attn_forward": 1, "attn_backward": 2}
    assert torch.equal(o.detach(), o0) and torch.equal(buf.grad[1:].view(qkv.shape), g0)


# ------------------------------------------------------------------------------------------ 2. dropout
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("B,S,H", [(2, 128, 4), (2, 77, 3)])
def test_dropout_mask_is_the_philox_mask(dtype, B, S, H):
    p = 0.1
    qkv, dout, mask = _inputs(B, S, H, dtype, 5 + S, [S, S // 2])
    o, g = _fused(qkv, dout, H, mask, p, cuda_seed=123)
    keep = keep_mask(seed_of(123), B, H, S, p)
    sigma = (p * (1 - p) / keep.numel()) ** 0.5
    assert abs(float(keep.float().mean()) - (1 - p)) < 6 * sigma
    od, gd = _run(lambda x: _formula(x, H, mask.double(), keep, p), qkv.double(), dout.double())
    of, gf = _run(lambda x: _formula(x, H, mask.to(dtype), keep, p), qkv, dout)
    _within(o, of, od, dtype, "O")
    _within(g, gf, gd, dtype, "dqkv")


def test_kept_fraction_of_the_kernel():
    """With V = identity rows and uniform P, O_i sums the kept weights of row i: the mean is about 1 - p."""
    B, S, H, p = 4, 128, 8, 0.1
    qkv = torch.zeros(B, S, 3 * H * D, device="cuda")
    qkv.view(B, S, 3, H, D)[:, :, 2, :, 0] = 1.0        # v_j = e_0: O_i[0] = sum_j keep_ij / (1-p) / S
    from oktopk_b200.ops.fused_attn import self_attention
    o = self_attention(qkv, H, None, p).view(B, S, H, D)[..., 0]
    frac = float(o.mean()) * (1 - p)
    sigma = (p * (1 - p) / (B * H * S * S)) ** 0.5
    assert abs(frac - (1 - p)) < 6 * sigma


@pytest.mark.parametrize("p", [1e-3, 0.5, 0.9, 0.99])
@pytest.mark.parametrize("dtype", DTYPES)
def test_dropout_mask_and_scale_are_exact_at_every_rate(dtype, p):
    """With q = 0 every P_ij is 1/S, and with S = D = 64, v_j = e_j and dO_i = e_i, O[b, i, h, j] and dV[b, j, h, i]
    are both keep(b,h,i,j) / (1-p) / S: the forward and the backward mask read off element by element.  Then O and
    d(qkv) of random inputs against the formula with keep_mask."""
    B, S, H = 2, 64, 3
    eye = torch.eye(S, device="cuda")
    x = torch.zeros(B, S, 3, H, D, device="cuda")
    x[:, :, 1] = torch.randn(B, S, H, D, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    x[:, :, 2] = eye[None, :, None, :]
    qkv = x.view(B, S, -1).to(dtype)
    dout = eye[None, :, None, :].expand(B, S, H, D).reshape(B, S, H * D).to(dtype)
    o, g = _fused(qkv, dout, H, None, p, cuda_seed=31)
    keep = keep_mask(seed_of(31), B, H, S, p)
    fo = o.view(B, S, H, D).permute(0, 2, 1, 3)                     # [b, h, i, j]
    dv = g.view(B, S, 3, H, D)[:, :, 2].permute(0, 2, 3, 1)         # [b, h, i, j]
    value = (1.0 / (1.0 - p)) / S
    for got, what in ((fo, "forward"), (dv, "backward")):
        assert torch.equal(got != 0, keep), what
        err = float((got[keep].double() - value).abs().max())
        assert err <= 2 * EPS[dtype] * value, (what, err, value)

    B, S, H = 2, 77, 3
    qkv, dout, mask = _inputs(B, S, H, dtype, 7 + S, [S, 40])
    o, g = _fused(qkv, dout, H, mask, p, cuda_seed=32)
    keep = keep_mask(seed_of(32), B, H, S, p)
    od, gd = _run(lambda x: _formula(x, H, mask.double(), keep, p), qkv.double(), dout.double())
    of, gf = _run(lambda x: _formula(x, H, mask.to(dtype), keep, p), qkv, dout)
    _within(o, of, od, dtype, "O")
    _within(g, gf, gd, dtype, "dqkv")


def test_dropout_counter_past_2_32():
    """B H S^2 > 2^34, so the Philox counter idx // 4 passes 2^32: (b, h) = (4095, 15) holds the counters just below
    it, (4096, 0) those from 2^32 on, whose high word is 1.  A forward-only launch of about 17 GB."""
    from oktopk_b200.ops.fused_attn import self_attention
    B, S, H, p, dtype = 4100, 512, 16, 0.1, torch.bfloat16
    if torch.cuda.mem_get_info()[0] < 24 * 2 ** 30:
        pytest.skip("needs about 24 GB of free device memory")
    assert ((4095 * H + 15) * S * S + S * S) // 4 == 2 ** 32 == (4096 * H * S * S) // 4
    qkv = torch.zeros(B, S, 3 * H * D, dtype=dtype, device="cuda")
    gen = torch.Generator("cuda").manual_seed(4)
    qkv[4095:4097] = torch.randn(2, S, 3 * H * D, device="cuda", generator=gen).to(dtype)
    torch.cuda.manual_seed(41)
    with torch.no_grad():
        o = self_attention(qkv, H, None, p)
    x, o = qkv[4095:4097].clone(), o[4095:4097].clone()
    del qkv
    torch.cuda.empty_cache()
    keep = keep_mask(seed_of(41), 2, H, S, p, b0=4095)
    od, of = _formula(x.double(), H, None, keep, p), _formula(x, H, None, keep, p)
    for b, h in ((0, 15), (1, 0)):
        c = (slice(b, b + 1), slice(None), slice(h * D, (h + 1) * D))
        _within(o[c], of[c], od[c], dtype, (4095 + b, h))


# ------------------------------------------------------------------------------------------ 3. determinism
def test_same_seed_is_bitwise_reproducible_and_seeds_differ():
    qkv, dout, mask = _inputs(8, 128, 12, torch.bfloat16, 9, [128, 100, 64, 1, 128, 7, 90, 128])
    a = _fused(qkv, dout, 12, mask, 0.1, cuda_seed=21)
    b = _fused(qkv, dout, 12, mask, 0.1, cuda_seed=21)
    c = _fused(qkv, dout, 12, mask, 0.1, cuda_seed=22)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    assert not torch.equal(a[0], c[0]) and not torch.equal(a[1], c[1])
    z1 = _fused(qkv, dout, 12, mask, 0.0)
    z2 = _fused(qkv, dout, 12, mask, 0.0)
    for u, v in zip(z1, z2):
        assert torch.equal(u, v)


# ------------------------------------------------------------------------------------------ 4. recompute, graphs
def test_checkpoint_recomputes_the_same_mask():
    from torch.utils.checkpoint import checkpoint
    from oktopk_b200.ops.fused_attn import self_attention
    qkv, dout, mask = _inputs(4, 128, 12, torch.float32, 11, [128, 50, 128, 3])
    torch.manual_seed(5)
    o1, g1 = _run(lambda x: self_attention(x, 12, mask, 0.1), qkv, dout)
    torch.manual_seed(5)
    n0 = _counts()
    o2, g2 = _run(lambda x: checkpoint(lambda t: self_attention(t, 12, mask, 0.1), x, use_reentrant=False), qkv, dout)
    assert _delta(n0) == {"attn_forward": 2, "attn_backward": 2}
    assert torch.equal(o1, o2) and torch.equal(g1, g2)


def _graphed(qkv, dout, H, mask, p):
    from oktopk_b200.ops.fused_attn import self_attention
    x = qkv.detach().clone().requires_grad_(True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            x.grad = None
            self_attention(x, H, mask, p).backward(dout)
    torch.cuda.current_stream().wait_stream(s)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        o = self_attention(x, H, mask, p)
        o.backward(dout)
    return graph, o, x


def test_graph_replays_draw_fresh_masks_and_match_eager_at_p0():
    qkv, dout, mask = _inputs(8, 128, 12, torch.bfloat16, 13, [128, 100, 64, 1, 128, 7, 90, 128])
    graph, o, x = _graphed(qkv, dout, 12, mask, 0.1)
    outs = []
    for _ in range(2):
        graph.replay()
        outs.append((o.clone(), x.grad.clone()))
    torch.cuda.synchronize()
    assert not torch.equal(outs[0][0], outs[1][0]) and not torch.equal(outs[0][1], outs[1][1])
    graph, o, x = _graphed(qkv, dout, 12, mask, 0.0)
    graph.replay()
    oe, ge = _fused(qkv, dout, 12, mask, 0.0)
    assert torch.equal(o, oe) and torch.equal(x.grad, ge)


# ------------------------------------------------------------------------------------------ 5. fp16 range
def test_fp16_overflow_reaches_the_gradient_as_inf():
    """Every query attends to key 0, so dV_0 = sum_i dO_i = 128 x 1000 > 65504."""
    B, S, H = 1, 128, 2
    qkv = torch.zeros(B, S, 3, H, D, device="cuda")
    qkv[:, :, 0, :, 0] = 8.0
    qkv[:, 0, 1, :, 0] = 8.0                            # s_i0 = 64 / 8 = 8 above the others
    qkv = qkv.view(B, S, -1).half()
    dout = torch.full((B, S, H * D), 1000.0, device="cuda").half()
    o, g = _fused(qkv, dout, H, None, 0.0)
    assert torch.isfinite(o).all()
    assert torch.isinf(g.view(B, S, 3, H, D)[:, 0, 2]).all()


# ------------------------------------------------------------------------------------------ 6. whole model
@pytest.mark.parametrize("autocast", [None, torch.bfloat16])
def test_bert_fused_matches_stock(autocast, monkeypatch):
    """Logits, loss and every parameter gradient of the whole model in eval mode (p = 0), fused and stock, against a
    float64 copy: the fused error within twice the stock error plus ULPS ulps of the attention's type."""
    from oktopk_b200.models import bert as bert_mod
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining, synthetic_batch
    torch.manual_seed(0)
    a = BertForPreTraining(BertConfig(num_hidden_layers=4), depth=2).cuda().eval()
    b = copy.deepcopy(a)
    r = copy.deepcopy(a).double()
    a.fuse_attn = True
    batch = synthetic_batch(4, 128, device="cuda", generator=torch.Generator().manual_seed(1))
    mask64 = bert_mod.extended_attention_mask
    res = []
    for net in (a, b, r):
        if net is r:                                     # the float64 model's SDPA takes the mask in its own type
            monkeypatch.setattr(bert_mod, "extended_attention_mask", lambda m: mask64(m, torch.float64))
        n0 = _counts()
        with torch.autocast("cuda", autocast or torch.bfloat16, enabled=autocast is not None and net is not r):
            scores, nsp = net(*batch[:3])
            loss = net(*batch)
        loss.backward()
        res.append((scores.detach(), nsp.detach(), loss.detach(), [q.grad for q in net.parameters()], _delta(n0)))
    (sa, na, la, ga, ca), (sb, nb, lb, gb, cb), (sr, nr, lr, gr, _) = res
    assert ca == {"attn_forward": 8, "attn_backward": 8} and cb == {"attn_forward": 0, "attn_backward": 0}
    dtype = autocast or torch.float32
    _within(sa, sb, sr, dtype, "scores")
    _within(na, nb, nr, dtype, "nsp")
    _within(la, lb, lr, dtype, "loss")
    for (n, _), u, v, w in zip(a.named_parameters(), ga, gb, gr):
        _within(u, v, w, dtype, n)


# ------------------------------------------------------------------------------------------ 7. trainer
def test_graphed_trainer_with_every_fused_bert_op():
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertConfig, synthetic_batch
    from oktopk_b200.train.trainer import Trainer
    cfg = BertConfig(num_hidden_layers=2)
    tr = Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=1e-4, compressor="oktopk", density=0.001,
                 cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128, cuda_graph=True,
                 autocast="bf16", model_kwargs={"config": cfg, "depth": 2, "fuse_ln": True, "fuse_xent": True,
                                                "sparse_mlm": True, "fuse_attn": True})
    assert tr.graphed is not None and tr.net.fuse_attn
    batches = [synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(40 + i)) for i in range(3)]
    n0 = _counts()
    losses = [float(tr.graphed.step(batches[i % 3])) for i in range(8)]
    torch.cuda.synchronize()
    assert tr.graphed.enabled and len(tr.graphed.graphs) >= 1, tr.graphed.why_disabled
    steps = 3 + len(tr.graphed.graphs)                   # eager warm-up steps and captures launch; replays are not counted
    assert _delta(n0) == {"attn_forward": 2 * steps, "attn_backward": 4 * steps}
    assert all(np.isfinite(losses))
    tr.check_mlm_overflow()
    tr.close()


# ------------------------------------------------------------------------------------------ 8. fallbacks
@pytest.mark.parametrize("case", ["d32", "mask_bss", "s513", "b65536", "fp64", "p1", "mask_grad"])
def test_fallbacks_run_the_stock_ops(case):
    from oktopk_b200.ops.fused_attn import self_attention
    B, S, H, p, dh = 2, 64, 4, 0.1, D
    mask = torch.zeros(B, 1, 1, S, device="cuda")
    dtype = torch.float32
    if case == "d32":
        dh = 32
    elif case == "mask_bss":
        mask = torch.randn(B, 1, S, S, device="cuda")
    elif case == "s513":
        S, mask = 513, None
    elif case == "b65536":                              # past the kernels' grid limit of 65535 sequences; p = 0, since
        B, S, H, mask, p = 65536, 1, 1, None, 0.0       # stock SDPA takes no dropout past 65535 sequences either
    elif case == "fp64":
        dtype = torch.float64
        mask = mask.double()
    elif case == "p1":
        p = 1.0
    elif case == "mask_grad":
        mask.requires_grad_(True)
    qkv = torch.randn(B, S, 3 * H * dh, device="cuda", dtype=dtype)
    dout = torch.randn(B, S, H * dh, device="cuda", dtype=dtype)
    n0 = _counts()
    res = []
    # stock SDPA's memory-efficient backward sums over key blocks in a varying order unless deterministic algorithms
    # are on, so without them two stock runs can differ in the last bit
    old = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        for fused in (True, False):
            torch.manual_seed(3)
            if fused:
                res.append(_run(lambda x: self_attention(x, H, mask, p), qkv, dout))
            else:
                def stock(x):
                    q, k, v = x.view(B, S, 3, H, dh).permute(2, 0, 3, 1, 4)
                    o = F.scaled_dot_product_attention(q, k, v, attn_mask=mask, dropout_p=p)
                    return o.transpose(1, 2).reshape(B, S, H * dh)
                res.append(_run(stock, qkv, dout))
    finally:
        torch.use_deterministic_algorithms(old)
    assert _delta(n0) == {"attn_forward": 0, "attn_backward": 0}
    for u, v in zip(*res):                              # p = 1: stock returns NaN (0 / 0), and so must the fallback
        torch.testing.assert_close(u, v, rtol=0, atol=0, equal_nan=True)


def test_default_bert_launches_no_attention_kernel():
    from oktopk_b200.models.bert import BertConfig, BertForPreTraining, synthetic_batch
    net = BertForPreTraining(BertConfig(num_hidden_layers=2), depth=2).cuda()
    batch = synthetic_batch(2, 128, device="cuda", generator=torch.Generator().manual_seed(1))
    n0 = _counts()
    net(*batch).backward()
    assert _delta(n0) == {"attn_forward": 0, "attn_backward": 0}
