"""The channel-sliced fused batch-norm kernels (csrc/bnrelu.cu, bn_*_sliced_kernel): which shapes take them, a host
model of the summation tree they share with the cooperative kernels, and, on the GPU, bit-for-bit equality of the two
kernel families (``MAX_CTAS = 1 << 30`` runs the cooperative kernels with an uncapped grid)."""
import numpy as np
import pytest
import torch

VGG16_SHAPES = [(16, 64, 32, 32), (16, 128, 16, 16), (16, 256, 8, 8), (16, 512, 4, 4), (16, 512, 2, 2)]
VGG16_LAYERS = [VGG16_SHAPES[i] for i in (0, 0, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4)]
RESNET20_SHAPES = [(32, 16, 32, 32), (32, 32, 16, 16), (32, 64, 8, 8)]
# sliced shapes beyond VGG-16's: a ragged last tile and a CTA that is not whole warps; two 256-column combine chunks;
# a CTA of 24 threads that owns 32 channels
SLICED_SHAPES = VGG16_SHAPES[2:] + [(3, 512, 5, 5), (4, 1024, 4, 4), (2, 1024, 3, 3)]
COOPERATIVE = 1 << 30


# ------------------------------------------------------------------------------------------ 1. selection (no GPU needed)
def _geom(M, C):
    """bn_geom of csrc/bnrelu.cu."""
    cv = C // 4
    tpr = min(cv, 256)
    rpi = max(1, 256 // tpr)
    want = min(512, max(1, (M * C + 8191) // 8192))
    rpb = max(rpi, (-(-M // want) + rpi - 1) // rpi * rpi)
    nblk = -(-M // rpb)
    hold = cv <= 256 and rpb // rpi <= 8
    sc = 1
    while hold and 2 * sc * nblk * rpi <= 256 and cv // (2 * sc) >= 32:
        sc *= 2
    sc = sc if hold and sc >= 2 and cv % sc == 0 else 0
    return dict(M=M, C=C, cv=cv, rpi=rpi, rpb=rpb, nblk=nblk, hold=hold, sc=sc)


def _mc(shape):
    N, C, H, W = shape
    return N * H * W, C


def test_which_shapes_are_sliced():
    from oktopk_b200.ops import ext
    C = ext.require()
    for shape in VGG16_SHAPES:
        M, Ch = _mc(shape)
        for W in (0, shape[3]):
            assert C.bn_sliced(M, Ch, W) == (Ch >= 256), shape      # layers 5 - 13; layers 1 - 4 stay cooperative
    for shape in RESNET20_SHAPES + [(128, 16, 32, 32), (128, 64, 32, 32), (8, 256, 56, 56), (8, 2048, 7, 7)]:
        assert not C.bn_sliced(*_mc(shape), 0), shape               # too few columns, or tiles too large to hold
    for shape in SLICED_SHAPES:
        assert C.bn_sliced(*_mc(shape), 0), shape
    assert not C.bn_sliced(64, 512, 3)                              # not a pool the fused kernels take
    for M in (1, 7, 64, 75, 256, 1000, 1024, 4096, 16384, 100000):
        for Ch in (4, 16, 64, 128, 252, 256, 260, 512, 600, 608, 1024, 1032, 2048):
            g = _geom(M, Ch)
            assert C.bn_tile_rows(M, Ch) == g["rpb"]
            assert C.bn_sliced(M, Ch, 0) == (g["sc"] > 0), (M, Ch)
            assert g["hold"] or not C.bn_sliced(M, Ch, 0)
            if g["sc"]:
                assert g["sc"] * g["nblk"] * g["rpi"] <= 256 and g["cv"] // g["sc"] >= 32


# ------------------------------------------------------------------------------------------ 2. the summation tree, on the host
def _lane_sums(x, g):
    """Step 1: per (tile, lane, column) the sequential fp32 sum over rows row0 + ty + k rpi, k ascending."""
    M, cv, rpi, rpb, nblk = g["M"], g["cv"], g["rpi"], g["rpb"], g["nblk"]
    pad = np.zeros((nblk * rpb, cv, 4), np.float32)
    pad[:M] = x
    valid = (np.arange(nblk * rpb) < M).reshape(nblk, rpb // rpi, rpi)
    v = pad.reshape(nblk, rpb // rpi, rpi, cv, 4)
    acc = np.zeros((nblk, rpi, cv, 4), np.float32)
    for k in range(rpb // rpi):
        acc = np.where(valid[:, k, :, None, None], acc + v[:, k], acc)
    return acc


def _tree_cooperative(x, g):
    """Steps 2 and 3 as bn_tile_partial and bn_combine_partials do them over partial rows [sum | second sum]."""
    cv, rpi, nblk = g["cv"], g["rpi"], g["nblk"]
    lane = [_lane_sums(x, g), _lane_sums(x[::-1].copy(), g)]       # any second quantity: the tree is the same
    partial = np.zeros((nblk, 2 * cv, 4), np.float32)
    for which in range(2):
        t = lane[which][:, 0].copy()
        for j in range(1, rpi):
            t = t + lane[which][:, j]
        partial[:, which * cv:(which + 1) * cv] = t
    tot = np.zeros((2 * cv, 4), np.float32)
    for c0 in range(0, 2 * cv, 256):
        w = min(256, 2 * cv - c0)
        groups = 256 // w
        accs = []
        for j in range(groups):
            acc = np.zeros((w, 4), np.float32)
            for b in range(j, nblk, groups):
                acc = acc + partial[b, c0:c0 + w]
            accs.append(acc)
        t = accs[0]
        for a in accs[1:]:
            t = t + a
        tot[c0:c0 + w] = t
    return tot


def _tree_sliced(x, g, sc):
    """bn_slice_reduce, index for index: CTA b, thread (t rpi + ty) sc + cx; s_lane, s_tile, s_tot."""
    cv, rpi, nblk = g["cv"], g["rpi"], g["nblk"]
    lanes = nblk * rpi
    lane = [_lane_sums(x, g), _lane_sums(x[::-1].copy(), g)]
    tot = np.zeros((2 * cv, 4), np.float32)
    for blk in range(cv // sc):
        s_lane = np.zeros((2 * lanes * sc, 4), np.float32)
        for tid in range(lanes * sc):
            cx, ln = tid % sc, tid // sc
            for which in range(2):
                s_lane[which * lanes * sc + tid] = lane[which][ln // rpi, ln % rpi, blk * sc + cx]
        s_tile = np.zeros((2 * nblk * sc, 4), np.float32)
        for i in range(2 * nblk * sc):
            which, t, cx = i // (nblk * sc), i // sc % nblk, i % sc
            src = (which * lanes + t * rpi) * sc + cx
            v = s_lane[src].copy()
            for j in range(1, rpi):
                v = v + s_lane[src + j * sc]
            s_tile[i] = v
        for i in range(2 * sc):
            which, cx = i // sc, i % sc
            pcol = which * cv + blk * sc + cx
            groups = 256 // min(256, 2 * cv - pcol // 256 * 256)
            t = None
            for j in range(groups):
                acc = np.zeros(4, np.float32)
                for b in range(j, nblk, groups):
                    acc = acc + s_tile[(which * nblk + b) * sc + cx]
                t = acc if j == 0 else t + acc
            tot[pcol] = t
    return tot


@pytest.mark.parametrize("shape", VGG16_SHAPES + RESNET20_SHAPES + SLICED_SHAPES[3:5] + [(1, 64, 24, 24)])
def test_host_model_of_the_two_summation_orders_agrees_bitwise(shape):
    """The sliced kernels' shared-memory passes add the same fp32 values in the same order as the cooperative kernels'
    per-tile partials and combine, at every VGG-16 and ResNet-20 shape (whatever slice width would cut them), at
    two combine chunks (C = 1024) and at a combine with 8 groups (C = 64)."""
    M, C = _mc(shape)
    g = _geom(M, C)
    rng = np.random.default_rng(M + C)
    x = (rng.standard_normal((M, g["cv"], 4)) * 1.7 + 0.3).astype(np.float32)
    x[rng.integers(0, M, 5), rng.integers(0, g["cv"], 5)] = [[np.inf, -np.inf, np.nan, -0.0]]
    want = _tree_cooperative(x, g)
    for sc in {g["sc"] or 2, 1, 4}:
        got = _tree_sliced(x, g, sc)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (shape, sc)


# ------------------------------------------------------------------------------------------ 3. the two kernel families on the GPU
def _bn(C):
    torch.manual_seed(C)
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        bn.weight.normal_(1.0, 0.3); bn.bias.normal_(0.0, 0.5)
        bn.running_mean.normal_(0.0, 0.1); bn.running_var.uniform_(0.5, 1.5)
    return bn


def _inputs(shape, mode, dtype, special):
    g = torch.Generator("cuda").manual_seed(sum(shape))
    cl = torch.channels_last
    N, C, H, W = shape
    x = torch.randn(shape, device="cuda", generator=g) * 1.7 + 0.3
    if special:                 # constant channels (one where E[x^2] - mean^2 cancels to rounding noise, either sign)
        x[:, 0] = 0.0
        x[:, 1] = 1000.1
        x[:, 2] = -3.3
        x[0, 5, 0, 0] = float("nan")
        x[N - 1, 6, H - 1, W - 1] = float("inf")
        x[0, 7, 0, 1] = float("-inf")
        x[:, 9] *= 1e-3
        x[:, 9] += 300.0
    ys = (N, C, H // 2, W // 2) if mode == "pool" else shape
    dy = torch.randn(ys, device="cuda", generator=g)
    if special:
        dy[0, 12, 0, 0] = float("nan")
        dy[0, 13, 0, 0] = float("inf")
    r = torch.randn(shape, device="cuda", generator=g) * 0.8
    return [t.to(dtype).contiguous(memory_format=cl) for t in (x, dy, r)]


def _run(x, dy, r, bn, mode, conv_bias):
    from oktopk_b200.ops.fused_bn import bias_bn_relu
    xa = x.detach().clone().requires_grad_(True)
    ra = r.detach().clone().requires_grad_(True) if mode == "res" else None
    bn.zero_grad(set_to_none=True)
    y = bias_bn_relu(xa, bn, conv_bias, True, torch.nn.MaxPool2d(2, 2) if mode == "pool" else None, fp16=True, residual=ra)
    y.backward(dy)
    return [y, xa.grad, bn.weight.grad, bn.bias.grad, bn.running_mean, bn.running_var, bn.num_batches_tracked] + (
        [ra.grad] if ra is not None else [])


def _same(a, b):
    """Bit for bit, NaNs included."""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(
        a.contiguous().reshape(-1).view(torch.uint8), b.contiguous().reshape(-1).view(torch.uint8))


MODES = ["plain", "pool", "res"]


@pytest.mark.gpu
@pytest.mark.parametrize("special", [False, True])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", SLICED_SHAPES)
def test_sliced_kernels_match_cooperative_kernels_bitwise(shape, mode, dtype, special, monkeypatch):
    """Forward, backward (arg-max-dependent dx, dres), dgamma, dbeta, running statistics and the batch counter of the
    channel-sliced kernels against the cooperative kernels on the same inputs; with ``special`` on constant channels
    (the variance clamp) and inf / NaN in x and dy."""
    from oktopk_b200.ops import ext, fused_bn
    if mode == "pool" and shape[2] % 2:
        pytest.skip("odd height: the pool is not folded in")
    assert ext.require().bn_sliced(*_mc(shape), shape[3] if mode == "pool" else 0)
    x, dy, r = _inputs(shape, mode, dtype, special)
    bias = torch.randn(shape[1], device="cuda")
    bn_a, bn_b = _bn(shape[1]), _bn(shape[1])
    got = [t.clone() for t in _run(x, dy, r, bn_a, mode, bias)]
    monkeypatch.setattr(fused_bn, "MAX_CTAS", COOPERATIVE)
    want = _run(x, dy, r, bn_b, mode, bias)
    for i, (a, b) in enumerate(zip(got, want)):
        assert _same(a, b), (i, shape, mode, dtype)
    assert int(bn_a.num_batches_tracked) == 1
    if not special:
        assert all(bool(torch.isfinite(t.float()).all()) for t in got)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_sliced_kernels_replayed_from_a_cuda_graph_match_eager(mode):
    shape = (16, 512, 4, 4)
    x, dy, r = _inputs(shape, mode, torch.float32, True)
    bn_e, bn_g = _bn(512), _bn(512)
    eager = [[t.clone() for t in _run(x, dy, r, bn_e, mode, None)] for _ in range(3)]
    state = {k: v.clone() for k, v in bn_g.state_dict().items()}
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _run(x, dy, r, bn_g, mode, None)                       # warm up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    bn_g.load_state_dict(state)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = _run(x, dy, r, bn_g, mode, None)
    bn_g.load_state_dict(state)                                # the capture itself runs nothing
    for want in eager:
        graph.replay()
        for a, b in zip(out, want):
            assert _same(a, b)


@pytest.mark.gpu
def test_sliced_call_leaves_the_hand_off_counters_alone(monkeypatch):
    """Sliced and cooperative calls interleaved on one module (one counter slot) stay bit for bit what a module that
    only ever ran the cooperative kernels computes."""
    from oktopk_b200.ops import fused_bn
    shape = (16, 256, 8, 8)
    x, dy, r = _inputs(shape, "plain", torch.float32, False)
    bn_a, bn_b = _bn(256), _bn(256)
    for step in range(4):
        monkeypatch.setattr(fused_bn, "MAX_CTAS", COOPERATIVE if step % 2 else 0)
        got = [t.clone() for t in _run(x, dy, r, bn_a, "plain", None)]
        monkeypatch.setattr(fused_bn, "MAX_CTAS", 5 if step % 2 else COOPERATIVE)
        want = _run(x, dy, r, bn_b, "plain", None)
        for a, b in zip(got, want):
            assert _same(a, b), step
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_vgg16_step_launches_as_many_kernels_sliced_as_cooperative(monkeypatch):
    """13 bn_forward and 13 bn_backward launches and no standalone pool, on either kernel family, with equal loss."""
    from oktopk_b200.models import create_net
    from oktopk_b200.ops import ext, fused_bn
    names = ("bn_forward", "bn_backward", "maxpool2_fwd", "maxpool2_bwd")
    torch.manual_seed(0)
    x = torch.randn(16, 3, 32, 32, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 10, (16,), device="cuda")
    seen = []
    for cap in (0, COOPERATIVE):
        monkeypatch.setattr(fused_bn, "MAX_CTAS", cap)
        torch.manual_seed(1)
        net = create_net(10, "vgg16")[0].cuda().to(memory_format=torch.channels_last)
        n0 = {k: ext.LAUNCH_COUNT.get(k, 0) for k in names}
        loss = torch.nn.functional.cross_entropy(net(x), y)
        loss.backward()
        seen.append(({k: ext.LAUNCH_COUNT.get(k, 0) - v for k, v in n0.items()}, float(loss.detach())))
    assert seen[0][0] == {"bn_forward": 13, "bn_backward": 13, "maxpool2_fwd": 0, "maxpool2_bwd": 0}
    assert seen[0] == seen[1]
