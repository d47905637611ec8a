"""Whole-step CUDA graphs for the AN4 DeepSpeech model over padded batches, on the GPU:

1. the persistent LSTM kernels stop at the longest length: y and dgates on [0, Tm) of a launch at T_b > Tm equal a
   launch at T = Tm bit for bit, and are exactly 0 after;
2. ``lstm_layer_device`` equals ``lstm_layer`` with host lengths bit for bit;
3. ``DeepSpeech.forward(device_lengths=True)`` equals the host path bit for bit, with no synchronisation, and raises
   for stock layers;
4. a graphed trainer at ``an4_pad_multiple=1`` follows today's eager trainer bit for bit;
5. graphed at m = 32 follows eager at m = 32 bit for bit (fp32, bf16, fp16 with dynamic loss scaling, bidirectional),
   with one graph per (padded length, flavour) and a replay loop without synchronisations;
6. the eager fallbacks (targets past the capacity, lengths past the cap) and the disabled graph step;
7. padding's one effect on the fused model: with the batch-norm statistics frozen, a batch padded to m = 32 gives the
   unpadded loss, valid-frame logits and gradients to rounding; with them live it does not."""
import pytest
import torch
import torch.nn as nn

from oktopk_b200.ops import ext, fused_lstm
from oktopk_b200.ops.ext import DTYPE_CODE

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _deterministic_convs():
    old = torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = True, False
    yield
    torch.backends.cudnn.deterministic, torch.backends.cudnn.benchmark = old


def _bits(t):
    t = t.detach().contiguous()
    return t.view({4: torch.int32, 2: torch.int16}[t.element_size()])


# ------------------------------------------------------------------------------------------------ 1. the kernel bound
def _launch(gx, dy, whh, lens, T, N, H, dt, dirs):
    """Both kernels on [dirs, T, N, .] inputs; y and dgates start as NaN, so every element they hold was written."""
    C = ext.require()
    geom = fused_lstm._device_geometry(H, N, gx.device, dt.itemsize, dirs)
    assert geom is not None
    stream = torch.cuda.current_stream().cuda_stream
    y = torch.full((dirs, T, N, H), float("nan"), device="cuda", dtype=dt)
    gates = torch.empty(dirs, T, N, 4 * H, device="cuda")
    cs = torch.empty(dirs, T, N, H, device="cuda")
    dg = torch.full((dirs, T, N, 4 * H), float("nan"), device="cuda", dtype=dt)
    w1 = whh[1].data_ptr() if dirs == 2 else 0
    C.lstm_forward(gx.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), y.data_ptr(), gates.data_ptr(), cs.data_ptr(),
                   torch.zeros(dirs, dtype=torch.int64, device="cuda").data_ptr(), T, N, H, geom.units, geom.fwd_rows,
                   stream, DTYPE_CODE[dt], w1)
    C.lstm_backward(dy.data_ptr(), gates.data_ptr(), cs.data_ptr(), whh[0].data_ptr(), lens.data_ptr(), dg.data_ptr(),
                    torch.zeros(dirs, dtype=torch.int64, device="cuda").data_ptr(), T, N, H, geom.units,
                    geom.bwd_rows, stream, DTYPE_CODE[dt], w1)
    return y, dg


@pytest.mark.parametrize("dt", [torch.float32, torch.bfloat16, torch.float16], ids=["fp32", "bf16", "fp16"])
@pytest.mark.parametrize("dirs", [1, 2])
@pytest.mark.parametrize("case", ["minus1_equal", "minus1_mixed", "far_equal", "far_mixed"])
def test_kernels_stop_at_the_longest_length(dt, dirs, case):
    g = torch.Generator(device="cuda").manual_seed(11)
    H, N, Tb = 800, 5, 64
    Tm = Tb - 1 if case.startswith("minus1") else 9
    lens = [Tm] * N if case.endswith("equal") else [Tm, 1, Tm - 1, max(1, Tm // 2), 3][:N]
    lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    whh = [(0.05 * torch.randn(4 * H, H, device="cuda", generator=g)).to(dt) for _ in range(dirs)]
    gx = torch.randn(dirs, Tb, N, 4 * H, device="cuda", generator=g).to(dt)      # garbage in the padded rows too
    dy = torch.randn(Tb, N, H, device="cuda", generator=g).to(dt)
    yb, dgb = _launch(gx, dy, whh, lens, Tb, N, H, dt, dirs)
    ym, dgm = _launch(gx[:, :Tm].contiguous(), dy[:Tm].contiguous(), whh, lens, Tm, N, H, dt, dirs)
    assert torch.isfinite(ym.float()).all() and torch.isfinite(dgm.float()).all()
    assert torch.equal(_bits(yb[:, :Tm]), _bits(ym)) and torch.equal(_bits(dgb[:, :Tm]), _bits(dgm))
    assert torch.equal(_bits(yb[:, Tm:]), torch.zeros_like(_bits(yb[:, Tm:])))      # +0, not -0 or NaN
    assert torch.equal(_bits(dgb[:, Tm:]), torch.zeros_like(_bits(dgb[:, Tm:])))


# ------------------------------------------------------------------------------------------ 2. the device-lengths entry
@pytest.mark.parametrize("mode", ["fp32", "bf16", "bidirectional"])
def test_device_entry_equals_the_host_entry(mode):
    torch.manual_seed(4)
    T, N, I, H = 57, 4, 320, 800
    bi = mode == "bidirectional"
    rnn = nn.LSTM(I, H, bidirectional=bi).cuda()
    x = torch.randn(T, N, I, device="cuda")
    dy = torch.randn(T, N, H, device="cuda")
    lens = torch.tensor([T, 20, T - 1, 5], dtype=torch.int32)
    ac = mode == "bf16"
    outs = []
    for fn in (lambda xi: fused_lstm.lstm_layer(xi, lens, rnn, autocast=ac, bidirectional=bi),
               lambda xi: fused_lstm.lstm_layer_device(xi, lens.cuda(), rnn, autocast=ac, bidirectional=bi)):
        for p in rnn.parameters():
            p.grad = None
        xi = x.clone().requires_grad_(True)
        n0 = ext.LAUNCH_COUNT.get("lstm_forward", 0)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
            y = fn(xi)
        assert ext.LAUNCH_COUNT.get("lstm_forward", 0) == n0 + 1
        (y.float() * dy).sum().backward()
        outs.append([y, xi.grad] + [p.grad for p in rnn.parameters()])
    for a, b in zip(*outs):
        assert torch.equal(_bits(a), _bits(b))


def test_device_entry_raises_where_the_layer_would_be_stock():
    rnn = nn.LSTM(32, 64).cuda()
    lens = torch.tensor([10, 7], dtype=torch.int32, device="cuda")
    x = torch.randn(10, 2, 32, device="cuda")
    with pytest.raises(RuntimeError, match="int32"):
        fused_lstm.lstm_layer_device(x, lens.long(), rnn)
    with pytest.raises(RuntimeError, match="do not apply"):
        fused_lstm.lstm_layer_device(x.double(), lens, rnn)
    with pytest.raises(RuntimeError, match="do not apply"):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            fused_lstm.lstm_layer_device(x, lens, rnn)          # autocast without autocast=True: stock


# ------------------------------------------------------------------------------------- 3. DeepSpeech.forward on device
@pytest.mark.parametrize("mode", ["fp32", "bf16"])
def test_model_device_lengths_equal_the_host_path(mode):
    from oktopk_b200.models import create_net
    torch.manual_seed(0)
    net, _ = create_net(29, "lstman4", fuse_lstm=True, fuse_lstm_autocast=True)
    net = net.cuda().train()
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 1, 161, 200, generator=g).cuda()
    lens = torch.tensor([200, 137], dtype=torch.int32)
    w = torch.randn(2, 100, 29, generator=g).cuda()
    dev_lens = lens.cuda()
    torch.cuda.synchronize()
    res = []
    for dev in (False, True):
        net.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
            if dev:
                torch.cuda.set_sync_debug_mode("error")
            try:
                out, out_lens = net(x, dev_lens if dev else lens, device_lengths=dev)
                (out.float() * w).sum().backward()
            finally:
                torch.cuda.set_sync_debug_mode(0)
        assert out_lens.is_cuda == dev
        res.append([out, out_lens.cpu()] + [p.grad for p in net.parameters()])
    assert res[0][1].tolist() == [100, 69]
    for a, b in zip(*res):
        assert torch.equal(_bits(a) if a.is_floating_point() else a, _bits(b) if b.is_floating_point() else b)


def test_model_device_lengths_raise_for_stock_layers():
    from oktopk_b200.models import create_net
    x = torch.randn(1, 1, 161, 40, device="cuda")
    lens = torch.tensor([40], dtype=torch.int32, device="cuda")
    net = create_net(29, "lstman4")[0].cuda()
    with pytest.raises(RuntimeError, match="fuse_lstm"):
        net(x, lens, device_lengths=True)
    net.fuse_lstm = True
    with pytest.raises(RuntimeError, match="fuse_lstm_autocast"):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            net(x, lens, device_lengths=True)
    bi = create_net(29, "lstman4", bidirectional=True, fuse_lstm=True)[0].cuda()
    with pytest.raises(RuntimeError, match="fuse_lstm_bidirectional"):
        bi(x, lens, device_lengths=True)


# ------------------------------------------------------------------------------------------------------- 4-6. trainers
KW = {"fuse_lstm": True, "fuse_ctc": True}


def _trainer(m, graph, autocast=None, loss_scale=None, model_kwargs=KW, warmup_iters=5):
    import bench
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    dnn, dataset, bs, lr, preset = bench.MODELS["lstman4"]
    cfg = okt.preset(preset, density=0.001, warmup_iters=warmup_iters)
    return Trainer(dnn=dnn, dataset=dataset, batch_size=bs, lr=lr, compressor="oktopk", density=0.001, cfg=cfg,
                   t_total=100000, warmup=0.1, seed=0, cuda_graph=graph, an4_pad_multiple=m, autocast=autocast,
                   loss_scale=loss_scale, model_kwargs=dict(model_kwargs))


def _pool(idx):
    import bench
    return [tuple(t.cuda() for t in bench.make_batch("lstman4", i, 0, 2, 128)) for i in idx]


def _same_state(a, b):
    for pa, pb in zip(a.net.parameters(), b.net.parameters()):
        assert torch.equal(_bits(pa), _bits(pb))
    for ba, bb in zip(a.net.buffers(), b.net.buffers()):
        assert torch.equal(ba, bb)


# bench.make_batch's lengths: i = 0, 1, 2, 3, 5 give 108, 240, 228, 192 and 396 frames
def _frames(pool):
    return [b[0].size(3) for b in pool]


def _padded_against_unpadded(device, model_kwargs, frozen_bn):
    """One batch (108 frames, lengths 108 and 75) unpadded and staged at m = 32 (128 frames) through one model:
    ``[loss, logits at each utterance's valid frames, parameter gradients]`` for each.  ``frozen_bn``: the batch-norm
    layers run on their running statistics, the rest of the model in training mode."""
    import bench
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="lstman4", dataset="an4", batch_size=2, lr=0.001, compressor="none", compression=False,
                 t_total=100, warmup=0.1, seed=0, device=torch.device(device), an4_pad_multiple=32,
                 model_kwargs=model_kwargs)
    x, tg, _, ts = (t.to(device) for t in bench.make_batch("lstman4", 0, 0, 2, 128))
    batch = (x, tg, torch.tensor([1.0, 0.7], device=device), ts)
    staged = tr.stage_batch(batch)
    assert staged.inputs.size(3) == 128 and x.size(3) == 108
    net = tr.net.train()
    if frozen_bn:
        for m in net.modules():
            if isinstance(m, nn.modules.batchnorm._BatchNorm):
                m.eval()
    params = [p for p in net.parameters()]
    res = []
    for b in (batch, staged):
        if b is batch:
            out, lens = net(x, (b[2] * x.size(3)).int())
        else:
            out, lens = net(b.inputs, b.lengths, device_lengths=b.inputs.is_cuda)
        lens = lens.tolist()
        loss, _ = tr._forward_loss(b)
        res.append([loss.detach()] + [out[n, :L].detach() for n, L in enumerate(lens)]
                   + list(torch.autograd.grad(loss, params)))
    assert lens == [54, 38]
    tr.close()
    return res


def _max_rel_err(a, b):
    return max(((x - y).abs().max() / y.abs().max().clamp_min(1e-30)).item() for x, y in zip(a, b))


def _check_padding_semantics(device, model_kwargs):
    """Padding changes the batch-norm statistics and nothing else: with them frozen, loss, valid-frame logits and
    every gradient agree with the unpadded batch to rounding (the convolutions and GEMMs run at other widths); with
    them live, the logits move far beyond that."""
    unpadded, padded = _padded_against_unpadded(device, model_kwargs, frozen_bn=True)
    assert _max_rel_err(padded[:3], unpadded[:3]) < 1e-4
    assert _max_rel_err(padded[3:], unpadded[3:]) < 1e-3
    unpadded, padded = _padded_against_unpadded(device, model_kwargs, frozen_bn=False)
    assert _max_rel_err(padded[1:3], unpadded[1:3]) > 1e-2


def test_padding_changes_only_the_batch_norm_statistics(monkeypatch):
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)
    monkeypatch.setattr(torch.backends.cuda.matmul, "allow_tf32", False)
    _check_padding_semantics("cuda", KW)


def test_graphed_at_multiple_one_follows_todays_eager_trainer():
    pool = _pool([0, 1, 2])
    assert len(set(_frames(pool))) == 3
    eager, graphed = _trainer(0, False), _trainer(1, True)
    assert graphed.graphed is not None and graphed.graphed.enabled, graphed.graphed.why_disabled
    flavours = []
    for it in range(12):
        b = pool[it % len(pool)]
        if it >= 3:
            flavours.append(graphed.graphed._key())
        la = eager.step(b)
        lb = graphed.step(b)
        assert torch.equal(_bits(la), _bits(lb)), it
    torch.cuda.synchronize()
    _same_state(eager, graphed)
    kinds = {f[1:] for f in flavours}
    assert any(p.kind == "dense" for k in kinds for p in k)                 # the dense warm-up, in graphs
    assert len([k for k in kinds if all(p.kind != "dense" for p in k)]) >= 2   # two sparse flavours
    assert {k[0][3] for k in graphed.graphed.graphs} == set(_frames(pool))
    assert graphed.graphed.fallbacks == {"shapes": 0, "targets": 0}
    for tr in (eager, graphed):
        tr.close()


@pytest.mark.parametrize("mode", ["fp32", "bf16", "fp16", "bidirectional"])
def test_graphed_padded_follows_eager_padded(mode):
    kw = dict(autocast={"bf16": "bf16", "fp16": "fp16"}.get(mode),
              loss_scale="dynamic" if mode == "fp16" else None,
              model_kwargs=dict(KW, fuse_lstm_autocast=True) if mode in ("bf16", "fp16")
              else dict(KW, bidirectional=True, fuse_lstm_bidirectional=True) if mode == "bidirectional" else KW)
    pool = _pool([0, 1, 3, 5])                       # T = 108, 240, 192, 396: padded to 128, 256, 192, 416
    eager, graphed = _trainer(32, False, **kw), _trainer(32, True, **kw)
    gs = graphed.graphed
    assert gs.enabled, gs.why_disabled
    n_sparse = len(gs._sparse_flavours())
    dense = set()
    for it in range(16):
        b = pool[it % len(pool)]
        if it >= 3 and gs._key()[1].kind == "dense":
            dense.add(((2, 1, 161, -(-b[0].size(3) // 32) * 32), gs._key()))
        la = eager.step(b)
        lb = graphed.step(b)
        assert torch.equal(_bits(la), _bits(lb)), (mode, it)
    # every shape is captured now: one more pass replays without a single synchronisation
    torch.cuda.synchronize()
    n_graphs = len(gs.graphs)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in pool:
            graphed.step(b)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for b in pool:
        eager.step(b)
    torch.cuda.synchronize()
    assert len(gs.graphs) == n_graphs
    _same_state(eager, graphed)
    shapes = {(2, 1, 161, Tb) for Tb in (128, 256, 192, 416)}
    assert {k[0] for k in gs.graphs} == shapes
    assert len(gs.graphs) == len(shapes) * n_sparse + len(dense), (len(gs.graphs), n_sparse, dense)
    assert gs.fallbacks == {"shapes": 0, "targets": 0}
    for tr in (eager, graphed):
        tr.close()


def test_fallbacks_run_eagerly_counted_and_equal_eager(monkeypatch):
    from oktopk_b200.train import graph_step
    monkeypatch.setattr(graph_step, "MAX_AN4_SHAPES", 1)
    pool = _pool([0, 1])                             # T = 108, 240: 128 and 256 frames at m = 32
    # over capacity: 2 utterances of 20 frames (T_b = 32, 16 output frames: 32 targets) with 40 targets
    x = torch.randn(2, 1, 161, 20, device="cuda")
    over = (x, torch.randint(1, 29, (40,), dtype=torch.int32, device="cuda"), torch.ones(2, device="cuda"),
            torch.tensor([20, 20], dtype=torch.int32, device="cuda"))
    seq = [pool[0]] * 6 + [pool[1], over, pool[0], pool[1]]
    eager, graphed = _trainer(32, False, warmup_iters=3), _trainer(32, True, warmup_iters=3)
    for it, b in enumerate(seq):
        la = eager.step(b)
        lb = graphed.step(b)
        assert torch.equal(_bits(la), _bits(lb)), it
    torch.cuda.synchronize()
    _same_state(eager, graphed)
    gs = graphed.graphed
    assert gs.enabled, gs.why_disabled
    assert gs.fallbacks == {"shapes": 2, "targets": 1}
    assert {k[0] for k in gs.graphs} == {(2, 1, 161, 128)}
    for tr in (eager, graphed):
        tr.close()


@pytest.mark.parametrize("kw,why", [({"fuse_lstm": True}, "fuse_ctc"), ({"fuse_ctc": True}, "fuse_lstm")])
def test_a_model_that_is_not_fused_disables_the_graph_step(kw, why):
    tr = _trainer(32, True, model_kwargs=kw)
    assert tr.graphed is not None and not tr.graphed.enabled and why in tr.graphed.why_disabled
    tr.train_step()                                  # the padded eager path
    assert torch.isfinite(torch.tensor(tr.last_loss()))
    tr.close()
