"""Whole-step CUDA graphs for the PTB language model, on the GPU.  A graphed ``Trainer(dnn="lstm", cuda_graph=True)``
against an eager one with the same seed, dropout on, through the dense warm-up, the dense-to-sparse transition (an
exact-threshold iteration) and threshold-reuse iterations, bit for bit: the loss at every step, ``tr.hidden`` after
every step, and at the end every parameter and the optimizer state (Ok-Topk residuals and thresholds, loss scale).

The two trainers run one after the other, not interleaved: both draw their dropout masks from the process's default
CUDA generator (and the stock layer from cuDNN's process-wide dropout state), which ``Trainer.__init__`` re-seeds; a
graph replay takes the same Philox offsets as the eager step it stands for.

Configurations: the fused stacked-layer LSTM in bf16, in fp16 with dynamic loss scaling and a forced overflow, and in
fp32, each with ``fuse_xent`` and ``fused_clip`` on and off; the stock cuDNN layer in fp32.  Further: a reset of the
state and ``Trainer.test()`` mid-run, a short batch, a replay loop without synchronisation, the graph count per flavour,
and the configurations that stay eager."""
import gc

import pytest
import torch

pytestmark = pytest.mark.gpu

N, T = 20, 35
MODES = {"bf16": ("bf16", {"fuse_lstm": True}), "fp16": ("fp16", {"fuse_lstm": True}),
         "fp32": (None, {"fuse_lstm": True, "fuse_lstm_fp32": True}), "stock_fp32": (None, {})}


def _trainer(mode, graph, fuse_xent=True, fused_clip=True, **kw):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    autocast, model_kwargs = MODES[mode]
    cfg = okt.preset("lstm_an4", density=0.02, warmup_iters=4)
    return Trainer(dnn="lstm", dataset="ptb", batch_size=N, lr=22.0, compressor="oktopk", density=0.02, cfg=cfg,
                   seed=0, autocast=autocast, loss_scale="dynamic" if mode == "fp16" else None, fused_clip=fused_clip,
                   cuda_graph=graph, model_kwargs=dict(model_kwargs, fuse_xent=fuse_xent), **kw)


def _batches(n, rows=N):
    """n consecutive [rows, T] batches of the synthetic stream, as the loader hands them over."""
    from oktopk_b200.train.data import SyntheticPTB
    ds = SyntheticPTB(batch_size=N, num_steps=T)
    out = []
    for b in range(n):
        r = [ds[b * N + i] for i in range(rows)]
        out.append((torch.stack([x[0] for x in r]).cuda(), torch.stack([x[1] for x in r]).cuda()))
    return out


def _bits(t):
    t = t.detach().contiguous()
    if not t.is_floating_point():
        return t
    return t.view({8: torch.int64, 4: torch.int32, 2: torch.int16}[t.element_size()])


def _leaves(o, out):
    if torch.is_tensor(o):
        out.append(o.detach().clone())
    elif isinstance(o, dict):
        for v in o.values():
            _leaves(v, out)
    elif isinstance(o, (list, tuple)):
        for v in o:
            _leaves(v, out)
    else:
        out.append(o)
    return out


def _run(mode, graph, seq, hooks=None, **kw):
    """Train on ``seq``; ``hooks[i](tr)`` runs before step i.  Returns the per-step (loss, hidden, loss scale state),
    the final parameters and optimizer state, and the graph step (None eager)."""
    tr = _trainer(mode, graph, **kw)
    if graph:
        assert tr.graphed is not None and tr.graphed.enabled, tr.graphed.why_disabled
    per_step = []
    for i, b in enumerate(seq):
        if hooks and i in hooks:
            hooks[i](tr)
        loss = tr.step(b).clone()
        per_step.append((loss, tuple(h.detach().clone() for h in tr.hidden), tr.optimizer.loss_scale_state()))
    torch.cuda.synchronize()
    final = [p.detach().clone() for p in tr.net.parameters()] + _leaves(tr.optimizer.state_dict(), [])
    gs = tr.graphed
    if graph:
        assert gs.enabled, gs.why_disabled
        assert tr.hidden[0] is gs._state[0] and tr.hidden[1] is gs._state[1]
    tr.close()
    del tr
    gc.collect()
    torch.cuda.empty_cache()
    return per_step, final, gs


def _same(a, b):
    (sa, fa, _), (sb, fb, _) = a, b
    assert len(sa) == len(sb)
    for i, ((la, ha, ca), (lb, hb, cb)) in enumerate(zip(sa, sb)):
        assert torch.equal(_bits(la), _bits(lb)), (i, float(la), float(lb))
        for u, v in zip(ha, hb):
            assert u.dtype == v.dtype and u.shape == v.shape and torch.equal(_bits(u), _bits(v)), i
        assert ca == cb, i
    assert len(fa) == len(fb)
    for j, (u, v) in enumerate(zip(fa, fb)):
        if torch.is_tensor(u):
            assert u.dtype == v.dtype and torch.equal(_bits(u), _bits(v)), j
        else:
            assert u == v, j


def _kinds(gs):
    """{"dense", "reuse", "exact"}: the flavours the graph step holds graphs for."""
    out = set()
    for key in gs.graphs:
        plan = key[1]
        out.add("dense" if plan.kind == "dense" else "exact" if plan.exact_local else "reuse")
    return out


def _overflow(tr):
    """Raise the loss scale to 2^40: the fp16 backward overflows and the optimizer skips the step on the device."""
    st = tr.optimizer._ls.state()
    tr.optimizer._ls.reset(2.0 ** 40, st["growth_tracker"], st["skipped_steps"], st["adam_step"])


CONFIGS = [(m, x, c) for m in ("bf16", "fp16", "fp32") for x in (True, False) for c in (True, False)]
CONFIGS.append(("stock_fp32", False, False))


@pytest.mark.parametrize("mode,fuse_xent,fused_clip", CONFIGS,
                         ids=["%s-%s-%s" % (m, "xent" if x else "stockxent", "fusedclip" if c else "stockclip")
                              for m, x, c in CONFIGS])
def test_graphed_follows_eager_bit_for_bit(mode, fuse_xent, fused_clip):
    seq = _batches(10)
    hooks = {6: _overflow} if mode == "fp16" else None
    kw = dict(fuse_xent=fuse_xent, fused_clip=fused_clip)
    eager = _run(mode, False, seq, hooks, **kw)
    graphed = _run(mode, True, seq, hooks, **kw)
    _same(eager, graphed)
    gs = graphed[2]
    # 3 eager warm-up steps, a dense graph for iteration 3, then the sparse phase (exact at iteration 4, reuse after)
    assert _kinds(gs) == {"dense", "reuse", "exact"}
    assert len(gs.graphs) == 3                    # one per flavour, in one pool
    assert gs.fallbacks == {"shapes": 0, "state": 0}
    h_dt = {"bf16": torch.bfloat16, "fp16": torch.float16}.get(mode, torch.float32)
    assert gs._state[0].dtype == h_dt and gs._state[1].dtype == torch.float32
    assert graphed[0][-1][1][0].dtype == h_dt
    if mode == "fp16":
        scales = [s[2]["scale"] for s in graphed[0]]
        skipped = [s[2]["skipped_steps"] for s in graphed[0]]
        assert skipped[6] == skipped[5] + 1 and scales[6] == 2.0 ** 39, (scales, skipped)
        assert not torch.equal(graphed[0][6][1][0], graphed[0][5][1][0])     # a skipped step still carries the state


def test_reset_and_test_mid_run_follow_eager():
    """``tr.hidden = None`` before step 5 (the graph starts from zeros) and ``tr.test()`` before step 8 (its final state,
    of the training batch size, is carried in), as eager does them."""
    seq = _batches(11)

    def reset(tr):
        tr.hidden = None

    def evaluate(tr):
        res = tr.test(max_batches=2)
        assert res["loss"] > 0 and tr.hidden[0].size(1) == N

    hooks = {5: reset, 8: evaluate}
    eager = _run("bf16", False, seq, hooks)
    graphed = _run("bf16", True, seq, hooks)
    _same(eager, graphed)
    assert graphed[2].fallbacks == {"shapes": 0, "state": 0}


def test_short_batch_runs_eagerly_and_the_next_starts_from_zeros():
    full = _batches(9)
    short = _batches(1, rows=N - 1)[0]
    seq = full[:6] + [short] + full[6:]
    eager = _run("bf16", False, seq)
    graphed = _run("bf16", True, seq)
    _same(eager, graphed)
    gs = graphed[2]
    assert gs.fallbacks == {"shapes": 1, "state": 0}
    assert graphed[0][6][1][0].size(1) == N - 1
    assert len(gs.graphs) == 3


def test_a_state_of_another_dtype_runs_eagerly_and_is_counted():
    """An fp32 h where the bf16 path carries bf16 (a state the user built with ``init_hidden``): that step runs eagerly,
    as eager would, and replay resumes on the next."""
    seq = _batches(9)

    def fp32_state(tr):
        tr.hidden = tuple(0.5 * torch.ones(2, N, 1500, device="cuda") for _ in range(2))

    eager = _run("bf16", False, seq, {6: fp32_state})
    graphed = _run("bf16", True, seq, {6: fp32_state})
    _same(eager, graphed)
    assert graphed[2].fallbacks == {"shapes": 0, "state": 1}


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_replay_loop_has_no_synchronisation(mode):
    tr = _trainer(mode, True)
    seq = _batches(8)
    for b in seq:
        tr.step(b)
    torch.cuda.synchronize()
    gs = tr.graphed
    n = len(gs.graphs)
    torch.cuda.set_sync_debug_mode("error")
    try:
        for b in seq:
            tr.step(b)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert gs.enabled and len(gs.graphs) == n == 3, gs.why_disabled
    assert all(torch.isfinite(p).all() for p in tr.net.parameters())
    tr.close()


@pytest.mark.parametrize("autocast", ["bf16", "fp16"])
def test_stock_layer_under_autocast_stays_eager(autocast):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    tr = Trainer(dnn="lstm", dataset="ptb", batch_size=N, lr=22.0, compressor="oktopk", density=0.02, seed=0,
                 cfg=okt.preset("lstm_an4", density=0.02, warmup_iters=4), autocast=autocast, cuda_graph=True,
                 loss_scale="dynamic" if autocast == "fp16" else None)
    gs = tr.graphed
    assert gs is not None and not gs.enabled
    assert "stock nn.LSTM under %s autocast" % {"bf16": "bfloat16", "fp16": "float16"}[autocast] in gs.why_disabled
    tr.train_step()
    assert torch.isfinite(torch.tensor(tr.last_loss())) and not gs.graphs
    tr.close()


def test_gradient_accumulation_stays_eager():
    tr = _trainer("bf16", True, nsteps_update=2)
    assert tr.graphed is None
    tr.close()
