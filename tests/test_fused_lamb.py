"""GPU tests of the fused LAMB update (csrc/optim.cu lamb_moments / lamb_ratio / lamb_apply through ``fused_lamb``, and
a wrapped ``okt.Lamb``): the step and the per-parameter norms against float64 at chunk and float4 boundaries, bitwise
repeatability, the fault flag and the skip verdict, Ok-Topk reading the gradients in place, fp16 loss scaling, the
global clip against torch's, graphed trainer steps against eager ones, the launch count, and two ranks.

Accuracy: each step starts the fused kernels, ``okt.Lamb``'s fp32 torch step and a float64 step from the same fp32
state; the fused step's largest error against float64 must be at most twice the torch step's (plus one ulp of the
tensor's largest weight, for tensors where torch's error happens to be 0)."""
import copy
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402

pytestmark = pytest.mark.gpu

B1, B2, EPS = 0.9, 0.999, 1e-6


def _C():
    from oktopk_b200.ops import ext
    return ext.require()


def _count(name):
    from oktopk_b200.ops import ext
    return ext.LAUNCH_COUNT.get(name, 0)


class _Slice:
    """One param-group slice laid out as a bucket lays it out, with 4-element alignment: segments of the given sizes,
    p, g, m, v and the tables ``fused_lamb`` reads."""

    def __init__(self, sizes, seed=0):
        C = _C()
        self.sizes = list(sizes)
        self.offs, o = [], 0
        for n in sizes:
            self.offs.append(o)
            o += -(-n // 4) * 4
        self.n = self.offs[-1] + sizes[-1]                # no padding after the last segment: a scalar tail
        blk = [0]
        for n in sizes:
            blk.append(blk[-1] + max(1, -(-n // C.SUMSQ_CHUNK)))
        ends = [self.offs[j + 1] // 4 for j in range(len(sizes) - 1)] + [2 ** 31 - 1]
        as_dev = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")      # noqa: E731
        self.tab = [as_dev(v) for v in (self.offs, sizes, blk, ends)]
        self.nblk = blk[-1]
        gen = torch.Generator(device="cuda").manual_seed(seed)
        cap = -(-self.n // 4) * 4
        self.p = torch.zeros(cap, device="cuda")
        self.g = torch.zeros(cap, device="cuda")
        self.m = torch.zeros(cap, device="cuda")
        self.v = torch.zeros(cap, device="cuda")
        for o, n in zip(self.offs, sizes):
            self.p[o:o + n] = torch.randn(n, device="cuda", generator=gen) * 0.05
        self.partial = torch.full((2, self.nblk), float("nan"), dtype=torch.float64, device="cuda")
        self.norm = torch.zeros(2, len(sizes), device="cuda")
        self.ratio = torch.zeros(len(sizes), device="cuda")
        self.gen = gen

    def views(self, t):
        return [t[o:o + n] for o, n in zip(self.offs, self.sizes)]

    def new_grad(self, scale=1.0):
        self.g.zero_()
        for o, n in zip(self.offs, self.sizes):
            self.g[o:o + n] = torch.randn(n, device="cuda", generator=self.gen) * scale

    def step(self, scal, fault=None, skip=None, coef=None, zero_grad=1):
        C = _C()
        C.fused_lamb(self.p.data_ptr(), self.g.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.n, B1, B2, EPS,
                     len(self.sizes), *(t.data_ptr() for t in self.tab), self.nblk, self.partial[0].data_ptr(),
                     self.partial[1].data_ptr(), self.norm[0].data_ptr(), self.norm[1].data_ptr(),
                     self.ratio.data_ptr(), zero_grad, torch.cuda.current_stream().cuda_stream, scal.data_ptr(),
                     fault.data_ptr() if fault is not None else 0, skip.data_ptr() if skip is not None else 0,
                     coef.data_ptr() if coef is not None else 0)


def _scal(lr, wd, t, bc=True):
    vals = [lr, wd, 1 - B1 ** t, 1 - B2 ** t] if bc else [lr, wd, 1.0, 1.0]
    return torch.tensor(vals, dtype=torch.float32, device="cuda")


def _group(lr, wd, bc=True):
    return {"lr": lr, "betas": (B1, B2), "eps": EPS, "weight_decay": wd, "bias_correction": bc}


def _f64_step(w, g, m, v, t, lr, wd, bc):
    """float64 LAMB step from the given (fp32) state: (w, m, v, ||w||, ||u||, r)."""
    w, g, m, v = (x.double() for x in (w, g, m, v))
    m = B1 * m + (1 - B1) * g
    v = B2 * v + (1 - B2) * g * g
    mh, vh = (m / (1 - B1 ** t), v / (1 - B2 ** t)) if bc else (m, v)
    u = mh / (vh.sqrt() + EPS) + wd * w
    wn, un = float(w.norm()), float(u.norm())
    r = wn / un if wd != 0 and wn > 0 and un > 0 else 1.0
    return w - lr * r * u, m, v, wn, un, r


CASES = {
    "1": [1], "3": [3], "4": [4], "5": [5], "mixed": [5, 3, 1, 4, 7],
    "chunk": [16383, 16384, 16385, 5, 2 * 16384 + 1],
    "big": [2 ** 20 + 3, 3, 2 ** 20 + 3],
}


@pytest.mark.parametrize("bc", [True, False])
@pytest.mark.parametrize("wd", [0.01, 0.0])
@pytest.mark.parametrize("case", list(CASES))
def test_step_against_float64(case, wd, bc):
    from oktopk_b200.optimizer import _lamb_param
    s = _Slice(CASES[case], seed=len(case))
    lr = 5e-3
    for t in (1, 2, 3):
        s.new_grad(scale=10.0 ** (t - 2))
        state = [x.clone() for x in (s.p, s.g, s.m, s.v)]
        s.step(_scal(lr, wd, t, bc))
        torch.cuda.synchronize()
        for j, (pw, gw, mw, vw) in enumerate(zip(*(s.views(x) for x in state))):
            w64, m64, v64, wn, un, r = _f64_step(pw, gw, mw, vw, t, lr, wd, bc)
            tw, tm, tv = pw.clone(), mw.clone(), vw.clone()
            _lamb_param(tw, gw.clone(), tm, tv, _group(lr, wd, bc), t)
            fw = s.views(s.p)[j]
            err_f = float((fw.double() - w64).abs().max())
            err_t = float((tw.double() - w64).abs().max())
            ulp = 2 ** -23 * float(w64.abs().max())
            assert err_f <= 2 * err_t + ulp, (case, j, t, err_f, err_t)
            for got, want in ((s.views(s.m)[j], m64), (s.views(s.v)[j], v64)):
                torch.testing.assert_close(got.double(), want, rtol=2e-6, atol=1e-6 * float(want.abs().max()))
            assert abs(float(s.norm[0, j]) - wn) <= 2 ** -23 * wn, (case, j, float(s.norm[0, j]), wn)
            assert abs(float(s.norm[1, j]) - un) <= 1e-5 * un, (case, j, float(s.norm[1, j]), un)
            if r == 1.0:
                assert float(s.ratio[j]) == 1.0
            else:
                assert abs(float(s.ratio[j]) - r) <= 2e-5 * r
        assert float(s.g.abs().max()) == 0.0                 # the gradient is cleared


def test_norms_of_a_segment_spanning_many_chunks():
    """BERT-base's word embedding, 30522 x 768 = 23.4 M elements (1431 chunks), between two small segments."""
    s = _Slice([5, 30522 * 768, 64], seed=9)
    s.new_grad()
    p0 = [x.clone() for x in s.views(s.p)]
    state = [x.clone() for x in (s.g, s.m, s.v)]
    s.step(_scal(1e-3, 0.01, 1))
    torch.cuda.synchronize()
    for j, (pw, gw, mw, vw) in enumerate(zip(p0, *(s.views(x) for x in state))):
        _, _, _, wn, un, r = _f64_step(pw, gw, mw, vw, 1, 1e-3, 0.01, True)
        assert abs(float(s.norm[0, j]) - wn) <= 2 ** -23 * wn
        assert abs(float(s.norm[1, j]) - un) <= 1e-5 * un
        assert abs(float(s.ratio[j]) - r) <= 2e-5 * r


def test_bitwise_repeatable():
    outs = []
    for _ in range(2):
        s = _Slice(CASES["chunk"] + [2 ** 20 + 3], seed=4)
        for t in (1, 2, 3):
            s.new_grad()
            s.step(_scal(1e-2, 0.01, t))
        torch.cuda.synchronize()
        outs.append([x.clone() for x in (s.p, s.m, s.v, s.norm, s.ratio, s.partial)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_fault_flag_stops_and_skip_verdict_clears_only_the_gradient():
    s = _Slice(CASES["mixed"] + [16385], seed=2)
    s.new_grad()
    s.step(_scal(1e-2, 0.01, 1))
    s.new_grad()
    before = [x.clone() for x in (s.p, s.g, s.m, s.v)]
    flag = torch.ones(1, dtype=torch.int32, device="cuda")
    s.step(_scal(1e-2, 0.01, 2), fault=flag)              # a timed-out reduction: nothing moves, not even the gradient
    torch.cuda.synchronize()
    for a, b in zip(before, (s.p, s.g, s.m, s.v)):
        assert torch.equal(a, b)
    s.step(_scal(1e-2, 0.01, 2), skip=flag)               # a skipped step: p, m, v stay, the gradient is cleared
    torch.cuda.synchronize()
    for a, b in zip(before[0:1] + before[2:], (s.p, s.m, s.v)):
        assert torch.equal(a, b)
    assert float(s.g.abs().max()) == 0.0


def test_clip_factor_scales_the_gradient_as_read():
    """A factor c: the same step as the gradient times c (one fp32 multiply), bit for bit."""
    a, b = _Slice(CASES["chunk"], seed=6), _Slice(CASES["chunk"], seed=6)
    c = torch.tensor([0.3125], device="cuda")
    for t in (1, 2):
        a.new_grad()
        b.new_grad()
        b.g.mul_(c)
        a.step(_scal(1e-2, 0.01, t), coef=c)
        b.step(_scal(1e-2, 0.01, t))
    torch.cuda.synchronize()
    for x, y in ((a.p, b.p), (a.m, b.m), (a.v, b.v)):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ wrapped Lamb
def _mlp(seed=0):
    torch.manual_seed(seed)
    return torch.nn.Sequential(torch.nn.Linear(256, 512), torch.nn.GELU(), torch.nn.Linear(512, 512), torch.nn.GELU(),
                               torch.nn.Linear(512, 10)).cuda()


def _mlp_groups(net):
    return [{"params": [p for p in net.parameters() if p.dim() > 1], "weight_decay": 0.01},
            {"params": [p for p in net.parameters() if p.dim() <= 1], "weight_decay": 0.0}]


def _mlp_batches(k, scale=3.0):
    g = torch.Generator(device="cuda").manual_seed(5)
    return [(torch.randn(64, 256, device="cuda", generator=g) * scale,
             torch.randint(0, 10, (64,), device="cuda", generator=g)) for _ in range(k)]


def _wrap(net, groups, **kw):
    import oktopk_b200 as okt
    from oktopk_b200.optimizer import Lamb
    kw.setdefault("compression", okt.compressors["none"])
    return okt.DistributedOptimizer(Lamb(groups, lr=1e-3), named_parameters=net.named_parameters(), **kw)


@pytest.mark.parametrize("clip", [False, True])
def test_launch_counts(clip):
    """Three update launches per bucket and param group; the global clip adds grad_sumsq (one bucket) and clip_coef."""
    from oktopk_b200.ops import ext
    net = _mlp()
    opt = _wrap(net, _mlp_groups(net), max_grad_norm=0.5 if clip else None)
    assert len(opt._buckets) == 1 and len(opt._buckets[0].group_slices) == 2 and opt._lamb is not None
    x, y = _mlp_batches(1)[0]
    for _ in range(2):
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.synchronize()
        n0, l0 = ext.LAUNCH_COUNT["total"], _count("fused_lamb")
        opt.step()
    assert _count("fused_lamb") - l0 == 3 * 2
    assert ext.LAUNCH_COUNT["total"] - n0 == 3 * 2 + (2 if clip else 0)
    opt.close()


def test_global_clip_equals_torch_clip_then_lamb():
    """Each step from the same state: the fused clipped step against clip_grad_norm_ over the reduced gradient, then
    okt.Lamb's torch step."""
    from oktopk_b200.optimizer import Lamb
    net = _mlp()
    opt = _wrap(net, _mlp_groups(net), max_grad_norm=0.5)
    assert opt._clip is not None
    params = list(net.parameters())
    for x, y in _mlp_batches(5):
        p0 = [p.detach().clone() for p in params]
        s0 = [{k: opt.state[p][k].clone() for k in ("exp_avg", "exp_avg_sq")} if "exp_avg" in opt.state[p] else {}
              for p in params]
        t0 = opt.counter
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.synchronize()
        grads = [p.grad.detach().clone() for p in params]
        opt.step()
        refs = [torch.nn.Parameter(q.clone()) for q in p0]
        for r, g in zip(refs, grads):
            r.grad = g
        assert float(torch.nn.utils.clip_grad_norm_(refs, 0.5)) > 0.5
        ref = Lamb([{"params": [r for r, p in zip(refs, params) if p.dim() > 1], "weight_decay": 0.01},
                    {"params": [r for r, p in zip(refs, params) if p.dim() <= 1], "weight_decay": 0.0}], lr=1e-3)
        for r, st in zip(refs, s0):
            if st:
                ref.state[r] = dict({k: v.clone() for k, v in st.items()}, step=torch.tensor(float(t0)))
        ref.step()
        torch.cuda.synchronize()
        for p, r in zip(params, refs):
            torch.testing.assert_close(p.detach(), r.detach(), rtol=1e-5, atol=1e-6)
    opt.close()


def test_fp16_overflow_step_leaves_state_and_does_not_advance_t():
    import oktopk_b200 as okt
    net = _mlp()
    opt = _wrap(net, _mlp_groups(net), loss_scale=okt.LossScale(init_scale=2.0 ** 10),
                compression=okt.compressors["oktopk"], is_sparse=True,
                cfg=okt.preset("vgg16", density=0.01, warmup_iters=2))
    assert opt._direct                                     # in-place reads: every update clears the bucket
    batches = _mlp_batches(5)

    def step(x, y, bad=False):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = torch.nn.functional.cross_entropy(net(x), y)
        opt.scale_loss(loss * float("inf") if bad else loss).backward()
        opt.step()

    for x, y in batches[:3]:
        step(x, y)
    torch.cuda.synchronize()
    before = [p.detach().clone() for p in net.parameters()] + [
        opt.state[p][k].clone() for p in net.parameters() for k in ("exp_avg", "exp_avg_sq")]
    st0 = opt._ls.state()
    step(*batches[3], bad=True)
    torch.cuda.synchronize()
    st1 = opt._ls.state()
    assert st1["skipped_steps"] == st0["skipped_steps"] + 1 and st1["adam_step"] == st0["adam_step"] == 3
    after = [p.detach().clone() for p in net.parameters()] + [
        opt.state[p][k].clone() for p in net.parameters() for k in ("exp_avg", "exp_avg_sq")]
    for a, b in zip(before, after):
        assert torch.equal(a, b)
    assert all(float(b.grad.abs().max()) == 0.0 for b in opt._buckets)
    step(*batches[4])                                      # the next applied step is t = 4
    torch.cuda.synchronize()
    for gi, g in enumerate(opt.param_groups):
        want = torch.tensor([g["lr"], g["weight_decay"], 1 - B1 ** 4, 1 - B2 ** 4], dtype=torch.float32)
        assert torch.equal(opt._lr_dev[4 * gi:4 * gi + 4].cpu(), want), gi
    assert opt.state_dict()["state"][0]["step"] == 4.0
    opt.close()


# ------------------------------------------------------------------------------------------------ BERT
def _bert_cfg():
    from oktopk_b200.models.bert import BertConfig
    return BertConfig(num_hidden_layers=2, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)


FUSED = {"fuse_ln": True, "fuse_xent": True, "fuse_attn": True, "fuse_emb": True}


def _bert_batches(k):
    from oktopk_b200.models.bert import synthetic_batch
    return [synthetic_batch(8, 128, device="cuda", generator=torch.Generator().manual_seed(40 + i)) for i in range(k)]


def test_oktopk_in_place_reads_equal_landing_bitwise():
    import oktopk_b200 as okt
    from oktopk_b200.models.bert import BertForPreTraining
    torch.manual_seed(0)
    base = BertForPreTraining(_bert_cfg(), depth=2, **FUSED).cuda()
    nets, opts = [], []
    for kind in ("direct", "land"):
        net = copy.deepcopy(base)
        named = list(net.named_parameters())
        groups = [{"params": [p for n, p in named if not any(k in n for k in ("bias", "norm", "LayerNorm"))],
                   "weight_decay": 0.01},
                  {"params": [p for n, p in named if any(k in n for k in ("bias", "norm", "LayerNorm"))],
                   "weight_decay": 0.0}]
        cfg = okt.preset("bert_base", density=0.001, warmup_iters=2)
        opt = _wrap(net, groups, compression=okt.compressors["oktopk"], is_sparse=True, density=0.001, cfg=cfg,
                    max_grad_norm=1.0)
        if kind == "land":
            opt._direct = False
        nets.append(net)
        opts.append(opt)
    assert opts[0]._direct and not opts[1]._direct
    for it, batch in enumerate(_bert_batches(8)):
        for k, (net, opt) in enumerate(zip(nets, opts)):
            opt.zero_grad()
            net(*batch).backward()
            opt.step()
            if k == 0:
                torch.cuda.synchronize()
                assert all(float(b.grad.abs().max()) == 0.0 for b in opt._buckets), it
    torch.cuda.synchronize()
    for (name, a), b in zip(nets[0].named_parameters(), nets[1].parameters()):
        assert torch.equal(a, b), name
    for ba, bb in zip(opts[0]._buckets, opts[1]._buckets):
        for key in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(opts[0]._flat_state[ba.index][key], opts[1]._flat_state[bb.index][key]), key
    for o in opts:
        o.close()


def _trainer(cuda_graph, autocast):
    import oktopk_b200 as okt
    from oktopk_b200.train.trainer import Trainer
    return Trainer(dnn="bert_base", dataset="wikipedia", batch_size=8, lr=1e-3, compressor="oktopk", density=0.001,
                   cfg=okt.preset("bert_base", density=0.001, warmup_iters=2), seed=0, seq_len=128,
                   cuda_graph=cuda_graph, autocast=autocast, t_total=12, warmup=0.25, lamb=True,
                   model_kwargs=dict(FUSED, config=_bert_cfg(), depth=2))


@pytest.mark.parametrize("autocast", [None, "bf16"])
def test_graphed_trainer_steps_equal_eager_bitwise(autocast):
    """Ten steps across the dense-to-sparse transition with the warmup_linear schedule moving the lr every step."""
    tg, te = _trainer(True, autocast), _trainer(False, autocast)
    assert tg.graphed is not None and te.graphed is None
    batches = _bert_batches(3)
    lrs = []
    for it in range(10):
        b = batches[it % 3]
        tg.step(b)
        te.step(b)
        lrs.append(tg.optimizer.param_groups[0]["lr"])
    torch.cuda.synchronize()
    assert tg.graphed.enabled and len(tg.graphed.graphs) >= 1, tg.graphed.why_disabled
    assert all(a != b for a, b in zip(lrs, lrs[1:])) and tg.optimizer.counter == te.optimizer.counter == 10
    for (name, a), b in zip(tg.net.named_parameters(), te.net.parameters()):
        assert torch.equal(a, b), name
    tg.close()
    te.close()


# ------------------------------------------------------------------------------------------------ two ranks
def _rank_worker(rank, P, steps):
    import oktopk_b200 as okt
    okt.init()
    net = _mlp()
    okt.broadcast_parameters(net)
    cfg = okt.preset("vgg16", density=0.02, warmup_iters=2, bucket_elems=100_000)
    opt = _wrap(net, _mlp_groups(net), compression=okt.compressors["oktopk"], is_sparse=True, cfg=cfg,
                max_grad_norm=1.0)
    for x, y in _mlp_batches(steps):
        x = x + rank                                       # different data per rank
        opt.zero_grad()
        torch.nn.functional.cross_entropy(net(x), y).backward()
        opt.step()
    torch.cuda.synchronize()
    flat = torch.cat([p.detach().view(-1) for p in net.parameters()]).cpu()
    opt.close()
    return flat


def test_two_ranks_end_bitwise_identical():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = run_distributed(_rank_worker, 2, (8,), backend="nccl", timeout=600)
    assert torch.equal(out[0], out[1])
