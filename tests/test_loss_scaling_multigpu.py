"""Loss scaling across GPUs (>= 2 devices): an inf on ONE rank makes EVERY rank skip the bucket's reduction, through the
device-side agreement of ``unscale_check`` (the verdict mailboxes of the symmetric block).  Every native path a verdict
guards: Ok-Topk reading autograd's tensors in place and reading the landed bucket, gTopk, a gather scheme (TopkA), the
dense warm-up (``dense_allreduce_kernel``) and the automatic dense switch (the residual carry-over).  A skipped call
leaves residual, thresholds, region edges and the call epoch bitwise unchanged on every rank, the next clean call matches
the oracle, and the scale halves on every rank."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from mp_util import run_distributed  # noqa: E402

pytestmark = [pytest.mark.gpu, pytest.mark.multigpu]

N = 200_003
INIT = 2.0 ** 10
# name -> (scheme, config overrides, read the gradient in place, call that is poisoned, exact match with the oracle)
CASES = {
    "oktopk-direct": ("oktopk", dict(), True, 1, True),
    "oktopk-landed": ("oktopk", dict(), False, 1, True),
    "gtopk": ("gtopk", dict(), False, 1, True),
    "topkA": ("topkA", dict(), False, 1, True),
    "dense-warmup": ("oktopk", dict(warmup_iters=100), False, 1, False),
    "dense-switch": ("oktopk", dict(density=0.1, dense_switch_density=0.05), False, 0, False),
}


def _cfg(case):
    from oktopk_b200.config import OkTopkConfig
    kw = dict(density=0.01, local_recompute_interval=2, global_recompute_interval=2, repartition_interval=2,
              slot_factor=64, gather_factor=64)
    kw.update(CASES[case][1])
    return OkTopkConfig(**kw)


def _grad(it, rank, n):
    g = torch.Generator().manual_seed(1000 * it + rank)
    return torch.randn(n, generator=g) * torch.linspace(0.2, 2.0, n)


def _residual0(rank, n):
    """A non-zero residual to start from, so that the dense switch has something to carry (or, skipped, to keep)."""
    return _grad(99, rank, n) * 0.01


def _poisoned(case, it, rank, P):
    return it == CASES[case][3] and rank == P - 1


def _worker(rank, P, case, iters):
    from oktopk_b200.config import LossScale
    from oktopk_b200.optimizer import _ScaleState
    from oktopk_b200.parallel.gpu_engine import CudaBucketEngine
    from oktopk_b200.parallel.world import World
    scheme, _, direct, _, _ = CASES[case]
    w = World()
    eng = CudaBucketEngine(N, _cfg(case), w, name="t")
    eng.enable_loss_scaling()
    ls = _ScaleState(LossScale(init_scale=INIT), torch.device("cuda"))
    eng.residual.copy_(_residual0(rank, N).cuda())
    recs = []
    for it in range(iters):
        scale = ls.state()["scale"]
        x = _grad(it, rank, N) * scale
        if _poisoned(case, it, rank, P):
            x[N // 3] = float("inf")
        before = (eng.residual.clone(), {k: v for k, v in eng.stats().items()
                                         if k in ("local_thr", "global_thr", "edges", "epoch")})
        src = x.cuda()
        if not direct:
            eng.grad.copy_(src)
        torch.cuda.synchronize()
        w.barrier()
        if direct:
            srcs = ([src.data_ptr()], [0], [N])
            eng.unscale_check(ls.ptr, srcs=srcs)
            eng.reduce(scheme, srcs=srcs, skip=eng.verdict_ptr)
        else:
            eng.unscale_check(ls.ptr)
            eng.reduce(scheme, skip=eng.verdict_ptr)
        torch.cuda.synchronize()
        found = ls.state()["found_inf"]
        st = eng.stats()
        rec = {"found": found, "scale_used": scale, "out": eng.grad.cpu().clone(),
               "residual_kept": bool(torch.equal(eng.residual, before[0])),
               "state_kept": {k: st[k] for k in before[1]} == before[1], "residual": eng.residual.cpu().clone()}
        ls.update()
        rec["scale_after"] = ls.state()["scale"]
        recs.append(rec)
        if direct or found:
            eng.grad.zero_()                      # what the fused update does after every step (skipped ones too)
    w.barrier()
    eng.close()
    return recs


@pytest.mark.parametrize("case", list(CASES))
def test_inf_on_one_rank_makes_every_rank_skip(case):
    _check(case, 2)


def _check(case, P, iters=3):
    from oktopk_b200.parallel.oracle import inv_scale_of, run_oracle_scaled
    from oktopk_b200.parallel.state import SparseState
    scheme, _, direct, poison_it, exact = CASES[case]
    got = run_distributed(_worker, P, (case, iters), backend="nccl", timeout=600)
    cfg = _cfg(case)
    states = [SparseState(N, P) for _ in range(P)]
    for r, st in enumerate(states):
        st.residual = _residual0(r, N)
    for it in range(iters):
        scale = got[0][it]["scale_used"]
        assert all(got[r][it]["scale_used"] == scale for r in range(P))
        grads = [_grad(it, r, N) * scale for r in range(P)]
        for r in range(P):
            if _poisoned(case, it, r, P):
                grads[r][N // 3] = float("inf")
        ref, skipped = run_oracle_scaled(scheme, grads, states, cfg, inv_scale_of(scale))
        assert skipped == (it == poison_it)
        for r in range(P):
            rec = got[r][it]
            assert rec["found"] == int(skipped), "%s it %d rank %d: verdict %d" % (case, it, r, rec["found"])
            assert rec["scale_after"] == (scale / 2 if skipped else scale), (case, it, r)
            if skipped:
                assert rec["residual_kept"] and rec["state_kept"], "%s rank %d: a skipped call changed state" % (case, r)
                if direct:
                    assert float(rec["out"].abs().max()) == 0.0, "the direct-path bucket must stay all-zero"
                continue
            if exact:
                assert torch.equal(rec["out"], ref[r]), "%s it %d rank %d differs from the oracle" % (case, it, r)
            else:                                 # the dense kernel sums in another order than the oracle
                torch.testing.assert_close(rec["out"], ref[r], rtol=1e-5, atol=1e-6)
            assert torch.equal(rec["residual"], states[r].residual), "%s it %d rank %d residual" % (case, it, r)
