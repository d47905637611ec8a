"""Every tunable of the sparse-allreduce engine in one dataclass.

The reference scatters these as literals inside ``AllReducer.run`` and the
compressors (``VGG/allreducer.py:27,209-211,573-579,673,696-699,1054-1057``,
``LSTM/allreducer.py:214-216,578-584,692-695,1034-1037``,
``BERT/bert/allreducer.py:188-190,355-361,412,434-437,728-731``,
``VGG/compression.py:393-404``).  Here they are explicit, per-workload presets
reproduce the three reference programs, and everything can be overridden.
"""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field
from typing import Dict, Optional, Sequence


@dataclass
class OkTopkConfig:
    # ---- what to run -----------------------------------------------------
    compressor: str = "oktopk"          # key of compression.compressors
    density: float = 0.01               # rho; k = int(n * rho) per bucket
    sparse: bool = True                 # False => dense allreduce regardless of compressor

    # ---- bucketing (reference: THRESHOLD = 640 Mi elements => one bucket) --
    bucket_elems: int = 64 * 1024 * 1024  # elements per bucket (reverse/backward order)

    # ---- schedule ---------------------------------------------------------
    warmup_iters: int = 0               # dense iterations before the sparse scheme kicks in
    local_recompute_interval: int = 32  # tau_l: exact local threshold every N iters
    global_recompute_interval: int = 32  # tau_g: exact global top-k every N iters
    repartition_interval: int = 64      # tau_r: balanced region re-partition every N iters
    topkaopt_recompute_interval: int = 32  # topkAopt exact threshold period (VGG/allreducer.py:1105)

    # ---- threshold-reuse guards / adaptation -----------------------------
    overselect_guard_num: int = 4       # raise thr while count > num/den * k ...
    overselect_guard_den: int = 3
    overselect_guard_factor: float = 1.03
    overselect_guard_loops: int = 5     # ... at most this many times (0 => no guard, BERT)
    # Hard over-selection cap (0 = off = the reference's behaviour).  The reference's guard can raise a stale threshold by
    # at most 1.03^5; its BERT variant has no guard at all and ships 10-80x k entries per rank early in training.  The
    # fused pack pass tallies a whole geometric ladder of thresholds for free, so when the count is still above
    # overselect_cap * k after the guard, the threshold keeps climbing coarse rungs (x overselect_cap_factor each) until it
    # is not: per-rank volume <= overselect_cap * k whatever the staleness.  The skipped entries stay in the residual.
    overselect_cap: float = 0.0
    overselect_cap_factor: float = 1.19
    overselect_cap_rungs: int = 40
    local_adapt_low: float = 2.0 / 3.0  # count < low*k  => thr /= local_adapt_factor
    local_adapt_high: float = 5.0 / 4.0  # count > high*k => thr *= local_adapt_factor
    local_adapt_factor: float = 1.012
    global_adapt_low: float = 2.0 / 3.0  # total < low*k  => gthr /= global_adapt_inc
    global_adapt_high: float = 4.0 / 3.0  # total > high*k => gthr *= global_adapt_dec
    global_adapt_inc: float = 1.008
    global_adapt_dec: float = 1.008

    # ---- exchange ----------------------------------------------------------
    throttle: int = 4                   # peers in flight in the pairwise exchange (min(4, P))
    balanced_allgather: bool = False    # BERT: re-slice global list to ceil(T/P) per rank
    dsa_dense_fallback_frac: float = 1.0 / 3.0  # TopkDSA: dense if total nnz >= frac * n

    # ---- Gaussiank ----------------------------------------------------------
    gaussian_low: float = 3.0 / 4.0
    gaussian_high: float = 5.0 / 4.0
    gaussian_factor: float = 1.02
    gaussian_loops: int = 20
    gaussian_mode: str = "vgg"          # 'vgg' | 'lstm' | 'bert' correction-loop flavour

    # ---- misc reference knobs ------------------------------------------------
    sigma_scale: float = 2.5
    norm_clip: Optional[float] = None   # TopkA/gTopk: clip bucket L2 to sqrt(1/P)*norm_clip
    dynamic_densities: Optional[Sequence[float]] = None  # per-epoch density schedule

    # ---- CUDA engine -----------------------------------------------------
    backend: str = "auto"               # 'auto' | 'cuda' (fused peer-memory kernels) | 'dist' (torch.distributed ops)
    fused: bool = True                  # one persistent kernel per bucket (False => phase-per-launch ablation)
    deterministic: bool = False         # fixed source order in the sparse reduce (bitwise run-to-run)
    # Slot capacities.  0 (default) = LOSSLESS: a destination's send slot is as long as its region and the gather slot as
    # long as the bucket, so no selected entry can ever be dropped, however stale the threshold (the reference gets this
    # from host-side count handshakes, VGG/allreducer.py:708-726); costs 24 B/element of symmetric memory per bucket.
    # > 0 = BOUNDED: per-(src,dst) capacity slot_factor * k / P (gather: gather_factor * k / P) with the in-kernel
    # overflow policy (Ok-Topk: raise the threshold and redo the pack pass; classic-residual schemes keep unsent entries in
    # the residual) -- 'bounded and conserved'.
    slot_factor: float = 0.0
    gather_factor: float = 0.0
    # Automatic dense switch: above this density the sparse schemes are predicted (at rho = 0.1 the fused kernel is
    # selection/scatter bound and loses to the NVLS dense kernel) to be slower than a
    # dense allreduce of the error-compensated gradient, which also is the better gradient -- so the engine adds the
    # residual into the bucket, clears it and takes the dense kernel.  0 = never switch.
    dense_switch_density: float = 0.05
    max_redo: int = 12                  # bounded slots: pack passes that may be repeated per call
    redo_factor: float = 1.5            # first threshold raise of the overflow policy (squared on every further attempt)
    land_grads: bool = True             # gradients land in the bucket with ONE multi-tensor copy kernel per bucket (not 1 add/param)
    nvls: str = "auto"                  # dense path through the NVSwitch multicast object: 'auto' | 'on' | 'off'
    comm_ctas: int = 0                  # CTAs of the persistent kernel (0 => 1 per SM)
    pull_mode: str = "tma"              # 'tma' (cp.async.bulk of remote chunks) | 'ldg' (128-bit peer loads)
    overlap: bool = True                # launch a bucket's exchange as soon as its last grad lands
    # threshold-reuse Ok-Topk calls pack a bucket's ready gradients during backward (parallel/early_pack.py): one segment
    # once early_pack_frac of the bucket is ready and unpacked, on at most early_pack_ctas CTAs.  OKTOPK_EARLY_PACK=0 in the
    # environment turns it off.
    early_pack: bool = True
    early_pack_frac: float = 0.85
    early_pack_ctas: int = 32
    # with a fused SGD update, each early-pack segment is followed by the zero-gradient update of its ranges (old values
    # stashed, 8 B per element of the bucket), so that after the call only the elements it wrote are recomputed
    # (csrc/optim.cu sgd_ahead_kernel).  OKTOPK_SGD_AHEAD=0 in the environment turns it off.
    sgd_ahead: bool = True
    gselect_mode: str = "auto"          # global selection over the reduced region: 'list' | 'scan' | 'auto' (density <= 0.5 % -> list)
    peer_timeout_s: float = 60.0        # bound of every cross-GPU flag wait inside the kernels (0 = wait forever)

    def k_for(self, numel: int, density: Optional[float] = None) -> int:
        d = self.density if density is None else density
        return int(numel * d)

    def replace(self, **kw) -> "OkTopkConfig":
        return dataclasses.replace(self, **kw)

    def to_dict(self) -> Dict:
        return dataclasses.asdict(self)


@dataclass(frozen=True)
class LossScale:
    """Dynamic loss scaling for fp16 training (``DistributedOptimizer(..., loss_scale=LossScale())``).

    The defaults are ``torch.amp.GradScaler``'s; ``growth_factor=1, backoff_factor=1`` is a fixed scale.  Use
    ``opt.scale_loss(loss).backward()`` and ``opt.step()`` as usual; ``torch.amp.GradScaler`` itself cannot be combined
    with the optimizer (it would read the gradients while their reduction is still running).

    Semantics, per step:
      1. Every bucket's gradient is multiplied by ``inv_scale`` (the fp32 reciprocal of the scale computed in double)
         before it reaches a residual, a threshold or a momentum: these stay in unscaled units across scale changes.
      2. Per bucket: if any rank sees a non-finite value in the bucket, every rank skips the bucket's reduction.  Its
         residual, thresholds, region edges and device trace stay bitwise unchanged.
      3. Per step: if any bucket was skipped, no parameter and no optimizer state is updated (the gradient bucket is
         still cleared) and the scale backs off; otherwise the growth tracker advances and the scale grows every
         ``growth_interval`` clean steps, exactly as ``torch._amp_update_scale_``.  Buckets that were clean and already
         reduced in a skipped step keep their residual update (a single-bucket model skips completely).
      4. A skipped step does not advance the wrapped fused Adam's bias-correction step.  BertAdam's schedule and the
         engines' iteration counters do advance: a skipped exact-threshold or re-partition iteration leaves the previous
         threshold and region edges in force.  SGD with ``dampening != 0`` whose very first step is skipped starts its
         momentum from a zero buffer rather than from a copy of the first gradient.
    """
    init_scale: float = 2.0 ** 16
    growth_factor: float = 2.0
    backoff_factor: float = 0.5
    growth_interval: int = 2000

    def __post_init__(self):
        if not (self.init_scale > 0 and self.growth_factor >= 1 and 0 < self.backoff_factor <= 1
                and self.growth_interval >= 1):
            raise ValueError("LossScale: need init_scale > 0, growth_factor >= 1, 0 < backoff_factor <= 1, "
                             "growth_interval >= 1")

    @staticmethod
    def parse(spec) -> Optional["LossScale"]:
        """``None`` / ``LossScale`` pass through; ``"dynamic"`` is the default dynamic scale; a number is a fixed scale."""
        if spec is None or isinstance(spec, LossScale):
            return spec
        if isinstance(spec, str) and spec.strip().lower() == "dynamic":
            return LossScale()
        return LossScale(init_scale=float(spec), growth_factor=1.0, backoff_factor=1.0)


def _vgg() -> OkTopkConfig:
    # VGG/allreducer.py:573-579,209-211,696-699,1054-1057; VGG/compression.py:393-404
    return OkTopkConfig(
        density=0.02, warmup_iters=512,
        local_recompute_interval=32, global_recompute_interval=32, repartition_interval=64,
        overselect_guard_num=4, overselect_guard_den=3, overselect_guard_loops=5,
        local_adapt_low=2 / 3, local_adapt_high=5 / 4, local_adapt_factor=1.012,
        global_adapt_low=2 / 3, global_adapt_high=4 / 3, global_adapt_inc=1.008, global_adapt_dec=1.008,
        gaussian_mode="vgg", gaussian_factor=1.02, gaussian_loops=20,
        overselect_cap=2.0,
    )


def _lstm() -> OkTopkConfig:
    # LSTM/allreducer.py:214-216,578-584,692-695,1034-1037; LSTM/compression.py:447-458
    return OkTopkConfig(
        density=0.02, warmup_iters=128,
        local_recompute_interval=32, global_recompute_interval=32, repartition_interval=64,
        overselect_guard_num=3, overselect_guard_den=2, overselect_guard_loops=5,
        local_adapt_low=3 / 4, local_adapt_high=5 / 4, local_adapt_factor=1.012,
        global_adapt_low=3 / 4, global_adapt_high=5 / 4, global_adapt_inc=1.01, global_adapt_dec=1.008,
        gaussian_mode="lstm", gaussian_factor=1.012, gaussian_loops=50,
        overselect_cap=2.0,
    )


def _bert() -> OkTopkConfig:
    # BERT/bert/allreducer.py:188-190,355-361,434-437,615-715,728-731; BERT/bert/compression.py:371-381
    return OkTopkConfig(
        density=0.01, warmup_iters=0,
        local_recompute_interval=128, global_recompute_interval=128, repartition_interval=64,
        overselect_guard_loops=0,
        local_adapt_low=4 / 5, local_adapt_high=5 / 4, local_adapt_factor=1.025,
        global_adapt_low=4 / 5, global_adapt_high=5 / 4, global_adapt_inc=1.036, global_adapt_dec=1.025,
        balanced_allgather=True, sigma_scale=1.0,
        gaussian_mode="bert", gaussian_factor=1.012, gaussian_loops=20,
        overselect_cap=2.0,
    )


PRESETS = {
    "vgg16": _vgg, "vgg": _vgg, "cnn": _vgg,
    "lstm_an4": _lstm, "lstman4": _lstm, "lstm": _lstm,
    "bert_base": _bert, "bert": _bert,
}


def preset(name: str, **overrides) -> OkTopkConfig:
    """Per-workload constants of SURVEY Appendix A.1 (``preset('bert_base', density=0.001)``)."""
    if name not in PRESETS:
        raise KeyError("unknown preset %r (have %s)" % (name, sorted(PRESETS)))
    return PRESETS[name]().replace(**overrides)


def sigma_scale_for_density(density: float) -> float:
    """``VGG/allreducer.py:460-470`` table (passed to compress_org, unused inside)."""
    if density > 0.7:
        return 0.5
    if density > 0.05:
        return 1.5
    if density > 0.01:
        return 2.0
    return 3.0
