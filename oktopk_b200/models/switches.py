"""The opt-in switches of the model zoo, one entry per command-line flag: the ``create_net`` keywords it sets, the models
that take them, and what else it needs.  ``train/cli.py`` builds its flags, their checks and ``model_args`` from this
table, and ``create_net`` refuses a switch keyword that the chosen model does not take."""
from __future__ import annotations

from typing import Dict, NamedTuple, Optional, Tuple

# the ResNets whose batch-norms take the fused kernels with ``fuse_bn=True`` (VGG fuses by default; the ImageNet
# ResNets keep the stock modules, see ROADMAP)
FUSED_BN_RESNETS = ("resnet20", "resnet32", "resnet44", "resnet56", "resnet110")
VGGS = ("vgg11", "vgg13", "vgg16", "vgg19")
BERTS = ("bert_base", "bert")

# precision requirements
FP16 = "--fp16"                     # needs --fp16
HALF = "--bf16 or --fp16"           # needs one of them
FP32 = "fp32"                       # neither


class Switch(NamedTuple):
    flag: str
    keywords: Tuple[str, ...]       # the create_net keywords the flag sets, each to the flag's value
    models: Tuple[str, ...]
    help: str
    needs: Tuple[str, ...] = ()     # flags that must be given with it
    precision: Optional[str] = None
    type: Optional[type] = None     # None: a store_true flag
    default: object = False
    metavar: Optional[str] = None

    @property
    def dest(self) -> str:
        return self.flag[2:].replace("-", "_")


SWITCHES = (
    Switch("--fused-bn-fp16", ("fuse_fp16",), VGGS + FUSED_BN_RESNETS, precision=FP16,
           help="with --fp16: VGG's Conv -> BN -> ReLU [-> pool] blocks take the fused fp16 batch-norm kernels "
                "(default: stock modules under fp16; a ResNet also needs --fused-bn)"),
    Switch("--fused-bn", ("fuse_bn",), FUSED_BN_RESNETS + ("lstman4",),
           help="CIFAR ResNets (resnet20 ... resnet110): every conv -> BN [+ shortcut] -> ReLU takes the fused "
                "batch-norm kernels (default: stock modules; VGG always fuses).  lstman4: the seven batch-norm "
                "sites take the fused kernels, their statistics over the frames of the longest utterance, so "
                "--an4-pad-multiple no longer changes them (default: stock modules)"),
    Switch("--fused-ln", ("fuse_ln",), BERTS,
           help="BERT: both LayerNorm(x + dropout(a)) sites of every encoder layer take the fused dropout + "
                "residual + LayerNorm kernels (default: stock ops)"),
    Switch("--fused-xent", ("fuse_xent",), BERTS + ("lstm",),
           help="BERT: the masked-LM loss takes the fused softmax cross-entropy kernels, which read only the "
                "labelled rows (default: stock cross_entropy)"),
    Switch("--sparse-mlm", ("sparse_mlm",), BERTS,
           help="BERT: the masked-LM head (transform, LayerNorm, decoder GEMM) runs on the labelled rows only, "
                "gathered into a fixed number of rows (default: every token row)"),
    Switch("--mlm-capacity", ("mlm_capacity",), BERTS, needs=("--sparse-mlm",), type=float, default=None,
           help="with --sparse-mlm: the gathered rows as a fraction of the batch's tokens, rounded up to a "
                "multiple of 8 (default 0.25; labelled rows past it stop training with an error; 1.0 never "
                "overflows)"),
    Switch("--fused-attn", ("fuse_attn",), BERTS,
           help="BERT: the self-attention of every encoder layer takes the fused attention kernels, which read "
                "the packed QKV projection and regenerate the dropout mask (default: stock "
                "scaled_dot_product_attention)"),
    Switch("--fused-emb", ("fuse_emb",), BERTS,
           help="BERT: the embedding sum + LayerNorm + dropout runs on the fused embedding kernels, one kernel "
                "forward and the table gradients without a sort (default: stock ops)"),
    Switch("--fused-lstm", ("fuse_lstm",), ("lstman4",),
           help="lstman4: the LSTM layers run on the persistent fused recurrence kernels, one launch per layer "
                "and pass, instead of packed sequences through cuDNN (default: stock)"),
    Switch("--fused-lstm-lm", ("fuse_lstm",), ("lstm",), precision=HALF,
           help="lstm (PTB), with --bf16 or --fp16: the stacked LSTM runs on the 16-bit stacked-layer fused "
                "recurrence kernels, the hidden state carried in and out (default: stock cuDNN layer)"),
    Switch("--fused-lstm-lm-fp32", ("fuse_lstm", "fuse_lstm_fp32"), ("lstm",), precision=FP32,
           help="lstm (PTB), in fp32 (no --bf16 / --fp16): the stacked LSTM runs on the fp32 stacked-layer fused "
                "recurrence kernels, W_hh partly read from L2 every step, the step product in 3xTF32 "
                "(default: stock cuDNN layer)"),
    Switch("--fused-lstm-autocast", ("fuse_lstm_autocast",), ("lstman4",), needs=("--fused-lstm",), precision=HALF,
           help="with --fused-lstm and --bf16 or --fp16: the LSTM layers take the 16-bit fused recurrence kernels "
                "(default: stock layers under autocast)"),
    Switch("--fused-ctc", ("fuse_ctc",), ("lstman4",),
           help="lstman4: the CTC loss runs on the fused softmax + CTC kernels, the lengths read on the device "
                "and the backward deterministic (default: stock log_softmax + nn.CTCLoss)"),
    Switch("--fused-lookahead", ("fuse_lookahead",), ("lstman4",),
           help="lstman4: the look-ahead convolution and its Hardtanh run on one fused kernel per pass, the lengths "
                "read on the device, the weight gradient deterministic and the weight kept in fp32 under autocast "
                "(default: stock pad -> depthwise conv1d -> Hardtanh; not with --bidirectional)"),
    # a Trainer argument, not a create_net keyword
    Switch("--an4-pad-multiple", (), ("lstman4",), type=int, default=0, metavar="M",
           help="lstman4: pad every training batch's frames up to a multiple of M and keep its lengths on the "
                "device; with --cuda-graph, --fused-lstm and --fused-ctc the steps are captured in CUDA graphs, "
                "one set per padded length.  The batch-norm statistics count the padded frames unless --fused-bn is "
                "on (default: 0, off)"),
    # a Trainer argument, not a create_net keyword
    Switch("--fused-clip", (), ("lstman4", "lstm"),
           help="lstman4 and lstm (PTB): clip the reduced gradient on the device inside the optimizer step, one "
                "deterministic norm pass with the factor applied by the fused update, instead of torch's "
                "clip_grad_norm_ before it (default: clip_grad_norm_)"),
    # a Trainer argument, not a create_net keyword
    Switch("--lamb", (), BERTS,
           help="BERT: train with LAMB (okt.Lamb: per-parameter trust ratios ||w|| / ||u||, bias correction, weight "
                "decay 0.01 except biases and LayerNorm) on the fused LAMB kernels, the reduced gradient clipped to "
                "a global norm of 1.0 on the device and the learning rate on BertAdam's warmup_linear schedule "
                "(default: BertAdam)"),
    Switch("--bidirectional", ("bidirectional",), ("lstman4",),
           help="lstman4: bidirectional LSTM layers, the two directions summed, and no look-ahead convolution "
                "(default: uni-directional)"),
    Switch("--fused-lstm-bidirectional", ("fuse_lstm_bidirectional",), ("lstman4",),
           needs=("--fused-lstm", "--bidirectional"),
           help="with --fused-lstm and --bidirectional: both directions of each LSTM layer run on the fused "
                "recurrence kernels in one launch (default: stock bidirectional layers)"),
)

# create_net keyword -> the models that take it
SWITCH_MODELS: Dict[str, Tuple[str, ...]] = {}
for _s in SWITCHES:
    for _k in _s.keywords:
        SWITCH_MODELS[_k] = tuple(dict.fromkeys(SWITCH_MODELS.get(_k, ()) + _s.models))
del _s, _k
