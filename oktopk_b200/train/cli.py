"""Command line (L0): one entry point for all three reference programs.

    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 -m oktopk_b200.train.cli \
        --dnn vgg16 --dataset cifar10 --batch-size 16 --lr 0.1 --compression --compressor oktopk --density 0.02

Flag parity with ``VGG/main_trainer.py:144-160`` (``--batch-size --nsteps-update --nworkers --nwpernode
--compression --compressor --sigma-scale --density --dataset --dnn --data-dir --lr --max-epochs --pretrain``)
and with the BERT driver's relevant flags (``BERT/bert/main_bert.py:645-765``: ``--train_batch_size
--max_seq_length --num_minibatches --gradient_accumulation_steps --checkpoint_dir --config_path --module``).
The SLURM/sbatch + ``exp_configs/*.conf`` layer of the reference becomes ``--preset`` + plain flags; launch is
``torchrun`` (one process per GPU) instead of ``srun python -m mpi4py``.
"""
from __future__ import annotations

import argparse
import os
import re
import sys

import torch


def build_parser() -> argparse.ArgumentParser:
    from ..compression import compressors
    from ..models import DNNS
    p = argparse.ArgumentParser(description="oktopk_b200 trainer")
    p.add_argument("--batch-size", "--train_batch_size", dest="batch_size", type=int, default=16)
    p.add_argument("--nsteps-update", "--gradient_accumulation_steps", dest="nsteps_update", type=int, default=1)
    p.add_argument("--nworkers", type=int, default=1, help="informational: world size comes from torchrun")
    p.add_argument("--nwpernode", type=int, default=1)
    p.add_argument("--compression", dest="compression", action="store_true")
    p.add_argument("--compressor", type=str, default="oktopk", choices=[k for k in compressors if k])
    p.add_argument("--sigma-scale", type=float, default=2.5)
    p.add_argument("--density", type=float, default=0.01)
    p.add_argument("--dataset", type=str, default=None, choices=["imagenet", "cifar10", "an4", "ptb", "mnist", "wikipedia"])
    p.add_argument("--dnn", type=str, default="vgg16", choices=DNNS)
    p.add_argument("--module", type=str, default=None, help="BERT style 'models.bert12.depth=4' (layers / depth)")
    p.add_argument("--config_path", type=str, default=None, help="BERT config json")
    p.add_argument("--data-dir", type=str, default=None)
    p.add_argument("--lr", type=float, default=0.1)
    p.add_argument("--max-epochs", type=int, default=1)
    p.add_argument("--max-iters", "--num_minibatches", dest="max_iters", type=int, default=None)
    p.add_argument("--max_seq_length", type=int, default=128)
    p.add_argument("--pretrain", type=str, default=None)
    p.add_argument("--checkpoint_dir", type=str, default=None)
    p.add_argument("--log-dir", type=str, default=None)
    p.add_argument("--preset", type=str, default=None, help="vgg16 | lstm_an4 | bert_base (SURVEY A.1 constants)")
    p.add_argument("--warmup-iters", type=int, default=None, help="dense warm-up iterations (preset default if omitted)")
    p.add_argument("--bucket-elems", type=int, default=None)
    p.add_argument("--backend", type=str, default=None, choices=["auto", "cuda", "dist"])
    p.add_argument("--no-fused", action="store_true", help="phase-per-launch ablation of the persistent kernel")
    p.add_argument("--slot-factor", type=float, default=None,
                   help="bounded send/gather slots of slot_factor*k/P entries with the in-kernel overflow policy (default 0: lossless layout)")
    p.add_argument("--overselect-cap", type=float, default=None,
                   help="hard bound on the per-rank selection, in units of k (preset: 2; 0 = the reference's behaviour)")
    p.add_argument("--dense-switch-density", type=float, default=None,
                   help="densities >= this take the dense kernel (default 0.05; 0 = never)")
    p.add_argument("--nvls", type=str, default=None, choices=["auto", "on", "off"], help="dense path through the NVSwitch multicast object")
    p.add_argument("--comm-ctas", type=int, default=None, help="CTAs of the persistent communication kernels (default: one per SM)")
    p.add_argument("--norm-clip", type=float, default=None, help="TopkA / TopkA2 / gTopk: clip the bucket's L2 norm to sqrt(1/P)*norm_clip")
    p.add_argument("--trace", type=str, default=None, help="directory: dump the device-side per-call trace ring of every bucket at the end")
    p.add_argument("--deterministic", action="store_true")
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--cuda-graph", action="store_true", help="capture forward+backward+allreduce+update into CUDA graphs")
    p.add_argument("--fp16", action="store_true", help="fp16 autocast (reference: apex amp O3, main_bert.py:1009-1023)")
    p.add_argument("--bf16", action="store_true", help="bf16 autocast")
    p.add_argument("--fused-bn-fp16", action="store_true",
                   help="with --fp16: VGG's Conv -> BN -> ReLU [-> pool] blocks take the fused fp16 batch-norm kernels "
                        "(default: stock modules under fp16; a ResNet also needs --fused-bn)")
    p.add_argument("--fused-bn", action="store_true",
                   help="CIFAR ResNets (resnet20 ... resnet110): every conv -> BN [+ shortcut] -> ReLU takes the fused "
                        "batch-norm kernels (default: stock modules; VGG always fuses).  lstman4: the seven batch-norm "
                        "sites take the fused kernels, their statistics over the frames of the longest utterance, so "
                        "--an4-pad-multiple no longer changes them (default: stock modules)")
    p.add_argument("--fused-ln", action="store_true",
                   help="BERT: both LayerNorm(x + dropout(a)) sites of every encoder layer take the fused dropout + "
                        "residual + LayerNorm kernels (default: stock ops)")
    p.add_argument("--fused-xent", action="store_true",
                   help="BERT: the masked-LM loss takes the fused softmax cross-entropy kernels, which read only the "
                        "labelled rows (default: stock cross_entropy)")
    p.add_argument("--sparse-mlm", action="store_true",
                   help="BERT: the masked-LM head (transform, LayerNorm, decoder GEMM) runs on the labelled rows only, "
                        "gathered into a fixed number of rows (default: every token row)")
    p.add_argument("--mlm-capacity", type=float, default=None,
                   help="with --sparse-mlm: the gathered rows as a fraction of the batch's tokens, rounded up to a "
                        "multiple of 8 (default 0.25; labelled rows past it stop training with an error; 1.0 never "
                        "overflows)")
    p.add_argument("--fused-attn", action="store_true",
                   help="BERT: the self-attention of every encoder layer takes the fused attention kernels, which read "
                        "the packed QKV projection and regenerate the dropout mask (default: stock "
                        "scaled_dot_product_attention)")
    p.add_argument("--fused-emb", action="store_true",
                   help="BERT: the embedding sum + LayerNorm + dropout runs on the fused embedding kernels, one kernel "
                        "forward and the table gradients without a sort (default: stock ops)")
    p.add_argument("--fused-lstm", action="store_true",
                   help="lstman4: the LSTM layers run on the persistent fused recurrence kernels, one launch per layer "
                        "and pass, instead of packed sequences through cuDNN (default: stock)")
    p.add_argument("--fused-lstm-lm", action="store_true",
                   help="lstm (PTB), with --bf16 or --fp16: the stacked LSTM runs on the 16-bit stacked-layer fused "
                        "recurrence kernels, the hidden state carried in and out (default: stock cuDNN layer)")
    p.add_argument("--fused-lstm-lm-fp32", action="store_true",
                   help="lstm (PTB), in fp32 (no --bf16 / --fp16): the stacked LSTM runs on the fp32 stacked-layer fused "
                        "recurrence kernels, W_hh partly read from L2 every step, the step product in 3xTF32 "
                        "(default: stock cuDNN layer)")
    p.add_argument("--fused-lstm-autocast", action="store_true",
                   help="with --fused-lstm and --bf16 or --fp16: the LSTM layers take the 16-bit fused recurrence kernels "
                        "(default: stock layers under autocast)")
    p.add_argument("--fused-ctc", action="store_true",
                   help="lstman4: the CTC loss runs on the fused softmax + CTC kernels, the lengths read on the device "
                        "and the backward deterministic (default: stock log_softmax + nn.CTCLoss)")
    p.add_argument("--an4-pad-multiple", type=int, default=0, metavar="M",
                   help="lstman4: pad every training batch's frames up to a multiple of M and keep its lengths on the "
                        "device; with --cuda-graph, --fused-lstm and --fused-ctc the steps are captured in CUDA graphs, "
                        "one set per padded length.  The batch-norm statistics count the padded frames unless --fused-bn is "
                        "on (default: 0, off)")
    p.add_argument("--bidirectional", action="store_true",
                   help="lstman4: bidirectional LSTM layers, the two directions summed, and no look-ahead convolution "
                        "(default: uni-directional)")
    p.add_argument("--fused-lstm-bidirectional", action="store_true",
                   help="with --fused-lstm and --bidirectional: both directions of each LSTM layer run on the fused "
                        "recurrence kernels in one launch (default: stock bidirectional layers)")
    p.add_argument("--loss-scale", type=str, default=None,
                   help="loss scaling: 'dynamic' (torch GradScaler's rule, checked on the device) or a fixed scale; off by default")
    p.add_argument("--recompute_step", action="store_true", help="activation recomputation in the BERT encoder")
    p.add_argument("--dataparallel", action="store_true", help="accepted for parity: data parallelism is the only mode")
    p.add_argument("--do_train", action="store_true", help="accepted for parity")
    p.add_argument("--do_lower_case", action="store_true", help="accepted for parity")
    p.add_argument("--train_path", type=str, default=None, help="BERT corpus (one sentence per line); implies --data-dir")
    p.add_argument("--vocab_path", type=str, default=None)
    p.add_argument("--bert_config_path", type=str, default=None)
    return p


def model_args(args: argparse.Namespace):
    """``(dnn, model_kwargs)`` for ``create_net`` from the parsed flags."""
    dnn = args.dnn
    model_kwargs = {}
    if args.module:                       # 'models.bert12.depth=4' => 12 layers run as 4 stage modules
        m = re.search(r"bert(\d+)\.depth=(\d+)", args.module)
        if m:
            dnn = "bert_base"
            model_kwargs.update(num_hidden_layers=int(m.group(1)), depth=int(m.group(2)))
    cfg_path = args.bert_config_path or (args.config_path if args.config_path and args.config_path.endswith(".json")
                                         and os.path.isfile(args.config_path) and "bert_config" in args.config_path else None)
    if cfg_path:
        model_kwargs["config"] = cfg_path
    if args.recompute_step:
        model_kwargs["recompute"] = True
    if args.fused_bn_fp16:
        model_kwargs["fuse_fp16"] = True
    if args.fused_bn:
        model_kwargs["fuse_bn"] = True
    if args.fused_ln:
        model_kwargs["fuse_ln"] = True
    if args.fused_xent:
        model_kwargs["fuse_xent"] = True
    if args.sparse_mlm:
        model_kwargs["sparse_mlm"] = True
    if args.mlm_capacity is not None:
        model_kwargs["mlm_capacity"] = args.mlm_capacity
    if args.fused_attn:
        model_kwargs["fuse_attn"] = True
    if args.fused_emb:
        model_kwargs["fuse_emb"] = True
    if args.fused_lstm or args.fused_lstm_lm or args.fused_lstm_lm_fp32:
        model_kwargs["fuse_lstm"] = True
    if args.fused_lstm_lm_fp32:
        model_kwargs["fuse_lstm_fp32"] = True
    if args.fused_lstm_autocast:
        model_kwargs["fuse_lstm_autocast"] = True
    if args.bidirectional:
        model_kwargs["bidirectional"] = True
    if args.fused_lstm_bidirectional:
        model_kwargs["fuse_lstm_bidirectional"] = True
    if args.fused_ctc:
        model_kwargs["fuse_ctc"] = True
    return dnn, model_kwargs


def check_fused_bn_args(parser: argparse.ArgumentParser, args: argparse.Namespace) -> None:
    """``--fused-bn`` is for the CIFAR ResNets and lstman4 only; on one of the ResNets, ``--fused-bn-fp16`` needs it."""
    from ..models import FUSED_BN_RESNETS
    if args.fused_bn and args.dnn not in FUSED_BN_RESNETS + ("lstman4",):
        parser.error("--fused-bn applies to %s and lstman4 (VGG fuses by default), not %s"
                     % (", ".join(FUSED_BN_RESNETS), args.dnn))
    if args.fused_bn_fp16 and args.dnn in FUSED_BN_RESNETS and not args.fused_bn:
        parser.error("--fused-bn-fp16 on %s needs --fused-bn" % args.dnn)


def check_fused_ln_args(parser: argparse.ArgumentParser, args: argparse.Namespace) -> None:
    """``--fused-ln``, ``--sparse-mlm``, ``--mlm-capacity``, ``--fused-attn`` and ``--fused-emb`` are for BERT only (``--dnn bert_base``
    / ``bert``, or a ``--module models.bertN.depth=M``), ``--fused-xent`` for BERT and the PTB model (``--dnn lstm``);
    ``--mlm-capacity`` needs ``--sparse-mlm`` and a value in (0, 1]."""
    dnn = model_args(args)[0]
    if args.fused_xent and dnn not in ("bert", "bert_base", "lstm"):
        parser.error("--fused-xent applies to BERT (bert_base, bert) and lstm, not %s" % dnn)
    for flag, on in (("--fused-ln", args.fused_ln), ("--sparse-mlm", args.sparse_mlm),
                     ("--mlm-capacity", args.mlm_capacity is not None), ("--fused-attn", args.fused_attn),
                     ("--fused-emb", args.fused_emb)):
        if on and dnn not in ("bert", "bert_base"):
            parser.error("%s applies to BERT (bert_base, bert), not %s" % (flag, dnn))
    if args.mlm_capacity is not None:
        if not args.sparse_mlm:
            parser.error("--mlm-capacity needs --sparse-mlm")
        if not 0.0 < args.mlm_capacity <= 1.0:
            parser.error("--mlm-capacity must be in (0, 1], got %r" % args.mlm_capacity)


def check_fused_lstm_args(parser: argparse.ArgumentParser, args: argparse.Namespace) -> None:
    """``--fused-lstm`` and ``--bidirectional`` are for the AN4 DeepSpeech model (``--dnn lstman4``) only;
    ``--fused-lstm-autocast`` needs ``--fused-lstm`` and one of ``--bf16`` / ``--fp16``; ``--fused-lstm-bidirectional``
    needs ``--fused-lstm`` and ``--bidirectional``.  ``--fused-lstm-lm`` is for the PTB model (``--dnn lstm``) and
    needs ``--bf16`` or ``--fp16``; ``--fused-lstm-lm-fp32`` is for the PTB model too, in fp32 only.  ``--fused-ctc`` is
    for ``lstman4`` only, as is ``--an4-pad-multiple`` (>= 0)."""
    if args.fused_lstm and model_args(args)[0] != "lstman4":
        parser.error("--fused-lstm applies to lstman4, not %s" % model_args(args)[0])
    if args.fused_lstm_lm and model_args(args)[0] != "lstm":
        parser.error("--fused-lstm-lm applies to lstm, not %s" % model_args(args)[0])
    if args.fused_lstm_lm and not (args.bf16 or args.fp16):
        parser.error("--fused-lstm-lm needs --bf16 or --fp16")
    if args.fused_lstm_lm_fp32 and model_args(args)[0] != "lstm":
        parser.error("--fused-lstm-lm-fp32 applies to lstm, not %s" % model_args(args)[0])
    if args.fused_lstm_lm_fp32 and (args.bf16 or args.fp16):
        parser.error("--fused-lstm-lm-fp32 runs fp32: with --bf16 or --fp16 use --fused-lstm-lm")
    if args.fused_lstm_autocast and not args.fused_lstm:
        parser.error("--fused-lstm-autocast needs --fused-lstm")
    if args.fused_lstm_autocast and not (args.bf16 or args.fp16):
        parser.error("--fused-lstm-autocast needs --bf16 or --fp16")
    if args.bidirectional and model_args(args)[0] != "lstman4":
        parser.error("--bidirectional applies to lstman4, not %s" % model_args(args)[0])
    if args.fused_lstm_bidirectional and not args.fused_lstm:
        parser.error("--fused-lstm-bidirectional needs --fused-lstm")
    if args.fused_lstm_bidirectional and not args.bidirectional:
        parser.error("--fused-lstm-bidirectional needs --bidirectional")
    if args.fused_ctc and model_args(args)[0] != "lstman4":
        parser.error("--fused-ctc applies to lstman4, not %s" % model_args(args)[0])
    if args.an4_pad_multiple and model_args(args)[0] != "lstman4":
        parser.error("--an4-pad-multiple applies to lstman4, not %s" % model_args(args)[0])
    if args.an4_pad_multiple < 0:
        parser.error("--an4-pad-multiple must be >= 1 (or 0, off), got %d" % args.an4_pad_multiple)


def main(argv=None) -> int:
    parser = build_parser()
    args = parser.parse_args(argv)
    if args.fused_bn_fp16 and not args.fp16:
        parser.error("--fused-bn-fp16 needs --fp16")
    check_fused_bn_args(parser, args)
    check_fused_ln_args(parser, args)
    check_fused_lstm_args(parser, args)
    import oktopk_b200 as okt
    from .trainer import preset_for, robust_ssgd
    okt.init()
    dnn, model_kwargs = model_args(args)
    if args.train_path and not args.data_dir:
        args.data_dir = os.path.dirname(os.path.abspath(args.train_path))
    cfg = okt.preset(args.preset or preset_for(dnn), density=args.density, sigma_scale=args.sigma_scale)
    over = {}
    if args.warmup_iters is not None:
        over["warmup_iters"] = args.warmup_iters
    if args.bucket_elems is not None:
        over["bucket_elems"] = args.bucket_elems
    if args.no_fused:
        over["fused"] = False
    if args.deterministic:
        over["deterministic"] = True
    if args.slot_factor is not None:
        over["slot_factor"] = over["gather_factor"] = args.slot_factor
    if args.overselect_cap is not None:
        over["overselect_cap"] = args.overselect_cap
    if args.dense_switch_density is not None:
        over["dense_switch_density"] = args.dense_switch_density
    if args.nvls is not None:
        over["nvls"] = args.nvls
    if args.comm_ctas is not None:
        over["comm_ctas"] = args.comm_ctas
    cfg = cfg.replace(**over)
    tr = robust_ssgd(dnn, args.dataset, args.data_dir, okt.size(), args.lr, args.batch_size, args.nsteps_update,
                     args.max_epochs, compression=args.compression, compressor=args.compressor,
                     nwpernode=args.nwpernode, sigma_scale=args.sigma_scale, pretrain=args.pretrain,
                     density=args.density, max_iters=args.max_iters, checkpoint_dir=args.checkpoint_dir, cfg=cfg,
                     log_dir=args.log_dir, seq_len=args.max_seq_length, seed=args.seed, backend=args.backend,
                     cuda_graph=args.cuda_graph, model_kwargs=model_kwargs or None, norm_clip=args.norm_clip,
                     autocast="bf16" if args.bf16 else ("fp16" if args.fp16 else None), loss_scale=args.loss_scale,
                     an4_pad_multiple=args.an4_pad_multiple)
    if args.trace:
        import json
        os.makedirs(args.trace, exist_ok=True)
        with open(os.path.join(args.trace, "trace_%s_rank%d.json" % (dnn, okt.rank())), "w") as f:
            json.dump(tr.optimizer._allreducer.trace(), f)
    if okt.rank() == 0:
        print("final loss %.5f after %d iterations" % (tr.last_loss(), tr.train_iter))
    tr.close()
    okt.shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
