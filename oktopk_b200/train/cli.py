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

from ..models.switches import FP16, FP32, FUSED_BN_RESNETS, HALF, SWITCHES


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
    p.add_argument("--cuda-graph", action="store_true", help="capture forward+backward+allreduce+update into CUDA graphs (PTB --dnn lstm: with "
                   "--fused-lstm-lm under --bf16 / --fp16, --fused-lstm-lm-fp32, or the stock layer in fp32)")
    p.add_argument("--fp16", action="store_true", help="fp16 autocast (reference: apex amp O3, main_bert.py:1009-1023)")
    p.add_argument("--bf16", action="store_true", help="bf16 autocast")
    for sw in SWITCHES:
        if sw.type is None:
            p.add_argument(sw.flag, action="store_true", help=sw.help)
        else:
            p.add_argument(sw.flag, type=sw.type, default=sw.default, metavar=sw.metavar, help=sw.help)
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
    for sw in SWITCHES:
        value = getattr(args, sw.dest)
        if value != sw.default:
            model_kwargs.update(dict.fromkeys(sw.keywords, value))
    return dnn, model_kwargs


def check_switch_args(parser: argparse.ArgumentParser, args: argparse.Namespace) -> None:
    """Each switch flag of ``models/switches.py`` that is given must apply to the model that ``model_args`` resolves
    (``--dnn``, or ``--module``), and come with the flags and the precision it needs."""
    dnn = model_args(args)[0]
    given = {sw.flag for sw in SWITCHES if getattr(args, sw.dest) != sw.default}
    half = args.bf16 or args.fp16
    for sw in SWITCHES:
        if sw.flag not in given:
            continue
        if dnn not in sw.models:
            parser.error("%s applies to %s, not %s" % (sw.flag, ", ".join(sw.models), dnn))
        for need in sw.needs:
            if need not in given:
                parser.error("%s needs %s" % (sw.flag, need))
        if (sw.precision == FP16 and not args.fp16) or (sw.precision == HALF and not half):
            parser.error("%s needs %s" % (sw.flag, sw.precision))
        if sw.precision == FP32 and half:
            alt = next(o.flag for o in SWITCHES if o.precision == HALF and o.models == sw.models)
            parser.error("%s runs fp32: with --bf16 or --fp16 use %s" % (sw.flag, alt))
    if args.fused_bn_fp16 and dnn in FUSED_BN_RESNETS and not args.fused_bn:
        parser.error("--fused-bn-fp16 on %s needs --fused-bn" % dnn)
    if args.mlm_capacity is not None and not 0.0 < args.mlm_capacity <= 1.0:
        parser.error("--mlm-capacity must be in (0, 1], got %r" % args.mlm_capacity)
    if args.an4_pad_multiple < 0:
        parser.error("--an4-pad-multiple must be >= 1 (or 0, off), got %d" % args.an4_pad_multiple)


# the names of the per-family checks that check_switch_args replaced, kept for their callers: each checks every switch
check_fused_bn_args = check_fused_ln_args = check_fused_lstm_args = check_switch_args


def main(argv=None) -> int:
    parser = build_parser()
    args = parser.parse_args(argv)
    check_switch_args(parser, args)
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
                     an4_pad_multiple=args.an4_pad_multiple, fused_clip=args.fused_clip, lamb=args.lamb)
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
