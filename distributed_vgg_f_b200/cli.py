"""Command line -- flag-for-flag compatible with the reference.

Reference (distributedVggf.py:239-302): ``-iu/--init_url`` (required), ``-rn/--rank`` (required),
``-ws/--world_size`` (required), ``-rd/--root_dir``, ``-ep/--epochs`` (20), ``-nc/--no_cuda``,
``-lr/--learning_rate`` (1e-3), ``-mb/--mini_batch`` (16); the parser prints the namespace and, as
a side effect, joins the process group when ``-ws > 1``; ``__main__`` then calls
``manage_training``.  Usage is one invocation per rank, e.g. (Readme.md:43-47)

    python -m distributed_vgg_f_b200 -iu tcp://10.0.0.1:23456 -rn 0 -ws 2 -rd /data -ep 5 \
        -lr 0.00001 -mb 64

All eight flags, short and long names and defaults are preserved; ``-rd`` is actually required
(the reference crashes with a TypeError without it, SURVEY 0.2).  Everything else is additive.
Under ``torchrun`` the three required flags may be omitted: they default from
``RANK / WORLD_SIZE / MASTER_ADDR:MASTER_PORT``.
"""
from __future__ import annotations

import argparse
import math
import os
import sys
from typing import Optional, Sequence

from .config import DATA, TRAIN

# Below 32 the fifth 2x2 pool of VGG leaves an empty feature map.
MIN_CROP = 32
MODELS = ["vggf", "vgg16", "vgg11", "vgg13", "vgg19", "vggf11", "vggf13", "vggf19", "vggf-tiny", "vggf-mini"]


def build_parser() -> argparse.ArgumentParser:
    desc = ("Trains a VGG-F convolutional neural network using a distributed cluster of machines. "
            "Train and validation data must be stored in folders TrainData and ValidationData under "
            "some root directory. Train and validation folders must have N subdirectories, one per "
            "class. The name of each of these N subdirectories is the class label.")
    env_ws = os.environ.get("WORLD_SIZE")
    env_rank = os.environ.get("RANK")
    env_url = None
    if "MASTER_ADDR" in os.environ and "MASTER_PORT" in os.environ:
        env_url = "tcp://%s:%s" % (os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"])
    parser = argparse.ArgumentParser(prog="distributed_vgg_f_b200", description=desc)
    required = parser.add_argument_group("required arguments")
    required.add_argument("-iu", "--init_url", type=str, required=env_url is None, default=env_url,
                          help="Initialization URL specifying the protocol and connection with a "
                               "master node like tcp://192.168.0.10:23456")
    required.add_argument("-rn", "--rank", type=int, required=env_rank is None,
                          default=int(env_rank) if env_rank is not None else 0,
                          help="Rank of the current instance (0..K-1).")
    required.add_argument("-ws", "--world_size", type=int, required=env_ws is None,
                          default=int(env_ws) if env_ws is not None else None,
                          help="Number of instances participating in the job")
    required.add_argument("-rd", "--root_dir", type=str, default=None,
                          help="Root directory for the training and validation sets")
    parser.add_argument("-ep", "--epochs", type=int, default=TRAIN.epochs,
                        help="Number of epochs. The default value is {}".format(TRAIN.epochs))
    parser.add_argument("-nc", "--no_cuda", action="store_true",
                        help="Flag to use the CPU in this instance. By default the program tries "
                             "to run on a GPU")
    parser.add_argument("-lr", "--learning_rate", type=float, default=TRAIN.learning_rate,
                        help="Selected learning rate. The default value is {}".format(
                            TRAIN.learning_rate))
    parser.add_argument("-mb", "--mini_batch", type=int, default=TRAIN.mini_batch,
                        help="Mini-batch size. The default value is {}".format(TRAIN.mini_batch))

    ext = parser.add_argument_group("extensions (not in the reference)")
    ext.add_argument("--model", default="vggf", choices=MODELS,
                     help="vggf = the reference's network (VGG-16 + funnel head); vggNN = torchvision's plain "
                          "VGG-NN; vggfNN = VGG-NN + funnel head; -tiny / -mini are test-sized")
    ext.add_argument("--num-classes", type=int, default=None,
                     help="override the class count (default: number of class folders)")
    ext.add_argument("--engine", default="auto", choices=["auto", "native", "oracle"],
                     help="native = sm_90a kernels; oracle = torch ops (CPU / reference numerics)")
    ext.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"],
                     help="bf16: the sm_90a engine (bf16 activations / weights / wire, fp32 master weights, moments and "
                          "accumulators).  fp32: the reference's arithmetic on the torch-op engine (the native kernels "
                          "have no tf32 path yet)")
    ext.add_argument("--optimizer", default="adam", choices=["adam", "adamw", "sgd", "lamb", "lars"],
                     help="adam / sgd: L2 weight decay (torch.optim.Adam / SGD); adamw: decoupled weight decay "
                          "(torch.optim.AdamW); lamb / lars: layer-wise trust ratio |w| / |update| per tensor for large "
                          "global batches (timm's Lamb with eps 1e-6, and Lars with trust coefficient 1e-3 and "
                          "--momentum).  Only tensors with a nonzero decay are adapted, so lamb / lars need "
                          "--weight-decay > 0 (--bias-weight-decay 0 keeps the biases unadapted), and --zero1 on is "
                          "refused with them at world size > 1")
    ext.add_argument("--momentum", type=float, default=TRAIN.momentum)
    ext.add_argument("--weight-decay", type=float, default=0.0,
                     help="weight decay of every parameter, >= 0 (default 0 = none, as the reference)")
    ext.add_argument("--bias-weight-decay", type=float, default=None,
                     help="weight decay of the biases, >= 0 (torchvision's --bias-weight-decay; default: "
                          "--weight-decay)")
    ext.add_argument("--lr-scheduler", default="step", choices=["step", "cosine"],
                     help="step: StepLR(--lr-step, --lr-gamma); cosine: CosineAnnealingLR over the epochs after "
                          "the warmup, down to --lr-min.  Stepped once per epoch")
    ext.add_argument("--lr-step", type=int, default=0,
                     help="StepLR period in epochs (0 = constant lr, as the reference)")
    ext.add_argument("--lr-gamma", type=float, default=TRAIN.decay_gamma)
    ext.add_argument("--lr-min", type=float, default=0.0, help="the cosine schedule's final rate (eta_min)")
    ext.add_argument("--lr-warmup-epochs", type=int, default=0,
                     help="epochs of warmup before the main schedule (torchvision's SequentialLR; 0 = none)")
    ext.add_argument("--lr-warmup-method", default="constant", choices=["linear", "constant"],
                     help="linear: LinearLR from --lr-warmup-decay x lr up to lr; constant: ConstantLR at "
                          "--lr-warmup-decay x lr")
    ext.add_argument("--lr-warmup-decay", type=float, default=0.01,
                     help="the warmup's (starting) factor of the rate, in (0, 1]")
    ext.add_argument("--backend", default=None, choices=[None, "gloo", "nccl"],
                     help="rendezvous backend (default: nccl on GPU, gloo on CPU)")
    ext.add_argument("--allreduce", default="auto",
                     choices=["auto", "oneshot", "twoshot", "nvls", "nccl"],
                     help="gradient all-reduce algorithm (nccl = library baseline)")
    ext.add_argument("--wire-dtype", default="bf16", choices=["bf16", "fp32"])
    ext.add_argument("--bucket-mb", type=float, default=32.0)
    ext.add_argument("--pipeline", default="auto", choices=["auto", "fused", "stream", "reference"],
                     help="input pipeline: fused GPU augment over a decoded uint8 cache (any image sizes, "
                          "resampled as PIL does), stream (no cache: each batch's JPEGs entropy-decoded on host "
                          "threads, IDCT and colour conversion on the GPU, for splits larger than host memory), "
                          "the reference's per-sample PIL transforms, or auto (fused when the split has one image "
                          "size and fits in host memory)")
    ext.add_argument("--decode-threads", type=int, default=8,
                     help="host threads decoding images: the fused pipeline's cache build, the stream pipeline's "
                          "per-batch decode")
    ext.add_argument("--pretrained", default=None,
                     help="path to a torchvision vgg16 state dict (offline pretrained=True)")
    ext.add_argument("--save", default=None, help="checkpoint path written by rank 0 every epoch")
    ext.add_argument("--resume", default=None, help="checkpoint path to resume from")
    ext.add_argument("--seed", type=int, default=0)
    ext.add_argument("--deterministic", action="store_true",
                     help="bit-reproducible training: two runs of the same command on the same GPU model, world size "
                          "and build give identical weights, optimizer state and losses.  Native engine: split-K and "
                          "column sums are reduced in a fixed order instead of with fp32 atomics (slightly slower; "
                          "refuses --allreduce nvls).  Torch-op engine: torch.use_deterministic_algorithms(True)")
    ext.add_argument("--synthetic", type=int, default=0,
                     help="generate a synthetic ImageFolder with this many train images per class "
                          "under --root_dir if it does not exist")
    ext.add_argument("--socket-ifname", default=None,
                     help="network interface for the rendezvous / gloo / NCCL bootstrap sockets (the reference "
                          "hard-codes GLOO_SOCKET_IFNAME=eth0, distributedVggf.py:296; default: auto-detect)")
    ext.add_argument("--eval-only", action="store_true",
                     help="one validation pass (typically with --resume <checkpoint>) and exit")
    ext.add_argument("--zero1", default="auto", choices=["auto", "on", "off"],
                     help="shard the Adam state of the FC weights (88 %% of the parameters) across the ranks of one "
                          "NVLink domain: reduce-scatter + optimizer + all-gather of the new bf16 weights in ONE "
                          "kernel per bucket (auto: from 4 ranks up)")
    ext.add_argument("--reference-order", action="store_true",
                     help="replay the reference's identical-shuffle-every-epoch behaviour")
    ext.add_argument("--shard-eval", action="store_true",
                     help="shard validation across ranks and all-reduce the metrics")
    ext.add_argument("--class-weights", default=None,
                     help="comma-separated per-class loss weights (the reference's commented-out "
                          "CLASS_OPTIM_WEIGHTS, distributedUtil.py:27-28)")
    ext.add_argument("--profile", default=None, choices=[None, "events", "nvtx", "timeline"],
                     help="events: per-phase CUDA-event timings each epoch; nvtx: emit NVTX ranges; timeline: print, for "
                          "the last training step of every epoch, when each layer's kernels and each bucket's reduction / "
                          "update finished (CUDA events, ms since the start of the step; native engine)")
    ext.add_argument("--log-jsonl", default=None, help="append one JSON record per epoch")
    ext.add_argument("--label-smoothing", type=float, default=0.0,
                     help="label smoothing of the training loss, 0 <= eps < 1 (torchvision's --label-smoothing; "
                          "0 = off).  The test loss stays plain cross-entropy")
    ext.add_argument("--mixup-alpha", type=float, default=0.0,
                     help="MixUp every training batch with lam ~ Beta(alpha, alpha) (torchvision's --mixup-alpha; 0 = off)")
    ext.add_argument("--cutmix-alpha", type=float, default=0.0,
                     help="CutMix every training batch with lam ~ Beta(alpha, alpha) (torchvision's --cutmix-alpha; "
                          "0 = off).  With both alphas > 0 each batch takes one of the two with probability 1/2")
    ext.add_argument("--accum-steps", type=int, default=1,
                     help="gradient accumulation: one optimizer update (and one gradient all-reduce) per K "
                          "mini-batches and after the last one of an epoch, with the mean of their gradients")
    ext.add_argument("--model-ema", action="store_true",
                     help="keep an exponential moving average of the weights (torchvision's --model-ema), evaluate it "
                          "every epoch after the raw weights and save it in the checkpoint")
    ext.add_argument("--model-ema-steps", type=int, default=32,
                     help="update the EMA after every N-th optimizer update of an epoch, from its first (default 32)")
    ext.add_argument("--freeze-layers", type=int, default=0,
                     help="fine-tune with the first N layers of the model frozen (convolutions, then Linears; VGG-F: "
                          "13 = all of features, 16 = only the last Linear trains), 0 <= N < number of layers.  "
                          "Frozen layers run forward in train mode and get no gradient, no exchange, no optimizer "
                          "state and no weight decay (torch's requires_grad_(False)); the EMA still averages them "
                          "(default 0 = everything trains)")
    ext.add_argument("--powersgd-rank", type=int, default=0,
                     help="compress the gradient exchange with PowerSGD at this rank, 1 <= r <= 8 (torch's "
                          "powerSGD_hook with error feedback and warm start, one bucket per tensor): every weight matrix "
                          "where it pays goes over the wire as rank-r fp32 factors P and Q (default 0 = off)")
    ext.add_argument("--powersgd-start-iter", type=int, default=1000,
                     help="optimizer updates exchanged uncompressed before PowerSGD starts, >= 2 (torch's "
                          "start_powerSGD_iter; default 1000)")
    ext.add_argument("--train-resize-size", type=int, default=DATA.resize,
                     help="size of the training RandomResizedCrop (default %d, the reference's)" % DATA.resize)
    ext.add_argument("--train-crop-size", type=int, default=DATA.crop,
                     help="CenterCrop after rotation and flip: the network's training input, <= --train-resize-size "
                          "(torchvision's --train-crop-size; default %d).  The native engine takes multiples of 8 from "
                          "64 to 512" % DATA.crop)
    ext.add_argument("--val-resize-size", type=int, default=DATA.resize,
                     help="Resize of the shorter side for validation (torchvision's --val-resize-size; default %d)"
                          % DATA.resize)
    ext.add_argument("--val-crop-size", type=int, default=DATA.crop,
                     help="CenterCrop after it: the network's evaluation input, <= --val-resize-size (torchvision's "
                          "--val-crop-size; default %d).  Training and evaluation sizes may differ (FixRes: e.g. "
                          "--train-crop-size 176 --val-resize-size 232 --val-crop-size 224)" % DATA.crop)
    ext.add_argument("--val-tta", default="none", choices=["none", "flip", "five-crop", "ten-crop"],
                     help="test-time augmentation of every validation pass: several --val-crop-size views of the "
                          "Resize(--val-resize-size) image, scored by the mean of their softmaxes.  flip: the centre "
                          "crop and its mirror image; five-crop: torchvision's five_crop; ten-crop: its ten_crop "
                          "(the five and those of the mirrored image).  Training does not change (default: none)")
    # SUPPRESS: without the flag the namespace (printed, and saved in checkpoints) is the one of earlier versions
    ext.add_argument("--val-metrics", action="store_true", default=argparse.SUPPRESS,
                     help="every validation pass also counts a confusion matrix (rows labels, columns predictions) and, "
                          "with more than 5 classes, the top-5 hits on the GPU, and reports balanced accuracy, acc@5 "
                          "and, up to 32 classes, per-class support, recall, precision and confusion row; the JSONL "
                          "records get test_confusion, test_recall, ... (default: off)")
    ext.add_argument("--model-ema-decay", type=float, default=0.99998,
                     help="EMA decay per image seen, 0 <= d < 1; the decay of one update is adjusted as torchvision "
                          "does: 1 - min(1, (1 - d) * world * mini_batch * accum_steps * model_ema_steps / epochs)")
    ext.add_argument("--distill-teacher", default=None,
                     help="knowledge distillation: train against the logits of this teacher as well as the labels.  A "
                          "checkpoint of this project (--save) or a plain state dict with torchvision names, loaded "
                          "whole (every tensor, right shapes, the student's class count).  The teacher runs in eval "
                          "mode on the student's augmented input; the train loss is (1 - alpha) CE + alpha T^2 "
                          "KL(softmax(teacher / T) || softmax(student / T)); the test loss stays plain cross-entropy "
                          "(default: off)")
    ext.add_argument("--distill-teacher-model", default=None, choices=MODELS,
                     help="the teacher's layer table (default: the checkpoint's --model, else the student's)")
    ext.add_argument("--distill-alpha", type=float, default=0.5,
                     help="weight of the distillation term, 0 < alpha <= 1 (default 0.5)")
    ext.add_argument("--distill-temperature", type=float, default=4.0,
                     help="softmax temperature T of the distillation term, finite and > 0 (default 4.0)")
    return parser


def check_sizes(args) -> Optional[str]:
    """What is wrong with the four input sizes, or None."""
    for split in ("train", "val"):
        resize, crop = getattr(args, split + "_resize_size"), getattr(args, split + "_crop_size")
        if crop < MIN_CROP:
            return "--%s-crop-size must be >= %d (got %d): the fifth 2x2 max-pool would leave an empty map" % (
                split, MIN_CROP, crop)
        if crop > resize:
            return "--%s-crop-size %d exceeds --%s-resize-size %d: the crop must lie inside the resized image" % (
                split, crop, split, resize)
    return None


def input_sizes(args) -> dict:
    """The four input sizes of a run (an args namespace without them: the reference's)."""
    return {k: int(getattr(args, k, DATA.resize if k.endswith("resize_size") else DATA.crop))
            for k in ("train_resize_size", "train_crop_size", "val_resize_size", "val_crop_size")}


def parse_command_line(argv: Optional[Sequence[str]] = None, init: bool = True):
    """Parse, print the namespace (as the reference does) and join the process group."""
    args = build_parser().parse_args(argv)
    if args.root_dir is None:
        build_parser().error("the following arguments are required: -rd/--root_dir")
    if args.accum_steps < 1:
        build_parser().error("--accum-steps must be >= 1")
    if not 0.0 <= args.label_smoothing < 1.0:
        build_parser().error("--label-smoothing must lie in [0, 1)")
    if args.mixup_alpha < 0.0 or args.cutmix_alpha < 0.0:
        build_parser().error("--mixup-alpha and --cutmix-alpha must be >= 0")
    if args.model_ema_steps < 1:
        build_parser().error("--model-ema-steps must be >= 1")
    if not 0.0 <= args.model_ema_decay < 1.0:
        build_parser().error("--model-ema-decay must lie in [0, 1)")
    if not args.weight_decay >= 0.0 or (args.bias_weight_decay is not None and not args.bias_weight_decay >= 0.0):
        build_parser().error("--weight-decay and --bias-weight-decay must be >= 0")
    if args.optimizer in ("lamb", "lars"):
        from .utils.optim import check_layerwise_decay
        try:
            check_layerwise_decay(args.optimizer, args.weight_decay)
        except ValueError as e:
            build_parser().error(str(e))
        if args.zero1 == "on" and args.world_size > 1:
            build_parser().error("--optimizer %s with --zero1 on: ZeRO-1 shards a tensor across ranks, and its trust "
                                 "ratio needs the whole tensor's norms; use --zero1 off (or auto)" % args.optimizer)
    if args.lr_warmup_epochs < 0:
        build_parser().error("--lr-warmup-epochs must be >= 0")
    if args.lr_scheduler == "cosine" and args.lr_warmup_epochs >= args.epochs:
        build_parser().error("--lr-scheduler cosine needs --lr-warmup-epochs < --epochs")
    if not 0.0 < args.lr_warmup_decay <= 1.0:
        build_parser().error("--lr-warmup-decay must lie in (0, 1]")
    if not args.lr_min >= 0.0:
        build_parser().error("--lr-min must be >= 0")
    err = check_sizes(args)
    if err:
        build_parser().error(err)
    if args.distill_teacher is not None:
        if not 0.0 < args.distill_alpha <= 1.0:
            build_parser().error("--distill-alpha must lie in (0, 1]")
        if not (math.isfinite(args.distill_temperature) and args.distill_temperature > 0.0):
            build_parser().error("--distill-temperature must be finite and > 0")
        if args.eval_only:
            build_parser().error("--distill-teacher trains a student; --eval-only scores a checkpoint (drop the teacher)")
    if args.freeze_layers:
        from .models.vggf import get_spec
        try:
            get_spec(args.model, args.num_classes or 3).check_freeze_layers(args.freeze_layers)
        except ValueError as e:
            build_parser().error("%s (%s)" % (e, args.model))
    if args.powersgd_rank:
        from .parallel import powersgd
        try:
            powersgd.check_config(args.powersgd_rank, args.powersgd_start_iter)
            powersgd.resolve_zero1({"auto": "auto", "on": True, "off": False}[args.zero1], args.powersgd_rank)
            powersgd.check_deterministic(args.powersgd_rank, args.deterministic, args.world_size)
        except ValueError as e:
            build_parser().error(str(e))
    print(args)
    if args.socket_ifname:
        os.environ["GLOO_SOCKET_IFNAME"] = args.socket_ifname
        os.environ.setdefault("NCCL_SOCKET_IFNAME", args.socket_ifname)
    if init and args.world_size > 1:
        from .parallel.process_group import init_distributed, pick_device

        device = pick_device(args.rank, args.no_cuda)
        init_distributed(args.init_url, args.rank, args.world_size, device, args.backend)
    return args


def main(argv: Optional[Sequence[str]] = None) -> int:
    from .train import manage_training

    args = parse_command_line(argv)
    from .parallel.process_group import shutdown
    from .parallel.watchdog import start_abort_watch

    watch = start_abort_watch(args.rank)          # None for single-process runs
    try:
        manage_training(args)
    except BaseException as e:                    # tell the peers before going down (they may be
        if watch is not None:                     # blocked in a collective this rank will never join)
            watch.signal("%s: %s" % (type(e).__name__, e))
            watch.stop()
        shutdown(graceful=False)
        raise
    if watch is not None:
        watch.stop()
    shutdown()
    return 0


if __name__ == "__main__":
    sys.exit(main())
