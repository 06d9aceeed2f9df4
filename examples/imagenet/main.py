"""ImageNet training with any algorithm — the command line of the reference's examples/imagenet/main.py:32-178 (``DIR``,
-a/--arch, -j/--workers, --epochs, --start-epoch, -b/--batch-size, --lr, --momentum, --wd, --milestones, --gama, --warmup-epochs,
-p/--print-freq, --resume, --save-checkpoint, -e/--evaluate, --pretrained, --seed, --amp, --prof, --algorithm,
--async-sync-interval, --async-warmup-steps) plus what is specific to this framework (--fused-shard, --fuse-optimizer, --dtype,
--synthetic and its shape flags, --cpu).

    python -m bagua_b200.distributed.launch --nproc_per_node=8 examples/imagenet/main.py -a resnet50 /data/imagenet --save-checkpoint
    python -m bagua_b200.distributed.launch --nproc_per_node=8 examples/imagenet/main.py -a vgg16 --synthetic --fused-shard

Recipe of the reference: SGD with momentum, multi-step decay (``lr · gama^(milestones passed)``) with a per-iteration linear
warm-up over ``--warmup-epochs`` (:562-581), top-1 / top-5 on the validation set after every epoch, the best top-1 kept next to
the latest checkpoint, the async algorithm resumed / aborted around every epoch (:326-334), ``--prof N`` wraps iterations in
NVTX ranges and brackets N..N+10 with cudaProfilerStart/Stop.

H100-first differences: parameters and activations are bf16 channels-last by default (``--dtype fp32`` restores the reference's
precision; ``--amp`` keeps fp32 parameters and runs the forward under bf16 autocast — no loss scaling needed, bf16 has fp32's
exponent range); batches are staged through pinned memory on a side stream (``bagua_b200.utils.data.DevicePrefetcher``) instead of
a blocking ``.cuda()`` in the loop; ``--fused-shard`` runs SGD inside the bucket kernels (reduce-scatter → update → all-gather).
``DIR`` expects ``DIR/train`` and ``DIR/val`` in torchvision ImageFolder layout; without it (or with ``--synthetic``) class-
dependent random images are generated so the script runs offline.  ``--batch-size`` is PER GPU (the reference passes its flag
straight to every rank's DataLoader as well, :300-316)."""
import argparse
import bisect
import contextlib
import logging
import os
import random
import shutil
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import bagua_b200 as bagua  # noqa: E402
from bagua_b200.models import get_model  # noqa: E402
from bagua_b200.parallel.algorithms import Algorithm, q_adam  # noqa: E402
from bagua_b200.parallel.algorithms.gradient_allreduce import FusedGradientAllReduceAlgorithm, make_sharded_fused_lars, make_sharded_fused_sgd  # noqa: E402


def parse():
    p = argparse.ArgumentParser(description="bagua_b200 ImageNet training")
    p.add_argument("data_pos", metavar="DIR", nargs="?", default="", help="dataset directory (train/ and val/)")
    p.add_argument("--data", default="", help="same as DIR")
    p.add_argument("-a", "--arch", default="resnet50", help="resnet50 / vgg16 (built in, fused NHWC epilogues) or any torchvision.models name")
    p.add_argument("-j", "--workers", type=int, default=4, metavar="N", help="data loading workers per rank")
    p.add_argument("--epochs", type=int, default=90, metavar="N")
    p.add_argument("--start-epoch", type=int, default=0, metavar="N", help="manual epoch number (useful on restarts)")
    p.add_argument("-b", "--batch-size", type=int, default=32, metavar="N", help="per GPU")
    p.add_argument("--lr", "--learning-rate", dest="lr", type=float, default=0.1, metavar="LR", help="for a global batch of 256; scaled linearly with the global batch")
    p.add_argument("--momentum", type=float, default=0.9, metavar="M")
    p.add_argument("--wd", "--weight-decay", dest="weight_decay", type=float, default=1e-4, metavar="W")
    p.add_argument("--milestones", default="60,70,80", help="epochs at which the learning rate is multiplied by --gama")
    p.add_argument("--gama", "--gamma", dest="gama", type=float, default=0.2)
    p.add_argument("--warmup-epochs", type=int, default=5)
    p.add_argument("-p", "--print-freq", type=int, default=10, metavar="N")
    p.add_argument("--resume", default="", metavar="PATH", help="checkpoint to continue from")
    p.add_argument("--save-checkpoint", action="store_true", default=False, help="rank 0 writes checkpoint.pth.tar (+ model_best.pth.tar) after every epoch")
    p.add_argument("--checkpoint-dir", "--save", dest="checkpoint_dir", default=".")
    p.add_argument("-e", "--evaluate", action="store_true", help="evaluate on the validation set and exit")
    p.add_argument("--pretrained", action="store_true", help="start from torchvision's weights (must already be in the local torch hub cache)")
    p.add_argument("--seed", type=int, default=None)
    p.add_argument("--amp", action="store_true", default=False, help="fp32 parameters, bf16 autocast")
    p.add_argument("--dtype", default="bf16", choices=["bf16", "fp32"], help="parameter / activation dtype when --amp is not given")
    p.add_argument("--prof", type=int, default=-1, help="profile 10 iterations starting at this one, then stop")
    p.add_argument("--algorithm", default="gradient_allreduce", help="gradient_allreduce, bytegrad, decentralized, low_precision_decentralized, qadam, async")
    p.add_argument("--async-sync-interval", type=int, default=500)
    p.add_argument("--async-warmup-steps", type=int, default=100)
    p.add_argument("--fused-shard", action="store_true", help="SGD inside the bucket kernels (reduce-scatter → update → all-gather); with "
                   "--optimizer lars the sharded LARS (reduce-scatter in the buckets, update in step())")
    p.add_argument("--optimizer", default="sgd", choices=["sgd", "lars"], help="momentum SGD, or LARS for large global batches (BatchNorm "
                   "and bias parameters get no weight decay and no layer adaptation)")
    p.add_argument("--trust-coefficient", type=float, default=1e-3, help="LARS trust coefficient (eta)")
    p.add_argument("--ema-decay", type=float, default=None, help="with --fused-shard: keep a sharded fp32 EMA of the weights with this decay; "
                   "validation then also reports the EMA weights' accuracy, and checkpoints carry the EMA in the optimizer state")
    p.add_argument("--ema-every", type=int, default=1, help="update the EMA on every N-th optimizer step")
    p.add_argument("--fuse-optimizer", action="store_true", help="generic fused optimizer (bagua.contrib.fuse_optimizer)")
    p.add_argument("--synthetic", action="store_true")
    p.add_argument("--steps-per-epoch", type=int, default=100, help="synthetic data only")
    p.add_argument("--num-classes", type=int, default=1000)
    p.add_argument("--image-size", type=int, default=224)
    p.add_argument("--cpu", action="store_true")
    args = p.parse_args()
    args.data = args.data or args.data_pos
    if args.ema_decay is not None and not args.fused_shard:
        p.error("--ema-decay needs --fused-shard")
    args.milestone_list = sorted(int(m) for m in args.milestones.split(",") if m.strip())
    return args


class Meter:
    """Running average with the reference's ``name val (avg)`` display (:510-533)."""

    def __init__(self, name, fmt=":f"):
        self.name, self.fmt, self.val, self.sum, self.count = name, fmt, 0.0, 0.0, 0

    def update(self, val, n=1):
        self.val = float(val)
        self.sum += float(val) * n
        self.count += n

    @property
    def avg(self):
        return self.sum / max(self.count, 1)

    def __str__(self):
        return ("{name} {val" + self.fmt + "} ({avg" + self.fmt + "})").format(name=self.name, val=self.val, avg=self.avg)


def show(prefix, i, total, meters):
    width = len(str(total))
    logging.info("\t".join([f"{prefix}[{i:>{width}}/{total}]"] + [str(m) for m in meters]))


class SyntheticImages(torch.utils.data.Dataset):
    def __init__(self, n, classes, size, seed):
        self.n, self.classes, self.size, self.seed = n, classes, size, seed

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1_000_003 + i)
        y = int(torch.randint(0, self.classes, (1,), generator=g))
        return torch.randn(3, self.size, self.size, generator=g) + (y % 7 - 3) * 0.1, y   # weak class signal


def make_loaders(args, rank, world, cuda):
    if args.data and not args.synthetic:
        import torchvision.datasets as D
        import torchvision.transforms as T

        norm = T.Normalize([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
        train = D.ImageFolder(os.path.join(args.data, "train"), T.Compose([T.RandomResizedCrop(args.image_size), T.RandomHorizontalFlip(), T.ToTensor(), norm]))
        val = D.ImageFolder(os.path.join(args.data, "val"), T.Compose([T.Resize(int(args.image_size * 256 / 224)), T.CenterCrop(args.image_size), T.ToTensor(), norm]))
        workers = args.workers
    else:
        train = SyntheticImages(args.steps_per_epoch * args.batch_size * world, args.num_classes, args.image_size, 1)
        val = SyntheticImages(4 * args.batch_size * world, args.num_classes, args.image_size, 2)
        workers = 0
    ts = torch.utils.data.distributed.DistributedSampler(train, num_replicas=world, rank=rank, shuffle=True)
    vs = torch.utils.data.distributed.DistributedSampler(val, num_replicas=world, rank=rank, shuffle=False)
    kw = dict(batch_size=args.batch_size, num_workers=workers, pin_memory=cuda)
    return torch.utils.data.DataLoader(train, sampler=ts, drop_last=True, **kw), torch.utils.data.DataLoader(val, sampler=vs, **kw), ts


def build_model(args, dev, dtype, cuda):
    if args.pretrained:
        import torchvision.models as tvm

        logging.info("=> using pre-trained model '%s'", args.arch)
        weights = tvm.get_model(args.arch, weights="DEFAULT").state_dict()   # raises when the file is not in the local hub cache: there is no network
        model = get_model(args.arch, num_classes=args.num_classes)
        missing = model.load_state_dict(weights, strict=False)
        logging.info("pre-trained weights loaded (missing %d, unexpected %d)", len(missing.missing_keys), len(missing.unexpected_keys))
    else:
        logging.info("=> creating model '%s'", args.arch)
        model = get_model(args.arch, num_classes=args.num_classes)
    model = model.to(dev).to(dtype)
    return model.to(memory_format=torch.channels_last) if cuda else model


def make_optimizer(args, model, lr, cuda, world):
    if args.algorithm == "qadam":
        opt = q_adam.QAdamOptimizer(model.parameters(), lr=lr * 1e-2, warmup_steps=100)
        return opt, q_adam.QAdamAlgorithm(opt)
    if args.optimizer == "lars":
        if args.algorithm != "gradient_allreduce":
            raise SystemExit("--optimizer lars runs with --algorithm gradient_allreduce")
        # the MLPerf recipe: parameters with ndim <= 1 (BatchNorm, biases) in a weight_decay = 0 group, i.e. plain momentum SGD
        groups = [{"params": [p for p in model.parameters() if p.dim() > 1], "weight_decay": args.weight_decay},
                  {"params": [p for p in model.parameters() if p.dim() <= 1], "weight_decay": 0.0}]
        kw = dict(lr=lr, momentum=args.momentum, trust_coefficient=args.trust_coefficient)
        if args.fused_shard and (cuda or args.ema_decay is not None):
            opt = make_sharded_fused_lars(groups, ema_decay=args.ema_decay, ema_every=args.ema_every, **kw)
            return opt, FusedGradientAllReduceAlgorithm(opt)
        return bagua.ops.FusedLARS(groups, **kw), Algorithm.init(args.algorithm)
    # with --ema-decay also on the CPU: the sharded optimizer's fallback keeps the EMA there
    if args.fused_shard and (cuda or args.ema_decay is not None) and args.algorithm == "gradient_allreduce":
        opt = make_sharded_fused_sgd(model.parameters(), lr=lr, momentum=args.momentum, weight_decay=args.weight_decay, ema_decay=args.ema_decay,
                                     ema_every=args.ema_every)
        return opt, FusedGradientAllReduceAlgorithm(opt)
    if cuda and not args.fuse_optimizer:
        opt = bagua.ops.FusedSGD(model.parameters(), lr=lr, momentum=args.momentum, weight_decay=args.weight_decay)   # one multi-tensor kernel per step
    else:
        opt = torch.optim.SGD(model.parameters(), lr=lr, momentum=args.momentum, weight_decay=args.weight_decay)
    kw = dict(sync_interval_ms=args.async_sync_interval, warmup_steps=args.async_warmup_steps) if args.algorithm == "async" else {}
    return opt, Algorithm.init(args.algorithm, **kw)


def learning_rate(args, base_lr, epoch, step, steps_per_epoch):
    """Multi-step decay with a linear per-iteration warm-up (reference :562-581)."""
    lr = base_lr * args.gama ** bisect.bisect_right(args.milestone_list, epoch)
    if epoch < args.warmup_epochs:
        lr *= (1 + step + epoch * steps_per_epoch) / (args.warmup_epochs * steps_per_epoch)
    return lr


def topk_hits(out, y, ks=(1, 5)):
    pred = out.topk(min(max(ks), out.shape[1]), 1).indices
    hit = pred.eq(y.view(-1, 1))
    return [hit[:, :k].any(1).float().sum() for k in ks]


def main():
    args = parse()
    if args.seed is not None:
        random.seed(args.seed)
        torch.manual_seed(args.seed)
        torch.backends.cudnn.deterministic = True
    else:
        torch.manual_seed(0)
        torch.backends.cudnn.benchmark = True
    cuda = torch.cuda.is_available() and not args.cpu
    if cuda:
        torch.cuda.set_device(bagua.get_local_rank())
    bagua.init_process_group()
    rank, world = bagua.get_rank(), bagua.get_world_size()
    logging.basicConfig(format=f"rank-{rank} %(asctime)s %(levelname)-8s %(message)s", datefmt="%H:%M:%S", level=logging.INFO if rank == 0 else logging.ERROR, stream=sys.stdout)
    dev = torch.device("cuda", bagua.get_local_rank()) if cuda else torch.device("cpu")
    dtype = torch.bfloat16 if (cuda and args.dtype == "bf16" and not args.amp) else torch.float32
    autocast = (lambda: torch.autocast(dev.type, dtype=torch.bfloat16)) if args.amp else contextlib.nullcontext

    model = build_model(args, dev, dtype, cuda)
    base_lr = args.lr * args.batch_size * world / 256.0
    optimizer, algorithm = make_optimizer(args, model, base_lr, cuda, world)
    best_acc1 = 0.0
    if args.resume:
        if os.path.isfile(args.resume):
            logging.info("=> loading checkpoint '%s'", args.resume)
            ck = torch.load(args.resume, map_location=dev)
            args.start_epoch, best_acc1 = ck["epoch"], float(ck.get("best_acc1", 0.0))
            model.load_state_dict(ck["state_dict"])
            if "optimizer" in ck and not args.evaluate:
                optimizer.load_state_dict(ck["optimizer"])   # before with_bagua: the engine broadcasts / re-shards it
            logging.info("=> loaded checkpoint '%s' (epoch %d)", args.resume, ck["epoch"])
        else:
            logging.info("=> no checkpoint found at '%s'", args.resume)
    model = model.with_bagua([optimizer], algorithm)
    if args.fuse_optimizer:
        optimizer = bagua.contrib.fuse_optimizer(optimizer)
    train_loader, val_loader, train_sampler = make_loaders(args, rank, world, cuda)

    def batches(loader):
        """Device batches; on GPUs the next one is already on its way (pinned memory → side stream, cast and layout change there too)."""
        from bagua_b200.utils.data import DevicePrefetcher

        def fix(x, y):
            x = x.to(dtype)
            return (x.contiguous(memory_format=torch.channels_last) if cuda else x), y

        return DevicePrefetcher(loader, dev, transform=fix)

    def nvtx(name):
        return torch.cuda.nvtx.range(name) if (cuda and args.prof >= 0) else contextlib.nullcontext()

    def validate(epoch):
        """Acc@1 of the live weights and, with --ema-decay, of the EMA weights (BatchNorm statistics stay the live model's)."""
        acc1 = score(epoch, "")
        if args.ema_decay is not None:
            with optimizer.ema_weights():   # collective: every rank validates its shard of the set
                score(epoch, "EMA ")
        return acc1

    @torch.no_grad()
    def score(epoch, label):
        model.eval()
        tot = torch.zeros(4, device=dev)   # top-1 hits, top-5 hits, samples, summed loss
        t0 = time.time()
        for i, (x, y) in enumerate(batches(val_loader)):
            with autocast():
                out = model(x).float()
            h1, h5 = topk_hits(out, y)
            tot += torch.stack([h1, h5, torch.tensor(float(len(y)), device=dev), F.cross_entropy(out, y, reduction="sum")])
            if i % args.print_freq == 0:
                logging.info("Test: [%d/%d]\tTime %.3f", i, len(val_loader), time.time() - t0)
        bagua.allreduce_inplace(tot, op=bagua.ReduceOp.SUM)   # every rank scored its own shard of the validation set
        acc1, acc5 = (100.0 * tot[0] / tot[2]).item(), (100.0 * tot[1] / tot[2]).item()
        logging.info(" * Epoch %d %sAcc@1 %.3f %sAcc@5 %.3f Loss %.4f", epoch, label, acc1, label, acc5, (tot[3] / tot[2]).item())
        return acc1

    def train(epoch):
        """One epoch; returns False when a --prof window has ended the run."""
        model.train()
        meters = [Meter("Time", ":6.3f"), Meter("Data", ":6.3f"), Meter("Loss", ":.4e"), Meter("Acc@1", ":6.2f"), Meter("Acc@5", ":6.2f"), Meter("img/s", ":8.0f")]
        bt, dt, lm, a1, a5, ips = meters
        n_steps = len(train_loader)
        end = time.time()
        for i, (x, y) in enumerate(batches(train_loader)):
            if args.prof >= 0 and i == args.prof and cuda:
                logging.info("Profiling begun at iteration %d", i)
                torch.cuda.cudart().cudaProfilerStart()
            dt.update(time.time() - end)
            for g in optimizer.param_groups:
                g["lr"] = learning_rate(args, base_lr, epoch, i, n_steps)
            with nvtx(f"Body of iteration {i}"):
                optimizer.zero_grad()
                with nvtx("forward"), autocast():
                    out = model(x)
                    loss = F.cross_entropy(out.float(), y)
                with nvtx("backward"):
                    loss.backward()
                with nvtx("optimizer.step()"):
                    optimizer.fuse_step() if args.fuse_optimizer else optimizer.step()
            if i % args.print_freq == 0:   # the only host syncs of the loop: every --print-freq iterations
                h1, h5 = topk_hits(out.detach().float(), y)
                lm.update(loss.item(), len(y))
                a1.update(100.0 * h1.item() / len(y), len(y))
                a5.update(100.0 * h5.item() / len(y), len(y))
                bt.update(time.time() - end)
                ips.update(len(y) * world / max(bt.val, 1e-9))
                show(f"Epoch: [{epoch}]", i, n_steps, meters)
            else:
                bt.update(time.time() - end)
            end = time.time()
            if args.prof >= 0 and i == args.prof + 10:
                logging.info("Profiling ended at iteration %d", i)
                if cuda:
                    torch.cuda.cudart().cudaProfilerStop()
                return False
        return True

    if args.evaluate:
        validate(args.start_epoch)
        return
    for epoch in range(args.start_epoch, args.epochs):
        train_sampler.set_epoch(epoch)
        if args.algorithm == "async":
            model.bagua_algorithm.resume(model)
        finished = train(epoch)
        if args.algorithm == "async":
            model.bagua_algorithm.abort(model)
        if not finished:
            break
        acc1 = validate(epoch)
        is_best, best_acc1 = acc1 > best_acc1, max(acc1, best_acc1)
        state = {"epoch": epoch + 1, "arch": args.arch, "state_dict": model.state_dict(), "best_acc1": best_acc1, "optimizer": optimizer.state_dict()}
        if rank == 0 and args.save_checkpoint:   # optimizer.state_dict() above is collective for sharded optimizers: every rank built it
            os.makedirs(args.checkpoint_dir, exist_ok=True)
            path = os.path.join(args.checkpoint_dir, "checkpoint.pth.tar")
            torch.save(state, path + ".tmp")
            os.replace(path + ".tmp", path)
            if is_best:
                shutil.copyfile(path, os.path.join(args.checkpoint_dir, "model_best.pth.tar"))


if __name__ == "__main__":
    main()
