#!/usr/bin/env python
"""Distributed synchronous SGD on (synthetic) MNIST -- the reference's ``train_dist.py`` scenario.

    python examples/train_mnist.py                       # CPU, gloo, world 2 (the reference default)
    python examples/train_mnist.py --backend b200 --size 8     # one process per GPU, fused engine
    python examples/train_mnist.py --backend b200 --size 8 --global-batch 32768   # large batch: wgmma batched engine
    python examples/train_mnist.py --backend b200 --size 8 --eval   # + test loss / accuracy after every epoch
    python examples/train_mnist.py --backend b200 --size 8 --weight-decay 5e-4 --nesterov   # torch.optim.SGD's options
    python examples/train_mnist.py --backend b200 --size 1 --global-batch 4096 --lr 0.32 --max-grad-norm 1.0   # clip_grad_norm_
    python examples/train_mnist.py --backend b200 --size 1 --global-batch 4096 --lr 0.32 --warmup-epochs 1 \
        --lr-decay cosine --eval                       # large batch: linearly scaled lr, 1 epoch of warmup, cosine decay
    python -m dist_tuto.pth_b200.spawn --size 8 --max-restarts 2 examples/train_mnist.py --external --backend b200 \
        --checkpoint run.pt --checkpoint-every 1       # supervised: a failed job is restarted and resumes from run.pt
    torchrun --nproc-per-node 8 examples/train_mnist.py --backend b200 --external

Prints ``Rank r, epoch e: mean loss`` per epoch like train_dist.py:125-127."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import dist_tuto.pth_b200 as dist  # noqa: E402

import json  # noqa: E402


def schedule_from(CFG):
    """The LRSchedule (epoch units) of the --warmup-* / --lr-* flags; None with the defaults (constant lr)."""
    if CFG["warmup_epochs"] == 0 and CFG["lr_decay"] == "constant":
        return None
    kw = {}
    if CFG["lr_decay"] == "multistep":
        kw = dict(milestones=CFG["lr_milestones"], gamma=CFG["lr_gamma"])
    elif CFG["lr_decay"] == "cosine":
        kw = dict(total_steps=CFG["epochs"], min_factor=CFG["lr_min_factor"])
    return dist.LRSchedule(warmup_steps=CFG["warmup_epochs"], warmup_start=CFG["warmup_start"], decay=CFG["lr_decay"],
                           unit="epoch", **kw)


def run(rank, size):
    CFG = json.loads(os.environ["B2_TRAIN_CFG"])          # spawned ranks re-import this file: pass the CLI through the env
    resume = CFG["resume"]
    if resume is None and CFG["ckpt"] and int(os.environ.get("B200DIST_RESTART_COUNT", "0")) > 0 and os.path.exists(CFG["ckpt"]):
        resume = CFG["ckpt"]                              # restarted by the launcher: continue from our own last checkpoint
    cfg = dist.TrainConfig(epochs=CFG["epochs"], lr=CFG["lr"], max_steps=CFG["max_steps"], checkpoint=CFG["ckpt"],
                           checkpoint_every=CFG["ckpt_every"], resume=resume, global_batch=CFG["global_batch"],
                           engine=CFG["engine"], trace=CFG["trace"],
                           eval_dataset="default" if CFG["eval"] else None, eval_every=CFG["eval_every"],
                           lr_schedule=schedule_from(CFG), weight_decay=CFG["weight_decay"], nesterov=CFG["nesterov"],
                           max_grad_norm=CFG.get("max_grad_norm"))
    out = dist.train(rank, size, cfg)
    if rank == 0:
        print(f"{out['steps']} steps, {out['samples_per_s']:.0f} samples/s (wall clock, whole job)")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=2)
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--lr", type=float, default=0.01)
    ap.add_argument("--max-steps", type=int, default=None)
    ap.add_argument("--checkpoint", default=None)
    ap.add_argument("--checkpoint-every", type=int, default=None, help="also checkpoint after every N-th epoch")
    ap.add_argument("--resume", default=None)
    ap.add_argument("--trace", default=None, help="write a Chrome / Perfetto trace of all ranks to this file")
    ap.add_argument("--global-batch", type=int, default=128, help="split over the ranks (train_dist.py:85: 128 // world)")
    ap.add_argument("--engine", default="auto", choices=["auto", "torch", "fused", "batched"])
    ap.add_argument("--external", action="store_true", help="rank/size from torchrun/mpirun env")
    ap.add_argument("--eval", action="store_true",
                    help="test loss / accuracy on the MNIST test split (or its synthetic stand-in) after every "
                         "--eval-every-th epoch and after the last one")
    ap.add_argument("--eval-every", type=int, default=1, help="with --eval: evaluate after every N-th epoch (default 1)")
    ap.add_argument("--warmup-epochs", type=float, default=0.0, help="linear lr warmup over this many epochs (default 0)")
    ap.add_argument("--warmup-start", type=float, default=1.0 / 3.0, help="lr factor at the first warmup step (default 1/3)")
    ap.add_argument("--lr-decay", default="constant", choices=["constant", "multistep", "cosine"],
                    help="after the warmup: constant lr, x gamma at each milestone, or cosine to --lr-min-factor at the end")
    ap.add_argument("--lr-milestones", type=float, nargs="*", default=[], help="multistep: epochs at which lr *= gamma")
    ap.add_argument("--lr-gamma", type=float, default=0.1, help="multistep: factor per milestone (default 0.1)")
    ap.add_argument("--lr-min-factor", type=float, default=0.0, help="cosine: final lr factor (default 0)")
    ap.add_argument("--weight-decay", type=float, default=0.0, help="L2 weight decay on every parameter (default 0)")
    ap.add_argument("--nesterov", action="store_true", help="Nesterov momentum")
    ap.add_argument("--max-grad-norm", type=float, default=None,
                    help="clip the averaged gradient to this L2 norm before every update (default: no clipping)")
    a = ap.parse_args()
    os.environ["B2_TRAIN_CFG"] = json.dumps(dict(epochs=a.epochs, lr=a.lr, max_steps=a.max_steps, ckpt=a.checkpoint, ckpt_every=a.checkpoint_every, resume=a.resume, trace=a.trace,
                                                 global_batch=a.global_batch, engine=a.engine, eval=a.eval,
                                                 eval_every=a.eval_every, warmup_epochs=a.warmup_epochs,
                                                 warmup_start=a.warmup_start, lr_decay=a.lr_decay,
                                                 lr_milestones=a.lr_milestones, lr_gamma=a.lr_gamma,
                                                 lr_min_factor=a.lr_min_factor, weight_decay=a.weight_decay,
                                                 nesterov=a.nesterov, max_grad_norm=a.max_grad_norm))
    if a.external:
        dist.init_from_env(run, backend=a.backend)
    else:
        dist.launch(run, size=a.size, backend=a.backend)
