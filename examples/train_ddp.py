#!/usr/bin/env python
"""Your own model, data-parallel: ``DistributedDataParallel`` + ``FlatSGD`` (or ``FlatAdamW``, ``FlatRMSprop``,
``FlatAdafactor``, ``FlatLAMB``, ``FlatLARS``) in the tutorial's loop, on synthetic data.

    python examples/train_ddp.py                                  # CPU, gloo, world 2
    python examples/train_ddp.py --sharded-optimizer              # momentum sharded over the ranks (ZeRO stage 1)
    python examples/train_ddp.py --backend b200 --size 8 --sharded-optimizer   # one process per GPU: per bucket ONE kernel
                                                                  # reduces, updates the owned slice and gathers the parameters
    python examples/train_ddp.py --optimizer adamw [--sharded-optimizer]   # FlatAdamW; sharded: both moments 1/size per rank
    python examples/train_ddp.py --optimizer adafactor            # FlatAdafactor: factored second moments (unsharded)
    python examples/train_ddp.py --optimizer rmsprop              # FlatRMSprop with torchvision's alpha 0.9, eps 0.0316,
                                                                  # momentum 0.9
    python examples/train_ddp.py --optimizer lamb                 # FlatLAMB / FlatLARS (--optimizer lars): per-tensor trust
                                                                  # ratios for large global batches
    python examples/train_ddp.py --backend b200 --size 1 --cuda-graph   # capturable=True: warm-up steps, then every step
                                                                  # is one replay of a captured CUDA graph
    python examples/train_ddp.py --accumulation-steps 4           # gradient accumulation: 4 micro-batches per step, the
                                                                  # first 3 backwards under model.no_sync()
    python examples/train_ddp.py --ema-decay 0.99 --ema-every 2   # FlatEMA: an EMA of the weights, updated after every
                                                                  # 2nd step, evaluated on a held-out batch at the end
    python examples/train_ddp.py --amp                            # fp16 autocast with torch.amp.GradScaler: the optimizer
                                                                  # unscales, and skips steps whose gradients overflow

The loop is ``backward(); average_gradients(model); optimizer.step()`` either way; with ``--accumulation-steps k`` the k - 1
backwards before the last run inside ``model.no_sync()`` on losses scaled by 1 / k.  With ``--sharded-optimizer`` the update
happens inside ``average_gradients`` (during backward, bucket by bucket) and ``step()`` only counts the step; with fp32
gradient buckets the parameters are bit for bit the same.  Prints ``Rank r, step s: loss`` for the last step, and with
``--ema-decay`` a second line per rank, ``Rank r, EMA model: held-out loss``, the loss of the EMA weights on a fixed batch."""
import argparse
import contextlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn as nn  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import dist_tuto.pth_b200 as dist  # noqa: E402


class SmallConvNet(nn.Module):
    """A generic model (not the library's fused MNIST Net): two convolutions and two linear layers."""

    def __init__(self):
        super().__init__()
        self.conv1, self.conv2 = nn.Conv2d(3, 16, 3, padding=1), nn.Conv2d(16, 32, 3, padding=1)
        self.fc1, self.fc2 = nn.Linear(32 * 4 * 4, 64), nn.Linear(64, 10)

    def forward(self, x):
        x = F.max_pool2d(F.relu(self.conv1(x)), 2)
        x = F.max_pool2d(F.relu(self.conv2(x)), 2)
        return self.fc2(F.relu(self.fc1(x.flatten(1))))


def batch(step, rank, dev, micro=0):
    # every rank its own part of the global batch; micro-batch 0 is the whole batch without accumulation
    g = torch.Generator().manual_seed(1000 * step + rank + 1_000_003 * micro)
    return torch.randn(16, 3, 16, 16, generator=g).to(dev), torch.randint(0, 10, (16,), generator=g).to(dev)


def train_step(model, optimizer, micro_batches, ema=None, scaler=None):
    """One optimizer step over ``micro_batches`` (a list of (x, y)): all but the last backward accumulate under no_sync(),
    the last one exchanges the buckets; then the EMA update, if any.  With ``scaler`` (--amp) the forwards run under fp16
    autocast, the losses are scaled, and ``scaler.step`` / ``scaler.update`` replace ``optimizer.step()``: the optimizer
    unscales the gradients and skips a step that overflowed.  Returns the last micro-batch's loss."""
    k = len(micro_batches)
    amp = contextlib.nullcontext() if scaler is None else torch.autocast(micro_batches[0][0].device.type, dtype=torch.float16)
    scale = (lambda t: t) if scaler is None else scaler.scale
    for x, y in micro_batches[:-1]:
        with model.no_sync():
            with amp:
                part = F.cross_entropy(model(x), y) / k
            scale(part).backward()
    x, y = micro_batches[-1]
    with amp:
        loss = F.cross_entropy(model(x), y)
    scale(loss / k).backward()
    dist.average_gradients(model)       # --sharded-optimizer: the parameters are updated when this returns
    if scaler is None:
        optimizer.step()
    else:
        scaler.step(optimizer)
        scaler.update()
    if ema is not None:
        ema.update()                    # a capturable optimizer: the kernel decides skip / copy / lerp from its step counter
    return loss


def train_graphed(model, optimizer, ema, rank, dev, steps, k, warmup=3, scaler=None):
    """--cuda-graph: ``warmup`` eager steps on a side stream (as torch requires before a capture), one step (all k
    micro-batches) captured, and every later step a ``copy_`` of its micro-batches into the static inputs and one replay.
    Returns the last step's loss."""
    static = [tuple(t.clone() for t in batch(0, rank, dev, j)) for j in range(k)]

    def load(i):
        for j, (x, y) in enumerate(static):
            for t, src in zip((x, y), batch(i, rank, dev, j)):
                t.copy_(src)

    def step():
        return train_step(model, optimizer, static, ema, scaler)

    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        for i in range(min(warmup, steps)):
            load(i)
            loss = step()
    torch.cuda.current_stream(dev).wait_stream(s)
    if steps <= warmup:
        return loss
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss = step()
    for i in range(warmup, steps):
        load(i)
        graph.replay()
    return loss


def run(rank, size):
    CFG = json.loads(os.environ["B2_DDP_CFG"])            # spawned ranks re-import this file: pass the CLI through the env
    dev = torch.device("cuda", torch.cuda.current_device()) if CFG["backend"] != "gloo" and torch.cuda.is_available() \
        else torch.device("cpu")
    torch.manual_seed(1234)
    model = dist.DistributedDataParallel(SmallConvNet().to(dev), bucket_cap_bytes=64 << 10)
    # --no-decay-bias-norm: biases and norm weights (ndim <= 1) in a group without weight decay, the usual recipe
    groups = [{"params": [p for p in model.parameters() if p.ndim <= 1], "weight_decay": 0.0}] if CFG["no_decay"] else None
    cap = {"capturable": True} if CFG["cuda_graph"] else {}
    if CFG["optimizer"] == "adamw":
        optimizer = dist.FlatAdamW(model, lr=2e-3, weight_decay=1e-2, sharded=CFG["sharded"], param_groups=groups, **cap)
    elif CFG["optimizer"] == "rmsprop":        # torchvision's classification reference: alpha 0.9, eps 0.0316, momentum 0.9
        optimizer = dist.FlatRMSprop(model, lr=1e-3, alpha=0.9, eps=0.0316, momentum=0.9, weight_decay=1e-4,
                                     sharded=CFG["sharded"], param_groups=groups, **cap)
    elif CFG["optimizer"] == "adafactor":      # torch.optim.Adafactor's defaults, with a little decoupled weight decay
        optimizer = dist.FlatAdafactor(model, lr=1e-2, weight_decay=1e-4, param_groups=groups)
    elif CFG["optimizer"] == "lamb":
        optimizer = dist.FlatLAMB(model, lr=2e-3, weight_decay=1e-2, sharded=CFG["sharded"])
    elif CFG["optimizer"] == "lars":
        optimizer = dist.FlatLARS(model, lr=2.0, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-2, sharded=CFG["sharded"])
    else:
        optimizer = dist.FlatSGD(model, lr=0.05, momentum=0.9, weight_decay=1e-4, sharded=CFG["sharded"], param_groups=groups,
                                 **cap)
    ema = None
    if CFG["ema_decay"] is not None:
        ema = dist.FlatEMA(optimizer, decay=CFG["ema_decay"], every=CFG["ema_every"], warmup_steps=CFG["ema_warmup_steps"])
    scaler = torch.amp.GradScaler(dev.type) if CFG.get("amp") else None
    loss = None
    if CFG["cuda_graph"]:
        loss = train_graphed(model, optimizer, ema, rank, dev, CFG["steps"], CFG["accumulation_steps"], scaler=scaler)
    for step in range(0 if CFG["cuda_graph"] else CFG["steps"]):
        optimizer.zero_grad()
        loss = train_step(model, optimizer, [batch(step, rank, dev, j) for j in range(CFG["accumulation_steps"])], ema, scaler)
    total = loss.detach().clone()
    dist.all_reduce(total)
    if CFG["optimizer"] in ("adamw", "lamb"):
        state = f"AdamW moment elements on this rank {sum(m.numel() for m in optimizer.exp_avg_flats + optimizer.exp_avg_sq_flats)}"
    elif CFG["optimizer"] == "rmsprop":
        flats = optimizer.square_avg_flats + optimizer.momentum_buffer_flats + optimizer.grad_avg_flats
        state = f"RMSprop state elements on this rank {sum(m.numel() for m in flats)}"
    elif CFG["optimizer"] == "adafactor":
        state = f"Adafactor state elements on this rank {sum(f.numel() for f in optimizer.state_flats)}"
    else:
        state = f"momentum elements on this rank {sum(m.numel() for m in optimizer.momentum_flats)}"
    print(f"Rank {rank}, step {CFG['steps']}: loss {float(loss.detach()):.6f} (mean over ranks {float(total) / size:.9f}), "
          + state)
    if ema is not None:
        x, y = batch(-1, rank, dev)     # a batch no step trains on
        with ema.average_parameters(), torch.no_grad():
            held_out = F.cross_entropy(model(x), y)
        print(f"Rank {rank}, EMA model: held-out loss {float(held_out):.6f}")
    if scaler is not None:
        print(f"Rank {rank}, loss scale {scaler.get_scale():g}, updates applied {optimizer.steps} of {CFG['steps']}")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=2)
    ap.add_argument("--backend", default="gloo")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--sharded-optimizer", action="store_true",
                    help="sharded=True: each rank keeps the optimizer state of, and updates, 1/size of every bucket")
    ap.add_argument("--optimizer", choices=("sgd", "adamw", "rmsprop", "adafactor", "lamb", "lars"),
                    default="sgd", help="FlatSGD (momentum SGD, the default), FlatAdamW, FlatRMSprop, FlatAdafactor, FlatLAMB or "
                                        "FlatLARS (adafactor unsharded; lamb / lars sharded on --backend b200 only)")
    ap.add_argument("--no-decay-bias-norm", action="store_true",
                    help="sgd / adamw / rmsprop / adafactor: no weight decay on biases and norm weights (a param_groups entry with "
                         "weight_decay=0)")
    ap.add_argument("--cuda-graph", action="store_true",
                    help="sgd / adamw / rmsprop on --backend b200: capturable=True, and every step after the warm-up one graph "
                         "replay")
    ap.add_argument("--accumulation-steps", type=int, default=1,
                    help="micro-batches of 16 samples per rank and optimizer step (gradient accumulation with no_sync())")
    ap.add_argument("--ema-decay", type=float, default=None,
                    help="keep an exponential moving average of the weights (FlatEMA) with this decay")
    ap.add_argument("--ema-every", type=int, default=1, help="with --ema-decay: update the EMA after every k-th step")
    ap.add_argument("--ema-warmup-steps", type=int, default=0,
                    help="with --ema-decay: copy the weights instead of averaging them up to this step")
    ap.add_argument("--amp", action="store_true",
                    help="fp16 autocast and torch.amp.GradScaler (dynamic loss scale; overflowing steps are skipped)")
    a = ap.parse_args()
    if a.amp and a.sharded_optimizer and a.size > 1:
        ap.error("--amp needs an unsharded optimizer when --size > 1: the sharded exchange applies the update during "
                 "backward, before GradScaler can check the gradients")
    if a.accumulation_steps < 1:
        ap.error("--accumulation-steps must be at least 1")
    if a.optimizer == "adafactor" and a.sharded_optimizer:
        ap.error("--optimizer adafactor cannot be sharded: a factored tensor's state is its row and column vectors, which do "
                 "not split along the flat slices of the sharded exchange")
    if a.optimizer in ("lamb", "lars") and a.sharded_optimizer and a.backend != "b200":
        ap.error(f"--optimizer {a.optimizer} is sharded on --backend b200 only: the per-tensor norms of the slices are exchanged "
                 "inside the peer-memory kernels")
    if a.optimizer == "adafactor" and a.cuda_graph:
        ap.error("--optimizer adafactor has no capturable form: --cuda-graph needs sgd / adamw / rmsprop")
    if a.cuda_graph and (a.optimizer not in ("sgd", "adamw", "rmsprop") or a.backend != "b200"):
        ap.error("--cuda-graph is for --optimizer sgd / adamw / rmsprop on --backend b200 (CUDA)")
    if a.no_decay_bias_norm and a.optimizer not in ("sgd", "adamw", "rmsprop", "adafactor"):
        ap.error("--no-decay-bias-norm is for --optimizer sgd / adamw / rmsprop / adafactor; FlatLAMB and FlatLARS exclude them already")
    os.environ["B2_DDP_CFG"] = json.dumps(dict(backend=a.backend, steps=a.steps, sharded=a.sharded_optimizer,
                                                optimizer=a.optimizer, no_decay=a.no_decay_bias_norm,
                                                cuda_graph=a.cuda_graph, accumulation_steps=a.accumulation_steps,
                                                ema_decay=a.ema_decay, ema_every=a.ema_every,
                                                ema_warmup_steps=a.ema_warmup_steps, amp=a.amp))
    dist.launch(run, size=a.size, backend=a.backend)
