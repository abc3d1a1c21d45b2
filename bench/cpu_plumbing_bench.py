"""BASELINE.json config #1: the tutorial's training loop on CPU / gloo, world_size 2, synthetic 28x28 data.

No GPU involved -- this measures the *plumbing*: data sharding + loader, model step on torch CPU ops, gradient
averaging over gloo, optimizer.  Two arms, same metric (samples/s, wall clock, max over ranks, K timed steps after W
warm-up steps, global batch 128 = 64 per rank):

  reference : the UNMODIFIED reference from oracle/_ref -- ``train_dist.Net``, ``train_dist.partition_dataset()``
              (torchvision MNIST on synthetic idx files + DataLoader), the tutorial-text ``average_gradients``
              (tuto.md:310-314: one all_reduce + one divide per parameter), ``optim.SGD`` -- loop body train_dist.py:115-124
  ours      : ``dist_tuto.pth_b200`` -- ``partition_dataset()`` (C++ prefetch thread into staging buffers), ``Net``,
              gradients as views of ONE flat bucket (one gloo all_reduce per step), ``FlatSGD``

Run here (no GPU):  python bench/cpu_plumbing_bench.py --steps 150 --warmup 10 --out cpu_plumbing_world2.json
"""
import argparse
import json
import os
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "baseline"))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import dist_tuto.pth_b200 as b2  # noqa: E402
from bench_common import max_over_ranks, synthetic_idx_dir  # noqa: E402


def _args():
    return json.loads(os.environ["B2_BENCH_ARGS"])


def _timed(step, batches, K, W):
    for _ in range(W):
        step(*next(batches))
    dist.barrier()
    t0 = time.perf_counter()
    loss = None
    for _ in range(K):
        loss = step(*next(batches))
    float(loss)
    dist.barrier()
    return max_over_ranks((time.perf_counter() - t0) * 1e3, torch.device("cpu"))


def _cycle(loader):
    while True:
        for b in loader:
            yield b


def w_reference(rank, size):
    a = _args()
    warnings.filterwarnings("ignore")
    torch.set_num_threads(a["threads"])
    from ref_harness import load_reference, tutorial_average_gradients
    ref, why = load_reference()
    if ref is None:
        if rank == 0:
            print(json.dumps({"impl": "reference", "unavailable": why}))
        return
    cwd = os.getcwd()
    os.chdir(synthetic_idx_dir(rank))
    try:
        train_set, bsz = ref.partition_dataset()                       # unmodified, train_dist.py:74-91
    finally:
        os.chdir(cwd)
    torch.manual_seed(1234)
    model = ref.Net()
    opt = torch.optim.SGD(model.parameters(), lr=0.01, momentum=0.5)

    def step(data, target):                                            # train_dist.py:118-124
        opt.zero_grad()
        loss = F.nll_loss(model(data), target)
        loss.backward()
        tutorial_average_gradients(model, dist)
        opt.step()
        return loss.detach()

    ms = _timed(step, _cycle(train_set), a["steps"], a["warmup"])
    if rank == 0:
        print(json.dumps({"impl": "reference", "samples_per_s": bsz * size * a["steps"] / (ms / 1e3), "ms_per_step": ms / a["steps"]}))


def w_ours(rank, size):
    a = _args()
    torch.set_num_threads(a["threads"])
    train_set, bsz = b2.partition_dataset(b2.SyntheticMNIST(n=60000, seed=1234), native=a["native"])
    torch.manual_seed(1234)
    model = b2.Net()
    b2.broadcast_parameters(model)
    opt = b2.FlatSGD(model, lr=0.01, momentum=0.5)                     # builds the flat bucket; grads/params are views

    def step(data, target):
        opt.zero_grad()
        loss = F.nll_loss(model(data), target)
        loss.backward()
        b2.average_gradients(model)                                    # ONE all_reduce on the flat bucket
        opt.step()
        return loss.detach()

    ms = _timed(step, _cycle(train_set), a["steps"], a["warmup"])
    if rank == 0:
        print(json.dumps({"impl": "ours", "samples_per_s": bsz * size * a["steps"] / (ms / 1e3), "ms_per_step": ms / a["steps"]}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=150)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--size", type=int, default=2)
    ap.add_argument("--threads", type=int, default=2, help="torch intra-op threads per rank")
    ap.add_argument("--python-loader", dest="native", action="store_false", help="vectorised Python loader instead of the C++ prefetch thread")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(args))
    rows = []
    for fn in (w_reference, w_ours):
        r, w = os.pipe()
        pid = os.fork()
        if pid == 0:                       # child: run one arm, forward its stdout JSON through the pipe
            os.close(r)
            os.dup2(w, 1)
            try:
                b2.launch(fn, size=args.size, backend="gloo", join_timeout_s=1200)
                os._exit(0)
            except BaseException as e:  # noqa: BLE001
                sys.stderr.write(f"{fn.__name__} failed: {e}\n")
                os._exit(1)
        os.close(w)
        out = b""
        while True:
            chunk = os.read(r, 65536)
            if not chunk:
                break
            out += chunk
        os.waitpid(pid, 0)
        for ln in out.decode().splitlines():
            if ln.startswith("{"):
                rows.append(json.loads(ln))
    res = {"config": "train_dist.py ConvNet on CPU/gloo world_size=%d, synthetic 28x28, global batch 128" % args.size,
           "steps": args.steps, "warmup": args.warmup, "threads_per_rank": args.threads,
           "ours_loader": "C++ prefetch thread (NativeBatchLoader)" if args.native else "vectorised Python BatchLoader", "timing": "wall clock, max over ranks",
           "rows": rows}
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
