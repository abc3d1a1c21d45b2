"""All-reduce bus bandwidth sweep (BASELINE.json config #4): fused peer-memory variants vs NCCL.

    python bench/allreduce_sweep.py --gpus N [--max-mb 1024] [--out gpurun_out/sweep_N.json]

For every size 1 KB .. max: LL (flag-in-data push, <= 64 KB) / one-shot / two-shot / NVLS (when exposed) on a symmetric
fp32 buffer (in place, 1/N scale fused) and ``dist.all_reduce`` (NCCL) with and without the ``div_`` the reference's
average_gradients issues per tensor.  Timed with CUDA events on the launching stream after warm-up, MAX over ranks.  Every
arm is measured twice in alternating order (A B .. B A) and the minimum kept, so that no arm owes its number to its position
(round 1's table had NCCL alone slower than NCCL + div).

Bandwidth columns:
  busbw   = 2(N-1)/N * bytes / t        the NCCL-tests convention (what a ring would push through each link)
  link_tx = bytes a GPU really sends:    two-shot (N-1)/N * bytes * 2 (gather slices + broadcast own slice);
            NVLS  bytes * (1 + 1/N) ... see `link_bytes()` (formulas checked against the NVLink counters, bench/nvlink_bytes.py);
            reported as link_GBs = link_tx / t against 770 GB/s measured peer copy.
``--emit-table`` writes parallel/allreduce_table.json (per-world variant thresholds) from the measured winners.

``--collective {reduce,broadcast,allgather,scatter,gather,reducescatter,alltoall,alltoallv}`` or ``--op {product,max,min}`` time
that collective instead: every variant of ours (forced, through the ``SymmWorld`` method ``comm.py`` routes to) against the
NCCL call on the same tensor, per size (for an all-gather, a scatter, a gather, a reduce-scatter and an all-to-all, the
size of one rank's segment; the root is rank 0 and its list is one block; reduce-scatter and all-to-all have an LL and a
pull arm only).  ``alltoallv`` times ``all_to_all_single`` with split sizes: seeded skewed splits of about the size
per pair, half of every rank's bytes to one hot destination and the rest at random, on the variable-segment kernel
against NCCL (no speed claim rests on it until it has run on a multi-GPU H100 machine).  ``--dtype {bf16,fp16,fp64,int8,uint8,int32,int64,bool}`` times the reductions (and the raw moves) on
a tensor of that dtype.  It compares GPUs, so it refuses to run on one.
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import dist_tuto.pth_b200 as b2  # noqa: E402
from dist_tuto.pth_b200.parallel import symm  # noqa: E402

import types
ARGS = types.SimpleNamespace(**json.loads(os.environ["B2_BENCH_ARGS"])) if "B2_BENCH_ARGS" in os.environ else None


def tmax(ms, dev):
    t = torch.tensor([ms], dtype=torch.float64, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def time_op(fn, iters, dev, graph=False):
    """ms per call, max over ranks.  ``graph=True`` replays a CUDA graph of ``iters`` calls so that small messages
    are timed at device speed rather than at the Python launch rate (applied to NCCL and to our kernels alike)."""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if graph:
        st = torch.cuda.Stream()
        g = torch.cuda.CUDAGraph()
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.graph(g, stream=st):
            for _ in range(iters):
                fn()
        g.replay()
        torch.cuda.synchronize()
        dist.barrier()
        torch.cuda.synchronize()
        e0.record()
        g.replay()
        e1.record()
        e1.synchronize()
        return tmax(e0.elapsed_time(e1) / iters, dev)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return tmax(e0.elapsed_time(e1) / iters, dev)


OPS = {"sum": dist.ReduceOp.SUM, "product": dist.ReduceOp.PRODUCT, "max": dist.ReduceOp.MAX, "min": dist.ReduceOp.MIN}
DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp16": torch.float16, "fp64": torch.float64, "int8": torch.int8,
          "uint8": torch.uint8, "int32": torch.int32, "int64": torch.int64, "bool": torch.bool}


def skewed_splits(size: int, n: int, seed: int) -> list:
    """``S[s][d]``: elements rank s sends rank d, about ``n`` per pair on average, drawn from ``seed`` (the same on every
    rank): one hot destination takes half of every rank's elements, the others share the rest at random."""
    g = torch.Generator().manual_seed(seed)
    hot = int(torch.randint(0, size, (1,), generator=g))
    S = []
    for _ in range(size):
        share = torch.rand(size, generator=g)
        share[hot] = 0.0
        share = share / share.sum() * (size * n - size * n // 2) if size > 1 else share * 0
        row = [int(x) for x in share]
        row[hot] += size * n - sum(row)
        S.append(row)
    return S


def body_collective(rank, size):
    """``--collective`` / ``--op``: ours per forced variant vs NCCL, per size, rows printed and written to ``--out``."""
    dev = torch.device("cuda", torch.cuda.current_device())
    w = symm.lookup_world(None)
    op = OPS[ARGS.op]
    coll = ARGS.collective
    rows = []
    s = 1024
    while s <= ARGS.max_mb << 20:
        dtype = DTYPES[ARGS.dtype]
        n = s // torch.empty((), dtype=dtype).element_size()
        t = torch.ones(n, dtype=dtype, device=dev)
        outs = [torch.empty_like(t) for _ in range(size)]
        lst = list(torch.empty(size * n, dtype=dtype, device=dev).view(size, n).unbind(0)) if rank == 0 else None  # scatter / gather
        iters = 100 if s <= (1 << 20) else 20
        whole = torch.ones(size * n, dtype=dtype, device=dev)  # reduce-scatter / all-to-all: world segments of s bytes
        outs_whole = torch.empty_like(whole)
        row = {"bytes": s, "collective": coll, "op": ARGS.op, "dtype": ARGS.dtype}
        arms = []
        segmented = coll in ("reducescatter", "alltoall")     # two kernels only: LL and pull
        if coll == "alltoallv":                                # one kernel: the variable-segment pull
            S = skewed_splits(size, n, s)
            v_in = torch.ones(sum(S[rank]), dtype=dtype, device=dev)
            v_out = torch.empty(sum(S[p][rank] for p in range(size)), dtype=dtype, device=dev)
            v_osplit = [S[p][rank] for p in range(size)]
            arms.append(("pull", lambda: w.all_to_all_v_(v_out, v_in, v_osplit, S[rank])))
        for name, v in (() if coll == "alltoallv" else (("ll", 3), ("pull", 0)) if segmented else
                        (("ll", 3), ("oneshot", 0), ("twoshot", 1))):
            if name == "ll" and s > symm.LL_CAP_VEC * 16:
                continue
            if coll == "reducescatter":
                arms.append((name, lambda v=v: w.reduce_scatter_(t, whole, op, variant=v)))
            elif coll == "alltoall":
                arms.append((name, lambda v=v: w.all_to_all_(outs_whole, whole, variant=v)))
            elif coll == "allreduce":
                arms.append((name, lambda v=v: w.all_reduce_(t, variant=v, op=op)))
            elif coll == "reduce":
                arms.append((name, lambda v=v: w.reduce_(t, 0, op, variant=v)))
            elif coll == "broadcast":
                arms.append((name, lambda v=v: w.broadcast_(t, 0, variant=v)))
            elif coll == "scatter":
                arms.append((name, lambda v=v: w.scatter_(t, lst, 0, variant=v)))
            elif coll == "gather":
                arms.append((name, lambda v=v: w.gather_(t, lst, 0, variant=v)))
            else:
                arms.append((name, lambda v=v: w.all_gather_(outs, t, variant=v)))
        nccl = {"allreduce": lambda: dist.all_reduce(t, op=op), "reduce": lambda: dist.reduce(t, 0, op=op),
                "broadcast": lambda: dist.broadcast(t, 0), "allgather": lambda: dist.all_gather(outs, t),
                "scatter": lambda: dist.scatter(t, scatter_list=lst, src=0),
                "gather": lambda: dist.gather(t, gather_list=lst, dst=0),
                "reducescatter": lambda: dist.reduce_scatter_tensor(t, whole, op=op),
                "alltoall": lambda: dist.all_to_all_single(outs_whole, whole),
                "alltoallv": lambda: dist.all_to_all_single(v_out, v_in, v_osplit, S[rank])}[coll]
        arms.append(("nccl", nccl))
        best = {}
        for order in (arms, arms[::-1]):
            for name, fn in order:
                t.fill_(1.0)
                best[name] = min(best.get(name, 1e30), time_op(fn, iters, dev, False))
        for name, ms in best.items():
            row[name + "_us"] = ms * 1e3
        ours = min((row[k], k) for k in row if k.endswith("_us") and k != "nccl_us")
        row["best"], row["speedup_vs_nccl"] = ours[1][:-3], row["nccl_us"] / ours[0]
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
        s *= 4
    if rank == 0:
        os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
        json.dump({"n_gpus": size, "symm": w.describe(), "rows": rows, "timing": "eager, CUDA events"}, open(ARGS.out, "w"),
                  indent=1)
        print("WROTE", ARGS.out, flush=True)
    dist.barrier()


def body(rank, size):
    if ARGS.collective != "allreduce" or ARGS.op != "sum" or ARGS.dtype != "fp32":
        return body_collective(rank, size)
    dev = torch.device("cuda", torch.cuda.current_device())
    w = symm.lookup_world(None)
    max_bytes = ARGS.max_mb << 20
    sizes = []
    s = 1024
    while s <= max_bytes:
        sizes.append(s)
        s *= 4 if s >= (1 << 20) else 2
    if sizes[-1] != max_bytes:
        sizes.append(max_bytes)
    hd = w.alloc(max_bytes // 4, torch.float32)
    rows = []
    variants = [("ll", 3), ("oneshot", 0), ("twoshot", 1)] + ([("nvls", 2)] if w.multicast else [])

    def link_bytes(name, nbytes):
        """Bytes one GPU transmits over its NVLink ports for one all-reduce of ``nbytes`` (receives the same), by algorithm;
        bench/nvlink_bytes.py checks these formulas against the GPU's own link counters.  The LL lines are 16-byte stores
        that carry 8 data bytes each -- it is a latency variant."""
        if name == "ll":
            return 2 * nbytes * (size - 1)                       # 16-byte lines carry 8 data bytes, to every peer
        if name == "oneshot":
            return nbytes * (size - 1)                           # every peer reads my whole buffer
        if name == "twoshot":
            return 2 * nbytes * (size - 1) / size                # peers read my slices + I push my reduced slice to them
        if name == "nvls":
            # multimem.ld_reduce of slice j makes the switch fetch slice j from EVERY GPU (mine included, over my link): the N
            # slices cost me nbytes of transmit; multimem.st of my reduced slice is one more nbytes / N (the switch replicates it)
            return nbytes * (1 + 1.0 / size)
        return 2 * nbytes * (size - 1) / size                    # NCCL ring / tree: the bus-bandwidth convention

    for nbytes in sizes:
        n = nbytes // 4
        t = hd.local[:n]
        plain = torch.ones(n, device=dev)
        iters = 100 if nbytes <= (1 << 20) else (40 if nbytes <= (64 << 20) else 10)
        gm = nbytes <= (4 << 20)          # graph-timed (device rate) for latency-bound sizes
        row = {"bytes": nbytes, "graph_timed": gm}
        arms = []
        for name, v in variants:
            if v == 0 and nbytes > (8 << 20):
                continue
            if v == 3 and nbytes > symm.LL_CAP_VEC * 16:
                continue

            def run(v=v):
                w.all_reduce_(t, scale=1.0 / size, handle=hd, variant=v)
            arms.append((name, run, True))
        arms.append(("nccl_div", lambda: (dist.all_reduce(plain), plain.div_(size)), False))
        arms.append(("nccl", lambda: dist.all_reduce(plain), False))
        best_ms = {}
        for order in (arms, arms[::-1]):                       # A B C .. then .. C B A: position effects cancel
            for name, fn, ours in order:
                if ours:
                    t.fill_(1.0)
                ms = time_op(fn, iters, dev, gm)
                best_ms[name] = min(best_ms.get(name, 1e30), ms)
                if ours:
                    assert abs(float(t[0]) - 1.0) < 1e-3, (name, float(t[0]))
        for name, ms in best_ms.items():
            row[name + "_us"] = ms * 1e3
            row[name + "_busbw_GBs"] = 2 * (size - 1) / size * nbytes / (ms * 1e-3) / 1e9
            row[name + "_link_GBs"] = link_bytes(name.split("_")[0], nbytes) / (ms * 1e-3) / 1e9
        best = min((row[k], k) for k in row if k.endswith("_us") and not k.startswith("nccl"))
        row["best"] = best[1][:-3]
        row["speedup_vs_nccl_div"] = row["nccl_div_us"] / best[0]
        # graph-replayed back-to-back NCCL all-reduces of one buffer are reproducibly SLOWER than the same calls with the
        # divide in between (both arm orders agree), so the competitor is the faster of the two NCCL arms
        row["nccl_best_us"] = min(row["nccl_us"], row["nccl_div_us"])
        row["speedup_vs_nccl_best"] = row["nccl_best_us"] / best[0]
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
    # the reference's actual pattern: 8 per-tensor all_reduce + 8 divides (ConvNet gradient shapes)
    shapes = [250, 10, 5000, 20, 16000, 50, 500, 10]
    grads = [torch.ones(s_, device=dev) for s_ in shapes]

    def ref_avg():
        for g in grads:
            dist.all_reduce(g)
            g.div_(size)
    per_tensor = time_op(ref_avg, 50, dev, True) * 1e3
    per_tensor_eager = time_op(ref_avg, 50, dev, False) * 1e3
    bucket = w.alloc(21888, torch.float32)
    fused = time_op(lambda: w.all_reduce_(bucket.local, scale=1.0 / size, handle=bucket, variant=0), 100, dev, True) * 1e3
    fused_eager = time_op(lambda: w.all_reduce_(bucket.local, scale=1.0 / size, handle=bucket, variant=0), 100, dev, False) * 1e3
    table = None
    if rank == 0:
        # variant thresholds from the measured winners: largest size at which LL / one-shot still wins, smallest at which NVLS does
        def last_win(name):
            sz = 0
            for r in rows:
                if r["best"] == name:
                    sz = r["bytes"]
            return sz
        nv = [r["bytes"] for r in rows if r["best"] == "nvls"]
        table = {"ll_max": last_win("ll"), "oneshot_max": max(last_win("oneshot"), last_win("ll")),
                 "nvls_min": (min(nv) if nv else (1 << 62))}
        if getattr(ARGS, "emit_table", False):
            path = os.path.join(ROOT, "dist_tuto.pth_b200", "parallel", "allreduce_table.json")
            try:
                cur = json.load(open(path))
            except Exception:
                cur = {"what": "per-world all-reduce variant thresholds (wire bytes), written by bench/allreduce_sweep.py --emit-table", "worlds": {}}
            cur["worlds"][str(size)] = table
            json.dump(cur, open(path, "w"), indent=1)
            for extra in (os.path.join(ROOT, "gpurun_out", f"allreduce_table_world{size}.json"),):
                os.makedirs(os.path.dirname(extra), exist_ok=True)
                json.dump({"world": size, **table}, open(extra, "w"), indent=1)
    if rank == 0:
        out = {"n_gpus": size, "symm": w.describe(), "rows": rows, "thresholds_from_this_sweep": table,
               "convnet_average_gradients": {"reference_8x(allreduce+div)_us": per_tensor, "fused_oneshot_bucket_us": fused,
                                             "speedup": per_tensor / fused, "timing": "CUDA-graph replay (device rate)",
                                             "eager_reference_us": per_tensor_eager, "eager_fused_us": fused_eager},
               "link_GBs_measured_ref": 770, "link_GBs_nominal": 900}
        os.makedirs(os.path.dirname(ARGS.out) or ".", exist_ok=True)
        json.dump(out, open(ARGS.out, "w"), indent=1)
        print("WROTE", ARGS.out, flush=True)
    dist.barrier()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=2)
    ap.add_argument("--max-mb", type=int, default=1024)
    ap.add_argument("--out", default=None)
    ap.add_argument("--emit-table", action="store_true", help="write the measured variant thresholds of this world size")
    ap.add_argument("--collective", choices=["allreduce", "reduce", "broadcast", "allgather", "scatter", "gather", "reducescatter",
                                                 "alltoall", "alltoallv"], default="allreduce")
    ap.add_argument("--op", choices=sorted(OPS), default="sum")
    ap.add_argument("--dtype", choices=list(DTYPES), default="fp32", help="tensor dtype of the reductions")
    ARGS = ap.parse_args()
    if ARGS.gpus < 2:
        ap.error("the sweep compares collectives across GPUs; it needs --gpus 2 or more")
    if ARGS.emit_table and (ARGS.collective != "allreduce" or ARGS.op != "sum" or ARGS.dtype != "fp32"):
        ap.error("--emit-table measures the fp32 SUM all-reduce thresholds")
    if ARGS.out is None:
        ARGS.out = f"gpurun_out/sweep_{ARGS.gpus}.json"
        if (ARGS.collective, ARGS.op, ARGS.dtype) != ("allreduce", "sum", "fp32"):    # one file per collective, op, dtype
            stem, ext = os.path.splitext(ARGS.out)
            ARGS.out = f"{stem}_{ARGS.collective}_{ARGS.op}" + ("" if ARGS.dtype == "fp32" else f"_{ARGS.dtype}") + ext
    os.environ["B2_BENCH_ARGS"] = json.dumps(vars(ARGS))
    if "RANK" in os.environ:
        b2.init_from_env(body, backend="b200")
    else:
        b2.launch(body, size=ARGS.gpus, backend="b200", join_timeout_s=1500)
