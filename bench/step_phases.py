"""Where the time of one training step goes, phase by phase, in the configuration of ``bench.py``'s ``value`` (global batch 128
on one GPU, CUDA graphs of 50 steps, PDL between the step kernel and the optimizer kernel).

Turns on the kernels' opt-in phase timestamps (``C.set_phase_ts``: thread 0 of every CTA reads ``%globaltimer`` at the ends of
the phases, see ``csrc/sgd_device.cuh``), replays the graphs and prints one JSON line:

* ``step_kernel_us``: median over CTAs and steps of each phase of ``convnet_step`` (entry -> griddepcontrol.wait returns ->
  S0 (input, RNG, staging barrier) -> S1 (conv1) -> S2 -> S4 -> S6 -> S7/S8a -> S8b -> gradient flush -> exit), and the CTA's
  whole life;
* ``optimizer_us``: from the last step CTA's exit to the optimizer kernel's first return from griddepcontrol.wait (``gap``),
  from there to its last CTA's exit (``work``), and the step period (first optimizer wait of one step to the next);
* ``optimizer_units_us``: per kind of reduction unit of ``reduce_sgd`` (``fc1``: fc1.weight tiles, ``other``: the other
  vectors), median and maximum over CTAs and steps of the optimizer's first wait -> this CTA's wait, wait -> the unit's loads
  have landed (its first barrier), loads -> emit done, emit -> exit; and how often each kind was the last CTA to exit.

The stamps cost a few barriers; ``bench.py`` never turns them on.  Run: ``python bench/step_phases.py [--out FILE]``."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dist_tuto.pth_b200.ops import _ext  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer  # noqa: E402

TS_STEPS, TS_CTAS, TS_PER_CTA = 64, 256, 16          # csrc/sgd_device.cuh
STEP_MARKS = ["entry", "waited", "s0", "s1", "s2", "s4", "s6", "s8a", "s8b", "flushed", "exit"]
EXIT = len(STEP_MARKS) - 1
OPT_UNIT, OPT_WAITED, OPT_EXIT, OPT_LOADED, OPT_EMITTED = 11, 12, 13, 14, 15
UNIT_KINDS = {1: "fc1", 2: "other"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bsz", type=int, default=128)
    ap.add_argument("--graph-steps", type=int, default=50)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "step_phases.py measures on a GPU"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    C = _ext.C()
    bsz, G = args.bsz, args.graph_steps
    assert G <= TS_STEPS
    tr = FusedTrainer(bsz, lr=0.01, momentum=0.5, seed=1234, device=dev, p_drop=0.5, raw_uint8=True)
    g = torch.Generator(device=dev).manual_seed(1234)
    px = torch.randn(G, bsz, 1, 28, 28, device=dev, generator=g)
    py = torch.randint(0, 10, (G, bsz), device=dev, generator=g)
    ts = torch.zeros(TS_STEPS * TS_CTAS * TS_PER_CTA, dtype=torch.int64, device=dev)
    C.set_phase_ts(ts)                                   # read at launch: baked into the captured graph
    st = tr.stream
    try:
        with torch.cuda.stream(st):
            for i in range(5):
                tr._kernels(px[i], py[i], bsz)
        st.synchronize()
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.graph(gr, stream=st):
            for i in range(G):
                tr._kernels(px[i], py[i], bsz)
    finally:
        C.set_phase_ts(None)
    n_cta = bsz                                          # one CTA per sample
    phases = {f"{a}->{b}": [] for a, b in zip(STEP_MARKS[:-1], STEP_MARKS[1:])}
    phases["cta_life"] = []
    gaps, works, periods = [], [], []
    unit_marks = [("first_wait->wait", None, OPT_WAITED), ("wait->loaded", OPT_WAITED, OPT_LOADED),
                  ("loaded->emitted", OPT_LOADED, OPT_EMITTED), ("emitted->exit", OPT_EMITTED, OPT_EXIT)]
    units = {kind: {name: [] for name, _, _ in unit_marks} for kind in UNIT_KINDS.values()}
    last_exit = {kind: 0 for kind in UNIT_KINDS.values()}
    for _ in range(args.replays):
        with torch.cuda.stream(st):                     # the clear is ordered before the replay on the same stream
            ts.zero_()
            gr.replay()
        st.synchronize()
        end = int(tr.step_counter.item())
        t = ts.view(TS_STEPS, TS_CTAS, TS_PER_CTA).cpu().numpy()
        prev_wait = None
        for s in range(end - G, end):
            row = t[s % TS_STEPS]
            cta = row[:n_cta]
            for k, (a, b) in enumerate(zip(STEP_MARKS[:-1], STEP_MARKS[1:])):
                phases[f"{a}->{b}"] += ((cta[:, k + 1] - cta[:, k]) / 1e3).tolist()
            phases["cta_life"] += ((cta[:, EXIT] - cta[:, 0]) / 1e3).tolist()
            opt = row[row[:, OPT_WAITED] > 0]
            if len(opt) == 0:
                continue
            w0 = int(opt[:, OPT_WAITED].min())
            gaps.append((w0 - int(cta[:, EXIT].max())) / 1e3)
            works.append((int(opt[:, OPT_EXIT].max()) - w0) / 1e3)
            for code, kind in UNIT_KINDS.items():
                u = opt[opt[:, OPT_UNIT] == code]
                for name, a, b in unit_marks:
                    start = u[:, a] if a is not None else w0
                    units[kind][name] += ((u[:, b] - start) / 1e3).tolist()
            last = int(opt[:, OPT_UNIT][opt[:, OPT_EXIT].argmax()])
            if last in UNIT_KINDS:
                last_exit[UNIT_KINDS[last]] += 1
            if prev_wait is not None:
                periods.append((w0 - prev_wait) / 1e3)
            prev_wait = w0
    med = lambda xs: round(statistics.median(xs), 2) if xs else None  # noqa: E731
    mx = lambda xs: round(max(xs), 2) if xs else None  # noqa: E731
    last_row = t[(end - 1) % TS_STEPS]
    res = {"gpu": torch.cuda.get_device_name(dev), "bsz": bsz, "steps": len(gaps),
           "step_kernel_us": {k: med(v) for k, v in phases.items()},
           "optimizer_us": {"gap_last_step_exit_to_wait": med(gaps), "work": med(works), "step_period": med(periods),
                            "ctas": int((last_row[:, OPT_WAITED] > 0).sum())},
           "optimizer_units_us": {kind: {"ctas": int((last_row[:, OPT_UNIT] == code).sum()),
                                         **{name: {"median": med(v), "max": mx(v)} for name, v in units[kind].items()}}
                                  for code, kind in UNIT_KINDS.items()},
           "optimizer_last_exit": last_exit}
    line = json.dumps(res)
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
