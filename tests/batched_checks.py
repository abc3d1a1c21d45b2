"""Checks shared by the batched-engine tests (tests/test_gpu_batched.py, tests/test_gpu_batched_sizes.py) and by the CPU
test that shows they catch planted faults (tests/test_batched_checks.py).

* Launch geometry: every wgmma kernel of csrc/convnet_batched.cu is a persistent grid of at most S CTAs (S = SM count) with
  an mbarrier ring whose phase parity flips only when one CTA handles more items than the ring has stages; the SIMT
  kernels loop over the batch once the grid is capped.  ``batch_sizes(S)`` is the set of batch sizes at which all of
  those paths run, and ``kernel_geometry()`` reads the stage counts and grid caps out of the kernel source, so that a
  change to the kernel's staging is seen by the CPU test of the set.
* Per-sample errors: ``row_errors`` gives each sample's error relative to the batch's RMS row norm, so one wrong sample
  out of thousands is as visible as a wrong batch.
* Reductions: ``synthetic`` builds the operands of one gradient kernel in the engine's buffer layouts, each sample's
  contribution with a random sign, plus the exact fp64 result; ``prefill_bucket`` / ``check_bucket`` pre-load the
  gradient bucket with the negated result and a sentinel in every slot the kernel must not touch.
"""
import os
import re

import torch
import torch.nn.functional as F

from dist_tuto.pth_b200.models.convnet import PARAM_SHAPES
from dist_tuto.pth_b200.ops import batched_reference as R
from dist_tuto.pth_b200.ops.convnet_fused import LAYOUT, NPAR_ALLOC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KERNEL_SRC = os.path.join(ROOT, "dist_tuto.pth_b200", "csrc", "convnet_batched.cu")

# ---------------------------------------------------------------------------------------------------------- geometry
SIZE_NAMES = ["1", "3", "4S+1", "8S+3", "2048", "4096", "32S+1", "8191"]


def batch_sizes(S: int) -> dict:
    """Batch sizes (by name) that cross every loop / ring threshold of the engine on a GPU with S SMs:
    1 and 3 (one tile, a half tile), 4S+1 (the conv2 data-gradient ring wraps), 8S+3 (odd; the conv2 forward and weight
    gradient rings wrap), 2048 (where train() switches to this engine), 4096 (bench.py's batch), 32S+1 (fc weight gradient
    takes ceil(B/S) samples per CTA) and 8191 (every ring wraps many times, 63 samples per CTA, odd)."""
    return {"1": 1, "3": 3, "4S+1": 4 * S + 1, "8S+3": 8 * S + 3, "2048": 2048, "4096": 4096, "32S+1": 32 * S + 1,
            "8191": 8191}


def kernel_geometry(src: str = KERNEL_SRC) -> dict:
    """Ring depths, the fc weight-gradient tile and chunk rule, and the grid caps of the launcher (in units of S)."""
    with open(src) as f:
        text = f.read()

    def const(name):
        m = re.search(rf"constexpr int {name} = (\d+);", text)
        assert m, f"{name} not found in {src}"
        return int(m.group(1))

    def cap(kernel):       # `kernel<<<n < sms * K ? n : sms * K, ...` (K = 1 when absent)
        m = re.search(rf"{kernel}<<<\w+ < sms(?: \* (\d+))? \?", text)
        assert m, f"launch of {kernel} not found in {src}"
        return int(m.group(1) or 1)

    dg = re.search(r"struct __align__\(1024\) DgSmem \{.*?uint64_t full\[(\d+)\]", text, re.S)
    fc = re.search(r"const int per = B >= sms \* (\d+) \? \(B \+ sms - 1\) / sms : (\d+);", text)
    assert dg and fc, "conv2 dgrad ring or fc_wgrad chunk rule not found"
    return {"C2F_NST": const("C2F_NST"), "WG_NST": const("WG_NST"), "DG_NST": int(dg.group(1)), "FW_TS": const("FW_TS"),
            "fc_from": int(fc.group(1)), "fc_per": int(fc.group(2)),
            "cap": {k: cap("bt_" + k) for k in ("conv1_fwd", "conv2_fwd", "conv2_wgrad", "conv2_dgrad", "conv1_wgrad")}}


def loop_depths(B: int, S: int, geo: dict) -> dict:
    """Per kernel: items the busiest CTA handles (``*_items``), phase flips of its ring (``*_flips`` = how often the
    stage index comes back to stage 0), and the fc weight-gradient chunk."""
    def per_cta(items, cap):
        grid = min(items, cap * S)
        return -(-items // grid) if grid else 0
    tiles, pairs = (B + 1) // 2, (B + 1) // 2
    out = {"conv1_fwd_items": per_cta(pairs, geo["cap"]["conv1_fwd"]),
           "conv1_wgrad_items": per_cta(B, geo["cap"]["conv1_wgrad"]),
           "conv2_fwd_items": per_cta(tiles, geo["cap"]["conv2_fwd"]),
           "conv2_wgrad_items": per_cta(B, geo["cap"]["conv2_wgrad"]),
           "conv2_dgrad_items": per_cta(tiles, geo["cap"]["conv2_dgrad"])}
    for k, nst in (("conv2_fwd", geo["C2F_NST"]), ("conv2_wgrad", geo["WG_NST"]), ("conv2_dgrad", geo["DG_NST"])):
        out[k + "_flips"] = max(out[k + "_items"] - 1, 0) // nst
    out["fc_per"] = -(-B // S) if B >= geo["fc_from"] * S else geo["fc_per"]
    return out


# ------------------------------------------------------------------------------------------------ per-sample errors
def row_errors(got: torch.Tensor, want: torch.Tensor) -> torch.Tensor:
    """[B] fp64: ||got_b - want_b|| / RMS_b ||want_b||."""
    B = want.shape[0]
    g, w = got.reshape(B, -1).double(), want.reshape(B, -1).double().to(got.device)
    scale = w.pow(2).sum(1).mean().sqrt().clamp_min(1e-30)
    return (g - w).norm(dim=1) / scale


def check_rows(report: dict, name: str, got, want, bound: float, batch_bound: float = None) -> list:
    """Record the worst sample of ``name`` in ``report``; return a failure line if any sample exceeds ``bound`` (or the
    whole batch's relative norm exceeds ``batch_bound``)."""
    e = row_errors(got, want)
    worst = int(e.argmax()) if e.numel() else 0
    n_over = int((e > bound).sum())
    batch = rel_norm(got, want.to(got.device))
    report[name] = {"worst": float(e.max()) if e.numel() else 0.0, "worst_sample": worst, "bound": bound,
                    "samples_over": n_over, "batch": batch}
    bad = [f"{name}: {n_over} samples above {bound:g} (worst {report[name]['worst']:.3g} at sample {worst})"] if n_over else []
    if batch_bound is not None and not batch <= batch_bound:
        bad.append(f"{name}: batch rel err {batch:.3g} > {batch_bound:g}")
    return bad


def pool_ties(pre: torch.Tensor, rel: float = 2.0 ** -14) -> torch.Tensor:
    """[B,C,H/2,W/2] bool: 2x2 windows of the pre-pool map ``pre`` [B,C,H,W] whose argmax or relu decision is a near-tie:
    the two largest candidates, or the largest and 0, within ``rel`` x max|pre| of that (sample, channel).  Summation
    order alone can flip such a decision."""
    B, C, H, W = pre.shape
    win = pre.reshape(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)
    top = win.topk(2, dim=-1).values
    tol = rel * pre.abs().amax(dim=(2, 3), keepdim=True)
    return ((top[..., 0] - top[..., 1]) <= tol) | (top[..., 0].abs() <= tol)


def check_codes(report: dict, name: str, got: torch.Tensor, want: torch.Tensor, ties: torch.Tensor, max_frac: float) -> list:
    """Pool codes of the engine vs the model: a code may differ only at a near-tie, and at most ``max_frac`` of all."""
    B = want.shape[0]
    diff = got.reshape(B, -1).to(torch.int64) != want.reshape(B, -1).to(torch.int64)
    at_tie = diff & ties.reshape(B, -1)
    n_diff, n_free = int(diff.sum()), int((diff & ~at_tie).sum())
    report[name] = {"mismatches": n_diff, "mismatches_not_at_a_tie": n_free, "samples_with_mismatch": int(diff.any(1).sum()),
                    "max_frac": max_frac}
    bad = []
    if n_free:
        bad.append(f"{name}: {n_free} codes differ without a near-tie in the model")
    if n_diff > max_frac * diff.numel():
        bad.append(f"{name}: {n_diff} of {diff.numel()} codes differ")
    return bad


def rel_norm(got, want) -> float:
    g, w = got.double(), want.double()
    return float((g - w).norm() / w.norm().clamp_min(1e-30))


# ------------------------------------------------------------------------------------------------ gradient bucket
SENTINEL = 2.0 ** -15          # finite and exactly representable; any red.add of a non-zero value changes it


def param_slots(name: str) -> slice:
    n = 1
    for s in dict(PARAM_SHAPES)[name]:
        n *= s
    return slice(LAYOUT[name], LAYOUT[name] + n)


def pad_slots() -> torch.Tensor:
    """Indices of the flat bucket that belong to no parameter (alignment padding of ``LAYOUT``)."""
    used = torch.zeros(NPAR_ALLOC, dtype=torch.bool)
    for name, _ in PARAM_SHAPES:
        used[param_slots(name)] = True
    return (~used).nonzero().flatten()


def prefill_bucket(want: dict, device) -> torch.Tensor:
    """fp32 bucket = -want[name] at the named parameters, SENTINEL everywhere else."""
    b = torch.full((NPAR_ALLOC,), SENTINEL, dtype=torch.float32, device=device)
    for name, v in want.items():
        b[param_slots(name)] = (-v.double()).reshape(-1).to(torch.float32).to(device)
    return b


def check_bucket(report: dict, tag: str, bucket: torch.Tensor, want: dict, bound: float) -> list:
    """After a kernel accumulated into ``prefill_bucket(want)``: every named gradient must land within ``bound`` of zero
    (relative to its fp64 norm), and every other slot -- padding and the other parameters -- must hold SENTINEL."""
    bad = []
    b = bucket.double().cpu()
    pre = prefill_bucket(want, "cpu").double()
    keep = torch.ones(NPAR_ALLOC, dtype=torch.bool)
    for name, v in want.items():
        s = param_slots(name)
        keep[s] = False
        # the kernel's sum = bucket - prefill (exact in fp64); its error against the exact result
        err = float((b[s] - pre[s] - v.double().reshape(-1).cpu()).norm() / v.double().norm().clamp_min(1e-30))
        report[f"{tag}/{name}"] = {"rel_err": err, "bound": bound}
        if not err <= bound:
            bad.append(f"{tag}/{name}: rel err {err:.3g} > {bound:g}")
    touched = (b[keep] != SENTINEL).nonzero().flatten()
    idx = keep.nonzero().flatten()[touched]
    report[f"{tag}/untouched_slots_written"] = idx.tolist()[:16]
    if idx.numel():
        bad.append(f"{tag}: slots outside the kernel's gradients were written: {idx.tolist()[:16]}")
    return bad


# ------------------------------------------------------------------------------------------------ synthetic operands
REDUCTIONS = {"conv2_wgrad": ("conv2.weight", "conv2.bias"), "conv1_wgrad": ("conv1.weight", "conv1.bias"),
              "fc_wgrad": ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias")}
# fp32 summation order is the only error left in the reductions (exact operands, exact fp64 result); dropping or
# doubling one sample of 8191 moves a gradient by ~1/sqrt(8191) = 1.1e-2 of its norm, 4e-3 at the least for the
# 10-wide fc2 rows (tests/test_batched_checks.py); the worst observed on an H100 is 4.3e-6 (conv2 weight, B = 8191)
REDUCTION_BOUND = 1e-4
# the conv2 data gradient's operands make every intermediate exact: it must match to the last bit of fp32
DGRAD_BOUND = 1e-6
STAGE_BIT = {"conv2_wgrad": 16, "conv2_dgrad": 32, "conv1_wgrad": 64, "fc_wgrad": 128}
MEAN, INV_STD = 0.1307, 1.0 / 0.3081


def normalize_u8(xu: torch.Tensor) -> torch.Tensor:
    """The kernels' in-register normalisation of raw pixels, in fp32: (u / 255 - mean) / std."""
    f32 = torch.float32
    inv255 = torch.tensor(1.0, dtype=f32) / torch.tensor(255.0, dtype=f32)
    inv_std = torch.tensor(1.0, dtype=f32) / torch.tensor(0.3081, dtype=f32)
    return (xu.to(f32) * inv255.to(xu.device) - torch.tensor(MEAN, dtype=f32, device=xu.device)) * inv_std.to(xu.device)


def _bf(t):
    return t.to(torch.bfloat16)


def _codes(B, gen, device):
    """Random conv1 pool codes [B,1440]: argmax 0..3 and the dead bit on ~30 % of the cells."""
    arg = torch.randint(0, 4, (B, 1440), generator=gen)
    dead = torch.rand(B, 1440, generator=gen) < 0.3
    return (arg | dead.to(torch.int64) * 4).to(torch.uint8).to(device)


def synthetic(kernel: str, B: int, seed: int, device, x_u8: bool = False, chunk: int = 1024) -> dict:
    """Operands of one engine kernel in ``BatchedBuffers`` layouts and its exact fp64 result.

    Every operand is exactly representable in the buffer's type.  For the three reductions each sample's operand carries a
    random sign (``signs``), so that dropping or doubling one sample moves the result by ~1/sqrt(B) of its norm.  The conv2
    data gradient uses small multiples of powers of two, so its bf16 staging tile and fp32 col2im sums are exact too.
    Returns {"bufs": {buffer name: tensor}, "x", "params", "want": {gradient name or "G1": fp64 tensor}, "signs"}."""
    gen = torch.Generator().manual_seed(seed)
    sign = (torch.randint(0, 2, (B,), generator=gen) * 2 - 1).double()
    out = {"bufs": {}, "signs": sign, "params": torch.zeros(NPAR_ALLOC, dtype=torch.float32)}
    if x_u8:
        out["x"] = torch.randint(0, 256, (B, 1, 28, 28), dtype=torch.uint8, generator=gen)
        xf = normalize_u8(out["x"]).double()
    else:
        out["x"] = _bf(torch.randn(B, 1, 28, 28, generator=gen)).float()
        xf = out["x"].double()
    want = {}
    if kernel == "conv2_wgrad":
        p1 = torch.zeros(B, 12, 12, 16)
        p1[..., :10] = _bf(torch.randn(B, 12, 12, 10, generator=gen)).float()
        p1[..., 10] = 1.0
        dc = torch.zeros(B, 32, 64)
        dc[:, :20] = _bf(torch.randn(B, 20, 64, generator=gen)).float() * sign.view(B, 1, 1).float()
        out["bufs"] = {"P1": _bf(p1), "DC": _bf(dc)}
        w, bsum = torch.zeros(20, 250, dtype=torch.float64), torch.zeros(20, dtype=torch.float64)
        for c0 in range(0, B, chunk):
            col = F.unfold(p1[c0:c0 + chunk, :, :, :10].permute(0, 3, 1, 2).double(), 5)      # [b, ci*25 + tap, 64]
            d = dc[c0:c0 + chunk, :20].double()
            w += torch.einsum("bkp,bcp->ck", col, d)
            bsum += d.sum((0, 2))
        want = {"conv2.weight": w.view(20, 10, 5, 5), "conv2.bias": bsum}
    elif kernel == "conv1_wgrad":
        code = _codes(B, gen, "cpu")
        g1 = _bf(torch.randn(B, 1440, generator=gen)).float() * sign.view(B, 1).float()
        g1[(code & 4) != 0] = 0.0                               # the engine's G1 is zero wherever conv1's pool is dead
        out["bufs"] = {"G1": g1, "A1": code}
        idx = R._unpool_index(code.view(B, 10, 12, 12), 24).view(B, 10, 144)
        w, bsum = torch.zeros(10, 25, dtype=torch.float64), torch.zeros(10, dtype=torch.float64)
        for c0 in range(0, B, chunk):
            g = g1[c0:c0 + chunk].double().view(-1, 10, 144)
            dc1 = torch.zeros(g.shape[0], 10, 576, dtype=torch.float64).scatter_(2, idx[c0:c0 + chunk], g)
            w += torch.einsum("bkp,bcp->ck", F.unfold(xf[c0:c0 + chunk], 5), dc1)
            bsum += g.sum((0, 2))
        want = {"conv1.weight": w.view(10, 1, 5, 5), "conv1.bias": bsum}
    elif kernel == "fc_wgrad":
        p2 = _bf(torch.randn(B, 320, generator=gen)).float()
        h, dh, dlog = torch.zeros(B, 64), torch.zeros(B, 64), torch.zeros(B, 16)
        h[:, :50] = _bf(torch.randn(B, 50, generator=gen)).float()
        dh[:, :50] = _bf(torch.randn(B, 50, generator=gen)).float() * sign.view(B, 1).float()
        dlog[:, :10] = _bf(torch.randn(B, 10, generator=gen)).float() * sign.view(B, 1).float()
        out["bufs"] = {"P2": _bf(p2), "H": _bf(h), "DH": _bf(dh), "DLOG": dlog}
        want = {"fc1.weight": dh[:, :50].double().t() @ p2.double(), "fc1.bias": dh[:, :50].double().sum(0),
                "fc2.weight": dlog[:, :10].double().t() @ h[:, :50].double(), "fc2.bias": dlog[:, :10].double().sum(0)}
    elif kernel == "conv2_dgrad":
        # |dA| <= 20 * 3 * 3 units of 2^-9 fits bf16's 8 significant bits; G1 sums <= 25 of them: exact in fp32
        w2 = torch.randint(-3, 4, (20, 10, 5, 5), generator=gen).float() * 2.0 ** -5
        out["params"][param_slots("conv2.weight")] = w2.reshape(-1)
        dc = torch.zeros(B, 32, 64)
        dc[:, :20] = torch.randint(-3, 4, (B, 20, 64), generator=gen).float() * 2.0 ** -4
        code = _codes(B, gen, "cpu")
        out["bufs"] = {"DC": _bf(dc), "A1": code}
        da = torch.einsum("ck,bcp->bkp", w2.double().view(20, 250), dc[:, :20].double())          # [B, ci*25 + tap, 64]
        g1 = F.fold(da, (12, 12), 5).view(B, 1440)
        g1[(code & 4) != 0] = 0.0
        want = {"G1": g1}
    else:
        raise ValueError(kernel)
    out["want"] = want
    dev = torch.device(device)
    out["x"] = out["x"].to(dev)
    out["params"] = out["params"].to(dev)
    out["bufs"] = {k: v.to(dev) for k, v in out["bufs"].items()}
    return out


# ------------------------------------------------------------------------------------------------ full pipeline
# Per-sample bounds of each stage (row error / batch RMS row norm), each >= 10x the worst sample observed at every size
# on an H100 and <= 1/10 of a swapped or zeroed sample.  fp32 stages differ by summation order only (<= 4e-7 observed).
# bf16-stored stages differ where the two fp32 values round to neighbouring bf16 numbers: one such flip of a sample's
# largest element moves it by up to 2^-8 (<= 6.2e-3 observed); the stages after dH inherit its flips.
STAGE_BOUNDS = {"hrelu": 1e-5, "dlog": 1e-5, "logp": 1e-5, "p2": 7e-2, "dh": 7e-2, "dp2": 7e-2, "dc": 7e-2, "g1": 7e-2}
BATCH_BOUND = 5e-3              # the same stages over the whole batch (one relative norm)
GRAD_BOUND = 2e-3               # pipeline gradients, relative norm per tensor (<= 1.4e-4 observed)
LOSS_BOUND = 1e-5               # mean NLL, relative (<= 1e-6 observed)
CODE_MISMATCH_FRAC = 1e-3       # pool codes: only at near-ties (none observed)


def engine_views(bufs, B: int) -> dict:
    """The first B samples of a ``BatchedBuffers`` in the model's shapes (fp32 / int64)."""
    p1 = bufs.P1[:B * 2304].view(B, 12, 12, 16)
    return {"p1": p1[..., :10].permute(0, 3, 1, 2).float(), "p1_raw": p1,
            "a1": bufs.A1[:B * 1440].view(B, 10, 12, 12).to(torch.int64),
            "a2": bufs.A2[:B * 320].view(B, 20, 4, 4).to(torch.int64),
            "p2": bufs.P2[:B * 320].view(B, 320).float(), "hrelu": bufs.Hrelu[:B * 64].view(B, 64)[:, :50],
            "hrelu_pad": bufs.Hrelu[:B * 64].view(B, 64)[:, 50:],
            "dlog": bufs.DLOG[:B * 16].view(B, 16), "dh": bufs.DH[:B * 64].view(B, 64).float(),
            "h": bufs.H[:B * 64].view(B, 64).float(), "dp2": bufs.dP2[:B * 320].view(B, 320).float(),
            "dc": bufs.DC[:B * 2048].view(B, 32, 64).float(), "g1": bufs.G1[:B * 1440].view(B, 10, 12, 12)}


def compare_pipeline(report: dict, bufs, params, x, y, m2, dm, grads=None, loss=None, backward: bool = True):
    """Every stage of one engine pass against the rounding-exact model, each on the engine's own inputs, sample by sample.

    ``x`` normalised fp32; ``m2``/``dm`` dropout scales (None = eval); ``grads`` the engine's flat gradient (any float
    dtype) and ``loss`` its mean NLL.  The model continues from the engine's conv1 output and pool codes, its conv2 pool
    codes, P2 and fc1 output, so pool routing and relu decisions are identical and each stage differs only by its own
    summation order and one bf16 rounding.  The pool codes themselves may differ only at near-ties of the model.
    Returns (failure lines, the model's outputs on the engine's inputs)."""
    B = y.numel()
    e = engine_views(bufs, B)
    bad = []
    ov = {"p1_override": e["p1"], "a1_override": e["a1"] & 3}
    r1 = R.forward_backward(params, x, y, m2, dm, a2_override=e["a2"], p2_override=e["p2"], **ov)
    p2_model = R.rbf(r1["mp2"].clamp_min(0)).view(B, 320)
    bad += check_rows(report, "p2", e["p2"], p2_model, STAGE_BOUNDS["p2"], BATCH_BOUND)
    bad += check_codes(report, "a2_codes", e["a2"], R.pool_codes(r1["a2"], r1["mp2"], 8), pool_ties(r1["c2"]),
                       CODE_MISMATCH_FRAC)
    bad += check_rows(report, "hrelu", e["hrelu"], r1["hrelu"], STAGE_BOUNDS["hrelu"], BATCH_BOUND)
    r2 = R.forward_backward(params, x, y, m2, dm, a2_override=e["a2"], p2_override=e["p2"], hrelu_override=e["hrelu"], **ov)
    if not backward:
        return bad, r2
    bad += check_rows(report, "dlog", e["dlog"][:, :10], r2["dlog"], STAGE_BOUNDS["dlog"], BATCH_BOUND)
    bad += check_rows(report, "dh", e["dh"][:, :50], r2["dh"], STAGE_BOUNDS["dh"], BATCH_BOUND)
    bad += check_rows(report, "dp2", e["dp2"], r2["dp2"], STAGE_BOUNDS["dp2"], BATCH_BOUND)
    bad += check_rows(report, "dc", e["dc"][:, :20], r2["dc"].reshape(B, 20, 64), STAGE_BOUNDS["dc"], BATCH_BOUND)
    bad += check_rows(report, "g1", e["g1"], r2["g1"], STAGE_BOUNDS["g1"], BATCH_BOUND)
    pads = {"p1_const_channels": bool((e["p1_raw"][..., 10] == 1).all() and (e["p1_raw"][..., 11:] == 0).all()),
            "dc_pad_zero": bool((e["dc"][:, 20:] == 0).all()), "dh_pad_zero": bool((e["dh"][:, 50:] == 0).all()),
            "dlog_pad_zero": bool((e["dlog"][:, 10:] == 0).all())}
    report["pads"] = pads
    bad += [f"pad not intact: {k}" for k, v in pads.items() if not v]
    if loss is not None:
        report["loss"] = abs(float(loss) - float(r2["loss"])) / abs(float(r2["loss"]))
        if not report["loss"] <= LOSS_BOUND:
            bad.append(f"loss rel err {report['loss']:.3g} > {LOSS_BOUND:g}")
    if grads is not None:
        from dist_tuto.pth_b200.ops.convnet_fused import unpack_params
        mine, want = unpack_params(grads), r2["named"]
        for n in want:
            err = rel_norm(mine[n], want[n])
            report["grad/" + n] = {"rel_err": err, "bound": GRAD_BOUND}
            if not err <= GRAD_BOUND:
                bad.append(f"grad/{n}: rel err {err:.3g} > {GRAD_BOUND:g}")
    return bad, r2
