"""FlatAdafactor's kernels on one GPU: ``adafactor_flat`` (csrc/adafactor.cu) bit for bit against tests/adafactor_model.py over
every layout a bucket view can have, with sentinels behind every flat, state and workspace and the tickets zero after every
call; two runs bit-identical; the clip and scaled instances against the plain one fed the clipped / unscaled gradient; the
kernel's error against fp64 within the model's bound and against torch's CUDA Adafactor; no host synchronisation in
``step()``; a ResNet-18 trained through ``DistributedDataParallel`` + ``FlatAdafactor`` under bf16 autocast."""
import math

import pytest
import torch

import adafactor_model as M
from adamw_model import clip_coef
from emulated_ranks import C  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

HP = dict(beta2_decay=-0.8, eps1=torch.finfo(torch.float32).eps, eps2=1e-3, d=1.0)
SENT = 4096
LAYOUTS = {
    "small": [((), None), ((1,), None), ((7,), None), ((5, 3), None), ((1, 6), None), ((6, 1), None), ((2, 3, 4), None),
              ((6, 4, 3, 3), "cl"), ((2, 3, 4, 5, 6), None)],
    "tiled": [((300, 300), None), ((3, 70, 200), None), ((130, 100), None), ((64, 129), "t"), ((8193,), None)],
    "conv": [((64, 32, 3, 3), "cl"), ((128, 64, 1, 1), "cl"), ((32, 64, 5, 5), None), ((16, 8, 7, 7), "cl")],
    "tiny": [((3,), None) if i % 3 else ((2, 2), None) for i in range(2000)],
    "tall": [((1 << 20, 1), None), ((5,), None)],
    "wide": [((1, 1 << 20), None), ((40000, 3), None)],
}


def _stride(shape, fmt):
    t = torch.empty(shape)
    if fmt == "cl":
        return t.to(memory_format=torch.channels_last).stride()
    if fmt == "t":                                        # a transposed 2-D weight (rows not contiguous)
        return torch.empty(shape[::-1]).t().stride()
    return t.stride()


def _layout(specs, groups=1):
    tensors, o = [], 0
    for i, (shape, fmt) in enumerate(specs):
        tensors.append((o, tuple(shape), _stride(shape, fmt), i % groups))
        o += (math.prod(shape) + 3) // 4 * 4
    return tensors, o


class Bucket:
    """One bucket on the device for adafactor_flat: flats and workspaces with SENT sentinel values behind each."""

    def __init__(self, C, tensors, n, n_groups=1):
        self.C, self.tensors, self.n = C, tensors, n
        soff, ns = M.state_offsets([s for _, s, _, _ in tensors])
        self.ns = ns
        table, self.n_chunks, n_rc, n_means = C.adafactor_table([t[0] for t in tensors], [list(t[1]) for t in tensors],
                                                                 [list(t[2]) for t in tensors], soff, [t[3] for t in tensors],
                                                                 n, max(ns, 1), n_groups, torch.device("cuda"))
        self.table = table
        nt = len(tensors)
        self.bufs = {}
        for name, size, dt, fill in (("p", n, torch.float32, 0.0), ("g", n, torch.float32, 0.0), ("state", max(ns, 1), torch.float32, 0.0),
                                     ("partials", 2 * self.n_chunks, torch.float32, 0.0), ("rc", max(n_rc, 1), torch.float32, 0.0),
                                     ("means", max(n_means, 1), torch.float32, 0.0), ("tickets", nt, torch.int32, 0),
                                     ("alpha", nt, torch.float64, 0.0), ("step", nt, torch.float32, 0.0)):
            full = torch.full((size + SENT,), fill, dtype=dt, device="cuda")
            full[size:] = 77 if dt == torch.int32 else 1234.5
            self.bufs[name] = (full, size)

    def __getitem__(self, k):
        full, size = self.bufs[k]
        return full[:size]

    def sentinels_intact(self):
        for k, (full, size) in self.bufs.items():
            assert bool((full[size:] == (77 if full.dtype == torch.int32 else 1234.5)).all()), f"{k}: a write past the end"
        assert int(self["tickets"].abs().sum()) == 0, "a ticket is not zero after the call"

    def step(self, t, groups, zero_grad=True, **kw):
        sc = [float(t) ** HP["beta2_decay"], HP["eps1"], HP["eps2"], HP["d"]]
        rho = [min(lr, 1 / (t ** 0.5)) for lr, _, _ in groups]
        decay = [1 - lr * wd for lr, wd, _ in groups]
        self.C.adafactor_flat(self["p"], self["state"], self["g"], self.table, self.n_chunks, self["partials"], self["rc"],
                              self["means"], self["tickets"], self["alpha"], self["step"], sc, rho, decay, zero_grad, **kw)


def _grad(n, t, seed, tensors):
    """A gradient flat: random on the tensors' elements, zero in the padding between them (as a bucket holds it)."""
    g = torch.Generator().manual_seed(seed * 31 + t)
    out = torch.zeros(n)
    for o, shape, _, _ in tensors:
        k = math.prod(shape)
        out[o:o + k] = torch.randn(k, generator=g) * (2.0 ** t)
    return out


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_kernel_matches_the_model_bit_for_bit(C, layout):
    """Three updates with decay and a second group: parameters, state, alpha and step scalars bit for bit the model's;
    sentinels intact and tickets zero after every call."""
    tensors, n = _layout(LAYOUTS[layout], groups=2)
    b = Bucket(C, tensors, n, n_groups=2)
    torch.manual_seed(1)
    p = torch.randn(n)
    state = torch.zeros(max(b.ns, 1))
    b["p"].copy_(p)
    groups = [(1e-2, 0.1, 1e-2), (3e-2, 0.0, 3e-2)]
    for t in (1, 2, 3):
        g = _grad(n, t, 5, tensors)
        b["g"].copy_(g)
        b.step(t, groups)
        p, state, alphas, steps = M.adafactor_step(p, g, state, tensors, groups, HP, t)
        torch.cuda.synchronize()
        b.sentinels_intact()
        assert torch.equal(b["p"].cpu(), p), (layout, t, "parameters")
        assert torch.equal(b["state"].cpu()[:b.ns], state[:b.ns]), (layout, t, "state")
        assert not b["g"].any(), "the gradients are re-zeroed"
        live = [i for i, a in enumerate(alphas) if a is not None]
        assert b["alpha"].cpu()[live].tolist() == [alphas[i] for i in live], (layout, t, "alpha")
        assert b["step"].cpu()[live].tolist() == [steps[i] for i in live], (layout, t, "step")


def test_two_runs_are_bit_identical(C):
    tensors, n = _layout(LAYOUTS["tiled"] + LAYOUTS["conv"])
    out = []
    for _ in range(2):
        b = Bucket(C, tensors, n)
        torch.manual_seed(2)
        b["p"].copy_(torch.randn(n))
        for t in (1, 2, 3):
            b["g"].copy_(_grad(n, t, 9, tensors))
            b.step(t, [(1e-2, 0.01, 1e-2)])
        out.append((b["p"].clone(), b["state"].clone()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


@pytest.mark.parametrize("clip, scaled", [(True, False), (False, True), (True, True)])
def test_clip_and_scaled_instances_equal_the_plain_one(C, clip, scaled):
    """The clip instance equals the plain one fed g * coef, the scaled one the plain one fed g * fp32(1 / double(S)); the
    clip instance writes the pre-clip norm."""
    tensors, n = _layout(LAYOUTS["small"] + LAYOUTS["tiled"])
    torch.manual_seed(3)
    p0 = torch.randn(n)
    S = 1000.0 if scaled else 1.0
    a, ref = Bucket(C, tensors, n), Bucket(C, tensors, n)
    a["p"].copy_(p0)
    ref["p"].copy_(p0)
    for t in (1, 2):
        g = _grad(n, t, 4, tensors)
        gs = (g * S) if scaled else g
        unscaled = (gs.cuda() * torch.tensor(1.0 / S, dtype=torch.float64).float().cuda()) if scaled else g.cuda()
        kw = {}
        if scaled:
            kw["grad_scale"] = torch.tensor([S], dtype=torch.float32, device="cuda")
        if clip:
            sq = torch.tensor([float((unscaled.double() ** 2).sum())], dtype=torch.float64, device="cuda")
            norm = torch.zeros(1, device="cuda")
            kw.update(max_grad_norm=0.5, sqnorms=sq, grad_norm_out=norm)
            coef = clip_coef([float(sq[0])], 0.5)
            unscaled = unscaled * torch.tensor(coef, dtype=torch.float32, device="cuda")
        a["g"].copy_(gs)
        a.step(t, [(1e-2, 0.1, 1e-2)], **kw)
        ref["g"].copy_(unscaled)
        ref.step(t, [(1e-2, 0.1, 1e-2)])
        torch.cuda.synchronize()
        a.sentinels_intact()
        assert torch.equal(a["p"], ref["p"]) and torch.equal(a["state"], ref["state"]), (clip, scaled, t)
        if clip:
            assert float(norm[0]) == float(torch.tensor(math.sqrt(float(sq[0])), dtype=torch.float32))


def test_error_against_fp64_and_torch_cuda_adafactor(C):
    """Over five updates with decay and d > 1: the kernel's error against fp64 Adafactor stays within the model's bound
    (4x torch's fp32 CPU error plus two ulps), and within 1e-5 relative of torch.optim.Adafactor on CUDA."""
    specs = LAYOUTS["small"] + LAYOUTS["tiled"] + LAYOUTS["conv"]
    tensors, n = _layout(specs)
    hp = dict(HP, d=1.5)
    b = Bucket(C, tensors, n)
    torch.manual_seed(5)
    p0 = torch.randn(n)
    b["p"].copy_(p0)
    views = lambda f: [f[o:o + math.prod(s)].as_strided(s, st) for o, s, st, _ in tensors]  # noqa: E731
    gs, lr, wd = [], 1e-2, 0.1
    for t in range(1, 6):
        g = _grad(n, t, 6, tensors)
        gs.append(g)
        b["g"].copy_(g)
        sc = [float(t) ** hp["beta2_decay"], hp["eps1"], hp["eps2"], hp["d"]]
        C.adafactor_flat(b["p"], b["state"], b["g"], b.table, b.n_chunks, b["partials"], b["rc"], b["means"], b["tickets"],
                         b["alpha"], b["step"], sc, [min(lr, 1 / t ** 0.5)], [1 - lr * wd], True)
    ref = M.adafactor_fp64(views(p0), [views(g) for g in gs], hp, [[lr] * len(tensors)] * 5, [[wd] * len(tensors)] * 5)
    for dev in ("cpu", "cuda"):
        ws = [torch.nn.Parameter(v.clone().to(dev)) for v in views(p0)]
        opt = torch.optim.Adafactor(ws, lr=lr, beta2_decay=hp["beta2_decay"], eps=(None, hp["eps2"]), d=hp["d"],
                                    weight_decay=wd, foreach=False)
        for g in gs:
            for w, gv in zip(ws, views(g)):
                w.grad = gv.clone().to(dev)
            opt.step()
        for k, (v, r, w) in enumerate(zip(views(b["p"].cpu()), ref, ws)):
            em = float((v.double() - r).abs().max())
            if dev == "cpu":
                et = float((w.detach().double().cpu() - r).abs().max())
                assert em <= 4 * et + 2 * float(r.abs().max()) * 2.0 ** -23, (specs[k], em, et)
            else:
                assert torch.allclose(v, w.detach().cpu(), rtol=1e-5, atol=1e-6), (specs[k], em)


def test_step_does_not_synchronise_and_tracks_the_model(C):
    """FlatAdafactor.step() on a DDP model with clipping, groups and a schedule runs under sync_debug_mode("error")."""
    import dist_tuto.pth_b200 as b2
    import adafactor_gpu_workers as WK
    b2.launch(WK.w_no_sync, size=1, backend="b200", join_timeout_s=600)


def test_ddp_resnet18_trains_like_torch_adafactor_under_bf16_autocast():
    import dist_tuto.pth_b200 as b2
    import adafactor_gpu_workers as WK
    b2.launch(WK.w_resnet, size=1, backend="b200", join_timeout_s=600)


def test_ddp_world_one_equals_one_bucket():
    import dist_tuto.pth_b200 as b2
    import adafactor_gpu_workers as WK
    b2.launch(WK.w_ddp, size=1, backend="b200", join_timeout_s=600)
