"""GPU-single tier: the per-sample step kernels -- ``convnet_step_kernel`` (csrc/convnet.cu, one CTA per sample) and
``convnet_cluster_kernel<2|4|8>`` (csrc/convnet_cluster.cu, one cluster per sample) -- sample by sample against the host
references of tests/step_oracle.py:

* the dropout scales they report equal the host Philox stream bit for bit (every p, 64-bit steps, seeds and sample indices,
  the draw that lands exactly on p);
* each sample's log-probs, loss, argmax and gradients match the fp64 oracle within the bound of ``check_per_sample``, read
  from the kernels' per-CTA slots (one sample per slot with inv_bsz = 1), from the one-GPU trainer's slots + fc1 factors,
  from slots that carry several samples, and from the double-buffered red.add bucket;
* the edges where the kernels branch: exact max-pool ties, ReLU at exactly 0, all logits tied, saturated softmax, blank
  and saturated images.

The largest error / bound ratio of every configuration is printed (run with -s to see them)."""
import math
from types import SimpleNamespace

import pytest
import torch

import step_oracle as O
from dist_tuto.pth_b200.models.convnet import PARAM_SHAPES, Net
from dist_tuto.pth_b200.ops import _ext
from dist_tuto.pth_b200.ops.convnet_fused import (FAC_STRIDE, LAYOUT, NPAR, NPAR_ALLOC, FusedTrainer, convnet_forward,
                                                 pack_params)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]
DEV = torch.device("cuda", 0)
SENTINEL = -1.25
SHAPES = dict(PARAM_SHAPES)


@pytest.fixture(scope="module")
def C():
    return _ext.C()


@pytest.fixture(scope="module")
def S():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


def _aux(params):
    """conv2.weight in the kernels' two shared-memory layouts, built by the trainer's own code."""
    aux = torch.zeros(13000, dtype=torch.float32, device=DEV)
    FusedTrainer._refresh_aux(SimpleNamespace(params=params, aux=aux, device=DEV))
    return aux


EDGES = ("conv1.weight = 0", "conv2.weight = 0", "conv1 = 0", "fc2 = 0", "fc2 x 500", "image 0", "image 255")


def _case(B, u8=False, seed=0, edge=None):
    torch.manual_seed(seed)
    net = Net()
    with torch.no_grad():
        if edge == "conv1.weight = 0":
            net.conv1.weight.zero_()                     # every pool1 window is an exact 4-way tie (= the bias)
        elif edge == "conv2.weight = 0":
            net.conv2.weight.zero_()                     # every pool2 window is an exact tie
        elif edge == "conv1 = 0":
            net.conv1.weight.zero_()
            net.conv1.bias.zero_()                       # every conv1 relu sits at exactly 0
        elif edge == "fc2 = 0":
            net.fc2.weight.zero_()
            net.fc2.bias.zero_()                         # all logits tied at 0: loss ln 10, argmax 0
        elif edge == "fc2 x 500":
            net.fc2.weight.mul_(500)
            net.fc2.bias.mul_(500)                       # saturated softmax: losses in the hundreds
    g = torch.Generator().manual_seed(seed + 1)
    if edge in ("image 0", "image 255"):
        x = torch.full((B, 1, 28, 28), 0 if edge == "image 0" else 255, dtype=torch.uint8)
    elif u8:
        x = torch.randint(0, 256, (B, 1, 28, 28), dtype=torch.uint8, generator=g)
    else:
        x = torch.randn(B, 1, 28, 28, generator=g)
    y = torch.randint(0, 10, (B,), generator=g)
    return pack_params(net).to(DEV), x.to(DEV), y.to(DEV)


def _rows(mat):
    """[rows, >= NPAR] flat gradient rows -> {name: [rows, *shape]} in fp64 on the CPU."""
    m = mat.detach().cpu().double()
    out = {}
    for n, shape in SHAPES.items():
        k = math.prod(shape)
        out[n] = m[:, LAYOUT[n]:LAYOUT[n] + k].reshape(m.shape[0], *shape)
    return out


def _launch(C, params, x, y, *, cluster=1, max_ctas=0, training=True, p=0.5, seed=1234, step=0, base=0, inv_bsz=1.0,
            aux=None, mode="slots"):
    """One convnet_step launch.  mode: "slots" (det_partials), "factors" (det_partials + factors: the one-GPU trainer's
    path), "bucket" (red.add into the bucket of parity step & 1, grad_stride = NPAR_ALLOC), "forward" (no gradients)."""
    B = y.numel()
    step_t = torch.tensor([step], dtype=torch.int64, device=DEV)
    masks = torch.full((B, 70), -1.0, device=DEV)
    logp = torch.full((B, 10), float("nan"), device=DEV)
    acc = torch.zeros(2, device=DEV)
    grads = slots = factors = None
    stride = 0
    if mode in ("slots", "factors"):
        grads = torch.full((NPAR_ALLOC,), SENTINEL, device=DEV)          # the slot paths must not touch the bucket
        slots = torch.full((B * cluster * NPAR_ALLOC,), float("nan"), device=DEV)
        if mode == "factors":
            factors = torch.full((B * FAC_STRIDE,), float("nan"), device=DEV)
    elif mode == "bucket":
        stride = NPAR_ALLOC
        grads = torch.full((2 * NPAR_ALLOC,), SENTINEL, device=DEV)
        par = step & 1
        grads[par * stride:par * stride + NPAR] = 0
    C.convnet_step(params, grads, x, y, acc, logp, masks, step_t, seed, base, training, inv_bsz, p, max_ctas, stride,
                   cluster, aux, None, slots, factors, False)
    torch.cuda.synchronize()
    return SimpleNamespace(masks=masks.cpu(), logp=logp.cpu(), acc=acc.cpu(), grads=grads, slots=slots, factors=factors,
                           stride=stride)


def _report(tag, rep):
    print(f"[ratio] {tag}: worst {rep.worst:.3g}x the bound at {rep.worst_at}")
    assert not rep.failures, f"{tag}\n{rep.message()}"


def _check_run(C, params, x, y, *, cluster=1, max_ctas=0, training=True, p=0.5, seed=1234, step=0, base=0, inv_bsz=1.0,
               aux=None, mode="slots", tag=""):
    """Launch, then compare masks, log-probs, per-slot loss / #correct / gradients (and, with factors, each sample's
    fc1.weight) with the host references.  Returns the kernel result."""
    B = y.numel()
    r = _launch(C, params, x, y, cluster=cluster, max_ctas=max_ctas, training=training, p=p, seed=seed, step=step,
                base=base, inv_bsz=inv_bsz, aux=aux, mode=mode)
    m = O.dropout_masks(seed, base, B, step, p, training)
    ref64 = O.scaled(O.per_sample_reference(params, x, y, m if training else None), inv_bsz)
    ref32 = O.scaled(O.per_sample_reference(params, x, y, m if training else None, torch.float32), inv_bsz)
    tag = tag or f"cluster {cluster} B {B} {mode}"
    _report(f"{tag} log-probs + masks", O.check_per_sample({"logp": r.logp, "masks": r.masks}, ref64, ref32, masks=m))
    G = B if max_ctas == 0 else min(B, max_ctas)                # slots (CTAs or clusters) that carry samples
    groups = [list(range(k, B, G)) for k in range(G)]
    labels = [f"slot {k} (samples {g[:3]}{'...' if len(g) > 3 else ''})" for k, g in enumerate(groups)]
    y_cpu = y.cpu()
    if mode in ("slots", "factors"):
        assert bool((r.grads == SENTINEL).all()), "the slot path wrote into the gradient bucket"
        sl = r.slots[:G * cluster * NPAR_ALLOC].view(G, cluster, NPAR_ALLOC).double().sum(1)   # a cluster's CTAs own disjoint slices
        got = _rows(sl)
        got["loss"] = sl[:, NPAR].cpu()
        if mode == "factors":
            f = r.factors.view(B, FAC_STRIDE).double().cpu()
            fc1 = f[:, :50, None] * f[:, None, 64:384]          # each sample's dh (x) p2
            _report(f"{tag} per-sample fc1.weight from the factors",
                    O.check_per_sample({"fc1.weight": fc1}, ref64, ref32))
            got["fc1.weight"] = torch.stack([fc1[g].sum(0) for g in groups])
        one = G == B
        _report(f"{tag} per-slot gradients and loss",
                O.check_per_sample(got, ref64 if one else O.fold(ref64, groups), ref32 if one else O.fold(ref32, groups),
                                   masks=m if one and training else None, labels=labels))
        want = [int(sum(int(ref64["argmax"][b]) == int(y_cpu[b]) for b in g)) for g in groups]
        assert sl[:, NPAR + 1].round().long().tolist() == want, "per-slot #correct"
        # padding between the tensors of a slot stays zero
        for n, shape in SHAPES.items():
            end = LAYOUT[n] + math.prod(shape)
            pad = (end + 3) // 4 * 4
            assert bool((sl[:, end:pad] == 0).all()), f"padding after {n}"
    elif mode == "bucket":
        par = step & 1
        bucket = r.grads[par * r.stride:par * r.stride + NPAR][None]
        whole = [list(range(B))]
        got = _rows(bucket)
        got["loss"] = r.acc[:1].double()
        _report(f"{tag} bucket sum", O.check_per_sample(got, O.fold(ref64, whole), O.fold(ref32, whole), labels=["batch"]))
        other = r.grads[(1 - par) * r.stride:(2 - par) * r.stride]
        assert bool((other == SENTINEL).all()), "the other parity's bucket was written"
        assert bool((r.grads[par * r.stride + NPAR:(par + 1) * r.stride] == SENTINEL).all()), "padding beyond NPAR written"
        assert int(r.acc[1]) == int((ref64["argmax"] == y_cpu).sum()), "#correct"
    return r, ref64


# ------------------------------------------------------------------------------------------------------- masks
KERNELS = [1, 2, 4, 8]
STEPS = [0, 1, 2 ** 32 + 1, 2 ** 40 + 3]


@pytest.mark.parametrize("cluster", KERNELS)
@pytest.mark.parametrize("p", [0.0, 0.25, 0.5, 0.9])
def test_masks_are_bit_exact_with_the_host_philox_reference(C, cluster, p):
    params, x, y = _case(16)
    seed, base = 0xC0FFEE0012345678, 12345                       # a seed with its high word set, sample_base != 0
    for step in STEPS:
        for training in (True, False):
            r = _launch(C, params, x, y, cluster=cluster, training=training, p=p, seed=seed, step=step, base=base,
                        mode="forward")
            want = O.dropout_masks(seed, base, 16, step, p, training)
            bad = torch.nonzero(r.masks != want)
            assert len(bad) == 0, (f"cluster {cluster} p {p} step {step} training {training}: {len(bad)} scales differ, "
                                   f"first (sample, column) {bad[0].tolist()}: {float(r.masks[tuple(bad[0])])} != "
                                   f"{float(want[tuple(bad[0])])}")


@pytest.mark.parametrize("cluster", KERNELS)
def test_the_draw_equal_to_p_is_kept(C, cluster):
    seed, sample, step, k = O.find_boundary_draw(0.5)
    params, x, y = _case(4)
    r = _launch(C, params, x, y, cluster=cluster, p=0.5, seed=seed, step=step, base=sample - 2, mode="forward")
    assert float(r.masks[2, k]) == 2.0, "u == p must keep the unit (u >= p)"
    assert torch.equal(r.masks, O.dropout_masks(seed, sample - 2, 4, step, 0.5))


@pytest.mark.parametrize("cluster", KERNELS)
def test_masks_depend_on_the_global_sample_index_only(C, cluster):
    params, x, y = _case(64)
    whole = _launch(C, params, x, y, cluster=cluster, p=0.25, seed=99, step=7, base=0, mode="forward").masks
    lo = _launch(C, params, x[:32].contiguous(), y[:32].contiguous(), cluster=cluster, p=0.25, seed=99, step=7, base=0,
                 mode="forward").masks
    hi = _launch(C, params, x[32:].contiguous(), y[32:].contiguous(), cluster=cluster, p=0.25, seed=99, step=7, base=32,
                 mode="forward").masks
    assert torch.equal(whole, torch.cat([lo, hi]))


# ------------------------------------------------------------------------------------------- per-sample numerics
# (cluster, B, max_ctas, mode, uint8, aux, training, p, step, sample_base); B may name a size in units of S
CONFIGS = [
    (1, 1, 0, "slots", False, True, True, 0.5, 0, 0),
    (1, 7, 0, "slots", True, False, True, 0.25, 2 ** 32 + 1, 1000),
    (1, 128, 0, "factors", True, True, True, 0.5, 3, 0),                  # the one-GPU trainer at its flagship batch
    (1, 128, 0, "slots", False, False, False, 0.5, 0, 0),
    (1, "4S+1", 0, "slots", False, True, True, 0.9, 2 ** 40 + 3, 7),      # one CTA per sample beyond 4 per SM
    (1, "4S+1", "4S", "factors", True, True, True, 0.5, 5, 0),            # the trainer's grid there: CTA 0 takes 2 samples
    (1, 64, 13, "slots", False, True, True, 0.5, 2, 0),                   # 13 CTAs carry 64 samples
    (1, 64, 13, "slots", True, False, False, 0.5, 0, 0),
    (2, 64, 0, "slots", True, True, True, 0.5, 1, 64),                    # pick_cluster's batches, rank 1's sample_base
    (4, 32, 0, "slots", False, False, True, 0.25, 2 ** 32 + 1, 32),
    (4, 16, 0, "slots", True, True, False, 0.5, 0, 0),
    (8, 8, 0, "slots", False, True, True, 0.5, 2 ** 40 + 3, 8),
    (2, 1, 0, "slots", True, False, True, 0.9, 4, 0),
    (4, 5, 0, "slots", False, True, True, 0.5, 3, 0),
    (8, 33, 0, "slots", True, True, True, 0.25, 9, 0),
    (2, 33, 3, "slots", False, True, True, 0.5, 6, 0),                    # 3 clusters carry 33 samples
    (8, 7, 3, "slots", True, False, False, 0.5, 0, 0),
]


def _size(v, S):
    return {"4S+1": 4 * S + 1, "4S": 4 * S}.get(v, v) if isinstance(v, str) else v


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: f"c{c[0]}-B{c[1]}-max{c[2]}-{c[3]}-{'u8' if c[4] else 'f32'}-"
                                                      f"{'aux' if c[5] else 'noaux'}-{'train' if c[6] else 'eval'}")
def test_every_sample_matches_the_fp64_oracle(C, S, cfg):
    cluster, B, max_ctas, mode, u8, use_aux, training, p, step, base = cfg
    B, max_ctas = _size(B, S), _size(max_ctas, S)
    params, x, y = _case(B, u8=u8, seed=B + cluster)
    _check_run(C, params, x, y, cluster=cluster, max_ctas=max_ctas, training=training, p=p, seed=4321, step=step,
               base=base, aux=_aux(params) if use_aux else None, mode=mode)


@pytest.mark.parametrize("cluster,B", [(1, 128), (4, 32)])
def test_slots_at_the_training_inv_bsz(C, cluster, B):
    """inv_bsz = 1/B as in training: every slot term (gradients and loss) is scaled by it."""
    params, x, y = _case(B, u8=True, seed=5)
    _check_run(C, params, x, y, cluster=cluster, inv_bsz=1.0 / B, step=3, aux=_aux(params), tag=f"cluster {cluster} 1/B")


@pytest.mark.parametrize("cluster,B", [(1, 128), (2, 64), (8, 8)])
@pytest.mark.parametrize("step", [6, 2 ** 32 + 1])
def test_red_add_bucket_at_both_parities(C, cluster, B, step):
    params, x, y = _case(B, seed=11)
    _check_run(C, params, x, y, cluster=cluster, inv_bsz=1.0 / B, step=step, base=B, aux=_aux(params), mode="bucket",
               tag=f"cluster {cluster} bucket parity {step & 1}")


# ------------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize("cluster", [1, 4])
@pytest.mark.parametrize("edge", EDGES)
def test_edge_weights_and_images(C, cluster, edge):
    B = 8
    params, x, y = _case(B, seed=17, edge=edge)
    y[:3] = 0                                                       # some labels are 0: the tied argmax is right for them
    r, ref64 = _check_run(C, params, x, y, cluster=cluster, p=0.5, step=1, aux=_aux(params), tag=f"cluster {cluster} {edge}")
    sl = r.slots[:B * cluster * NPAR_ALLOC].view(B, cluster, NPAR_ALLOC).sum(1).cpu()
    if edge == "conv1 = 0":
        assert int(torch.count_nonzero(sl[:, :LAYOUT["conv2.weight"]])) == 0, "relu'(0) must be 0: conv1 gradients are 0"
    if edge == "fc2 = 0":
        assert torch.allclose(sl[:, NPAR].double(), torch.full((B,), math.log(10), dtype=torch.float64), rtol=1e-6)
        assert sl[:, NPAR + 1].tolist() == (y.cpu() == 0).float().tolist(), "all logits tied: the argmax is class 0"
    if edge == "fc2 x 500":
        assert float(ref64["loss"].max()) > 100, "the case must saturate the softmax"


def test_forward_only_log_probs_per_sample(S):
    B = 4 * S + 1
    params, x, y = _case(B, seed=23)
    out = convnet_forward(params, x)
    ref64 = O.per_sample_reference(params, x, y, None)
    ref32 = O.per_sample_reference(params, x, y, None, torch.float32)
    _report("forward-only 4S+1", O.check_per_sample({"logp": out.cpu()}, ref64, ref32))


# ------------------------------------------------------------------------------------------------ binding checks
def test_misaligned_buffers_are_refused_before_launch(C):
    # Every call below would fault on the device if it reached the kernel: require the binding that refuses them.
    assert "16-byte aligned" in (C.convnet_step.__doc__ or ""), "convnet_step without its alignment checks"
    params, x, y = _case(2)
    B = 2

    def off(t):
        """A view of t's data shifted by one element (4 bytes for fp32, 1 byte for uint8): contiguous, not 16-byte aligned."""
        buf = torch.zeros(t.numel() + 16, dtype=t.dtype, device=DEV)
        v = buf[1:1 + t.numel()].view_as(t)
        v.copy_(t)
        return v

    step = torch.zeros(1, dtype=torch.int64, device=DEV)
    grads = torch.zeros(2 * NPAR_ALLOC, device=DEV)
    aux = _aux(params)
    slots = torch.zeros(B * NPAR_ALLOC, device=DEV)
    factors = torch.zeros(B * FAC_STRIDE, device=DEV)
    calls = {
        "params": lambda: C.convnet_step(off(params), grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5),
        "x": lambda: C.convnet_step(params, grads, off(x), y, None, None, None, step, 1, 0, True, 0.5, 0.5),
        "x uint8": lambda: C.convnet_step(params, grads, off(x.to(torch.uint8)), y, None, None, None, step, 1, 0, True, 0.5, 0.5),
        "grads": lambda: C.convnet_step(params, off(grads), x, y, None, None, None, step, 1, 0, True, 0.5, 0.5),
        "aux": lambda: C.convnet_step(params, grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5, 0, 0, 1, off(aux)),
        "det_partials": lambda: C.convnet_step(params, grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5, 0, 0, 1,
                                               aux, None, off(slots)),
        "factors": lambda: C.convnet_step(params, grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5, 0, 0, 1, aux,
                                          None, slots, off(factors)),
        "grad_stride": lambda: C.convnet_step(params, grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5, 0, 6),
    }
    for what, call in calls.items():
        with pytest.raises(RuntimeError, match="16-byte aligned|multiple of 4"):
            call()
    # the cluster kernel goes through the same checks
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        C.convnet_step(off(params), grads, x, y, None, None, None, step, 1, 0, True, 0.5, 0.5, 0, 0, 2)
    torch.cuda.synchronize()
    # and aligned buffers still run
    r = _launch(C, params, x, y, aux=aux)
    assert torch.isfinite(r.logp).all()
