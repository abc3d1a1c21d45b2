"""CPU checks of the batched-engine test helpers (tests/batched_checks.py).

* The batch-size set wraps every mbarrier ring of csrc/convnet_batched.cu at least twice and runs every persistent loop
  more than once, for the SM counts of the H100 SXM (132) and PCIe (114), with the stage counts read from the kernel.
* The per-sample, reduction and bucket checks flag faults planted in the model's own outputs, each by at least 10x its
  bound: a swapped sample, a zeroed sample in the last tile, one sample missing from a reduction of 8191, a padding slot
  written."""
import pytest
import torch

import batched_checks as BC
import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.ops import batched_reference as R
from dist_tuto.pth_b200.ops.convnet_fused import pack_params


@pytest.mark.parametrize("S", [132, 114])
def test_size_set_wraps_every_ring_twice(S):
    geo = BC.kernel_geometry()
    depths = {n: BC.loop_depths(B, S, geo) for n, B in BC.batch_sizes(S).items()}
    for ring in ("conv2_fwd", "conv2_wgrad", "conv2_dgrad"):
        assert max(d[ring + "_flips"] for d in depths.values()) >= 2, (ring, geo, depths)
    for loop in ("conv1_fwd", "conv1_wgrad"):
        assert max(d[loop + "_items"] for d in depths.values()) >= 2, (loop, geo, depths)
    # fc weight gradient: ceil(B/S) samples per CTA, a chunk that is not a whole number of shared-memory tiles
    assert any(d["fc_per"] != geo["fc_per"] and d["fc_per"] % geo["FW_TS"] for d in depths.values()), (geo, depths)
    sizes = BC.batch_sizes(S)
    assert sizes["1"] == 1 and any(B % 2 for B in sizes.values() if B > 1)      # one sample; a half-full last tile
    assert sizes["2048"] == 2048 and sizes["4096"] == 4096


def _engine_buffers(out, B):
    """Buffers laid out like ``BatchedBuffers`` holding the model's own outputs: what a correct engine would write."""
    class Bufs:
        pass
    f = Bufs()
    p1 = torch.zeros(B, 12, 12, 16)
    p1[..., :10] = out["p1"].permute(0, 2, 3, 1)
    p1[..., 10] = 1.0
    f.P1 = p1.to(torch.bfloat16).view(-1)
    f.A1 = R.pool_codes(out["a1"], out["m1"], 24).to(torch.uint8).view(-1)
    f.A2 = R.pool_codes(out["a2"], out["mp2"], 8).to(torch.uint8).view(-1)
    f.P2 = out["p2"].to(torch.bfloat16).view(-1)
    f.Hrelu, f.DLOG, f.DH, f.H = torch.zeros(B, 64), torch.zeros(B, 16), torch.zeros(B, 64), torch.zeros(B, 64)
    f.Hrelu[:, :50], f.DLOG[:, :10], f.DH[:, :50] = out["hrelu"], out["dlog"], out["dh"]
    f.Hrelu, f.DLOG, f.DH, f.H = f.Hrelu.view(-1), f.DLOG.view(-1), f.DH.to(torch.bfloat16).view(-1), f.H.view(-1)
    f.dP2 = out["dp2"].to(torch.bfloat16).view(-1)
    dc = torch.zeros(B, 32, 64)
    dc[:, :20] = out["dc"].reshape(B, 20, 64)
    f.DC = dc.to(torch.bfloat16).view(-1)
    f.G1 = out["g1"].reshape(-1).clone()
    return f


def _model_case(B=8, seed=3):
    torch.manual_seed(seed)
    params = pack_params(b2.Net())
    x = torch.randn(B, 1, 28, 28)
    y = torch.randint(0, 10, (B,))
    m2 = (torch.rand(B, 20) >= 0.5).float() * 2.0
    dm = (torch.rand(B, 50) >= 0.5).float() * 2.0
    out = R.forward_backward(params, x, y, m2, dm)
    return params, x, y, m2, dm, out


def test_pipeline_checks_pass_the_model_itself():
    params, x, y, m2, dm, out = _model_case()
    rep = {}
    bad, _ = BC.compare_pipeline(rep, _engine_buffers(out, 8), params, x, y, m2, dm, grads=out["grads"], loss=out["loss"])
    assert not bad, (bad, rep)
    assert all(v["worst"] == 0.0 for k, v in rep.items() if isinstance(v, dict) and "worst" in v), rep


def test_swapped_sample_is_flagged():
    params, x, y, m2, dm, out = _model_case()
    f = _engine_buffers(out, 8)
    p2 = f.P2.view(8, 320)
    p2[[2, 5]] = p2[[5, 2]].clone()
    rep = {}
    bad, _ = BC.compare_pipeline(rep, f, params, x, y, m2, dm)
    assert any(b.startswith("p2:") for b in bad), bad
    assert rep["p2"]["worst"] >= 10 * BC.STAGE_BOUNDS["p2"], rep["p2"]
    assert rep["p2"]["samples_over"] == 2


def test_second_sample_of_the_last_tile_zeroed_is_flagged():
    params, x, y, m2, dm, out = _model_case()          # B = 8: tiles of 2 samples, the last one (index 3) holds 6 and 7
    for buf, name, rows in (("G1", "g1", 1440), ("DC", "dc", 2048), ("DH", "dh", 64)):
        f = _engine_buffers(out, 8)
        getattr(f, buf).view(8, rows)[7] = 0
        rep = {}
        bad, _ = BC.compare_pipeline(rep, f, params, x, y, m2, dm)
        assert any(b.startswith(name + ":") for b in bad), (name, bad)
        assert rep[name]["worst_sample"] == 7 and rep[name]["worst"] >= 10 * BC.STAGE_BOUNDS[name], rep[name]


def test_one_sample_missing_from_a_reduction_of_8191_is_flagged():
    B, j = 8191, 4000
    op = BC.synthetic("fc_wgrad", B, seed=5, device="cpu")
    want = op["want"]
    bufs = {k: v.double() for k, v in op["bufs"].items()}
    dh, p2, h, dlog = bufs["DH"][:, :50], bufs["P2"], bufs["H"][:, :50], bufs["DLOG"][:, :10]
    drop = {"fc1.weight": torch.outer(dh[j], p2[j]), "fc1.bias": dh[j], "fc2.weight": torch.outer(dlog[j], h[j]),
            "fc2.bias": dlog[j]}
    # a kernel that accumulated every sample: passes; one that skipped sample j: flagged on every gradient
    for missing in (False, True):
        bucket = BC.prefill_bucket(want, "cpu").double()
        for n, v in want.items():
            bucket[BC.param_slots(n)] += (v - drop[n] if missing else v).reshape(-1)
        rep = {}
        bad = BC.check_bucket(rep, "fc_wgrad", bucket.float(), want, BC.REDUCTION_BOUND)
        if not missing:
            assert not bad, (bad, rep)
        else:
            assert len(bad) == 4, (bad, rep)
            assert min(rep[f"fc_wgrad/{n}"]["rel_err"] for n in want) >= 10 * BC.REDUCTION_BOUND, rep


def test_padding_slot_written_is_flagged():
    op = BC.synthetic("conv2_wgrad", 64, seed=6, device="cpu")
    for slot in BC.pad_slots().tolist()[::7] + [BC.LAYOUT["conv1.weight"]]:      # padding, or another kernel's gradient
        bucket = BC.prefill_bucket(op["want"], "cpu")
        for n, v in op["want"].items():
            bucket[BC.param_slots(n)] = 0.0
        bucket[slot] += 1e-3
        rep = {}
        bad = BC.check_bucket(rep, "conv2_wgrad", bucket, op["want"], BC.REDUCTION_BOUND)
        assert len(bad) == 1 and rep["conv2_wgrad/untouched_slots_written"] == [slot], (slot, bad)


def test_pad_slots_are_the_layout_gaps():
    assert BC.pad_slots().tolist() == [250, 251, 262, 263, 21334, 21335] + list(range(21846, 21888))
