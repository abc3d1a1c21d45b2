"""The driver's bench.py contract: one JSON line with the required keys (checked on CPU with synthetic numbers)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_result_line_has_every_required_key():
    from bench_common import result_line
    line = result_line(impl="ours", value=123.0, ms=10.0, n_gpus=2, steps=5, warmup=3,
                       clocks={"sm_mhz": 1965.0, "sm_max_mhz": 1965.0, "reasons": []}, e2e_value=100.0, h2d=10, d2h=8,
                       gpu_launches=10, dtype="fp32", extra_config={"l2": "pool"})
    d = json.loads(line)
    assert "\n" not in line
    for k in ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
              "vs_baseline", "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "impl"]:
        assert k in d, k
    assert d["scaling"] == "strong" and d["higher_is_better"] is True and d["vs_baseline"] is None
    assert d["config"]["global_batch"] == 128 and d["config"]["parallelism"] == "dp2" and d["config"]["per_gpu_batch"] == 64
    assert set(d["e2e"]) == {"value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step"}
    assert d["ms_per_step"] == 2.0


def test_reference_arm_reports_unavailable_or_runs_without_gpu():
    """On a box without CUDA the reference arm must print a single JSON line and exit 0."""
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1", "--warmup", "1"],
                       capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, r.stderr[-500:]
    last = [ln for ln in r.stdout.strip().splitlines() if ln.startswith("{")][-1]
    d = json.loads(last)
    assert d["impl"] == "reference" and ("unavailable" in d or "value" in d)


def test_pick_cluster_policy():
    from dist_tuto.pth_b200.ops.convnet_fused import pick_cluster
    assert [pick_cluster(b) for b in (128, 64, 32, 16, 8, 1)] == [1, 2, 4, 4, 8, 8]
    os.environ["B200DIST_CONVNET_CLUSTER"] = "1"
    try:
        assert pick_cluster(16) == 1
    finally:
        del os.environ["B200DIST_CONVNET_CLUSTER"]


def test_reference_net_matches_golden():
    """The project's Net against the original tutorial's Net (train_dist.py): tests/golden/reference_net.npz holds what the
    original computed with torch.manual_seed(1234) at construction -- its initial parameters (a fixed sample of 2048 entries
    and the sum of every tensor), the eval-mode log-probs of a stored batch, and three training steps on stored batches (SGD
    lr 0.01 momentum 0.5, dropout stream torch.manual_seed(7)): the losses and the parameters after them."""
    import numpy as np
    import torch
    import torch.nn.functional as F
    from dist_tuto.pth_b200.models.convnet import Net
    g = np.load(os.path.join(ROOT, "tests", "golden", "reference_net.npz"))
    torch.manual_seed(1234)
    net = Net()
    flat = lambda m: torch.cat([p.detach().reshape(-1) for p in m.parameters()]).numpy()
    sums = lambda m: np.array([float(p.detach().double().sum()) for p in m.parameters()])
    idx = g["sample_idx"]
    assert np.array_equal(flat(net)[idx], g["init_sample"])
    np.testing.assert_allclose(sums(net), g["init_sums"], rtol=1e-9, atol=1e-9)
    x, y = torch.from_numpy(g["x"]), torch.from_numpy(g["y"])
    net.eval()
    with torch.no_grad():
        np.testing.assert_allclose(net(x[0]).numpy(), g["logp_eval"], rtol=1e-5, atol=1e-6)
    net.train()
    opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.5)
    torch.manual_seed(7)
    losses = []
    for i in range(3):
        opt.zero_grad()
        loss = F.nll_loss(net(x[i]), y[i])
        loss.backward()
        opt.step()
        losses.append(loss.item())
    np.testing.assert_allclose(losses, g["train_losses"], rtol=1e-5)
    np.testing.assert_allclose(flat(net)[idx], g["final_sample"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(sums(net), g["final_sums"], rtol=1e-5, atol=1e-5)


def test_aligned_start_gives_every_rank_the_same_instant():
    """The e2e window of both bench arms starts at a common instant (bench_common.aligned_start), gloo world 2 on the CPU."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import dist_tuto.pth_b200 as b2
    import dist_workers as W
    b2.launch(W.w_aligned_start, size=2, backend="gloo", join_timeout_s=120)
