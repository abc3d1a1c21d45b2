"""GPU-single tier: every sm_90a kernel against a plain PyTorch fp32 oracle (SURVEY §4)."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


@pytest.fixture(scope="module")
def dev():
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda", 0)


def _net(dev, seed=0):
    from dist_tuto.pth_b200.models.convnet import Net
    torch.manual_seed(seed)
    return Net().to(dev)


def _batch(dev, B, seed=1):
    g = torch.Generator(device="cpu").manual_seed(seed)
    x = torch.randn(B, 1, 28, 28, generator=g).to(dev)
    y = torch.randint(0, 10, (B,), generator=g).to(dev)
    return x, y


def _masked_forward(net, x, m2, mh):
    """Oracle forward with explicit dropout scales (m2: [B,20] channel scales, mh: [B,50])."""
    h = F.relu(F.max_pool2d(net.conv1(x), 2))
    h = net.conv2(h) * m2[:, :, None, None]
    h = F.relu(F.max_pool2d(h, 2)).reshape(-1, 320)
    h = F.relu(net.fc1(h)) * mh
    return F.log_softmax(net.fc2(h), dim=1)


def test_extension_is_loaded_not_a_fallback():
    from dist_tuto.pth_b200.ops import _ext
    C = _ext.C()
    assert C.convnet_npar() == 21848 and C.gemm_available()


@pytest.mark.parametrize("B", [1, 7, 128, 300])
def test_convnet_forward_matches_torch(dev, B):
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_forward, pack_params
    net = _net(dev).eval()
    x, _ = _batch(dev, B)
    out = convnet_forward(pack_params(net), x)
    ref = net(x)
    assert out.shape == (B, 10)
    assert torch.allclose(out, ref, atol=2e-4, rtol=1e-4), (out - ref).abs().max()


@pytest.mark.parametrize("B", [1, 16, 128, 200])
def test_convnet_loss_and_grads_match_autograd(dev, B):
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads, pack_params, unpack_params
    net = _net(dev, seed=3).eval()                       # eval: dropout off, autograd still on
    x, y = _batch(dev, B, seed=5)
    loss, grads = convnet_loss_and_grads(pack_params(net), x, y, training=False)
    net64 = net.double()                                 # fp64 oracle: immune to TF32 / algorithm choices in cuDNN
    ref_loss = F.nll_loss(net64(x.double()), y)
    ref_loss.backward()
    assert torch.allclose(loss.double(), ref_loss, atol=1e-4, rtol=1e-4)
    views = unpack_params(grads)
    errs = {}
    for name, p in net64.named_parameters():
        scale = p.grad.abs().max().clamp_min(1e-9)
        errs[name] = float((views[name].double() - p.grad).abs().max() / scale)
    assert max(errs.values()) < 1e-3, errs
    # padding between tensors stays zero
    assert float(grads[250:252].abs().sum()) == 0.0


def test_convnet_training_dropout_matches_masked_oracle(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads, pack_params, unpack_params
    net = _net(dev, seed=4).eval()
    B = 64
    x, y = _batch(dev, B, seed=6)
    step = torch.tensor([3], dtype=torch.int64, device=dev)
    loss, grads, masks = convnet_loss_and_grads(pack_params(net), x, y, training=True, seed=77, step=step,
                                                return_masks=True)
    vals = set(masks.unique().tolist())
    assert vals <= {0.0, 2.0} and len(vals) == 2          # p=0.5 -> scale 2 or dropped
    assert 0.3 < float((masks > 0).float().mean()) < 0.7
    params_flat = pack_params(net)
    net64 = net.double()
    ref_loss = F.nll_loss(_masked_forward(net64, x.double(), masks[:, :20].double(), masks[:, 20:].double()), y)
    ref_loss.backward()
    assert torch.allclose(loss.double(), ref_loss, atol=1e-4, rtol=1e-4)
    views = unpack_params(grads)
    errs = {}
    for name, p in net64.named_parameters():
        scale = p.grad.abs().max().clamp_min(1e-9)
        errs[name] = float((views[name].double() - p.grad).abs().max() / scale)
    assert max(errs.values()) < 1e-3, errs
    net = net64.float()
    # different step -> different masks; same step -> same masks
    _, _, m_same = convnet_loss_and_grads(params_flat, x, y, training=True, seed=77, step=step, return_masks=True)
    _, _, m_diff = convnet_loss_and_grads(params_flat, x, y, training=True, seed=77, step=step + 1,
                                          return_masks=True)
    assert torch.equal(masks, m_same) and not torch.equal(masks, m_diff)


def test_convnet_uint8_input_normalised_in_kernel(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_forward, pack_params
    net = _net(dev).eval()
    xu = torch.randint(0, 256, (32, 1, 28, 28), dtype=torch.uint8, device=dev)
    xf = (xu.float() / 255.0 - 0.1307) / 0.3081
    assert torch.allclose(convnet_forward(pack_params(net), xu), net(xf), atol=3e-4, rtol=1e-4)


def test_sgd_flat_matches_torch(dev):
    from dist_tuto.pth_b200.ops import _ext
    C = _ext.C()
    n = 10007
    p = torch.randn(n, device=dev)
    g = torch.randn(n, device=dev)
    m = torch.zeros(n, device=dev)
    ref = p.clone().requires_grad_(True)
    opt = torch.optim.SGD([ref], lr=0.01, momentum=0.5)
    for _ in range(3):
        ref.grad = g.clone()
        opt.step()
        C.sgd_flat(p, m, g, 0.01, 0.5, 0.0, False)
    assert torch.allclose(p, ref.detach(), atol=1e-6)


def test_fused_trainer_matches_torch_sgd_single_gpu(dev):
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer, unpack_params
    torch.manual_seed(11)
    ref = Net(p_drop=0.0).to(dev)
    tr = FusedTrainer(32, lr=0.05, momentum=0.5, seed=11, device=dev, p_drop=0.0, init_from=ref)
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    losses = []
    for i in range(6):
        x, y = _batch(dev, 32, seed=100 + i)
        xp, yp = x.cpu().pin_memory(), y.cpu().pin_memory()
        tr.step(xp, yp)                                  # graph path, pinned host input
        opt.zero_grad()
        loss = F.nll_loss(ref(x), y)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    got = tr.pop_loss_sum()
    assert abs(got - sum(losses)) < 1e-3 * max(1.0, abs(sum(losses)))
    views = unpack_params(tr.params)
    for name, p in ref.named_parameters():
        assert torch.allclose(views[name], p.detach(), atol=2e-4, rtol=1e-3), name
    sd = tr.state_dict()
    assert sd["steps"] == 6 and set(sd["model"]) == {n for n, _ in ref.named_parameters()}
    # eval forward through the trainer == torch module with the same weights
    x, _ = _batch(dev, 8, seed=999)
    assert torch.allclose(tr.eval()(x), tr.to_module().to(dev).eval()(x), atol=2e-4)


def test_fused_trainer_short_batch_and_device_input(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    tr = FusedTrainer(16, seed=1, device=dev, p_drop=0.5)
    x, y = _batch(dev, 5)
    tr.step(x, y)                                        # eager path: short batch, device tensors
    assert tr.pop_loss_sum() > 0


@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (256, 50, 320), (1000, 10, 512), (300, 200, 136), (64, 32, 8),
                                   (4096, 512, 1024), (4096, 256, 512), (2000, 1000, 264), (8192, 1003, 520),
                                   (2500, 2048, 2056), (8192, 4096, 4096)])
def test_tcgen05_gemm_matches_torch(dev, M, N, K):
    from dist_tuto.pth_b200.ops.gemm import linear_bf16
    g = torch.Generator(device="cpu").manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).to(dev).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(dev).to(torch.bfloat16)
    bias = torch.randn(N, generator=g).to(dev)
    ref = a.float() @ w.float().t() + bias
    out = linear_bf16(a, w, bias, relu=False, out_dtype=torch.float32)
    assert out.shape == (M, N)
    assert torch.allclose(out, ref, atol=2e-2, rtol=2e-2), float((out - ref).abs().max())
    out_r = linear_bf16(a, w, bias, relu=True, out_dtype=torch.bfloat16)
    assert torch.allclose(out_r.float(), ref.relu(), atol=6e-2, rtol=3e-2)


@pytest.mark.parametrize("lead,K,N", [((256,), 320, 50), ((96,), 200, 10), ((8, 50), 512, 1000), ((1000,), 64, 64)])
def test_tc_linear_forward_backward_on_tcgen05(dev, lead, K, N):
    """`linear_tc`: forward, data gradient and weight gradient all on csrc/gemm_tcgen05.cu, vs the same op in fp32 on the same
    bf16-rounded operands (the only differences left: accumulation order and the bf16 rounding of dY)."""
    from dist_tuto.pth_b200.ops.gemm import TcLinear
    g = torch.Generator().manual_seed(K + N)
    m = TcLinear(K, N).to(dev)
    x = torch.randn(*lead, K, generator=g).to(dev).requires_grad_()
    gy = torch.randn(*lead, N, generator=g).to(dev)
    y = m(x)
    y.backward(gy)
    xr = x.detach().to(torch.bfloat16).float().requires_grad_()
    wr = m.weight.detach().to(torch.bfloat16).float().requires_grad_()
    br = m.bias.detach().clone().requires_grad_()
    yr = F.linear(xr, wr, br)
    yr.backward(gy.to(torch.bfloat16).float())
    for got, ref, name in ((y, yr, "y"), (x.grad, xr.grad, "dx"), (m.weight.grad, wr.grad, "dw")):
        scale = float(ref.abs().max())
        assert got.shape == ref.shape and float((got - ref).abs().max()) < 2e-3 * scale + 1e-5, (name, float((got - ref).abs().max()), scale)
    assert torch.allclose(m.bias.grad, gy.reshape(-1, N).sum(0), atol=1e-3, rtol=1e-4)
    # and it trains: a few SGD steps reduce a regression loss
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    tgt = torch.randn(*lead, N, generator=g).to(dev)
    losses = []
    for _ in range(5):
        opt.zero_grad()
        loss = F.mse_loss(m(x.detach()), tgt)
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0]


def test_train_loop_single_gpu_fused(dev):
    import dist_tuto.pth_b200 as b2
    from dist_tuto.pth_b200.data import SyntheticMNIST
    ds = SyntheticMNIST(n=2048, seed=5)
    out = {}

    def fn(rank, size):
        out.update(b2.train(rank, size, b2.TrainConfig(epochs=3, dataset=ds, lr=0.1, log=lambda *a: None)))

    b2.init_processes(0, 1, fn, backend="b200", master_port=b2.find_free_port())
    assert out["loss"][-1] < out["loss"][0] - 0.05, out["loss"]


def test_train_loop_picks_the_batched_engine_for_large_batches(dev):
    """train(): engine="auto" takes the wgmma batched engine from 2048 samples per GPU up (short tail batch included)."""
    import dist_tuto.pth_b200 as b2
    from dist_tuto.pth_b200.data import SyntheticMNIST
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    ds = SyntheticMNIST(n=2048 * 3 + 500, seed=5)
    out = {}

    def fn(rank, size):
        out.update(b2.train(rank, size, b2.TrainConfig(epochs=4, dataset=ds, lr=0.1, global_batch=2048, log=lambda *a: None)))

    b2.init_processes(0, 1, fn, backend="b200", master_port=b2.find_free_port())
    assert isinstance(out["model"], BatchedTrainer) and out["bsz"] == 2048 and out["steps"] == 16
    assert out["loss"][-1] < out["loss"][0] - 0.02, out["loss"]


@pytest.mark.parametrize("num_buffers", [4, 5, 6, 7, 8, 12, 24, 100])
def test_native_executor_matches_python_loop(dev, num_buffers):
    """C++ StepExecutor (prefetch thread -> kernel launches) == stepping the same loader from Python.
    The ring depth sets how many steps are in flight (num_buffers - 2) and how many device blocks the executor feeds;
    4 is the shallowest ring a NativeBatchLoader has."""
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    ds = D.SyntheticMNIST(n=1000, seed=2)                 # 1000 = 15 x 64 + 40 -> exercises the short tail batch
    part = D.Partition(ds, list(range(1000)))
    res = []
    for native in (True, False):
        loader = D.NativeBatchLoader(part, 64, seed=9, raw_uint8=True, pin_memory=True, num_buffers=num_buffers)
        tr = FusedTrainer(64, lr=0.05, seed=3, device=dev, p_drop=0.5, raw_uint8=True)
        if native:
            done, finished = tr.run_native(loader)
            assert done == 16 and finished
            torch.cuda.synchronize()                      # the epoch ended with the eager short batch: its loss is the last one
            assert tr.last_loss_cumulative() == float(tr.loss_acc[0].item())
            ex = tr._executors[id(loader)][0]                # what bench.py reads from the executor
            stats = ex.stats()
            assert stats and all(isinstance(v, (int, float)) for v in stats.values()), stats
            ex.reset_stats()
            assert ex.flag_mode() is False and ex.chunking() is False
            done2, _ = tr.run_native(loader, max_steps=6)        # second epoch, budgeted
            assert done2 == 6 and ex.stats()["steps"] == 6
        else:
            n = 0
            for x, y in loader:
                tr.step(x, y)
                n += 1
            assert n == 16
            for i, (x, y) in enumerate(loader):
                if i == 6:
                    break
                tr.step(x, y)
        torch.cuda.synchronize()                          # the python loop's last steps are still in flight on tr.stream
        res.append((tr.params.clone(), tr.pop_loss_sum(), int(tr.step_counter.item())))
    assert res[0][2] == res[1][2] == 22
    assert abs(res[0][1] - res[1][1]) < 1e-3 * abs(res[1][1])
    assert torch.allclose(res[0][0], res[1][0], atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("cluster,B", [(2, 1), (2, 64), (4, 5), (4, 32), (8, 1), (8, 16), (8, 40)])
def test_convnet_cluster_per_sample_matches_fp64_oracle(dev, cluster, B):
    """One thread-block cluster (2/4/8 CTAs, DSMEM broadcasts) per sample: same numerics as the one-CTA kernel."""
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads, pack_params, unpack_params
    net = _net(dev, seed=3).eval()
    x, y = _batch(dev, B, seed=5)
    flat = pack_params(net)
    loss, grads = convnet_loss_and_grads(flat, x, y, training=False, cluster=cluster)
    net64 = net.double()
    ref_loss = F.nll_loss(net64(x.double()), y)
    ref_loss.backward()
    assert torch.allclose(loss.double(), ref_loss, atol=1e-4, rtol=1e-4)
    views = unpack_params(grads)
    errs = {}
    for name, p in net64.named_parameters():
        scale = p.grad.abs().max().clamp_min(1e-9)
        errs[name] = float((views[name].double() - p.grad).abs().max() / scale)
    assert max(errs.values()) < 1e-3, errs
    assert float(grads[250:252].abs().sum()) == 0.0


def test_convnet_cluster_dropout_masks_match_single_cta_kernel(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import convnet_loss_and_grads, pack_params
    net = _net(dev, seed=4).eval()
    x, y = _batch(dev, 16, seed=6)
    flat = pack_params(net)
    step = torch.tensor([5], dtype=torch.int64, device=dev)
    l1, g1, m1 = convnet_loss_and_grads(flat, x, y, training=True, seed=9, step=step, return_masks=True, cluster=1)
    l8, g8, m8 = convnet_loss_and_grads(flat, x, y, training=True, seed=9, step=step, return_masks=True, cluster=8)
    assert torch.equal(m1, m8)
    assert torch.allclose(l1, l8, atol=1e-5)
    assert torch.allclose(g1, g8, atol=1e-5, rtol=1e-4)


def test_fused_trainer_uses_clusters_for_small_batches(dev):
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer, pick_cluster
    assert [pick_cluster(b) for b in (128, 64, 32, 16, 8)] == [1, 2, 4, 4, 8]
    res = []
    for cluster in (1, 8):
        tr = FusedTrainer(16, lr=0.05, seed=3, device=dev, p_drop=0.5, cluster=cluster)
        g = torch.Generator().manual_seed(1)
        for i in range(8):
            tr.step(torch.randn(16, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (16,), generator=g).pin_memory())
        res.append((tr.pop_loss_sum(), tr.params.clone()))
    assert abs(res[0][0] - res[1][0]) < 1e-3
    assert torch.allclose(res[0][1], res[1][1], atol=1e-5, rtol=1e-4)


def test_load_state_dict_rewinds_step_parity_and_buckets(dev):
    """load_state_dict() may move the step counter to the other parity: the double-buffered gradient buckets must both be
    clean afterwards (the kernels only re-zero the bucket of the previous parity)."""
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    tr = FusedTrainer(32, lr=0.05, seed=8, device=dev, p_drop=0.5)

    def batch(i):
        g = torch.Generator().manual_seed(1000 + i)
        return torch.randn(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).pin_memory()

    for i in range(7):
        tr.step(*batch(i))
    snap = tr.state_dict()
    for i in range(7, 11):                   # ends at step 11 (odd); snap is step 7 (odd) -> take one more to flip parity
        tr.step(*batch(i))
    tr.step(*batch(11))
    tr.load_state_dict(snap)                 # 12 (even) -> 7 (odd)
    for i in range(7, 11):
        tr.step(*batch(i))
    tr.sync_lag(0)
    torch.cuda.synchronize()
    again = tr.params.clone()
    fresh = FusedTrainer(32, lr=0.05, seed=8, device=dev, p_drop=0.5)
    fresh.load_state_dict(snap)
    for i in range(7, 11):
        fresh.step(*batch(i))
    fresh.sync_lag(0)
    torch.cuda.synchronize()
    assert int(tr.step_counter.item()) == int(fresh.step_counter.item()) == 11
    # (not bit-equal: the per-CTA gradient flush is a float atomic, its order varies run to run)
    assert torch.allclose(again, fresh.params, atol=2e-5, rtol=1e-4)


def test_fused_trainer_checkpoint_roundtrip_restores_momentum_and_steps(dev, tmp_path):
    """save_checkpoint / load_checkpoint on the fused trainer: parameters, momentum AND the device step counter."""
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    from dist_tuto.pth_b200.utils.checkpoint import load_checkpoint, save_checkpoint

    def batch(i):
        g = torch.Generator().manual_seed(2000 + i)
        return torch.randn(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).pin_memory()

    a = FusedTrainer(32, lr=0.05, momentum=0.9, seed=1, device=dev, p_drop=0.0)
    for i in range(5):
        a.step(*batch(i))
    path = save_checkpoint(str(tmp_path / "t.pt"), a, history=[0.5])
    for i in range(5, 8):
        a.step(*batch(i))
    a.sync_lag(0)
    b = FusedTrainer(32, lr=0.05, momentum=0.9, seed=99, device=dev, p_drop=0.0)      # different init
    blob = load_checkpoint(path, b)
    assert blob["steps"] == 5 and int(b.step_counter.item()) == 5 and float(b.momentum.abs().sum()) > 0
    for i in range(5, 8):
        b.step(*batch(i))
    b.sync_lag(0)
    torch.cuda.synchronize()
    assert torch.allclose(a.params, b.params, atol=2e-5, rtol=1e-4)
    assert torch.allclose(a.momentum, b.momentum, atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("bsz", [128, 32])
def test_deterministic_mode_is_bit_reproducible(dev, bsz):
    """deterministic=True: per-CTA gradient slots summed in CTA order -> two runs are bit-equal (the default float red.add
    flush is only equal to ~1e-6); and the result agrees with the default mode to rounding."""
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer

    def run(det):
        tr = FusedTrainer(bsz, lr=0.05, seed=13, device=dev, p_drop=0.5, deterministic=det)
        g = torch.Generator().manual_seed(99)
        for _ in range(12):
            tr.step(torch.randn(bsz, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (bsz,), generator=g).pin_memory())
        tr.sync_lag(0)
        torch.cuda.synchronize()
        return tr.params.clone(), tr.momentum.clone(), tr.pop_loss_sum()

    a, b, c = run(True), run(True), run(False)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]      # parameters, momentum AND the loss sum
    assert torch.allclose(a[0], c[0], atol=2e-5, rtol=1e-4)
