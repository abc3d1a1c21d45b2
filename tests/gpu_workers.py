"""Workers for the GPU-multi tier (spawned, one process per GPU, backend 'b200')."""
import os

import torch
import torch.distributed as dist
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200 import ring
from dist_tuto.pth_b200.parallel import symm


def _dev():
    # the torch models these workers compare against must be fp32 references: cuDNN / cuBLAS default to TF32 (10-bit
    # mantissa) for fp32 convolutions, which by itself moves 5 SGD steps by ~1e-3
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda", torch.cuda.current_device())


def w_symm_allreduce(rank, size):
    dev = _dev()
    w = symm.lookup_world(None)
    assert w is not None and w.world == size
    info = w.describe()
    if rank == 0:
        print("SYMM", info, flush=True)
    variants = [0, 1, 3] + ([2] if w.multicast else [])       # one-shot, two-shot, LL (falls back to one-shot > 64 KB), NVLS
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 2e-2)):
        for n in (1, 7, 64, 1000, 21888, 65536 + 3, 1 << 20):
            g = torch.Generator(device="cpu").manual_seed(1000 + rank)
            local = torch.randn(n, generator=g).to(dev).to(dtype)
            ref = local.clone().float()
            dist.all_reduce(ref)                      # NCCL oracle (fp32 accumulate)
            ref = ref / size
            # (a) zero-copy symmetric buffer, every variant
            hd = w.alloc(n, dtype)
            for v in variants:
                hd.local.zero_()
                hd.local[:n].copy_(local)
                torch.cuda.synchronize()
                dist.barrier()
                w.all_reduce_(hd.local, scale=1.0 / size, handle=hd, variant=v)
                torch.cuda.synchronize()
                got = hd.local[:n].float()
                assert torch.allclose(got, ref, atol=tol, rtol=tol), (str(dtype), n, v, float((got - ref).abs().max()))
                # bit-identical on every rank (fixed reduction order)
                mine = hd.local[:n].clone()
                other = mine.clone()
                dist.broadcast(other, src=0)
                assert torch.equal(mine, other), ("replica mismatch", str(dtype), n, v)
            # (b) arbitrary tensor through the staging buffer (fused copy-in/out or ragged path)
            for v in variants:
                t = local.clone()
                w.all_reduce_(t, scale=1.0 / size, variant=v)
                torch.cuda.synchronize()
                assert torch.allclose(t.float(), ref, atol=tol, rtol=tol), ("staged", str(dtype), n, v)
    # (c) fp32 tensor, bf16 on the wire
    t = torch.randn(4096, generator=torch.Generator().manual_seed(5 + rank)).to(dev)
    ref = t.clone()
    dist.all_reduce(ref)
    w.all_reduce_(t, wire=torch.bfloat16)
    torch.cuda.synchronize()
    assert torch.allclose(t, ref, atol=5e-2, rtol=5e-2)
    # (d) repeated calls: flag reuse must not race
    hd = w.alloc(4096, torch.float32)
    for it in range(200):
        hd.local.fill_(float(rank + it))
        w.all_reduce_(hd.local, handle=hd, variant=it % len(variants))
    torch.cuda.synchronize()
    expect = float(sum(r + 199 for r in range(size)))
    assert torch.allclose(hd.local, torch.full_like(hd.local, expect)), float(hd.local[0])
    # (e) public API routes CUDA float SUM to the fused kernels
    t = torch.ones(10, device=dev)
    b2.all_reduce(t)
    assert float(t[0]) == size
    dist.barrier()


def w_average_gradients_gpu(rank, size):
    dev = _dev()
    torch.manual_seed(1234)
    model = b2.Net().to(dev).eval()
    g = torch.Generator().manual_seed(50 + rank)
    x = torch.randn(8, 1, 28, 28, generator=g).to(dev)
    y = torch.randint(0, 10, (8,), generator=g).to(dev)
    F.nll_loss(model(x), y).backward()
    local = [p.grad.clone() for p in model.parameters()]
    ref = []
    for gl in local:
        r = gl.clone()
        dist.all_reduce(r)
        ref.append(r / size)
    b2.average_gradients(model)
    for p, r in zip(model.parameters(), ref):
        assert torch.allclose(p.grad, r, atol=1e-6)
    # overlapped bucketed DDP on symmetric buckets
    from dist_tuto.pth_b200.parallel.ddp import DistributedDataParallel
    torch.manual_seed(7 + rank)
    m2 = b2.Net().to(dev).eval()
    ddp = DistributedDataParallel(m2, bucket_cap_bytes=16 << 10)
    assert len(ddp.buckets) >= 2 and ddp.buckets[0].world is not None
    m3 = b2.Net().to(dev).eval()
    m3.load_state_dict(m2.state_dict())
    F.nll_loss(m3(x), y).backward()
    ref = []
    for p in m3.parameters():
        r = p.grad.clone()
        dist.all_reduce(r)
        ref.append(r / size)
    for it in range(3):
        ddp.zero_grad()
        F.nll_loss(ddp(x), y).backward()
        b2.average_gradients(m2)
        torch.cuda.synchronize()
        for p, r in zip(m2.parameters(), ref):
            assert torch.allclose(p.grad, r, atol=1e-6), it
    dist.barrier()


def w_fused_trainer(rank, size):
    """World-N fused trainer == single-process torch SGD on the concatenated global batch."""
    dev = _dev()
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer, unpack_params
    bsz = 16
    torch.manual_seed(21)
    ref = Net(p_drop=0.0).to(dev)
    tr = FusedTrainer(bsz, lr=0.05, momentum=0.5, seed=21, device=dev, p_drop=0.0, init_from=ref, grad_wire=torch.float32)
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    for i in range(5):
        g = torch.Generator().manual_seed(300 + i)
        xg = torch.randn(bsz * size, 1, 28, 28, generator=g)
        yg = torch.randint(0, 10, (bsz * size,), generator=g)
        xs, ys = xg[rank * bsz:(rank + 1) * bsz].contiguous().pin_memory(), yg[rank * bsz:(rank + 1) * bsz].contiguous().pin_memory()
        tr.step(xs, ys)
        opt.zero_grad()
        F.nll_loss(ref(xg.to(dev)), yg.to(dev)).backward()     # mean over the GLOBAL batch
        opt.step()
    tr.sync_lag(0)
    torch.cuda.synchronize()
    views = unpack_params(tr.params)
    for name, p in ref.named_parameters():
        assert torch.allclose(views[name], p.detach(), atol=5e-4, rtol=5e-3), (name, float((views[name] - p.detach()).abs().max()))
    # replicas bit-identical
    mine = tr.params.clone()
    other = mine.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(mine, other)
    # with dropout on: still bit-identical replicas, finite loss
    tr2 = FusedTrainer(bsz, seed=5, device=dev, p_drop=0.5)
    for i in range(20):
        g = torch.Generator().manual_seed(900 + i * size + rank)
        tr2.step(torch.randn(bsz, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (bsz,), generator=g).pin_memory())
    loss = tr2.pop_loss_sum()
    assert loss == loss and loss > 0
    mine = tr2.params.clone()
    other = mine.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(mine, other)
    dist.barrier()


def w_push_exchange_equals_barrier_exchange(rank, size):
    """allreduce_sgd_push_kernel (flag-in-data stores into the peers' inboxes) == barrier + peer loads,
    through the Python graph path, the C++ executor and a load_state_dict() rewind of the step counter (epoch reuse)."""
    import os
    dev = _dev()
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    bsz = 16
    ds = D.SyntheticMNIST(n=bsz * size * 12 + 5 * size, seed=4)        # 12 full batches + a short tail per rank
    idx = list(range(rank, len(ds), size))
    results = {}
    # the optimizer kernel after the step kernel: barrier + peer loads | push (default)
    for push in ("0", "1"):
        os.environ["B200DIST_SGD_PUSH"] = push
        tr = FusedTrainer(bsz, lr=0.05, seed=11, device=dev, p_drop=0.5, raw_uint8=True, grad_wire=torch.float32)
        assert (tr.inbox_handle is not None) == (push == "1")
        assert tr.gpu_launches_per_step == 2
        for i in range(7):                                             # python graph path, odd count -> both parities
            g = torch.Generator().manual_seed(50 + i * size + rank)
            tr.step(torch.randint(0, 255, (bsz, 1, 28, 28), generator=g, dtype=torch.uint8).pin_memory(),
                    torch.randint(0, 10, (bsz,), generator=g).pin_memory())
        tr.sync_lag(0)
        snap = tr.state_dict()
        loader = D.NativeBatchLoader(D.Partition(ds, idx), bsz, seed=3, raw_uint8=True, pin_memory=True)
        done, fin = tr.run_native(loader)                              # C++ executor + eager short tail
        assert done == 13 and fin
        tr.load_state_dict(snap)                                       # rewinds the step counter: inbox epochs are reused
        done, _ = tr.run_native(loader, max_steps=9)
        assert done == 9
        torch.cuda.synchronize()
        results[push] = (tr.params.clone(), tr.momentum.clone(), int(tr.step_counter.item()))
        mine = tr.params.clone()
        other = mine.clone()
        dist.broadcast(other, src=0)
        assert torch.equal(mine, other), ("replicas differ", push)
        del tr
    os.environ.pop("B200DIST_SGD_PUSH", None)
    assert results["0"][2] == results["1"][2] == 16
    # same maths in the same rank order; run-to-run differences only from the float-atomic gradient flush inside a GPU
    assert torch.allclose(results["0"][0], results["1"][0], atol=2e-5, rtol=1e-4)
    assert torch.allclose(results["0"][1], results["1"][1], atol=2e-5, rtol=1e-4)
    dist.barrier()


def w_p2p_ring_gpu(rank, size):
    dev = _dev()
    t = torch.zeros(4, device=dev)
    if rank == 0:
        t += 1
        b2.send(t, dst=1)
    elif rank == 1:
        b2.recv(t, src=0)
        assert float(t[0]) == 1.0
    send = torch.arange(6, dtype=torch.float32, device=dev) * (rank + 1)
    recv = torch.zeros(6, device=dev)
    b2.allreduce(send, recv)
    torch.cuda.synchronize()
    assert torch.allclose(recv, torch.arange(6, dtype=torch.float32, device=dev) * sum(r + 1 for r in range(size)))
    recv2 = torch.zeros(1000, device=dev)
    src = torch.randn(1000, generator=torch.Generator().manual_seed(rank)).to(dev)
    ring.allreduce_chunked(src, recv2)
    ref = src.clone()
    dist.all_reduce(ref)
    assert torch.allclose(recv2, ref, atol=1e-4)
    dist.barrier()


def w_train_fused_e2e(rank, size):
    from dist_tuto.pth_b200.data import SyntheticMNIST
    ds = SyntheticMNIST(n=2048, seed=5)
    logs = []
    cfg = b2.TrainConfig(epochs=3, dataset=ds, lr=0.1, log=lambda *a: logs.append(a))
    out = b2.train(rank, size, cfg)
    assert out["loss"][-1] < out["loss"][0] - 0.05, out["loss"]
    dist.barrier()


def w_train_torch_engine_gpu(rank, size):
    """The tutorial loop on torch CUDA ops (engine='torch'): gradients in ONE symmetric flat bucket averaged by the fused
    peer-memory all-reduce, update + zero_grad by the `sgd_flat` kernel (`FlatSGD`).  Replicas stay bit-identical."""
    from dist_tuto.pth_b200.data import SyntheticMNIST
    ds = SyntheticMNIST(n=2048, seed=5)
    cfg = b2.TrainConfig(epochs=2, dataset=ds, lr=0.1, engine="torch", log=lambda *a: None)
    out = b2.train(rank, size, cfg)
    assert out["loss"][-1] == out["loss"][-1] and out["loss"][-1] < out["loss"][0], out["loss"]
    model = out["model"]
    assert model._grad_bucket.world is not None and model._grad_bucket.flat.numel() >= model._grad_bucket.numel
    flat = torch.cat([p.detach().reshape(-1) for p in model.parameters()])
    other = flat.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(flat, other)
    # generic model: bucketed overlapped DDP (symmetric, padded buckets) + FlatSGD, bf16 autocast, channels_last
    from dist_tuto.pth_b200.models.resnet import ResNet18
    dev = _dev()
    torch.manual_seed(3 + rank)                                  # broadcast inside DDP must make the replicas equal
    net = ResNet18(num_classes=10).to(dev).to(memory_format=torch.channels_last)
    ddp = b2.DistributedDataParallel(net, bucket_cap_bytes=4 << 20)
    opt = b2.FlatSGD(ddp, lr=0.01, momentum=0.5)
    assert len(opt.buckets) > 1 and all(b.world is not None for b in opt.buckets)
    for it in range(3):
        g = torch.Generator().manual_seed(700 + it * size + rank)
        x = torch.randn(8, 3, 64, 64, generator=g).to(dev).to(memory_format=torch.channels_last)
        y = torch.randint(0, 10, (8,), generator=g).to(dev)
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(ddp(x), y)
        loss.backward()
        b2.average_gradients(net)
        opt.step()
    torch.cuda.synchronize()
    assert bool(torch.isfinite(loss))
    flat = torch.cat([p.detach().reshape(-1) for p in net.parameters()])
    other = flat.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(flat, other)
    ddp.remove_hooks()
    dist.barrier()


def w_suite_odd_world(rank, size):
    """Everything that touches the peer-memory protocols, at a world size the power-of-two tests never see (the reference's
    gloo.py:59 runs 7 ranks): all-reduce variants incl. sizes that are not multiples of the world, the fused trainer against
    global-batch SGD, and the three exchange flavours against each other."""
    dev = _dev()
    w = symm.lookup_world(None)
    assert w is not None and w.world == size
    variants = [0, 1, 3] + ([2] if w.multicast else [])       # one-shot, two-shot, LL (falls back to one-shot > 64 KB), NVLS
    for dtype, tol in ((torch.float32, 1e-5), (torch.bfloat16, 2e-2)):
        for n in (1, 5, 64, 21888, 65536 + 3, (1 << 20) + 7):
            g = torch.Generator(device="cpu").manual_seed(1000 + rank)
            local = torch.randn(n, generator=g).to(dev).to(dtype)
            ref = local.clone().float()
            dist.all_reduce(ref)
            ref = ref / size
            hd = w.alloc(n, dtype)
            for v in variants:
                hd.local.zero_()
                hd.local[:n].copy_(local)
                torch.cuda.synchronize()
                dist.barrier()
                w.all_reduce_(hd.local, scale=1.0 / size, handle=hd, variant=v)
                torch.cuda.synchronize()
                got = hd.local[:n].float()
                assert torch.allclose(got, ref, atol=tol, rtol=tol), (size, str(dtype), n, v, float((got - ref).abs().max()))
                mine = hd.local[:n].clone()
                other = mine.clone()
                dist.broadcast(other, src=0)
                assert torch.equal(mine, other), ("replica mismatch", size, str(dtype), n, v)
            t = local.clone()
            w.all_reduce_(t, scale=1.0 / size)
            torch.cuda.synchronize()
            assert torch.allclose(t.float(), ref, atol=tol, rtol=tol), ("staged", size, str(dtype), n)
    w_fused_trainer(rank, size)
    w_push_exchange_equals_barrier_exchange(rank, size)


def w_flag_reuse_stress(rank, size):
    """10^5 back-to-back fused all-reduces with the variant changing every call (signal-pad epochs, SURVEY 7.4 hard part 1),
    then 20000 one-kernel training steps replayed from CUDA graphs (inbox epochs / parity double-buffer of the push exchange)."""
    dev = _dev()
    w = symm.lookup_world(None)
    variants = [0, 1, 3] + ([2] if w.multicast else [])       # one-shot, two-shot, LL (falls back to one-shot > 64 KB), NVLS
    hd = w.alloc(4096, torch.float32)
    n_it = int(os.environ.get("B200DIST_STRESS_ITERS", "100000"))
    hd.local.fill_(1.0)
    torch.cuda.synchronize()
    dist.barrier()
    for it in range(n_it):                       # t <- mean over ranks of t  (stays exactly 1.0: any lost/duplicated add shows)
        w.all_reduce_(hd.local, scale=1.0 / size, handle=hd, variant=variants[it % len(variants)])
        if it % 10000 == 9999:
            torch.cuda.synchronize()
            assert torch.allclose(hd.local, torch.ones_like(hd.local), atol=1e-4), (it, float(hd.local.min()), float(hd.local.max()))
    torch.cuda.synchronize()
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    bsz = max(1, 128 // size)
    tr = FusedTrainer(bsz, lr=0.001, seed=3, device=dev, p_drop=0.5)
    g = torch.Generator(device=dev).manual_seed(7 + rank)
    xs = torch.randn(8, bsz, 1, 28, 28, device=dev, generator=g)
    ys = torch.randint(0, 10, (8, bsz), device=dev, generator=g)
    st = tr.stream
    with torch.cuda.stream(st):
        tr._kernels(xs[0], ys[0], bsz)
    st.synchronize()
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr, stream=st):
        for i in range(8):
            tr._kernels(xs[i], ys[i], bsz)
    with torch.cuda.stream(st):
        for _ in range(2500):
            gr.replay()
    st.synchronize()
    assert int(tr.step_counter.item()) == 20001
    assert bool(torch.isfinite(tr.params).all())
    mine = tr.params.clone()
    other = mine.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(mine, other)
    dist.barrier()


def w_large_sizes_vs_nccl(rank, size):
    """Full-tensor comparison against NCCL up to 1 GiB (BASELINE B3 range), every variant the host exposes."""
    dev = _dev()
    w = symm.lookup_world(None)
    variants = [1] + ([2] if w.multicast else [])
    for n in (16 << 20, 64 << 20, 256 << 20):            # fp32 elements: 64 MiB, 256 MiB, 1 GiB
        g = torch.Generator(device=dev).manual_seed(11 + rank)
        hd = w.alloc(n, torch.float32)
        src = torch.randn(n, device=dev, generator=g)
        ref = src.clone()
        dist.all_reduce(ref)
        for v in variants:
            hd.local[:n].copy_(src)
            torch.cuda.synchronize()
            dist.barrier()
            w.all_reduce_(hd.local, handle=hd, variant=v)
            torch.cuda.synchronize()
            err = float((hd.local[:n] - ref).abs().max())
            assert err < 1e-3, (n, v, err)
        del src, ref
    dist.barrier()


def w_subgroup_symmetric_world(rank, size):
    """tuto.md:176-186: collectives on a sub-group.  A symmetric world (own mappings, own signal pads) over a subset of
    the GPUs, used by all_reduce and by a fused trainer, while the other ranks idle."""
    dev = _dev()
    members = list(range(1, size)) if size > 2 else [0, 1]
    grp = b2.new_group(members)
    if rank in members:
        t = torch.full((1000,), float(rank + 1), device=dev)
        b2.all_reduce(t, group=grp)
        assert float(t[0]) == float(sum(r + 1 for r in members))
        wg = symm.lookup_world(grp) or symm.init_world(grp)
        assert wg.world == len(members)
        from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
        tr = FusedTrainer(8, seed=2, device=dev, p_drop=0.5, group=grp)
        for i in range(6):
            g = torch.Generator().manual_seed(40 + i * size + rank)
            tr.step(torch.randn(8, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (8,), generator=g).pin_memory())
        tr.sync_lag(0)
        torch.cuda.synchronize()
        mine = tr.params.clone()
        other = mine.clone()
        dist.broadcast(other, src=members[0], group=grp)
        assert torch.equal(mine, other)
    dist.barrier()


def w_batched_trainer(rank, size):
    """Batched tensor-core engine, world N == torch SGD on the concatenated global batch (eval-mode network)."""
    dev = _dev()
    from dist_tuto.pth_b200.models.convnet import Net
    from dist_tuto.pth_b200.ops.convnet_batched import BatchedTrainer
    from dist_tuto.pth_b200.ops.convnet_fused import unpack_params
    bsz = 192
    torch.manual_seed(33)
    ref = Net(p_drop=0.0).to(dev).eval()
    tr = BatchedTrainer(bsz, lr=0.05, momentum=0.5, seed=21, device=dev, p_drop=0.0, init_from=ref)
    tr.eval()
    opt = torch.optim.SGD(ref.parameters(), lr=0.05, momentum=0.5)
    for i in range(6):
        g = torch.Generator().manual_seed(500 + i)
        xg = torch.randn(bsz * size, 1, 28, 28, generator=g)
        yg = torch.randint(0, 10, (bsz * size,), generator=g)
        tr.step(xg[rank * bsz:(rank + 1) * bsz].contiguous().pin_memory(), yg[rank * bsz:(rank + 1) * bsz].contiguous().pin_memory())
        opt.zero_grad()
        F.nll_loss(ref(xg.to(dev)), yg.to(dev)).backward()
        opt.step()
    tr.stream.synchronize()
    views = unpack_params(tr.params)
    for name, p in ref.named_parameters():
        rel = float((views[name] - p.detach()).norm() / p.detach().norm())
        assert rel < 2e-2, (name, rel)
    mine = tr.params.clone()
    other = mine.clone()
    dist.broadcast(other, src=0)
    assert torch.equal(mine, other)
    dist.barrier()


def w_bf16_wire_exchange(rank, size):
    """FusedTrainer(grad_wire=bf16): same training curve as the fp32 wire within bf16 rounding of the exchanged gradients,
    replicas still bit-identical, through both the Python graph path and the C++ executor."""
    dev = _dev()
    from dist_tuto.pth_b200 import data as D
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    bsz = 16
    ds = D.SyntheticMNIST(n=bsz * size * 10, seed=4)
    idx = list(range(rank, len(ds), size))
    out = {}
    for wire in (torch.float32, torch.bfloat16):
        tr = FusedTrainer(bsz, lr=0.05, seed=11, device=dev, p_drop=0.0, raw_uint8=True, grad_wire=wire)
        assert tr.wire_bf16 == (wire == torch.bfloat16)
        for i in range(9):
            g = torch.Generator().manual_seed(70 + i * size + rank)
            tr.step(torch.randint(0, 255, (bsz, 1, 28, 28), generator=g, dtype=torch.uint8).pin_memory(),
                    torch.randint(0, 10, (bsz,), generator=g).pin_memory())
        tr.sync_lag(0)
        loader = D.NativeBatchLoader(D.Partition(ds, idx), bsz, seed=3, raw_uint8=True, pin_memory=True)
        done, _ = tr.run_native(loader)
        assert done == 10
        torch.cuda.synchronize()
        mine = tr.params.clone()
        other = mine.clone()
        dist.broadcast(other, src=0)
        assert torch.equal(mine, other), "replicas differ with wire %s" % wire
        out[wire] = (mine, tr.pop_loss_sum())
        del tr
    a, b = out[torch.float32], out[torch.bfloat16]
    rel = float((a[0] - b[0]).norm() / a[0].norm())
    assert rel < 6e-3, rel                       # 19 steps of lr 0.05 with gradients rounded to 8 mantissa bits
    assert abs(a[1] - b[1]) < 2e-2 * abs(a[1]), (a[1], b[1])
    dist.barrier()


def w_suite_world_rest(rank, size):
    """Second half of the one-launch suite (the 8-GPU box time is the scarce resource)."""
    import time
    t0 = time.time()
    for fn in (w_bf16_wire_exchange, w_batched_trainer, w_flag_reuse_stress, w_large_sizes_vs_nccl):
        t1 = time.time()
        fn(rank, size)
        torch.cuda.synchronize()
        dist.barrier()
        if rank == 0:
            print(f"SUITE world={size} {fn.__name__} ok in {time.time() - t1:.1f}s (total {time.time() - t0:.1f}s)", flush=True)


def w_suite_world(rank, size):
    """Every multi-GPU worker in ONE launch (process start-up dominates on an 8-GPU box: 13 launches would cost minutes)."""
    import time
    t0 = time.time()
    for fn in (w_symm_allreduce, w_average_gradients_gpu, w_fused_trainer, w_p2p_ring_gpu, w_push_exchange_equals_barrier_exchange,
               w_bf16_wire_exchange, w_batched_trainer, w_train_fused_e2e, w_train_torch_engine_gpu, w_flag_reuse_stress,
               w_large_sizes_vs_nccl):
        t1 = time.time()
        fn(rank, size)
        torch.cuda.synchronize()
        dist.barrier()
        if rank == 0:
            print(f"SUITE world={size} {fn.__name__} ok in {time.time() - t1:.1f}s (total {time.time() - t0:.1f}s)", flush=True)
