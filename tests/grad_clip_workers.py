"""Multi-process workers of tests/test_grad_clip.py (dist_tuto.pth_b200.launch runs them, one process per rank)."""
import os

import torch
import torch.distributed as dist

import dist_tuto.pth_b200 as b2


class _Stop(Exception):
    pass


def w_torch_engine_clip_resume(rank, size):
    """train(engine="torch", max_grad_norm=...) at world 2 on gloo: the replicas stay equal, every epoch reports a norm,
    and a run stopped after its first in-progress checkpoint and resumed from it ends bit-equal to the uninterrupted run.
    Dropout is off and each epoch's shuffle is seeded by the epoch index (see tests/lr_workers.py)."""
    from dist_tuto.pth_b200.data import BatchLoader, SyntheticMNIST
    it = BatchLoader.__iter__

    def epoch_seeded_iter(self):
        self._gen.manual_seed(1000 + self._epoch)
        self._epoch += 1
        return it(self)
    BatchLoader._epoch = 0
    BatchLoader.__iter__ = epoch_seeded_iter
    ckdir = os.environ["B2_CLIP_TEST_DIR"]
    ds = SyntheticMNIST(n=1024, seed=5)

    def cfg(**kw):
        return b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0, max_grad_norm=0.05,
                              weight_decay=1e-3, nesterov=True, log=kw.pop("log", lambda *a: None), **kw)

    whole = b2.train(rank, size, cfg())
    assert whole["steps"] == 24 and len(whole["grad_norm"]) == 3
    assert all(n > 0.05 for n in whole["grad_norm"]), whole["grad_norm"]     # the clip was in force
    flat = torch.cat([p.detach().reshape(-1) for p in whole["model"].parameters()])
    peers = [torch.empty_like(flat) for _ in range(size)]
    dist.all_gather(peers, flat)
    assert all(torch.equal(peers[0], q) for q in peers[1:]), "replicas differ"
    plain = b2.train(rank, size, b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0,
                                                weight_decay=1e-3, nesterov=True, log=lambda *a: None))
    assert "grad_norm" not in plain
    assert any(not torch.equal(a, b) for a, b in zip(whole["model"].parameters(), plain["model"].parameters()))

    ck = os.path.join(ckdir, "run.pt")

    def stop_in_epoch_1(*a):
        if a[:4] == ("Rank ", rank, ", epoch ", 1):
            raise _Stop()
    try:
        b2.train(rank, size, cfg(checkpoint=ck, checkpoint_every=1, log=stop_in_epoch_1))
        raise AssertionError("the run was not stopped")
    except _Stop:
        pass
    b2.barrier()
    blob = torch.load(ck, map_location="cpu")
    assert blob["in_progress"] and blob["epoch"] == 1 and blob["optim"]["max_grad_norm"] == 0.05
    resumed = b2.train(rank, size, cfg(resume=ck))
    assert resumed["steps"] == 16 and resumed["grad_norm"] == whole["grad_norm"][1:]
    for (n, a), (_, b) in zip(whole["model"].named_parameters(), resumed["model"].named_parameters()):
        assert torch.equal(a.detach(), b.detach()), n
    b2.barrier()


def w_two_gpu_clip(rank, size):
    """Two GPUs, push exchange with an fp32 and a bf16 wire, clipping in force: the replicas stay bit-identical and
    report the same norm."""
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    for wire in (torch.float32, torch.bfloat16):
        tr = FusedTrainer(32, lr=0.05, seed=4, device=dev, grad_wire=wire, max_grad_norm=0.1, weight_decay=1e-3)
        assert tr.inbox_handle is not None
        for k in range(8):
            g = torch.Generator().manual_seed(50 + k * size + rank)
            x, y = torch.randn(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).pin_memory()
            tr.step(x, y)
        norm = torch.tensor([tr.grad_norm()], device=dev)
        tr.sync_lag(0)
        torch.cuda.synchronize()
        both = [torch.empty_like(tr.params) for _ in range(size)]
        dist.all_gather(both, tr.params)
        norms = [torch.empty_like(norm) for _ in range(size)]
        dist.all_gather(norms, norm)
        assert torch.equal(both[0], both[1]) and torch.equal(norms[0], norms[1]), wire
        assert float(norm) > 0.1
