"""Per-rank bodies of the multi-process lr-schedule tests (spawned processes import them from here)."""
import os

import torch

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.data import SyntheticMNIST


class _Stop(Exception):
    pass


def w_torch_engine_schedule_resume(rank, size):
    """train(engine="torch") with a warmup + multistep schedule: a run stopped after its first in-progress checkpoint
    (mid-warmup) and resumed from it ends with the parameters of the uninterrupted run, bit for bit.  Dropout is off:
    the torch engine does not checkpoint the host RNG that draws its masks.  The CPU loader draws each epoch's shuffle from
    one running generator; here it is seeded by the epoch index instead, as the native loader does, so that a resumed
    run sees the batches of the uninterrupted one."""
    from dist_tuto.pth_b200.data import BatchLoader
    it = BatchLoader.__iter__

    def epoch_seeded_iter(self):
        self._gen.manual_seed(1000 + self._epoch)
        self._epoch += 1
        return it(self)
    BatchLoader._epoch = 0                  # train() sets it to the first epoch of a resumed run
    BatchLoader.__iter__ = epoch_seeded_iter
    ckdir = os.environ["B2_LR_TEST_DIR"]
    ds = SyntheticMNIST(n=1024, seed=5)
    # 8 steps per epoch and rank: the warmup ends at step 12, the milestone is at step 18
    sched = b2.LRSchedule(warmup_steps=1.5, decay="multistep", milestones=[2.25], gamma=0.5, unit="epoch")

    def cfg(**kw):
        return b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0, lr_schedule=sched,
                              log=lambda *a: None, **kw)

    whole = b2.train(rank, size, cfg())
    assert whole["steps"] == 24
    r = sched.resolve(8)
    assert whole["lr"] == [r.lr_at(0.05, 7), r.lr_at(0.05, 15), r.lr_at(0.05, 23)]
    assert whole["lr"][0] < whole["lr"][1] > whole["lr"][2]

    ck = os.path.join(ckdir, "run.pt")

    def stop_in_epoch_1(*a):
        if a[:4] == ("Rank ", rank, ", epoch ", 1):
            raise _Stop()
    try:
        b2.train(rank, size, b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.05, p_drop=0.0,
                                            lr_schedule=sched, checkpoint=ck, checkpoint_every=1, log=stop_in_epoch_1))
        raise AssertionError("the run was not stopped")
    except _Stop:
        pass
    b2.barrier()
    blob = torch.load(ck, map_location="cpu")
    assert blob["in_progress"] and blob["epoch"] == 1 and blob["steps"] == 8 and blob["optim"]["steps"] == 8
    resumed = b2.train(rank, size, cfg(resume=ck))
    assert resumed["steps"] == 16 and resumed["lr"] == whole["lr"][1:]
    for (n, a), (_, b) in zip(whole["model"].named_parameters(), resumed["model"].named_parameters()):
        assert torch.equal(a.detach(), b.detach()), n
    b2.barrier()


def w_two_gpu_schedule(rank, size):
    """Two GPUs, push exchange with an fp32 and a bf16 wire: every update applies lr_at(step) and the replicas stay
    bit-identical."""
    import torch.distributed as dist
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    sched = b2.LRSchedule(warmup_steps=5, decay="multistep", milestones=[9], gamma=0.3)
    for wire in (torch.float32, torch.bfloat16):
        tr = FusedTrainer(32, lr=0.05, seed=4, device=dev, grad_wire=wire, lr_schedule=sched)
        assert tr.inbox_handle is not None
        for k in range(12):
            g = torch.Generator().manual_seed(50 + k * size + rank)
            x, y = torch.randn(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).pin_memory()
            tr.sync_lag(0)
            torch.cuda.synchronize()
            p_old = tr.params.clone()
            tr.step(x, y)
            tr.sync_lag(0)
            torch.cuda.synchronize()
            m = tr.momentum
            sel = m.abs() > m.abs().median()
            d, mm = (p_old - tr.params)[sel].double(), m[sel].double()
            got, want = float((d * mm).sum() / (mm * mm).sum()), sched.lr_at(0.05, k)
            assert abs(got - want) <= 1e-4 * want, (wire, k, got, want)
            other = tr.params.clone()
            dist.broadcast(other, src=0)
            assert torch.equal(other, tr.params), (wire, k)
    dist.barrier()
