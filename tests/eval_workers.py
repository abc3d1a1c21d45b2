"""Per-rank bodies of the multi-process evaluation tests (spawned processes import them from here)."""
import torch
import torch.nn.functional as F

import dist_tuto.pth_b200 as b2
from dist_tuto.pth_b200.data import SyntheticMNIST
from dist_tuto.pth_b200.models.convnet import Net


def _gathered(obj):
    out = [None] * b2.get_world_size()
    torch.distributed.all_gather_object(out, obj)
    return out


def w_evaluate_cpu_net(rank, size):
    """evaluate(Net on CPU) over the ranks == one process evaluating the whole set, and the same dict on every rank."""
    ds = SyntheticMNIST(n=1001, seed=21)
    torch.manual_seed(5)
    net = Net()
    net.train()
    got = b2.evaluate(net, ds)
    assert net.training, "evaluate() must restore the train / eval mode"
    net.eval()
    with torch.no_grad():
        x = ((ds.images.double() / 255.0 - ds.mean) / ds.std).unsqueeze(1)
        out = net.double()(x)
        loss = float(F.nll_loss(out, ds.labels, reduction="sum"))
        correct = int((out.argmax(1) == ds.labels).sum())
    assert got["n"] == 1001 and got["correct"] == correct, (got, correct)
    assert abs(got["loss"] * 1001 - loss) <= 1e-6 * abs(loss), (got["loss"] * 1001, loss)
    assert got["accuracy"] == correct / 1001
    assert all(d == got for d in _gathered(got))
    b2.barrier()


def w_train_torch_with_eval(rank, size):
    """train(engine="torch", eval_dataset=...): one extra line per evaluated epoch, the loss history of the run without
    evaluation, the same "eval" entries on every rank."""
    ds, test = SyntheticMNIST(n=1024, seed=5), SyntheticMNIST(n=301, seed=9)
    runs = []
    for eval_ds in (None, test):
        logs = []
        cfg = b2.TrainConfig(epochs=3, dataset=ds, engine="torch", device="cpu", lr=0.1, eval_dataset=eval_ds, eval_every=2,
                             log=lambda *a: logs.append(a))
        runs.append((b2.train(rank, size, cfg), logs))
    (off, off_logs), (on, on_logs) = runs
    assert off["eval"] == [] and off["eval_seconds"] == 0.0
    assert on["loss"] == off["loss"] and len(on["loss"]) == 3
    assert [e["epoch"] for e in on["eval"]] == [1, 2]               # every 2nd epoch, and the last one
    assert all(e["n"] == 301 and 0.0 <= e["accuracy"] <= 1.0 for e in on["eval"])
    extra = [a for a in on_logs if ": test loss " in a]
    assert len(extra) == 2 and len(on_logs) == len(off_logs) + 2
    assert extra[0] == ("Rank ", rank, ", epoch ", 1, ": test loss ", on["eval"][0]["loss"], ", accuracy ",
                        on["eval"][0]["accuracy"])
    assert on_logs.index(extra[0]) == on_logs.index(off_logs[1]) + 1     # right after the epoch's loss line
    assert all(e == on["eval"] for e in _gathered(on["eval"]))
    b2.barrier()


def w_fused_evaluate_world(rank, size):
    """FusedTrainer.evaluate over the ranks == a one-process evaluation of the same parameters on the whole set."""
    from dist_tuto.pth_b200.ops.convnet_eval import convnet_evaluate
    from dist_tuto.pth_b200.ops.convnet_fused import FusedTrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    train_ds, test = SyntheticMNIST(n=128 * 4, seed=3), SyntheticMNIST(n=10007, seed=8)
    tr = FusedTrainer(128 // size, lr=0.05, seed=2, device=dev)
    for i in range(4):
        idx = torch.arange(i * 128 + rank * (128 // size), i * 128 + (rank + 1) * (128 // size))
        x, y = train_ds.gather(idx)
        tr.step(x.pin_memory(), y.pin_memory())
    got = tr.evaluate(test)
    assert got == b2.evaluate(tr, test)
    assert all(d == got for d in _gathered(got))
    torch.cuda.synchronize()
    whole = convnet_evaluate(tr.params, test.images.to(dev), test.labels.to(dev), test.mean, test.std).tolist()
    assert got["n"] == 10007 == int(whole[2]) and got["correct"] == int(whole[1]), (got, whole)
    assert abs(got["loss"] * 10007 - whole[0]) <= 1e-6 * abs(whole[0]), (got, whole)
    b2.barrier()
