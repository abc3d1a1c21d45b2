"""The capturable instances of the sharded exchange kernel at emulated worlds 1..8 on one GPU (the harness of
tests/emulated_ranks.py): fed the same scalars they equal the existing instances bit for bit, and W graphs of
each rank's exchange plus step-counter advance, replayed concurrently for 50 steps across a schedule change, equal the
existing instances launched eagerly with the model's scalars (tests/capturable_model.py) at every step."""
import pytest
import torch

import capturable_model as CM
from dist_tuto.pth_b200.ops.optim import LRSchedule, schedule_tuple
from emulated_ranks import C, World, _untouched, _with_sentinel  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

MU, BETAS, EPS = 0.9, (0.8, 0.95), 1e-6
LRS, WDS = [0.05, 0.01], [0.02, 0.0]
SCHED = LRSchedule(warmup_steps=5, decay="multistep", milestones=(30,), gamma=0.25)
STEPS = 50


def _ranks(C, world, kind, wire, n_vec, grouped, seed):
    """Fresh world, per-rank parameters, state shards, gradients (with sentinels), group maps and device scalar state."""
    epv = 8 if wire == torch.bfloat16 else 4
    n, per = n_vec * epv, n_vec * epv // world
    gen = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=gen)
    s0 = [torch.randn(per, generator=gen).abs() for _ in range(2)]
    g0 = [torch.randn(n, generator=gen) for _ in range(world)]
    gmap = torch.randint(0, len(LRS), (n // 4,), generator=gen, dtype=torch.uint8)
    lay = C.flat_scalars_layout()
    R = dict(n=n, per=per, bf16=wire == torch.bfloat16, lay=lay,
             params=[_with_sentinel(p0) for _ in range(world)], st=[[_with_sentinel(s) for s in s0] for _ in range(world)],
             grads=[_with_sentinel(g, wire) for g in g0],
             maps=[gmap[r * per // 4:(r + 1) * per // 4].cuda() if grouped else None for r in range(world)],
             dev=[(torch.zeros(lay["table_bytes"], dtype=torch.uint8, device="cuda"), torch.zeros(1, dtype=torch.int64, device="cuda"),
                   torch.zeros(lay["block_bytes"], dtype=torch.uint8, device="cuda")) for _ in range(world)])
    lrs, wds = (LRS, WDS) if grouped else (LRS[:1], WDS[:1])
    for t, c, b in R["dev"]:
        C.flat_scalars_sync(t, c, b, lrs, wds, *BETAS, EPS, schedule_tuple(SCHED), steps=0)
    return R


def _cap(C, R, W, kind, n_vec, r, max_blocks):
    gp, pp = [x.data_ptr() for x in R["grads"]], [x.data_ptr() for x in R["params"]]
    st, blk = R["st"][r], R["dev"][r][2]
    if kind == "adamw":
        C.sharded_adamw_cap(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], st[1][:R["per"]], R["maps"][r], blk, n_vec,
                            1.0 / W.world, False, r, W.world, max_blocks)
    else:
        C.sharded_sgd_cap(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], R["maps"][r], blk, n_vec, MU, kind == "sgd_nesterov",
                          1.0 / W.world, False, r, W.world, max_blocks)


def _ref(C, R, W, kind, n_vec, r, max_blocks, s, grouped):
    """The existing instance of rank r with the model's scalars of the update at counter s."""
    gp, pp = [x.data_ptr() for x in R["grads"]], [x.data_ptr() for x in R["params"]]
    st = R["st"][r]
    blocks = [CM.block(SCHED.lr_at(lr, s), wd, BETAS, EPS, s) for lr, wd in zip(LRS, WDS)]
    if kind == "adamw":
        if grouped:
            C.sharded_adamw_grouped(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], st[1][:R["per"]], R["maps"][r], n_vec,
                                    blocks[-1]["adamw"], [b["decay"] for b in blocks], [b["step_size"] for b in blocks],
                                    1.0 / W.world, False, r, W.world, max_blocks)
        else:
            C.sharded_adamw(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], st[1][:R["per"]], n_vec, blocks[0]["adamw"],
                            1.0 / W.world, False, r, W.world, max_blocks)
    elif grouped:
        C.sharded_sgd_grouped(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], R["maps"][r], n_vec, [b["lr"] for b in blocks],
                              [b["wd"] for b in blocks], MU, kind == "sgd_nesterov", 1.0 / W.world, False, r, W.world, max_blocks)
    else:
        C.sharded_sgd(R["bf16"], gp, pp, W.sig_ptrs, st[0][:R["per"]], n_vec, blocks[0]["lr"], MU, blocks[0]["wd"],
                      kind == "sgd_nesterov", 1.0 / W.world, False, r, W.world, max_blocks)


def _same(R, Q, world):
    ib = torch.int16 if R["bf16"] else torch.int32
    for r in range(world):
        assert torch.equal(R["params"][r].view(torch.int32), Q["params"][r].view(torch.int32)), f"params of rank {r}"
        for a, b in zip(R["st"][r], Q["st"][r]):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"state of rank {r}"
        assert torch.equal(R["grads"][r].view(ib), Q["grads"][r].view(ib))
        assert _untouched(R["params"][r][R["n"]:]) and all(_untouched(s[R["per"]:]) for s in R["st"][r])
    for r in range(1, world):
        assert torch.equal(R["params"][r][:R["n"]], R["params"][0][:R["n"]]), "replicas differ"


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("kind", ["sgd", "sgd_nesterov", "adamw"])
def test_graph_replays_equal_the_existing_instances(C, world, kind):
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for wire in (torch.float32, torch.bfloat16):
        for grouped in (False, True):
            n_vec, max_blocks = world * 1031, max(1, min(2, sms // world))
            blocks = min(max_blocks, max(1, ((n_vec // world + 511) // 512 + 1) // 2))
            what = f"{kind} world {world} {wire} grouped {grouped}"
            # one eager step of each: the same scalars, the same bits
            Wa, Wb = World(world, sms), World(world, sms)
            A = _ranks(C, world, kind, wire, n_vec, grouped, world)
            B = _ranks(C, world, kind, wire, n_vec, grouped, world)
            Wa.launch(blocks, lambda r: _cap(C, A, Wa, kind, n_vec, r, max_blocks))
            Wb.launch(blocks, lambda r: _ref(C, B, Wb, kind, n_vec, r, max_blocks, 0, grouped))
            _same(A, B, world)
            # every rank's exchange + advance captured, the W graphs replayed concurrently
            graphs = []
            for r in range(world):
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g, stream=Wa.streams[r]):
                    _cap(C, A, Wa, kind, n_vec, r, max_blocks)
                    C.flat_scalars_advance(*A["dev"][r])
                graphs.append(g)
            for t, c, b in A["dev"]:                   # the eager step above did not advance: counter 1 from here
                C.flat_scalars_advance(t, c, b)
            for s in range(1, STEPS + 1):
                Wa.launch(blocks, lambda r: graphs[r].replay())
                Wb.launch(blocks, lambda r: _ref(C, B, Wb, kind, n_vec, r, max_blocks, s, grouped))
                try:
                    _same(A, B, world)
                except AssertionError as e:
                    raise AssertionError(f"{what} replay {s}: {e}") from None
            assert all(int(c.item()) == STEPS + 1 for _, c, _ in A["dev"])
