"""The sharded LAMB / LARS kernels (csrc/sharded_layerwise.cu) on ONE GPU, with W emulated ranks.

``C.sharded_lamb`` / ``C.sharded_lars`` take raw per-rank pointers, so W "ranks" are W sets of buffers on one device, each
with its own gradient bucket, parameter flat, sums buffer, table, workspaces, state shards, signal pad and stream (the
``World`` harness of tests/emulated_ranks.py: the W launches go out back to back on W streams, and
``world x blocks <= SM count`` is asserted before any launch).  Every rank's parameters, state shards, ratios and gradient
bucket are compared bit for bit with tests/sharded_layerwise_model.py after each of 3 steps with fresh gradients, sentinels
sit behind every buffer, the tickets are zero after every call, and every rank writes the same ratios.  For fp32 buckets the
tensors inside one slice also equal the one-shot and two-shot all-reduce followed by ``lamb_flat`` / ``lars_flat``.
"""
import pytest
import torch

import comm_model as M
import sharded_layerwise_model as S
import sharded_sgd_model as SM
from emulated_ranks import C, SERIAL_SKIP, World, _untouched, _with_sentinel, sms  # noqa: F401

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800), SERIAL_SKIP]

CHUNK = S.CHUNK
LAMB_HP = dict(lr=2e-2, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.01)
LARS_HP = dict(lr=0.1, momentum=0.9, weight_decay=1e-4, trust_coefficient=1e-3, eps=1e-8, nesterov=True)
SUMS_SENTINEL = 12345.0


def lay(numels, n_vec_min=0, world=1, epv=4):
    """Offsets (multiples of 4) of tensors of ``numels`` elements laid out in turn, and the padded bucket's vectors."""
    offsets, o = [], 0
    for k in numels:
        offsets.append(o)
        o += (k + 3) // 4 * 4
    n_vec = max((o + epv - 1) // epv, n_vec_min)
    return offsets, list(numels), (n_vec + world - 1) // world * world


def layouts(world):
    """(name, numels, n_vec_min or 0, zero_tensors): the shapes the issue lists, at this world."""
    out = []
    for sl in (1, 511, 512, 513):                            # slices of sl vectors, one tensor with a tail spanning all
        n = world * sl * 4
        out.append((f"slices of {sl}", [max(n - 3, 1)], world * sl, ()))
    out.append(("chunk multiples +- 1, tails 1-3", [CHUNK - 1, 1, CHUNK + 1, 2, 2 * CHUNK, 3, 2 * CHUNK - 1, 7, 9], 0, ()))
    out.append(("straddle one boundary", [5] * 3 + [world * 700 + 3] + [6] * 3, 0, ()))
    if world > 1:
        out.append(("a slice of padding only", [13, 4], world * 512, ()))
    out.append(("3000 tiny tensors", [1 + i % 3 for i in range(3000)], 0, ()))
    out.append(("excluded and all-zero tensors", [300, 301, 64, 65, 1, 2000], 0, (1, 2)))
    return out


def _sums_buf(T):
    b = torch.zeros(2 * T + 2, dtype=torch.float64, device="cuda")
    b[2 * T:] = SUMS_SENTINEL
    return b


def run(C, W, kind, numels, n_vec_min, zeros, wire, max_blocks, zero_grad, seed, steps=3, against_kernels=False):
    world, epv = W.world, M.elems_per_vec(wire)
    offsets, numels, n_vec = lay(numels, n_vec_min, world, epv)
    n, T = n_vec * epv, len(numels)
    per = n // world
    adapt = [k > 3 and i % 5 != 4 for i, k in enumerate(numels)]
    hp = LAMB_HP if kind == "lamb" else LARS_HP
    gen = torch.Generator().manual_seed(seed)
    p0 = torch.randn(n, generator=gen)
    for z in zeros[:1]:                                    # an all-zero parameter tensor
        p0[offsets[z]:offsets[z] + numels[z]] = 0
    n_states = 2 if kind == "lamb" else 1
    st_full = [torch.zeros(n) for _ in range(n_states)]
    params = [_with_sentinel(p0) for _ in range(world)]
    grads = [_with_sentinel(torch.zeros(n), wire) for _ in range(world)]
    shards = [[_with_sentinel(torch.zeros(per)) for _ in range(world)] for _ in range(n_states)]
    work = [_with_sentinel(torch.zeros(per)) for _ in range(world)]
    sums = [_sums_buf(T) for _ in range(world)]
    ratios = [_with_sentinel(torch.ones(T)) for _ in range(world)]
    tabs = [C.sharded_layerwise_table(offsets, numels, adapt, n, r, world, torch.device("cuda")) for r in range(world)]
    parts = [_with_sentinel(torch.zeros(2 * tb.n_chunks)) for tb in tabs]
    tickets = [torch.zeros(T + 4, dtype=torch.int32, device="cuda") for _ in range(world)]
    gp, pp, sp = ([x.data_ptr() for x in xs] for xs in (grads, params, sums))
    blocks = SM.grid_blocks(n_vec, world, max_blocks)
    what = f"{kind} world {world} n_vec {n_vec} tensors {T} max_blocks {max_blocks} {wire} zero_grad {zero_grad}"
    inside = S.tensors_inside_one_slice(offsets, numels, n, world)
    if against_kernels:
        assert wire == torch.float32
        ut, unc = C.layerwise_table(offsets, numels, adapt, n, torch.device("cuda"))
        ref = {v: dict(p=p0.cuda(), st=[torch.zeros(n, device="cuda") for _ in range(n_states)],
                       ws=(torch.zeros(2 * unc, device="cuda"), torch.zeros(T, dtype=torch.int32, device="cuda"),
                           torch.zeros(2 * T, dtype=torch.float64, device="cuda")), r=torch.ones(T, device="cuda"))
               for v in (M.TWOSHOT, M.ONESHOT)}

    def launch(r, t):
        tb, nc = tabs[r], tabs[r].n_chunks
        if kind == "lamb":
            sc = [1 - hp["betas"][0], hp["betas"][1], 1 - hp["betas"][1], (1 - hp["betas"][1] ** t) ** 0.5, hp["eps"],
                  1 / (1 - hp["betas"][0] ** t), hp["lr"], hp["weight_decay"]]
            C.sharded_lamb(wire == torch.bfloat16, gp, pp, sp, W.sig_ptrs, shards[0][r][:per], shards[1][r][:per], tb,
                           parts[r][:2 * nc], tickets[r][:T], ratios[r][:T], n_vec, sc, 1.0 / world, zero_grad, r, world,
                           max_blocks)
        else:
            C.sharded_lars(wire == torch.bfloat16, gp, pp, sp, W.sig_ptrs, shards[0][r][:per], work[r][:per], tb,
                           parts[r][:2 * nc], tickets[r][:T], ratios[r][:T], n_vec, hp["lr"], hp["momentum"],
                           hp["weight_decay"], hp["trust_coefficient"], hp["eps"], hp["nesterov"], 1.0 / world, zero_grad, r,
                           world, max_blocks)

    p_cur = p0
    for it in range(steps):
        gs = M.make_inputs(world, n, wire, 7919 * seed + it, specials=False)
        for z in zeros[1:]:                                # an all-zero gradient tensor
            for x in gs:
                x[offsets[z]:offsets[z] + numels[z]] = 0
        for r in range(world):
            if zero_grad and it > 0:
                assert not bool(grads[r][:n].any()), f"{what} step {it}: rank {r}'s bucket was not left zeroed"
            grads[r][:n].copy_(gs[r])
        if against_kernels:
            for v in (M.TWOSHOT, M.ONESHOT):
                bufs = [g[:n].clone() for g in grads]
                bptr = [b.data_ptr() for b in bufs]
                W.launch(M.grid_blocks(v, n_vec, world, max_blocks),
                         lambda r: C.allreduce(v, False, bptr, W.sig_ptrs, 0, None, None, n_vec, 1.0 / world, r, world,
                                               max_blocks))
                R = ref[v]
                if kind == "lamb":
                    b1, b2 = hp["betas"]
                    t = it + 1
                    C.lamb_flat(R["p"], R["st"][0], R["st"][1], bufs[0], ut, unc, *R["ws"], R["r"],
                                [1 - b1, b2, 1 - b2, (1 - b2 ** t) ** 0.5, hp["eps"], 1 / (1 - b1 ** t), hp["lr"],
                                 hp["weight_decay"]], False)
                else:
                    C.lars_flat(R["p"], R["st"][0], bufs[0], ut, unc, *R["ws"], R["r"], hp["lr"], hp["momentum"],
                                hp["weight_decay"], hp["trust_coefficient"], hp["eps"], hp["nesterov"], False)
        W.launch(blocks, lambda r: launch(r, it + 1))
        want = S.step(kind, gs, p_cur, st_full, offsets, numels, adapt, hp, 1.0 / world, t=it + 1, zero_grad=zero_grad)
        tag = f"{what} step {it}"
        M.assert_bits_equal(f"{tag}: params", [p[:n] for p in params], want["params"], 4)
        for k in range(n_states):
            M.assert_bits_equal(f"{tag}: state {k}", [s[:per] for s in shards[k]], want["shards"][k], 4)
        M.assert_bits_equal(f"{tag}: gradient buckets", [g[:n] for g in grads], want["grads"], epv)
        want_r = torch.tensor(want["ratios"][0], dtype=torch.float32)
        for r in range(world):
            assert torch.equal(ratios[r][:T].cpu(), want_r), f"{tag}: rank {r}'s ratios"
            assert not bool(tickets[r].any()), f"{tag}: rank {r}'s tickets are not zero"
            assert _untouched(params[r][n:]) and _untouched(grads[r][n:]) and _untouched(ratios[r][T:]), (
                f"{tag}: rank {r} wrote behind its parameters, gradients or ratios")
            assert all(_untouched(s[r][per:]) for s in shards) and _untouched(work[r][per:]), f"{tag}: rank {r}: state shards"
            assert _untouched(parts[r][2 * tabs[r].n_chunks:]), f"{tag}: rank {r}: partials"
            assert bool((sums[r][2 * T:] == SUMS_SENTINEL).all()), f"{tag}: rank {r}: sums"
            if kind == "lars":
                inner = [(o - r * per, o - r * per + k) for o, k in zip(offsets, numels)]
                wk = work[r][:per].cpu()
                for a, b in inner:
                    a, b = max(a, 0), min(b, per)
                    if a < b:
                        assert torch.equal(wk[a:b], want["g"][r * per + a:r * per + b]), f"{tag}: rank {r}: gradient workspace"
        if zeros:                       # all-zero parameters (before the first update), and LARS on all-zero gradients
            assert it > 0 or want["ratios"][0][zeros[0]] == 1.0
            assert kind == "lamb" or want["ratios"][0][zeros[1]] == 1.0
        if against_kernels:
            for v in (M.TWOSHOT, M.ONESHOT):
                R = ref[v]
                rp = R["p"].cpu()
                for i in inside:
                    s = slice(offsets[i], offsets[i] + numels[i])
                    name = f"{tag}: {M.VARIANT_NAMES[v]} all-reduce + {kind}_flat, tensor {i}"
                    assert torch.equal(params[0][s].cpu(), rp[s]), name + ": params"
                    assert float(ratios[0][i]) == float(R["r"][i]), name + ": ratio"
                    for k in range(n_states):
                        assert torch.equal(want["states"][k][s], R["st"][k].cpu()[s]), name + f": state {k}"
        p_cur, st_full = want["params"][0], want["states"]


def cases(world, sms):
    """(layout, max_blocks, wire, zero_grad): every layout at max_blocks 1, 3 and SMs // world in turn, fp32 and bf16 and
    zero_grad rotating."""
    out = []
    for i, lo in enumerate(layouts(world)):
        mb = [1, 3, sms // world][i % 3]
        out.append((lo, mb, torch.bfloat16 if i % 2 else torch.float32, (i // 2) % 2 == 0))
    return out


@pytest.mark.parametrize("kind", ["lamb", "lars"])
@pytest.mark.parametrize("world", range(1, 9))
def test_sharded_layerwise_matches_the_model_bit_for_bit(C, sms, kind, world):
    for k, ((name, numels, nvm, zeros), mb, wire, zero_grad) in enumerate(cases(world, sms)):
        run(C, World(world, sms), kind, numels, nvm, zeros, wire, mb, zero_grad, seed=100 * world + k)


@pytest.mark.parametrize("kind", ["lamb", "lars"])
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_fp32_tensors_inside_one_slice_equal_the_allreduce_and_the_unsharded_kernels(C, sms, kind, world):
    numels = [5, 3, world * 3000 + 1, CHUNK + 1, 9, 2 * CHUNK - 1, 130, 7]
    run(C, World(world, sms), kind, numels, 0, (), torch.float32, sms // world, world % 2 == 0, seed=7 * world,
        against_kernels=True)


def test_refusals(C):
    pad = torch.zeros(M.SIGNAL_WORDS, dtype=torch.int32, device="cuda")
    g, p, m, v = (torch.zeros(64, device="cuda") for _ in range(4))
    sums = torch.zeros(8, dtype=torch.float64, device="cuda")
    dev = torch.device("cuda")
    tabs = {(r, w): C.sharded_layerwise_table([0], [64], [True], 64, r, w, dev) for r, w in ((0, 2), (1, 2), (0, 1))}
    one = lambda t, k: [t.data_ptr()] * k          # noqa: E731

    def args(k, nv, tb):
        return (one(g, k), one(p, k), one(sums, k), one(pad, k), m, v, tb, torch.zeros(2 * tb.n_chunks, device="cuda"),
                torch.zeros(1, dtype=torch.int32, device="cuda"), torch.ones(1, device="cuda"), nv)

    sc = [0.1, 0.999, 0.001, 0.03, 1e-6, 10.0, 1e-3, 0.01]
    assert (tabs[0, 2].rank, tabs[0, 2].world, tabs[0, 2].n, tabs[0, 2].n_chunks) == (0, 2, 64, 1)
    assert tabs[1, 2].n_chunks == 1
    assert C.sharded_layerwise_table([0], [8], [True], 64, 1, 2, dev).n_chunks == 0        # a slice of padding only
    with pytest.raises(RuntimeError, match="multiple of world"):
        C.sharded_lamb(False, *args(3, 16, tabs[0, 2]), sc, 1.0, True, 0, 3)
    with pytest.raises(RuntimeError, match="world"):
        C.sharded_lamb(False, *args(9, 18, tabs[0, 2]), sc, 1.0, True, 0, 9)
    with pytest.raises(RuntimeError, match="scalars"):
        C.sharded_lamb(False, *args(2, 16, tabs[0, 2]), sc[:7], 1.0, True, 0, 2)
    with pytest.raises(RuntimeError, match="nesterov"):
        C.sharded_lars(False, *args(2, 16, tabs[0, 2]), 0.1, 0.0, 0.0, 1e-3, 1e-8, True, 1.0, True, 0, 2)
    # a table built for another rank, world size or bucket size would index the state shards outside the slice
    for (r, w), tb in (((1, 2), tabs[0, 2]), ((0, 2), tabs[1, 2]), ((0, 2), tabs[0, 1])):
        with pytest.raises(RuntimeError, match="table was built for"):
            C.sharded_lamb(False, *args(w, 16, tb), sc, 1.0, True, r, w)
        with pytest.raises(RuntimeError, match="table was built for"):
            C.sharded_lars(False, *args(w, 16, tb), 0.1, 0.9, 0.0, 1e-3, 1e-8, False, 1.0, True, r, w)
    with pytest.raises(RuntimeError, match="table was built for"):
        C.sharded_lamb(True, *args(2, 16, tabs[0, 2]), sc, 1.0, True, 0, 2)      # bf16: 128 elements, not 64
    with pytest.raises(RuntimeError, match="slices"):
        C.sharded_layerwise_table([0], [60], [True], 60, 0, 8, dev)
