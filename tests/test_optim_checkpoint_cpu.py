"""The checkpoint forms of every flat optimizer on CPU, no process group: ``state_dict`` round-trips bit for bit, and
``load_state_dict`` / ``load_named_state`` refuse a malformed state with ``ValueError`` before they write anything -- a bad
option, a shard of another world, buffers of other sizes, a per-name entry without one of its states."""
import pytest
import torch
import torch.nn as nn

from dist_tuto.pth_b200.ops.optim import FlatAdafactor, FlatAdamW, FlatLAMB, FlatLARS, FlatRMSprop, FlatSGD

# optimizer, constructor options of the one that loads and of the one that saved, state flats, option attributes, and one
# option value its constructor refuses
CASES = {
    "sgd": (FlatSGD, dict(lr=0.05, momentum=0.5, weight_decay=0.01), dict(lr=0.2, momentum=0.9, nesterov=True),
            ["momentum_flats"], ["lr", "momentum", "weight_decay", "nesterov"], dict(weight_decay=-1.0)),
    "adamw": (FlatAdamW, dict(lr=0.01), dict(lr=0.03, betas=(0.8, 0.99), eps=1e-6, weight_decay=0.1),
              ["exp_avg_flats", "exp_avg_sq_flats"], ["lr", "betas", "eps", "weight_decay"], dict(betas=(0.9, 1.5))),
    "rmsprop": (FlatRMSprop, dict(lr=0.01, momentum=0.5, centered=True), dict(lr=0.02, alpha=0.9, momentum=0.9, centered=True),
                ["square_avg_flats", "momentum_buffer_flats", "grad_avg_flats"],
                ["lr", "alpha", "eps", "weight_decay", "momentum", "centered"], dict(alpha=-0.5)),
    "adafactor": (FlatAdafactor, dict(lr=0.01), dict(lr=0.02, beta2_decay=-0.5, eps=(1e-30, 1e-3), d=2.0),
                  ["state_flats"], ["lr", "beta2_decay", "eps", "d", "weight_decay", "eps1", "eps2"], dict(d=0.5)),
    "lamb": (FlatLAMB, dict(lr=0.01), dict(lr=0.03, betas=(0.8, 0.99), weight_decay=0.1),
             ["exp_avg_flats", "exp_avg_sq_flats"], ["lr", "betas", "eps", "weight_decay"], dict(betas=(0.9, 1.5))),
    "lars": (FlatLARS, dict(lr=0.05), dict(lr=0.2, momentum=0.5, trust_coefficient=0.01, eps=1e-6),
             ["momentum_flats"], ["lr", "momentum", "weight_decay", "nesterov", "trust_coefficient", "eps"],
             dict(weight_decay=-1.0)),
}
NAMED = ["adamw", "rmsprop", "adafactor", "lamb"]          # the optimizers with torch's per-name state (named_state)


def _trained(case: str, saved: bool, steps: int):
    cls, mine, theirs = CASES[case][:3]
    torch.manual_seed(0)
    net = nn.Sequential(nn.Linear(5, 4), nn.Tanh(), nn.Linear(4, 3))
    opt = cls(net, max_grad_norm=1.0 if saved else None, **(theirs if saved else mine))
    for _ in range(steps):
        net(torch.randn(6, 5)).square().sum().backward()
        opt.step()
    return net, opt


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.reshape(-1).view(torch.int32)


def _snapshot(case: str, opt) -> tuple:
    flats, options = CASES[case][3], CASES[case][4]
    return ([_bits(f).clone() for name in flats for f in getattr(opt, name)],
            [(name, getattr(opt, name)) for name in options + ["max_grad_norm", "steps"]])


def _assert_same(a: tuple, b: tuple) -> None:
    assert len(a[0]) == len(b[0]) and all(torch.equal(x, y) for x, y in zip(a[0], b[0]))
    assert a[1] == b[1] and [type(v) for _, v in a[1]] == [type(v) for _, v in b[1]]


def _refused(case: str, load, *args, match=None) -> None:
    """``load(*args)`` raises ValueError and leaves every buffer, option and ``steps`` of the loading optimizer as it was."""
    opt = load.__self__
    before = _snapshot(case, opt)
    with pytest.raises(ValueError, match=match):
        load(*args)
    _assert_same(_snapshot(case, opt), before)


@pytest.mark.parametrize("case", list(CASES))
def test_state_dict_round_trip_is_bit_exact(case):
    _, saved = _trained(case, True, 3)
    _, opt = _trained(case, False, 2)
    opt.load_state_dict(saved.state_dict())
    _assert_same(_snapshot(case, opt), _snapshot(case, saved))
    assert opt.steps == 3 and opt.max_grad_norm == 1.0


@pytest.mark.parametrize("case", list(CASES))
def test_a_refused_option_writes_nothing(case):
    _, saved = _trained(case, True, 3)
    _, opt = _trained(case, False, 2)
    _refused(case, opt.load_state_dict, dict(saved.state_dict(), **CASES[case][5]))


def test_sgd_refuses_nesterov_without_momentum_as_its_constructor_does():
    _, saved = _trained("sgd", True, 3)
    _, opt = _trained("sgd", False, 2)
    with pytest.raises(ValueError, match="nesterov"):
        FlatSGD(nn.Linear(2, 2), momentum=0.0, nesterov=True)
    _refused("sgd", opt.load_state_dict, dict(saved.state_dict(), momentum=0.0, nesterov=True))


@pytest.mark.parametrize("case", list(CASES))
def test_a_shard_of_another_world_writes_nothing(case):
    _, saved = _trained(case, True, 3)
    _, opt = _trained(case, False, 2)
    _refused(case, opt.load_state_dict, dict(saved.state_dict(), sharded=True, world=2, rank=1))


@pytest.mark.parametrize("case", list(CASES))
def test_buffers_of_another_size_write_nothing(case):
    _, saved = _trained(case, True, 3)
    _, opt = _trained(case, False, 2)
    sd = saved.state_dict()
    key = [k for k, v in sd.items() if isinstance(v, list) and v][-1]          # the last state the state_dict holds
    for buffers in (sd[key][:-1] + [sd[key][-1][:-1]], sd[key] + [sd[key][-1]]):     # one element short, one bucket more
        _refused(case, opt.load_state_dict, dict(sd, **{key: buffers}), match="other sizes")


@pytest.mark.parametrize("case", NAMED)
def test_a_named_entry_without_a_state_writes_nothing(case):
    saved_net, saved = _trained(case, True, 3)
    net, opt = _trained(case, False, 2)
    named = saved.named_state(saved_net)
    last = list(named)[-2]                                  # the last weight matrix: every state it has is written last
    named[last] = {k: v for k, v in named[last].items() if k != list(named[last])[-1]}
    _refused(case, opt.load_named_state, net, named)
