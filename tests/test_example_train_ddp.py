"""examples/train_ddp.py (DistributedDataParallel + FlatSGD on a generic conv model) as a real process on CPU / gloo: the
sharded optimizer prints the same final loss as the unsharded one and holds half the momentum per rank."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.timeout(300)


def run(*args):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), CUDA_VISIBLE_DEVICES="")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "examples", "train_ddp.py"), *args], capture_output=True, text=True,
                       timeout=280, env=env, cwd=ROOT)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = re.findall(r"Rank (\d), step 6: loss ([0-9.]+) \(mean over ranks ([0-9.]+)\), momentum elements on this rank (\d+)",
                       p.stdout)
    assert sorted(r for r, *_ in lines) == ["0", "1"], p.stdout
    return {int(r): (loss, mean, int(mom)) for r, loss, mean, mom in lines}


def test_train_ddp_with_and_without_the_sharded_optimizer_prints_the_same_loss():
    plain = run("--size", "2", "--steps", "6")
    sharded = run("--size", "2", "--steps", "6", "--sharded-optimizer")
    for r in (0, 1):
        assert plain[r][:2] == sharded[r][:2]                        # the printed losses, digit for digit
        assert 0.5 < float(plain[r][0]) < 5.0
        assert plain[r][2] // 2 <= sharded[r][2] <= plain[r][2] // 2 + 64   # half the momentum (+ padding) per rank
