"""The tutorial's MNIST ConvNet (layer L5).

Parity: ``Net`` of train_dist.py:53-71 -- conv1 1->10 k5 -> maxpool2 -> relu;
conv2 10->20 k5 -> Dropout2d -> maxpool2 -> relu; flatten 320; fc1 320->50 +
relu; dropout; fc2 50->10; log_softmax(dim=1).  NOTE the order is
conv -> pool -> relu.  21,840 parameters in 8 tensors, registered in the same
order and under the same names as the reference so state_dicts interchange.

Two execution paths share one set of parameters:
  * ``forward`` -- plain torch ops (CPU, and the oracle for kernel tests);
  * the fused sm_90a training step in ``ops/convnet_fused.py`` which reads the
    parameters from a flat fp32 buffer (see ``FlatParams``) and runs
    forward + loss + backward in one kernel.
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ["Net", "PARAM_SHAPES", "PARAM_NUMEL", "param_offsets"]

# (name, shape) in ``model.parameters()`` order (train_dist.py:58-62)
PARAM_SHAPES: List[Tuple[str, Tuple[int, ...]]] = [
    ("conv1.weight", (10, 1, 5, 5)), ("conv1.bias", (10,)),
    ("conv2.weight", (20, 10, 5, 5)), ("conv2.bias", (20,)),
    ("fc1.weight", (50, 320)), ("fc1.bias", (50,)),
    ("fc2.weight", (10, 50)), ("fc2.bias", (10,)),
]


def _numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


PARAM_NUMEL = sum(_numel(s) for _, s in PARAM_SHAPES)  # 21840


def param_offsets(align: int = 1):
    """Element offsets of each parameter inside the flat buffer."""
    offs, o = {}, 0
    for name, shape in PARAM_SHAPES:
        offs[name] = o
        o += (_numel(shape) + align - 1) // align * align
    return offs, o


class Net(nn.Module):
    """MNIST ConvNet, same architecture / init / parameter order as the reference."""

    def __init__(self, p_drop: float = 0.5):
        super().__init__()
        self.conv1 = nn.Conv2d(1, 10, kernel_size=5)
        self.conv2 = nn.Conv2d(10, 20, kernel_size=5)
        self.conv2_drop = nn.Dropout2d(p_drop)
        self.fc1 = nn.Linear(320, 50)
        self.fc2 = nn.Linear(50, 10)
        self.p_drop = p_drop

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        x = F.relu(F.max_pool2d(self.conv1(x), 2))
        x = F.relu(F.max_pool2d(self.conv2_drop(self.conv2(x)), 2))
        x = x.reshape(-1, 320)
        x = F.relu(self.fc1(x))
        x = F.dropout(x, p=self.p_drop, training=self.training)
        x = self.fc2(x)
        return F.log_softmax(x, dim=1)
