"""ResNet-18 (BASELINE.json config #3: "ResNet-18 bf16 on 8 GPUs, bucketed fused allreduce").

The reference repo has no second model; BASELINE.json adds ResNet-18 as the *larger-gradient* workload for
the data-parallel engine: 11,689,512 parameters in 62 tensors (44.6 MB fp32 / 22.3 MB bf16 per step),
which exercises the two-shot / NVLS all-reduce variants and the bucket/overlap machinery that the 87 KB
ConvNet gradient never reaches.

Architecture = the standard 18-layer residual network (7x7/2 stem, 4 stages of 2 BasicBlocks, 64..512
channels, global average pool, linear classifier), parameter names compatible with torchvision's
``resnet18`` so state_dicts interchange.  Convolutions/batch-norm run on the library kernels (cuDNN) in
channels_last bf16; the classifier can run on our wgmma GEMM (``use_tc_fc=True``, inference/forward);
gradient communication is entirely ours (``parallel.ddp.DistributedDataParallel``).
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

__all__ = ["ResNet18", "BasicBlock"]


class BasicBlock(nn.Module):
    """conv3x3-BN-ReLU-conv3x3-BN + identity / 1x1 downsample (torchvision parameter names)."""
    expansion = 1

    def __init__(self, cin: int, cout: int, stride: int = 1):
        super().__init__()
        self.conv1 = nn.Conv2d(cin, cout, 3, stride, 1, bias=False)
        self.bn1 = nn.BatchNorm2d(cout)
        self.conv2 = nn.Conv2d(cout, cout, 3, 1, 1, bias=False)
        self.bn2 = nn.BatchNorm2d(cout)
        self.downsample = None
        if stride != 1 or cin != cout:
            self.downsample = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.BatchNorm2d(cout))

    def forward(self, x):
        idt = x if self.downsample is None else self.downsample(x)
        out = F.relu(self.bn1(self.conv1(x)), inplace=True)
        out = self.bn2(self.conv2(out))
        return F.relu(out + idt, inplace=True)


class ResNet18(nn.Module):
    """The larger-gradient model of BASELINE config #3 (11,689,512 parameters at 1000 classes; state_dict keys match
    torchvision's ``resnet18``).  Only its gradients matter here: 45 MB in ~60 tensors exercise the bucketed, overlapped
    all-reduce.  ``use_tc_fc`` routes the inference-time classifier through the wgmma GEMM."""

    def __init__(self, num_classes: int = 1000, in_channels: int = 3, use_tc_fc: bool = False):
        super().__init__()
        self.conv1 = nn.Conv2d(in_channels, 64, 7, 2, 3, bias=False)
        self.bn1 = nn.BatchNorm2d(64)
        self.maxpool = nn.MaxPool2d(3, 2, 1)
        chans, layers, cin = [64, 128, 256, 512], [], 64
        for i, c in enumerate(chans):
            layers.append(nn.Sequential(BasicBlock(cin, c, 1 if i == 0 else 2), BasicBlock(c, c, 1)))
            cin = c
        self.layer1, self.layer2, self.layer3, self.layer4 = layers
        self.avgpool = nn.AdaptiveAvgPool2d(1)
        self.fc = nn.Linear(512, num_classes)
        self.use_tc_fc = use_tc_fc
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
            elif isinstance(m, nn.BatchNorm2d):
                nn.init.ones_(m.weight)
                nn.init.zeros_(m.bias)

    def forward(self, x):
        x = self.maxpool(F.relu(self.bn1(self.conv1(x)), inplace=True))
        x = self.layer4(self.layer3(self.layer2(self.layer1(x))))
        x = torch.flatten(self.avgpool(x), 1)
        if self.use_tc_fc and x.is_cuda:
            from ..ops.gemm import linear_bf16, linear_tc
            if not torch.is_grad_enabled():
                return linear_bf16(x, self.fc.weight, self.fc.bias, out_dtype=torch.float32)
            return linear_tc(x.float(), self.fc.weight, self.fc.bias)     # trainable: dgrad + wgrad on the same wgmma kernel
        return self.fc(x)
