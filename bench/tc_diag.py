"""Diagnostic: fused ConvNet kernel, SIMT vs wgmma conv2 path vs fp64 oracle (errors per tensor, training curves)."""
import json
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from dist_tuto.pth_b200.models.convnet import Net  # noqa: E402
from dist_tuto.pth_b200.ops import _ext  # noqa: E402
from dist_tuto.pth_b200.ops.convnet_fused import (FusedTrainer, convnet_forward, convnet_loss_and_grads, pack_params,  # noqa: E402
                                                  unpack_params)

C = _ext.C()
dev = torch.device("cuda", 0)
out = {}
for B in (1, 2, 16, 128):
    torch.manual_seed(3)
    net = Net().to(dev).eval()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, 1, 28, 28, generator=g).to(dev)
    y = torch.randint(0, 10, (B,), generator=g).to(dev)
    flat = pack_params(net)
    net64 = Net().to(dev).double().eval()
    net64.load_state_dict({k: v.double() for k, v in net.state_dict().items()})
    ref_out = net64(x.double())
    ref_loss = F.nll_loss(ref_out, y)
    ref_loss.backward()
    row = {}
    for mode in (0, 1):
        C.convnet_set_tc(bool(mode))
        o = convnet_forward(flat, x)
        loss, grads = convnet_loss_and_grads(flat, x, y, training=False)
        torch.cuda.synchronize()
        views = unpack_params(grads)
        errs = {n: float((views[n].double() - p.grad).abs().max() / p.grad.abs().max().clamp_min(1e-12)) for n, p in net64.named_parameters()}
        per_sample = (o.double() - ref_out).abs().max(dim=1).values
        row["tc" if mode else "simt"] = {"fwd_max_abs_err": float(per_sample.max()), "fwd_err_per_sample_first8": [round(float(v), 4) for v in per_sample[:8]],
                                         "loss": float(loss), "ref_loss": float(ref_loss), "grad_rel_err": {k: round(v, 5) for k, v in errs.items()}}
    out[f"B{B}"] = row
curves = {}
for mode in (0, 1):
    C.convnet_set_tc(bool(mode))
    tr = FusedTrainer(64, lr=0.01, seed=1, device=dev, p_drop=0.5)
    g = torch.Generator().manual_seed(0)
    xs = torch.randn(64, 1, 28, 28, generator=g).pin_memory()
    ys = torch.randint(0, 10, (64,), generator=g).pin_memory()
    c = []
    for i in range(40):
        tr.step(xs, ys)
        c.append(round(tr.pop_loss_sum(), 4))
    curves["tc" if mode else "simt"] = c[::4]
out["train_curve_same_batch_lr0.01"] = curves
C.convnet_set_tc(False)
print(json.dumps(out, indent=1))
