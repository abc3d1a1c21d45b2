"""Per-rank body of the two-GPU weight-decay / Nesterov test (spawned processes import it from here)."""
import torch

import sgd_options_model as SM


def w_two_gpu_options(rank, size):
    """Two GPUs, push exchange with an fp32 and a bf16 wire, weight decay and Nesterov on: every update is the model's
    update of the exchanged gradient, and the replicas stay bit-identical."""
    import torch.distributed as dist
    from dist_tuto.pth_b200.ops.convnet_fused import NPAR_ALLOC, FusedTrainer
    dev = torch.device("cuda", torch.cuda.current_device())
    for wire in (torch.float32, torch.bfloat16):
        tr = FusedTrainer(32, lr=0.05, seed=4, device=dev, grad_wire=wire, weight_decay=1e-2, nesterov=True)
        assert tr.inbox_handle is not None
        for k in range(8):
            g = torch.Generator().manual_seed(50 + k * size + rank)
            x, y = torch.randn(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).pin_memory()
            tr.sync_lag(0)
            torch.cuda.synchronize()
            p0, m0 = tr.params.clone(), tr.momentum.clone()
            tr.step(x, y)
            tr.sync_lag(0)
            torch.cuda.synchronize()
            # this step's bucket (parity k & 1) is re-zeroed only by the next step: the exchanged gradient is the rank
            # sum of the buckets, bf16-rounded per term on a bf16 wire, times 1/world
            cur = tr.grads[(k & 1) * NPAR_ALLOC:(k & 1) * NPAR_ALLOC + NPAR_ALLOC].clone()
            if wire == torch.bfloat16:
                cur = cur.to(torch.bfloat16).float()
            terms = [torch.empty_like(cur) for _ in range(size)]
            dist.all_gather(terms, cur)
            acc = torch.zeros_like(cur)
            for t in terms:
                acc = acc + t
            gsum = acc * torch.tensor(1.0 / size, dtype=torch.float32)
            p, m = SM.sgd_update(gsum, p0, m0, tr.mu, tr.lr, tr.weight_decay, True)
            assert torch.equal(p, tr.params) and torch.equal(m, tr.momentum), (wire, k)
            other = tr.params.clone()
            dist.broadcast(other, src=0)
            assert torch.equal(other, tr.params), (wire, k)
    dist.barrier()
