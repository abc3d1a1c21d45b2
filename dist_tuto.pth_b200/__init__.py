"""dist_tuto.pth_b200 -- a Blackwell-native minimal data-parallel training library
with the API of the PyTorch distributed tutorial ``seba-1511/dist_tuto.pth``.

Public surface (tutorial names kept; see each module for file:line parity):

    init_processes / launch / init_from_env            launch.py
    send recv isend irecv                               comm.py
    P2POp batch_isend_irecv                             comm.py
    all_reduce reduce broadcast scatter gather gather_to_root all_gather barrier new_group
    reduce_scatter reduce_scatter_tensor all_to_all_single all_to_all all_gather_into_tensor      comm.py
    reduce_op get_rank get_world_size                   comm.py
    allreduce (ring) / allreduce_chunked                ring.py
    Partition DataPartitioner partition_dataset         data.py
    Net                                                 models/convnet.py
    average_gradients GradBucket DistributedDataParallel parallel/ddp.py
    SyncBatchNorm (global-batch statistics)            parallel/sync_bn.py
    FlatSGD (one-launch momentum SGD over flat buffers) ops/optim.py
    FlatAdamW (one-launch AdamW over flat buffers)      ops/optim.py
    FlatRMSprop (one-launch RMSprop over flat buffers)  ops/optim.py
    FlatAdafactor (factored second moments, no sync)    ops/optim.py
    FlatLAMB FlatLARS (per-tensor trust ratios)         ops/optim.py
    FlatEMA (EMA of the weights, one launch per update) ops/optim.py
    GradScaler support (fp16 loss scaling, in-kernel)   ops/optim.py
    run / train / TrainConfig                           train.py
    evaluate (test loss / accuracy, sharded over ranks) ops/convnet_eval.py
    partition_eval_dataset default_eval_dataset         data.py
"""
from .comm import (reduce_op, ReduceOp, send, recv, isend, irecv, broadcast, reduce, all_reduce,  # noqa: F401
                   scatter, gather, gather_to_root, all_gather, barrier, new_group, get_rank, get_world_size,
                   is_initialized, group, reduce_scatter, reduce_scatter_tensor, all_to_all_single,
                   all_gather_into_tensor, all_to_all, P2POp, batch_isend_irecv)
from .launch import (init_processes, init_process, launch, init_from_env, shutdown, find_free_port,  # noqa: F401
                     LaunchError)
from .ring import allreduce, allreduce_chunked  # noqa: F401
from .data import (Partition, DataPartitioner, partition_dataset, SyntheticMNIST, TensorImageDataset,  # noqa: F401
                   BatchLoader, partition_eval_dataset, default_eval_dataset)
from .models.convnet import Net  # noqa: F401
from .parallel.ddp import (average_gradients, GradBucket, DistributedDataParallel,  # noqa: F401
                           broadcast_parameters)
from .parallel.sync_bn import SyncBatchNorm  # noqa: F401
from .ops.optim import FlatAdafactor, FlatAdamW, FlatEMA, FlatLAMB, FlatLARS, FlatRMSprop, FlatSGD, LRSchedule  # noqa: F401
from .ops.convnet_eval import evaluate  # noqa: F401
from .train import run, train, TrainConfig  # noqa: F401

__version__ = "0.1.0"
