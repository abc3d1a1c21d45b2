"""dist_tuto.pth_b200 -- a Blackwell-native minimal data-parallel training library
with the API of the PyTorch distributed tutorial ``seba-1511/dist_tuto.pth``.

Public surface (tutorial names kept; see each module for file:line parity):

    init_processes / launch / init_from_env            launch.py
    send recv isend irecv                               comm.py
    all_reduce reduce broadcast scatter gather gather_to_root all_gather barrier new_group
    reduce_op get_rank get_world_size                   comm.py
    allreduce (ring) / allreduce_chunked                ring.py
    Partition DataPartitioner partition_dataset         data.py
    Net                                                 models/convnet.py
    average_gradients GradBucket DistributedDataParallel parallel/ddp.py
    FlatSGD (one-launch momentum SGD over flat buffers) ops/optim.py
    run / train / TrainConfig                           train.py
    evaluate (test loss / accuracy, sharded over ranks) ops/convnet_eval.py
    partition_eval_dataset default_eval_dataset         data.py
"""
from .comm import (reduce_op, ReduceOp, send, recv, isend, irecv, broadcast, reduce, all_reduce,  # noqa: F401
                   scatter, gather, gather_to_root, all_gather, barrier, new_group, get_rank, get_world_size,
                   is_initialized, group)
from .launch import (init_processes, init_process, launch, init_from_env, shutdown, find_free_port,  # noqa: F401
                     LaunchError)
from .ring import allreduce, allreduce_chunked  # noqa: F401
from .data import (Partition, DataPartitioner, partition_dataset, SyntheticMNIST, TensorImageDataset,  # noqa: F401
                   BatchLoader, partition_eval_dataset, default_eval_dataset)
from .models.convnet import Net  # noqa: F401
from .parallel.ddp import (average_gradients, GradBucket, DistributedDataParallel,  # noqa: F401
                           broadcast_parameters)
from .ops.optim import FlatSGD, LRSchedule  # noqa: F401
from .ops.convnet_eval import evaluate  # noqa: F401
from .train import run, train, TrainConfig  # noqa: F401

__version__ = "0.1.0"
