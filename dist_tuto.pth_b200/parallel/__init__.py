"""Data-parallel engine: gradient buckets, overlapped fused all-reduce, symmetric peer memory, SyncBatchNorm."""
from .ddp import GradBucket, average_gradients, DistributedDataParallel, broadcast_parameters  # noqa: F401
from .sync_bn import SyncBatchNorm, sync_batch_norm  # noqa: F401
