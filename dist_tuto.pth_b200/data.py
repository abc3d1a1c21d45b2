"""Data partitioning for synchronous data-parallel SGD (layer L4).

Parity map (reference = /root/reference):
  * ``Partition``            train_dist.py:17-29, tuto.md:222-233
  * ``DataPartitioner``      train_dist.py:32-50, tuto.md:236-253
  * ``partition_dataset()``  train_dist.py:74-91, tuto.md:260-274
      global batch 128, ``bsz = 128 // world_size`` (fixes D5: the tutorial
      text divides by a float), shard ``rank`` of ``world_size`` equal shards,
      shuffled loader.

GPU-first differences:
  * the dataset is tensor-backed (uint8 images + int64 labels in one block) so a
    batch is produced by a vectorised gather + fused normalise straight into a
    *pinned* staging buffer (optionally by the native C++ prefetcher in
    ``csrc/loader.cpp``), ready for one async H2D copy per step -- instead of a
    Python ``__getitem__`` + PIL + collate per sample;
  * there is no network in this environment, so the default dataset is a
    deterministic synthetic MNIST-shaped set (60000 x 1 x 28 x 28); real MNIST
    idx files are used when present (fixes D7).
"""
from __future__ import annotations

import gzip
import os
import struct
from random import Random
from typing import Iterator, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import comm

__all__ = ["Partition", "DataPartitioner", "partition_dataset", "SyntheticMNIST", "TensorImageDataset",
           "BatchLoader", "NativeBatchLoader", "load_mnist", "write_idx", "MNIST_MEAN", "MNIST_STD", "GLOBAL_BATCH",
           "partition_eval_dataset", "default_eval_dataset", "eval_shard_range", "EVAL_SEED"]

MNIST_MEAN, MNIST_STD = 0.1307, 0.3081   # train_dist.py:82
GLOBAL_BATCH = 128                       # train_dist.py:85


class Partition:
    """Dataset-like view restricted to a list of indices (train_dist.py:17-29)."""

    def __init__(self, data, index: Sequence[int]):
        self.data = data
        self.index = index

    def __len__(self) -> int:
        return len(self.index)

    def __getitem__(self, i):
        return self.data[self.index[i]]

    # vectorised access used by BatchLoader (not in the reference)
    def index_tensor(self) -> torch.Tensor:
        t = getattr(self, "_index_t", None)
        if t is None:
            t = self._index_t = torch.as_tensor(list(self.index), dtype=torch.int64)
        return t


class DataPartitioner:
    """Split ``data`` into disjoint shuffled chunks (train_dist.py:32-50).

    Every rank builds the same permutation from the same seed, so the shards
    are disjoint without any communication.  ``int(frac * len)`` samples per
    chunk; the remainder is dropped, exactly like the reference (world 7 on
    60000 samples -> 8571 each, 3 dropped)."""

    def __init__(self, data, sizes: Sequence[float] = (0.7, 0.2, 0.1), seed: int = 1234):
        self.data = data
        self.partitions: List[List[int]] = []
        rng = Random()
        rng.seed(seed)
        n = len(data)
        order = list(range(n))
        rng.shuffle(order)
        start = 0
        for frac in sizes:
            k = int(frac * n)
            self.partitions.append(order[start:start + k])
            start += k

    def use(self, partition: int) -> Partition:
        return Partition(self.data, self.partitions[partition])


class TensorImageDataset:
    """uint8 images ``[N,H,W]`` + int64 labels, normalised on access.

    ``ds[i]`` mimics torchvision MNIST with ToTensor+Normalize
    (train_dist.py:76-83): ``(float32 [1,H,W], int)``."""

    def __init__(self, images: torch.Tensor, labels: torch.Tensor,
                 mean: float = MNIST_MEAN, std: float = MNIST_STD):
        assert images.dtype == torch.uint8 and images.dim() == 3
        assert labels.shape[0] == images.shape[0]
        self.images = images.contiguous()
        self.labels = labels.to(torch.int64).contiguous()
        self.mean, self.std = float(mean), float(std)

    def __len__(self) -> int:
        return self.images.shape[0]

    def __getitem__(self, i: int):
        x = self.images[i].to(torch.float32).div_(255.0).sub_(self.mean).div_(self.std).unsqueeze(0)
        return x, int(self.labels[i])

    def gather(self, idx: torch.Tensor, out_x: Optional[torch.Tensor] = None,
               out_y: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """Vectorised batch fetch: normalised ``[B,1,H,W]`` float32 + ``[B]`` int64."""
        b = idx.numel()
        h, w = self.images.shape[1:]
        if out_x is None:
            out_x = torch.empty(b, 1, h, w, dtype=torch.float32)
        if out_y is None:
            out_y = torch.empty(b, dtype=torch.int64)
        ox, oy = out_x[:b], out_y[:b]
        raw = self.images.index_select(0, idx)
        ox.view(b, h, w).copy_(raw)                      # uint8 -> float32
        ox.mul_(1.0 / (255.0 * self.std)).sub_(self.mean / self.std)
        torch.index_select(self.labels, 0, idx, out=oy)
        return ox, oy

    def gather_raw(self, idx: torch.Tensor, out_x: torch.Tensor, out_y: torch.Tensor):
        """uint8 batch (normalisation is then fused into the first device kernel)."""
        b = idx.numel()
        torch.index_select(self.images, 0, idx, out=out_x[:b].view(b, *self.images.shape[1:]))
        torch.index_select(self.labels, 0, idx, out=out_y[:b])
        return out_x[:b], out_y[:b]


class SyntheticMNIST(TensorImageDataset):
    """Deterministic MNIST-shaped synthetic data: class-dependent blob + noise.

    Learnable (loss falls quickly) so loss-curve parity tests mean something;
    generated from ``seed`` only, identical on every rank."""

    def __init__(self, n: int = 60000, seed: int = 1234, num_classes: int = 10, hw: int = 28):
        g = torch.Generator().manual_seed(seed)
        labels = torch.randint(0, num_classes, (n,), generator=g, dtype=torch.int64)
        yy, xx = torch.meshgrid(torch.arange(hw, dtype=torch.float32),
                                torch.arange(hw, dtype=torch.float32), indexing="ij")
        protos = []
        for c in range(num_classes):
            ang = 2.0 * np.pi * c / num_classes
            cy, cx = hw / 2 + 6.0 * np.sin(ang), hw / 2 + 6.0 * np.cos(ang)
            blob = torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * 3.0 ** 2))
            stripe = 0.5 + 0.5 * torch.cos((xx * np.cos(ang) + yy * np.sin(ang)) * (0.35 + 0.05 * c))
            protos.append((0.75 * blob + 0.25 * stripe * blob.clamp(min=0.15)).clamp(0, 1))
        protos = torch.stack(protos)                                   # [C,H,W]
        images = torch.empty(n, hw, hw, dtype=torch.uint8)
        step = 8192
        for s in range(0, n, step):
            e = min(n, s + step)
            noise = torch.rand(e - s, hw, hw, generator=g) * 0.35
            img = (protos[labels[s:e]] * (0.65 + 0.35 * torch.rand(e - s, 1, 1, generator=g)) + noise)
            images[s:e] = (img.clamp_(0, 1) * 255.0).to(torch.uint8)
        super().__init__(images, labels)


# ------------------------------------------------------------------ idx I/O --
_IDX_FILES = {True: ("train-images-idx3-ubyte", "train-labels-idx1-ubyte"),
              False: ("t10k-images-idx3-ubyte", "t10k-labels-idx1-ubyte")}


def _open_maybe_gz(path):
    if os.path.isfile(path):
        return open(path, "rb")
    if os.path.isfile(path + ".gz"):
        return gzip.open(path + ".gz", "rb")
    return None


def load_mnist(root: str = "./data", train: bool = True) -> Optional[TensorImageDataset]:
    """Read MNIST idx files under ``root/MNIST/raw`` if they exist (else None)."""
    img_name, lab_name = _IDX_FILES[train]
    for sub in (os.path.join(root, "MNIST", "raw"), root):
        fi, fl = _open_maybe_gz(os.path.join(sub, img_name)), _open_maybe_gz(os.path.join(sub, lab_name))
        if fi is None or fl is None:
            for f in (fi, fl):
                if f is not None:
                    f.close()
            continue
        with fi, fl:
            magic, n, h, w = struct.unpack(">IIII", fi.read(16))
            if magic != 2051:
                raise ValueError(f"bad idx3 magic {magic}")
            images = torch.from_numpy(np.frombuffer(fi.read(n * h * w), dtype=np.uint8).copy()).view(n, h, w)
            magic, n2 = struct.unpack(">II", fl.read(8))
            if magic != 2049 or n2 != n:
                raise ValueError("bad idx1 header")
            labels = torch.from_numpy(np.frombuffer(fl.read(n), dtype=np.uint8).copy()).to(torch.int64)
        return TensorImageDataset(images, labels)
    return None


def write_idx(root: str, ds: TensorImageDataset, test_n: int = 1000) -> str:
    """Write ``ds`` as MNIST idx files under ``root/MNIST/raw`` (used to feed the
    *unmodified* reference ``partition_dataset()`` offline, see baseline/)."""
    raw = os.path.join(root, "MNIST", "raw")
    os.makedirs(raw, exist_ok=True)

    def dump(img_name, lab_name, images, labels):
        n, h, w = images.shape
        with open(os.path.join(raw, img_name), "wb") as f:
            f.write(struct.pack(">IIII", 2051, n, h, w))
            f.write(images.numpy().tobytes())
        with open(os.path.join(raw, lab_name), "wb") as f:
            f.write(struct.pack(">II", 2049, n))
            f.write(labels.to(torch.uint8).numpy().tobytes())

    dump(*_IDX_FILES[True], ds.images, ds.labels)
    k = min(test_n, len(ds))
    dump(*_IDX_FILES[False], ds.images[:k], ds.labels[:k])
    return raw


# ------------------------------------------------------------------ loader ---
class BatchLoader:
    """Shuffled mini-batch iterator over a :class:`Partition` (DataLoader stand-in).

    Yields ``(data [b,1,28,28] float32, target [b] int64)`` host tensors; the
    buffers are pinned when CUDA is present so the training step can issue one
    async H2D copy.  ``len(loader)`` = number of batches (last one may be short,
    like ``DataLoader(drop_last=False)``); ``loader.dataset`` is the partition
    (train_dist.py:112 uses ``len(train_set.dataset)``)."""

    def __init__(self, partition, batch_size: int, shuffle: bool = True, drop_last: bool = False,
                 pin_memory: Optional[bool] = None, seed: Optional[int] = None, raw_uint8: bool = False,
                 num_buffers: int = 4):
        self.dataset = partition
        self.batch_size = int(batch_size)
        if self.batch_size <= 0:
            raise ValueError("batch_size must be a positive integer (128 // world_size)")
        self.shuffle, self.drop_last, self.raw_uint8 = shuffle, drop_last, raw_uint8
        self._gen = torch.Generator()
        if seed is not None:
            self._gen.manual_seed(seed)
        else:
            self._gen.manual_seed(int(torch.initial_seed()) & 0x7FFFFFFF)
        base = partition.data if isinstance(partition, Partition) else partition
        self._base = base if hasattr(base, "gather") else None
        self._index = partition.index_tensor() if isinstance(partition, Partition) else \
            torch.arange(len(partition), dtype=torch.int64)
        pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        self._bufs = []
        if self._base is not None:
            h, w = self._base.images.shape[1:]
            for _ in range(num_buffers):
                x = torch.empty(self.batch_size, 1, h, w, dtype=torch.uint8 if raw_uint8 else torch.float32)
                y = torch.empty(self.batch_size, dtype=torch.int64)
                if pin:
                    x, y = x.pin_memory(), y.pin_memory()
                self._bufs.append((x, y))

    def __len__(self) -> int:
        n = len(self.dataset)
        return n // self.batch_size if self.drop_last else (n + self.batch_size - 1) // self.batch_size

    def __iter__(self) -> Iterator[Tuple[torch.Tensor, torch.Tensor]]:
        n = len(self.dataset)
        order = torch.randperm(n, generator=self._gen) if self.shuffle else torch.arange(n)
        nb = len(self)
        for b in range(nb):
            sel = order[b * self.batch_size:(b + 1) * self.batch_size]
            idx = self._index.index_select(0, sel)
            if self._base is not None:
                x, y = self._bufs[b % len(self._bufs)]
                if self.raw_uint8:
                    yield self._base.gather_raw(idx, x, y)
                else:
                    yield self._base.gather(idx, x, y)
            else:  # generic dataset: per-sample path (reference behaviour)
                items = [self.dataset.data[int(i)] if isinstance(self.dataset, Partition) else self.dataset[int(i)]
                         for i in idx]
                xs = torch.stack([torch.as_tensor(it[0]) for it in items])
                ys = torch.as_tensor([int(it[1]) for it in items], dtype=torch.int64)
                yield xs, ys


class NativeBatchLoader:
    """Same contract as :class:`BatchLoader`, served by the C++ prefetcher (csrc/loader.cpp).

    A worker thread gathers + normalises the next batches into a ring of pinned
    buffers while the GPU trains; the yielded tensors alias those buffers (the
    fused trainer adopts them as CUDA-graph copy sources -> zero extra copies).
    A buffer is recycled ``num_buffers - 1`` batches after it was yielded."""

    def __init__(self, partition, batch_size: int, shuffle: bool = True, drop_last: bool = False,
                 pin_memory: Optional[bool] = None, seed: Optional[int] = None, raw_uint8: bool = False,
                 num_buffers: int = 24):
        from .ops import _ext
        base = partition.data if isinstance(partition, Partition) else partition
        if not hasattr(base, "images"):
            raise TypeError("NativeBatchLoader needs a tensor-backed dataset (TensorImageDataset)")
        self.dataset = partition
        self.batch_size = int(batch_size)
        idx = partition.index_tensor() if isinstance(partition, Partition) else torch.arange(len(partition))
        pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        seed = int(torch.initial_seed()) & 0x7FFFFFFF if seed is None else seed
        # >= 4: FusedTrainer.step() adopts these pinned buffers as graph H2D sources and keeps up to 2 steps in flight, so a
        # slot may only be refilled 3 yields later (with 3 buffers batch 0's captured copy could still be pending)
        self.num_buffers = max(4, num_buffers)
        self._l = _ext.C().NativeLoader(base.images, base.labels, idx, self.batch_size, self.num_buffers, shuffle,
                                        drop_last, raw_uint8, base.mean, base.std, seed, pin)
        self._epoch = 0
        self.before_recycle = None     # optional callable: make sure the oldest yielded batch was consumed

    def __len__(self) -> int:
        return int(self._l.num_batches())

    def begin_epoch(self) -> None:
        """Start the prefetch thread on a freshly shuffled epoch (used by the native step executor)."""
        self._l.start_epoch(self._epoch)
        self._epoch += 1

    def __iter__(self):
        self._l.start_epoch(self._epoch)
        self._epoch += 1
        out = 0
        try:
            while True:
                if out >= self.num_buffers - 1:
                    if self.before_recycle is not None:
                        self.before_recycle()
                    self._l.release()
                    out -= 1
                r = self._l.next()
                if r is None:
                    break
                out += 1
                yield r
        finally:
            if self.before_recycle is not None:
                self.before_recycle()
            self._l.stop()


_DATASET_CACHE = {}


def default_dataset(root: str = "./data", n: int = 60000, seed: int = 1234) -> TensorImageDataset:
    """Real MNIST when its idx files are on disk, else the synthetic stand-in."""
    key = (os.path.abspath(root), n, seed)
    ds = _DATASET_CACHE.get(key)
    if ds is None:
        ds = load_mnist(root, train=True) or SyntheticMNIST(n=n, seed=seed)
        _DATASET_CACHE[key] = ds
    return ds


EVAL_SEED = 4321        # synthetic test set: same class prototypes as the training set, different samples


def default_eval_dataset(root: str = "./data", n: int = 10000) -> TensorImageDataset:
    """The real MNIST test split (``t10k``) when its idx files are on disk, else ``SyntheticMNIST(n, seed=EVAL_SEED)``."""
    key = (os.path.abspath(root), n, "eval")
    ds = _DATASET_CACHE.get(key)
    if ds is None:
        ds = load_mnist(root, train=False) or SyntheticMNIST(n=n, seed=EVAL_SEED)
        _DATASET_CACHE[key] = ds
    return ds


def eval_shard_range(n: int, rank: int, world_size: int) -> Tuple[int, int]:
    """``[lo, hi)`` of rank ``rank``'s evaluation shard: ``n // world_size`` samples, one more on the first
    ``n % world_size`` ranks, in rank order."""
    q, r = divmod(n, world_size)
    lo = rank * q + min(rank, r)
    return lo, lo + q + (1 if rank < r else 0)


def partition_eval_dataset(dataset=None, rank: Optional[int] = None, world_size: Optional[int] = None) -> Partition:
    """This rank's contiguous shard of an evaluation set, without shuffling and without dropping a remainder: over all
    ranks every sample is evaluated exactly once (``DataPartitioner`` drops the remainder, which is right for training)."""
    size = comm.get_world_size() if world_size is None else world_size
    rank = comm.get_rank() if rank is None else rank
    if dataset is None:
        dataset = default_eval_dataset()
    if not 0 <= rank < size:
        raise ValueError(f"rank {rank} outside a world of {size}")
    lo, hi = eval_shard_range(len(dataset), rank, size)
    return Partition(dataset, range(lo, hi))


def partition_dataset(dataset=None, global_batch: int = GLOBAL_BATCH, seed: int = 1234,
                      rank: Optional[int] = None, world_size: Optional[int] = None, native: Optional[bool] = None,
                      **loader_kw):
    """Shard the training set for this rank; returns ``(loader, bsz)``.

    Same contract as train_dist.py:74-91: equal shards ``[1/size] * size``,
    this rank's shard, ``bsz = global_batch // size`` so the *global* batch
    stays 128 at every world size (tuto.md:277)."""
    size = comm.get_world_size() if world_size is None else world_size
    rank = comm.get_rank() if rank is None else rank
    if dataset is None:
        dataset = default_dataset()
    bsz = global_batch // size
    if bsz < 1:
        raise ValueError(f"world size {size} exceeds the global batch {global_batch}")
    sizes = [1.0 / size for _ in range(size)]
    part = DataPartitioner(dataset, sizes, seed=seed).use(rank)
    if native is None:
        native = hasattr(dataset, "images") and torch.cuda.is_available()
    if native:
        return NativeBatchLoader(part, batch_size=bsz, shuffle=True, **loader_kw), bsz
    return BatchLoader(part, batch_size=bsz, shuffle=True, **loader_kw), bsz
