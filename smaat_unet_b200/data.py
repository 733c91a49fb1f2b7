"""Input pipeline for the GPU path (SURVEY 8 f3): pre-decompressed shards + a pinned, threaded batch loader.

The reference reads gzip-9 HDF5 sample by sample through one DataLoader worker (utils/dataset_precip.py:23-44,63-77,
models/regression_lightning.py:177-199) -- a few hundred frames/s at best, far below what the GPU path consumes in
training and in inference.  This module keeps the reference's *indexing semantics* and removes the
decompression and the per-sample Python overhead from the step:

  * ``write_shard`` / ``convert_h5`` -- one-off conversion of ``<file>[train|test]["images"]`` into a raw float32
    ``.npy`` (memory-mappable; the page cache holds it after the first epoch).  ``convert_h5`` needs ``h5py`` and is
    the only place that does.
  * ``precipitation_maps_oversampled_shard`` / ``precipitation_maps_shard`` -- ``torch.utils.data.Dataset``s with the
    constructor arguments, ``__len__`` and ``__getitem__`` results of the reference's
    ``precipitation_maps_oversampled_h5`` (utils/dataset_precip.py:47-77) and ``precipitation_maps_h5`` (:6-44):
    ``imgs = images[index]`` (resp. ``images[index : index + seq]``), ``input = imgs[:num_input]``, ``target = imgs[-1]``.
  * ``precipitation_maps_classification_shard`` -- ``precipitation_maps_classification_h5`` (:83-127): the same sliding
    window with the target frame bucketed into 8 rain-rate classes (int64).
  * ``PinnedBatchLoader`` -- a background thread gathers whole batches straight into pinned host buffers (a small
    ring), in the order of a sampler (sequential, seeded shuffle, or an explicit index list such as the reference's
    train/valid split), sharded across ranks like ``DistributedSampler``; it yields ``(x, y)`` pinned tensors that
    ``TrainSession.step`` / ``InferenceSession.submit`` copy asynchronously.

Pure host code (numpy + torch CPU tensors): no kernels, nothing here touches the device.
"""
from __future__ import annotations

import queue
import threading

import numpy as np
import torch
from torch.utils.data import Dataset


# ------------------------------------------------------------------------------------------------ shards
def write_shard(path, images):
    """Store ``images`` (float32-convertible array, e.g. (N, T, H, W) or (N, H, W)) as a memory-mappable .npy shard."""
    arr = np.ascontiguousarray(np.asarray(images, dtype=np.float32))
    np.save(path, arr, allow_pickle=False)
    return path


def convert_h5(in_file, out_prefix, splits=("train", "test"), chunk=256):
    """Decompress ``in_file[split]["images"]`` into ``<out_prefix>_<split>.npy`` (needs h5py; streaming, `chunk` rows at a time)."""
    import h5py  # only needed for the one-off conversion
    out = {}
    with h5py.File(in_file, "r") as f:
        for split in splits:
            src = f[split]["images"]
            dst = np.lib.format.open_memmap(f"{out_prefix}_{split}.npy", mode="w+", dtype=np.float32, shape=src.shape)
            for i in range(0, src.shape[0], chunk):
                dst[i:i + chunk] = src[i:i + chunk]
            dst.flush()
            out[split] = f"{out_prefix}_{split}.npy"
    return out


def _open(images):
    if isinstance(images, (str, bytes)) or hasattr(images, "__fspath__"):
        return np.load(images, mmap_mode="r", allow_pickle=False)
    return images


class precipitation_maps_oversampled_shard(Dataset):
    """Same samples as ``precipitation_maps_oversampled_h5`` (utils/dataset_precip.py:47-77) over a (samples, T, H, W) shard."""

    def __init__(self, in_file, num_input_images, num_output_images, train=True, transform=None):
        super().__init__()
        self.file_name = in_file
        self.dataset = _open(in_file)
        self.samples = self.dataset.shape[0]
        self.num_input = num_input_images
        self.num_output = num_output_images
        self.train = train
        self.transform = transform

    def __getitem__(self, index):
        imgs = np.array(self.dataset[index], dtype="float32")
        if self.transform is not None:
            imgs = self.transform(imgs)
        return imgs[: self.num_input], imgs[-1]

    def __len__(self):
        return self.samples

    # fast path used by PinnedBatchLoader: write sample `index` straight into the batch buffers
    def read_into(self, index, x_out, y_out):
        if self.transform is not None:
            x, y = self[index]
            x_out[...] = x
            y_out[...] = y
            return
        imgs = self.dataset[index]
        x_out[...] = imgs[: self.num_input]
        y_out[...] = imgs[-1]

    def sample_shapes(self):
        t, h, w = self.dataset.shape[1:]
        return (min(self.num_input, t), h, w), (h, w)


class precipitation_maps_shard(Dataset):
    """Same samples as ``precipitation_maps_h5`` (utils/dataset_precip.py:6-44): a sliding window over an (n_images, H, W) shard."""

    def __init__(self, in_file, num_input_images, num_output_images, train=True, transform=None):
        super().__init__()
        self.file_name = in_file
        self.dataset = _open(in_file)
        self.n_images, self.nx, self.ny = self.dataset.shape
        self.num_input = num_input_images
        self.num_output = num_output_images
        self.sequence_length = num_input_images + num_output_images
        self.train = train
        self.size_dataset = self.n_images - (num_input_images + num_output_images)
        self.transform = transform

    def __getitem__(self, index):
        imgs = np.array(self.dataset[index: index + self.sequence_length], dtype="float32")
        if self.transform is not None:
            imgs = self.transform(imgs)
        return imgs[: self.num_input], imgs[-1]

    def __len__(self):
        return self.size_dataset

    def read_into(self, index, x_out, y_out):
        if self.transform is not None:
            x, y = self[index]
            x_out[...] = x
            y_out[...] = y
            return
        x_out[...] = self.dataset[index: index + self.num_input]
        y_out[...] = self.dataset[index + self.sequence_length - 1]

    def sample_shapes(self):
        return (self.num_input, self.nx, self.ny), (self.nx, self.ny)


class precipitation_maps_classification_shard(Dataset):
    """Same samples as ``precipitation_maps_classification_h5`` (utils/dataset_precip.py:83-127) over an (n_images, H, W)
    shard: the sliding window of ``precipitation_maps_shard`` with the target frame turned into 8 rain-rate classes,
    ``np.digitize(target * 47.83 * 12, [0, 0.5, 1, 2, 5, 10, 30], right=True)`` (mm/h bins of the de-normalised frame),
    as int64 class indices for ``CrossEntropyLoss`` / ``TrainSession(loss="cross_entropy")``."""

    target_dtype = torch.int64
    num_classes = 8

    def __init__(self, in_file, num_input_images, img_to_predict, train=True, transform=None):
        super().__init__()
        self.file_name = in_file
        self.dataset = _open(in_file)
        self.n_images, self.nx, self.ny = self.dataset.shape
        self.num_input = num_input_images
        self.img_to_predict = img_to_predict
        self.sequence_length = num_input_images + img_to_predict
        self.bins = np.array([0.0, 0.5, 1, 2, 5, 10, 30])
        self.train = train
        self.size_dataset = self.n_images - (num_input_images + img_to_predict)
        self.transform = transform

    def _buckets(self, target_img):
        # float32 frame times Python floats stays float32 (as in the reference), then the bin search in float64
        return np.digitize(target_img * 47.83 * 12, self.bins, right=True)

    def __getitem__(self, index):
        imgs = np.array(self.dataset[index: index + self.sequence_length], dtype="float32")
        if self.transform is not None:
            imgs = self.transform(imgs)
        return imgs[: self.num_input], self._buckets(imgs[-1])

    def __len__(self):
        return self.size_dataset

    def read_into(self, index, x_out, y_out):
        if self.transform is not None:
            x, y = self[index]
            x_out[...] = x
            y_out[...] = y
            return
        x_out[...] = self.dataset[index: index + self.num_input]
        y_out[...] = self._buckets(np.asarray(self.dataset[index + self.sequence_length - 1], dtype=np.float32))

    def sample_shapes(self):
        return (self.num_input, self.nx, self.ny), (self.nx, self.ny)


# ------------------------------------------------------------------------------------------------ loader
def shard_indices(indices, rank, world, drop_last=False):
    """This rank's share of ``indices`` with ``DistributedSampler`` semantics: padded by wrapping around (or truncated
    with ``drop_last``) to a multiple of ``world``, then strided ``rank::world``."""
    indices = list(indices)
    n = len(indices)
    if world <= 1:
        return indices
    if drop_last:
        total = (n // world) * world
        indices = indices[:total]
    else:
        total = -(-n // world) * world
        pad = total - n
        if pad:
            indices = indices + (indices * (-(-pad // max(n, 1))))[:pad]
    return indices[rank:total:world]


class PinnedBatchLoader:
    """Iterate ``(x, y)`` batches of a shard dataset; a background thread fills a ring of pinned host buffers.

    ``indices``: explicit sample order (e.g. the reference's train / valid split); default = all samples.
    ``shuffle``: reshuffle every epoch with ``seed + epoch`` (call ``set_epoch`` like a DistributedSampler).
    ``rank`` / ``world``: shard the (shuffled) index list across data-parallel ranks.
    The yielded tensors are views of a ring slot that is handed back to the filler thread when the NEXT batch is
    requested.  If the consumer only *enqueued* an asynchronous host->device copy of the batch (``TrainSession.step``,
    ``InferenceSession.submit``), it must say when that copy is done: ``loader.guard(event)`` attaches a CUDA event to
    the slot just yielded and the filler thread waits for it before overwriting the slot::

        for x, y in loader:
            sess.step(x, y)
            loader.guard(sess.last_h2d_event())
    """

    def __init__(self, dataset, batch_size, indices=None, shuffle=False, seed=0, drop_last=True, rank=0, world=1, ring=3,
                 pin_memory=None):
        self.dataset, self.batch_size = dataset, int(batch_size)
        self.indices = list(range(len(dataset))) if indices is None else list(indices)
        self.shuffle, self.seed, self.drop_last = bool(shuffle), int(seed), bool(drop_last)
        self.rank, self.world, self.ring = int(rank), int(world), max(2, int(ring))
        self.epoch = 0
        pin = torch.cuda.is_available() if pin_memory is None else bool(pin_memory)
        xs, ys = dataset.sample_shapes()
        ydt = getattr(dataset, "target_dtype", torch.float32)      # int64 class indices for the classification shard
        self._x = [torch.empty((self.batch_size,) + tuple(xs), dtype=torch.float32, pin_memory=pin) for _ in range(self.ring)]
        self._y = [torch.empty((self.batch_size,) + tuple(ys), dtype=ydt, pin_memory=pin) for _ in range(self.ring)]
        self._guard = [None] * self.ring      # per slot: event that must complete before the slot is refilled
        self._held = None

    def guard(self, event):
        """The slot yielded last must not be overwritten before ``event`` (anything with ``.synchronize()``) completes."""
        if self._held is not None and event is not None:
            self._guard[self._held] = event

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def epoch_indices(self):
        idx = list(self.indices)
        if self.shuffle:
            rng = np.random.default_rng(self.seed + self.epoch)
            idx = [idx[i] for i in rng.permutation(len(idx))]
        return shard_indices(idx, self.rank, self.world, drop_last=False)

    def __len__(self):
        n = len(shard_indices(self.indices, self.rank, self.world))
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def __iter__(self):
        idx = self.epoch_indices()
        nb = len(self)
        free = queue.Queue()
        ready = queue.Queue()
        for s in range(self.ring - 1):      # one slot always belongs to the consumer
            free.put(s)
        held = [self.ring - 1]
        stop = threading.Event()

        def work():
            try:
                for bi in range(nb):
                    s = free.get()
                    if stop.is_set():
                        return
                    ev, self._guard[s] = self._guard[s], None
                    if ev is not None:
                        ev.synchronize()     # the consumer's asynchronous copy out of this slot has finished
                    chunk = idx[bi * self.batch_size:(bi + 1) * self.batch_size]
                    xb, yb = self._x[s].numpy(), self._y[s].numpy()
                    for j, i in enumerate(chunk):
                        self.dataset.read_into(i, xb[j], yb[j])
                    ready.put((s, len(chunk)))
                ready.put(None)
            except BaseException as e:  # surface loader errors in the consumer
                ready.put(e)

        t = threading.Thread(target=work, daemon=True)
        t.start()
        try:
            while True:
                item = ready.get()
                if item is None:
                    break
                if isinstance(item, BaseException):
                    raise item
                s, n = item
                free.put(held[0])        # the previously yielded slot may be refilled now (after its guard event)
                held[0] = s
                self._held = s
                yield self._x[s][:n], self._y[s][:n]
        finally:
            self._held = None
            stop.set()
            free.put(0)
            t.join(timeout=5)
