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
  * ``convert_voc`` / ``voc_segmentation_shard`` -- the VOC segmentation set (utils/dataset_VOC.py:73-168): the one-off
    decode + ``Resize(256)`` + ``CenterCrop(224)`` into uint8 shards, and a ``Dataset`` over them whose per-sample random
    augmentation choices are drawn on the host, in the reference's order, and applied either on the CPU (``__getitem__``)
    or on the device (``ops.voc_augment``, one kernel per batch).
  * ``PinnedBatchLoader`` -- a background thread gathers whole batches straight into pinned host buffers (a small
    ring), in the order of a sampler (sequential, seeded shuffle, or an explicit index list such as the reference's
    train/valid split), sharded across ranks like ``DistributedSampler``; it yields ``(x, y)`` pinned tensors that
    ``TrainSession.step`` / ``InferenceSession.submit`` copy asynchronously (``(x, y, aug)`` for an augmenting VOC shard).

Pure host code (numpy + torch CPU tensors): no kernels, nothing here touches the device.
"""
from __future__ import annotations

import math
import queue
import random
import threading

import numpy as np
import torch
from torch.utils.data import Dataset

from .parallel import shard_range


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


# ------------------------------------------------------------------------------------------------ VOC segmentation
VOC_MEAN = (0.485, 0.456, 0.406)     # the reference's Normalize (utils/dataset_VOC.py:152-155)
VOC_STD = (0.229, 0.224, 0.225)


def convert_voc(voc_root, image_set, out_prefix):
    """Decode ``<voc_root>/VOC2012`` (the reference's ``root``) split ``image_set`` once, run the training script's
    deterministic ``transformations`` (``Resize(256)`` + ``CenterCrop(224)``, train_SmaAtUNet.py:149) on every image and mask,
    and write ``<out_prefix>_images.npy`` (N, 224, 224, 3) and ``<out_prefix>_masks.npy`` (N, 224, 224) uint8 in the split
    file's order.  Needs PIL and torchvision (only here).  Returns the two paths."""
    import os

    from PIL import Image
    from torchvision import transforms

    voc = os.path.join(os.fspath(voc_root), "VOC2012")
    with open(os.path.join(voc, "ImageSets", "Segmentation", image_set + ".txt")) as f:
        names = [x.strip() for x in f.readlines()]
    tf = transforms.Compose([transforms.Resize(256), transforms.CenterCrop(224)])
    paths = (f"{out_prefix}_images.npy", f"{out_prefix}_masks.npy")
    imgs = np.lib.format.open_memmap(paths[0], mode="w+", dtype=np.uint8, shape=(len(names), 224, 224, 3))
    masks = np.lib.format.open_memmap(paths[1], mode="w+", dtype=np.uint8, shape=(len(names), 224, 224))
    for i, n in enumerate(names):
        imgs[i] = np.asarray(tf(Image.open(os.path.join(voc, "JPEGImages", n + ".jpg")).convert("RGB")))
        masks[i] = np.asarray(tf(Image.open(os.path.join(voc, "SegmentationClass", n + ".png"))))
    imgs.flush()
    masks.flush()
    return paths


def _pil_rotation(deg, w, h):
    """PIL's ``Image.rotate(deg, expand=False)`` affine matrix (a, b, c, d, e, f), in its own double arithmetic."""
    angle = -math.radians(deg % 360.0)
    a, b = round(math.cos(angle), 15), round(math.sin(angle), 15)
    d, e = round(-math.sin(angle), 15), round(math.cos(angle), 15)
    cx, cy = w / 2, h / 2
    return a, b, a * -cx + b * -cy + 0.0 + cx, d, e, d * -cx + e * -cy + 0.0 + cy


def rotation_source(deg, h, w):
    """Source (ys, xs) int64 (h, w) of every output pixel of PIL's NEAREST ``rotate(deg)`` of an (h, w) image (out of range:
    the fill).  PIL walks the rows in 16.16 fixed point when the four corners map inside +-32768 and in doubles otherwise
    (ImagingTransformAffine); both are restated with PIL's rounding."""
    a = _pil_rotation(deg, w, h)

    def inside(x, y):
        return abs(x * a[0] + y * a[1] + a[2]) < 32768.0 and abs(x * a[3] + y * a[4] + a[5]) < 32768.0

    if inside(0, 0) and inside(w, h) and inside(0, h) and inside(w, 0):
        def fix(v):
            return math.floor(v * 65536.0 + 0.5)
        X, Y = np.arange(w, dtype=np.int64), np.arange(h, dtype=np.int64)[:, None]
        xx = fix(a[2] + a[0] * 0.5 + a[1] * 0.5) + Y * fix(a[1]) + X * fix(a[0])
        yy = fix(a[5] + a[3] * 0.5 + a[4] * 0.5) + Y * fix(a[4]) + X * fix(a[3])
        return yy >> 16, xx >> 16
    # the double walk: every coordinate is a running sum, so the order of the additions is kept (add.accumulate is serial)
    xo = np.add.accumulate(np.array([a[2] + a[1] * 0.5 + a[0] * 0.5] + [a[1]] * (h - 1)))
    yo = np.add.accumulate(np.array([a[5] + a[4] * 0.5 + a[3] * 0.5] + [a[4]] * (h - 1)))
    xs, ys = np.empty((h, w)), np.empty((h, w))
    for y in range(h):
        xs[y] = np.add.accumulate(np.array([xo[y]] + [a[0]] * (w - 1)))
        ys[y] = np.add.accumulate(np.array([yo[y]] + [a[3]] * (w - 1)))
    coord = lambda v: np.where(v < 0.0, -1, np.trunc(np.maximum(v, 0.0))).astype(np.int64)  # noqa: E731  (PIL's COORD)
    return coord(ys), coord(xs)


def voc_augment_u8(img, mask, aug):
    """``apply_augmentations`` (utils/dataset_VOC.py:150-168) with the choices ``aug`` = (flip, rot, bright) on uint8 arrays:
    img (H, W, 3), mask (H, W) -> augmented uint8 copies, PIL's arithmetic exactly (what smaat_voc_augment_fwd computes)."""
    flip, rot, bright = (int(v) for v in aug)
    img, mask = np.asarray(img, np.uint8), np.asarray(mask, np.uint8)
    if flip:
        img, mask = img[:, ::-1], mask[:, ::-1]
    if rot:
        h, w = mask.shape
        ys, xs = rotation_source(10.0 if rot > 0 else -10.0, h, w)
        ok = (xs >= 0) & (xs < w) & (ys >= 0) & (ys < h)
        ri, rm = np.zeros_like(img), np.zeros_like(mask)
        ri[ok], rm[ok] = img[ys[ok], xs[ok]], mask[ys[ok], xs[ok]]
        img, mask = ri, rm
    if bright:
        # ImageEnhance.Brightness: ImagingBlend with black at fp32 alpha, truncated, clamped when alpha > 1
        alpha = np.float32(1.2 if bright > 0 else 1.2 - 0.4)
        img = np.minimum(alpha * img.astype(np.float32), np.float32(255)).astype(np.uint8)
    return np.ascontiguousarray(img), np.ascontiguousarray(mask)


def voc_normalize_u8(img, mask, mean=VOC_MEAN, std=VOC_STD):
    """``ToTensor`` + ``Normalize(mean, std)`` of an (H, W, 3) uint8 image and ``target[target == 255] = 0`` of the mask, as
    the reference returns them: (3, H, W) float32 and (H, W) int64 torch tensors."""
    v = np.asarray(img, np.uint8).transpose(2, 0, 1).astype(np.float32) / np.float32(255)
    v = (v - np.asarray(mean, np.float32)[:, None, None]) / np.asarray(std, np.float32)[:, None, None]
    t = np.asarray(mask, np.uint8).astype(np.int64)
    t[t == 255] = 0
    return torch.from_numpy(np.ascontiguousarray(v)), torch.from_numpy(t)


class voc_segmentation_shard(Dataset):
    """``VOCSegmentation`` (utils/dataset_VOC.py:73-168) with ``transformations=Resize(256) + CenterCrop(224)`` over the
    uint8 shards of ``convert_voc``: ``__len__`` and the ``(img (3, 224, 224) float32, target (224, 224) int64)`` samples of
    the reference.  ``augmentations``: the reference's random flip / rotation / brightness; ``__getitem__`` draws them from
    its own ``random.Random(seed)`` and applies them on the CPU.  ``PinnedBatchLoader`` instead carries the uint8 sample and
    its drawn ``aug`` row, and ``ops.voc_augment`` (or a ``TrainSession`` with ``input_transform=ops.VOCNormalize()``) applies
    them on the device with the same result."""

    input_dtype = torch.uint8
    target_dtype = torch.uint8
    num_classes = 21

    def __init__(self, prefix, augmentations=False, seed=0, mean=VOC_MEAN, std=VOC_STD):
        super().__init__()
        self.images = _open(f"{prefix}_images.npy")
        self.masks = _open(f"{prefix}_masks.npy")
        if self.images.ndim != 4 or self.images.shape[3] != 3 or self.masks.shape != self.images.shape[:3]:
            raise ValueError(f"voc_segmentation_shard: images {self.images.shape} and masks {self.masks.shape} are not "
                             "(N, H, W, 3) and (N, H, W)")
        self.augmentations = bool(augmentations)
        self.rng = random.Random(seed)
        self.mean, self.std = tuple(mean), tuple(std)

    @staticmethod
    def draw_augmentation(rng):
        """One sample's (flip, rot, bright) from ``rng`` with exactly the ``random.random()`` calls of the reference's
        ``apply_augmentations`` (utils/dataset_VOC.py:150-168), in its order and under its conditions (3 to 5 draws):
        flip 1 = hflip; rot +1 / -1 = rotate(+10) / rotate(-10); bright +1 / -1 = brightness 1.2 / 1.2 - 0.4; 0 = none."""
        flip = int(rng.random() > 0.5)
        rot = 0
        if rng.random() > 0.5:
            rot = -1 if rng.random() > 0.5 else 1
        bright = 0
        if rng.random() > 0.5:
            bright = -1 if rng.random() > 0.5 else 1
        return flip, rot, bright

    def __getitem__(self, index):
        img, mask = self.images[index], self.masks[index]
        if self.augmentations:
            img, mask = voc_augment_u8(img, mask, self.draw_augmentation(self.rng))
        return voc_normalize_u8(img, mask, self.mean, self.std)

    def __len__(self):
        return self.images.shape[0]

    def read_into(self, index, x_out, y_out):
        x_out[...] = self.images[index]
        y_out[...] = self.masks[index]

    def sample_shapes(self):
        return tuple(self.images.shape[1:]), tuple(self.masks.shape[1:])


# ------------------------------------------------------------------------------------------------ loader
def shard_indices(indices, rank, world, drop_last=False, disjoint=False):
    """This rank's share of ``indices`` with ``DistributedSampler`` semantics: padded by wrapping around (or truncated
    with ``drop_last``) to a multiple of ``world``, then strided ``rank::world``.  Every rank gets the same count.

    ``disjoint=True`` gives every index to exactly one rank instead (validation and test sets, where a sample counted
    twice would bias the metrics): rank ``r`` takes the contiguous slice ``parallel.shard_range(n, r, world)``, unpadded,
    so the ranks' counts may differ by one and a rank may get none."""
    indices = list(indices)
    n = len(indices)
    if world <= 1:
        return indices
    if disjoint:
        lo, hi = shard_range(n, rank, world)
        return indices[lo:hi]
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
    ``rank`` / ``world``: shard the (shuffled) index list across data-parallel ranks (``shard_indices``): wrap-padded to
    equal counts by default, or, with ``disjoint=True``, each sample on exactly one rank (validation and test sets).
    The yielded tensors are views of a ring slot that is handed back to the filler thread when the NEXT batch is
    requested.  If the consumer only *enqueued* an asynchronous host->device copy of the batch (``TrainSession.step``,
    ``InferenceSession.submit``), it must say when that copy is done: ``loader.guard(event)`` attaches a CUDA event to
    the slot just yielded and the filler thread waits for it before overwriting the slot::

        for x, y in loader:
            sess.step(x, y)
            loader.guard(sess.last_h2d_event())

    The batch buffers take the dataset's ``input_dtype`` / ``target_dtype`` (default float32).  A dataset with
    ``augmentations`` on (``voc_segmentation_shard``) yields ``(x, y, aug)``: ``aug`` (n, 3) int8 holds each sample's
    choices, drawn by ``dataset.draw_augmentation`` from ``augmentation_rng()`` (seeded by ``seed``, the epoch and the rank)
    in the order the samples are loaded, so an epoch's augmentations are reproducible::

        for x, y, aug in loader:
            sess.step(x, y, aug=aug)          # TrainSession(..., input_transform=ops.VOCNormalize())
            loader.guard(sess.last_h2d_event())
    """

    def __init__(self, dataset, batch_size, indices=None, shuffle=False, seed=0, drop_last=True, rank=0, world=1, ring=3,
                 pin_memory=None, disjoint=False):
        self.dataset, self.batch_size = dataset, int(batch_size)
        self.indices = list(range(len(dataset))) if indices is None else list(indices)
        self.shuffle, self.seed, self.drop_last = bool(shuffle), int(seed), bool(drop_last)
        self.rank, self.world, self.ring = int(rank), int(world), max(2, int(ring))
        self.disjoint = bool(disjoint)
        self.epoch = 0
        pin = torch.cuda.is_available() if pin_memory is None else bool(pin_memory)
        xs, ys = dataset.sample_shapes()
        xdt = getattr(dataset, "input_dtype", torch.float32)       # uint8 for the VOC shard
        ydt = getattr(dataset, "target_dtype", torch.float32)      # int64 class indices for the classification shard
        self._x = [torch.empty((self.batch_size,) + tuple(xs), dtype=xdt, pin_memory=pin) for _ in range(self.ring)]
        self._y = [torch.empty((self.batch_size,) + tuple(ys), dtype=ydt, pin_memory=pin) for _ in range(self.ring)]
        self.augmentations = bool(getattr(dataset, "augmentations", False))
        self._aug = [torch.zeros((self.batch_size, 3), dtype=torch.int8, pin_memory=pin) for _ in range(self.ring)] \
            if self.augmentations else None
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
        return shard_indices(idx, self.rank, self.world, drop_last=False, disjoint=self.disjoint)

    def augmentation_rng(self):
        """The generator this epoch's augmentation choices on this rank are drawn from."""
        return random.Random(f"augment/{self.seed}/{self.epoch}/{self.rank}")

    def __len__(self):
        n = len(shard_indices(self.indices, self.rank, self.world, disjoint=self.disjoint))
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def __iter__(self):
        idx = self.epoch_indices()
        rng = self.augmentation_rng() if self.augmentations else None
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
                        if rng is not None:
                            self._aug[s].numpy()[j] = self.dataset.draw_augmentation(rng)
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
                if self._aug is not None:
                    yield self._x[s][:n], self._y[s][:n], self._aug[s][:n]
                else:
                    yield self._x[s][:n], self._y[s][:n]
        finally:
            self._held = None
            stop.set()
            free.put(0)
            t.join(timeout=5)
