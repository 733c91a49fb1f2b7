"""The reference's rain-thresholded precipitation datasets (``create_datasets.py``), built natively from the frame shards.

    python -m smaat_unet_b200.create_datasets --frames-prefix precip --out-dir data/precipitation

The input is what ``data.convert_h5(raw.h5, prefix)`` writes: ``<prefix>_<split>.npy``, (n_images, H, W) float32.  Each
split is read once:

  * **Scan.** ``chunk`` frames at a time go from the memory-mapped shard into a ring of two pinned buffers (the rows
    copied by a few host threads, which a single-threaded copy would leave the bottleneck), cross to the
    device on a side stream, and ``ops.rain_pixel_counts`` (``smaat_rain_pixels_fwd``) counts their rain pixels on the
    compute stream into one device buffer.  The host waits only for the copy out of the pinned buffer it is about to
    refill; the counts come back once per split.
  * **Selection** on the host, from the same counts for every threshold, as the reference decides it
    (create_datasets.py:22-23, :75-82): ``seq = input_length + image_ahead``; frame ``i`` in ``range(seq, n_images)`` is
    kept when ``count[i] >= num_pixels * thresh``, with ``num_pixels = H * H`` (the reference takes ``images.shape[1]``
    as the image size); the sample is ``images[i - seq : i]``, so frame ``i`` itself is not in it and the target
    (``imgs[-1]``) is frame ``i - 1``.
  * **Output.** One ``(samples, seq, H, W)`` float32 ``.npy`` per threshold and split, named with the reference's formula
    (:25-27, ``int(thresh * 100)``, so 0.29 gives 28) plus ``_<split>.npy``; samples in ascending ``i``, values copied bit
    for bit.  Each kept window is read once and written to every threshold's shard that keeps it.
    ``precipitation_maps_oversampled_shard`` reads these shards as they are.

Timestamps are not written: ``convert_h5`` does not keep them and nothing here or in the reference reads them.
"""
from __future__ import annotations

import argparse
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import ops


def dataset_file_name(input_length, image_ahead, thresh, split):
    """The reference's file name (create_datasets.py:25-27) with ``_<split>.npy`` in place of ``.h5``."""
    return (f"train_test_2016-2019_input-length_{input_length}_img-ahead_{image_ahead}_rain-threshold_"
            f"{int(thresh * 100)}_{split}.npy")


def _open_frames(path):
    frames = np.load(path, mmap_mode="r", allow_pickle=False)
    if frames.ndim != 3 or frames.dtype != np.float32:
        raise ValueError(f"create_datasets: {path} must hold (n_images, H, W) float32 frames, got {frames.dtype} {frames.shape}")
    return frames


def select_indices(counts, input_length, image_ahead, thresh, img_size):
    """Frames ``i`` whose window ``images[i - seq : i]`` the reference keeps: ``i >= seq`` and
    ``count[i] >= img_size * img_size * thresh`` (a Python float; every count below 2^53 compares exactly as a float64)."""
    seq = input_length + image_ahead
    counts = np.asarray(counts)
    bound = img_size * img_size * float(thresh)
    idx = np.arange(seq, counts.shape[0])
    return idx[counts[seq:].astype(np.float64) >= bound]


def write_split(frames, counts, out_dir, split, input_length=12, image_ahead=6, thresholds=(0.2, 0.5)):
    """Write every threshold's shard of one split from its frames ((n_images, H, W) array or memmap) and their rain-pixel
    counts.  Returns ``{thresh: (path, samples)}`` and the bytes written."""
    seq = input_length + image_ahead
    n, H, W = frames.shape
    keep = {t: select_indices(counts, input_length, image_ahead, t, H) for t in thresholds}
    outs, rows = {}, {}
    for t in thresholds:
        path = os.path.join(out_dir, dataset_file_name(input_length, image_ahead, t, split))
        outs[t] = (path, np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=(len(keep[t]), seq, H, W)))
        rows[t] = 0
    union = np.unique(np.concatenate([keep[t] for t in thresholds])) if thresholds else np.zeros(0, np.int64)
    members = {t: np.isin(union, keep[t]) for t in thresholds}
    nbytes = 0
    for j, i in enumerate(union):
        window = np.asarray(frames[i - seq:i])        # read once, written to every shard that keeps frame i
        for t in thresholds:
            if members[t][j]:
                outs[t][1][rows[t]] = window
                rows[t] += 1
                nbytes += window.nbytes
    res = {}
    for t in thresholds:
        path, arr = outs[t]
        arr.flush()
        res[t] = (path, rows[t])
    return res, nbytes


def _fill(pool, k, dst, src):
    """dst[:] = src, the rows split across k threads of the pool (numpy copies run without the GIL, and the memory map's
    page faults are taken in parallel)."""
    bounds = [len(src) * j // k for j in range(k + 1)]
    list(pool.map(lambda j: dst.__setitem__(slice(bounds[j], bounds[j + 1]), src[bounds[j]:bounds[j + 1]]), range(k)))


def scan_rain_pixels(frames, chunk=256, device=None, workers=None):
    """Rain-pixel count of every frame of an (n_images, H, W) float32 array / memmap, on the GPU: ``chunk`` frames at a
    time through two pinned buffers (filled by ``workers`` host threads), the copy on a side stream, the count on the
    current stream.  Returns (n_images,) int64 on the host."""
    if not torch.cuda.is_available():
        raise RuntimeError("create_datasets: counting rain pixels needs a CUDA device; there is no CPU fallback")
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    n, H, W = frames.shape
    chunk = max(1, min(int(chunk), n))
    workers = max(1, min(8, os.cpu_count() or 1) if workers is None else int(workers))
    with torch.cuda.device(device), ThreadPoolExecutor(workers) as pool:
        compute = torch.cuda.current_stream()
        side = torch.cuda.Stream()
        counts = torch.empty((n,), device=device, dtype=torch.int32)
        pinned = [torch.empty((chunk, H, W), dtype=torch.float32, pin_memory=True) for _ in range(2)]
        staged = [torch.empty((chunk, H, W), dtype=torch.float32, device=device) for _ in range(2)]
        copied = [None, None]        # the H2D copy out of pinned[s] / into staged[s]
        counted = [None, None]       # the count that read staged[s]
        for c, f0 in enumerate(range(0, n, chunk)):
            s, m = c % 2, min(chunk, n - f0)
            if copied[s] is not None:
                copied[s].synchronize()                  # pinned[s] is free again
            _fill(pool, workers, pinned[s].numpy()[:m], frames[f0:f0 + m])
            with torch.cuda.stream(side):
                if counted[s] is not None:
                    side.wait_event(counted[s])          # staged[s] was read by the count two chunks ago
                staged[s][:m].copy_(pinned[s][:m], non_blocking=True)
                copied[s] = torch.cuda.Event()
                copied[s].record(side)
            compute.wait_event(copied[s])
            ops.rain_pixel_counts(staged[s][:m], out=counts[f0:f0 + m])
            counted[s] = torch.cuda.Event()
            counted[s].record(compute)
        host = counts.cpu()                              # the split's one wait for the device
    return host.numpy().astype(np.int64)


def create_datasets(frames_prefix, out_dir, input_length=12, image_ahead=6, thresholds=(0.2, 0.5), splits=("train", "test"),
                    chunk=256, verbose=True):
    """Build the reference's oversampled datasets for every threshold from ``<frames_prefix>_<split>.npy``.  Returns
    ``{thresh: {split: path}}``.  Raises ``ValueError`` before any work when a split's frames are not square or the splits
    differ in size (the reference writes (samples, seq, imgSize, imgSize) with imgSize = H)."""
    thresholds = tuple(dict.fromkeys(float(t) for t in thresholds))
    if len({int(t * 100) for t in thresholds}) < len(thresholds):
        raise ValueError(f"create_datasets: thresholds {thresholds} share a file name (rain-threshold_{{int(t * 100)}})")
    if int(input_length) < 0 or int(image_ahead) < 0 or int(input_length) + int(image_ahead) < 1:
        raise ValueError(f"create_datasets: input_length {input_length} and image_ahead {image_ahead} give no window")
    frames = {sp: _open_frames(f"{frames_prefix}_{sp}.npy") for sp in splits}
    shapes = {sp: f.shape[1:] for sp, f in frames.items()}
    for sp, (H, W) in shapes.items():
        if H != W:
            raise ValueError(f"create_datasets: frames of split {sp!r} are {H}x{W}; the reference's datasets hold square "
                             "frames (imgSize x imgSize with imgSize = H)")
    if len(set(shapes.values())) > 1:
        raise ValueError(f"create_datasets: the splits' frame sizes differ: {shapes}")
    os.makedirs(out_dir, exist_ok=True)
    files = {t: {} for t in thresholds}
    for sp, fr in frames.items():
        t0 = time.perf_counter()
        counts = scan_rain_pixels(fr, chunk)
        t1 = time.perf_counter()
        res, nbytes = write_split(fr, counts, out_dir, sp, input_length, image_ahead, thresholds)
        t2 = time.perf_counter()
        for t, (path, _) in res.items():
            files[t][sp] = path
        if verbose:
            kept = ", ".join(f"{res[t][1]} at {t:g}" for t in thresholds)
            print(f"{sp}: {fr.shape[0]} frames scanned in {t1 - t0:.2f} s; samples kept: {kept}; "
                  f"{nbytes} bytes written in {t2 - t1:.2f} s", flush=True)
    return files


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="Create the rain-thresholded precipitation datasets (the reference's "
                                "create_datasets.py) from the frame shards of data.convert_h5, counting rain pixels on the GPU")
    p.add_argument("--frames-prefix", required=True, help="reads <prefix>_<split>.npy, (n_images, H, W) float32")
    p.add_argument("--out-dir", required=True, help="where the (samples, seq, H, W) shards go")
    p.add_argument("--input-length", type=int, default=12)
    p.add_argument("--image-ahead", type=int, default=6)
    p.add_argument("--thresholds", type=float, nargs="+", default=[0.2, 0.5],
                   help="fractions of rain pixels the target frame needs (one shard per threshold and split)")
    p.add_argument("--splits", nargs="+", default=["train", "test"])
    p.add_argument("--chunk", type=int, default=256, help="frames per host-to-device copy")
    return p.parse_args(argv)


def main(argv=None):
    a = parse_args(argv)
    return create_datasets(a.frames_prefix, a.out_dir, a.input_length, a.image_ahead, a.thresholds, a.splits, a.chunk)


if __name__ == "__main__":
    main()
