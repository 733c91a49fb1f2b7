"""Dataset creation throughput: the GPU rain-pixel scan of create_datasets against the reference's per-frame numpy scan.

  python tools/bench_create_datasets.py [--frames N] [--chunk C] [--rounds R]

On a seeded synthetic 288^2 frame shard pair (<prefix>_train.npy with 80 % of N frames, <prefix>_test.npy with the rest;
each frame rains on a fraction of its pixels drawn from a spread: most frames nearly dry, some half covered), written to a
temporary directory by this run (so the page cache holds it: the scan figures are warm-cache figures), reports:
  * pinned host-to-device bandwidth: a (C, 288, 288) pinned buffer copied to the device, CUDA events over 20 copies;
  * ``smaat_rain_pixels_fwd`` alone on device-resident frames: C frames per launch and all N in one launch, CUDA events
    over 50 launches, frames/s and GB/s over its 4 B/px floor;
  * ``scan_rain_pixels`` end to end (memory map -> pinned ring -> side-stream copy -> count, counts read back once):
    frames/s and GB/s, medians over R rounds;
  * the reference's scan (create_datasets.py:79-82): ``np.sum(images[i] > 0)`` for one frame at a time from the same
    memory map, medians over R rounds;
  * ``create_datasets`` end to end for thresholds 0.2 and 0.5 and both splits (scan, selection and writing the shards into
    the same temporary directory), once; the bytes written and the samples kept.
The card's name and power limit are printed first.  Nothing is written outside the temporary directory, which is removed.
"""
import argparse
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from smaat_unet_b200 import create_datasets as CD  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402

SIZE = 288


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def write_frames(path, n, rng, block=128):
    """n seeded frames, written `block` at a time: per frame a rain fraction (75 % of frames below 0.15, 15 % in
    0.15-0.45, 10 % in 0.45-0.9), rain values in (0, 1], dry pixels 0."""
    out = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=(n, SIZE, SIZE))
    for f0 in range(0, n, block):
        m = min(block, n - f0)
        kind = rng.random(m)
        frac = np.where(kind < 0.75, rng.uniform(0, 0.15, m), np.where(kind < 0.9, rng.uniform(0.15, 0.45, m),
                                                                     rng.uniform(0.45, 0.9, m)))
        v = rng.random((m, SIZE, SIZE), dtype=np.float32)
        out[f0:f0 + m] = np.where(v < frac[:, None, None].astype(np.float32), np.float32(1) - v, np.float32(0))
    out.flush()
    del out


def events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=2048)
    ap.add_argument("--chunk", type=int, default=256)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    torch.cuda.set_device(0)
    print(card(), flush=True)
    plane_bytes = SIZE * SIZE * 4
    tmp = tempfile.mkdtemp(prefix="bench_create_datasets_")
    try:
        free = shutil.disk_usage(tmp).free
        print(f"temporary directory: {free / 1e9:.1f} GB free", flush=True)
        n_train = int(a.frames * 0.8)
        sizes = {"train": n_train, "test": a.frames - n_train}
        prefix = os.path.join(tmp, "frames")
        rng = np.random.default_rng(20261019)
        for sp, n in sizes.items():
            write_frames(f"{prefix}_{sp}.npy", n, rng)
        frames = np.load(f"{prefix}_train.npy", mmap_mode="r")
        n = frames.shape[0]
        print(f"shard: {n} + {sizes['test']} frames of {SIZE}x{SIZE} fp32 ({a.frames * plane_bytes / 1e9:.2f} GB); page cache: "
              "warm (the shards were written by this run)", flush=True)

        # pinned host-to-device bandwidth
        c = min(a.chunk, n)
        pinned = torch.empty((c, SIZE, SIZE), dtype=torch.float32, pin_memory=True)
        pinned.numpy()[:] = frames[:c]
        dev = torch.empty_like(pinned, device="cuda")
        ms = events_ms(lambda: dev.copy_(pinned, non_blocking=True), 20)
        h2d = c * plane_bytes / ms / 1e6
        print(f"pinned H2D: {c} frames in {ms:.3f} ms = {h2d:.1f} GB/s", flush=True)

        # the kernel alone
        out = torch.empty((c,), device="cuda", dtype=torch.int32)
        ms = events_ms(lambda: ops.rain_pixel_counts(dev, out=out), 50)
        print(f"smaat_rain_pixels_fwd, {c} device-resident frames per launch: {ms * 1e3:.1f} us = {c / ms * 1e3:,.0f} frames/s, "
              f"{c * plane_bytes / ms / 1e6:.0f} GB/s over 4 B/px", flush=True)
        alldev = torch.from_numpy(np.array(frames)).cuda()
        outall = torch.empty((n,), device="cuda", dtype=torch.int32)
        ms = events_ms(lambda: ops.rain_pixel_counts(alldev, out=outall), 50)
        print(f"smaat_rain_pixels_fwd, all {n} frames in one launch: {ms * 1e3:.1f} us = {n / ms * 1e3:,.0f} frames/s, "
              f"{n * plane_bytes / ms / 1e6:.0f} GB/s over 4 B/px", flush=True)
        want = np.sum(np.asarray(frames) > 0, axis=(1, 2))
        assert np.array_equal(outall.cpu().numpy(), want), "device counts differ from numpy's"
        del alldev, outall

        # scan end to end, and the reference's per-frame numpy scan, alternated
        CD.scan_rain_pixels(frames, a.chunk)
        gpu_s, np_s = [], []
        for _ in range(a.rounds):
            t0 = time.perf_counter()
            got = CD.scan_rain_pixels(frames, a.chunk)
            gpu_s.append(time.perf_counter() - t0)
            assert np.array_equal(got, want)
            t0 = time.perf_counter()
            ref = [np.sum(frames[i] > 0) for i in range(n)]
            np_s.append(time.perf_counter() - t0)
            assert np.array_equal(np.asarray(ref), want)
        g, r = statistics.median(gpu_s), statistics.median(np_s)
        print(f"scan_rain_pixels (memmap -> pinned ring -> H2D -> count), chunk {a.chunk}: {g:.3f} s "
              f"(min {min(gpu_s):.3f}, max {max(gpu_s):.3f}) = {n / g:,.0f} frames/s, {n * plane_bytes / g / 1e9:.2f} GB/s "
              f"(pinned H2D alone: {h2d:.1f} GB/s)", flush=True)
        print(f"reference scan (np.sum(images[i] > 0) per frame, same memmap): {r:.3f} s (min {min(np_s):.3f}, max "
              f"{max(np_s):.3f}) = {n / r:,.0f} frames/s, {n * plane_bytes / r / 1e9:.2f} GB/s; GPU scan {r / g:.1f}x faster",
              flush=True)

        # create_datasets end to end, once
        out_dir = os.path.join(tmp, "out")
        t0 = time.perf_counter()
        files = CD.create_datasets(prefix, out_dir, 12, 6, (0.2, 0.5), chunk=a.chunk)
        e2e = time.perf_counter() - t0
        written = sum(os.path.getsize(p) for d in files.values() for p in d.values())
        print(f"create_datasets, {a.frames} frames, thresholds 0.2 and 0.5, both splits: {e2e:.2f} s, {written / 1e9:.2f} GB of "
              f"shards written ({a.frames / e2e:,.0f} frames/s, output into the temporary directory)", flush=True)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
