"""Data-parallel epoch time of the training driver, the same epoch as bare steps, the loader alone, and evaluate's rate.

  torchrun --nproc-per-node G tools/bench_fit_multi.py [--samples 4400] [--distinct 256] [--epochs 3] [--test-samples 2048]
  python tools/bench_fit_multi.py ...          # one GPU, no process group

Run it once per GPU count (1, 2, 4, 8): every rank runs the same program and rank 0 prints the card's name and power limit,
the GPU count, then one JSON line.  The workload is ``fit precip``'s: UNetDSAttention (SmaAt_UNet(12, 1), k = 2),
``batch_size`` 16 per rank, 12 x 288 x 288 inputs, valid_size 0.1, over a seeded synthetic shard of ``--samples`` samples
(4 400 by default: 3 960 train samples, so every rank of 8 runs 31 steps; the same shard at every GPU count, so the epoch
times compare as strong scaling).  The shard repeats ``--distinct`` seeded samples (a 4.3 MB .npy each, memory-mapped
from a temporary directory and shared through the page cache), so the loader copies 4.3 MB per sample as it would from a
real shard without the benchmark writing GBs.  Reported, as the slowest rank's times:
  * ``loader``: one epoch of every rank's train loader alone, all ranks at once, no GPU work: samples/s per rank and in
    all; whether the host feeds the GPUs;
  * ``driver``: ``fit_precipitation``'s epoch time (``history.jsonl``'s ``epoch_seconds``: steps, validation, epoch-end
    reductions, rank 0's checkpoint files, barrier), median over the epochs after the first;
  * ``steps``: the same epoch's batch sizes through the driver's own ``TrainSession.step`` (NCCL all-reduce included) on
    device-resident batches, host clock after a synchronise and a barrier; ``driver - steps`` is the driver's cost;
  * ``evaluate``: ``evaluate_precipitation`` with the persistence baseline and SmaAt-UNet over ``--test-samples`` samples
    (batch 32 per rank), samples/s of the whole call, session capture included, second of two calls.
"""
import argparse
import json
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

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import evaluate as E  # noqa: E402
from smaat_unet_b200 import fit as F  # noqa: E402
from smaat_unet_b200 import parallel as P  # noqa: E402
from smaat_unet_b200.data import PinnedBatchLoader, precipitation_maps_oversampled_shard  # noqa: E402

H = W = 288
BATCH = 16


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"unknown ({e})"
    return name, q


class Tiled:
    """``n`` samples of an (distinct, T, H, W) array, sample i being row i % distinct: a shard-shaped array for the
    datasets of smaat_unet_b200.data."""

    def __init__(self, base, n):
        self.base, self.shape = base, (int(n),) + tuple(base.shape[1:])

    def __getitem__(self, i):
        return self.base[int(i) % self.base.shape[0]]


def make_distinct(path, n):
    rng = np.random.default_rng(0)
    a = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=(n, 13, H, W))
    for i in range(n):
        v = rng.random((12, H, W), dtype=np.float32) ** 3 * np.float32(0.06)
        a[i, :12] = v
        a[i, 12] = v[-1]
    a.flush()
    del a


def loader_rate(shard, rank, world, dev):
    ds = precipitation_maps_oversampled_shard(shard, 12, 1)
    train_idx, _ = F.train_valid_split(len(ds), 0.1, 0)
    loader = PinnedBatchLoader(ds, BATCH, indices=train_idx, shuffle=True, seed=0, drop_last=False, rank=rank, world=world)
    P.barrier(dev)
    t0 = time.perf_counter()
    n = sum(int(b[0].shape[0]) for b in loader)
    dt = P.reduce_max(time.perf_counter() - t0, dev)
    return n, dt


def step_seconds(sess, sizes, dev):
    x = torch.rand((BATCH,) + sess.in_shape, device=dev) * 0.06
    y = torch.rand((BATCH,) + sess.in_shape[1:], device=dev) * 0.06
    for n in sorted(set(sizes)):
        sess.step(x[:n], y[:n])
    P.barrier(dev)
    t0 = time.perf_counter()
    for n in sizes:
        sess.step(x[:n], y[:n])
    torch.cuda.synchronize(dev)
    return P.reduce_max(time.perf_counter() - t0, dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=4400)
    ap.add_argument("--distinct", type=int, default=256)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3, help="timed repetitions of the bare step epoch")
    ap.add_argument("--test-samples", type=int, default=2048)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fit_multi: needs a GPU")
    with P.process_group_from_env() as (rank, world, local):
        dev = torch.device("cuda", local)
        torch.cuda.set_device(dev)
        name, limit = card()
        tmp = P.broadcast_from_rank0(tempfile.mkdtemp(prefix="bench_fit_multi_") if rank == 0 else None, dev)
        try:
            path = os.path.join(tmp, "distinct.npy")
            if rank == 0:
                print(f"{name}, power limit / max SM clock: {limit}; {world} GPU(s)", flush=True)
                make_distinct(path, a.distinct)
            P.barrier(dev)
            base = np.load(path, mmap_mode="r")
            shard = Tiled(base, a.samples)
            n_loaded, t_loader = loader_rate(shard, rank, world, dev)

            res = F.fit_precipitation("UNetDSAttention", shard, os.path.join(tmp, "out"), batch_size=BATCH, epochs=a.epochs,
                                      seed=0, verbose=False)
            epochs = [P.reduce_max(h["epoch_seconds"], dev) for h in res.history]
            sizes = F._EpochLoop._sizes(res.train_loader)
            steps = [step_seconds(res.session, sizes, dev) for _ in range(a.rounds)]
            res.session.close()
            del res
            torch.cuda.empty_cache()

            test = precipitation_maps_oversampled_shard(Tiled(base, a.test_samples), 12, 6, train=False)
            torch.manual_seed(0)
            models = {E.PERSISTENCE: S.PersistenceModel(), "UNetDSAttention": S.SmaAt_UNet(12, 1, kernels_per_layer=2)}
            evals = []
            for _ in range(2):
                P.barrier(dev)
                t0 = time.perf_counter()
                E.evaluate_precipitation(models, test, batch=32, device=dev)
                evals.append(P.reduce_max(time.perf_counter() - t0, dev))
            driver = statistics.median(epochs[1:] or epochs)
            step = statistics.median(steps)
            out = {"card": name, "power_limit_max_sm_clock": limit, "gpus": world, "batch_per_rank": BATCH,
                   "samples": a.samples, "steps_per_rank": len(sizes), "step_sizes": sorted(set(sizes)),
                   "loader_samples_per_s_per_rank": n_loaded / t_loader, "loader_samples_per_s": world * n_loaded / t_loader,
                   "driver_epoch_s": driver, "driver_epochs_s": epochs, "steps_epoch_s": step, "steps_epochs_s": steps,
                   "driver_overhead_s": driver - step, "train_samples_per_s": world * sum(sizes) / driver,
                   "evaluate_samples_per_s": a.test_samples / evals[-1], "evaluate_calls_s": evals}
            if rank == 0:
                print(json.dumps(out), flush=True)
        finally:
            P.barrier(dev)
            if rank == 0:
                shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
