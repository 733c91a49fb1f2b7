"""Epoch time of the training driver (smaat_unet_b200.fit) against the step alone and against the eager loop.

  python tools/bench_fit.py [--samples 1000] [--epochs 3] [--rounds 3] [--batch 16]

On a seeded synthetic (N, 13, 288, 288) train shard held in memory (12 input frames, the target the last), for
UNetDSAttention (SmaAt_UNet(12, 1), k = 2), B = 16, valid_size 0.1, reports per epoch:
  * the driver's epoch wall time (``fit_precipitation``: train steps, validation, checkpoints, history), once with the
    uncaptured serving forward for validation and once with a re-captured InferenceSession;
  * the device time of the same epoch's ``TrainSession.step`` calls alone: the same sequence of batch sizes replayed back to
    back on device-resident batches, CUDA events around it.  The difference to the driver's wall time is the driver's
    loader, validation and checkpoint overhead;
  * the same epoch as an eager loop, what the Lightning route executes minus Lightning: the native blocks through autograd,
    the reference's ``loss_func`` (``mse_loss(sum) / B``), ``PrecipitationMetrics.update``, ``loss.backward()`` and
    ``torch.optim.Adam``, then the eager validation forward.
The three runs alternate within each round; medians and (min-max) over every epoch of every round.  The card's name and
power limit are printed first.
"""
import argparse
import gc
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.nn.functional as TF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import fit as F  # noqa: E402
from smaat_unet_b200.data import PinnedBatchLoader, precipitation_maps_oversampled_shard  # noqa: E402

H = W = 288


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def make_shard(n):
    rng = np.random.default_rng(0)
    a = np.empty((n, 13, H, W), np.float32)
    for i in range(n):
        v = rng.random((12, H, W), dtype=np.float32) ** 3 * np.float32(0.06)
        a[i, :12] = v
        a[i, 12] = v[-1]
    return a


def free():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def step_only_ms(sess, sizes, batch):
    """Device time of one epoch's steps: the epoch's batch sizes back to back on device-resident batches."""
    x = torch.rand((batch,) + sess.in_shape, device=sess.device) * 0.06
    y = torch.rand((batch,) + sess.in_shape[1:], device=sess.device) * 0.06
    for n in sorted(set(sizes)):
        sess.step(x[:n], y[:n])
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for n in sizes:
        sess.step(x[:n], y[:n])
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / 1e3


def driver(shard, a, validation):
    with tempfile.TemporaryDirectory() as out:
        res = F.fit_precipitation("UNetDSAttention", shard, out, batch_size=a.batch, epochs=a.epochs, seed=0,
                                  validation=validation, verbose=False)
        secs = [h["epoch_seconds"] for h in res.history]
        ckpt = [h["checkpoint_seconds"] for h in res.history]
        steps = step_only_ms(res.session, F._EpochLoop._sizes(res.train_loader), a.batch)
    del res
    free()
    return secs, steps, ckpt


def eager(shard, a):
    ds = precipitation_maps_oversampled_shard(shard, 12, 1)
    train_idx, valid_idx = F.train_valid_split(len(ds), 0.1, 0)
    train = PinnedBatchLoader(ds, a.batch, indices=train_idx, shuffle=True, seed=0, drop_last=False)
    valid = PinnedBatchLoader(ds, a.batch, indices=valid_idx, shuffle=True, seed=0, drop_last=False)
    torch.manual_seed(0)
    model = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)
    tm, vm = S.PrecipitationMetrics(), S.PrecipitationMetrics()
    secs = []
    for epoch in range(a.epochs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        model.train()
        train.set_epoch(epoch)
        for x, y in train:
            xd, yd = x.cuda(non_blocking=True), y.cuda(non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            train.guard(ev)
            pred = model(xd)
            loss = TF.mse_loss(pred.squeeze(1), yd, reduction="sum") / yd.size(0)     # regression_lightning.py:57-65
            tm.update(pred.detach(), yd)
            opt.zero_grad()
            loss.backward()
            opt.step()
        model.eval()
        valid.set_epoch(epoch)
        with torch.no_grad():
            for x, y in valid:
                xd, yd = x.cuda(non_blocking=True), y.cuda(non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                valid.guard(ev)
                pred = model(xd)
                TF.mse_loss(pred.squeeze(1), yd, reduction="sum") / yd.size(0)
                vm.update(pred, yd)
        tm.compute()
        vm.compute()
        tm.reset()
        vm.reset()
        torch.cuda.synchronize()
        secs.append(time.perf_counter() - t0)
    del model, opt
    free()
    return secs


def fmt(vals):
    return f"{statistics.median(vals):.3f} s ({min(vals):.3f}-{max(vals):.3f})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=1000)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fit: needs a GPU")
    print(card(), flush=True)
    shard = make_shard(a.samples)
    n_train = len(shard) - int(np.floor(0.1 * len(shard)))
    print(f"UNetDSAttention k=2, B={a.batch}, 12x{H}x{W}, {a.samples} samples ({n_train} train), {a.epochs} epochs x "
          f"{a.rounds} rounds", flush=True)
    runs = {"driver (serving validation)": [], "driver (captured validation)": [], "eager loop": []}
    steps, ckpts = [], []
    for r in range(a.rounds):
        for mode in ("serving", "captured"):
            s, st, ck = driver(shard, a, mode)
            runs[f"driver ({mode} validation)"] += s
            steps.append(st)
            ckpts += ck
        runs["eager loop"] += eager(shard, a)
        print(f"round {r}: " + "; ".join(f"{k} {', '.join(f'{v:.3f}' for v in vals[-a.epochs:])}" for k, vals in runs.items()),
              flush=True)
    print(f"TrainSession.step alone, one epoch of batches: {fmt(steps)}")
    print(f"driver's checkpoint files (best and last, written to a temporary directory): {fmt(ckpts)} per epoch")
    for k, vals in runs.items():
        print(f"{k}: epoch {fmt(vals)}")
    base = statistics.median(steps)
    for k in ("driver (serving validation)", "driver (captured validation)"):
        m = statistics.median(runs[k])
        print(f"{k}: overhead over the steps {m - base:.3f} s per epoch ({(m - base) / m * 100:.1f} % of the epoch)")
    print(f"eager loop / driver (serving validation): {statistics.median(runs['eager loop']) / statistics.median(runs['driver (serving validation)']):.2f}x")


if __name__ == "__main__":
    main()
