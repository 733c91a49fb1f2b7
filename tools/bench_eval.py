"""Test-set evaluation throughput: evaluate_precipitation against the batch-1 loop of the reference's script.

  python tools/bench_eval.py [--samples N] [--batch1-samples M] [--rounds R]

On a seeded synthetic (N, 18, 288, 288) test shard held in memory, for the persistence baseline plus SmaAt_UNet(12, 1)
k = 2, UNetDS(12, 1) k = 2, UNetDSAttention4CBAMs(12, 1) k = 2, UNet(12, 1) and UNetAttention(12, 1) (tf32x3, eval), reports:
  * samples/s of the evaluator's loop (``evaluate.score_batches``: B = 32, six thresholds 0.5 / 1 / 2 / 5 / 10 / 30, every
    model, one pass from the pinned loader to the final ``compute()``), on sessions captured beforehand;
  * samples/s of what calc_metrics_test_set.py amounts to on the same native models: one sample at a time, the eager
    forward (plain module calls) and one ``PrecipitationMetrics`` update per threshold, over the first M samples;
  * ``smaat_precip_sweep_fwd`` alone at B = 32, 288^2 for T = 1 and T = 6, model-output and strided persistence reads:
    device time (CUDA events over 200 launches) and GB/s against its floor of 8 bytes per pixel.
Medians over R rounds.  The card's name and power limit are printed first.
"""
import argparse
import ctypes
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200.data import PinnedBatchLoader  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402
from smaat_unet_b200.evaluate import evaluate_precipitation, score_batches  # noqa: E402

TH = (0.5, 1.0, 2.0, 5.0, 10.0, 30.0)
H = W = 288


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def models():
    torch.manual_seed(0)
    out = {"PersistenceModel": S.PersistenceModel(), "SmaAt-UNet": S.SmaAt_UNet(12, 1, kernels_per_layer=2),
           "UNetDS": S.UNetDS(12, 1, kernels_per_layer=2),
           "UNetDS Attention 4CBAMs": S.UNetDSAttention4CBAMs(12, 1, kernels_per_layer=2),
           "UNet": S.UNet(12, 1), "UNet Attention": S.UNetAttention(12, 1)}
    for m in out.values():
        for mod in m.modules():
            if isinstance(mod, S.OutConv):
                torch.nn.init.normal_(mod.conv.weight, 0, 0.002)
                torch.nn.init.constant_(mod.conv.bias, 0.005)
    return {k: m.cuda().eval() for k, m in out.items()}


def shard(n):
    rng = np.random.default_rng(0)
    a = np.empty((n, 18, H, W), np.float32)
    for i in range(n):
        v = rng.random((18, H, W), dtype=np.float32) ** 3 * np.float32(0.06)
        v[rng.random((18, H, W), dtype=np.float32) < 0.5] = 0
        a[i] = v
    return S.precipitation_maps_oversampled_shard(a, 12, 6, train=False)


def batch1_loop(ms, ds, m):
    mets = {name: [S.PrecipitationMetrics(threshold=t) for t in TH] for name in ms}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        for i in range(m):
            x, y = ds[i]
            xd = torch.from_numpy(x).cuda()[None]
            yd = torch.from_numpy(y).cuda()[None]
            for name, model in ms.items():
                pred = model(xd)
                for met in mets[name]:
                    met.update(pred, yd)
    torch.cuda.synchronize()
    return m / (time.perf_counter() - t0)


def sweep_kernel(T, persistence, iters=200):
    B, P = 32, H * W
    x = torch.rand(B, 12, H, W, device="cuda") * 0.06
    y = torch.rand(B, H, W, device="cuda") * 0.06
    src = x if persistence else x[:, :1].contiguous()
    pred, bstride = (src.data_ptr() + 11 * P * 4, 12 * P) if persistence else (src.data_ptr(), P)
    per = torch.empty(B, 3, dtype=torch.float64, device="cuda")
    hist = torch.empty(B, T + 1, T + 1, dtype=torch.int32, device="cuda")
    thr = (ctypes.c_float * T)(*TH[:T])
    lib = S._lib.load()

    def launch():
        S._lib.check(lib.smaat_precip_sweep_fwd(pred, bstride, y.data_ptr(), B, P, 47.83, thr, T, 1, per.data_ptr(),
                                                hist.data_ptr(), torch.cuda.current_stream().cuda_stream), "sweep")
    for _ in range(10):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        launch()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return ms, 8 * B * P / (ms * 1e-3) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=192)
    ap.add_argument("--batch1-samples", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    print(card(), flush=True)
    ms = models()
    ds = shard(a.samples)
    evaluate_precipitation(ms, ds, batch=32, thresholds=TH)          # one full pass, as a user runs it (warm-up)
    # the timed passes run the evaluator's loop on sessions captured once, so capture time is not in the rate
    sessions = {name: InferenceSession(m, 32, (12, H, W)) for name, m in ms.items() if not isinstance(m, S.PersistenceModel)}
    loader = PinnedBatchLoader(ds, 32, drop_last=False)
    ev, b1 = [], []
    for _ in range(a.rounds):
        accs = {name: S.PrecipitationMetricsSweep(TH) for name in ms}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        score_batches(loader, sessions, accs, torch.device("cuda", 0))
        for acc in accs.values():
            acc.compute()                                                # ends in a device -> host copy
        ev.append(a.samples / (time.perf_counter() - t0))
        b1.append(batch1_loop(ms, ds, a.batch1_samples))
    evm, b1m = statistics.median(ev), statistics.median(b1)
    print(f"evaluate_precipitation (B=32, 6 thresholds, 6 models incl. persistence): {evm:.1f} samples/s "
          f"(rounds {', '.join(f'{v:.1f}' for v in ev)})")
    print(f"batch-1 loop (eager forward + 6 PrecipitationMetrics per model): {b1m:.1f} samples/s "
          f"(rounds {', '.join(f'{v:.1f}' for v in b1)});  speed-up {evm / b1m:.1f}x")
    for T in (1, 6):
        for pers in (False, True):
            t, gbs = sweep_kernel(T, pers)
            print(f"smaat_precip_sweep_fwd B=32 288^2 T={T} {'persistence (strided)' if pers else 'model output'}: "
                  f"{t * 1e3:.1f} us, {gbs:.0f} GB/s of 8 B/px")


if __name__ == "__main__":
    main()
