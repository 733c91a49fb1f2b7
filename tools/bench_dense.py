"""Dense baselines (UNet, UNetAttention) on one GPU: H100 drop-ins vs the torch port on cuDNN.

    python tools/bench_dense.py [--batch 32] [--size 288] [--iters 10]

Run from the repository root after build().  Prints one line per measurement with the GPU name and power limit, plus the
per-layer times of the 18 dense 3x3 convs and of their weight gradients (CUDA events).  Achieved TFLOP/s use the shape-derived forward work of the
reference modules (102.06 GFLOP per 12 x 288 x 288 frame, scaled by area); tf32x3 also reports the issued MMA work (3x).
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import smaat_unet_b200 as S                                   # noqa: E402
from oracle import dense_oracle as D                          # noqa: E402
from smaat_unet_b200 import ops                               # noqa: E402
from smaat_unet_b200.engine import InferenceSession           # noqa: E402
from smaat_unet_b200.train import TrainSession                # noqa: E402

GFLOP_288 = 102.06


def gpu_label():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        pl = "unknown"
    return f"{name}, power limit {pl or 'unknown'}"


def timed(fn, iters, warmup=2):
    """ms per call, wall clock between device synchronisations (the sessions enqueue on their own streams)."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=288)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    B, Sz = a.batch, a.size
    gf = GFLOP_288 * (Sz / 288) ** 2
    label = gpu_label()
    torch.manual_seed(0)
    x = torch.rand(B, 12, Sz, Sz, device="cuda")

    def report(what, ms, mult=1):
        fps = B / (ms / 1e3)
        extra = f", issued {mult * fps * gf / 1e3:.1f} TFLOP/s" if mult != 1 else ""
        print(f"{what:46s} {ms:9.2f} ms  {fps:8.1f} frames/s  {fps * gf / 1e3:6.1f} TFLOP/s{extra}   [{label}]", flush=True)

    for cls in (S.UNet, S.UNetAttention):
        m = cls(12, 1).cuda().eval()
        sd = {k: v.detach().clone() for k, v in m.state_dict().items()}
        for mode in ("tf32x3", "tf32"):
            ops.set_pointwise_mode(mode)
            sess = InferenceSession(m, B, (12, Sz, Sz))
            y = sess.forward(x)
            torch.backends.cudnn.allow_tf32 = mode == "tf32"
            torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
            with torch.no_grad():
                ref = D.port_unet_forward(x[:2], sd, attention=cls is S.UNetAttention)
            err = float((y[:2] - ref).abs().max() / ref.abs().max())
            assert err < (2e-2 if mode == "tf32" else 1e-3), (cls.__name__, mode, err)
            report(f"{cls.__name__} forward, InferenceSession, {mode}", timed(sess.replay, a.iters), 3 if mode == "tf32x3" else 1)
            del sess
        for allow in (True, False):
            torch.backends.cudnn.allow_tf32 = allow
            torch.backends.cuda.matmul.allow_tf32 = allow
            with torch.no_grad():
                ms = timed(lambda: D.port_unet_forward(x, sd, attention=cls is S.UNetAttention), a.iters)
            report(f"{cls.__name__} forward, torch port cuDNN allow_tf32={allow}", ms)
        del m
        torch.cuda.empty_cache()

    ops.set_pointwise_mode("tf32x3")
    m = S.UNet(12, 1).cuda().train()
    sess = TrainSession(m, B, (12, Sz, Sz), lr=1e-4)
    xt, yt = torch.rand(B, 12, Sz, Sz, device="cuda"), torch.rand(B, Sz, Sz, device="cuda")
    report("UNet train step, TrainSession, tf32x3", timed(lambda: sess.step(xt, yt), max(2, a.iters // 3), warmup=1), 3)
    sess.close()
    del sess, m
    torch.cuda.empty_cache()

    # per-layer forward conv times (eager eval forward under ops.profile)
    for mode in ("tf32x3", "tf32"):
        ops.set_pointwise_mode(mode)
        m = S.UNet(12, 1).cuda().eval()
        with torch.no_grad():
            m(x)
            with ops.profile() as prof:
                m(x)
        print(f"per-layer 3x3 conv forward, {mode}, B={B}  [{label}]")
        for k, v in prof.summary(by_shape=True).items():
            if k.startswith("smaat_conv3x3"):
                print(f"  {k:52s} {v['launches']:2d} x  {v['ms'] / v['launches']:8.3f} ms  {v['flops'] / v['ms'] / 1e9:7.1f} TFLOP/s")
        del m

    # per-layer weight-gradient times (eager train-mode forward + backward)
    for mode in ("tf32x3", "tf32"):
        ops.set_pointwise_mode(mode)
        m = S.UNet(12, 1).cuda().train()
        m(x).sum().backward()
        with ops.profile() as prof:
            m(x).sum().backward()
        print(f"per-layer 3x3 conv weight gradient, {mode}, B={B}  [{label}]")
        for k, v in prof.summary(by_shape=True).items():
            if k.startswith("smaat_conv3x3_bwd_weight"):
                print(f"  {k:52s} {v['launches']:2d} x  {v['ms'] / v['launches']:8.3f} ms  {v['flops'] / v['ms'] / 1e9:7.1f} TFLOP/s")
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
