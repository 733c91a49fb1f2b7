"""Probability serving timings: InferenceSession(output="logits") + torch.softmax against InferenceSession(output="probs"),
alternated rounds, medians and spread, with the card's name and power limit.

    python tools/bench_probs.py [--rounds 7] [--iters 10]

For SmaAt_UNet(3, 21) at B = 8, 3x224x224 (VOC) and SmaAt_UNet(12, 8) at B = 32, 12x288x288 (the rain-bucket classifier):
  dev_logits_softmax     sess.forward(x) on a device-resident batch, then torch.softmax(logits, 1) on the device
  dev_probs              the "probs" session's forward: the last conv, OutConv and smaat_softmax_channels_fwd inside the graph
the last DS conv alone (up4's second conv: 64 -> 64 channels, k = 2): smaat_dsconv_classify_fwd (class map only) against the
probability route (smaat_dsconv_fwd, smaat_outconv_fwd, smaat_softmax_channels_fwd); and smaat_softmax_channels_fwd alone on
(B, K, H, W) logits against its HBM floor (8 K bytes per pixel: the logits read once, the probabilities written once), with
torch.softmax beside it.
Each round runs every variant once, in turn, timed with CUDA events.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402

CONFIGS = {"voc_3x224_k21_b8": (3, 21, 8, 224), "rain_12x288_k8_b32": (12, 8, 32, 288)}


def card():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        limit = float(out.splitlines()[0])
    except Exception:
        pass
    return name, limit


def timed_dev(fn, iters):
    """Mean ms per call, CUDA events around `iters` calls, synchronised at both ends."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def variants_for(n_ch, K, B, HW):
    torch.manual_seed(K)
    m = S.SmaAt_UNet(n_ch, K).cuda().eval()
    x = torch.rand(B, n_ch, HW, HW, device="cuda")
    sl = InferenceSession(m, B, (n_ch, HW, HW))
    sp = InferenceSession(m, B, (n_ch, HW, HW), output="probs")
    sink = {}

    def dev_logits_softmax():
        sink["a"] = torch.softmax(sl.forward(x), 1)

    def dev_probs():
        sink["c"] = sp.forward(x)

    # the last DS conv alone, at its own shape
    g = torch.Generator().manual_seed(1)
    y = torch.rand(B, 64, HW, HW, generator=g).cuda()
    dw_w, dw_b = (torch.rand(128, 1, 3, 3, generator=g) - 0.5).cuda(), (torch.rand(128, generator=g) - 0.5).cuda() * 0.1
    pw_w = ((torch.rand(64, 128, 1, 1, generator=g) - 0.5) * 0.2).cuda()
    sc_, sh_ = (torch.rand(64, generator=g) + 0.5).cuda(), (torch.rand(64, generator=g) - 0.5).cuda() * 0.2
    ow, ob = ((torch.rand(K, 64, generator=g) - 0.5) * 0.4).cuda(), (torch.rand(K, generator=g) - 0.5).cuda() * 0.2
    split = ops.split_tf32(pw_w.view(64, -1))
    args = (y, dw_w, dw_b, 2, pw_w, sc_, sh_, True)

    def conv_classify():
        sink["d"] = ops.dsconv_classify(*args, ow, ob, w_split=split)

    def conv_unfused_probs():
        a = ops.dsconv(*args, w_split=split)
        sink["f"] = ops.softmax_channels(ops.outconv(a, ow, ob))

    # the softmax kernel alone on logits of the model's output shape
    lg = torch.randn(B, K, HW, HW, generator=g).cuda() * 4.0

    def softmax_kernel():
        sink["g"] = ops.softmax_channels(lg)

    def softmax_torch():
        sink["h"] = torch.softmax(lg, 1)

    dev = {"dev_logits_softmax": dev_logits_softmax, "dev_probs": dev_probs, "last_conv_classify": conv_classify,
           "last_conv_unfused_outconv_softmax": conv_unfused_probs, "softmax_channels_kernel": softmax_kernel,
           "torch_softmax": softmax_torch}
    extra = {"d2h_bytes_logits": sl.d2h_bytes_per_step, "d2h_bytes_probs": sp.d2h_bytes_per_step,
             "launches_per_forward": {"logits": sl.launches_per_forward, "probs": sp.launches_per_forward},
             "softmax_hbm_bytes": 8 * K * B * HW * HW}
    with torch.no_grad():
        p = sp.forward(x).clone()
        pt = torch.softmax(sl.forward(x), 1)
        extra["max_abs_diff_probs_vs_logits_torch_softmax"] = float((p - pt).abs().max())
    return dev, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_probs.py times the GPU path: it needs a CUDA device"
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "rounds": a.rounds, "iters": a.iters, "pointwise_mode": S.get_pointwise_mode()}
    with torch.no_grad():
        for tag, cfg in CONFIGS.items():
            dev, extra = variants_for(*cfg)
            for f in dev.values():          # warm-up
                for _ in range(3):
                    f()
            res = {k: [] for k in dev}
            for _ in range(a.rounds):
                for k, f in dev.items():
                    res[k].append(timed_dev(f, a.iters))
            med = {k: statistics.median(v) for k, v in res.items()}
            out[tag] = {"median_ms": med,
                        "spread_pct": {k: 100.0 * (max(v) - min(v)) / statistics.median(v) for k, v in res.items()},
                        "softmax_channels_gbps": extra["softmax_hbm_bytes"] / med["softmax_channels_kernel"] / 1e6, **extra}
            del dev
            torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
