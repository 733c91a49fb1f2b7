"""Class-map serving timings: InferenceSession(output="logits") + torch.argmax against InferenceSession(output="classes"),
alternated rounds, medians, with the card's name and power limit.

    python tools/bench_classes.py [--rounds 7] [--iters 10]

For SmaAt_UNet(3, 21) at B = 8, 3x224x224 (VOC) and SmaAt_UNet(12, 8) at B = 32, 12x288x288 (the rain-bucket classifier):
  dev_logits_argmax      sess.forward(x) on a device-resident batch, then torch.argmax(logits, 1) on the device
  dev_classes            the "classes" session's forward: OutConv + argmax in the last DS conv's epilogue, inside the graph
  dev_classes_unfused    the "classes" session built with ops.set_fused_classify(False): the last conv, OutConv and
                         smaat_argmax_channels_fwd as separate launches inside the graph
  host_logits_devargmax  pinned batch copied in, the logits session's forward, torch.argmax on the device, the map copied back
  host_classes           submit(pinned x) / collect() of the "classes" session (only the int64 map crosses PCIe)
  host_classes_unfused   the same for the unfused class session
and the last DS conv alone (up4's second conv: 64 -> 64 channels, k = 2): smaat_dsconv_outconv_fwd (one class) against
smaat_dsconv_classify_fwd with K classes, with and without the logits output, and against the unfused route (smaat_dsconv_fwd,
smaat_outconv_fwd, smaat_argmax_channels_fwd), so the per-class epilogue cost is visible.
Each round runs every variant once, in turn; device variants are timed with CUDA events, host variants with the host clock
around work that ends in a synchronise.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

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


def timed_host(fn, iters):
    """Mean ms per call, host clock; every call ends in a synchronise (collect())."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        fn()
    return (time.perf_counter() - t0) * 1e3 / iters


def variants_for(n_ch, K, B, HW):
    torch.manual_seed(K)
    m = S.SmaAt_UNet(n_ch, K).cuda().eval()
    x = torch.rand(B, n_ch, HW, HW, device="cuda")
    xh = x.cpu().pin_memory()
    sl = InferenceSession(m, B, (n_ch, HW, HW))
    sc = InferenceSession(m, B, (n_ch, HW, HW), output="classes")
    ops.set_fused_classify(False)         # the same class map through the unfused last conv, OutConv and argmax kernel
    su = InferenceSession(m, B, (n_ch, HW, HW), output="classes")
    ops.set_fused_classify(True)
    map_host = torch.empty((B, HW, HW), dtype=torch.int64, pin_memory=True)
    sink = {}

    def dev_logits_argmax():
        sink["a"] = torch.argmax(sl.forward(x), 1)

    def dev_classes():
        sink["b"] = sc.forward(x)

    def dev_classes_unfused():
        sink["h"] = su.forward(x)

    def host_logits_devargmax():
        # the logits route done well: pinned batch in, torch.argmax on the device, only the map copied back
        xd = xh.to("cuda", non_blocking=True)
        map_host.copy_(torch.argmax(sl.forward(xd), 1), non_blocking=True)
        torch.cuda.synchronize()

    def host_classes():
        sc.submit(xh)
        sink["d"] = sc.collect()

    def host_classes_unfused():
        su.submit(xh)
        sink["i"] = su.collect()

    # the last DS conv alone, at its own shape
    g = torch.Generator().manual_seed(1)
    y = torch.rand(B, 64, HW, HW, generator=g).cuda()
    dw_w, dw_b = (torch.rand(128, 1, 3, 3, generator=g) - 0.5).cuda(), (torch.rand(128, generator=g) - 0.5).cuda() * 0.1
    pw_w = ((torch.rand(64, 128, 1, 1, generator=g) - 0.5) * 0.2).cuda()
    sc_, sh_ = (torch.rand(64, generator=g) + 0.5).cuda(), (torch.rand(64, generator=g) - 0.5).cuda() * 0.2
    ow, ob = ((torch.rand(K, 64, generator=g) - 0.5) * 0.4).cuda(), (torch.rand(K, generator=g) - 0.5).cuda() * 0.2
    split = ops.split_tf32(pw_w.view(64, -1))
    args = (y, dw_w, dw_b, 2, pw_w, sc_, sh_, True)

    def conv_outconv_1():
        sink["e"] = ops.dsconv(*args, w_split=split, outconv=(ow[:1].contiguous(), ob[:1]))

    def conv_classify():
        sink["f"] = ops.dsconv_classify(*args, ow, ob, w_split=split)

    def conv_classify_logits():
        sink["g"] = ops.dsconv_classify(*args, ow, ob, w_split=split, want_logits=True)

    def conv_unfused_classes():
        a = ops.dsconv(*args, w_split=split)
        sink["j"] = ops.argmax_channels(ops.outconv(a, ow, ob))

    host = {"host_logits_devargmax": host_logits_devargmax, "host_classes": host_classes, "host_classes_unfused": host_classes_unfused}
    dev = {"dev_logits_argmax": dev_logits_argmax, "dev_classes": dev_classes, "dev_classes_unfused": dev_classes_unfused,
           "last_conv_outconv_1class": conv_outconv_1,
           "last_conv_classify": conv_classify, "last_conv_classify_with_logits": conv_classify_logits,
           "last_conv_unfused_outconv_argmax": conv_unfused_classes}
    extra = {"d2h_bytes_logits": sl.d2h_bytes_per_step, "d2h_bytes_classes": sc.d2h_bytes_per_step,
             "launches_per_forward": {"logits": sl.launches_per_forward, "classes": sc.launches_per_forward}}
    with torch.no_grad():
        cls = sc.forward(x).clone()
        lg = sl.forward(x)
        extra["pixels_differing_from_argmax_of_logits"] = int((cls != lg.argmax(1)).sum())
        extra["unfused_route_equals_argmax_of_logits"] = bool(torch.equal(su.forward(x), lg.argmax(1)))
    return dev, host, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_classes.py times the GPU path: it needs a CUDA device"
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "rounds": a.rounds, "iters": a.iters, "pointwise_mode": S.get_pointwise_mode()}
    with torch.no_grad():
        for tag, cfg in CONFIGS.items():
            dev, host, extra = variants_for(*cfg)
            fns = {**{k: (f, timed_dev) for k, f in dev.items()}, **{k: (f, timed_host) for k, f in host.items()}}
            for f, _ in fns.values():          # warm-up
                for _ in range(3):
                    f()
            res = {k: [] for k in fns}
            for _ in range(a.rounds):
                for k, (f, timer) in fns.items():
                    res[k].append(timer(f, a.iters))
            out[tag] = {"median_ms": {k: statistics.median(v) for k, v in res.items()},
                        "spread_pct": {k: 100.0 * (max(v) - min(v)) / statistics.median(v) for k, v in res.items()}, **extra}
            del dev, host
            torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
