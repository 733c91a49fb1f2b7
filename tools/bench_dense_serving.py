"""Dense-network serving timings: the OutConv (+ argmax / softmax) in the last 3x3 conv's epilogue against the separate launches,
alternated rounds, medians and spread, with the card's name and power limit.

    python tools/bench_dense_serving.py [--rounds 7] [--iters 10]

For UNet(12, 1) at B = 32, 12x288x288 (logits) and UNet(3, 21) / UNetAttention(3, 21) at B = 8, 3x224x224 (logits, class map,
probabilities), in tf32 and tf32x3:
  session_<output>_fused     InferenceSession(output=...).forward on a device-resident batch, built with
                             ops.set_fused_dense_head(True): up4's last conv applies OutConv (and the argmax / softmax) in its
                             epilogue, inside the graph
  session_<output>_unfused   the same session with the default ops.set_fused_dense_head(False): the last conv, OutConv and the
                             argmax / softmax kernel as separate launches inside the graph
  last_conv_<output>_fused / _unfused   up4's last conv alone (64 -> 64 channels at the full resolution), fused and unfused
Each round runs every variant once, in turn, timed with CUDA events.  The fused and unfused outputs are compared bit for bit on
the timed inputs.  Writes nothing.
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

# tag: (model class, n_channels, n_classes, B, H = W, outputs)
CONFIGS = {"unet_12x288_k1_b32": (S.UNet, 12, 1, 32, 288, ("logits",)),
           "unet_3x224_k21_b8": (S.UNet, 3, 21, 8, 224, ("logits", "classes", "probs")),
           "unet_attention_3x224_k21_b8": (S.UNetAttention, 3, 21, 8, 224, ("logits", "classes", "probs"))}


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


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def variants_for(cls, n_ch, K, B, HW, outputs):
    torch.manual_seed(K)
    m = cls(n_ch, K).cuda().eval()
    with torch.no_grad():
        m.outc.conv.weight.mul_(50.0)           # spread the logits over the classes
    x = torch.rand(B, n_ch, HW, HW, device="cuda")
    sink, dev, extra = {}, {}, {"launches_per_forward": {}, "bit_identical": {}}
    for o in outputs:
        ops.set_fused_dense_head(True)
        sf = InferenceSession(m, B, (n_ch, HW, HW), output=o)
        ops.set_fused_dense_head(False)
        su = InferenceSession(m, B, (n_ch, HW, HW), output=o)
        dev[f"session_{o}_fused"] = lambda sf=sf, o=o: sink.__setitem__(o + "f", sf.forward(x))
        dev[f"session_{o}_unfused"] = lambda su=su, o=o: sink.__setitem__(o + "u", su.forward(x))
        extra["launches_per_forward"][o] = {"fused": sf.launches_per_forward, "unfused": su.launches_per_forward}
        extra["bit_identical"][f"session_{o}"] = bool(torch.equal(_bits(sf.forward(x).clone()), _bits(su.forward(x).clone())))

    # up4's last conv alone: 64 -> 64 channels at the full resolution, the model's own OutConv
    dc = m.up4.conv
    g = torch.Generator().manual_seed(1)
    y = torch.rand(B, 64, HW, HW, generator=g).cuda()
    s1, t1 = dc._folded(3)
    wp, hi, lo = dc.packed(3, 64)
    split = (hi, lo) if hi is not None else None
    ow, ob = m.outc.conv.weight.detach(), m.outc.conv.bias.detach()
    args = (y, wp, 64, s1, t1, True, ow, ob)

    def unfused(o):
        lg = ops.outconv(ops.conv3x3(y, wp, 64, s1, t1, True, w_split=split), ow, ob)
        return lg if o == "logits" else (ops.argmax_channels(lg) if o == "classes" else ops.softmax_channels(lg))

    def fused(o):
        if o == "probs":
            return ops.conv3x3_probs(*args, w_split=split)
        return ops.conv3x3_classify(*args, w_split=split, want_logits=o == "logits", want_classes=o == "classes")

    for o in outputs:
        dev[f"last_conv_{o}_fused"] = lambda o=o: sink.__setitem__("cf", fused(o))
        dev[f"last_conv_{o}_unfused"] = lambda o=o: sink.__setitem__("cu", unfused(o))
        extra["bit_identical"][f"last_conv_{o}"] = bool(torch.equal(_bits(fused(o)), _bits(unfused(o))))
    return dev, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--modes", default="tf32,tf32x3")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_serving.py times the GPU path: it needs a CUDA device"
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "rounds": a.rounds, "iters": a.iters}
    with torch.no_grad():
        for mode in a.modes.split(","):
            ops.set_pointwise_mode(mode)
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
                out[f"{tag}_{mode}"] = {"median_ms": med,
                                        "spread_pct": {k: 100.0 * (max(v) - min(v)) / statistics.median(v) for k, v in res.items()},
                                        **extra}
                del dev
                torch.cuda.empty_cache()
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()
