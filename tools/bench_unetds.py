"""UNetDS and UNetDSAttention4CBAMs (12, 1), k = 2, B = 32, 12 x 288 x 288: the fused DS conv's max-pool epilogue per layer, and
the whole networks, reference-order plain calls against the native serving session.

  layers    UNetDS's producing convs inc.1, down1.1, down2.1, down3.1 alone, in tf32x3 (fp32 maps) and with bf16 storage (bf16
            maps; the max-pool in the dtype of the level it feeds): 'epilogue' (one launch writing y and its max-pool), 'plain'
            (the conv alone) and 'standalone' (the conv, then the max-pool kernel: smaat_maxpool2_fwd for fp32 maps; for bf16
            maps the project has no standalone pool, so torch's max_pool2d stands in).  A conv the fused kernel does not take
            is reported as such
  networks  'plain' (model(x): the reference's plain calls in its order, eager, tf32x3), 'session' (InferenceSession replay,
            tf32x3), 'session_bf16' (InferenceSession(dtype=torch.bfloat16) replay) and, for UNetDS, 'session_no_epilogue'
            (tf32x3 with the max-pool epilogue declined, so down1-down4 pool with smaat_maxpool2_fwd)

Each setup is timed with CUDA events over --reps launches (or replays) per round, the setups alternated over --rounds rounds;
the report gives the median and the min-max spread in ms.  The card name and power limit are read in the same run.  Writes
one JSON document to --out and prints it.

    python tools/bench_unetds.py --out /tmp/unetds.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402

B, SHAPE = 32, (12, 288, 288)
# (layer, Cin, Cout, H): the convs whose output the next DownDS pools; the max-pool dtype with bf16 storage
LAYERS = [("inc.1", 64, 64, 288, torch.bfloat16), ("down1.1", 128, 128, 144, torch.bfloat16),
          ("down2.1", 256, 256, 72, torch.float32), ("down3.1", 512, 512, 36, torch.float32)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def alternate(setups, rounds, reps):
    for fn in setups.values():          # warm-up: caches, algorithms, graph uploads
        fn()
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in setups}
    for _ in range(rounds):
        for k, fn in setups.items():
            times[k].append(timed(fn, reps))
    return {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in times.items()}


def layer_setups(Cin, Cout, H, pdt, bf16):
    g = torch.Generator(device="cuda").manual_seed(Cin + H)
    x = torch.randn((B, Cin, H, H), generator=g, device="cuda")
    K = 2 * Cin
    w, b = torch.randn((K, 1, 3, 3), generator=g, device="cuda") / 3, torch.randn((K,), generator=g, device="cuda") * 0.1
    pw = torch.randn((Cout, K), generator=g, device="cuda") * K ** -0.5
    sc, sh = torch.rand((Cout,), generator=g, device="cuda") + 0.5, torch.randn((Cout,), generator=g, device="cuda") * 0.1
    if bf16:
        xb, pack = x.to(torch.bfloat16), (ops.pack_bf16(pw), None)
        if not ops.dsconv_maxpool_bf16_takes(xb, None, pw, 2):
            return None
        return {
            "epilogue": lambda: ops.dsconv_maxpool_bf16(xb, w, b, 2, pw, sc, sh, True, w_split=pack, pooled_dtype=pdt),
            "plain": lambda: ops.dsconv_bf16(xb, w, b, 2, pw, sc, sh, True, w_split=pack),
            "standalone": lambda: F.max_pool2d(ops.dsconv_bf16(xb, w, b, 2, pw, sc, sh, True, w_split=pack), 2).to(pdt),
        }
    split = ops.split_tf32(pw)
    if not ops.dsconv_maxpool_takes(x, None, pw, 2, "tf32x3"):
        return None
    return {
        "epilogue": lambda: ops.dsconv_maxpool(x, w, b, 2, pw, sc, sh, True, mode="tf32x3", w_split=split),
        "plain": lambda: ops.dsconv(x, w, b, 2, pw, sc, sh, True, mode="tf32x3", w_split=split),
        "standalone": lambda: ops.maxpool2(ops.dsconv(x, w, b, 2, pw, sc, sh, True, mode="tf32x3", w_split=split)),
    }


def net_setups(ctor, x):
    torch.manual_seed(0)
    model = ctor().cuda().eval()
    out = {}
    nograd = torch.no_grad()

    def plain():
        with nograd:
            model(x)
    out["plain"] = plain
    s = InferenceSession(model, B, SHAPE)
    out["session"] = lambda: s.forward(x)
    sb = InferenceSession(model, B, SHAPE, dtype=torch.bfloat16)
    xb = x.to(torch.bfloat16)
    out["session_bf16"] = lambda: sb.forward(xb)
    if isinstance(model, S.UNetDS):
        real = ops.dsconv_maxpool_takes
        ops.dsconv_maxpool_takes = lambda *a, **k: False
        try:
            sn = InferenceSession(model, B, SHAPE)
        finally:
            ops.dsconv_maxpool_takes = real
        out["session_no_epilogue"] = lambda: sn.forward(x)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_unetds needs a GPU"
    ops.set_pointwise_mode("tf32x3")
    res = {"card": card(), "batch": B, "shape": SHAPE, "rounds": a.rounds, "reps": a.reps, "layers": {}, "networks": {}}
    for name, Cin, Cout, H, pdt in LAYERS:
        for storage in ("tf32x3", "bf16"):
            setups = layer_setups(Cin, Cout, H, pdt, storage == "bf16")
            key = f"{name}_{storage}"
            res["layers"][key] = "not taken by the fused kernel" if setups is None else alternate(setups, a.rounds, 5 * a.reps)
            print(key, res["layers"][key], flush=True)
    x = torch.rand((B,) + SHAPE, generator=torch.Generator(device="cuda").manual_seed(1), device="cuda")
    for name, ctor in (("UNetDS_12_1", lambda: S.UNetDS(12, 1, kernels_per_layer=2)),
                       ("UNetDSAttention4CBAMs_12_1", lambda: S.UNetDSAttention4CBAMs(12, 1, kernels_per_layer=2))):
        res["networks"][name] = alternate(net_setups(ctor, x), a.rounds, a.reps)
        print(name, res["networks"][name], flush=True)
        torch.cuda.empty_cache()
    doc = json.dumps(res, indent=1)
    print(doc)
    if a.out:
        with open(a.out, "w") as f:
            f.write(doc)


if __name__ == "__main__":
    main()
