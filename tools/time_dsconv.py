"""Time the fused DS conv alone at bench.py's shapes with Cout <= 128 (B = 32, 3xTF32, k = 2), with CUDA events (a tool, not a
test).

For each shape it times two entry points over the same tiles, main loop and affine:
  smaat_dsconv_fwd          writes the Cout-channel activation (the layer as the forward runs it);
  smaat_dsconv_outconv_fwd  writes one float per pixel (the fused 1-class OutConv) instead of Cout.
Their difference bounds what the output stores cost.  Each timing is 5 warm-up launches, then 40 launches between two CUDA
events.  `hbm_ms` is the algorithmic HBM floor: input + output bytes at 3.35 TB/s (H100 SXM data sheet).

With --cbam it times instead the serving forward's CBAM fusions (smaat_dsconv_cbam_fwd) against the plain fused conv on the same
tiles: the second DS conv of inc / down1 / down2 with and without the epilogue pools (partial sums / maxima + 2x2 max-pool), and
the first DS conv of up4 / up3 / up2 with and without the gate applied on load.

With --wide it times instead bench.py's three 256-channel layers (down2.0, down2.1, up2.0 at 72^2; up2.0 also with the CBAM
gate on load) as wide tiles and in two 128-channel passes (ops.set_dsconv_wide), the two alternated --rounds times; medians,
beside each layer's HBM floor and its tensor floor (the issued tf32 MMA flops, 3 per product in 3xTF32, at the data-sheet
495 TFLOP/s).

  python tools/time_dsconv.py [--tree DIR] [--mode tf32x3|tf32] [--json] [--cbam | --wide [--rounds N]]

--tree imports smaat_unet_b200 from another checkout (a built one), to compare two builds in one session."""
import argparse
import json
import os
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--mode", default="tf32x3", choices=["tf32", "tf32x3"])
ap.add_argument("--json", action="store_true", help="one JSON line per shape instead of a table")
ap.add_argument("--cbam", action="store_true", help="time the CBAM fusions (epilogue pools, gate on load) instead")
ap.add_argument("--wide", action="store_true", help="time the 256-channel layers as wide tiles and in two passes instead")
ap.add_argument("--rounds", type=int, default=3, help="--wide: alternated rounds per route")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))

import torch  # noqa: E402

from smaat_unet_b200 import _lib, ops  # noqa: E402

B, K_PL = 32, 2
# (C0, C1, S, Cout): C1 > 0 is Up's concat, read virtually.  Each runs once per SmaAt-UNet forward
SHAPES = [
    (12, 0, 288, 64),
    (64, 0, 288, 64),
    (64, 64, 288, 64),
    (64, 0, 144, 128),
    (128, 0, 144, 128),
    (128, 128, 144, 128),
    (128, 0, 144, 64),
    (256, 0, 72, 128),
]
WARMUP, ITERS = 5, 40
HBM_BPS = 3.35e12


def timed(fn):
    for _ in range(WARMUP):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / ITERS


# (C0, C1, S, Cout, what): producers of the CBAM level 1-3 maps (pools) and the up-block convs reading them (gate)
CBAM_SHAPES = [
    (64, 0, 288, 64, "pools"),
    (128, 0, 144, 128, "pools"),
    (256, 0, 72, 256, "pools"),
    (64, 64, 288, 64, "gate"),
    (128, 128, 144, 128, "gate"),
    (256, 256, 72, 256, "gate"),
]


def main_cbam():
    g = torch.Generator(device="cuda").manual_seed(7)
    rows = []
    for C0, C1, S, Cout, what in CBAM_SHAPES:
        Cin = C0 + C1
        K = K_PL * Cin
        x0 = torch.rand(B, C0, S, S, device="cuda", generator=g)
        x1 = torch.rand(B, C1, S, S, device="cuda", generator=g) if C1 else None
        dw_w = torch.randn(K, 1, 3, 3, device="cuda", generator=g) * 0.3
        dw_b = torch.randn(K, device="cuda", generator=g) * 0.1
        pw_w = torch.randn(Cout, K, device="cuda", generator=g) * 0.1
        scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
        shift = torch.randn(Cout, device="cuda", generator=g) * 0.1
        split = ops.split_tf32(pw_w) if args.mode == "tf32x3" else None
        gate = (torch.rand(B, C0, device="cuda", generator=g), torch.rand(B, 1, S, S, device="cuda", generator=g)) if what == "gate" else None
        common = (dw_w, dw_b, K_PL, pw_w, scale, shift, True)
        ms_plain = timed(lambda: ops.dsconv(x0, *common, x1=x1, mode=args.mode, w_split=split))
        ms_fused = timed(lambda: ops.dsconv_cbam(x0, *common, x1=x1, mode=args.mode, w_split=split, gate=gate, pools=what == "pools"))
        name = f"C{Cin}->{Cout} {S}^2" + (" (concat)" if C1 else "")
        rows.append({"layer": name, "fusion": what, "plain_ms": round(ms_plain, 4), "fused_ms": round(ms_fused, 4),
                     "extra_ms": round(ms_fused - ms_plain, 4)})
        del x0, x1
    dev = torch.cuda.get_device_name()
    if args.json:
        for r in rows:
            print(json.dumps(r))
        print(json.dumps({"device": dev, "mode": args.mode}))
        return
    print(f"{dev}, {args.mode}, B = {B}, k = {K_PL}; {WARMUP} warm-up + {ITERS} timed launches each")
    print(f"{'layer':28s} {'fusion':>6s} {'plain ms':>9s} {'fused ms':>9s} {'extra ms':>9s}")
    for r in rows:
        print(f"{r['layer']:28s} {r['fusion']:>6s} {r['plain_ms']:9.3f} {r['fused_ms']:9.3f} {r['extra_ms']:9.3f}")


# (C0, C1, S, Cout, gated): bench.py's layers with 128 < Cout <= 256
WIDE_SHAPES = [
    (128, 0, 72, 256, False),
    (256, 0, 72, 256, False),
    (256, 256, 72, 256, False),
    (256, 256, 72, 256, True),
]
TF32_FLOPS = 495e12


def main_wide():
    g = torch.Generator(device="cuda").manual_seed(7)
    rows = []
    for C0, C1, S, Cout, gated in WIDE_SHAPES:
        Cin = C0 + C1
        K = K_PL * Cin
        x0 = torch.rand(B, C0, S, S, device="cuda", generator=g)
        x1 = torch.rand(B, C1, S, S, device="cuda", generator=g) if C1 else None
        dw_w = torch.randn(K, 1, 3, 3, device="cuda", generator=g) * 0.3
        dw_b = torch.randn(K, device="cuda", generator=g) * 0.1
        pw_w = torch.randn(Cout, K, device="cuda", generator=g) * 0.1
        scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
        shift = torch.randn(Cout, device="cuda", generator=g) * 0.1
        split = ops.split_tf32(pw_w) if args.mode == "tf32x3" else None
        gate = (torch.rand(B, C0, device="cuda", generator=g), torch.rand(B, 1, S, S, device="cuda", generator=g)) if gated else None
        common = (dw_w, dw_b, K_PL, pw_w, scale, shift, True)
        fn = lambda: ops.dsconv_cbam(x0, *common, x1=x1, mode=args.mode, w_split=split, gate=gate)
        times = {True: [], False: []}
        for _ in range(args.rounds):
            for wide in (False, True):
                ops.set_dsconv_wide(wide)
                times[wide].append(timed(fn))
        ops.set_dsconv_wide(True)
        med = {w: sorted(t)[len(t) // 2] for w, t in times.items()}
        hbm = 4.0 * B * S * S * (Cin + Cout) / HBM_BPS * 1e3
        mma = (3 if args.mode == "tf32x3" else 1) * 2.0 * B * S * S * K * Cout / TF32_FLOPS * 1e3
        name = f"C{Cin}->{Cout} {S}^2" + (" (concat)" if C1 else "") + (" gated" if gated else "")
        rows.append({"layer": name, "two_pass_ms": round(med[False], 4), "wide_ms": round(med[True], 4),
                     "change": round(med[True] / med[False] - 1, 4), "hbm_ms": round(hbm, 4), "tensor_ms": round(mma, 4),
                     "two_pass_runs": [round(t, 4) for t in times[False]], "wide_runs": [round(t, 4) for t in times[True]]})
        del x0, x1
    dev = torch.cuda.get_device_name()
    if args.json:
        for r in rows:
            print(json.dumps(r))
        print(json.dumps({"device": dev, "mode": args.mode, "rounds": args.rounds}))
        return
    print(f"{dev}, {args.mode}, B = {B}, k = {K_PL}; {args.rounds} alternated rounds of {WARMUP} warm-up + {ITERS} timed launches")
    print(f"{'layer':32s} {'two-pass ms':>11s} {'wide ms':>8s} {'change':>7s} {'HBM floor':>9s} {'tensor floor':>12s}")
    for r in rows:
        print(f"{r['layer']:32s} {r['two_pass_ms']:11.3f} {r['wide_ms']:8.3f} {100 * r['change']:6.1f}% {r['hbm_ms']:9.3f} "
              f"{r['tensor_ms']:12.3f}")


def main():
    assert torch.cuda.is_available(), "time_dsconv.py needs a GPU"
    if args.cbam:
        return main_cbam()
    if args.wide:
        return main_wide()
    lib = _lib.load()
    mode = ops.PW_MODES[args.mode]
    g = torch.Generator(device="cuda").manual_seed(7)
    p = ops._ptr
    st = ops._stream()
    rows = []
    for C0, C1, S, Cout in SHAPES:
        Cin = C0 + C1
        K = K_PL * Cin
        x0 = torch.rand(B, C0, S, S, device="cuda", generator=g)
        x1 = torch.rand(B, C1, S, S, device="cuda", generator=g) if C1 else None
        dw_w = torch.randn(K, 1, 3, 3, device="cuda", generator=g) * 0.3
        dw_b = torch.randn(K, device="cuda", generator=g) * 0.1
        pw_w = torch.randn(Cout, K, device="cuda", generator=g) * 0.1
        scale = torch.rand(Cout, device="cuda", generator=g) + 0.5
        shift = torch.randn(Cout, device="cuda", generator=g) * 0.1
        oc_w = torch.randn(Cout, device="cuda", generator=g) * 0.1
        oc_b = torch.randn(1, device="cuda", generator=g)
        hi, lo = ops.split_tf32(pw_w) if args.mode == "tf32x3" else (pw_w, None)
        y = torch.empty(B, Cout, S, S, device="cuda")
        logits = torch.empty(B, 1, S, S, device="cuda")
        bs0, bs1 = C0 * S * S, C1 * S * S

        def fwd():
            _lib.check(lib.smaat_dsconv_fwd(p(x0), C0, bs0, p(x1), C1, bs1, p(dw_w), p(dw_b), p(hi), p(lo), p(scale), p(shift),
                                            p(y), Cout * S * S, None, B, S, S, K_PL, Cout, 1, mode, st), "smaat_dsconv_fwd")

        def outconv():
            _lib.check(lib.smaat_dsconv_outconv_fwd(p(x0), C0, bs0, p(x1), C1, bs1, p(dw_w), p(dw_b), p(hi), p(lo), p(scale),
                                                    p(shift), p(oc_w), p(oc_b), p(logits), B, S, S, K_PL, Cout, 1, mode, st),
                       "smaat_dsconv_outconv_fwd")

        ms_fwd = timed(fwd)
        ms_oc = timed(outconv)
        hbm = 4.0 * B * S * S * (Cin + Cout) / HBM_BPS * 1e3
        name = f"C{Cin}->{Cout} {S}^2" + (" (concat)" if C1 else "")
        rows.append({"layer": name, "fwd_ms": round(ms_fwd, 4), "outconv_ms": round(ms_oc, 4), "gap_ms": round(ms_fwd - ms_oc, 4),
                     "hbm_ms": round(hbm, 4)})
        del x0, x1, y
    total_gap = sum(r["gap_ms"] for r in rows)
    dev = torch.cuda.get_device_name()
    if args.json:
        for r in rows:
            print(json.dumps(r))
        print(json.dumps({"device": dev, "mode": args.mode, "sum_fwd_ms": round(sum(r["fwd_ms"] for r in rows), 4),
                          "sum_gap_ms": round(total_gap, 4)}))
        return
    print(f"{dev}, {args.mode}, B = {B}, k = {K_PL}; {WARMUP} warm-up + {ITERS} timed launches per entry point")
    print(f"{'layer':28s} {'fwd ms':>8s} {'outconv ms':>10s} {'gap ms':>8s} {'HBM floor ms':>12s}")
    for r in rows:
        print(f"{r['layer']:28s} {r['fwd_ms']:8.3f} {r['outconv_ms']:10.3f} {r['gap_ms']:8.3f} {r['hbm_ms']:12.3f}")
    print(f"sum of gaps (each layer runs once per forward): {total_gap:.3f} ms")


if __name__ == "__main__":
    main()
