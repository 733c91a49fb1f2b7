"""tf32x3 / tf32 / bf16 side by side, alternated within every round (the three arithmetic modes of the tensor-core GEMMs).

  python tools/bench_precision.py [--rounds R] [--iters N]

Reports, for each mode, the median over the rounds and the spread ((max - min) / median) of:
  * each fused DS conv layer of bench.py's network (SmaAt_UNet(12, 1, kernels_per_layer=2), B = 32, 12 x 288 x 288, eval
    epilogue), the pointwise GEMMs of the layers the fused kernel declines (36 x 36, 18 x 18) and UNet(12, 1)'s dense 3x3
    convs, each timed alone (CUDA events over N launches) with its GEMM's achieved TFLOP/s;
  * InferenceSession per batch: SmaAt_UNet(12, 1) logits (k = 2, B = 32, 288^2), SmaAt_UNet(3, 21) classes (B = 8, 224^2) and
    UNet(12, 1) logits (B = 32, 288^2);
  * one SmaAt_UNet(12, 1) TrainSession step (B = 32, 288^2; its weight gradients run tf32 kernels in bf16 mode).
The card's name and power limit are printed first: an absolute number is only worth something with them.
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402
from smaat_unet_b200.train import TrainSession  # noqa: E402

MODES = ("tf32x3", "tf32", "bf16")
KPL = 2
# (name, C0, C1, Cout, S) of bench.py's network (tests/test_gpu_ds_forward_kernels.py LAYERS)
DS_LAYERS = [
    ("inc.0", 12, 0, 64, 288), ("inc.1", 64, 0, 64, 288), ("down1.0", 64, 0, 128, 144), ("down1.1", 128, 0, 128, 144),
    ("down2.0", 128, 0, 256, 72), ("down2.1", 256, 0, 256, 72), ("down3.0", 256, 0, 512, 36), ("down3.1", 512, 0, 512, 36),
    ("down4.0", 512, 0, 512, 18), ("down4.1", 512, 0, 512, 18), ("up1.0", 512, 512, 512, 36), ("up1.1", 512, 0, 256, 36),
    ("up2.0", 256, 256, 256, 72), ("up2.1", 256, 0, 128, 72), ("up3.0", 128, 128, 128, 144), ("up3.1", 128, 0, 64, 144),
    ("up4.0", 64, 64, 64, 288), ("up4.1", 64, 0, 64, 288),
]
# (C0, C1, Cout, S) of UNet(12, 1)'s tensor-core 3x3 convs (down4's 18 x 18 ones run on the CUDA cores in every mode)
DENSE = [(12, 0, 64, 288), (64, 0, 64, 288), (64, 0, 128, 144), (128, 0, 128, 144), (128, 0, 256, 72), (256, 0, 256, 72),
         (256, 0, 512, 36), (512, 0, 512, 36), (512, 512, 256, 36), (256, 256, 128, 72), (128, 128, 64, 144), (64, 64, 64, 288)]
B = 32


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:       # the number still needs its card: say what is missing
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def time_fn(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def layer_cases():
    """(label, GEMM flops, {mode: callable}) per timed layer; the weight operands are prepared outside the timed call."""
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for name, C0, C1, Cout, H in DS_LAYERS:
        Cin = C0 + C1
        K = KPL * Cin
        x = torch.randn((B, Cin, H, H), generator=g, device="cuda")
        x0, x1 = (x[:, :C0].contiguous(), x[:, C0:].contiguous()) if C1 else (x, None)
        w = torch.randn((K, 1, 3, 3), generator=g, device="cuda") / 3
        b = torch.randn((K,), generator=g, device="cuda") * 0.1
        pw = torch.randn((Cout, K), generator=g, device="cuda") * K ** -0.5
        sc, sh = torch.rand(Cout, generator=g, device="cuda") + 0.5, torch.randn(Cout, generator=g, device="cuda") * 0.1
        fns = {}
        fused = ops.dsconv_takes(x0, x1, pw, KPL, "tf32x3")
        for mode in MODES:
            wops = ops.weight_operands(pw, ops.PW_MODES[mode])
            if fused:
                assert ops.dsconv_takes(x0, x1, pw, KPL, mode), (name, mode)
                fns[mode] = (lambda x0=x0, x1=x1, w=w, b=b, pw=pw, sc=sc, sh=sh, mode=mode, wops=wops:
                             ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=wops))
            else:
                d = torch.randn((B, K, H, H), generator=g, device="cuda") if mode == MODES[0] else d
                fns[mode] = (lambda d=d, pw=pw, sc=sc, sh=sh, mode=mode, wops=wops:
                             ops.pw1x1(d, pw, sc, sh, True, mode=mode, w_split=wops))
        out.append((f"{'dsconv' if fused else 'pw1x1 '} {name:8s} {Cin:4d}->{Cout:4d} S{H}", 2.0 * B * H * H * K * Cout, fns))
        del x
    for C0, C1, Cout, H in DENSE:
        x = torch.randn((B, C0 + C1, H, H), generator=g, device="cuda")
        x0, x1 = (x[:, :C0].contiguous(), x[:, C0:].contiguous()) if C1 else (x, None)
        w = torch.randn((Cout, C0 + C1, 3, 3), generator=g, device="cuda") * (9 * (C0 + C1)) ** -0.5
        wp = ops.conv3x3_pack_weight(w, C0, C1)
        sc, sh = torch.rand(Cout, generator=g, device="cuda") + 0.5, torch.randn(Cout, generator=g, device="cuda") * 0.1
        fns = {}
        for mode in MODES:
            wops = ops.weight_operands(wp, ops.PW_MODES[mode])
            fns[mode] = (lambda x0=x0, x1=x1, wp=wp, sc=sc, sh=sh, mode=mode, wops=wops, Cout=Cout:
                         ops.conv3x3(x0, wp, Cout, sc, sh, True, x1=x1, mode=mode, w_split=wops))
        out.append((f"conv3x3 {C0:4d}{'+' + str(C1) if C1 else '':5s}->{Cout:4d} S{H}", 18.0 * B * H * H * (C0 + C1) * Cout, fns))
        del x
    return out


def session_cases():
    """(label, {mode: callable}), one session per mode: a session captures the mode set when it is built."""
    out = []
    specs = [
        ("session SmaAt_UNet(12, 1) k=2 logits B=32 288^2", lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=2), 32, (12, 288, 288), "logits"),
        ("session SmaAt_UNet(3, 21) classes B=8 224^2", lambda: S.SmaAt_UNet(3, 21, kernels_per_layer=2), 8, (3, 224, 224), "classes"),
        ("session UNet(12, 1) logits B=32 288^2", lambda: S.UNet(12, 1), 32, (12, 288, 288), "logits"),
    ]
    for label, ctor, bs, shape, output in specs:
        torch.manual_seed(0)
        model = ctor().cuda().eval()
        x = torch.rand((bs,) + shape, device="cuda")
        fns = {}
        for mode in MODES:
            ops.set_pointwise_mode(mode)
            sess = InferenceSession(model, bs, shape, output=output)
            fns[mode] = (lambda sess=sess, x=x: sess.forward(x))
        out.append((label, fns))
    ops.set_pointwise_mode("tf32x3")
    return out


def train_step_times(rounds, iters):
    """One TrainSession per mode and round (three sessions at B = 32 do not fit beside each other), modes alternated."""
    x = torch.rand((B, 12, 288, 288), device="cuda")
    y = torch.rand((B, 288, 288), device="cuda")
    times = {m: [] for m in MODES}
    for _ in range(rounds):
        for mode in MODES:
            ops.set_pointwise_mode(mode)
            torch.manual_seed(0)
            m = S.SmaAt_UNet(12, 1, kernels_per_layer=2).cuda().train()
            sess = TrainSession(m, B, (12, 288, 288), lr=1e-4)
            times[mode].append(time_fn(lambda: sess.step(x, y), iters))
            sess.close()
            del sess, m
            torch.cuda.empty_cache()
    ops.set_pointwise_mode("tf32x3")
    return times


def report(label, times, flops=None):
    cells = []
    for mode in MODES:
        t = times[mode]
        med = statistics.median(t)
        spread = (max(t) - min(t)) / med
        cell = f"{mode} {med:8.3f} ms ±{100 * spread:4.1f}%"
        if flops:
            cell += f" {flops / med / 1e9:6.1f} TF/s"
        cells.append(cell)
    ratio = statistics.median(times["tf32"]) / statistics.median(times["bf16"])
    print(f"{label:44s} | " + " | ".join(cells) + f" | tf32/bf16 {ratio:.2f}x", flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_precision: needs a GPU")
    S._lib.load()
    print(card(), flush=True)
    print(f"rounds {args.rounds}, iters {args.iters}; median over rounds, spread = (max - min) / median", flush=True)

    def run(cases, iters, with_flops):
        for case in cases:
            label, fns = case[0], case[-1]
            times = {m: [] for m in MODES}
            for _ in range(args.rounds):
                for mode in MODES:                # alternate the modes within every round
                    times[mode].append(time_fn(fns[mode], iters))
            report(label, times, case[1] if with_flops else None)

    with torch.no_grad():
        run(layer_cases(), args.iters, True)
        torch.cuda.empty_cache()
        run(session_cases(), args.iters, False)
    torch.cuda.empty_cache()
    report("TrainSession SmaAt_UNet(12, 1) k=2 step B=32 288^2", train_step_times(args.rounds, max(2, args.iters // 4)))


if __name__ == "__main__":
    main()
