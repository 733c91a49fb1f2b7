"""SmaAt-UNet at kernels_per_layer = 1, 2 and 4 on the H100 path (a tool, not a test).

  python tools/bench_kpl.py [--rounds R] [--iters N] [--parent DIR] [--json]

Reports, each with the device name and power limit:
  * InferenceSession logits of SmaAt_UNet(12, 1, kernels_per_layer=k), k in {1, 2, 4}, B = 32, 12 x 288 x 288: ms per batch;
  * at k = 4 the fused DS conv against the unfused route (dw3x3 + pw1x1, ops.set_fused_dsconv(False)), two sessions in this
    process timed in alternated rounds: median and spread (min-max) of the rounds;
  * each k = 4 fused DS conv (smaat_dsconv_fwd at B = 32, 3xTF32) beside its HBM floor 4 B S^2 (Cin + Cout) / 3.35 TB/s;
  * one k = 4 TrainSession step (B = 32, mse) of this tree and, with --parent, of another built checkout (tools/time_dsconv.py
    --tree does the same), each in its own subprocess, alternated.
A round is `iters` CUDA-graph replays between two CUDA events after a warm-up."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--parent", default=None, help="another built checkout to time the k = 4 training step against")
ap.add_argument("--json", action="store_true")
ap.add_argument("--train-only", default=None, help=argparse.SUPPRESS)     # subprocess mode: time one tree's training step
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.train_only or ROOT))

import torch  # noqa: E402

B, S_, C_IN, HBM_BPS = 32, 288, 12, 3.35e12


def device_info():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        pl = "unknown"
    return {"device": name, "power_limit": pl}


def events_ms(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def stats(xs):
    return {"median_ms": round(statistics.median(xs), 3), "min_ms": round(min(xs), 3), "max_ms": round(max(xs), 3)}


def train_step_ms(rounds, iters):
    import smaat_unet_b200 as S
    from smaat_unet_b200.train import TrainSession
    torch.manual_seed(0)
    m = S.SmaAt_UNet(C_IN, 1, kernels_per_layer=4).cuda().train()
    sess = TrainSession(m, B, (C_IN, S_, S_), lr=1e-4)
    x = torch.rand(B, C_IN, S_, S_, device="cuda")
    y = torch.rand(B, S_, S_, device="cuda")
    for _ in range(3):
        sess.step(x, y)
    torch.cuda.synchronize()
    return [events_ms(lambda: sess.step(x, y), iters) for _ in range(rounds)]


def main():
    assert torch.cuda.is_available(), "bench_kpl.py needs a GPU"
    if args.train_only:
        print(json.dumps(train_step_ms(args.rounds, args.iters)))
        return
    import smaat_unet_b200 as S
    from smaat_unet_b200 import ops
    from smaat_unet_b200.engine import InferenceSession
    info = device_info()
    out = []
    x = torch.rand(B, C_IN, S_, S_, device="cuda")

    # ---- InferenceSession logits at k = 1, 2, 4; at k = 4 also the unfused route, alternated with the fused one
    sess = {}
    for k in (1, 2, 4):
        torch.manual_seed(0)
        m = S.SmaAt_UNet(C_IN, 1, kernels_per_layer=k).cuda().eval()
        sess[f"k{k}"] = InferenceSession(m, B, (C_IN, S_, S_))
        if k == 4:
            ops.set_fused_dsconv(False)
            try:
                sess["k4_unfused"] = InferenceSession(m, B, (C_IN, S_, S_))
            finally:
                ops.set_fused_dsconv(True)
    same = torch.equal(sess["k4"].forward(x).clone(), sess["k4"].forward(x).clone())
    ref = sess["k4_unfused"].forward(x).clone()
    rel = float((sess["k4"].forward(x) - ref).abs().max() / ref.abs().max())
    times = {n: [] for n in sess}
    for n, s in sess.items():
        events_ms(lambda: s.forward(x), 3)
    for _ in range(args.rounds):
        for n, s in sess.items():
            times[n].append(events_ms(lambda: s.forward(x), args.iters))
    for n, t in times.items():
        out.append({"what": f"InferenceSession logits {n}", "B": B, **stats(t), **info})
    out.append({"what": "k4 fused vs unfused", "speedup_median": round(statistics.median(times["k4_unfused"]) / statistics.median(times["k4"]), 3),
                "fused_repeatable": same, "max_rel_diff_vs_unfused": rel, **info})
    del sess

    # ---- each k = 4 fused DS conv at B = 32 beside its HBM floor
    layers = [("inc.0", 12, 0, 64, 288), ("inc.1", 64, 0, 64, 288), ("down1.0", 64, 0, 128, 144), ("down1.1", 128, 0, 128, 144),
              ("down2.0", 128, 0, 256, 72), ("down2.1", 256, 0, 256, 72), ("up2.0", 256, 256, 256, 72), ("up2.1", 256, 0, 128, 72),
              ("up3.0", 128, 128, 128, 144), ("up3.1", 128, 0, 64, 144), ("up4.0", 64, 64, 64, 288), ("up4.1", 64, 0, 64, 288)]
    g = torch.Generator(device="cuda").manual_seed(7)
    total = floor_total = 0.0
    for name, C0, C1, Cout, S in layers:
        Cin = C0 + C1
        x0 = torch.rand(B, C0, S, S, device="cuda", generator=g)
        x1 = torch.rand(B, C1, S, S, device="cuda", generator=g) if C1 else None
        dw_w = torch.randn(4 * Cin, 1, 3, 3, device="cuda", generator=g) * 0.3
        dw_b = torch.randn(4 * Cin, device="cuda", generator=g) * 0.1
        pw = torch.randn(Cout, 4 * Cin, device="cuda", generator=g) * 0.05
        sc, sh = torch.rand(Cout, device="cuda", generator=g) + 0.5, torch.randn(Cout, device="cuda", generator=g) * 0.1
        split = ops.split_tf32(pw)
        fn = lambda: ops.dsconv(x0, dw_w, dw_b, 4, pw, sc, sh, True, x1=x1, mode="tf32x3", w_split=split)
        assert fn() is not None, f"{name}: not fused"
        events_ms(fn, 3)
        ms = statistics.median(events_ms(fn, args.iters) for _ in range(args.rounds))
        floor = 4.0 * B * S * S * (Cin + Cout) / HBM_BPS * 1e3
        total += ms
        floor_total += floor
        out.append({"what": f"k4 fused {name} C{Cin}->{Cout} {S}^2", "ms": round(ms, 4), "hbm_floor_ms": round(floor, 4),
                    "share_of_floor": round(floor / ms, 3), **info})
        del x0, x1
    out.append({"what": "k4 fused DS convs, sum", "ms": round(total, 3), "hbm_floor_ms": round(floor_total, 3), **info})
    torch.cuda.empty_cache()

    # ---- one k = 4 training step, this tree against --parent, alternated subprocesses
    trees = [("this", ROOT)] + ([("parent", os.path.abspath(args.parent))] if args.parent else [])
    tt = {n: [] for n, _ in trees}
    for _ in range(2):
        for n, tree in trees:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--train-only", tree, "--rounds", str(args.rounds),
                                "--iters", "5"], capture_output=True, text=True, cwd=tree)
            if r.returncode != 0:
                tt[n] = None
                out.append({"what": f"TrainSession k4 step ({n})", "error": r.stderr.strip().splitlines()[-1:], **info})
                continue
            if tt[n] is not None:
                tt[n] += json.loads(r.stdout.strip().splitlines()[-1])
    for n, t in tt.items():
        if t:
            out.append({"what": f"TrainSession k4 step B={B} ({n})", **stats(t), **info})
    for r in out:
        print(json.dumps(r) if args.json else "  ".join(f"{k}={v}" for k, v in r.items()))


if __name__ == "__main__":
    main()
