"""bf16 activations in HBM against fp32 ones: SmaAt-UNet's serving sessions in three setups, alternated round by round.

  fp32+bf16ops  fp32 storage, set_pointwise_mode('bf16') (bf16 GEMM operands)
  bf16          bf16 storage: InferenceSession(dtype=torch.bfloat16) (bf16 operands at levels 1-3; levels 4-5 in 'bf16' mode too)
  tf32x3        fp32 storage, the default mode: the anchor

Sessions: SmaAt_UNet(12, 1) logits at B = 32, 12 x 288 x 288 and SmaAt_UNet(3, 21) class maps at B = 8, 3 x 224 x 224.  For
each: device time per graph replay (CUDA events over --replays replays per round, --rounds rounds with the setups alternated:
median and min-max), the submit / collect time per batch over --batches pinned-host batches (host clock, ends in collect's
synchronise), the memory the session reserved (torch.cuda.memory_reserved across its construction, empty cache before), and the
input / output bytes per batch.  A torch.profiler run of its own (one eager serving forward per setup after warm-up) gives the
per-launch device times of the DS convs, the CBAM kernels and the upsample.  The card name and power limit are read in the same
run.  Writes one JSON document to --out.

    python tools/bench_bf16_activations.py --out /tmp/bf16_activations.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402

SETUPS = {"fp32+bf16ops": ("bf16", torch.float32), "bf16": ("bf16", torch.bfloat16), "tf32x3": ("tf32x3", torch.float32)}
SESSIONS = {
    "smaat_12_1_logits_b32_288": (lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=2), 32, (12, 288, 288), "logits"),
    "smaat_3_21_classes_b8_224": (lambda: S.SmaAt_UNet(3, 21, kernels_per_layer=2), 8, (3, 224, 224), "classes"),
}
KERNEL_GROUPS = ("dsconv", "cbam", "upsample")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def build(setup, sess_name):
    mode, dtype = SETUPS[setup]
    ctor, B, shape, output = SESSIONS[sess_name]
    ops.set_pointwise_mode(mode)
    torch.manual_seed(0)
    model = ctor().cuda().eval()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r0 = torch.cuda.memory_reserved()
    sess = InferenceSession(model, B, shape, output=output, dtype=dtype)
    torch.cuda.synchronize()
    reserved = torch.cuda.memory_reserved() - r0
    x = torch.rand((B,) + shape, generator=torch.Generator().manual_seed(1)).to(dtype)
    sess.static_in.copy_(x.cuda())
    return {"sess": sess, "mode": mode, "x_host": x.pin_memory(), "reserved_MiB": reserved / 2 ** 20,
            "h2d_bytes": sess.h2d_bytes_per_step, "d2h_bytes": sess.d2h_bytes_per_step}


def replay_ms(entry, n):
    ops.set_pointwise_mode(entry["mode"])
    sess = entry["sess"]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.cuda.stream(sess.compute):
        e0.record()
        for _ in range(n):
            sess.replay()
        e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def submit_collect_ms(entry, n):
    sess, x = entry["sess"], entry["x_host"]
    sess.submit(x)
    sess.collect()
    t0 = time.perf_counter()
    for i in range(n):
        sess.submit(x)
        if i >= 1:
            sess.collect()
    sess.collect()
    return (time.perf_counter() - t0) * 1e3 / n


def profile(entries, out_dir):
    res = {}
    for (setup, sess_name), entry in entries.items():
        sess = entry["sess"]
        ops.set_pointwise_mode(entry["mode"])
        x = sess.static_in
        fwd = sess._fwd
        with torch.no_grad():
            fwd(x)
            torch.cuda.synchronize()
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                fwd(x)
                torch.cuda.synchronize()
        per = {}
        for ev in prof.key_averages():
            name = ev.key
            grp = next((g for g in KERNEL_GROUPS if g in name), None)
            if grp is None:
                continue
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            per.setdefault(grp, {"us": 0.0, "launches": 0, "kernels": {}})
            per[grp]["us"] += t
            per[grp]["launches"] += ev.count
            per[grp]["kernels"][name[:90]] = {"us": t, "launches": ev.count}
        res[f"{setup}/{sess_name}"] = per
        if out_dir:
            prof.export_chrome_trace(os.path.join(out_dir, f"trace_{setup}_{sess_name}.json"))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--replays", type=int, default=20)
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--traces", action="store_true", help="also write the profiler traces beside --out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bf16_activations: needs a GPU")
    doc = {"card": card(), "rounds": a.rounds, "replays": a.replays, "batches": a.batches, "sessions": {}}
    entries = {(s, n): build(s, n) for n in SESSIONS for s in SETUPS}
    for e in entries.values():                      # warm-up
        replay_ms(e, 3)
    times = {k: [] for k in entries}
    sc = {k: [] for k in entries}
    for _ in range(a.rounds):
        for k, e in entries.items():
            times[k].append(replay_ms(e, a.replays))
        for k, e in entries.items():
            sc[k].append(submit_collect_ms(e, a.batches))
    for (s, n), e in entries.items():
        t, c = times[(s, n)], sc[(s, n)]
        doc["sessions"].setdefault(n, {})[s] = {
            "replay_ms_median": statistics.median(t), "replay_ms_min": min(t), "replay_ms_max": max(t),
            "submit_collect_ms_median": statistics.median(c), "submit_collect_ms_min": min(c), "submit_collect_ms_max": max(c),
            "reserved_MiB": e["reserved_MiB"], "h2d_bytes": e["h2d_bytes"], "d2h_bytes": e["d2h_bytes"]}
    out_dir = os.path.dirname(a.out) if (a.out and a.traces) else None
    doc["profile_us"] = profile(entries, out_dir)
    ops.set_pointwise_mode("tf32x3")
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
