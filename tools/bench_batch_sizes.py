"""Partial batches through InferenceSession: device time and memory of each captured size.

  python tools/bench_batch_sizes.py [--rounds R] [--iters N]

For bench.py's network (SmaAt_UNet(12, 1, kernels_per_layer=2), 12 x 288 x 288, tf32x3, eval) in one session of capacity
32 with batch_sizes (1, 2, 4, 8, 16), reports:
  * the device time of one replay per captured size B in {1, 2, 4, 8, 16, 32}, per batch and per frame (CUDA events over N
    replays, the sizes alternated within every round);
  * the memory each captured size adds: the reserved memory of a session with that one extra size minus that of a session
    with none, both measured after the allocator's cache is emptied;
  * a one-sample request through forward(): served by its own graph (batch_sizes=(1,)) against the same request padded to
    32 (a session without batch_sizes), alternated within every round.
Medians over the rounds with the spread ((max - min) / median).  The card's name and power limit are printed first.
"""
import argparse
import gc
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402

CAP = 32
SIZES = (1, 2, 4, 8, 16)
SHAPE = (12, 288, 288)


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip()
    except Exception as e:       # the number still needs its card: say what is missing
        q = f"unknown ({e})"
    return f"{name}, power limit / max SM clock: {q}"


def model():
    torch.manual_seed(0)
    m = S.SmaAt_UNet(12, 1, kernels_per_layer=2)
    g = torch.Generator().manual_seed(1)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, torch.nn.BatchNorm2d):
                mod.running_mean.copy_(torch.randn(mod.running_mean.shape, generator=g) * 0.1)
                mod.running_var.copy_(torch.rand(mod.running_var.shape, generator=g) + 0.5)
                mod.weight.copy_(torch.rand(mod.weight.shape, generator=g) + 0.5)
                mod.bias.copy_(torch.randn(mod.bias.shape, generator=g) * 0.1)
    return m.cuda().eval()


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


def med(t):
    m = statistics.median(t)
    return m, (max(t) - min(t)) / m


def reserved_after(build):
    """Reserved bytes held by what build() returns, with the allocator's cache emptied before and after."""
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r0 = torch.cuda.memory_reserved()
    obj = build()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    r = torch.cuda.memory_reserved() - r0
    del obj
    gc.collect()
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_batch_sizes: needs a GPU")
    S._lib.load()
    print(card(), flush=True)
    print(f"SmaAt_UNet(12, 1) k=2, {SHAPE[0]}x{SHAPE[1]}x{SHAPE[2]}, {S.get_pointwise_mode()}, capacity {CAP}; rounds {args.rounds}, "
          f"iters {args.iters}; median over rounds, spread = (max - min) / median", flush=True)
    m = model()

    reserved_after(lambda: InferenceSession(m, CAP, SHAPE))     # the model's weight caches stay: count them in neither
    base = reserved_after(lambda: InferenceSession(m, CAP, SHAPE))
    print(f"memory: session of capacity {CAP} without extra sizes: {base / 2**20:8.1f} MiB reserved", flush=True)
    for n in SIZES:
        r = reserved_after(lambda n=n: InferenceSession(m, CAP, SHAPE, batch_sizes=(n,)))
        print(f"memory: batch_sizes=({n},) adds {(r - base) / 2**20:8.1f} MiB", flush=True)
    again = reserved_after(lambda: InferenceSession(m, CAP, SHAPE))
    print(f"memory: session without extra sizes, measured again: {again / 2**20:8.1f} MiB reserved", flush=True)

    with torch.no_grad():
        sess = InferenceSession(m, CAP, SHAPE, batch_sizes=SIZES)
        sess.forward(torch.rand((CAP,) + SHAPE, device="cuda"))
        sizes = SIZES + (CAP,)
        times = {n: [] for n in sizes}
        with torch.cuda.stream(sess.compute):          # replay() runs on the session's stream: time it there
            for _ in range(args.rounds):
                for n in sizes:
                    times[n].append(time_fn(lambda n=n: sess.replay(n), args.iters))
        for n in sizes:
            t, sp = med(times[n])
            print(f"replay B={n:2d}: {t:8.3f} ms per batch ±{100 * sp:4.1f}%, {1e3 * t / n:8.1f} us per frame", flush=True)
        del sess
        gc.collect()
        torch.cuda.empty_cache()

        one = torch.rand((1,) + SHAPE, device="cuda")
        own = InferenceSession(m, CAP, SHAPE, batch_sizes=(1,))
        padded = InferenceSession(m, CAP, SHAPE)
        assert torch.equal(own.forward(one), padded.forward(one)), "the B = 1 graph and the padded request disagree"
        t_own, t_pad = [], []
        for _ in range(args.rounds):
            t_own.append(time_fn(lambda: own.forward(one), args.iters))
            t_pad.append(time_fn(lambda: padded.forward(one), args.iters))
        (a, sa), (b, sb) = med(t_own), med(t_pad)
        print(f"one-sample forward(): own B=1 graph {a:8.3f} ms ±{100 * sa:4.1f}%, padded to {CAP} {b:8.3f} ms ±{100 * sb:4.1f}%, "
              f"{b / a:.1f}x", flush=True)


if __name__ == "__main__":
    main()
