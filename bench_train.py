#!/usr/bin/env python
"""bench_train.py -- BASELINE configs[2]/[3]: SmaAt-UNet training step (fwd + bwd + Adam) on H100.

  python bench_train.py [--batch 32] [--steps 10] [--warmup 3] [--mode tf32x3]
  torchrun --nproc-per-node N bench_train.py --global-batch 256      # configs[3]: DDP, one flat gradient all-reduce

Loss = mse_loss(pred.squeeze(1), y, reduction="sum") / B and Adam(lr=1e-3) as in the reference
(models/regression_lightning.py:47-65).  BatchNorm statistics stay per rank (no SyncBatchNorm in the reference).
Separate from bench.py; prints one JSON line.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import parallel as PAR  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--global-batch", type=int, default=0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mode", default="tf32x3")
    ap.add_argument("--no-graph", action="store_true")
    a = ap.parse_args()
    rank, world, local = PAR.env_rank_world()
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    PAR.init_from_env("nccl", dev)
    S.set_pointwise_mode(a.mode)
    B = a.global_batch // world if a.global_batch else a.batch
    torch.manual_seed(0)
    model = S.SmaAt_UNet(12, 1, kernels_per_layer=2).to(dev).train()
    from smaat_unet_b200.train import TrainSession
    sess = TrainSession(model, B, (12, 288, 288), lr=1e-3, device=dev, use_graph=not a.no_graph)
    gen = torch.Generator().manual_seed(1 + rank)
    # a few distinct pinned host batches: every step copies its inputs host -> device (inside the timed region)
    xs = [torch.rand((B, 12, 288, 288), generator=gen).pin_memory() for _ in range(2)]
    ys = [torch.rand((B, 288, 288), generator=gen).pin_memory() for _ in range(2)]

    for i in range(a.warmup):
        loss = sess.step(xs[i % 2], ys[i % 2])
    PAR.barrier(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(a.steps):
        loss = sess.step(xs[i % 2], ys[i % 2])
    e1.record()
    PAR.barrier(dev)
    ms = PAR.reduce_max(e0.elapsed_time(e1), dev)
    if rank == 0:
        m = {k: float(v) for k, v in sess.metrics.compute().items()}
        print(json.dumps({"task": "train step fwd+bwd+Adam (TrainSession: loss+metrics fused, h2d of the batch every step)",
                          "frames_per_s": world * B * a.steps / (ms * 1e-3), "ms_per_step": ms / a.steps,
                          "n_gpus": world, "batch_per_gpu": B, "pointwise": a.mode, "cuda_graph": not a.no_graph, "final_loss": float(loss),
                          "gpu_launches_per_step": sess.launches_per_step, "metrics_mse": m["mse"],
                          "max_mem_GB": torch.cuda.max_memory_allocated() / 1e9}))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
