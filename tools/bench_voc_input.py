"""VOC segmentation input pipeline (train_SmaAtUNet.py:139-173: SmaAt_UNet(3, 21), batch 8, 224x224), alternated rounds.

    python tools/bench_voc_input.py [--samples 96] [--rounds 5] [--steps 24] [--kernel-iters 200]

A synthetic VOC tree (JPEG images of 500x375 / 375x500, P-mode masks with 255 borders, like VOC2012) is generated from a
seed in a temporary directory, converted once with data.convert_voc, and deleted at the end.
(a) samples/s of the reference's per-sample pipeline (oracle/voc_reference_pipeline.py: decode, Resize(256) + CenterCrop(224),
    augmentations, ToTensor / Normalize) through DataLoader(batch_size=8, shuffle=True, num_workers=0, pin_memory=True);
    "not measured" when PIL or torchvision is missing
(b) samples/s of PinnedBatchLoader on the uint8 shards with augmentation draws (host only)
(c) smaat_voc_augment_fwd per batch (CUDA events, mixed augmentations), with bytes/s against its HBM floor of
    (3 + 1) bytes read and (12 + 8) written per pixel
(d) TrainSession(SmaAt_UNet(3, 21), 8, (3, 224, 224), loss="cross_entropy") steps/s fed by (a), by (b) + the kernel
    (input_transform=ops.VOCNormalize()), and on a device-resident batch (no input at all)
Every round runs each leg once, in turn; medians over the rounds are printed with the card's name and power limit, and one
JSON line at the end.  Writes nothing outside the temporary directory.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200 import data as D  # noqa: E402
from smaat_unet_b200 import ops  # noqa: E402
from smaat_unet_b200.train import TrainSession  # noqa: E402

B, HW, HBM_TBS = 8, 224, 3.35


def card():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        limit = float(out.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return name, limit


def make_tree(root, n, seed):
    from PIL import Image
    rng = np.random.default_rng(seed)
    voc = os.path.join(root, "VOC2012")
    for d in ("JPEGImages", "SegmentationClass", os.path.join("ImageSets", "Segmentation")):
        os.makedirs(os.path.join(voc, d))
    names = []
    for i in range(n):
        h, w = (375, 500) if i % 3 else (500, 375)
        yy, xx = np.mgrid[0:h, 0:w]
        img = np.stack([xx * 255 // w, yy * 255 // h, (xx * yy) % 256], -1).astype(np.int16)
        img = np.clip(img + rng.integers(-30, 31, img.shape), 0, 255).astype(np.uint8)
        Image.fromarray(img).save(os.path.join(voc, "JPEGImages", f"{i:06d}.jpg"), quality=90)
        m = rng.integers(0, 21, (h // 25 + 1, w // 25 + 1), dtype=np.uint8).repeat(25, 0).repeat(25, 1)[:h, :w].copy()
        m[:4], m[:, :4] = 255, 255
        Image.fromarray(m, mode="P").save(os.path.join(voc, "SegmentationClass", f"{i:06d}.png"))
        names.append(f"{i:06d}")
    with open(os.path.join(voc, "ImageSets", "Segmentation", "train.txt"), "w") as f:
        f.write("\n".join(names) + "\n")


def forever(make_iter):
    """Batches from a fresh iterator per epoch, without end."""
    epoch = 0
    while True:
        for b in make_iter(epoch):
            yield b
        epoch += 1


def rate(batches, steps, consume):
    """Samples/s over `steps` batches (host clock, device synchronised at both ends)."""
    torch.cuda.synchronize()
    t0, n = time.perf_counter(), 0
    for _ in range(steps):
        b = next(batches)
        consume(b)
        n += b[0].shape[0]
    torch.cuda.synchronize()
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=96)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=24)
    ap.add_argument("--kernel-iters", type=int, default=200)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_voc_input.py measures on a GPU"
    name, limit = card()
    print(f"card: {name}, power limit {limit} W")
    try:
        import PIL  # noqa: F401
        import torchvision  # noqa: F401
        have_pil = True
    except ImportError:
        have_pil = False
    if not have_pil:
        print("PIL / torchvision missing: no synthetic JPEG tree, legs (a) and (d, fed by a) not measured; "
              "the shards are generated directly")
    res = {"card": name, "power_limit_w": limit, "batch": B, "hw": HW}
    with tempfile.TemporaryDirectory() as tmp:
        prefix = os.path.join(tmp, "shard")
        if have_pil:
            make_tree(tmp, a.samples, 20261017)
            D.convert_voc(tmp, "train", prefix)
        else:
            rng = np.random.default_rng(20261017)
            np.save(prefix + "_images.npy", rng.integers(0, 256, (a.samples, HW, HW, 3), dtype=np.uint8))
            np.save(prefix + "_masks.npy", rng.integers(0, 21, (a.samples, HW, HW), dtype=np.uint8))
        shard = D.voc_segmentation_shard(prefix, augmentations=True)
        loader = D.PinnedBatchLoader(shard, B, shuffle=True, seed=0)

        def pinned_epoch(e):
            loader.set_epoch(e)
            return iter(loader)

        ref_batches = None
        if have_pil:
            from oracle.voc_reference_pipeline import VOCReferencePipeline
            dl = torch.utils.data.DataLoader(VOCReferencePipeline(tmp), batch_size=B, shuffle=True, num_workers=0,
                                             pin_memory=True, drop_last=True)
            ref_batches = forever(lambda e: iter(dl))
        pin_batches = forever(pinned_epoch)

        torch.manual_seed(0)
        m_u8, m_f = S.SmaAt_UNet(3, 21), S.SmaAt_UNet(3, 21)
        m_f.load_state_dict(m_u8.state_dict())
        s_u8 = TrainSession(m_u8, B, (3, HW, HW), loss="cross_entropy", input_transform=ops.VOCNormalize())
        s_f = TrainSession(m_f, B, (3, HW, HW), loss="cross_entropy")

        # (c) the kernel alone
        g = torch.Generator().manual_seed(1)
        xk = torch.randint(0, 256, (B, HW, HW, 3), dtype=torch.uint8, generator=g).cuda()
        yk = torch.randint(0, 256, (B, HW, HW), dtype=torch.uint8, generator=g).cuda()
        augk = torch.tensor([[i % 2, (i // 2) % 3 - 1, i % 3 - 1] for i in range(B)], dtype=torch.int8).cuda()
        ox, oy = torch.empty(B, 3, HW, HW, device="cuda"), torch.empty(B, HW, HW, dtype=torch.int64, device="cuda")

        def kernel_ms():
            for _ in range(10):
                ops.voc_augment(xk, yk, augk, out_x=ox, out_y=oy)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.kernel_iters):
                ops.voc_augment(xk, yk, augk, out_x=ox, out_y=oy)
            e1.record()
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / a.kernel_iters

        def step_u8(b):
            x, y, aug = b
            s_u8.step(x, y, aug=aug)
            loader.guard(s_u8.last_h2d_event())

        legs = {
            "b_loader_samples_s": lambda: rate(pin_batches, a.steps, lambda b: None),
            "c_kernel_ms": kernel_ms,
            "d_steps_s_loader_kernel": lambda: rate(pin_batches, a.steps, step_u8) / B,
            "d_steps_s_device_resident": lambda: rate(forever(lambda e: [(s_f.x,)] * a.steps), a.steps, lambda b: s_f.step()) / B,
        }
        if have_pil:
            legs["a_reference_samples_s"] = lambda: rate(ref_batches, a.steps, lambda b: None)
            legs["d_steps_s_reference_input"] = lambda: rate(ref_batches, a.steps, lambda b: s_f.step(b[0], b[1])) / B
        for fn in legs.values():            # warm-up of every leg
            fn()
        got = {k: [] for k in legs}
        for _ in range(a.rounds):
            for k, fn in legs.items():
                got[k].append(fn())
        for k, v in got.items():
            res[k] = statistics.median(v)
            print(f"{k:30s} median {res[k]:10.3f}   rounds {[round(x, 3) for x in v]}")
        nbytes = 24 * B * HW * HW
        res["c_kernel_gbs"] = nbytes / (res["c_kernel_ms"] * 1e-3) / 1e9
        res["c_kernel_hbm_floor_us"] = nbytes / (HBM_TBS * 1e12) * 1e6
        print(f"kernel: {res['c_kernel_ms'] * 1e3:.1f} us per batch, {res['c_kernel_gbs']:.0f} GB/s over {nbytes} B "
              f"(floor {res['c_kernel_hbm_floor_us']:.2f} us at {HBM_TBS} TB/s)")
        if not have_pil:
            res["a_reference_samples_s"] = res["d_steps_s_reference_input"] = "not measured"
        loader_rate, dev_rate = res["b_loader_samples_s"], res["d_steps_s_device_resident"] * B
        print(f"training step consumes {dev_rate:.0f} samples/s on device-resident batches; the shard loader supplies "
              f"{loader_rate:.0f} samples/s" + (f", the reference pipeline {res['a_reference_samples_s']:.0f}" if have_pil else ""))
        s_u8.close()
        s_f.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
