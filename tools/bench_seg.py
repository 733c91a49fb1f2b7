"""Segmentation workflow timings (train_SmaAtUNet.py:139-199: SmaAt_UNet(3, 21), batch 8, 3x224x224), alternated runs.

    python tools/bench_seg.py [--rounds 7] [--iters 20]

(a) one training step: TrainSession(loss="cross_entropy") vs the reference loop on the same modules (model(x),
    nn.CrossEntropyLoss, backward, torch.optim.Adam -- train_SmaAtUNet.py:54-57)
(b) one validation batch: the reference's eager forward + loss.item() + argmax(softmax) + host bincount of IoU.add
    (train_SmaAtUNet.py:69-77, metric/confusionmatrix.py:40-69) vs InferenceSession + ce_step (no host sync per batch)
(a') one training step with TrainSession(loss=CrossEntropyLossWithOptions(weight=w, label_smoothing=0.1)) (smaat_cross_entropy_fwd)
    against loss="cross_entropy" (smaat_ce_fwd), same shapes
(c) the loss kernels alone (loss + gradient + confusion matrix) at B = 32, K = 8, 288x288, each against its HBM floor
    over 2 654 208 px:
      ce_fwd        smaat_ce_fwd                                   32 B logits + 32 B gradient + 8 B target   = 72 B/px
      ce_weighted   smaat_cross_entropy_fwd, weights + eps = 0.1   the same bytes                             = 72 B/px
      ce_prob       smaat_cross_entropy_fwd, probability targets   32 B logits + 32 B targets + 32 B gradient = 96 B/px
      ce_none       ce_weighted + the per-pixel loss map           + 4 B                                      = 76 B/px
Each round runs every variant once, in turn; the medians over the rounds are printed, with the card's name and power limit.
Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import smaat_unet_b200 as S  # noqa: E402
from smaat_unet_b200.engine import InferenceSession  # noqa: E402
from smaat_unet_b200.segmentation import ce_forward, ce_forward_opts  # noqa: E402
from smaat_unet_b200.train import TrainSession  # noqa: E402

K, B, HW = 21, 8, 224


def card():
    name, limit = torch.cuda.get_device_name(0), None
    try:
        import pynvml
        pynvml.nvmlInit()
        limit = pynvml.nvmlDeviceGetEnforcedPowerLimit(pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())) / 1000.0
    except Exception:
        pass
    return name, limit


def timed(fn, iters):
    """Mean ms per call over `iters` calls, CUDA events around the batch, synchronised at both ends."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    torch.manual_seed(0)
    x = torch.rand(B, 3, HW, HW, device="cuda")
    y = torch.randint(0, K, (B, HW, HW), device="cuda")
    y_host = y.cpu()

    # (a) training step
    m_ours = S.SmaAt_UNet(3, K).cuda()
    m_ref = S.SmaAt_UNet(3, K).cuda().train()
    m_ref.load_state_dict(m_ours.state_dict())
    sess = TrainSession(m_ours, B, (3, HW, HW), loss="cross_entropy")
    opt = torch.optim.Adam(m_ref.parameters(), lr=1e-3)
    crit = torch.nn.CrossEntropyLoss()

    def ref_train():
        loss = crit(m_ref(x), y)
        opt.zero_grad()
        loss.backward()
        opt.step()

    def ours_train():
        sess.step(x, y)

    # (a') the same step with a weighted, smoothed loss
    cw = torch.rand(K) + 0.5
    m_w = S.SmaAt_UNet(3, K).cuda()
    m_w.load_state_dict(m_ref.state_dict())
    sess_w = TrainSession(m_w, B, (3, HW, HW), loss=S.CrossEntropyLossWithOptions(weight=cw, label_smoothing=0.1))

    def ours_train_weighted():
        sess_w.step(x, y)

    # (b) validation batch
    m_val = S.SmaAt_UNet(3, K).cuda().eval()
    inf = InferenceSession(m_val, B, (3, HW, HW))
    iou = S.IoU(K)
    conf_host = np.zeros((K, K), np.int64)

    def ref_val():
        with torch.no_grad():
            yp = m_val(x)
            float(crit(yp, y))                                         # val_loss += loss.item()
            pc = torch.argmax(torch.nn.functional.softmax(yp, dim=1), dim=1).cpu().numpy().reshape(-1)
            t = y_host.numpy().reshape(-1)
            conf_host[...] += np.bincount((pc + K * t).astype(np.int32), minlength=K * K).reshape(K, K)

    def ours_val():
        with torch.no_grad():
            S.ce_step(inf.forward(x), y_host, iou)

    # (c) the kernel alone
    lg = torch.randn(32, 8, 288, 288, device="cuda")
    tg = torch.randint(0, 8, (32, 288, 288), device="cuda")
    conf = torch.zeros(8, 8, dtype=torch.int64, device="cuda")
    dl = {}

    w8 = torch.rand(8, device="cuda") + 0.5
    q8 = torch.softmax(torch.randn_like(lg), dim=1)

    def kern():
        dl["acc"], dl["g"] = ce_forward(lg, tg, -100, True, want_grad=True, conf=conf)

    def kern_weighted():
        dl["acc"], _, dl["g"] = ce_forward_opts(lg, tg, w8, 0.1, -100, True, want_grad=True, conf=conf)

    def kern_prob():
        dl["acc"], _, dl["g"] = ce_forward_opts(lg, q8, w8, 0.1, -100, False, want_grad=True, conf=conf)

    def kern_none():
        dl["acc"], dl["map"], dl["g"] = ce_forward_opts(lg, tg, w8, 0.1, -100, True, want_grad=True, want_map=True, conf=conf)

    variants = {"train_ref": ref_train, "train_ours": ours_train, "train_ours_weighted": ours_train_weighted, "val_ref": ref_val,
                "val_ours": ours_val, "ce_fwd": kern, "ce_weighted": kern_weighted, "ce_prob": kern_prob, "ce_none": kern_none}
    for fn in variants.values():          # warm-up (allocator, caches, graphs)
        for _ in range(3):
            fn()
    res = {k: [] for k in variants}
    for _ in range(a.rounds):
        for k, fn in variants.items():
            res[k].append(timed(fn, a.iters))
    med = {k: statistics.median(v) for k, v in res.items()}
    floor_bytes = 32 * 288 * 288 * (8 * 4 + 8 * 4 + 8)
    px = 32 * 288 * 288
    floors = {"ce_weighted": 72 * px, "ce_prob": 96 * px, "ce_none": 76 * px}
    name, limit = card()
    out = {"card": name, "power_limit_w": limit, "rounds": a.rounds, "iters": a.iters,
           "train_step_ms": {"reference_loop": med["train_ref"], "train_session": med["train_ours"],
                             "train_session_weighted_smoothed": med["train_ours_weighted"]},
           "val_batch_ms": {"reference_loop": med["val_ref"], "inference_session_ce_step": med["val_ours"]},
           "ce_fwd_us": med["ce_fwd"] * 1e3, "ce_fwd_floor_bytes": floor_bytes,
           "ce_fwd_gbps": floor_bytes / (med["ce_fwd"] * 1e-3) / 1e9,
           "ce_options": {k: {"us": med[k] * 1e3, "floor_bytes": f, "gbps": f / (med[k] * 1e-3) / 1e9} for k, f in floors.items()},
           "spread_pct": {k: 100.0 * (max(v) - min(v)) / statistics.median(v) for k, v in res.items()}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
