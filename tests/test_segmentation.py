"""Segmentation workflow, CPU side: IoU / ConfusionMatrix host math vs the reference's own outputs, the classification shard vs
the reference dataset class, argument checks of the new C entry points, and their kernels' resource usage."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle.make_golden_seg import CONFIGS, INDICES, K, classification_array
from smaat_unet_b200 import _lib
from smaat_unet_b200 import data as D

GOLD_DIR = os.path.join(os.path.dirname(__file__), "golden")
SEG = np.load(os.path.join(GOLD_DIR, "seg_metrics.npz"))
CLS = np.load(os.path.join(GOLD_DIR, "dataset_classification.npz"))


def _injected(normalized, ignore, invalid=0):
    m = S.IoU(K, normalized=normalized, ignore_index=ignore, device="cpu")
    m.load_totals(torch.cat([torch.from_numpy(SEG["counts"]).reshape(-1), torch.tensor([invalid])]))
    return m


@pytest.mark.parametrize("tag", sorted(CONFIGS))
def test_iou_host_math_on_injected_counts_equals_reference(tag):
    normalized, ignore = CONFIGS[tag]
    m = _injected(normalized, ignore)
    conf = m.conf_metric.value()
    want = SEG[f"{tag}/int/conf"]
    assert conf.dtype == want.dtype and np.array_equal(conf, want)
    iou, miou = m.value()
    assert iou.dtype == SEG[f"{tag}/int/iou"].dtype
    assert np.array_equal(iou, SEG[f"{tag}/int/iou"], equal_nan=True)      # NaN positions included
    assert np.isnan(iou[int(SEG["absent"])])
    assert miou == SEG[f"{tag}/int/miou"]
    # value() leaves the counts alone (the reference's IoU.value zeroes ignored rows of its own matrix in place)
    assert np.array_equal(m.conf_metric.counts()[0], SEG["counts"])


def test_out_of_range_labels_make_value_raise_and_reset_clears():
    m = _injected(False, None, invalid=3)
    with pytest.raises(AssertionError, match="not between 0 and k-1"):
        m.value()
    m.reset()
    iou, miou = m.value()
    assert np.isnan(iou).all() and np.isnan(miou)


def test_constructors_refuse_what_has_no_kernel():
    with pytest.raises(NotImplementedError):
        S.CrossEntropyLoss(weight=torch.ones(3))
    with pytest.raises(NotImplementedError):
        S.CrossEntropyLoss(label_smoothing=0.1)
    with pytest.raises(NotImplementedError):
        S.CrossEntropyLoss(reduction="none")
    with pytest.raises(NotImplementedError):
        S.IoU(2000, device="cpu")
    with pytest.raises(ValueError):
        S.IoU(4, ignore_index=1.5, device="cpu")
    assert S.IoU(4, ignore_index=[1, 2], device="cpu").ignore_index == (1, 2)
    assert S.CrossEntropyLoss(ignore_index=255).ignore_index == 255


@pytest.mark.parametrize("train", [True, False])
def test_classification_shard_reproduces_the_reference_samples(tmp_path, train):
    seq = classification_array()
    tag = "train" if train else "test"
    arr = seq if train else seq[::-1].copy()
    ds = D.precipitation_maps_classification_shard(D.write_shard(str(tmp_path / "seq.npy"), arr), 12, 6, train=train)
    assert len(ds) == int(CLS[f"{tag}/len"])
    for i in INDICES:
        x, y = ds[i]
        gx, gy = CLS[f"{tag}/{i}/x"], CLS[f"{tag}/{i}/y"]
        assert x.dtype == gx.dtype and np.array_equal(x, gx)
        assert y.dtype == gy.dtype == np.int64 and np.array_equal(y, gy)
        xs, ys = ds.sample_shapes()
        xb, yb = np.empty(xs, np.float32), np.empty(ys, np.int64)
        ds.read_into(i, xb, yb)
        assert np.array_equal(xb, gx) and np.array_equal(yb, gy)


def test_loader_target_dtype_follows_the_dataset():
    seq = classification_array()
    cls = D.precipitation_maps_classification_shard(seq, 12, 6)
    reg = D.precipitation_maps_shard(seq, 12, 6)
    for ds, dt in ((cls, torch.int64), (reg, torch.float32)):
        batches = [(x.clone(), y.clone()) for x, y in D.PinnedBatchLoader(ds, batch_size=5, pin_memory=False)]
        assert batches and all(x.dtype == torch.float32 and y.dtype == dt for x, y in batches)
    ys = torch.cat([y.clone() for _, y in D.PinnedBatchLoader(cls, batch_size=5, pin_memory=False)])
    assert torch.equal(ys, torch.from_numpy(np.stack([cls[i][1] for i in range(len(ys))])))


def test_new_entry_points_reject_bad_arguments_on_the_host():
    lib = _lib.load()
    acc = 16                                    # any non-null address: validation fails before anything is enqueued
    assert lib.smaat_ce_fwd(None, 8, 2, 4, 16, -100, 1, acc, None, None, None) == -1
    assert b"ce_fwd" in lib.smaat_last_error()
    assert lib.smaat_ce_fwd(16, 8, 2, 1, 16, -100, 1, acc, None, None, None) == -1            # K < 2
    assert lib.smaat_ce_fwd(16, 8, 2, 4, 0, -100, 1, acc, None, None, None) == -1             # no pixels
    assert lib.smaat_ce_fwd(16, 12, 2, 4, 16, -100, 1, acc, None, None, None) == -1           # misaligned int64 target
    assert lib.smaat_ce_fwd(16, 8, 2, 1025, 16, -100, 1, acc, None, None, None) == -3         # K > 1024: unsupported
    assert lib.smaat_confusion_add(None, 8, 10, 4, 16, None, None) == -1
    assert b"confusion_add" in lib.smaat_last_error()
    assert lib.smaat_confusion_add(8, 8, 10, 4, None, None, None) == -1
    assert lib.smaat_confusion_add(8, 8, 10, 2048, 16, None, None) == -3


def test_new_kernels_use_no_local_memory():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    usage = subprocess.run([exe, "--dump-resource-usage", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if "ce_fwd_kernel" in m.group(1) or "confusion_add_kernel" in m.group(1):
            seen += 1
            local = re.search(r"LOCAL:(\d+)", m.group(2))
            assert local and int(local.group(1)) == 0, f"{m.group(1)} uses local memory: {m.group(2)}"
    assert seen == 6          # ce_fwd: {vector, scalar} x {shared, global histogram}; confusion_add: {shared, global}
