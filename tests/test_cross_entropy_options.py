"""Cross-entropy options, CPU side: argument checks of smaat_cross_entropy_fwd / smaat_onehot_classes, their kernels'
resource usage, the host-side validation of CrossEntropyLossWithOptions / cross_entropy (torch's messages), and
TrainSession's refusal of a per-pixel loss before it touches a device."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib
from smaat_unet_b200.segmentation import cross_entropy


def test_cross_entropy_entry_points_reject_bad_arguments_before_launch():
    lib = _lib.load()
    f = lib.smaat_cross_entropy_fwd
    acc = 64                      # any non-null address: validation fails before anything is enqueued
    #     logits target prob weight B  K  P   eps  ign  use acc  map   dl    conf  stream
    assert f(None, 8, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1
    assert b"cross_entropy_fwd" in lib.smaat_last_error()
    assert f(16, 8, None, None, 2, 4, 16, 0.0, -100, 1, None, None, None, None, None) == -1     # no batch_acc
    assert f(16, None, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1   # no target at all
    assert f(16, 8, 16, None, 2, 4, 16, 0.0, -100, 0, acc, None, None, None, None) == -1        # both kinds of target
    assert f(16, 8, None, None, 2, 1, 16, 0.0, -100, 1, acc, None, None, None, None) == -1      # K < 2
    assert f(16, 8, None, None, 2, 4, 0, 0.0, -100, 1, acc, None, None, None, None) == -1       # no pixels
    assert f(16, 8, None, None, 0, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1      # no images
    assert f(16, 8, None, None, 2, 4, 16, 1.5, -100, 1, acc, None, None, None, None) == -1      # smoothing > 1
    assert f(16, 8, None, None, 2, 4, 16, -0.1, -100, 1, acc, None, None, None, None) == -1     # smoothing < 0
    assert f(16, 8, None, None, 2, 4, 16, float("nan"), -100, 1, acc, None, None, None, None) == -1
    assert f(16, None, 16, None, 2, 4, 16, 0.0, 255, 1, acc, None, None, None, None) == -1      # ignore with probabilities
    assert f(16, 12, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1     # misaligned int64 target
    assert f(18, 8, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1      # misaligned logits
    assert f(16, 8, None, 18, 2, 4, 16, 0.0, -100, 1, acc, None, None, None, None) == -1        # misaligned weight
    assert f(16, 8, None, None, 2, 4, 16, 0.0, -100, 1, 68, None, None, None, None) == -1       # misaligned batch_acc
    assert f(16, 8, None, None, 2, 4, 16, 0.0, -100, 1, acc, 18, None, None, None) == -1        # misaligned loss map
    assert f(16, 8, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, 18, None, None) == -1        # misaligned dlogits
    assert f(16, 8, None, None, 2, 4, 16, 0.0, -100, 1, acc, None, None, 12, None) == -1        # misaligned conf
    assert f(16, 8, None, None, 2, 1025, 16, 0.0, -100, 1, acc, None, None, None, None) == -3   # K > 1024: unsupported
    g = lib.smaat_onehot_classes
    assert g(None, 8, 2, 4, 16, None) == -1
    assert b"onehot_classes" in lib.smaat_last_error()
    assert g(16, None, 2, 4, 16, None) == -1
    assert g(16, 8, 2, 0, 16, None) == -1
    assert g(16, 8, 2, 4, 0, None) == -1
    assert g(18, 8, 2, 4, 16, None) == -1
    assert g(16, 12, 2, 4, 16, None) == -1
    assert g(16, 8, 2, 1025, 16, None) == -3


def test_cross_entropy_option_kernels_use_no_local_memory():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    usage = subprocess.run([exe, "--dump-resource-usage", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if "cross_entropy_kernel" in m.group(1) or "onehot_classes_kernel" in m.group(1):
            seen += 1
            local = re.search(r"LOCAL:(\d+)", m.group(2))
            assert local and int(local.group(1)) == 0, f"{m.group(1)} uses local memory: {m.group(2)}"
    assert seen == 10         # cross_entropy: {vector, scalar} x {shared, global histogram} x {class, probability}; onehot: 2


def test_host_validation_uses_torchs_messages():
    x = torch.zeros(2, 4, 3, 3)                  # the checks run before the logits are looked at: no device needed
    t = torch.zeros(2, 3, 3, dtype=torch.int64)
    with pytest.raises(RuntimeError, match="weight tensor should be defined either for all 4 classes"):
        cross_entropy(x, t, weight=torch.ones(3))
    with pytest.raises(RuntimeError, match="weight tensor should be defined either for all 4 classes"):
        cross_entropy(x, t, weight=torch.ones(4, 1))
    with pytest.raises(RuntimeError, match=r"label_smoothing must be between 0.0 and 1.0. Got: 1.5"):
        cross_entropy(x, t, label_smoothing=1.5)
    with pytest.raises(RuntimeError, match="label_smoothing must be between 0.0 and 1.0"):
        S.CrossEntropyLossWithOptions(label_smoothing=-0.1)
    with pytest.raises(RuntimeError, match="ignore_index is not supported for floating point target"):
        cross_entropy(x, torch.rand(2, 4, 3, 3), ignore_index=255)
    with pytest.raises(RuntimeError, match="ignore_index is not supported for floating point target"):
        S.CrossEntropyLossWithOptions(ignore_index=0, weight=torch.ones(4))(x, torch.rand(2, 4, 3, 3))
    with pytest.raises(RuntimeError, match="floating-point target must have the logits' shape"):
        cross_entropy(x, torch.rand(2, 3, 3))
    with pytest.raises(NotImplementedError, match="at most 1024"):
        cross_entropy(torch.zeros(1, 1025, 2, 2), torch.zeros(1, 2, 2, dtype=torch.int64), label_smoothing=0.1)
    with pytest.raises(RuntimeError, match="no CPU fallback"):     # valid options, CPU logits: still no fallback
        cross_entropy(x, t, weight=torch.ones(4), label_smoothing=0.1)


def test_options_class_takes_torchs_constructor_and_the_plain_class_points_to_it():
    for cls in (S.CrossEntropyLoss, S.CrossEntropyLossWithOptions):
        with pytest.raises(NotImplementedError):
            cls(size_average=True)
        with pytest.raises(NotImplementedError):
            cls(reduce=False)
        with pytest.raises(NotImplementedError):
            cls(reduction="batchmean")
        assert cls(ignore_index=255).ignore_index == 255 and cls().weight is None
    for kw in ({"weight": torch.ones(3)}, {"label_smoothing": 0.1}, {"reduction": "none"}):
        with pytest.raises(NotImplementedError, match="CrossEntropyLossWithOptions"):
            S.CrossEntropyLoss(**kw)
    loss = S.CrossEntropyLossWithOptions(weight=torch.tensor([1.0, 2.0, 0.5]), label_smoothing=0.1, reduction="none")
    assert loss.reduction == "none" and loss.label_smoothing == 0.1
    assert "weight" in dict(loss.named_buffers())                # a buffer, as in torch: .to() moves it
    assert loss.to(torch.float64).weight.dtype == torch.float64


def test_train_session_rejects_a_per_pixel_loss_before_touching_a_device():
    from smaat_unet_b200.train import TrainSession
    model = torch.nn.Conv2d(3, 4, 1)
    with pytest.raises(ValueError, match="reduction='none'"):
        TrainSession(model, 2, (3, 8, 8), device="cpu",
                     loss=S.CrossEntropyLossWithOptions(weight=torch.ones(4), reduction="none"))
    with pytest.raises(ValueError, match="loss="):
        TrainSession(model, 2, (3, 8, 8), device="cpu", loss=torch.nn.CrossEntropyLoss())
    assert next(model.parameters()).device.type == "cpu"
