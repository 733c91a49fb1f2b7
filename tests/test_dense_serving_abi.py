"""CPU-side checks of the dense networks' OutConv epilogue (smaat_conv3x3_classify_fwd, smaat_conv3x3_probs_fwd,
smaat_conv3x3_classify_eligible): the header declares them, the library exports them, and bad or unsupported requests are
refused on the host before any CUDA call; UNet / UNetAttention offer the serving forward InferenceSession looks up."""
import ctypes
import os
import re

import pytest
import torch

import smaat_unet_b200 as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BADARG, UNSUPPORTED = -1, -3
# fake, 16-byte aligned addresses: never dereferenced, validation fails first
A = 1 << 20
NAMES = ("smaat_conv3x3_classify_eligible", "smaat_conv3x3_classify_fwd", "smaat_conv3x3_probs_fwd")
TF32, TF32X3 = 1, 2


def test_header_declares_and_library_exports_the_entry_points():
    src = open(os.path.join(ROOT, "include", "smaat_b200.h")).read()
    decl = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    lib = ctypes.CDLL(S._lib.LIB_PATH)
    for name in NAMES:
        assert re.search(rf"\bint {name}\s*\(", decl), f"{name} is not declared in include/smaat_b200.h"
        assert hasattr(lib, name), f"{name} is not exported"
        assert name in S._lib.SIGNATURES
    assert "bit for bit" in src and "smaat_conv3x3_fwd -> smaat_outconv_fwd" in src


def _eligible(lib, x0=A, x1=None, C1=0, wp=A, W=64, Cout=64, K=8, mode=TF32X3):
    return lib.smaat_conv3x3_classify_eligible(x0, 64 * 64 * 64, x1, C1, 64 * 64 * 64, wp, W, Cout, K, mode)


def test_eligibility():
    lib = S._lib.load()
    assert _eligible(lib) == 1 and _eligible(lib, mode=TF32) == 1
    assert _eligible(lib, K=1) == 1 and _eligible(lib, K=32) == 1 and _eligible(lib, Cout=8) == 1
    assert _eligible(lib, x1=A, C1=64) == 1
    assert _eligible(lib, mode=0) == 0                 # fp32: the exact CUDA-core conv has no epilogue OutConv
    assert _eligible(lib, K=0) == 0 and _eligible(lib, K=33) == 0
    assert _eligible(lib, Cout=65) == 0 and _eligible(lib, Cout=7) == 0
    assert _eligible(lib, W=18) == 0                   # W % 4 != 0: the tensor-core conv declines
    assert _eligible(lib, x0=A + 4) == 0 and _eligible(lib, wp=A + 8) == 0 and _eligible(lib, x1=A + 4, C1=64) == 0


# up4's last conv at 64 x 64: x0 (2, 64, 64, 64), Cout = 64
def _classify(lib, x0=A, oc_w=A, oc_b=None, K=8, logits=A, classes=A, Cout=64, W=64, mode=TF32X3):
    return lib.smaat_conv3x3_classify_fwd(x0, 64, 64 * 64 * 64, None, 0, 0, A, A, A, A, oc_w, oc_b, K, logits, classes,
                                          2, 64, W, Cout, 1, mode, None)


def _probs(lib, x0=A, oc_w=A, K=8, probs=A, Cout=64, mode=TF32X3):
    return lib.smaat_conv3x3_probs_fwd(x0, 64, 64 * 64 * 64, None, 0, 0, A, A, A, A, oc_w, None, K, probs, 2, 64, 64, Cout, 1, mode, None)


def test_classify_rejects_bad_arguments_before_launch():
    lib = S._lib.load()
    assert _classify(lib, logits=None, classes=None) == BADARG and b"logits or a classes" in lib.smaat_last_error()
    assert _classify(lib, oc_w=None) == BADARG and b"null pointer" in lib.smaat_last_error()
    assert _classify(lib, x0=None) == BADARG
    assert _classify(lib, K=0) == BADARG and b"K=0" in lib.smaat_last_error()
    assert _classify(lib, classes=A + 4) == BADARG and b"8-byte" in lib.smaat_last_error()
    assert _classify(lib, logits=A + 2) == BADARG and b"4-byte" in lib.smaat_last_error()
    assert _classify(lib, oc_b=A + 1) == BADARG
    assert _classify(lib, mode=7) == BADARG and b"unknown mode" in lib.smaat_last_error()
    assert _classify(lib, mode=0) == UNSUPPORTED and b"smaat_outconv_fwd" in lib.smaat_last_error()
    assert _classify(lib, K=33) == UNSUPPORTED and b"K <= 32" in lib.smaat_last_error()
    assert _classify(lib, Cout=128) == UNSUPPORTED
    assert _classify(lib, W=18) == UNSUPPORTED
    assert _classify(lib, x0=A + 4) == UNSUPPORTED


def test_probs_rejects_bad_arguments_before_launch():
    lib = S._lib.load()
    assert _probs(lib, probs=None) == BADARG and b"probs output" in lib.smaat_last_error()
    assert _probs(lib, oc_w=None) == BADARG
    assert _probs(lib, K=-1) == BADARG
    assert _probs(lib, probs=A + 2) == BADARG and b"4-byte" in lib.smaat_last_error()
    assert _probs(lib, mode=0) == UNSUPPORTED
    assert _probs(lib, K=33) == UNSUPPORTED and _probs(lib, Cout=96) == UNSUPPORTED


def test_dense_models_offer_the_serving_forward():
    for cls in (S.UNet, S.UNetAttention):
        for bilinear in (True, False):
            m = cls(3, 21, bilinear)
            for name in ("forward_serving", "forward_classes", "forward_probs"):
                assert callable(getattr(m, name, None)), f"{cls.__name__}.{name}"


def test_blocks_refuse_an_unknown_head_before_touching_a_tensor():
    # CPU tensors: a check that reached them would raise RuntimeError (no CPU fallback), not ValueError
    x, low, oc = torch.zeros(1, 64, 8, 8), torch.zeros(1, 128, 4, 4), S.OutConv(64, 3)
    calls = {"DoubleConv.run": lambda **kw: S.DoubleConv(64, 64).run(x, **kw),
             "DoubleConvDS.run": lambda **kw: S.DoubleConvDS(64, 64).run(x, **kw),
             "Up.forward": lambda **kw: S.Up(128, 64)(low, x, **kw),
             "UpDS.forward": lambda **kw: S.UpDS(128, 64)(low, x, **kw)}
    for call in calls.values():
        for head in ("class", "logit", "argmax", None):
            with pytest.raises(ValueError, match="head must be one of"):
                call(outconv=oc, head=head)
        for head in ("classes", "probs"):
            with pytest.raises(ValueError, match="needs the OutConv"):
                call(head=head)
