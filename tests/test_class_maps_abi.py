"""CPU-side checks of the class-map entry points (smaat_dsconv_classify_fwd / _eligible, smaat_argmax_channels_fwd): bad
arguments are rejected on the host, before any CUDA call, with SMAAT_E_BADARG or SMAAT_E_UNSUPPORTED; InferenceSession
refuses an unknown output kind."""
import pytest
import torch

import smaat_unet_b200 as S

BADARG, UNSUPPORTED = -1, -3
# fake, 16-byte aligned addresses: never dereferenced, validation fails first
A = 1 << 20


def _classify(lib, oc_w=A, K=8, logits=A, classes=A, x0=A, Cout=64):
    # up4's last conv at 64 x 64: x0 (B, 64, H, W), k = 2, Cout = 64, tf32x3
    return lib.smaat_dsconv_classify_fwd(x0, 64, 64 * 64 * 64, None, 0, 0, A, None, A, A, None, None, oc_w, None, K, logits, classes,
                                         2, 64, 64, 2, Cout, 1, 2, None)


def test_dsconv_classify_rejects_bad_arguments_before_launch():
    lib = S._lib.load()
    assert _classify(lib, oc_w=None) == BADARG and b"OutConv weight" in lib.smaat_last_error()
    assert _classify(lib, logits=None, classes=None) == BADARG
    assert _classify(lib, x0=None) == BADARG
    assert _classify(lib, K=0) == BADARG and b"K=0" in lib.smaat_last_error()
    assert _classify(lib, K=-3) == BADARG
    assert _classify(lib, K=33) == UNSUPPORTED and b"at most 32" in lib.smaat_last_error()
    assert _classify(lib, classes=A + 4) == BADARG and b"8-byte" in lib.smaat_last_error()
    # Cout > 128: the OutConv needs every channel in one pass
    assert _classify(lib, Cout=256) == UNSUPPORTED


def test_dsconv_classify_eligible_query():
    lib = S._lib.load()

    def q(K=8, Cout=64, mode=2, H=64, W=64):
        return lib.smaat_dsconv_classify_eligible(A, 64, 64 * H * W, None, 0, 0, A, H, W, 2, Cout, K, mode)

    assert q() == 1 and q(mode=1) == 1 and q(K=1) == 1 and q(K=32) == 1
    assert q(K=0) == 0 and q(K=33) == 0 and q(mode=0) == 0 and q(Cout=256) == 0 and q(W=62) == 0


def test_argmax_channels_rejects_bad_arguments_before_launch():
    lib = S._lib.load()
    f = lib.smaat_argmax_channels_fwd
    assert f(None, A, 2, 8, 64, None) == BADARG
    assert f(A, None, 2, 8, 64, None) == BADARG
    assert f(A, A, 0, 8, 64, None) == BADARG
    assert f(A, A, 2, 8, 0, None) == BADARG
    assert f(A, A, 2, 0, 64, None) == BADARG and b"K=0" in lib.smaat_last_error()
    assert f(A, A, 2, 1025, 64, None) == UNSUPPORTED and b"at most 1024" in lib.smaat_last_error()
    assert f(A + 2, A, 2, 8, 64, None) == BADARG and b"aligned" in lib.smaat_last_error()
    assert f(A, A + 4, 2, 8, 64, None) == BADARG


def test_inference_session_rejects_unknown_output():
    from smaat_unet_b200.engine import InferenceSession
    with pytest.raises(ValueError, match="'logits' or 'classes'"):
        InferenceSession(S.SmaAt_UNet(3, 4), 1, (3, 32, 32), output="probabilities")


def test_every_model_offers_a_class_map():
    for m in (S.SmaAt_UNet(3, 21), S.UNet(3, 21), S.UNetAttention(3, 21)):
        assert callable(getattr(m, "forward_classes", None))
    with pytest.raises(RuntimeError, match="no CPU fallback"), torch.no_grad():
        S.ops.argmax_channels(torch.zeros(1, 4, 8, 8))
