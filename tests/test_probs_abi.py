"""CPU-side checks of the probability entry point (smaat_softmax_channels_fwd): bad arguments are rejected on the host,
before any CUDA call, with SMAAT_E_BADARG or SMAAT_E_UNSUPPORTED; InferenceSession refuses an unknown
output kind before it touches the device; every model offers probabilities."""
import pytest
import torch

import smaat_unet_b200 as S

BADARG, UNSUPPORTED = -1, -3
# fake, 16-byte aligned addresses: never dereferenced, validation fails first
A = 1 << 20


def test_softmax_channels_rejects_bad_arguments_before_launch():
    lib = S._lib.load()
    f = lib.smaat_softmax_channels_fwd
    assert f(None, A, 2, 8, 64, None) == BADARG
    assert f(A, None, 2, 8, 64, None) == BADARG
    assert f(A, A, 0, 8, 64, None) == BADARG
    assert f(A, A, 2, 8, 0, None) == BADARG
    assert f(A, A, 2, 0, 64, None) == BADARG and b"K=0" in lib.smaat_last_error()
    assert f(A, A, 2, 1025, 64, None) == UNSUPPORTED and b"at most 1024" in lib.smaat_last_error()
    assert f(A + 2, A, 2, 8, 64, None) == BADARG and b"aligned" in lib.smaat_last_error()
    assert f(A, A + 2, 2, 8, 64, None) == BADARG and b"aligned" in lib.smaat_last_error()


@pytest.mark.parametrize("output", ["probabilities", "prob", "softmax", None])
def test_inference_session_rejects_unknown_output_before_touching_the_device(output):
    from smaat_unet_b200.engine import InferenceSession
    with pytest.raises(ValueError, match="'probs'"):
        InferenceSession(S.SmaAt_UNet(3, 4), 1, (3, 32, 32), device="cpu", output=output)


def test_every_model_offers_probabilities():
    for m in (S.SmaAt_UNet(3, 21), S.UNet(3, 21), S.UNetAttention(3, 21)):
        assert callable(getattr(m, "forward_probs", None))
    assert callable(getattr(S.OutConv(64, 8), "probs", None))
    with pytest.raises(RuntimeError, match="no CPU fallback"), torch.no_grad():
        S.ops.softmax_channels(torch.zeros(1, 4, 8, 8))
