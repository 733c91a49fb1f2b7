"""CPU-side checks of the bf16 storage route: host-side argument validation of the *_bf16 entry points (fake aligned addresses
that are never dereferenced), which DS convs the bf16-activation kernel takes, the model-level rejections (they raise before
any device work, so they run without a GPU), and the session's byte counts from its buffers' shapes and dtypes."""
import pytest
import torch

import smaat_unet_b200 as S
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession

A = 1 << 20      # fake, 16-byte aligned address
BADARG, UNSUPPORTED = -1, -3
BF = torch.bfloat16


def _elig(lib, C0, C1, S_, Cout, k=2, ncls=0, W=None, bs_pad=0):
    W = S_ if W is None else W
    return lib.smaat_dsconv_bf16_eligible(A, C0, C0 * S_ * W + bs_pad, A if C1 else None, C1, C1 * S_ * W, A, S_, W, k, Cout, ncls)


# (C0, C1, S, Cout) of the level 1-3 DS convs of SmaAt_UNet(12, 1) at 288 and SmaAt_UNet(3, 21) at 224
LEVELS_1_3 = [(12, 0, 288, 64), (64, 0, 288, 64), (64, 0, 144, 128), (128, 0, 144, 128), (128, 0, 72, 256), (256, 0, 72, 256),
              (256, 256, 72, 256), (256, 0, 72, 128), (128, 128, 144, 128), (128, 0, 144, 64), (64, 64, 288, 64),
              (3, 0, 224, 64), (64, 0, 112, 128), (128, 0, 56, 256), (256, 256, 56, 256), (64, 64, 224, 64)]


def test_the_bf16_kernel_takes_every_level_1_3_conv():
    lib = S._lib.load()
    for k in (1, 2):
        for C0, C1, S_, Cout in LEVELS_1_3:
            if k == 1 and C1 and C0 % 32:
                continue
            # the 3-channel input conv too (K = 3 or 6: the fp32 kernel needs K % 4 == 0, the bf16 pack pads K to 32)
            assert _elig(lib, C0, C1, S_, Cout, k) == 1, (k, C0, C1, S_, Cout)
    for K in (1, 21, 22):
        assert _elig(lib, 64, 0, 288, 64, ncls=K) == 1 and _elig(lib, 64, 0, 224, 64, ncls=K) == 1
    assert _elig(lib, 64, 0, 288, 64, ncls=33) == 0


def test_the_bf16_kernel_declines_what_it_has_no_instance_for():
    lib = S._lib.load()
    assert _elig(lib, 64, 0, 288, 64, k=4) == 0                  # k = 4: no bf16-activation instance
    assert _elig(lib, 64, 0, 100, 64, W=100) == 0                # W % 8 != 0: no 16-byte bf16 rows
    assert _elig(lib, 64, 0, 288, 64, bs_pad=4) == 0             # batch stride not a multiple of 8
    assert _elig(lib, 64, 0, 72, 512) == 1 and _elig(lib, 64, 0, 72, 640) == 0 and _elig(lib, 64, 0, 36, 64) == 0
    assert lib.smaat_set_dsconv_impl(1) == 0                    # the shared-memory A form has no bf16 instances
    try:
        assert _elig(lib, 64, 0, 288, 64) == 0
    finally:
        assert lib.smaat_set_dsconv_impl(0) == 0


def test_dsconv_bf16_entry_points_validate_their_arguments():
    lib = S._lib.load()
    ds = lambda x0, W, y, k=2: lib.smaat_dsconv_bf16_fwd(x0, 64, 64 * 8 * W, None, 0, 0, A, None, A, A, A, y, 64 * 8 * W,  # noqa: E731
                                                          None, None, 2, 8, W, k, 64, 1, None)
    assert ds(None, 64, A) == BADARG and ds(A, 64, None) == BADARG
    assert ds(A, 60, A) == UNSUPPORTED and ds(A, 64, A, k=4) == UNSUPPORTED
    assert b"dsconv_bf16" in lib.smaat_last_error()
    # the CBAM gate needs both sc and sa
    assert lib.smaat_dsconv_bf16_fwd(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, A, 64 * 512, A, None, 2, 8, 64, 2, 64, 1,
                                     None) == BADARG
    oc = lib.smaat_dsconv_outconv_bf16_fwd
    assert oc(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, None, None, A, 2, 8, 64, 2, 64, 1, None) == BADARG
    assert oc(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, A, None, A + 1, 2, 8, 64, 2, 64, 1, None) == BADARG
    cl = lib.smaat_dsconv_classify_bf16_fwd
    assert cl(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, A, None, 33, None, A, 2, 8, 64, 2, 64, 1, None) == UNSUPPORTED
    assert cl(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, A, None, 0, None, A, 2, 8, 64, 2, 64, 1, None) == BADARG
    assert cl(A, 64, 64 * 512, None, 0, 0, A, None, A, A, A, A, None, 21, None, None, 2, 8, 64, 2, 64, 1, None) == BADARG


def test_cbam_upsample_and_head_entry_points_validate_their_arguments():
    lib = S._lib.load()
    pm = lambda x, H, W, C=64, pooled=A: lib.smaat_cbam_pool_mlp_bf16_fwd(x, A, A, pooled, 1, A, A, A, A, A, A, 2, C, H, W, 4,  # noqa: E731
                                                                          None)
    assert pm(None, 8, 8) == BADARG and pm(A, 8, 8, pooled=None) == BADARG
    assert pm(A, 7, 8) == UNSUPPORTED and pm(A, 8, 6) == UNSUPPORTED and pm(A, 8, 8, C=60) == UNSUPPORTED
    assert pm(A + 4, 8, 8) == UNSUPPORTED                        # 8-byte loads of four bf16 columns
    mp = lib.smaat_cbam_pool_maxpool_bf16_fwd
    assert mp(A, A, A, None, 1, 4, 8, 8, None) == BADARG and mp(A, A, A, A, 1, 4, 9, 8, None) == UNSUPPORTED
    assert mp(A, A, A, A + 4, 0, 4, 8, 8, None) == UNSUPPORTED   # an fp32 max-pool takes 8-byte stores
    assert lib.smaat_cbam_reduce_bf16_fwd(None, A, A, 2, 64, 64, None) == BADARG
    assert lib.smaat_cbam_reduce_bf16_fwd(A, A, A, 70000, 64, 64, None) == BADARG
    up = lambda y, Ho, Wo, ybs=None: lib.smaat_upsample2x_pad_bf16_fwd(A, 0, y, ybs or 4 * Ho * Wo, 2, 4, 8, 8, Ho, Wo, None)  # noqa: E731
    assert up(None, 16, 16) == BADARG and up(A, 15, 16) == BADARG and up(A, 16, 16, ybs=10) == BADARG
    assert up(A, 18, 18) == UNSUPPORTED and up(A + 2, 16, 16) == UNSUPPORTED
    assert lib.smaat_outconv_bf16_fwd(None, A, None, A, 2, 64, 1, 64, None) == BADARG
    assert lib.smaat_outconv_bf16_fwd(A + 1, A, None, A, 2, 64, 1, 64, None) == BADARG
    for f in (lib.smaat_argmax_channels_bf16_fwd, lib.smaat_softmax_channels_bf16_fwd):
        assert f(A, A, 2, 0, 64, None) == BADARG and f(A, A, 2, 1025, 64, None) == UNSUPPORTED
        assert f(None, A, 2, 4, 64, None) == BADARG and f(A + 1, A, 2, 4, 64, None) == BADARG
    assert lib.smaat_argmax_channels_bf16_fwd(A, A + 4, 2, 4, 64, None) == BADARG


def _x(shape=(2, 12, 64, 64)):
    return torch.zeros(shape, dtype=BF)


def test_requests_without_a_bf16_route_raise_naming_the_supported_entry_points():
    model = S.SmaAt_UNet(12, 1).eval()
    with torch.no_grad():
        for call in (lambda: model(_x()), lambda: model.forward_serving(_x((2, 12, 64, 48))),
                     lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=4).eval().forward_serving(_x()),
                     lambda: S.SmaAt_UNet(12, 1, bilinear=False).eval().forward_classes(_x()),
                     lambda: S.UNet(12, 1).eval().forward_serving(_x()), lambda: S.UNet(12, 1)(_x()),
                     lambda: S.UNetAttention(12, 1).eval().forward_probs(_x()), lambda: S.UNetAttention(12, 1)(_x())):
            with pytest.raises(ValueError, match="forward_serving / forward_classes / forward_probs"):
                call()
        model.train()
        with pytest.raises(ValueError, match="train mode"):
            model.forward_serving(_x())
    model.eval()
    with pytest.raises(ValueError, match="autograd"):
        model.forward_serving(_x())


def test_session_dtype_and_byte_counts():
    with pytest.raises(ValueError, match="dtype"):
        InferenceSession(S.SmaAt_UNet(12, 1), 2, (12, 64, 64), dtype=torch.float16)
    # the byte counts follow the buffers' shapes and dtypes (meta tensors: no device needed)
    sess = InferenceSession.__new__(InferenceSession)
    sess.batch, sess.dtype, sess.in_shape = 32, BF, (12, 288, 288)
    sess.static_in = torch.empty((32, 12, 288, 288), dtype=BF, device="meta")
    sess._outs = {32: torch.empty((32, 1, 288, 288), dtype=BF, device="meta")}
    assert sess.h2d_bytes_per_step == 32 * 12 * 288 * 288 * 2
    assert sess.d2h_bytes_per_step == 32 * 288 * 288 * 2
    sess._outs = {32: torch.empty((32, 288, 288), dtype=torch.int64, device="meta")}
    assert sess.d2h_bytes_per_step == 32 * 288 * 288 * 8
    with pytest.raises(ValueError, match="bfloat16"):
        sess._rows(torch.empty((2, 12, 288, 288), device="meta"))


def test_ops_accept_bf16_only_on_the_route():
    x = torch.zeros((2, 4, 8, 8), dtype=BF)
    with pytest.raises(RuntimeError, match="float32"):
        ops._req(x, "x")
    with pytest.raises(RuntimeError, match="CUDA"):          # accepted dtype, still no CPU fallback
        ops._req(x, "x", bf16=True)
