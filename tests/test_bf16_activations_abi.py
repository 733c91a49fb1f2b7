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


def _model_ds_convs(n_ch, n_cls, H, W):
    """(name, C0, C1, Cout, H, W, ncls) of SmaAt_UNet(n_ch, n_cls)'s level 1-3 DS convs on an H x W input (C1: the upsampled
    half of the decoder's virtual concat; ncls: the classes of the OutConv up4's last conv carries for class maps, else 0)."""
    convs = []
    for blk, s, cin, mid, cout, cat in (("inc", 1, n_ch, 64, 64, False), ("down1", 2, 64, 128, 128, False),
                                        ("down2", 4, 128, 256, 256, False), ("up2", 4, 512, 256, 128, True),
                                        ("up3", 2, 256, 128, 64, True), ("up4", 1, 128, 64, 64, True)):
        C0, C1 = (cin // 2, cin // 2) if cat else (cin, 0)
        convs.append((f"{blk}.0", C0, C1, mid, H // s, W // s, 0))
        convs.append((f"{blk}.1", mid, 0, cout, H // s, W // s, 0))
    if n_cls <= 32:
        convs.append(("up4.1+outc", 64, 0, 64, H, W, n_cls))
    return convs


def test_the_bf16_shape_check_admits_only_what_every_level_1_3_conv_takes():
    """For H, W multiples of 32 up to 640: an input shape SmaAt_UNet's bf16 route admits has every level 1-3 DS conv (and the
    class-map head) taken by the bf16 kernel, so a request it admits never stops half-way on a declined layer.  W = 32 is
    refused: its 8-wide level-3 maps waste half of a 16- or 32-pixel patch."""
    from smaat_unet_b200.model import bf16_shape_refusal
    lib = S._lib.load()
    sizes = range(32, 641, 32)
    for k in (1, 2):
        for n_ch, n_cls in ((12, 1), (3, 21), (1, 2)):
            for H in sizes:
                for W in sizes:
                    admitted = bf16_shape_refusal((2, n_ch, H, W)) is None
                    assert admitted == (W >= 64), (H, W)
                    if not admitted:
                        continue
                    for name, C0, C1, Cout, h, w, ncls in _model_ds_convs(n_ch, n_cls, H, W):
                        if k == 1 and C1 and C0 % 32:
                            continue     # no concat conv of the model has C0 < 32
                        got = lib.smaat_dsconv_bf16_eligible(A, C0, C0 * h * w, A if C1 else None, C1, C1 * h * w, A, h, w, k, Cout,
                                                             ncls)
                        assert got == 1, (k, n_ch, n_cls, H, W, name)
    # the check and the kernel agree on why: at W = 32, level 3 (8 wide) is what the kernel declines
    assert _elig(lib, 128, 0, 8, 256, W=8) == 0 and _elig(lib, 256, 256, 8, 256, W=8) == 0
    assert _elig(lib, 128, 0, 16, 256, W=16) == 1


def test_w32_is_refused_before_any_device_work():
    model = S.SmaAt_UNet(12, 1).eval()
    with torch.no_grad():
        for call in (model.forward_serving, model.forward_classes, model.forward_probs):
            with pytest.raises(ValueError, match="level-3 maps are 8 wide"):
                call(_x((2, 12, 64, 32)))
        # a 32-row, 64-column image is admitted: it fails later, at the first kernel, because x is on the CPU
        with pytest.raises(RuntimeError, match="CUDA"):
            model.forward_serving(_x((1, 12, 32, 64)))


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
