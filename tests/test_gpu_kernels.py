"""-m gpu: every kernel behind the C ABI vs the numpy oracle on the same seeded inputs."""
import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle import smaat_oracle as O
from smaat_unet_b200 import ops
from tests._util import PW_TOL, assert_close, dev

pytestmark = pytest.mark.gpu
RNG = np.random.default_rng(1234)


def rnd(*shape, lo=-1.0, hi=1.0):
    return RNG.uniform(lo, hi, shape).astype(np.float32)


# ------------------------------------------------------------------------------ depthwise
DW_CASES = [
    # B, C0, C1, H, W, k, loaders
    (2, 5, 0, 9, 11, 1, (0, 1)),        # W % 4 != 0 -> LDG loader / one-warp-per-plane kernel (auto)
    (2, 6, 0, 12, 8, 2, (1, 2)),
    (1, 4, 0, 7, 5, 3, (1,)),           # generic k
    (2, 3, 5, 16, 20, 2, (1, 2)),       # virtual concat
    (1, 8, 0, 18, 18, 2, (0, 1)),       # the 18x18 layers (72-byte rows: no TMA): auto = one warp per plane
    (3, 5, 4, 18, 18, 2, (0, 1)),       # ... over a virtual concat, several images
    (2, 4, 0, 36, 36, 2, (1, 2)),
    (1, 3, 0, 72, 72, 2, (1, 2)),
    (1, 2, 2, 144, 144, 2, (1, 2)),
    (1, 3, 0, 288, 288, 2, (1, 2)),
    (1, 2, 0, 100, 148, 1, (1, 2)),     # W = 4*37: no nice divisor -> 64-wide tiles with a ragged edge
    (1, 2, 0, 40, 576, 2, (1, 2)),
]


@pytest.mark.parametrize("case", DW_CASES)
def test_dw3x3_matches_oracle(case):
    B, C0, C1, H, W, k, loaders = case
    C = C0 + C1
    x = rnd(B, C, H, W)
    w = rnd(k * C, 1, 3, 3)
    b = rnd(k * C)
    ref = O.depthwise3x3(x.astype(np.float64), w, b, k)
    x0 = dev(x[:, :C0])
    x1 = dev(x[:, C0:]) if C1 else None
    outs = []
    for ld in loaders:
        y = ops.dw3x3(x0, dev(w), dev(b), k, x1=x1, loader=ld)
        torch.cuda.synchronize()
        assert_close(y, ref, 2e-6, f"dw3x3 loader={ld} {case}")
        outs.append(y)
    if len(outs) == 2:   # TMA-staged and LDG-staged tiles must agree bit for bit
        assert torch.equal(outs[0], outs[1])
    y = ops.dw3x3(x0, dev(w), None, k, x1=x1)      # no bias
    assert_close(y, O.depthwise3x3(x.astype(np.float64), w, None, k), 2e-6, "dw3x3 no-bias")


@pytest.mark.parametrize("loader", [0, 1, 2])
def test_dw3x3_prologue_bn_relu_then_zero_pad(loader):
    B, C, H, W, k = (2, 6, 12, 16, 2) if loader else (2, 6, 9, 10, 2)     # loader 0 on a W % 4 != 0 plane: one-warp-per-plane kernel
    x, w, b = rnd(B, C, H, W), rnd(k * C, 1, 3, 3), rnd(k * C)
    s, t = rnd(C, lo=0.5, hi=1.5), rnd(C)
    act = np.maximum(x.astype(np.float64) * s[None, :, None, None] + t[None, :, None, None], 0)
    ref = O.depthwise3x3(act, w, b, k)
    y = ops.dw3x3(dev(x), dev(w), dev(b), k, in_scale=dev(s), in_shift=dev(t), loader=loader)
    assert_close(y, ref, 2e-6, "dw3x3 prologue")


def test_dw3x3_batch_strided_input():
    # reading a channel slice of a wider tensor through the batch stride (no copy)
    B, Cw, C, H, W = 2, 10, 4, 8, 8
    wide = dev(rnd(B, Cw, H, W))
    x = wide[:, 2:2 + C]
    w, b = rnd(2 * C, 1, 3, 3), rnd(2 * C)
    ref = O.depthwise3x3(x.double().cpu().numpy(), w, b, 2)
    for ld in (1, 2):
        assert_close(ops.dw3x3(x, dev(w), dev(b), 2, loader=ld), ref, 2e-6, f"dw3x3 strided loader={ld}")


# ------------------------------------------------------------------------------ pointwise
PW_CASES = [
    # B, K, Cout, H, W
    (2, 24, 64, 16, 16),      # inc.0 shape class (single k-chunk, K < 32)
    (1, 128, 64, 32, 32),     # inc.3 / up4.3
    (2, 128, 128, 16, 24),
    (1, 256, 128, 16, 16),
    (1, 256, 256, 12, 12),    # N_TILE 256, P = 144 (ragged M tile)
    (2, 512, 256, 8, 8),      # P = 64 < 128
    (1, 1024, 512, 18, 18),   # down4 shape: P = 324, two N tiles
    (1, 2048, 512, 6, 6),     # up1.0 K
    (1, 40, 24, 8, 12),       # K % 32 != 0 tail, Cout < N_TILE
    (2, 16, 16, 5, 7),        # P % 4 != 0 -> exact CUDA-core kernel in every mode
]


@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
@pytest.mark.parametrize("case", PW_CASES)
def test_pw1x1_matches_oracle(case, mode):
    B, K, Cout, H, W = case
    x, w = rnd(B, K, H, W), rnd(Cout, K, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    acc = O.pointwise1x1(x.astype(np.float64), w, None)
    ref = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    y = ops.pw1x1(dev(x), dev(w), dev(scale), dev(shift), True, mode=mode)
    torch.cuda.synchronize()
    assert_close(y, ref, PW_TOL[mode], f"pw1x1 {mode} {case}")
    # no affine, no relu: plain conv + nothing
    y2 = ops.pw1x1(dev(x), dev(w), None, None, False, mode=mode)
    assert_close(y2, acc, PW_TOL[mode], f"pw1x1 plain {mode} {case}")


@pytest.mark.parametrize("mode", ["fp32", "tf32x3"])
def test_pw1x1_stats_and_strided_output(mode):
    B, K, Cout, H, W = 2, 64, 48, 12, 12
    x, w, bias = rnd(B, K, H, W), rnd(Cout, K, 1, 1, lo=-0.3, hi=0.3), rnd(Cout)
    pre = O.pointwise1x1(x.astype(np.float64), w, bias)
    stats = torch.zeros(2 * Cout, device="cuda", dtype=torch.float64)
    wide = torch.zeros(B, Cout + 8, H, W, device="cuda")
    out = wide[:, 8:]
    ops.pw1x1(dev(x), dev(w), None, dev(bias), False, mode=mode, stats=stats, out=out)
    assert_close(out, pre, PW_TOL[mode], "pw1x1 strided out")
    assert float(wide[:, :8].abs().max()) == 0.0
    assert_close(stats[:Cout], pre.sum(axis=(0, 2, 3)), 1e-4, "channel sums")
    assert_close(stats[Cout:], (pre ** 2).sum(axis=(0, 2, 3)), 1e-4, "channel sums of squares")


def test_split_tf32_is_exact():
    w = dev(rnd(1000))
    hi, lo = ops.split_tf32(w)
    assert torch.equal(hi + lo, w)
    assert int((hi.view(torch.int32) & 0x1FFF).abs().max()) == 0


# ------------------------------------------------------------------------------ glue
@pytest.mark.parametrize("shape", [(2, 3, 8, 8), (1, 2, 13, 18), (2, 4, 36, 36), (1, 2, 7, 9), (1, 2, 288, 288)])
def test_maxpool2(shape):
    x = rnd(*shape)
    y = ops.maxpool2(dev(x))
    assert np.array_equal(y.cpu().numpy(), O.maxpool2(x))       # bit-exact: pure selection


@pytest.mark.parametrize("case", [((2, 3, 6, 8), 12, 16), ((1, 2, 4, 6), 9, 13), ((1, 2, 18, 18), 36, 36), ((1, 1, 1, 1), 2, 2),
                                  ((1, 2, 5, 5), 11, 10)])
def test_upsample2x_pad(case):
    shape, Ho, Wo = case
    x = rnd(*shape)
    ref = O.pad_to(O.upsample_bilinear2x(x.astype(np.float64)), Ho, Wo)
    assert_close(ops.upsample2x_pad(dev(x), Ho, Wo), ref, 2e-6, f"upsample {case}")


@pytest.mark.parametrize("case", [(2, 64, 1, 16, 16), (1, 64, 5, 8, 12), (1, 64, 21, 9, 7), (2, 16, 2, 6, 6)])
def test_outconv(case):
    B, Cin, ncls, H, W = case
    x, w, b = rnd(B, Cin, H, W), rnd(ncls, Cin, 1, 1, lo=-0.3, hi=0.3), rnd(ncls)
    assert_close(ops.outconv(dev(x), dev(w), dev(b)), O.pointwise1x1(x.astype(np.float64), w, b), 1e-5, f"outconv {case}")


def test_bn_fold():
    C = 70
    g, b, rm, rv, cb = rnd(C, lo=0.5, hi=1.5), rnd(C), rnd(C), rnd(C, lo=0.5, hi=1.5), rnd(C)
    s, t = ops.bn_fold(dev(g), dev(b), dev(rm), dev(rv), dev(cb), 1e-5)
    es = g.astype(np.float64) / np.sqrt(rv.astype(np.float64) + 1e-5)
    assert_close(s, es, 1e-6, "bn scale")
    assert_close(t, b + (cb.astype(np.float64) - rm) * es, 1e-6, "bn shift")


# ------------------------------------------------------------------------------ CBAM pieces
@pytest.mark.parametrize("shape", [(2, 32, 14, 10), (1, 64, 9, 9), (2, 16, 72, 72), (1, 8, 36, 36), (1, 4, 288, 288), (2, 32, 18, 18)])
def test_cbam_pool_reduce_scale(shape):
    B, C, H, W = shape
    x = rnd(*shape)
    avg, mx = ops.cbam_pool(dev(x))
    assert_close(avg, x.astype(np.float64).mean(axis=(2, 3)), 1e-5, "cbam avg")
    assert np.array_equal(mx.cpu().numpy(), x.max(axis=(2, 3)))
    sc = rnd(B, C, lo=0.1, hi=1.0)
    xs = x.astype(np.float64) * sc[:, :, None, None]
    pooled = ops.cbam_reduce(dev(x), dev(sc))
    assert_close(pooled[:, 0], xs.mean(axis=1), 1e-5, "cbam channel mean")
    assert_close(pooled[:, 1], xs.max(axis=1), 1e-6, "cbam channel max")
    sa = rnd(B, 1, H, W, lo=0.1, hi=1.0)
    assert_close(ops.cbam_scale(dev(x), dev(sc), dev(sa)), xs * sa, 1e-6, "cbam scale")


@pytest.mark.parametrize("ks", [3, 7])
def test_cbam_gate(ks):
    B, H, W = 2, 37, 45
    pooled, w = rnd(B, 2, H, W), rnd(1, 2, ks, ks, lo=-0.3, hi=0.3)
    aff = np.array([1.3, -0.2], dtype=np.float32)
    a = O.conv2d_same(pooled.astype(np.float64), w, ks // 2)
    sa, raw = ops.cbam_gate(dev(pooled), dev(w), dev(aff), want_raw=True)
    assert_close(raw, a, 1e-5, "gate conv")
    assert_close(sa, O.sigmoid(a * 1.3 - 0.2), 1e-5, "gate sigmoid")


# ------------------------------------------------------------------------------ fused depthwise -> pointwise
DS_CASES = [
    # B, C0, C1, H, W, k, Cout
    (2, 12, 0, 32, 32, 2, 64),     # inc.0 class: Cin < chunk (zero-filled channels), single chunk
    (1, 64, 0, 32, 64, 2, 64),     # K = 128, 32-wide patches
    (1, 64, 0, 48, 48, 2, 128),    # 16-wide patches (48 % 32 != 0), N_TILE 128
    (1, 16, 16, 16, 32, 2, 32),    # virtual concat, Cout < N_TILE
    (2, 32, 0, 24, 32, 1, 48),     # k = 1 (32 input channels per chunk), ragged channel tail
    (1, 8, 0, 36, 52, 2, 16),      # ragged patches in x and y
    (1, 128, 128, 16, 16, 2, 64),  # K = 512: many chunks, both producer groups, concat boundary mid-loop
    (3, 24, 0, 8, 96, 2, 40),      # odd chunk count (3 per tile) -> groups alternate across tiles
    (8, 16, 0, 128, 128, 2, 64),   # 1024 tiles: 7-8 per CTA -> every ring wraps many times across tiles
    (8, 16, 0, 128, 64, 2, 128),   # 512 tiles, N_TILE 128: one producer group feeds several tiles per CTA
    (2, 32, 32, 40, 72, 2, 96),    # ragged right / bottom patches, concat, Cout between the tile sizes
    (2, 32, 0, 32, 32, 2, 256),    # Cout = 256: two output-channel passes of 128 over the same patches
    (1, 48, 16, 16, 64, 2, 512),   # Cout = 512: four passes, concat
]


@pytest.fixture(params=["smem", "regs"])
def ds_impl(request):
    """Both ways the fused kernel hands the depthwise result to the tensor core behind the same ABI entry: K-major tiles
    that wgmma reads from shared memory / tiles loaded into registers for wgmma's register-A form."""
    ops.set_dsconv_impl(request.param)
    yield request.param
    ops.set_dsconv_impl("auto")


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", DS_CASES)
def test_dsconv_fused_matches_oracle(case, mode, ds_impl):
    B, C0, C1, H, W, k, Cout = case
    C = C0 + C1
    x = rnd(B, C, H, W)
    dw_w, dw_b = rnd(k * C, 1, 3, 3), rnd(k * C)
    pw_w = rnd(Cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    d = O.depthwise3x3(x.astype(np.float64), dw_w, dw_b, k)
    acc = O.pointwise1x1(d, pw_w, None)
    ref = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    x0 = dev(x[:, :C0])
    x1 = dev(x[:, C0:]) if C1 else None
    y = ops.dsconv(x0, dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True, x1=x1, mode=mode)
    assert y is not None, f"fused kernel refused an eligible shape {case}"
    torch.cuda.synchronize()
    assert_close(y, ref, PW_TOL[mode], f"dsconv {mode} {case}")
    # no bias / no affine / no relu (+ statistics: Cout <= 128, all channels in one pass)
    pre = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, None, k), pw_w, None)
    if Cout > 128:
        y2 = ops.dsconv(x0, dev(dw_w), None, k, dev(pw_w), None, None, False, x1=x1, mode=mode)
        assert_close(y2, pre, PW_TOL[mode], f"dsconv plain {mode} {case}")
        return
    stats = torch.zeros(2 * Cout, device="cuda", dtype=torch.float64)
    y2 = ops.dsconv(x0, dev(dw_w), None, k, dev(pw_w), None, None, False, x1=x1, mode=mode, stats=stats)
    assert_close(y2, pre, PW_TOL[mode], f"dsconv plain {mode} {case}")
    assert_close(stats[:Cout], pre.sum(axis=(0, 2, 3)), 2e-3 if mode == "tf32" else 1e-4, "dsconv channel sums")


@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", [DS_CASES[1], DS_CASES[2], DS_CASES[3], DS_CASES[5], DS_CASES[8]])
def test_dsconv_with_fused_outconv_matches_oracle(case, mode, ds_impl):
    """smaat_dsconv_outconv_fwd: DS conv -> BN/ReLU -> OutConv(Cout -> 1) with the activation kept in registers."""
    B, C0, C1, H, W, k, Cout = case
    C = C0 + C1
    x = rnd(B, C, H, W)
    dw_w, dw_b = rnd(k * C, 1, 3, 3), rnd(k * C)
    pw_w = rnd(Cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    ow, ob = rnd(1, Cout, 1, 1), rnd(1)
    acc = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, dw_b, k), pw_w, None)
    act = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    ref = O.pointwise1x1(act, ow, ob)
    x0 = dev(x[:, :C0])
    x1 = dev(x[:, C0:]) if C1 else None
    y = ops.dsconv(x0, dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True, x1=x1, mode=mode, outconv=(dev(ow), dev(ob)))
    assert y is not None and tuple(y.shape) == (B, 1, H, W)
    assert_close(y, ref, PW_TOL[mode], f"dsconv+outconv {mode} {case}")
    y = ops.dsconv(x0, dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True, x1=x1, mode=mode, outconv=(dev(ow), None))
    assert_close(y, ref - ob[0], PW_TOL[mode], f"dsconv+outconv without bias {mode} {case}")


def test_dsconv_ineligible_shapes_fall_back():
    # Cout > 128 / tiny planes are not fused: ops.dsconv says so and the module path still gives the right answer
    assert ops.dsconv(dev(rnd(1, 16, 8, 8)), dev(rnd(32, 1, 3, 3)), None, 2, dev(rnd(256, 32, 1, 1)), None, None, False) is None
    # Cout = 256 is fused in passes of 128, but the fused OutConv needs every channel in one pass: declined, not an error
    x32, w256 = dev(rnd(1, 16, 32, 32)), dev(rnd(256, 32, 1, 1))
    assert ops.dsconv(x32, dev(rnd(32, 1, 3, 3)), None, 2, w256, None, None, True) is not None
    assert ops.dsconv(x32, dev(rnd(32, 1, 3, 3)), None, 2, w256, None, None, True, outconv=(dev(rnd(1, 256, 1, 1)), None)) is None
    m = S.DepthwiseSeparableConv(16, 256, 3, padding=1, kernels_per_layer=2).cuda().eval()
    x = rnd(1, 16, 18, 18)
    sd = {k_: v.detach().cpu().numpy() for k_, v in m.state_dict().items()}
    ref = O.ds_conv(x.astype(np.float64), {"m." + k_: v for k_, v in sd.items()}, "m", 2)
    with torch.no_grad():
        assert_close(m(dev(x)), ref, PW_TOL["tf32x3"], "unfused fallback")


def test_dsconv_with_batch_statistics_only_where_a_kernel_has_them():
    """smaat_dsconv_eligible2(with_stats): batch statistics need all channels in one pass, so a request with `stats` is
    either taken by the fused kernel (Cout <= 128) or declined (Cout = 256, passes of 128) -- never an error -- and
    DepthwiseSeparableConv.run(stats=...) gives the same result and the same sums either way."""
    for cout, fused in ((64, True), (256, False)):
        m = S.DepthwiseSeparableConv(16, cout, 3, padding=1, kernels_per_layer=2).cuda().eval()
        x = dev(rnd(2, 16, 32, 32))
        assert m.fused_takes(x) is True                      # without statistics both shapes are fused (Cout 256: passes of 128)
        assert m.fused_takes(x, stats=True) is fused
        with torch.no_grad():
            st = ops.new_stats(cout, x.device)
            z = m.run(x, stats=st)
            ref = m(x)
        assert_close(z, ref.double().cpu().numpy(), 1e-5, f"run(stats) Cout={cout}")
        zs = z.double()
        sums = torch.stack([zs.sum(dim=(0, 2, 3)), (zs * zs).sum(dim=(0, 2, 3))]).reshape(-1)
        assert_close(st, sums.cpu().numpy(), 1e-5, f"batch statistics Cout={cout}")


@pytest.mark.parametrize("shape", [(2, 3, 8, 12), (1, 5, 64, 64), (2, 2, 288, 288), (3, 4, 18, 20)])
def test_cbam_pool_with_fused_maxpool(shape):
    """smaat_cbam_pool_maxpool_fwd: global avg/max pools and MaxPool2d(2) from one read (layers.py:107-108, parts_ds.py:48)."""
    x = rnd(*shape)
    avg, mx, pooled = ops.cbam_pool_maxpool(dev(x))
    B, C, H, W = shape
    assert_close(avg, x.astype(np.float64).mean(axis=(2, 3)), 1e-5, "avg")
    assert np.array_equal(mx.cpu().numpy(), x.max(axis=(2, 3)))
    ref = x.reshape(B, C, H // 2, 2, W // 2, 2).max(axis=(3, 5))
    assert np.array_equal(pooled.cpu().numpy(), ref)
    assert ops.cbam_pool_maxpool(dev(rnd(1, 2, 9, 12))) is None and ops.cbam_pool_maxpool(dev(rnd(1, 2, 8, 10))) is None


# ------------------------------------------------------------------------------ CBAM in three launches
@pytest.mark.parametrize("shape,hidden,with_pool", [((2, 64, 64, 64), 4, True), ((3, 128, 18, 18), 8, False), ((2, 512, 12, 16), 32, True),
                                                    ((1, 256, 72, 72), 16, True), ((4, 8, 6, 8), 2, True)])
def test_cbam_pool_mlp_one_launch(shape, hidden, with_pool):
    """smaat_cbam_pool_mlp_fwd: the last pooling CTA of an image finishes the shared MLP + sigmoid (layers.py:98-109), both
    plane-size variants, with and without the fused 2x2 max-pool; twice in a row (the counters must come back at zero)."""
    B, C, H, W = shape
    x = rnd(*shape)
    w1, b1, w2, b2 = rnd(hidden, C, lo=-0.3, hi=0.3), rnd(hidden), rnd(C, hidden, lo=-0.3, hi=0.3), rnd(C)
    x64 = x.astype(np.float64)
    avg_r, mx_r = x64.mean(axis=(2, 3)), x64.max(axis=(2, 3))
    mlp = lambda v: np.maximum(v @ w1.astype(np.float64).T + b1, 0) @ w2.astype(np.float64).T + b2   # noqa: E731
    sc_r = O.sigmoid(mlp(avg_r) + mlp(mx_r))
    for rep in range(2):
        got = ops.cbam_pool_mlp(dev(x), dev(w1), dev(b1), dev(w2), dev(b2), with_maxpool=with_pool)
        assert got is not None
        sc, avg, mx, pooled = got
        torch.cuda.synchronize()
        assert_close(avg, avg_r, 1e-5, "avg")
        assert np.array_equal(mx.cpu().numpy(), x.max(axis=(2, 3)))
        assert_close(sc, sc_r, 1e-5, f"channel gate (call {rep})")
        if with_pool and W % 4 == 0 and H % 2 == 0:
            assert np.array_equal(pooled.cpu().numpy(), x.reshape(B, C, H // 2, 2, W // 2, 2).max(axis=(3, 5)))
        else:
            assert pooled is None
        assert int(ops._counters(torch.device("cuda", torch.cuda.current_device()), B).abs().sum()) == 0
    assert ops.cbam_pool_mlp(dev(rnd(1, 12, 8, 8)), dev(rnd(2, 12)), dev(rnd(2)), dev(rnd(12, 2)), dev(rnd(12))) is None   # C % 8


@pytest.mark.parametrize("ks", [3, 7])
@pytest.mark.parametrize("shape", [(2, 64, 40, 72), (1, 512, 18, 20), (3, 24, 33, 36), (1, 8, 288, 288)])
def test_cbam_gate_scale_one_launch(shape, ks):
    """smaat_cbam_gate_scale_fwd = smaat_cbam_gate_fwd + smaat_cbam_scale_fwd (layers.py:126-128, :110), any channel split."""
    B, C, H, W = shape
    x, sc = rnd(*shape), rnd(B, C, lo=0.1, hi=1.0)
    pooled, w = rnd(B, 2, H, W), rnd(1, 2, ks, ks, lo=-0.3, hi=0.3)
    aff = np.array([1.3, -0.2], dtype=np.float32)
    gate = O.sigmoid(O.conv2d_same(pooled.astype(np.float64), w, ks // 2) * 1.3 - 0.2)
    ref = x.astype(np.float64) * sc[:, :, None, None] * gate
    y = ops.cbam_gate_scale(dev(x), dev(sc), dev(pooled), dev(w), dev(aff))
    assert y is not None
    assert_close(y, ref, 1e-5, f"gate+scale {shape} k{ks}")
    # into a channel slice of a wider tensor (batch stride > C*H*W), as the virtual-concat consumers use it
    wide = torch.zeros(B, C + 8, H, W, device="cuda")
    ops.cbam_gate_scale(dev(x), dev(sc), dev(pooled), dev(w), dev(aff), out=wide[:, 8:])
    assert_close(wide[:, 8:], ref, 1e-5, "gate+scale into a slice")
    assert float(wide[:, :8].abs().max()) == 0.0
    assert ops.cbam_gate_scale(dev(rnd(1, 8, 6, 10)), dev(rnd(1, 8)), dev(rnd(1, 2, 6, 10)), dev(w), dev(aff)) is None   # W % 4
