"""SmaAt-UNet's bf16 storage route against float64 at its edges.

tests/test_gpu_bf16_activations.py checks the bf16-activation kernels at the layer shapes of two square networks (288^2 with
12 channels, 224^2 with 3), k = 2.  This file adds the shapes where those kernels go wrong:

  A  the fused DS conv on bf16 activations (ops.dsconv_bf16, ops.dsconv_head_bf16): W < PW (24 wide, level 3 of a 96-px
     image, PW 32), odd H (99 x 96), partial tiles both ways at Cout 40 (70 x 104, PW 16), Cout 8 at odd H, tall and narrow
     (300 x 16) and wide and short (8 x 200), Cout 384 (three 128-channel passes), 1- and 3-channel inputs at k = 1 and 2
     (K padded to 32 in the pack), the virtual concat with one 16- or 32-channel chunk of x0 and an odd C1, B = 1 and 5,
     batch-strided channel slices (and one whose batch stride is not a multiple of 8, refused before any launch), relu off,
     and the CBAM gate with an sa band of exact 0s on some rows, exact 1s on some columns and sc = 0 on every fifth channel.
     Heads at W < PW and odd H: the one-class OutConv and the class map at K = 2, 21 and 32 (K = 33 is declined).  Through
     the C ABI, the partial-tile outputs and the heads are written into NaN-poisoned buffers with guard tails (y with a
     batch stride larger than Cout H W, over-allocated logits and class maps), and nothing outside the image's region may
     change
  B  CBAM from bf16: the pools + MLP + max-pool on planes under 2 048 pixels (8 planes per CTA and its MLP tail), the
     pools + max-pool with B C not a multiple of 8, the channel reduce at P % 4 != 0, C = 13, P = 8 188 / 8 192 (each side
     of its float4 switch) and B = 7
  C  the upsample to bf16 from fp32 and bf16 with odd vertical pads (Ho = 2H + 1, 2H + 3), Wo = 2W + 4, odd W, 1-row and
     1-column sources; a Wo that is not a multiple of 4 is refused without a write
  D  the unfused heads on bf16: OutConv at K = 1, 2, 9 with and without P % 4 == 0 (also into a guarded buffer), the argmax
     with exact ties, NaN and +-inf logits, K = 1 and 1024 and more pixels than one grid pass, the softmax at K = 2, 21 and
     1024 with torch's NaN / 0 / 1 pattern on non-finite rows
  E  whole networks through InferenceSession(dtype=torch.bfloat16): non-square, k = 1, 1-channel input, 2 classes and 40
     classes (the unfused class and probability heads on bf16 maps), odd B with a captured partial batch
  F  W = 32 is refused before any launch (its level-3 maps are 8 wide, which the fused bf16 DS conv does not tile)

Two oracles for every DS conv case (A):
  1. float64 on the same bf16 inputs (``_ds_ref``), within one bf16 ulp of the once-rounded result plus the fused DS conv's
     fp32 accumulation bound (``_one_ulp``); class maps exact where the top two logits are clearly apart;
  2. the fp32-storage fused kernel in 'bf16' mode on the same values, rounded to bf16 once: bit-equal.  The two instances
     share pick_pw, N_TILE, the chunk order, the stencil, the __fmul_rn gate and the epilogue formula; only the storage type
     differs.  Where the fp32 kernel does not take the shape (K = k (C0 + C1) not a multiple of 4: C0 = 1 or 3, C1 = 3 at
     k = 1) only oracle 1 applies.  The heads compare with ops.dsconv(outconv=...) and ops.dsconv_classify in 'bf16' mode.

Oracle 2 held bit for bit at every shape where the fp32 kernel runs, gated or not, heads included.  Bounds were set from
the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x above it; everything
else is bit-exact and was:

  quantity                                                      worst observed                   bound
  A  DS conv y, heads' logits: |err| / (1 ulp + 1.5e-5 max)     0.498 (24^2 concat + gate)       1
  B  pool avg (8 planes per CTA, 39 planes)                     1.2e-7                           1e-6
     MLP gate sc                                                2.6e-7                           2e-6
     reduce mean / max                                          3.3e-7 / 4.5e-8                  2e-6 / 2e-7
  C  upsample to bf16: |err| / (1 ulp + coordinate term)        0.500 (7 -> 16 columns)          1
  D  outconv / softmax: |err| / (1 ulp + atol)                  0.492 / 0.499                    1
  E  logits vs emulated port / unrounded port, max over nets    6.1e-3 / 6.7e-3                  1.5e-2 - 2e-2 (per net)
     probabilities vs emulated port                             4.0e-3 (64 x 96, 2 classes)      1e-2
     class map agreement with the emulated port                 1.00000                          >= 0.99

Mutations of the csrc, one at a time, and what failed (the existing file is tests/test_gpu_bf16_activations.py):
  * the bf16 upsample launched with pad_t = pad_l = 0: the 12 upsample cases with a top or left pad (from fp32 and bf16);
    no existing test (every map it sees is exactly 2H x 2W, and so is every map in part E);
  * the 8-planes-per-CTA pool grid as N / 8 instead of ceil_div64(N, 8): the 39-plane pool + max-pool case (bf16 and fp32
    max-pool); no existing test (every B C there is a multiple of 8);
  * the bf16 argmax with v >= m: the exact-ties and the K = 1024 / several-pass argmax tests; the existing file's
    test_unfused_heads_from_bf16 at K = 21 and 40 also failed (224^2 random bf16 logits hold exact ties);
  * the outconv scalar store with pp + q <= P: the guarded outconv at P = 63, K = 1, 2 and 9 (the write lands one element
    past the last plane); no existing test;
  * the v0 / v1 masks dropped from the fused one-class head's logit store, and, apart, from the class-map store: both
    guarded head tests (24^2 and 99 x 96: tiles that overhang the image); no existing test (their maps tile exactly).  Those
    two mutants write past every image whose tiles overhang it, so they were run on the guarded tests only.
The whole file runs in ~5 s on one H100 at a peak of 0.45 GiB allocated.
"""
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200.engine import InferenceSession
from tests.test_gpu_bf16 import _bn_randomise, _port
from tests.test_gpu_bf16_activations import DS_ATOL, HEAD_ATOL, _ds_ref, _one_ulp, _port_bf16, _sd64, r16
from tests.test_gpu_ds_forward_kernels import _check, _exact, _gen, _randn

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
NAN16 = 0x7FC0          # bf16 quiet NaN bits: the poison of the guarded buffers
UNSUPPORTED = -3
GUARD = 4096            # guard tail, in elements, past every guarded buffer


def _poisoned(n, dtype):
    """n elements of NaN bits (bf16) or -7 (int64): what a guarded buffer holds before the launch."""
    if dtype == BF:
        return torch.full((n,), NAN16, dtype=torch.int16, device="cuda").view(BF)
    return torch.full((n,), -7, dtype=torch.int64, device="cuda")


def _untouched(buf, keep, what):
    """Every element of ``buf`` outside the bool mask ``keep`` still holds its poison."""
    bits = buf.view(torch.int16) if buf.dtype == BF else buf
    poison = NAN16 if buf.dtype == BF else -7
    n = int((bits[~keep] != poison).sum())
    print(f"ERR {what}: {n} writes outside the output region")
    assert n == 0, f"{what}: {n} elements outside the output region were written"


# ============================================================================================== A: the fused DS conv on bf16
# (id, C0, C1, Cout, H, W, k, B, gate, relu)
DS_CASES = [
    ("wltpw_24", 256, 0, 256, 24, 24, 2, 2, False, True),
    ("wltpw_24_cat_gate", 256, 256, 256, 24, 24, 2, 2, True, True),
    ("oddh_99x96", 64, 0, 64, 99, 96, 2, 2, False, True),
    ("oddh_99x96_gate", 64, 0, 64, 99, 96, 2, 2, True, True),
    ("cout40_70x104_k1", 64, 0, 40, 70, 104, 1, 2, False, True),
    ("cout8_37x40", 64, 0, 8, 37, 40, 2, 2, False, True),
    ("tall_300x16", 32, 0, 96, 300, 16, 2, 2, False, True),
    ("wide_8x200", 64, 0, 64, 8, 200, 2, 2, False, True),
    ("cout384_12x64", 64, 0, 384, 12, 64, 2, 2, False, True),
    ("c1_64x96_k1", 1, 0, 64, 64, 96, 1, 2, False, True),
    ("c1_64x96_k2", 1, 0, 64, 64, 96, 2, 2, False, True),
    ("c3_96x160_k1", 3, 0, 64, 96, 160, 1, 2, False, True),
    ("cat_16_24_k2", 16, 24, 64, 40, 56, 2, 2, False, True),
    ("cat_32_3_k1", 32, 3, 64, 40, 56, 1, 2, False, True),
    ("b1_oddh", 64, 0, 64, 99, 96, 2, 1, False, True),
    ("b5_cout40", 64, 0, 40, 70, 104, 1, 5, False, True),
    ("norelu_oddh", 64, 0, 64, 99, 96, 2, 2, False, False),
    ("norelu_wltpw_gate", 256, 256, 256, 24, 24, 2, 2, True, False),
]


def _gate(B, C0, H, W, g):
    """sc (B, C0) with every fifth channel 0, sa (B, 1, H, W) exactly 0 on a row band and 1 on a column band."""
    sc = torch.rand((B, C0), generator=g, device="cuda") + 0.5
    sc[:, ::5] = 0.0
    sa = torch.rand((B, 1, H, W), generator=g, device="cuda")
    sa[:, :, H // 3:H // 3 + 3] = 0.0
    sa[:, :, :, W // 2:W // 2 + 5] = 1.0
    return sc, sa


def _make(C0, C1, Cout, H, W, k, B, gate=False, relu=True, seed=0):
    g = _gen(seed + C0 * 131 + C1 * 17 + Cout * 7 + H * 3 + W + k)
    Cin, K = C0 + C1, k * (C0 + C1)
    x = r16(_randn((B, Cin, H, W), g)).float()           # bf16 values, held in fp32 for the references
    w, b = _randn((K, 1, 3, 3), g, 1.0 / 3.0), _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc = torch.rand((Cout,), generator=g, device="cuda") + 0.5
    sh = _randn((Cout,), g, 0.1) - (0.0 if relu else 0.2)     # relu off: signed outputs
    gt = _gate(B, C0, H, W, g) if gate else None
    return g, x, w, b, pw, sc, sh, gt


def _fp32_rounded(x, C0, w, b, k, pw, sc, sh, relu, gt):
    """Oracle 2: the fp32-storage fused kernel in 'bf16' mode on the same values, rounded once; None where it does not take
    the shape."""
    x0, x1 = x[:, :C0].contiguous(), (x[:, C0:].contiguous() if x.shape[1] > C0 else None)
    if gt is None:
        y = ops.dsconv(x0, w, b, k, pw, sc, sh, relu, x1=x1, mode="bf16")
    elif ops.dsconv_cbam_takes(x0, x1, pw, k, gate=True, mode="bf16"):
        y = ops.dsconv_cbam(x0, w, b, k, pw, sc, sh, relu, x1=x1, mode="bf16", gate=gt)
    else:
        y = None
    return None if y is None else y.to(BF)


@pytest.mark.parametrize("case", DS_CASES, ids=[c[0] for c in DS_CASES])
def test_dsconv_bf16_edges(case):
    name, C0, C1, Cout, H, W, k, B, gate, relu = case
    g, x, w, b, pw, sc, sh, gt = _make(C0, C1, Cout, H, W, k, B, gate, relu)
    x0, x1 = x[:, :C0].to(BF), (x[:, C0:].to(BF) if C1 else None)
    assert ops.dsconv_bf16_takes(x0, x1, pw, k)
    y = ops.dsconv_bf16(x0, w, b, k, pw, sc, sh, relu, x1=x1, gate=gt)
    assert y.dtype == BF and y.shape == (B, Cout, H, W)
    _one_ulp(y, _ds_ref(x, w, b, k, pw, sc, sh, C0, *(gt or (None, None)), relu=relu), f"dsconv bf16 {name}", DS_ATOL)
    ref2 = _fp32_rounded(x, C0, w, b, k, pw, sc, sh, relu, gt)
    if (k * (C0 + C1)) % 4 == 0:
        assert ref2 is not None, f"{name}: the fp32 kernel in 'bf16' mode should take this shape"
        _exact(y, ref2, f"dsconv bf16 {name} vs the fp32-storage kernel rounded once")
    else:
        assert ref2 is None


def test_dsconv_bf16_batch_strided_channel_slices():
    """x0 and x1 as channel slices of larger bf16 buffers (batch strides 48 H W and 40 H W): the same output as contiguous
    copies.  A view whose batch stride is not a multiple of 8 is not taken, and dsconv_bf16 raises before any launch."""
    C0, C1, Cout, H, W, k, B = 32, 32, 64, 40, 56, 2, 3
    g, x, w, b, pw, sc, sh, _ = _make(C0, C1, Cout, H, W, k, B)
    big0 = torch.randn((B, 48, H, W), generator=g, device="cuda").to(BF)
    big1 = torch.randn((B, 40, H, W), generator=g, device="cuda").to(BF)
    big0[:, 8:40] = x[:, :C0].to(BF)
    big1[:, 3:35] = x[:, C0:].to(BF)
    x0, x1 = big0[:, 8:40], big1[:, 3:35]
    assert x0.stride(0) == 48 * H * W and x1.stride(0) == 40 * H * W
    assert ops.dsconv_bf16_takes(x0, x1, pw, k)
    y = ops.dsconv_bf16(x0, w, b, k, pw, sc, sh, True, x1=x1)
    _exact(y, ops.dsconv_bf16(x0.contiguous(), w, b, k, pw, sc, sh, True, x1=x1.contiguous()), "dsconv bf16 slices vs copies")
    _one_ulp(y, _ds_ref(x, w, b, k, pw, sc, sh, C0, None, None), "dsconv bf16 channel slices", DS_ATOL)
    _exact(y, _fp32_rounded(x, C0, w, b, k, pw, sc, sh, True, None), "dsconv bf16 slices vs the fp32-storage kernel rounded once")
    # a batch stride of C0 H W + 4: 16-byte aligned rows, but not the 16-byte plane strides TMA needs
    buf = torch.zeros((B * (C0 * H * W + 4),), dtype=BF, device="cuda")
    odd = torch.as_strided(buf, (B, C0, H, W), (C0 * H * W + 4, H * W, W, 1))
    pw1 = pw[:, :k * C0].contiguous()
    assert not ops.dsconv_bf16_takes(odd, None, pw1, k)
    n0 = _lib.launch_count()
    with pytest.raises(RuntimeError, match="does not take"):
        ops.dsconv_bf16(odd, w[:k * C0], b[:k * C0], k, pw1, sc, sh, True)
    assert _lib.launch_count() == n0


# (id, C0, C1, Cout, H, W, k, B): the partial-tile and narrow cases, written through the C ABI into guarded buffers
GUARDED = [("wltpw_24", 256, 0, 256, 24, 24, 2, 2), ("oddh_99x96", 64, 0, 64, 99, 96, 2, 2), ("cout40_70x104_k1", 64, 0, 40, 70, 104, 1, 3),
           ("cout8_37x40", 64, 0, 8, 37, 40, 2, 2), ("cout384_12x64", 64, 0, 384, 12, 64, 2, 2), ("cat_32_3_k1", 32, 3, 64, 40, 56, 1, 2)]


@pytest.mark.parametrize("case", GUARDED, ids=[c[0] for c in GUARDED])
def test_dsconv_bf16_guarded_output(case):
    """y with a batch stride of Cout H W + 64 in a NaN-poisoned buffer with a guard tail: the (Cout, H, W) region of each image
    equals ops.dsconv_bf16's output, and nothing else is written (a store box past W, H or Cout would show here)."""
    name, C0, C1, Cout, H, W, k, B = case
    g, x, w, b, pw, sc, sh, _ = _make(C0, C1, Cout, H, W, k, B, seed=1)
    x0, x1 = x[:, :C0].to(BF), (x[:, C0:].to(BF).contiguous() if C1 else None)
    ref = ops.dsconv_bf16(x0, w, b, k, pw, sc, sh, True, x1=x1)
    chw = Cout * H * W
    ybs = chw + 64
    buf = _poisoned(B * ybs + GUARD, BF)
    pack = ops.pack_bf16(pw)
    torch.cuda.synchronize()
    rc = _lib.load().smaat_dsconv_bf16_fwd(x0.data_ptr(), C0, C0 * H * W, x1.data_ptr() if C1 else None, C1, C1 * H * W,
                                           w.data_ptr(), b.data_ptr(), pack.data_ptr(), sc.data_ptr(), sh.data_ptr(),
                                           buf.data_ptr(), ybs, None, None, B, H, W, k, Cout, 1, ops._stream())
    assert rc == 0, _lib.load().smaat_last_error()
    torch.cuda.synchronize()
    _exact(buf[:B * ybs].view(B, ybs)[:, :chw].reshape(B, Cout, H, W), ref, f"guarded dsconv bf16 {name}")
    keep = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    keep[:B * ybs].view(B, ybs)[:, :chw] = True
    _untouched(buf, keep, f"guarded dsconv bf16 {name}")


# (id, C0, Cout, H, W): the heads at W < PW (C0 = 256 at level 3 of a 96-px image) and at odd H
HEAD_SHAPES = [("wltpw_24", 256, 64, 24, 24), ("oddh_99x96", 64, 64, 99, 96)]


def _head_case(C0, Cout, H, W, K, B=2):
    g, x, w, b, pw, sc, sh, _ = _make(C0, 0, Cout, H, W, 2, B, seed=K)
    ow, ob = _randn((K, Cout), g, Cout ** -0.5), _randn((K,), g, 0.3)
    act = _ds_ref(x, w, b, 2, pw, sc, sh, C0, None, None)
    ref = torch.einsum("kc,bchw->bkhw", ow.double(), act) + ob.double().view(1, -1, 1, 1)
    return x, w, b, pw, sc, sh, ow, ob, ref


def _clear_classes(cls, ref, what):
    """Class map = the float64 argmax where the top two logits are apart by more than the fp32 accumulation can move them."""
    top2 = ref.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-5 * ref.abs().max()
    _exact(cls[clear], ref.argmax(dim=1)[clear], f"{what} (clear pixels)")
    assert float(clear.double().mean()) > 0.99


@pytest.mark.parametrize("shape", HEAD_SHAPES, ids=[s[0] for s in HEAD_SHAPES])
def test_dsconv_head_bf16_edges(shape):
    name, C0, Cout, H, W = shape
    x, w, b, pw, sc, sh, ow, ob, ref = _head_case(C0, Cout, H, W, 1)
    x0 = x.to(BF)
    lg = ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow, ob, "logits")
    assert lg.dtype == BF and lg.shape == (x.shape[0], 1, H, W)
    _one_ulp(lg, ref, f"outconv head bf16 {name}", HEAD_ATOL)
    _exact(lg, ops.dsconv(x, w, b, 2, pw, sc, sh, True, mode="bf16", outconv=(ow, ob)).to(BF),
           f"outconv head bf16 {name} vs the fp32-storage head rounded once")
    for K in (2, 21, 32):
        x, w, b, pw, sc, sh, ow, ob, ref = _head_case(C0, Cout, H, W, K)
        cls = ops.dsconv_head_bf16(x.to(BF), w, b, 2, pw, sc, sh, True, ow, ob, "classes")
        assert cls.dtype == torch.int64 and cls.shape == (x.shape[0], H, W)
        _clear_classes(cls, ref, f"classify head bf16 {name} K={K}")
        _exact(cls, ops.dsconv_classify(x, w, b, 2, pw, sc, sh, True, ow, ob, mode="bf16"),
               f"classify head bf16 {name} K={K} vs the fp32-storage head")
    x, w, b, pw, sc, sh, ow, ob, _ = _head_case(C0, Cout, H, W, 33, B=1)
    assert not ops.dsconv_bf16_takes(x.to(BF), None, pw, 2, ncls=33)
    n0 = _lib.launch_count()
    assert ops.dsconv_head_bf16(x.to(BF), w, b, 2, pw, sc, sh, True, ow, ob, "classes") is None
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("shape", HEAD_SHAPES, ids=[s[0] for s in HEAD_SHAPES])
def test_dsconv_head_bf16_guarded(shape):
    """The heads through the C ABI into over-allocated, poisoned logits and class maps: the image's pixels equal the ops' output
    (and the class map's logits, class by class, the one-class head's), nothing past them is written."""
    name, C0, Cout, H, W = shape
    B, P = 2, H * W
    lib = _lib.load()
    for K in (1, 2, 21, 32):
        x, w, b, pw, sc, sh, ow, ob, ref = _head_case(C0, Cout, H, W, K, B)
        x0 = x.to(BF)
        pack = ops.pack_bf16(pw)
        args = (x0.data_ptr(), C0, C0 * P, None, 0, 0, w.data_ptr(), b.data_ptr(), pack.data_ptr(), sc.data_ptr(), sh.data_ptr(),
                ow.data_ptr(), ob.data_ptr())
        if K == 1:
            lbuf = _poisoned(B * P + GUARD, BF)
            rc = lib.smaat_dsconv_outconv_bf16_fwd(*args, lbuf.data_ptr(), B, H, W, 2, Cout, 1, ops._stream())
            assert rc == 0, lib.smaat_last_error()
            _exact(lbuf[:B * P].view(B, 1, H, W), ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow, ob, "logits"),
                   f"guarded outconv head {name}")
            keep = torch.zeros(lbuf.shape, dtype=torch.bool, device="cuda")
            keep[:B * P] = True
            _untouched(lbuf, keep, f"guarded outconv head {name}")
            continue
        lbuf, cbuf = _poisoned(B * K * P + GUARD, BF), _poisoned(B * P + GUARD, torch.int64)
        rc = lib.smaat_dsconv_classify_bf16_fwd(*args, K, lbuf.data_ptr(), cbuf.data_ptr(), B, H, W, 2, Cout, 1, ops._stream())
        assert rc == 0, lib.smaat_last_error()
        _exact(cbuf[:B * P].view(B, H, W), ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow, ob, "classes"),
               f"guarded classify head {name} K={K}")
        lg = lbuf[:B * K * P].view(B, K, H, W)
        _one_ulp(lg, ref, f"guarded classify head {name} K={K} logits", HEAD_ATOL)
        for j in (0, K - 1):      # class j's logits are the one-class head's with OutConv row j
            _exact(lg[:, j:j + 1], ops.dsconv_head_bf16(x0, w, b, 2, pw, sc, sh, True, ow[j:j + 1], ob[j:j + 1], "logits"),
                   f"guarded classify head {name} K={K} class {j} logits vs the one-class head")
        for buf, n in ((lbuf, B * K * P), (cbuf, B * P)):
            keep = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
            keep[:n] = True
            _untouched(buf, keep, f"guarded classify head {name} K={K} {buf.dtype}")


# ========================================================================================================== B: CBAM from bf16
# max |err| / max |ref| against float64 (tighter than tests/test_gpu_bf16_activations.py's 1e-5: see the table above)
POOL_AVG, POOL_GATE, REDUCE_MEAN, REDUCE_MAX = 1e-6, 2e-6, 2e-6, 2e-7
POOL_MLP_CASES = [(64, 32, 32), (128, 16, 40), (256, 8, 24), (256, 8, 8)]


@pytest.mark.parametrize("C,H,W", POOL_MLP_CASES, ids=[f"C{c}_{h}x{w}" for c, h, w in POOL_MLP_CASES])
@pytest.mark.parametrize("pdt", [BF, torch.float32], ids=["bf16_pool", "fp32_pool"])
def test_cbam_pool_mlp_small_planes(C, H, W, pdt):
    """Planes under 2 048 pixels: the 8-planes-per-CTA kernel and the MLP tail that the last CTA of each image runs."""
    B = 3
    g = _gen(C + H * 7 + W)
    xf = r16(_randn((B, C, H, W), g, 1.0, 1.0)).float()
    x = xf.to(BF)
    hid = C // 16
    w1, b1 = _randn((hid, C), g, C ** -0.5), _randn((hid,), g, 0.1)
    w2, b2 = _randn((C, hid), g, hid ** -0.5), _randn((C,), g, 0.1)
    sc, avg, mx, pooled = ops.cbam_pool_mlp(x, w1, b1, w2, b2, with_maxpool=True, pooled_dtype=pdt)
    xd = xf.double()
    _check(avg, xd.mean(dim=(2, 3)), POOL_AVG, f"pool_mlp bf16 avg C{C} {H}x{W}")
    _exact(mx, xf.amax(dim=(2, 3)), f"pool_mlp bf16 max C{C} {H}x{W}")
    assert pooled.dtype == pdt
    _exact(pooled.float(), F.max_pool2d(xf, 2), f"pool_mlp bf16 max-pool C{C} {H}x{W}")
    mlp = lambda v: F.linear(F.relu(F.linear(v, w1.double(), b1.double())), w2.double(), b2.double())  # noqa: E731
    _check(sc, torch.sigmoid(mlp(avg.double()) + mlp(mx.double())), POOL_GATE, f"pool_mlp bf16 gate C{C} {H}x{W}")


@pytest.mark.parametrize("pdt", [BF, torch.float32], ids=["bf16_pool", "fp32_pool"])
def test_cbam_pool_maxpool_planes_not_a_multiple_of_8(pdt):
    B, C, H, W = 3, 13, 10, 12           # 39 planes: the last CTA holds 7
    g = _gen(39)
    xf = r16(_randn((B, C, H, W), g, 1.0, 1.0)).float()
    avg, mx, pooled = ops.cbam_pool_maxpool(xf.to(BF), pooled_dtype=pdt)
    _check(avg, xf.double().mean(dim=(2, 3)), POOL_AVG, "pool_maxpool bf16 avg 39 planes")
    _exact(mx, xf.amax(dim=(2, 3)), "pool_maxpool bf16 max 39 planes")
    _exact(pooled.float(), F.max_pool2d(xf, 2), "pool_maxpool bf16 max-pool 39 planes")


REDUCE_CASES = [(3, 64, 9, 13), (3, 13, 16, 16), (2, 13, 9, 13), (7, 64, 46, 178), (7, 64, 64, 128), (2, 13, 64, 128)]


@pytest.mark.parametrize("B,C,H,W", REDUCE_CASES, ids=[f"B{b}_C{c}_{h}x{w}" for b, c, h, w in REDUCE_CASES])
def test_cbam_reduce_from_bf16_edges(B, C, H, W):
    """P % 4 != 0 (the scalar kernel), C = 13 (the C % 8 tail), P = 8 188 / 8 192 (each side of the float4 kernel's switch)."""
    g = _gen(B * 1000 + C * 10 + H + W)
    xf = r16(_randn((B, C, H, W), g, 1.0, 1.0)).float()
    sc = torch.rand((B, C), generator=g, device="cuda") + 0.5
    red = ops.cbam_reduce(xf.to(BF), sc)
    xs = xf.double() * sc.double().view(B, C, 1, 1)
    _check(red[:, 0], xs.mean(dim=1), REDUCE_MEAN, f"reduce bf16 mean B{B} C{C} {H}x{W}")
    _check(red[:, 1], xs.amax(dim=1), REDUCE_MAX, f"reduce bf16 max B{B} C{C} {H}x{W}")


# ============================================================================================================ C: upsample
# (B, C, H, W, Ho, Wo)
UP_CASES = [(2, 16, 12, 16, 25, 32), (2, 16, 12, 16, 27, 36), (2, 8, 6, 7, 12, 16), (2, 8, 9, 7, 21, 16), (2, 8, 1, 16, 2, 32),
            (2, 8, 1, 16, 3, 36), (2, 8, 16, 1, 32, 4), (2, 8, 16, 1, 35, 4)]


def _up_ref(xd, Ho, Wo):
    up = F.interpolate(xd, scale_factor=2, mode="bilinear", align_corners=True)
    dY, dX = Ho - up.shape[2], Wo - up.shape[3]
    return F.pad(up, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2])


@pytest.mark.parametrize("case", UP_CASES, ids=[f"{c[2]}x{c[3]}_to_{c[4]}x{c[5]}" for c in UP_CASES])
@pytest.mark.parametrize("src", [torch.float32, BF], ids=["from_fp32", "from_bf16"])
def test_upsample_to_bf16_with_pads(case, src):
    B, C, H, W, Ho, Wo = case
    g = _gen(H * 100 + W * 10 + Ho + Wo)
    xf = _randn((B, C, H, W), g)
    if src == BF:
        xf = r16(xf).float()
    y = ops.upsample2x_pad(xf.to(src), Ho, Wo, out_dtype=BF)
    assert y.dtype == BF and y.shape == (B, C, Ho, Wo)
    what = f"upsample {str(src)[6:]} -> bf16 {H}x{W} -> {Ho}x{Wo}"
    _exact(y, ops.upsample2x_pad(xf, Ho, Wo).to(BF), what + " vs fp32 kernel rounded")
    # the source coordinate is taken in fp32 (as torch's fp32 kernel does): off by ~2 max(H, W) 6e-8 pixels
    _one_ulp(y, _up_ref(xf.double(), Ho, Wo), what, atol_rel=4 * max(H, W) * 6e-8)


def test_upsample_to_bf16_refuses_wo_not_a_multiple_of_4_without_writing():
    B, C, H, W, Ho, Wo = 2, 8, 6, 7, 12, 14
    x = torch.randn((B, C, H, W), device="cuda").to(BF)
    with pytest.raises(RuntimeError):
        ops.upsample2x_pad(x, Ho, Wo, out_dtype=BF)
    buf = _poisoned(B * C * Ho * Wo + GUARD, BF)
    n0 = _lib.launch_count()
    rc = _lib.load().smaat_upsample2x_pad_bf16_fwd(x.data_ptr(), 1, buf.data_ptr(), C * Ho * Wo, B, C, H, W, Ho, Wo, ops._stream())
    assert rc == UNSUPPORTED and _lib.launch_count() == n0
    torch.cuda.synchronize()
    _untouched(buf, torch.zeros(buf.shape, dtype=torch.bool, device="cuda"), "refused upsample")


# ======================================================================================================= D: unfused heads
@pytest.mark.parametrize("K", [1, 2, 9])
@pytest.mark.parametrize("H,W", [(16, 20), (7, 9)], ids=["P320", "P63"])
def test_outconv_bf16_edges(K, H, W):
    B, Cin, P = 2, 24, H * W
    g = _gen(K * 100 + P)
    xf = r16(torch.relu(_randn((B, Cin, H, W), g))).float()
    w, b = _randn((K, Cin), g, Cin ** -0.5), _randn((K,), g, 0.3)
    xb = xf.to(BF)
    lg = ops.outconv(xb, w, b)
    assert lg.dtype == BF
    ref = torch.einsum("kc,bchw->bkhw", w.double(), xf.double()) + b.double().view(1, -1, 1, 1)
    _one_ulp(lg, ref, f"outconv bf16 K={K} {H}x{W}", HEAD_ATOL)
    # into a poisoned, over-allocated buffer: the scalar path's stores stop at P
    buf = _poisoned(B * K * P + GUARD, BF)
    rc = _lib.load().smaat_outconv_bf16_fwd(xb.data_ptr(), w.data_ptr(), b.data_ptr(), buf.data_ptr(), B, Cin, K, P,
                                            ops._stream())
    assert rc == 0
    _exact(buf[:B * K * P].view(B, K, H, W), lg, f"guarded outconv bf16 K={K} {H}x{W}")
    keep = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    keep[:B * K * P] = True
    _untouched(buf, keep, f"guarded outconv bf16 K={K} {H}x{W}")


def _argmax_ref(x):
    """torch.argmax's rule, spelled out: the first NaN if the pixel has one, else the first index of the maximum."""
    xd = x.double()
    K = xd.shape[1]
    idx = torch.arange(K, device=x.device).view(1, K, *([1] * (xd.dim() - 2)))
    isn = xd.isnan()
    first_nan = torch.where(isn, idx, K).amin(dim=1)
    m = torch.where(isn, -torch.inf, xd).amax(dim=1, keepdim=True)
    first_max = torch.where(xd == m, idx, K).amin(dim=1)
    return torch.where(isn.any(dim=1), first_nan, first_max)


def test_argmax_bf16_ties_and_non_finite_logits():
    B, K, H, W = 2, 7, 24, 40
    g = _gen(77)
    x = torch.randint(0, 3, (B, K, H, W), generator=g, device="cuda").to(BF)      # three values: ties everywhere
    assert float((x == x.amax(dim=1, keepdim=True)).sum(dim=1).gt(1).double().mean()) > 0.5
    _exact(ops.argmax_channels(x), _argmax_ref(x), "argmax bf16 exact ties")
    _exact(ops.argmax_channels(x), torch.argmax(x, dim=1), "argmax bf16 exact ties vs torch")
    y = _randn((B, K, H, W), g).to(BF)
    y[0, 3, 0, :8] = float("nan")                      # a NaN wins
    y[0, 5, 0, 4:12] = float("nan")                    # the first NaN
    y[0, 2, 1, :8] = float("inf")                      # +inf wins over finite
    y[0, 6, 1, 4:8] = float("inf")                     # a tie of +infs: the first
    y[1, :, 2, :8] = float("-inf")                     # all -inf: index 0
    y[1, :4, 3, :8] = float("-inf")                    # -inf among finite logits
    y[1, 4, 3, 4:8] = float("nan")
    y[1, 1, 4, :] = float("inf")
    y[1, 0, 4, :6] = float("nan")                      # NaN before +inf
    _exact(ops.argmax_channels(y), _argmax_ref(y), "argmax bf16 non-finite logits")
    _exact(ops.argmax_channels(y), torch.argmax(y.float(), dim=1), "argmax bf16 non-finite logits vs torch")


def test_argmax_bf16_k1_k1024_and_several_grid_passes():
    g = _gen(78)
    x1 = _randn((2, 1, 8, 12), g).to(BF)
    _exact(ops.argmax_channels(x1), torch.zeros((2, 8, 12), dtype=torch.int64, device="cuda"), "argmax bf16 K=1")
    xk = torch.randint(-50, 50, (2, 1024, 6, 10), generator=g, device="cuda").to(BF)
    _exact(ops.argmax_channels(xk), _argmax_ref(xk), "argmax bf16 K=1024")
    # more pixels than the capped grid (16 CTAs per SM, 256 threads) covers in one pass
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    B, H = 3, 512
    W = -(-(16 * sms * 256 + 10000) // (B * H))
    xl = torch.randint(-4, 4, (B, 3, H, W), generator=g, device="cuda").to(BF)
    assert B * H * W > 16 * sms * 256
    _exact(ops.argmax_channels(xl), _argmax_ref(xl), f"argmax bf16 {B * H * W} pixels")


@pytest.mark.parametrize("K", [2, 21, 1024])
def test_softmax_bf16_edges(K):
    B, H, W = 2, 8, 12 if K < 1024 else 6
    g = _gen(K + 5)
    lg = (_randn((B, K, H, W), g) * 3).to(BF)
    pr = ops.softmax_channels(lg)
    assert pr.dtype == BF
    _one_ulp(pr, torch.softmax(lg.double(), dim=1), f"softmax bf16 K={K}")
    # non-finite rows: torch's pattern
    nf = lg.clone()
    nf[0, 1, 0, :3] = float("nan")
    nf[0, 0, 1, :3] = float("inf")
    nf[1, :, 2, :3] = float("-inf")
    nf[1, 0, 3, :3] = float("-inf")
    if K > 2:
        nf[1, 1, 3, 3:6] = float("-inf")
    pr = ops.softmax_channels(nf)
    ref = torch.softmax(nf.double(), dim=1)
    _exact(pr.isnan(), ref.isnan(), f"softmax bf16 K={K} NaN pattern")
    fin = ~ref.isnan()
    _exact(pr[fin & (ref == 0)].double(), ref[fin & (ref == 0)], f"softmax bf16 K={K} exact zeros")
    _one_ulp(pr[fin], ref[fin], f"softmax bf16 K={K} with non-finite rows")
    if K == 2:
        one = torch.tensor([[[0.0]], [[float("-inf")]]], device="cuda").to(BF).view(1, 2, 1, 1)
        _exact(ops.softmax_channels(one).float().view(-1), torch.tensor([1.0, 0.0], device="cuda"), "softmax bf16 K=2 [0, -inf]")


# ====================================================================================================== E: whole networks
# max |err| / max |ref| of the whole networks against the emulated port / the unrounded port (see the table above)
NET_BOUND = {
    "smaat_3_21_k2_96x160": (1.5e-2, 1.5e-2), "smaat_3_21_k2_96x160_probs": 1e-2,
    "smaat_12_1_k1_128x64": (1.8e-2, 1.5e-2),
    "smaat_1_2_k2_64x96": (2e-2, 2e-2), "smaat_1_2_k2_64x96_probs": 1e-2,
    "smaat_3_40_k2_96x96": (1.5e-2, 1.6e-2), "smaat_3_40_k2_96x96_probs": 1e-2,
}
MIN_CLASS_AGREEMENT = 0.99


def _model(n_ch, n_cls, k):
    torch.manual_seed(3 + n_cls)
    return _bn_randomise(S.SmaAt_UNet(n_ch, n_cls, kernels_per_layer=k), 4 + k).cuda().eval()


# (name, n_ch, n_cls, k, H, W, B, outputs)
NETS = [
    ("smaat_3_21_k2_96x160", 3, 21, 2, 96, 160, 3, ("logits", "probs", "classes")),
    ("smaat_12_1_k1_128x64", 12, 1, 1, 128, 64, 2, ("logits",)),
    ("smaat_1_2_k2_64x96", 1, 2, 2, 64, 96, 3, ("logits", "probs", "classes")),
    ("smaat_3_40_k2_96x96", 3, 40, 2, 96, 96, 2, ("logits", "probs", "classes")),
]


@pytest.mark.parametrize("net", NETS, ids=[n[0] for n in NETS])
def test_whole_network_sessions(net):
    name, n_ch, n_cls, k, H, W, B, outputs = net
    model = _model(n_ch, n_cls, k)
    shape = (n_ch, H, W)
    x = torch.rand((B,) + shape, generator=_gen(H + W + n_cls), device="cuda").to(BF)
    sd = _sd64(model)
    emul = _port_bf16(x.double(), sd, fused_head=n_cls == 1)
    eager = {"logits": model.forward_serving, "classes": model.forward_classes, "probs": model.forward_probs}
    for out in outputs:
        sess = InferenceSession(model, B, shape, output=out, dtype=BF, batch_sizes=(1,))
        got = sess.forward(x).clone()
        part = sess.forward(x[1:2]).clone()
        with torch.no_grad():
            _exact(got, eager[out](x), f"{name} {out} session vs eager")
            _exact(part, eager[out](x[1:2]), f"{name} {out} 1-row session vs eager")
        if out == "logits":
            assert got.dtype == BF
            bound_emul, bound_port = NET_BOUND[name]
            _check(got, emul, bound_emul, f"{name} logits vs float64 port with the bf16 roundings")
            _check(got, _port(model, x.float()), bound_port, f"{name} logits vs the unrounded float64 port")
        elif out == "probs":
            assert got.dtype == BF
            _check(got, torch.softmax(emul, dim=1), NET_BOUND[name + "_probs"], f"{name} probabilities vs emulated port")
        else:
            # up4's last conv feeds the fused class head unrounded (n_classes <= 32); the unfused head reads bf16 maps
            ref = _port_bf16(x.double(), sd, fused_head=True) if n_cls <= 32 else emul
            agree = float((got == ref.argmax(dim=1)).double().mean())
            print(f"ERR {name} class map agreement with the emulated port: {agree:.5f}")
            assert agree >= MIN_CLASS_AGREEMENT


# ============================================================================================================= F: W = 32
def test_w32_raises_before_any_launch():
    model = _model(12, 1, 2)
    x = torch.rand((2, 12, 64, 32), device="cuda").to(BF)
    for fwd in (model.forward_serving, model.forward_classes, model.forward_probs):
        n0 = _lib.launch_count()
        with torch.no_grad(), pytest.raises(ValueError, match="level-3 maps are 8 wide"):
            fwd(x)
        assert _lib.launch_count() == n0, "a refused W = 32 request launched kernels"
    n0 = _lib.launch_count()
    with pytest.raises(ValueError, match="level-3 maps are 8 wide"):
        InferenceSession(model, 2, (12, 64, 32), dtype=BF)
    assert _lib.launch_count() == n0
    sess = InferenceSession(model, 2, (12, 64, 64), dtype=BF)         # the device is still fine
    xs = torch.rand((2, 12, 64, 64), device="cuda").to(BF)
    with torch.no_grad():
        _exact(sess.forward(xs).clone(), model.forward_serving(xs), "session after a refused W = 32 session")
    # the fp32 route still takes W = 32
    with torch.no_grad():
        y = model.forward_serving(x.float())
    assert y.dtype == torch.float32 and bool(torch.isfinite(y).all())
