"""The SmaAt-UNet forward kernels and the depthwise backward against high-precision references, at the layer shapes
SmaAt_UNet(12, 1, kernels_per_layer=2, bilinear=True) runs at 288x288 (the network bench.py measures).

The other forward tests use planes of at most 128x128 (a fused DS-conv CTA then sees ~8 tiles), <= 8 channels for the
depthwise kernels and batches <= 4 for CBAM.  The production launches are much larger: 20 736 fused tiles at B = 32,
1 024-channel concats, 2.65 M-term weight reductions.  Here every entry point is called directly (through ``ops`` /
``functional`` or the C ABI) at those shapes:

  A  the references themselves, on the CPU: fma32 against exact rational arithmetic, the emulated depthwise against
     F.conv2d, the backward references against autograd, tf32 truncation and the hi / lo split on bit patterns
  B  smaat_dw3x3_fwd at all 18 depthwise layers: loader auto (one warp per plane at 18x18), LDG and TMA, the BN+ReLU
     prologue on every conv 1, the concat on every up block's conv 0, batch-strided channel slices, misaligned copies
  C  smaat_dsconv_fwd at the 12 fused layers: eval epilogue (scale, shift, ReLU) and train epilogue (shift, BatchNorm
     statistics), tf32 and tf32x3, A operand from shared memory and from registers; smaat_dsconv_outconv_fwd at up4.1
  D  exact-integer production launches at B = 32, 288x288: inc.0, up4.0 (concat), up4.1 + OutConv
  E  smaat_pw1x1_fwd at the 18 pointwise shapes, fp32 / tf32 / tf32x3, train epilogue everywhere and the eval epilogue at
     the six layers the fused kernel declines (36x36, 18x18)
  F  the CBAM forward at the five CBAMs, serving chain and train chain; maxpool2 and upsample2x_pad into the concat slice
  G  smaat_dw3x3_bwd_input (TMA and tiled) and smaat_dw3x3_bwd_weight (TMA and tiled, with and without the prologue)

Conventions:
  * the depthwise kernels all compute a = bias; a = fmaf(w[t], x[t], a) for the 9 taps in row-major order, the prologue
    as fmaxf(fmaf(v, scale, shift), 0) and zero outside the image.  ``fma32`` reproduces fp32 fmaf exactly (a float64
    product is exact, a two-sum recovers the error of the float64 add, and ties of the final fp32 rounding are broken by
    the sign of that error), so ``dw_emul`` is bit-equal to the kernels and is compared with torch.equal;
  * tf32 mode hands raw fp32 bits to the tensor core, which ignores the low 13 mantissa bits: the reference multiplies
    truncated operands exactly in float64, so only the tensor core's fp32 accumulation is measured.  tf32x3 splits
    a = hi + lo (lo = a - hi is exact; the tensor core truncates it again) and w the same way (smaat_split_tf32): the
    reference is hi.Whi + trunc(lo).Whi + hi.trunc(Wlo) in float64, without the dropped lo.lo term;
  * part D uses integer data (inputs and weights in {-1, 0, 1}, integer biases, power-of-two scales, shifts on a 1/8 grid):
    every product and partial sum is exact in fp32, so y, the logits and the BatchNorm sums must be bit-equal to float64
    whatever the summation order.  The stats epilogue's fp32 16-value sums of squares stay exact while |pre-activation|
    < 2^10, which the test asserts on its reference first;
  * accumulating outputs (the depthwise dW and db) start from a non-zero buffer and are checked as init + gradient;
  * errors are max |got - ref| / max |ref|, as tests/_util.assert_close measures them.

The shared-memory and register forms of the fused kernel feed the tensor core the same operand bits in the same MMA order,
and are bit-equal (asserted); so are repeated calls.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x
above it (everything else is bit-exact and was):

  quantity                                                   worst observed                 bound
  C  fused DS conv y and logits, tf32 / tf32x3               3.3e-6 / 9.7e-6                3e-5 / 9e-5
     its BatchNorm sums, tf32 / tf32x3                       1.7e-6 / 5.4e-6                1.5e-5 / 5e-5
  E  pointwise y, fp32 / tf32 / tf32x3                       2.2e-6 / 5.8e-6 / 1.8e-5       2e-5 / 5e-5 / 1.5e-4
     its BatchNorm sums, fp32 / tf32 / tf32x3                2.7e-8 / 4.5e-6 / 1.4e-5       2.5e-7 / 4e-5 / 1.4e-4
  F  channel mean, MLP gate sc, pixel channel mean           4.3e-7                         4e-6
     spatial gate and scaled output (serving and train)      4.6e-7                         4e-6
     upsample, kernel / torch fp32 error                     1.0x                           3x + 1e-6
  G  depthwise dx                                            2.2e-7                         2e-6
     depthwise dW, db                                        1.3e-6                         1e-5

With the truncation-aware reference the fused kernel's tf32 error is that of an fp32 accumulation (3.3e-6).  Producers
that rounded the A operand to tf32 nearest instead of passing it raw measured 5.7e-4 here: inside the PW_TOL["tf32"] =
4e-3 the other tests hold this kernel to, 19x over this file's bound.  tf32x3 sits ~3x above tf32: three MMAs per k-step
accumulate into the same fp32 registers.  The whole file runs in ~9 s on one H100 at a peak of 4.6 GiB allocated.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200 import functional as Fn

gpu = pytest.mark.gpu
KPL = 2                      # kernels_per_layer of the network under test
MODES = ("fp32", "tf32", "tf32x3")

# max |got - ref| / max |ref| bounds per quantity (see the module docstring for the observed figures)
ERR_BOUND = {
    "fused": {"tf32": 3e-5, "tf32x3": 9e-5},            # fused DS conv y / logits against the truncation / split-aware reference
    "fused_stats": {"tf32": 1.5e-5, "tf32x3": 5e-5},    # its BatchNorm sums
    "pw": {"fp32": 2e-5, "tf32": 5e-5, "tf32x3": 1.5e-4},
    "pw_stats": {"fp32": 2.5e-7, "tf32": 4e-5, "tf32x3": 1.4e-4},
    "cbam_pool": 4e-6,        # channel mean (fp32 plane sums), MLP gate sc, per-pixel channel mean
    "cbam_out": 4e-6,         # spatial gate (raw conv, sigmoid) and the scaled output
    "dw_dx": 2e-6,
    "dw_dw": 1e-5,            # dW and db (fp32 partial sums merged by atomics)
}
UPSAMPLE_FACTOR = 3.0        # upsample: error <= this x torch fp32's own error + 1e-6 (both use fp32 source coordinates)
CHUNK = 1 << 23              # elements per chunk of the float64 references (bounds their temporaries to a few 100 MB)


# ------------------------------------------------------------------------------------------------------------------ helpers
def _p(t):
    return None if t is None else t.data_ptr()


def _abi(name, *args):
    _lib.check(getattr(_lib.load(), name)(*args), name)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=g, device="cuda") * scale + shift


def _rel(got, ref):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _check(got, ref, tol, what):
    e = _rel(got, ref)
    print(f"ERR {what}: {e:.3e} (bound {tol:.1e})")
    assert e == e and e <= tol, f"{what}: max rel err {e:.3e} > {tol:.1e}"
    return e


def _exact(got, ref, what):
    """torch.equal, with the first differing position in the message."""
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = got != ref
    n = int(bad.sum())
    print(f"ERR {what}: {n} of {got.numel()} differ (bit-exact)")
    if n:
        idx = tuple(int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{what}: {n} values differ, first at {idx}: {got[idx].item()!r} vs {ref[idx].item()!r}")


def _offset(t):
    """A copy of ``t`` whose data starts one element past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def _slice_of_wider(t, before=4, after=3):
    """``t`` as a channel slice of a wider tensor (read through its batch stride); 16-byte aligned when H W % 4 == 0."""
    B, C, H, W = t.shape
    wide = torch.full((B, before + C + after, H, W), float("nan"), device=t.device)
    wide[:, before:before + C] = t
    return wide[:, before:before + C]


def _chunks(n, per):
    step = max(1, CHUNK // max(per, 1))
    return [(i, min(n, i + step)) for i in range(0, n, step)]


# ------------------------------------------------------------------------------------------------- exact fp32 arithmetic
def fma32(a, b, c):
    """fp32 tensors -> fmaf(a, b, c) in fp32, exactly (one rounding of the exact a * b + c)."""
    p = a.double() * b.double()                 # exact: 24 + 24 bits
    cd = c.double()
    s = p + cd
    bb = s - p
    err = (p - (s - bb)) + (cd - bb)            # two-sum: s + err == p + c exactly
    r = s.float()
    up = torch.nextafter(r, torch.full_like(r, float("inf")))
    dn = torch.nextafter(r, torch.full_like(r, float("-inf")))
    rd = r.double()
    tie_up = s == (rd + up.double()) / 2        # s sits on an fp32 midpoint: the sign of err decides the side
    tie_dn = s == (rd + dn.double()) / 2
    r = torch.where(tie_up & (err > 0), up, r)
    return torch.where(tie_dn & (err < 0), dn, r)


def tf32(t):
    """fp32 -> the tf32 value the tensor core multiplies: the low 13 mantissa bits cleared."""
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32)


def split_hi_lo(t):
    """The tf32x3 split as the kernels make it: hi = tf32(t), lo = t - hi (exact in fp32), lo as the tensor core reads it."""
    hi = tf32(t)
    return hi, tf32(t - hi)


def prologue(x, scale, shift):
    """fmaxf(fmaf(x, scale[c], shift[c]), 0) per channel, in fp32 exactly as the kernels apply it."""
    C = x.shape[1]
    return fma32(x, scale.view(1, C, 1, 1).expand_as(x), shift.view(1, C, 1, 1).expand_as(x)).clamp_min(0.0)


def dw_emul(x, w, bias, k, scale=None, shift=None):
    """The depthwise forward bit for bit: x (B, Cin, H, W) fp32 (the concat), w (k Cin, 1, 3, 3), bias (k Cin) or None,
    optional prologue -> fp32 (B, k Cin, H, W)."""
    B, Cin, H, W = x.shape
    out = torch.empty((B, k * Cin, H, W), device=x.device, dtype=torch.float32)
    w9 = w.reshape(k * Cin, 9)
    for b in range(B):
        for c0, c1 in _chunks(Cin, k * H * W):
            xa = x[b:b + 1, c0:c1]
            if scale is not None:
                xa = prologue(xa, scale[c0:c1], shift[c0:c1])
            xe = F.pad(xa[0], (1, 1, 1, 1)).repeat_interleave(k, dim=0)          # zero outside the image
            o0, o1 = k * c0, k * c1
            if bias is None:
                a = torch.zeros((o1 - o0, H, W), device=x.device)
            else:
                a = bias[o0:o1].view(-1, 1, 1).expand(o1 - o0, H, W).contiguous()
            for t in range(9):
                dy, dx = divmod(t, 3)
                a = fma32(w9[o0:o1, t].view(-1, 1, 1).expand(o1 - o0, H, W), xe[:, dy:dy + H, dx:dx + W], a)
            out[b, o0:o1] = a
    return out


# ------------------------------------------------------------------------------------------------ float64 references
def pw_ref(d, w, mode):
    """float64 Z[b] = W . D[b] as the pointwise GEMM computes it in ``mode``: exact operands (fp32), truncated operands (tf32)
    or the three split products (tf32x3)."""
    B, K, H, W_ = d.shape
    w = w.reshape(w.shape[0], K)
    if mode == "fp32":
        wt = [w.double()]
    elif mode == "tf32":
        wt = [tf32(w).double()]
    else:
        wh, wl = split_hi_lo(w)
        wt = [wh.double(), wl.double()]
    out = torch.empty((B, w.shape[0], H, W_), device=d.device, dtype=torch.float64)
    for b in range(B):
        a = d[b].reshape(K, -1)
        if mode == "fp32":
            z = wt[0] @ a.double()
        elif mode == "tf32":
            z = wt[0] @ tf32(a).double()
        else:
            ah, al = split_hi_lo(a)
            ah = ah.double()
            z = wt[0] @ ah + wt[0] @ al.double() + wt[1] @ ah
        out[b] = z.view(-1, H, W_)
    return out


def dw_input_grad_ref(dd, w, k):
    """float64 input gradient of the depthwise conv: dx[b, c] = sum_kk sum_t w[c k + kk, t] dd[b, c k + kk, y + 1 - dy, x + 1 - dx]."""
    B, KC, H, W = dd.shape
    Cin = KC // k
    w9 = w.reshape(KC, 9).double()
    out = torch.empty((B, Cin, H, W), device=dd.device, dtype=torch.float64)
    for b0, b1 in _chunks(B, KC * H * W):
        gp = F.pad(dd[b0:b1].double(), (1, 1, 1, 1))
        acc = torch.zeros((b1 - b0, KC, H, W), device=dd.device, dtype=torch.float64)
        for t in range(9):
            dy, dx = divmod(t, 3)
            acc += w9[:, t].view(1, KC, 1, 1) * gp[:, :, 2 - dy:2 - dy + H, 2 - dx:2 - dx + W]
        out[b0:b1] = acc.view(b1 - b0, Cin, k, H, W).sum(dim=2)
    return out


def dw_weight_grad_ref(dd, xa, k):
    """float64 (dW (k Cin, 9), db (k Cin)) of the depthwise conv on the (already activated) input xa."""
    B, KC, H, W = dd.shape
    dW = torch.zeros((KC, 9), device=dd.device, dtype=torch.float64)
    db = torch.zeros(KC, device=dd.device, dtype=torch.float64)
    for b0, b1 in _chunks(B, KC * H * W):
        g = dd[b0:b1].double()
        xe = F.pad(xa[b0:b1].double(), (1, 1, 1, 1)).repeat_interleave(k, dim=1)
        for t in range(9):
            dy, dx = divmod(t, 3)
            dW[:, t] += (g * xe[:, :, dy:dy + H, dx:dx + W]).sum(dim=(0, 2, 3))
        db += g.sum(dim=(0, 2, 3))
    return dW, db


# ---------------------------------------------------------------------------------------------------------- layer shapes
# (name, C0, C1, Cout, S): the 18 DS convs of SmaAt_UNet(12, 1, kernels_per_layer=2, bilinear=True) at 288x288.  Cin = [C0 | C1]
# is UpDS's concat [skip | upsampled]; K = 2 Cin.  Conv 1 of each block reads relu(BN(conv 0)) through the prologue in training.
LAYERS = [
    ("inc.0", 12, 0, 64, 288), ("inc.1", 64, 0, 64, 288),                # fused, PW 32, N_TILE 64
    ("down1.0", 64, 0, 128, 144), ("down1.1", 128, 0, 128, 144),         # fused, PW 16, N_TILE 128
    ("down2.0", 128, 0, 256, 72), ("down2.1", 256, 0, 256, 72),          # fused, PW 16, two 128-channel passes
    ("down3.0", 256, 0, 512, 36), ("down3.1", 512, 0, 512, 36),          # dw3x3 (TMA) + pw1x1
    ("down4.0", 512, 0, 512, 18), ("down4.1", 512, 0, 512, 18),          # dw3x3_small + pw1x1
    ("up1.0", 512, 512, 512, 36), ("up1.1", 512, 0, 256, 36),            # dw3x3 + pw1x1
    ("up2.0", 256, 256, 256, 72), ("up2.1", 256, 0, 128, 72),            # fused
    ("up3.0", 128, 128, 128, 144), ("up3.1", 128, 0, 64, 144),           # fused
    ("up4.0", 64, 64, 64, 288), ("up4.1", 64, 0, 64, 288),               # fused (+ OutConv 64 -> 1)
]
FUSED = [l for l in LAYERS if l[4] >= 72]
UNFUSED = [l for l in LAYERS if l[4] < 72]


def _lid(layer):
    name, C0, C1, Cout, H = layer
    return f"{name}_{C0}{'+' + str(C1) if C1 else ''}to{Cout}_S{H}"


def _batch(H):
    return {288: 8, 144: 16}.get(H, 32)


def _seed(layer):
    name, C0, C1, Cout, H = layer
    return C0 * 131 + C1 * 17 + Cout * 7 + H + len(name)


def _split(x, C0, C1):
    return x[:, :C0].contiguous(), (x[:, C0:].contiguous() if C1 else None)


def _dw_params(Cin, g):
    return _randn((KPL * Cin, 1, 3, 3), g, 1.0 / 3.0), _randn((KPL * Cin,), g, 0.1)


def _bn_affine(C, g):
    return torch.rand(C, generator=g, device="cuda") + 0.5, _randn((C,), g, 0.5, 0.2)


# ====================================================================================================== A: the references
def _fma_exact(a, b, c):
    """fp32 fmaf by exact rational arithmetic, rounded to nearest-even at 24 bits."""
    v = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    r = np.float32(float(v))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    return min(cands, key=lambda q: (abs(Fraction(float(q)) - v), int(np.array(q, dtype=np.float32).view(np.int32)) & 1))


def test_fma32_matches_exact_rounding():
    """fma32 against Fraction on random triples and on triples aimed at fp32 ties (a b within 2^-46 of half an ulp of c),
    where rounding a float64 a b + c to fp32 (two roundings) is wrong about half the time."""
    rng = np.random.default_rng(5)
    n = 3000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-30, 30, n)).astype(np.float32)
    m = 2000
    ct = (rng.uniform(1, 2, m) * 2.0 ** rng.integers(-10, 10, m) * rng.choice([-1, 1], m)).astype(np.float32)
    h = np.spacing(np.abs(ct)).astype(np.float64) / 2                   # half an ulp of c: a power of two
    kk = rng.integers(1, 64, m).astype(np.float64)
    ea = rng.integers(-8, 8, m).astype(np.float64)
    at = ((1 + kk * 2.0 ** -23) * 2.0 ** ea).astype(np.float32)
    bt = ((1 - kk * 2.0 ** -23) * h / 2.0 ** ea * rng.choice([-1, 1], m)).astype(np.float32)   # a b = +-h (1 - k^2 2^-46)
    A, Bv, Cv = (np.concatenate(v) for v in ((a, at), (b, bt), (c, ct)))
    ta, tb, tc = (torch.from_numpy(v) for v in (A, Bv, Cv))
    got = fma32(ta, tb, tc).numpy()
    ref = np.array([_fma_exact(x, y, z) for x, y, z in zip(A, Bv, Cv)], dtype=np.float32)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32)), int((got != ref).sum())
    naive = (ta.double() * tb.double() + tc.double()).float().numpy()
    assert (naive != ref).sum() > 100, "the tie-aimed triples no longer reach the double-rounding cases"


def test_depthwise_emulation_matches_float64_conv():
    """dw_emul (bias, concat, prologue, zero padding) against float64 F.conv2d(groups=Cin) within fp32 rounding: a shift > 0
    makes relu(shift) != 0, so padding with the activated value instead of 0 would show at every border."""
    gen = torch.Generator().manual_seed(11)
    for B, C0, C1, H, W, pro in ((2, 5, 3, 7, 10, True), (1, 4, 0, 6, 5, False), (3, 2, 2, 4, 4, True)):
        Cin = C0 + C1
        x = torch.randn(B, Cin, H, W, generator=gen)
        w = torch.randn(KPL * Cin, 1, 3, 3, generator=gen) / 3
        b = torch.randn(KPL * Cin, generator=gen) * 0.1
        sc = torch.rand(Cin, generator=gen) + 0.5 if pro else None
        sh = torch.rand(Cin, generator=gen) * 0.5 + 0.25 if pro else None
        got = dw_emul(x, w, b, KPL, sc, sh)
        xa = x.double()
        if pro:
            xa = torch.relu(xa * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
        ref = F.conv2d(xa, w.double(), b.double(), padding=1, groups=Cin)
        assert _rel(got, ref) < 1e-6
        assert torch.equal(dw_emul(x, w, None, KPL, sc, sh), dw_emul(x, w, torch.zeros_like(b), KPL, sc, sh))


def test_backward_references_match_autograd():
    gen = torch.Generator().manual_seed(12)
    for B, Cin, H, W in ((2, 3, 7, 9), (1, 4, 5, 4)):
        x = torch.randn(B, Cin, H, W, generator=gen, dtype=torch.float64, requires_grad=True)
        w = torch.randn(KPL * Cin, 1, 3, 3, generator=gen, dtype=torch.float64, requires_grad=True)
        b = torch.randn(KPL * Cin, generator=gen, dtype=torch.float64, requires_grad=True)
        dd = torch.randn(B, KPL * Cin, H, W, generator=gen, dtype=torch.float64)
        F.conv2d(x, w, b, padding=1, groups=Cin).backward(dd)
        assert torch.allclose(dw_input_grad_ref(dd, w.detach(), KPL), x.grad, rtol=1e-12, atol=1e-12)
        dW, db = dw_weight_grad_ref(dd, x.detach(), KPL)
        assert torch.allclose(dW.view_as(w), w.grad, rtol=1e-12, atol=1e-12)
        assert torch.allclose(db, b.grad, rtol=1e-12, atol=1e-12)


def test_tf32_truncation_and_split():
    v = torch.tensor([1 + 2 ** -10, 1 + 2 ** -11, -(1 + 2 ** -11), 1 + 2 ** -11 + 2 ** -20 + 2 ** -23, 3.0, -0.0], dtype=torch.float32)
    assert tf32(v).tolist() == [1 + 2 ** -10, 1.0, -1.0, 1.0, 3.0, -0.0]
    hi, lo = split_hi_lo(v)
    assert hi.tolist() == tf32(v).tolist()
    assert lo.tolist() == [0.0, 2 ** -11, -2 ** -11, 2 ** -11 + 2 ** -20, 0.0, 0.0]       # 2^-23 is past lo's 11 bits
    assert torch.equal(hi + (v - hi), v)
    d = torch.randn(4096, generator=torch.Generator().manual_seed(1))
    h, _ = split_hi_lo(d)
    assert bool(((d - h).abs() < d.abs() * 2.0 ** -10).all()) and bool(((h.view(torch.int32) & 8191) == 0).all())


def test_pw_reference_modes():
    """pw_ref in tf32 / tf32x3 against exact products of hand-truncated operands; fp32 against a plain float64 GEMM."""
    gen = torch.Generator().manual_seed(13)
    d = torch.randn(2, 40, 3, 5, generator=gen)
    w = torch.randn(24, 40, generator=gen)
    exact = torch.einsum("ok,bkp->bop", w.double(), d.double().flatten(2)).view(2, 24, 3, 5)
    assert torch.allclose(pw_ref(d, w, "fp32"), exact, rtol=1e-13, atol=1e-13)
    t = torch.einsum("ok,bkp->bop", tf32(w).double(), tf32(d).double().flatten(2)).view(2, 24, 3, 5)
    assert torch.allclose(pw_ref(d, w, "tf32"), t, rtol=1e-13, atol=1e-13)
    assert _rel(pw_ref(d, w, "tf32"), exact) > 1e-5                          # truncation is visible
    assert _rel(pw_ref(d, w, "tf32x3"), exact) < 1e-5                        # the split recovers fp32-grade products


# ============================================================================================ B: depthwise forward, bit-exact
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
def test_depthwise_forward_is_bit_exact(layer):
    """smaat_dw3x3_fwd against dw_emul with torch.equal: loader auto (TMA where W % 4 == 0, else the one-warp-per-plane
    kernel at 18x18), LDG, TMA; batch-strided channel slices; a copy one float off alignment (LDG, or the small kernel)."""
    name, C0, C1, Cout, H = layer
    B, Cin = _batch(H), C0 + C1
    g = _gen(_seed(layer))
    x = _randn((B, Cin, H, H), g)
    w, b = _dw_params(Cin, g)
    sc, sh = _bn_affine(Cin, g) if name.endswith(".1") else (None, None)
    x0, x1 = _split(x, C0, C1)
    ref = dw_emul(x, w, b, KPL, sc, sh)
    for loader in (0, 1, 2) if H % 4 == 0 else (0, 1):
        y = ops.dw3x3(x0, w, b, KPL, x1=x1, in_scale=sc, in_shift=sh, loader=loader)
        _exact(y, ref, f"dw fwd {_lid(layer)} loader {loader}")
        del y
    s0, s1 = _slice_of_wider(x0), (_slice_of_wider(x1, 1, 5) if C1 else None)
    assert s0.data_ptr() % 16 == 0 and not s0.is_contiguous()
    _exact(ops.dw3x3(s0, w, b, KPL, x1=s1, in_scale=sc, in_shift=sh), ref, f"dw fwd {_lid(layer)} channel slices")
    del s0, s1
    o0, o1 = _offset(x0), (_offset(x1) if C1 else None)
    _exact(ops.dw3x3(o0, w, b, KPL, x1=o1, in_scale=sc, in_shift=sh), ref, f"dw fwd {_lid(layer)} misaligned")


# ============================================================================================== C: fused DS conv forward
@gpu
@pytest.mark.parametrize("layer", FUSED, ids=_lid)
def test_fused_dsconv_at_network_shapes(layer):
    """smaat_dsconv_fwd at the 12 layers it runs: eval epilogue relu(scale z + shift), and for Cout <= 128 the train
    epilogue z + bias with the BatchNorm sums; tf32 and tf32x3, A operand from shared memory and from registers (bit-equal
    to each other), each call repeated (bit-equal); at up4.1 also the fused OutConv with and without its bias."""
    name, C0, C1, Cout, H = layer
    B, Cin = _batch(H), C0 + C1
    K = KPL * Cin
    g = _gen(_seed(layer) + 1)
    x = _randn((B, Cin, H, H), g)
    w, b = _dw_params(Cin, g)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    pb = _randn((Cout,), g, 0.3)
    ow, ob = _randn((1, Cout), g, Cout ** -0.5), _randn((1,), g, 0.3)
    x0, x1 = _split(x, C0, C1)
    d = dw_emul(x, w, b, KPL)
    split = ops.split_tf32(pw)
    train = Cout <= 128
    what = f"fused {_lid(layer)}"
    try:
        for mode in ("tf32", "tf32x3"):
            ws = split if mode == "tf32x3" else None
            z = pw_ref(d, pw, mode)
            ref_eval = torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
            got = {}
            for impl in ("smem", "regs"):
                ops.set_dsconv_impl(impl)
                y = ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws)
                assert y is not None, "the fused kernel declined a layer it runs in the network"
                _check(y, ref_eval, ERR_BOUND["fused"][mode], f"{what} {mode} {impl} eval")
                _exact(ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws), y, f"{what} {mode} {impl} repeat")
                got[impl, "eval"] = y
                if train:
                    zb = z + pb.double().view(1, -1, 1, 1)
                    stats = ops.new_stats(Cout, x.device)
                    y = ops.dsconv(x0, w, b, KPL, pw, None, pb, False, x1=x1, mode=mode, w_split=ws, stats=stats)
                    _check(y, zb, ERR_BOUND["fused"][mode], f"{what} {mode} {impl} train")
                    _check(stats[:Cout], zb.sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"][mode], f"{what} {mode} {impl} stats sum")
                    _check(stats[Cout:], (zb * zb).sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"][mode],
                           f"{what} {mode} {impl} stats sum of squares")
                    got[impl, "train"] = y
                    del zb
                if name == "up4.1":
                    for bias in (ob, None):
                        lg = ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws, outconv=(ow, bias))
                        ref = torch.einsum("c,bchw->bhw", ow.double().view(-1), ref_eval).unsqueeze(1)
                        if bias is not None:
                            ref = ref + bias.double()
                        _check(lg, ref, ERR_BOUND["fused"][mode], f"{what} {mode} {impl} outconv bias={bias is not None}")
                        got[impl, f"oc{bias is not None}"] = lg
            for key in {k for _, k in got}:
                _exact(got["regs", key], got["smem", key], f"{what} {mode} {key} regs vs smem")
            del got, z, ref_eval
    finally:
        ops.set_dsconv_impl("auto")


# ======================================================================================== D: exact-integer production launches
def _int_data(shape, g, lo=-1, hi=1):
    return torch.randint(lo, hi + 1, shape, generator=g, device="cuda").float()


@gpu
@pytest.mark.parametrize("name", ["inc.0", "up4.0", "up4.1"])
def test_fused_dsconv_exact_integers_at_production_size(name):
    """B = 32 at 288x288 (20 736 tiles, ~157 per CTA): with integer data every partial sum is exact, so y, the logits and
    the BatchNorm sums must equal the float64 reference bit for bit in tf32 and tf32x3 (lo parts zero), both A forms."""
    layer = next(l for l in LAYERS if l[0] == name)
    _, C0, C1, Cout, H = layer
    B, Cin = 32, C0 + C1
    K = KPL * Cin
    g = _gen(_seed(layer) + 2)
    x = _int_data((B, Cin, H, H), g)
    w = _int_data((K, 1, 3, 3), g)
    b = _int_data((K,), g, -2, 2)
    pw = _int_data((Cout, K), g)
    sc = 2.0 ** _int_data((Cout,), g)                       # 1/2, 1, 2
    sh = _int_data((Cout,), g, -32, 32) / 8
    pb = _int_data((Cout,), g, -32, 32) / 8
    ow, ob = _int_data((1, Cout), g), _int_data((1,), g, -16, 16) / 8
    x0, x1 = _split(x, C0, C1)
    # float64 reference, one image at a time; every value below is exact, so the fp32 copies are too
    y_eval = torch.empty((B, Cout, H, H), device="cuda")
    zb = torch.empty_like(y_eval)
    logits = torch.empty((B, 1, H, H), device="cuda") if name == "up4.1" else None
    stats_ref = torch.zeros(2 * Cout, device="cuda", dtype=torch.float64)
    zmax = 0.0
    for i in range(B):
        d = F.conv2d(x[i:i + 1].double(), w.double(), b.double(), padding=1, groups=Cin)
        z = (pw.double() @ d.view(K, -1)).view(1, Cout, H, H)
        zmax = max(zmax, z.abs().max().item())
        ye = torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
        y_eval[i] = ye[0].float()
        if logits is not None:
            logits[i] = (torch.einsum("c,chw->hw", ow.double().view(-1), ye[0]) + ob.double()).float()
        z += pb.double().view(1, -1, 1, 1)
        zb[i] = z[0].float()
        stats_ref += torch.cat([z.sum(dim=(0, 2, 3)), (z * z).sum(dim=(0, 2, 3))])
    del x, d, z, ye
    assert zmax < 2 ** 10, f"pre-activations reach {zmax}: the stats epilogue's fp32 sums of squares would round"
    split = ops.split_tf32(pw)
    assert bool((split[1] == 0).all())
    try:
        for mode in ("tf32", "tf32x3"):
            ws = split if mode == "tf32x3" else None
            for impl in ("smem", "regs"):
                ops.set_dsconv_impl(impl)
                what = f"integers {name} B32 {mode} {impl}"
                _exact(ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws), y_eval, f"{what} eval y")
                stats = ops.new_stats(Cout, x0.device)
                _exact(ops.dsconv(x0, w, b, KPL, pw, None, pb, False, x1=x1, mode=mode, w_split=ws, stats=stats), zb, f"{what} train y")
                _exact(stats, stats_ref, f"{what} stats")
                if logits is not None:
                    lg = ops.dsconv(x0, w, b, KPL, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws, outconv=(ow, ob))
                    _exact(lg, logits, f"{what} outconv logits")
    finally:
        ops.set_dsconv_impl("auto")


# ============================================================================================== E: pointwise forward
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
@pytest.mark.parametrize("mode", MODES)
def test_pointwise_forward_at_network_shapes(layer, mode):
    """smaat_pw1x1_fwd on the layer's own depthwise output (an exact fp32 operand): the train epilogue z + bias with the
    BatchNorm sums (functional.ds_conv_fwd) everywhere, the eval epilogue relu(scale z + shift) where the fused kernel
    declines (36x36, 18x18)."""
    name, C0, C1, Cout, H = layer
    B, Cin = _batch(H), C0 + C1
    K = KPL * Cin
    g = _gen(_seed(layer) + 3)
    x = _randn((B, Cin, H, H), g)
    w, b = _dw_params(Cin, g)
    d = ops.dw3x3(x, w, b, KPL)
    del x
    pw = _randn((Cout, K), g, K ** -0.5)
    pb = _randn((Cout,), g, 0.3)
    sc, sh = _bn_affine(Cout, g)
    if mode != "fp32":
        assert ops.tc_eligible(d, pw)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    z = pw_ref(d, pw, mode)
    what = f"pw {_lid(layer)} {mode}"
    stats = ops.new_stats(Cout, d.device)
    y = ops.pw1x1(d, pw, None, pb, False, mode=mode, w_split=ws, stats=stats)
    zb = z + pb.double().view(1, -1, 1, 1)
    _check(y, zb, ERR_BOUND["pw"][mode], f"{what} train")
    _check(stats[:Cout], zb.sum(dim=(0, 2, 3)), ERR_BOUND["pw_stats"][mode], f"{what} stats sum")
    _check(stats[Cout:], (zb * zb).sum(dim=(0, 2, 3)), ERR_BOUND["pw_stats"][mode], f"{what} stats sum of squares")
    del zb, y
    if H < 72:
        y = ops.pw1x1(d, pw, sc, sh, True, mode=mode, w_split=ws)
        _check(y, torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)), ERR_BOUND["pw"][mode], f"{what} eval")


# ============================================================================================================ F: CBAM forward
# (C, H): the five CBAMs of SmaAt-UNet (hidden C / 16, kernel 7)
CBAMS = [(64, 288), (128, 144), (256, 72), (512, 36), (512, 18)]
GATE_BN = (1.3, -0.2)        # the spatial gate's BatchNorm2d(1) as an eval affine


def _cbam_params(C, g):
    hidden = C // 16
    w1, b1 = _randn((hidden, C), g, C ** -0.5), _randn((hidden,), g, 0.1, 0.2)
    w2, b2 = _randn((C, hidden), g, hidden ** -0.5), _randn((C,), g, 0.1)
    wsp = _randn((1, 2, 7, 7), g, 0.3 / 7)
    return w1, b1, w2, b2, wsp


def _cbam_input(B, C, H, g):
    x = torch.relu(_randn((B, C, H, H), g))           # the DoubleConv output: about half exact zeros
    x[0, min(3, C - 1)] = 0.0                          # a dead plane
    return x


def _mlp64(v, w1, b1, w2, b2):
    return F.linear(torch.relu(F.linear(v, w1.double(), b1.double())), w2.double(), b2.double())


@gpu
@pytest.mark.parametrize("C, H", CBAMS, ids=[f"C{c}_S{h}" for c, h in CBAMS])
def test_cbam_forward_serving_chain(C, H):
    """What CBAM.run launches in inference: smaat_cbam_pool_mlp_fwd with the fused max-pool for C < 512 (twice: its
    last-CTA counters must come back at zero), cbam_pool_maxpool / cbam_pool + cbam_mlp at 512; cbam_reduce; then
    cbam_gate_scale into a channel slice of a wider buffer, or cbam_gate + cbam_scale at 18x18.  Max-pools, global maxima and
    the channel maximum of the fp32 products x sc are bit-exact."""
    B = _batch(H)
    g = _gen(C * 3 + H)
    w1, b1, w2, b2, wsp = _cbam_params(C, g)
    x = _cbam_input(B, C, H, g)
    bn_aff = torch.tensor(GATE_BN, device="cuda")
    what = f"cbam serve C{C} S{H}"
    avg_ref, mx_ref = x.double().mean(dim=(2, 3)), x.amax(dim=(2, 3))
    mp_ref = F.max_pool2d(x, 2) if H % 2 == 0 else None
    if C < 512:
        cnt = ops._counters(x.device, B)
        first = None
        for rep in range(2):
            sc, avg, mx, pooled = ops.cbam_pool_mlp(x, w1, b1, w2, b2, with_maxpool=True)
            torch.cuda.synchronize()
            assert int(cnt[:B].abs().sum()) == 0, "cbam_pool_mlp left its counters non-zero"
            if first is None:
                first = sc
            else:
                _exact(sc, first, f"{what} pool_mlp repeat sc")
    else:
        fused = ops.cbam_pool_maxpool(x)
        if H % 4 == 0:
            avg, mx, pooled = fused
        else:
            assert fused is None
            avg, mx = ops.cbam_pool(x)
            pooled = None
        sc = ops.cbam_mlp(avg, mx, w1, b1, w2, b2)
    _exact(mx, mx_ref, f"{what} global max")
    if pooled is not None:
        _exact(pooled, mp_ref, f"{what} max-pool")
    _check(avg, avg_ref, ERR_BOUND["cbam_pool"], f"{what} avg")
    _check(sc, torch.sigmoid(_mlp64(avg_ref, w1, b1, w2, b2) + _mlp64(mx_ref.double(), w1, b1, w2, b2)), ERR_BOUND["cbam_pool"], f"{what} sc")

    red = ops.cbam_reduce(x, sc)
    u32 = x * sc[:, :, None, None]                    # the fp32 products the kernel forms
    _exact(red[:, 1], u32.amax(dim=1), f"{what} channel max of x sc")
    _check(red[:, 0], (x.double() * sc.double()[:, :, None, None]).mean(dim=1), ERR_BOUND["cbam_pool"], f"{what} channel mean")
    del u32
    sa_ref = torch.sigmoid(F.conv2d(red.double(), wsp.double(), padding=3) * GATE_BN[0] + GATE_BN[1])
    out_ref = x.double() * sc.double()[:, :, None, None] * sa_ref
    wide = torch.full((B, C + 7, H, H), float("nan"), device="cuda")
    sl = wide[:, 4:4 + C]
    if H % 4 == 0:
        assert ops.cbam_gate_scale(x, sc, red, wsp, bn_aff, out=sl) is not None
    else:
        assert ops.cbam_gate_scale(x, sc, red, wsp, bn_aff, out=sl) is None
        sa = ops.cbam_gate(red, wsp, bn_aff)
        _check(sa, sa_ref, ERR_BOUND["cbam_out"], f"{what} gate")
        ops.cbam_scale(x, sc, sa, out=sl)
    _check(sl, out_ref, ERR_BOUND["cbam_out"], f"{what} out")
    assert bool(wide[:, :4].isnan().all()) and bool(wide[:, 4 + C:].isnan().all())


@gpu
@pytest.mark.parametrize("C, H", CBAMS, ids=[f"C{c}_S{h}" for c, h in CBAMS])
def test_cbam_forward_train_chain(C, H):
    """functional.cbam_fwd (the training forward): pools, MLP, channel reduce, the gate's raw conv, its batch statistics
    (channel_stats + bn_finalize) and the sigmoid gate, and the scaled output, against float64."""
    B = _batch(H)
    g = _gen(C * 5 + H)
    w1, b1, w2, b2, wsp = _cbam_params(C, g)
    mod = S.CBAM(C, reduction_ratio=16, kernel_size=7).cuda().train()
    with torch.no_grad():
        l1, l2, sp = mod.channel_att.MLP[1], mod.channel_att.MLP[3], mod.spatial_att
        for p, v in ((l1.weight, w1), (l1.bias, b1), (l2.weight, w2), (l2.bias, b2), (sp.conv.weight, wsp)):
            p.copy_(v)
        sp.bn.weight.fill_(1.3)
        sp.bn.bias.fill_(-0.2)
    x = _cbam_input(B, C, H, g)
    out, s = Fn.cbam_fwd(mod, x)
    what = f"cbam train C{C} S{H}"
    avg_ref, mx_ref = x.double().mean(dim=(2, 3)), x.amax(dim=(2, 3))
    _exact(s["mx"], mx_ref, f"{what} global max")
    _check(s["avg"], avg_ref, ERR_BOUND["cbam_pool"], f"{what} avg")
    sc = s["sc"]
    _check(sc, torch.sigmoid(_mlp64(avg_ref, w1, b1, w2, b2) + _mlp64(mx_ref.double(), w1, b1, w2, b2)), ERR_BOUND["cbam_pool"], f"{what} sc")
    _exact(s["pooled"][:, 1], (x * sc[:, :, None, None]).amax(dim=1), f"{what} channel max of x sc")
    raw_ref = F.conv2d(s["pooled"].double(), wsp.double(), padding=3)
    _check(s["raw"], raw_ref, ERR_BOUND["cbam_out"], f"{what} raw")
    sa_ref = torch.sigmoid(F.batch_norm(s["raw"].double(), None, None, torch.tensor([1.3], device="cuda", dtype=torch.float64),
                                        torch.tensor([-0.2], device="cuda", dtype=torch.float64), training=True, eps=sp.bn.eps))
    _check(s["sa"], sa_ref, ERR_BOUND["cbam_out"], f"{what} gate")
    _check(out, x.double() * sc.double()[:, :, None, None] * s["sa"].double(), ERR_BOUND["cbam_out"], f"{what} out")


# (h, C): the decoder's upsamplings h -> 2 h into the concat [skip (C) | upsampled (C)], and the encoder's max-pools 2 h -> h
UPS = [(18, 512), (36, 256), (72, 128), (144, 64)]


@gpu
@pytest.mark.parametrize("h, C", UPS, ids=[f"{h}to{2 * h}_C{c}" for h, c in UPS])
def test_upsample_into_concat_and_maxpool(h, C):
    """smaat_upsample2x_pad_fwd writes its C channels into the upper half of a [skip | up] concat buffer (batch stride 2 C);
    against float64 F.interpolate, calibrated on torch fp32's own error (both round the source coordinates to fp32).  The
    skip half stays untouched.  maxpool2 at 2h -> h is bit-exact."""
    B = _batch(2 * h)
    g = _gen(h + C)
    x = _randn((B, C, h, h), g)
    wide = torch.full((B, 2 * C, 2 * h, 2 * h), float("nan"), device="cuda")
    up = wide[:, C:]
    _abi("smaat_upsample2x_pad_fwd", _p(x), _p(up), wide.stride(0), B, C, h, h, 2 * h, 2 * h, ops._stream())
    ref = F.interpolate(x.double(), scale_factor=2, mode="bilinear", align_corners=True)
    noise = _rel(F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True), ref)
    _check(up, ref, UPSAMPLE_FACTOR * noise + 1e-6, f"upsample {h}->{2 * h} C{C} into concat (torch fp32 {noise:.2e})")
    assert bool(wide[:, :C].isnan().all())
    skip = _randn((B, C, 2 * h, 2 * h), g)
    _exact(ops.maxpool2(skip), F.max_pool2d(skip, 2), f"maxpool2 {2 * h}->{h} C{C}")


# ============================================================================================== G: depthwise backward
@gpu
@pytest.mark.parametrize("layer", LAYERS, ids=_lid)
def test_depthwise_backward_at_network_shapes(layer):
    """smaat_dw3x3_bwd_input (TMA where W % 4 == 0, the tiled kernel at 18x18 and on a misaligned dd) split over the
    concat, and smaat_dw3x3_bwd_weight (TMA / tiled the same way) accumulating into non-zero dW, db, with the BN+ReLU
    prologue on conv 1 and without it, against float64.  inc.0 runs at B = 32 (2.65 M-term weight reductions)."""
    name, C0, C1, Cout, H = layer
    B = 32 if name == "inc.0" else _batch(H)
    Cin = C0 + C1
    K = KPL * Cin
    g = _gen(_seed(layer) + 4)
    x = _randn((B, Cin, H, H), g)
    w, _ = _dw_params(Cin, g)
    dd = _randn((B, K, H, H), g)
    x0, x1 = _split(x, C0, C1)
    what = f"dw bwd {_lid(layer)}"
    st = ops._stream()
    dx_ref = dw_input_grad_ref(dd, w, KPL)
    for variant in ("aligned", "misaligned"):
        ddv = dd if variant == "aligned" else _offset(dd)
        dx0 = torch.full((B, C0, H, H), float("nan"), device="cuda")
        dx1 = torch.full((B, C1, H, H), float("nan"), device="cuda") if C1 else None
        _abi("smaat_dw3x3_bwd_input", _p(ddv), _p(w), _p(dx0), C0, C0 * H * H, _p(dx1), C1, C1 * H * H, B, H, H, KPL, st)
        _check(dx0, dx_ref[:, :C0], ERR_BOUND["dw_dx"], f"{what} dx0 {variant}")
        if C1:
            _check(dx1, dx_ref[:, C0:], ERR_BOUND["dw_dx"], f"{what} dx1 {variant}")
        del ddv, dx0, dx1
    del dx_ref
    pros = [False, True] if name.endswith(".1") else [False]
    for pro in pros:
        sc, sh = _bn_affine(Cin, g) if pro else (None, None)
        xa = prologue(x, sc, sh) if pro else x
        dW_ref, db_ref = dw_weight_grad_ref(dd, xa, KPL)
        del xa
        dW0 = _randn((K, 9), g, 0.3 * dW_ref.abs().max().item())
        db0 = _randn((K,), g, 0.3 * db_ref.abs().max().item())
        for variant in ("aligned", "misaligned"):
            ddv = dd if variant == "aligned" else _offset(dd)
            dW, db = dW0.clone(), db0.clone()
            _abi("smaat_dw3x3_bwd_weight", _p(ddv), _p(x0), C0, C0 * H * H, _p(x1), C1, C1 * H * H, _p(sc), _p(sh), _p(dW), _p(db), B, H,
                 H, KPL, st)
            _check(dW, dW0.double() + dW_ref, ERR_BOUND["dw_dw"], f"{what} dW prologue={pro} {variant}")
            _check(db, db0.double() + db_ref, ERR_BOUND["dw_dw"], f"{what} db prologue={pro} {variant}")
            del ddv
