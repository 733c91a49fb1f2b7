"""The serving forward's CBAM fusions (smaat_dsconv_cbam_fwd, smaat_cbam_mlp_partials_fwd) against float64 at their edges.

Levels 1-3 of SmaAt_UNet.forward_serving never write their CBAM output: the first DS conv of up2 / up3 / up4 reads the skip
as (x * sc) * sa while it loads it (the gate), and the same entry point can write the channel gate's per half-patch partial
pools and MaxPool2d(2) of its output from the staged epilogue (the pools).  tests/test_gpu_cbam_serving_fusion.py checks
both against the library's own unfused kernels at the 288 network's shapes in the register A form.  This file adds a
float64 reference, the shared-memory A form and the shapes where these paths go wrong:

  A  the dispatch table, on the CPU: DsCfg's ST_BUFS restated for all 16 instances (N_TILE {64, 128} x k {1, 2} x PW
     {16, 32} x {tf32, tf32x3} x {smem, regs}); smaat_dsconv_cbam_eligible(with_pools=1) follows it under every
     smaat_set_dsconv_impl, with_gate never declines, the direct-store instances (ST_BUFS = 0) are k = 1 in tf32x3 at
     N_TILE 64 in the smem form and at N_TILE 128 in the register form; smaat_dsconv_pool_parts against a restated pick_pw
  B  the gate, tf32 and tf32x3, both A forms: up2.0 / up3.0 / up4.0 of the 288 and 576 networks, k = 1 on the
     direct-store instances, H = 99 x W = 96 (PW 32, odd H: the sa halo box at the bottom edge), H = 70 x W = 100 (PW 16,
     partial tiles both ways), B = 1, x0 alone (C1 = 0, a partial last chunk), batch-strided channel slices, Cout 40 and
     96; sa exactly 0 on a row band and 1 on a column band, sc = 0 on every fifth channel, everywhere.  One production
     launch (B = 32, up4.0 of the 288 network).  Refusals: a misaligned sa or sc without sa raise and write nothing; fp32
     is declined and DoubleConvDS.run(gate=...) materialises the CBAM output with cbam_scale instead
  C  the pools through the C ABI into NaN-poisoned buffers with guard tails, wherever part A says they are taken (and
     refused without a write where it says not): k = 1 and 2, Cout 40 / 64 / 96 / 128 / 256, 288^2 at Cout 128 (PW 32 with
     N_TILE 128, four 32-channel slices per warpgroup), H = 45 x W = 52 (warpgroup 1 of the last tile row lies wholly
     below the image: pmax = -inf), H = 37 x W = 40, level 1 at 576 (npart = 5 184), signed outputs (relu=False), and
     one launch with gate and pools together
  D  UpDS with gate=cbam.serving_gates(skip) against UpDS on cbam(skip) at up2 / up3 / up4 of both networks (B = 2, fp32
     / tf32 / tf32x3, both forms); forward_serving against forward in fp32 at 288 and 576; forward_serving at 576
     (B = 2, tf32x3) against the float64 port; the 576 serving forward's CBAM launch inventory, derived from the model

Conventions:
  * references are those of tests/test_gpu_ds_forward_kernels.py (dw_emul is bit-equal to the depthwise stencil, pw_ref
    multiplies tf32-truncated or split operands exactly in float64); the gated input is formed in fp32 on the CPU, whose
    multiply rounds as __fmul_rn does, in the CBAM kernels' order (x * sc) * sa;
  * the gated conv must be bit-equal to ops.dsconv on ops.cbam_scale's output (same products, same stencil, same MMAs), and
    the smem and register forms bit-equal to each other;
  * a partial pool covers one warpgroup's half-patch: rows ty PH + wg PH / 2 .. + PH / 2, columns tx PW .. + PW, clipped
    to the image, at index 2 (ty tiles_x + tx) + wg.  Its maximum must be exact, its sum within 64 2^-24 x that
    half-patch's sum of |y| (a 64-term fp32 sum's worst case);
  * errors are max |got - ref| / max |ref|, as tests/_util.assert_close measures them.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than
10x above it, with one exception: the partial sums are held to the analytical worst case of a 64-term fp32 sum, which
cannot fail on a correct kernel whatever the data (everything else is bit-exact and was):

  quantity                                                   worst observed                 bound
  B  gated DS conv y, tf32 / tf32x3 (288 up2.0)              1.9e-6 / 5.9e-6                1.5e-5 / 5e-5
  C  partial sums, |err| / (64 2^-24 sum |y|)                0.046                          1 (analytical)
     channel mean, MLP gate sc from the partials             2.9e-7                         2.5e-6
  D  576 serving logits against the float64 port             3.5e-7                         max(2e-6, 5 x 3.2e-7)
                                                             (port fp32 vs float64: 3.2e-7)

The gate bounds are half of the fused DS conv's in tests/test_gpu_ds_forward_kernels.py, which observes the same kernel
without the gate.  Mutations of csrc/dsconv_fused.cu, one at a time, and what failed:
  * (x * sa) * sc in the smem form's stencil only: every part B and D case, in its smem form only (tf32 and tf32x3); the
    fp32 and register-form checks and tests/test_gpu_cbam_serving_fusion.py (register form) pass;
  * the partial sums without the second-row mask: the odd-H pool cases (45 x 52, 37 x 40, gate + pools);
  * warpgroup partials written at 2 (ty tiles_x + tx) + (1 - wg): every part C case, on the per-partial maxima, while
    tests/test_gpu_cbam_serving_fusion.py's totals after the MLP still pass;
  * the sa halo box loaded at y0 instead of y0 - 1: every part B and D gated case and the 576 serving forward.
The whole file runs in ~8 s on one H100 at a peak of 4.0 GiB allocated.
"""
import math
from collections import Counter

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import _lib, ops
from tests._util import load_np_state_dict
from tests.test_gpu_ds_forward_kernels import (_abi, _bn_affine, _cbam_params, _check, _exact, _gen, _mlp64, _offset, _p,
                                               _randn, _rel, _slice_of_wider, dw_emul, pw_ref)

gpu = pytest.mark.gpu
IMPLS = ("smem", "regs")
TC_MODES = ("tf32", "tf32x3")
MODE_CODE = {"fp32": 0, "tf32": 1, "tf32x3": 2}
GATE_BOUND = {"tf32": 1.5e-5, "tf32x3": 5e-5}   # gated DS conv y against the float64 reference (half of the fused DS conv bounds of test_gpu_ds_forward_kernels)
MLP_BOUND = 2.5e-6           # channel mean and gate sc from the partials against float64 pools and MLP
PART_SUM_TERMS = 64          # pixels per half-patch: the partial sums' worst-case rounding is 64 2^-24 sum |y|
NET_NOISE_FACTOR, NET_FLOOR = 5.0, 2e-6      # as tests/test_gpu_576_kernels.py part G


@pytest.fixture
def ds_impl():
    """ops.set_dsconv_impl for the test's own calls; 'auto' and the pointwise mode are restored afterwards."""
    mode = ops.get_pointwise_mode()
    try:
        yield ops.set_dsconv_impl
    finally:
        ops.set_dsconv_impl("auto")
        ops.set_pointwise_mode(mode)


# ============================================================================================== A: dispatch table (CPU)
def pick_pw(H, W):
    """csrc/dsconv_fused.cu pick_pw: patch width 32 (4 rows) or 16 (8 rows), whichever pads the plane less (32 on a tie),
    0 when even the better one pads it by more than 35 %."""
    best, pw = 1e9, 0
    for c in (32, 16):
        ph = 128 // c
        waste = (-(-W // c) * c / W) * (-(-H // ph) * ph / H)
        if waste < best - 1e-9:
            best, pw = waste, c
    return pw if best <= 1.35 else 0


def st_bufs(n_tile, k, pw, x3, a_smem):
    """DsCfg<N_TILE, KPL, PW, X3, A_SMEM>::ST_BUFS: output staging buffers per consumer warpgroup, from the shared memory
    the A, weight and input rings leave (2 wanted, 1 where 2 would leave the input ring under 2 stages, 0 = direct stores)."""
    ph = 128 // pw
    in_bytes = (32 // k) * (ph + 2) * (pw + 8) * 4
    a_bytes, b_bytes = 128 * 32 * 4, n_tile * 32 * 4
    ng = 1 if n_tile > 64 else 2
    ast = (2 if x3 and a_smem else 1) * a_bytes
    bst = (2 if x3 else 1) * b_bytes
    n_as = ((2 if n_tile > 64 else 3) if a_smem else 2 + ng) if x3 else 4
    n_bs = (2 if a_smem and n_tile > 64 else 3) if x3 else 4
    free = 224 * 1024 - 1024 - 512 - 3 * 512 * 4 - n_as * ast - n_bs * bst
    box = 32 * 64 * 4
    if (free - 2 * 2 * box) // in_bytes >= 2:
        return 2
    return 1 if (free - 2 * box) // in_bytes >= 2 else 0


INSTANCES = [(nt, k, pw, x3, sm) for nt in (64, 128) for k in (1, 2) for pw in (16, 32) for x3 in (False, True) for sm in (True, False)]
PLANE_OF_PW = {32: (64, 64), 16: (72, 72)}      # square planes pick_pw sends to each patch width


def _eligible(lib, k, Cout, H, W, mode, gate, pools):
    x0, w = 1 << 20, 3 << 20                     # 16-byte aligned dummy pointers: eligibility never dereferences them
    return lib.smaat_dsconv_cbam_eligible(x0, 32, 32 * H * W, None, 0, 0, w, H, W, k, Cout, mode, int(gate), int(pools))


def test_dispatch_table_st_bufs_and_eligibility(ds_impl):
    """The pools are taken exactly where the dispatched instance stages its output (ST_BUFS > 0), under each A form ('auto'
    is the register form); the gate is taken by every instance; fp32 takes neither."""
    lib = _lib.load()
    direct = {i for i in INSTANCES if st_bufs(*i) == 0}
    assert direct == {(64, 1, pw, True, True) for pw in (16, 32)} | {(128, 1, pw, True, False) for pw in (16, 32)}, direct
    assert all(st_bufs(128, 1, pw, x3, True) == 1 for pw in (16, 32) for x3 in (False, True))     # single-buffer staging
    for pw, (H, W) in PLANE_OF_PW.items():
        assert pick_pw(H, W) == pw
    for impl in ("auto", "smem", "regs"):
        ds_impl(impl)
        smem = impl == "smem"
        for nt, k, pw, x3, sm in INSTANCES:
            if sm != smem:
                continue
            H, W = PLANE_OF_PW[pw]
            Cout = 64 if nt == 64 else 128
            mode = MODE_CODE["tf32x3" if x3 else "tf32"]
            what = (impl, nt, k, pw, x3)
            assert _eligible(lib, k, Cout, H, W, mode, False, True) == int(st_bufs(nt, k, pw, x3, sm) > 0), what
            assert _eligible(lib, k, Cout, H, W, mode, True, False) == 1, what
            assert _eligible(lib, k, Cout, H, W, mode, True, True) == int(st_bufs(nt, k, pw, x3, sm) > 0), what
            for gate, pools in ((1, 0), (0, 1), (1, 1)):
                assert _eligible(lib, k, Cout, H, W, MODE_CODE["fp32"], gate, pools) == 0, what


def test_pool_parts_matches_restated_pick_pw():
    lib = _lib.load()
    sizes = list(range(1, 160, 3)) + [288, 576, 1000]
    for H in sizes:
        for W in sizes:
            pw = pick_pw(H, W)
            want = 2 * math.ceil(W / pw) * math.ceil(H / (128 // pw)) if pw else 0
            assert lib.smaat_dsconv_pool_parts(H, W) == want, (H, W, pw)
    assert lib.smaat_dsconv_pool_parts(0, 64) == 0 and lib.smaat_dsconv_pool_parts(64, 0) == 0
    assert lib.smaat_dsconv_pool_parts(576, 576) == 5184 and lib.smaat_dsconv_pool_parts(45, 52) == 2 * 2 * 12


# ================================================================================================== shared GPU helpers
def _conv_params(Cin, Cout, k, g):
    K = k * Cin
    return dict(dw_w=_randn((K, 1, 3, 3), g, 1.0 / 3.0), dw_b=_randn((K,), g, 0.1), pw=_randn((Cout, K), g, K ** -0.5),
                scale=_bn_affine(Cout, g)[0], shift=_randn((Cout,), g, 0.5, 0.2))


def _gate_inputs(B, C0, C1, H, W, g):
    """The un-attended skip (post-ReLU), the decoder map, and gates with exact 0 / 1 bands and dead channels."""
    x0 = torch.relu(_randn((B, C0, H, W), g))
    x1 = _randn((B, C1, H, W), g) if C1 else None
    sc = torch.rand((B, C0), generator=g, device="cuda")
    sc[:, ::5] = 0.0
    sa = torch.rand((B, 1, H, W), generator=g, device="cuda")
    sa[:, :, H // 3:H // 3 + 3] = 0.0
    sa[:, :, :, W // 2:W // 2 + 5] = 1.0
    return x0, x1, sc, sa


def _gated_input(x0, sc, sa):
    """(x0 * sc) * sa in fp32 on the CPU: two correctly rounded products, the CBAM kernels' order."""
    return ((x0.cpu() * sc.cpu()[:, :, None, None]) * sa.cpu()).to(x0.device)


def _eval_ref(d, prm, mode):
    z = pw_ref(d, prm["pw"], mode)
    return torch.relu(z * prm["scale"].double().view(1, -1, 1, 1) + prm["shift"].double().view(1, -1, 1, 1))


# ============================================================================================================ B: the gate
# (id, B, C0, C1, H, W, Cout, k, batch-strided slices)
GATE_CASES = [
    ("288_up2.0", 2, 256, 256, 72, 72, 256, 2, False),
    ("288_up3.0", 2, 128, 128, 144, 144, 128, 2, False),
    ("288_up4.0", 2, 64, 64, 288, 288, 64, 2, False),
    ("576_up2.0", 2, 256, 256, 144, 144, 256, 2, False),
    ("576_up3.0", 1, 128, 128, 288, 288, 128, 2, False),
    ("576_up4.0", 1, 64, 64, 576, 576, 64, 2, False),
    ("k1_N64_direct_smem_x3", 2, 64, 32, 64, 64, 64, 1, False),
    ("k1_N128_direct_regs_x3", 2, 32, 64, 48, 48, 128, 1, False),
    ("H99_W96_pw32", 2, 32, 32, 99, 96, 64, 2, False),
    ("H70_W100_pw16", 2, 32, 32, 70, 100, 64, 2, False),
    ("B1", 1, 64, 64, 96, 96, 64, 2, False),
    ("x0_only_C40", 2, 40, 0, 64, 64, 64, 2, False),
    ("slices", 2, 64, 64, 72, 72, 128, 2, True),
    ("Cout40", 2, 32, 32, 64, 64, 40, 2, False),
    ("Cout96", 2, 32, 32, 64, 64, 96, 2, False),
]


@gpu
@pytest.mark.parametrize("case", GATE_CASES, ids=lambda c: c[0])
def test_gated_conv_against_float64_and_the_materialised_path(case, ds_impl):
    name, B, C0, C1, H, W, Cout, k, sliced = case
    g = _gen(sum(map(ord, name)))
    x0, x1, sc, sa = _gate_inputs(B, C0, C1, H, W, g)
    prm = _conv_params(C0 + C1, Cout, k, g)
    xg = _gated_input(x0, sc, sa)
    _exact(ops.cbam_scale(x0, sc, sa), xg, f"gate {name} cbam_scale vs fp32 CPU products")
    d = dw_emul(torch.cat([xg, x1], 1) if C1 else xg, prm["dw_w"], prm["dw_b"], k)
    del xg
    if sliced:
        x0, x1 = _slice_of_wider(x0), _slice_of_wider(x1, 1, 5)
        assert not x0.is_contiguous() and x0.data_ptr() % 16 == 0
    split = ops.split_tf32(prm["pw"])
    n_tile = 64 if Cout <= 64 else 128
    direct = [(m, i) for m in TC_MODES for i in IMPLS if st_bufs(n_tile, k, pick_pw(H, W), m == "tf32x3", i == "smem") == 0]
    if name.startswith("k1_"):
        assert direct, "this case is meant to reach a direct-store instance"
    for mode in TC_MODES:
        ws = split if mode == "tf32x3" else None
        ref = _eval_ref(d, prm, mode)
        got = {}
        for impl in IMPLS:
            ds_impl(impl)
            what = f"gate {name} {mode} {impl}{' (direct store)' if (mode, impl) in direct else ''}"
            assert ops.dsconv_cbam_takes(x0, x1, prm["pw"], k, gate=True, mode=mode), f"{what}: declined"
            y = ops.dsconv_cbam(x0, prm["dw_w"], prm["dw_b"], k, prm["pw"], prm["scale"], prm["shift"], True, x1=x1, mode=mode,
                                w_split=ws, gate=(sc, sa))
            mat = ops.dsconv(ops.cbam_scale(x0, sc, sa), prm["dw_w"], prm["dw_b"], k, prm["pw"], prm["scale"], prm["shift"], True,
                             x1=x1, mode=mode, w_split=ws)
            assert mat is not None
            _exact(y, mat, f"{what} vs dsconv on cbam_scale")
            _check(y, ref, GATE_BOUND[mode], f"{what} vs float64")
            got[impl] = y
            del mat
        _exact(got["regs"], got["smem"], f"gate {name} {mode} regs vs smem")
        del ref, got


@gpu
def test_gated_conv_production_launch(ds_impl):
    """B = 32 at up4.0 of the 288 network (20 736 tiles): bit-equal to the conv on the materialised CBAM output."""
    B, C, S_ = 32, 64, 288
    g = _gen(77)
    x0, x1, sc, sa = _gate_inputs(B, C, C, S_, S_, g)
    prm = _conv_params(2 * C, C, 2, g)
    ws = ops.split_tf32(prm["pw"])
    mat = ops.dsconv(ops.cbam_scale(x0, sc, sa), prm["dw_w"], prm["dw_b"], 2, prm["pw"], prm["scale"], prm["shift"], True, x1=x1,
                     mode="tf32x3", w_split=ws)
    for impl in IMPLS:
        ds_impl(impl)
        y = ops.dsconv_cbam(x0, prm["dw_w"], prm["dw_b"], 2, prm["pw"], prm["scale"], prm["shift"], True, x1=x1, mode="tf32x3",
                            w_split=ws, gate=(sc, sa))
        _exact(y, mat, f"gate production B32 up4.0 tf32x3 {impl}")
        del y


def _cbam_fwd_abi(x0, x1, prm, k, mode, y, sc=None, sa=None, psum=None, pmax=None, pooled=None, relu=True, x0_bstride=None,
                  x1_bstride=None):
    B, C0, H, W = x0.shape
    C1 = x1.shape[1] if x1 is not None else 0
    Cout = prm["pw"].shape[0]
    hi, lo = ops.split_tf32(prm["pw"]) if mode == "tf32x3" else (prm["pw"], None)
    _abi("smaat_dsconv_cbam_fwd", _p(x0), C0, x0_bstride or C0 * H * W, _p(x1), C1, x1_bstride or C1 * H * W, _p(prm["dw_w"]),
         _p(prm["dw_b"]), _p(hi), _p(lo), _p(prm["scale"]), _p(prm["shift"]), _p(y), Cout * H * W, _p(sc), _p(sa), _p(psum), _p(pmax),
         _p(pooled), B, H, W, k, Cout, int(relu), MODE_CODE[mode], ops._stream())


@gpu
def test_gate_refusals(ds_impl):
    """A misaligned sa, or sc without sa: an error before any launch, y untouched.  fp32: declined by dsconv_cbam_takes and
    refused by dsconv_cbam; DoubleConvDS.run(gate=...) then materialises (x * sc) * sa with cbam_scale and runs the plain convs."""
    B, C, S_ = 2, 64, 64
    g = _gen(78)
    x0, x1, sc, sa = _gate_inputs(B, C, C, S_, S_, g)
    prm = _conv_params(2 * C, C, 2, g)
    y = torch.full((B, C, S_, S_), float("nan"), device="cuda")
    for what, sc_, sa_, msg in (("misaligned sa", sc, _offset(sa), "16-byte aligned"), ("sc without sa", sc, None, "both sc and sa")):
        with pytest.raises(RuntimeError, match=msg):
            _cbam_fwd_abi(x0, x1, prm, 2, "tf32x3", y, sc=sc_, sa=sa_)
        torch.cuda.synchronize()
        assert bool(y.isnan().all()), f"{what}: the refused call wrote its output"
    assert not ops.dsconv_cbam_takes(x0, x1, prm["pw"], 2, gate=True, mode="fp32")
    with pytest.raises(RuntimeError, match="does not take"):
        ops.dsconv_cbam(x0, prm["dw_w"], prm["dw_b"], 2, prm["pw"], prm["scale"], prm["shift"], True, x1=x1, mode="fp32", gate=(sc, sa))
    m = _model()
    conv = m.up4.conv                                     # DoubleConvDS(128, 64, 64): skip 64 | upsampled 64
    ops.set_pointwise_mode("fp32")
    with torch.no_grad():
        with ops.profile() as prof:
            got = conv.run(x0, x1=x1, gate=(sc, sa))
        names = [r[0].split("[")[0] for r in prof.records]
        ref = conv.run(ops.cbam_scale(x0, sc, sa), x1=x1)
    assert names.count("smaat_cbam_scale_fwd") == 1 and "smaat_dsconv_fwd" not in names, names
    _exact(got, ref, "DoubleConvDS.run(gate) in fp32 vs run(cbam_scale(x))")


# ============================================================================================================ C: the pools
def _partials_ref(y, pw):
    """float64 (sum, max, sum |y|) over each warpgroup's half-patch, in the kernel's partial layout (B, npart, C)."""
    B, C, H, W = y.shape
    ph = 128 // pw
    tx, ty = -(-W // pw), -(-H // ph)
    pad = (0, tx * pw - W, 0, ty * ph - H)
    yd = y.double()

    def fold(t, op):
        t = t.view(B, C, ty, 2, ph // 2, tx, pw)
        t = t.amax(dim=(4, 6)) if op == "max" else t.sum(dim=(4, 6))
        return t.permute(0, 2, 4, 3, 1).reshape(B, ty * tx * 2, C)

    return (fold(F.pad(yd, pad), "sum"), fold(F.pad(yd, pad, value=float("-inf")), "max"), fold(F.pad(yd.abs(), pad), "sum"))


def _poisoned(n, guard=37):
    buf = torch.full((n + guard,), float("nan"), device="cuda")
    return buf, buf[:n]


# (id, B, Cin, H, W, Cout, k, relu)
POOL_CASES = [
    ("k2_N64_H45_W52", 2, 32, 45, 52, 64, 2, True),          # wg 1 of the last tile row wholly below the image
    ("k1_N40_H37_W40_signed", 2, 24, 37, 40, 40, 1, False),  # odd H (half a row pair in the image), Cout 40, k = 1
    ("k2_N96_H37_W40_signed", 2, 48, 37, 40, 96, 2, False),  # N_TILE 128 with three slices
    ("k1_N64_64x96", 2, 16, 64, 96, 64, 1, True),            # tf32x3 smem is a direct-store instance: refused there
    ("k1_N128_64x64", 2, 32, 64, 64, 128, 1, True),          # ST_BUFS = 1 (smem), tf32x3 regs refused
    ("k2_N128_288_pw32", 1, 128, 288, 288, 128, 2, True),    # level 2 of the 576 network: PW 32 with N_TILE 128
    ("k2_N256_72_signed", 2, 128, 72, 72, 256, 2, False),    # two channel passes
    ("k2_N64_576_level1", 1, 64, 576, 576, 64, 2, True),     # npart = 5 184
]


def _check_pools(name, y, psum, pmax, pooled, H, W, g):
    B, Cout = y.shape[:2]
    pw = pick_pw(H, W)
    s_ref, m_ref, a_ref = _partials_ref(y, pw)
    assert psum.shape == s_ref.shape
    _exact(pmax.double(), m_ref, f"{name} partial maxima")
    if H % (128 // pw) and (H % (128 // pw)) <= (64 // pw):
        assert bool((m_ref == float("-inf")).any()), f"{name}: expected half-patches wholly below the image"
    err = (psum.double() - s_ref).abs()
    lim = PART_SUM_TERMS * 2.0 ** -24 * a_ref
    ratio = (err / lim.clamp_min(1e-300)).max().item()
    print(f"ERR {name} partial sums: {ratio:.3e} of the 64-term bound")
    assert bool((err <= lim).all()), f"{name} partial sums: worst {ratio:.3f} x the bound"
    _exact(pooled, ops.maxpool2(y), f"{name} max-pool vs maxpool2")
    _exact(pooled, F.max_pool2d(y, 2), f"{name} max-pool vs F.max_pool2d (floor)")
    w1, b1, w2, b2, _ = _cbam_params(Cout, g)
    out = ops.cbam_mlp_partials(psum.view(B, -1, Cout), pmax.view(B, -1, Cout), H, W, w1, b1, w2, b2)
    if Cout % 16:
        assert out is None
        return
    sc, avg, mx = out
    avg_ref, mx_ref = y.double().mean(dim=(2, 3)), y.amax(dim=(2, 3))
    _exact(mx, mx_ref, f"{name} channel max from the partials")
    _check(avg, avg_ref, MLP_BOUND, f"{name} channel mean from the partials")
    _check(sc, torch.sigmoid(_mlp64(avg_ref, w1, b1, w2, b2) + _mlp64(mx_ref.double(), w1, b1, w2, b2)), MLP_BOUND,
           f"{name} gate sc from the partials")


def _run_pools(name, x0, x1, prm, k, mode, relu, gate=None):
    """One pools launch into poisoned buffers: (y, psum, pmax, pooled), each checked fully written and its guard untouched."""
    B, _, H, W = x0.shape
    Cout = prm["pw"].shape[0]
    npart = _lib.load().smaat_dsconv_pool_parts(H, W)
    bufs = [_poisoned(n) for n in (B * Cout * H * W, B * npart * Cout, B * npart * Cout, B * Cout * (H // 2) * (W // 2))]
    (yb, y), (sb, ps), (mb, pm), (pb, po) = bufs
    sc, sa = gate if gate is not None else (None, None)
    _cbam_fwd_abi(x0, x1, prm, k, mode, y, sc=sc, sa=sa, psum=ps, pmax=pm, pooled=po, relu=relu)
    torch.cuda.synchronize()
    for what, (buf, v) in zip(("y", "psum", "pmax", "pooled"), bufs):
        assert not bool(v.isnan().any()), f"{name}: {int(v.isnan().sum())} of {v.numel()} {what} elements not written"
        assert bool(buf[v.numel():].isnan().all()), f"{name}: {what} written past its end"
    return y.view(B, Cout, H, W), ps.view(B, npart, Cout), pm.view(B, npart, Cout), po.view(B, Cout, H // 2, W // 2)


@gpu
@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: c[0])
def test_epilogue_pools_against_float64_half_patches(case, ds_impl):
    name, B, Cin, H, W, Cout, k, relu = case
    g = _gen(sum(map(ord, name)) + 1)
    x = _randn((B, Cin, H, W), g)
    prm = _conv_params(Cin, Cout, k, g)
    pw, n_tile = pick_pw(H, W), (64 if Cout <= 64 else 128)
    taken = 0
    for mode in TC_MODES:
        ws = ops.split_tf32(prm["pw"]) if mode == "tf32x3" else None
        for impl in IMPLS:
            ds_impl(impl)
            what = f"pools {name} {mode} {impl}"
            staged = st_bufs(n_tile, k, pw, mode == "tf32x3", impl == "smem") > 0
            assert ops.dsconv_cbam_takes(x, None, prm["pw"], k, pools=True, mode=mode) == staged, what
            if not staged:
                npart = _lib.load().smaat_dsconv_pool_parts(H, W)
                (sb, ps), y = _poisoned(B * npart * Cout), torch.full((B, Cout, H, W), float("nan"), device="cuda")
                pm, po = torch.empty_like(ps), torch.empty((B, Cout, H // 2, W // 2), device="cuda")
                with pytest.raises(RuntimeError, match="staged epilogue"):
                    _cbam_fwd_abi(x, None, prm, k, mode, y, psum=ps, pmax=pm, pooled=po, relu=relu)
                torch.cuda.synchronize()
                assert bool(sb.isnan().all()) and bool(y.isnan().all()), f"{what}: the refused call wrote"
                continue
            taken += 1
            y, ps, pm, po = _run_pools(what, x, None, prm, k, mode, relu)
            _exact(y, ops.dsconv(x, prm["dw_w"], prm["dw_b"], k, prm["pw"], prm["scale"], prm["shift"], relu, mode=mode, w_split=ws),
                   f"{what} y vs dsconv")
            _check_pools(what, y, ps, pm, po, H, W, g)
            del y, ps, pm, po
    assert taken >= 2


@gpu
def test_gate_and_pools_in_one_launch(ds_impl):
    """Both fusions at once (not a serving-forward combination, but one entry point takes it): y bit-equal to the conv on the
    materialised CBAM output, the pools checked on that y."""
    B, C0, C1, H, W, Cout = 2, 32, 32, 37, 40, 64
    g = _gen(91)
    x0, x1, sc, sa = _gate_inputs(B, C0, C1, H, W, g)
    prm = _conv_params(C0 + C1, Cout, 2, g)
    for mode in TC_MODES:
        ws = ops.split_tf32(prm["pw"]) if mode == "tf32x3" else None
        for impl in IMPLS:
            ds_impl(impl)
            what = f"gate+pools {mode} {impl}"
            assert ops.dsconv_cbam_takes(x0, x1, prm["pw"], 2, gate=True, pools=True, mode=mode)
            y, ps, pm, po = _run_pools(what, x0, x1, prm, 2, mode, True, gate=(sc, sa))
            mat = ops.dsconv(ops.cbam_scale(x0, sc, sa), prm["dw_w"], prm["dw_b"], 2, prm["pw"], prm["scale"], prm["shift"], True, x1=x1,
                             mode=mode, w_split=ws)
            _exact(y, mat, f"{what} y vs dsconv on cbam_scale")
            _check_pools(what, y, ps, pm, po, H, W, g)


@gpu
def test_mlp_partials_declines_untaken_shapes():
    """C % 16 != 0, C > 512 or hidden > 64: None before any launch."""
    for C, hidden in ((40, 2), (528, 33), (512, 65)):
        ps = torch.zeros((1, 4, C), device="cuda")
        w1, b1 = torch.zeros((hidden, C), device="cuda"), torch.zeros(hidden, device="cuda")
        w2, b2 = torch.zeros((C, hidden), device="cuda"), torch.zeros(C, device="cuda")
        assert ops.cbam_mlp_partials(ps, ps, 8, 8, w1, b1, w2, b2) is None, (C, hidden)


# ================================================================================================ D: blocks and networks
_MODELS = {}


def _model():
    """SmaAt_UNet(12, 1, kernels_per_layer=2) with the schema-filled weights of the 576 file (seed 5), eval, cached."""
    if "m" not in _MODELS:
        sd = cast_sd(fill_schema(smaat_unet_schema(12, 1, 2), 5), np.float32)
        _MODELS["sd"] = sd
        _MODELS["m"] = load_np_state_dict(S.SmaAt_UNet(12, 1, kernels_per_layer=2), sd).cuda().eval()
    return _MODELS["m"]


# (up block, the CBAM whose gates it applies, that level's index): the three gated decoder blocks
GATED_UPS = [("up2", "cbam3", 2), ("up3", "cbam2", 1), ("up4", "cbam1", 0)]
NETS = (288, 576)


@gpu
@pytest.mark.parametrize("net", NETS)
@pytest.mark.parametrize("up, cbam, lvl", GATED_UPS, ids=[u for u, _, _ in GATED_UPS])
def test_up_block_with_serving_gates_is_bit_equal(up, cbam, lvl, net, ds_impl):
    """UpDS(y, skip, gate=cbam.serving_gates(skip)) against UpDS(y, cbam(skip)), bit for bit: fp32 (cbam_scale fallback),
    tf32 and tf32x3 (gate on load), both A forms; up4 also with the fused OutConv."""
    m = _model()
    C, S_ = (64, 128, 256)[lvl], net >> lvl
    g = _gen(net + lvl)
    skip = torch.relu(_randn((2, C, S_, S_), g))
    y_in = _randn((2, C, S_ // 2, S_ // 2), g)
    block, att = getattr(m, up), getattr(m, cbam)
    with torch.no_grad():
        for mode in ("fp32", "tf32", "tf32x3"):
            ops.set_pointwise_mode(mode)
            for impl in IMPLS:
                ds_impl(impl)
                sc, sa, _ = att.serving_gates(skip)
                got = block(y_in, skip, gate=(sc, sa))
                ref = block(y_in, att(skip))
                _exact(got, ref, f"{net} {up} {mode} {impl} gate vs cbam output")
                if up == "up4":
                    _exact(block(y_in, skip, outconv=m.outc, gate=(sc, sa)), block(y_in, att(skip), outconv=m.outc),
                           f"{net} {up} {mode} {impl} + OutConv gate vs cbam output")
                del got, ref


def _frames(B, S_, seed):
    return torch.from_numpy(np.random.default_rng(seed).uniform(0, 1, (B, 12, S_, S_)).astype(np.float32)).cuda()


@gpu
@pytest.mark.parametrize("net", NETS)
def test_forward_serving_is_forward_in_fp32(net, ds_impl):
    """In fp32 nothing is fused: the gated blocks materialise (x * sc) * sa with cbam_scale, the product cbam_gate_scale
    forms in forward, so the logits are the same bits."""
    m = _model()
    x = _frames(2, net, net)
    ops.set_pointwise_mode("fp32")
    with torch.no_grad():
        _exact(m.forward_serving(x), m(x), f"forward_serving vs forward fp32 at {net}")


class _NoTF32:
    def __enter__(self):
        self.old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False

    def __exit__(self, *exc):
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = self.old
        return False


@gpu
def test_forward_serving_at_576_against_float64_port(ds_impl):
    """The path configs[4] times: B = 2, tf32x3, bounded as the plain forward is in tests/test_gpu_576_kernels.py."""
    m = _model()
    x = _frames(2, 576, 9)
    with torch.no_grad():
        ref = TP.smaat_unet_forward(x.double(), TP.to_torch_sd(_MODELS["sd"], torch.float64, "cuda"))
        with _NoTF32():
            noise = _rel(TP.smaat_unet_forward(x, TP.to_torch_sd(_MODELS["sd"], torch.float32, "cuda")), ref)
        ops.set_pointwise_mode("tf32x3")
        y = m.forward_serving(x)
    _check(y, ref, max(NET_FLOOR, NET_NOISE_FACTOR * noise), f"forward_serving 576 B2 tf32x3 vs float64 port (port fp32 {noise:.2e})")


def _expected_cbam_launches(model, S_):
    """The CBAM launches SmaAt_UNet._serving makes at plane S_ (modules.CBAM.forward / serving_gates): levels 1-3 with an
    eval BatchNorm compute sa alone (cbam_gate); the others run cbam_gate_scale where W % 4 == 0, else cbam_gate +
    cbam_scale.  The gated blocks all take the fused conv here, so no cbam_scale materialises a gated skip."""
    gate, scale, gate_scale = 0, 0, Counter()
    for lvl in range(5):
        cbam = getattr(model, f"cbam{lvl + 1}")
        C, Sl, bn = cbam.channel_att.MLP[1].in_features, S_ >> lvl, cbam.spatial_att.bn
        if lvl < 3 and not bn.training and bn.track_running_stats:
            gate += 1
        elif Sl % 4 == 0:
            gate_scale[f"smaat_cbam_gate_scale_fwd[C{C}_S{Sl}]"] += 1
        else:
            gate, scale = gate + 1, scale + 1
    return gate, scale, gate_scale


@gpu
def test_serving_cbam_launch_inventory_at_576(ds_impl):
    m = _model()
    x = _frames(2, 576, 3)
    ops.set_pointwise_mode("tf32x3")
    gate, scale, gate_scale = _expected_cbam_launches(m, 576)
    assert (gate, scale, dict(gate_scale)) == (3, 0, {"smaat_cbam_gate_scale_fwd[C512_S72]": 1, "smaat_cbam_gate_scale_fwd[C512_S36]": 1})
    with torch.no_grad():
        m.forward_serving(x)                      # caches built outside the profile
        torch.cuda.synchronize()
        with ops.profile() as prof:
            m.forward_serving(x)
        names = [r[0] for r in prof.records]
    assert sum(n.split("[")[0] == "smaat_cbam_gate_fwd" for n in names) == gate, names
    assert sum(n.split("[")[0] == "smaat_cbam_scale_fwd" for n in names) == scale, names
    assert Counter(n for n in names if n.startswith("smaat_cbam_gate_scale_fwd")) == gate_scale, names
