"""Each backward kernel of the SmaAt-UNet training step against float64 torch autograd of the plain operation, at the
shapes SmaAt-UNet(12, 1, kernels_per_layer=2) runs at 288x288 and at the edges where the kernels switch variants.

The whole-network gradient tests run on small frames (32x32, 48x48) or under a noise-calibrated bound at 288x288; neither
reaches the large-plane vector paths nor would notice a small slip in one kernel.  Here every entry point is called
directly (through ``functional`` / ``ops`` or the C ABI) and compared with a float64 reference computed on the GPU:

  A  smaat_pw1x1_bwd_weight_tc (tf32, tf32x3) and smaat_pw1x1_bwd_weight (CUDA cores), with the bias gradient
  B  functional.pw_bwd's input gradient (smaat_transpose + the forward GEMM with K and Cout swapped), smaat_transpose
  C  smaat_channel_stats, smaat_bn_finalize, smaat_bn_act_bwd_reduce -> smaat_bn_bwd_coeffs -> smaat_bn_act_bwd_apply
  D  the CBAM chain: smaat_cbam_bwd_gate_in, BatchNorm(1) backward, smaat_cbam_gate_bwd, smaat_cbam_bwd_dsc,
     smaat_cbam_mlp_bwd, smaat_cbam_bwd_dx
  E  smaat_maxpool2_bwd, smaat_upsample2x_pad_bwd, smaat_outconv_bwd, smaat_pixel_shuffle2_pad_bwd,
     smaat_convt2x2_unpack_wgrad

Conventions:
  * accumulating outputs (dW, db, dgamma, dbeta, dz_sum, dsc, the MLP and gate-conv gradients) start from a non-zero
    buffer and are checked as init + gradient;
  * where an entry point has a 128-bit and a scalar variant, both run on the same data; the scalar one is forced with a
    copy that starts one float past a 16-byte boundary (``_offset``) or with P % 4 != 0.  Element-wise outputs must then
    be bit-equal, selections (argmax routing) identical, reductions within the bound of the reference;
  * the CBAM reference decides its max routing on the fp32 values the kernels see (first index on ties) and applies it
    in float64 with ``gather``, so that near-ties cannot flip between the two;
  * errors are max |got - ref| / max |ref|, as tests/_util.assert_close measures them.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x
above it (selections, copies and the argmax routing are bit-exact and were):

  quantity                                                   worst observed        bound
  A  pointwise dW, CUDA cores (fp32)                         1.1e-6                1e-5
     pointwise dW, tensor cores tf32x3                       3.3e-5                1e-4
     pointwise dW, tensor cores tf32                         7.6e-4                PW_TOL["tf32"] = 4e-3
     bias gradients (pointwise, OutConv, transposed conv)    7.4e-7                5e-6
  B  pointwise input gradient fp32 / tf32x3 / tf32           1.2e-6 / 6.0e-6 / 8.9e-4   1e-5 / 3e-5 / 4e-3
  C  channel_stats, bn_finalize, backward sums               5.3e-7                4e-6
     dz train / eval                                         5.2e-7 / 0            5e-6 / 0
     dgamma, dbeta, dz_sum                                   5.9e-7                5e-6
     offset-heavy channels, kernel / torch fp32 error        2.3x (dgamma)         10x
  D  CBAM dx                                                 6.4e-7                5e-6
     dpre, draw, dpooled, dsc, davg, dmx                     8.1e-7                5e-6
     MLP, gate conv and BatchNorm(1) parameter gradients     3.3e-6                3e-5
  E  upsample adjoint, kernel / torch fp32 error             1.7x (1.15e-5)        3x + 1e-6
     OutConv dx / dW                                         1.1e-7 / 2.6e-7       1e-6 / 1e-5
     transposed conv dW (through the CUDA-core wgrad)        2.6e-7                1e-5

The tf32x3 weight gradient sits ~30x above the CUDA-core one: each CTA accumulates ~1200 k-steps of three MMAs in the
tensor core's fp32 accumulator before the atomics merge the splits.  The upsample adjoint's error is the fp32 rounding
of the forward's source coordinates, which torch's fp32 upsample shares.  The whole file runs in ~10 s on one H100 at a
peak of 6.5 GiB.
"""
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200 import functional as Fn
from tests._util import PW_TOL

pytestmark = pytest.mark.gpu

# max |got - ref| / max |ref| bounds per quantity (see the module docstring for the observed figures)
ERR_BOUND = {
    "wgrad_fp32": 1e-5,   # pointwise / OutConv / transposed-conv weight gradients on the CUDA cores (fp32 atomics)
    "wgrad_x3": 1e-4,     # pointwise weight gradient on the tensor cores in 3xTF32
    "bias": 5e-6,         # bias gradients (fp32 channel sums)
    "pw_input": {"fp32": 1e-5, "tf32x3": PW_TOL["tf32x3"], "tf32": PW_TOL["tf32"]},
    "bn_stats": 4e-6,     # channel_stats, bn_finalize, the backward's per-channel sums (fp64 merged)
    "bn_dz": 5e-6,        # train-mode dz (batch-statistics terms from the fp64 sums)
    "bn_dz_eval": 0.0,    # eval: dz = 2 dA exactly for the affine used here
    "bn_param": 5e-6,     # dgamma / dbeta / dz_sum
    "cbam_dx": 5e-6,
    "cbam_inner": 5e-6,   # dpre, draw, dpooled, dsc, davg / dmx
    "cbam_param": 3e-5,   # MLP, gate conv and BatchNorm(1) parameter gradients
    "outconv_dx": 1e-6,
}
OFFSET_BN_FACTOR = 10.0   # offset-heavy BatchNorm: kernel error <= this x torch fp32's own error (+ a small floor)
UPSAMPLE_FACTOR = 3.0     # upsample adjoint: error <= this x torch fp32's own error + 1e-6 (both use fp32 source coordinates)


def _abi(name, *args):
    _lib.check(getattr(_lib.load(), name)(*args), name)


def _rc(name, *args):
    return getattr(_lib.load(), name)(*args)


def _p(t):
    return None if t is None else t.data_ptr()


def _st():
    return ops._stream()


def _rel(got, ref):
    got, ref = got.double(), ref.double()
    assert got.shape == ref.shape, (got.shape, ref.shape)
    return (got - ref).abs().max().item() / max(ref.abs().max().item(), 1e-30)


def _check(got, ref, tol, what):
    e = _rel(got, ref)
    print(f"ERR {what}: {e:.3e} (bound {tol:.1e})")
    assert e == e and e <= tol, f"{what}: max rel err {e:.3e} > {tol:.1e}"
    return e


def _offset(t):
    """A copy of ``t`` whose data starts one element past a 16-byte boundary: kernels that need 128-bit access take their
    scalar variant on it."""
    buf = torch.empty(t.numel() + 4, device=t.device, dtype=t.dtype)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 != 0
    return v


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(shape, g, scale=1.0, shift=0.0):
    return torch.randn(shape, generator=g, device="cuda") * scale + shift


def _first_argmax(v, dim):
    """Index of the first maximum along ``dim`` (keepdim), by an explicit rule: torch's CUDA max does not specify ties."""
    n = v.shape[dim]
    shape = [1] * v.dim()
    shape[dim] = n
    ar = torch.arange(n, device=v.device).view(shape)
    return torch.where(v == v.amax(dim=dim, keepdim=True), ar, n).amin(dim=dim, keepdim=True)


def _batch(H):
    return 32 if H <= 72 else 4


# =====================================================================================================================
# A / B: pointwise 1x1 backward
# =====================================================================================================================
# (K, Cout, H): the pointwise layers (K = kernels_per_layer * Cin) of SmaAt-UNet(12, 1, k=2) at 288x288, encoder then decoder
PW_LAYERS = [(24, 64, 288), (128, 64, 288), (128, 128, 144), (256, 128, 144), (256, 256, 72), (512, 256, 72), (512, 512, 36),
             (1024, 512, 36), (1024, 512, 18), (2048, 512, 36), (1024, 256, 36), (1024, 256, 72), (512, 128, 72),
             (512, 128, 144), (256, 64, 144), (256, 64, 288)]
# (B, K, Cout, H, W) edges: K / Cout not tile multiples (both sides of the Cout <= 64 < K operand swap, N_TILE 64 and 128),
# P % 32 != 0, a single 32-pixel chunk in total
PW_EDGES = [(3, 24, 40, 20, 20), (2, 136, 24, 12, 12), (2, 40, 136, 12, 12), (5, 136, 136, 9, 12), (1, 64, 64, 4, 4),
            (1, 8, 8, 4, 4), (2, 72, 8, 6, 6)]


def _pw_data(B, K, Cout, H, W, seed):
    g = _gen(seed)
    dz = _randn((B, Cout, H, W), g, 1.0, 0.25)
    d = _randn((B, K, H, W), g, 1.0, 0.5)
    return dz, d


def _pw_wgrad_ref(dz, d):
    dz64, d64 = dz.double().flatten(2), d.double().flatten(2)
    return torch.einsum("bop,bcp->oc", dz64, d64), dz64.sum(dim=(0, 2))


def _run_pw_wgrad(dz, d, mode, seed, ref_w, ref_b, tol, what):
    B, Cout, H, W = dz.shape
    K = d.shape[1]
    g = _gen(seed + 7)
    dW0 = _randn((Cout, K), g, 0.3 * ref_w.abs().max().item())
    db0 = _randn((Cout,), g, 0.3 * ref_b.abs().max().item() + 1.0)
    dW, db = dW0.clone(), db0.clone()
    if mode == "fp32":
        _abi("smaat_pw1x1_bwd_weight", _p(dz), _p(d), _p(dW), _p(db), B, K, Cout, H * W, _st())
    else:
        _abi("smaat_pw1x1_bwd_weight_tc", _p(dz), _p(d), _p(dW), _p(db), B, K, Cout, H * W, ops.PW_MODES[mode], _st())
    _check(dW, dW0.double() + ref_w, tol, f"{what} dW")
    _check(db, db0.double() + ref_b, ERR_BOUND["bias"], f"{what} db")


@pytest.mark.parametrize("layer", PW_LAYERS, ids=lambda l: f"K{l[0]}_N{l[1]}_S{l[2]}")
def test_pw_weight_gradient_at_network_shapes(layer):
    """dW += dz . d^T, db += sum dz over B*H*W pixels: tensor cores in tf32x3 and tf32, CUDA cores in fp32.  B = 4 at 144 and
    288 reaches the production split count (2 x SMs / tiles), B = 32 below."""
    K, Cout, H = layer
    B = _batch(H)
    seed = K * 7 + Cout * 3 + H
    dz, d = _pw_data(B, K, Cout, H, H, seed)
    ref_w, ref_b = _pw_wgrad_ref(dz, d)
    for mode in ("tf32x3", "fp32", "tf32"):
        tol = {"tf32": PW_TOL["tf32"], "tf32x3": ERR_BOUND["wgrad_x3"], "fp32": ERR_BOUND["wgrad_fp32"]}[mode]
        _run_pw_wgrad(dz, d, mode, seed, ref_w, ref_b, tol, f"pw wgrad {mode} K{K} N{Cout} S{H}")


@pytest.mark.parametrize("case", PW_EDGES, ids=lambda c: "B{}_K{}_N{}_{}x{}".format(*c))
def test_pw_weight_gradient_edges(case):
    B, K, Cout, H, W = case
    seed = B + K * 11 + Cout * 5 + H * W
    dz, d = _pw_data(B, K, Cout, H, W, seed)
    ref_w, ref_b = _pw_wgrad_ref(dz, d)
    for mode in ("tf32x3", "fp32", "tf32"):
        tol = {"tf32": PW_TOL["tf32"], "tf32x3": ERR_BOUND["wgrad_x3"], "fp32": ERR_BOUND["wgrad_fp32"]}[mode]
        _run_pw_wgrad(dz, d, mode, seed, ref_w, ref_b, tol, f"pw wgrad {mode} {case}")


def test_pw_weight_gradient_tc_rejects_what_tma_cannot_describe():
    """P % 4 != 0 or a misaligned operand: the tensor-core entry point returns SMAAT_E_UNSUPPORTED and leaves dW alone; the
    CUDA-core kernel takes the same data."""
    for (B, K, Cout, H, W), misalign in (((2, 64, 64, 5, 5), False), ((3, 40, 24, 7, 9), False), ((2, 64, 64, 8, 8), True)):
        dz, d = _pw_data(B, K, Cout, H, W, 99 + H)
        if misalign:
            dz = _offset(dz)
        ref_w, ref_b = _pw_wgrad_ref(dz, d)
        dW = torch.ones(Cout, K, device="cuda")
        db = torch.ones(Cout, device="cuda")
        for m in (1, 2):
            assert _rc("smaat_pw1x1_bwd_weight_tc", _p(dz), _p(d), _p(dW), _p(db), B, K, Cout, H * W, m, _st()) == -3
        torch.cuda.synchronize()
        assert bool((dW == 1).all()) and bool((db == 1).all())
        _run_pw_wgrad(dz, d, "fp32", 5, ref_w, ref_b, ERR_BOUND["wgrad_fp32"], f"pw wgrad fp32 fallback {(B, K, Cout, H, W)}")


@pytest.mark.parametrize("layer", PW_LAYERS, ids=lambda l: f"K{l[0]}_N{l[1]}_S{l[2]}")
@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "fp32"])
def test_pw_input_gradient_at_network_shapes(layer, mode):
    """functional.pw_bwd: dd = W^T dz, i.e. smaat_transpose then the forward GEMM with K and Cout swapped (Cout up to 2048,
    K down to 64 there)."""
    K, Cout, H = layer
    B = _batch(H)
    seed = K + Cout * 13 + H * 3
    dz, d = _pw_data(B, K, Cout, H, H, seed)
    w = _randn((Cout, K, 1, 1), _gen(seed + 1), K ** -0.5)
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    try:
        dd = Fn.pw_bwd(dz, d, w, torch.zeros(Cout, K, device="cuda"), None)
    finally:
        ops.set_pointwise_mode(old)
    ref = torch.einsum("oc,bop->bcp", w.double().view(Cout, K), dz.double().flatten(2)).view(B, K, H, H)
    _check(dd, ref, ERR_BOUND["pw_input"][mode], f"pw input grad {mode} K{K} N{Cout} S{H}")


@pytest.mark.parametrize("rows, cols", [(1, 1), (1, 70), (33, 65), (100, 37), (24, 136), (512, 2048), (2048, 512)])
def test_transpose_is_exact(rows, cols):
    src = _randn((rows, cols), _gen(rows * 3 + cols))
    dst = torch.full((cols, rows), float("nan"), device="cuda")
    _abi("smaat_transpose", _p(src), _p(dst), rows, cols, _st())
    assert torch.equal(dst, src.t().contiguous())


# =====================================================================================================================
# C: BatchNorm(+ReLU) statistics and backward
# =====================================================================================================================
# (B, C, H, W, mode, act).  mode: train (batch statistics), eval (running statistics, exactly representable affine with
# planted zero pre-activations), offset (train, channel means 1e2..1e3 standard deviations away from 0)
BN_CASES = [(32, 1, 288, 288, "train", 0), (32, 1, 288, 288, "eval", 0), (4, 64, 288, 288, "train", 1),
            (4, 64, 288, 288, "eval", 1), (16, 128, 36, 36, "train", 0), (8, 24, 17, 19, "train", 1), (8, 24, 17, 19, "eval", 1),
            (8, 16, 64, 64, "offset", 1), (8, 16, 64, 64, "offset", 0)]
BN_EPS, BN_MOM = 1e-5, 0.1


def _bn_data(B, C, H, W, mode, act, g):
    if mode == "eval":
        # pre-activation 2 z - 1 with z on a 1/8 grid around 0.5: exact in fp32 and fp64, about 1 in 16 exactly 0
        z = torch.round(_randn((B, C, H, W), g, 8.0, 4.0)) / 8.0
        return z
    m = _randn((1, C, 1, 1), g, 3.0)
    s = torch.rand((1, C, 1, 1), generator=g, device="cuda") + 0.5
    if mode == "offset":
        ratio = 10.0 ** (2.0 + torch.rand((1, C, 1, 1), generator=g, device="cuda"))      # |mean| / std in 1e2..1e3
        sign = torch.where(torch.arange(C, device="cuda").view(1, C, 1, 1) % 2 == 0, 1.0, -1.0)
        m = sign * ratio * s
    v = _randn((B, C, H, W), g)
    if act:   # keep every value 0.1 std away from the batch mean: the ReLU threshold (beta = 0) then never flips with rounding
        v = torch.sign(v) * (v.abs() + 0.1)
        v[:, :, 0, 0] = 0.1          # no sign(0)
        v[:, :, 0, 1] = -0.1
    return m + s * v


@pytest.mark.parametrize("case", BN_CASES, ids=lambda c: "B{}_C{}_{}x{}_{}_act{}".format(*c))
def test_batchnorm_statistics_and_backward(case):
    B, C, H, W, mode, act = case
    P, n = H * W, B * H * W
    g = _gen(B * 1000 + C * 10 + H + act + len(mode))
    z = _bn_data(B, C, H, W, mode, act, g)
    dy = _randn((B, C, H, W), g)
    train = mode != "eval"
    gamma = torch.rand(C, generator=g, device="cuda") + 0.5
    beta = torch.zeros(C, device="cuda") if act else _randn((C,), g, 0.3)
    rm0, rv0 = _randn((C,), g, 0.5), torch.rand(C, generator=g, device="cuda") + 0.5
    what = f"bn {case}"

    # ---- forward statistics (train): channel_stats (+= into a non-zero buffer) and bn_finalize vs torch's BatchNorm2d
    if mode == "offset":
        # the one-pass variance s2/n - mean^2 is not what this case is about: hand the backward exact statistics
        z64 = z.double()
        mu = z64.mean(dim=(0, 2, 3))
        istd = 1.0 / torch.sqrt(z64.var(dim=(0, 2, 3), unbiased=False) + BN_EPS)
        mean, invstd = mu.float(), istd.float()
        scale = (gamma.double() * istd).float()
        shift = (beta.double() - mu * gamma.double() * istd).float()
    elif train:
        z64 = z.double()
        s_ref = torch.cat([z64.sum(dim=(0, 2, 3)), (z64 * z64).sum(dim=(0, 2, 3))])
        s0 = torch.randn(2 * C, device="cuda", dtype=torch.float64)
        stats = s0.clone()
        _abi("smaat_channel_stats", _p(z), _p(stats), B, C, P, _st())
        _check(stats - s0, s_ref, ERR_BOUND["bn_stats"], f"{what} channel_stats")
        stats = torch.zeros(2 * C, device="cuda", dtype=torch.float64)
        _abi("smaat_channel_stats", _p(z), _p(stats), B, C, P, _st())
        rm, rv = rm0.clone(), rv0.clone()
        nbt = torch.full((), 7, device="cuda", dtype=torch.int64)
        scale, shift, mean, invstd = (torch.empty(C, device="cuda") for _ in range(4))
        _abi("smaat_bn_finalize", _p(stats), float(n), _p(gamma), _p(beta), BN_EPS, BN_MOM, _p(rm), _p(rv), _p(scale), _p(shift),
             _p(mean), _p(invstd), _p(nbt), C, _st())
        bn = torch.nn.BatchNorm2d(C, eps=BN_EPS, momentum=BN_MOM).cuda().double().train()
        with torch.no_grad():
            bn.running_mean.copy_(rm0)
            bn.running_var.copy_(rv0)
            bn.num_batches_tracked.fill_(7)
            bn(z64)
        mu = z64.mean(dim=(0, 2, 3))
        istd = 1.0 / torch.sqrt(z64.var(dim=(0, 2, 3), unbiased=False) + BN_EPS)
        _check(mean, mu, ERR_BOUND["bn_stats"], f"{what} mean")
        _check(invstd, istd, ERR_BOUND["bn_stats"], f"{what} invstd")
        _check(rm, bn.running_mean, ERR_BOUND["bn_stats"], f"{what} running_mean")
        _check(rv, bn.running_var, ERR_BOUND["bn_stats"], f"{what} running_var")
        assert int(nbt) == int(bn.num_batches_tracked) == 8
        _check(scale, gamma.double() * istd, ERR_BOUND["bn_stats"], f"{what} scale")
        _check(shift, beta.double() - mu * gamma.double() * istd, ERR_BOUND["bn_stats"], f"{what} shift")
    else:
        # affine 2 z - 1 exactly: mean 0.25, invstd 0.5, gamma 4, beta -0.5
        mean = torch.full((C,), 0.25, device="cuda")
        invstd = torch.full((C,), 0.5, device="cuda")
        gamma = torch.full((C,), 4.0, device="cuda")
        beta = torch.full((C,), -0.5, device="cuda")
        scale, shift = torch.full((C,), 2.0, device="cuda"), torch.full((C,), -1.0, device="cuda")
        assert bool(((2 * z - 1) == 0).any())

    # ---- float64 reference: F.batch_norm (+ReLU) autograd
    zr = z.double().requires_grad_(True)
    gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    if train:
        y = F.batch_norm(zr, None, None, gr, br, training=True, eps=BN_EPS)
    else:   # BatchNorm2d.eval written out with the saved mean / inv-std: exact for this affine, so zeros stay exact zeros
        y = (zr - mean.double()[:, None, None]) * invstd.double()[:, None, None] * gr[:, None, None] + br[:, None, None]
    if act:
        y = torch.relu(y)
    y.backward(dy.double())

    # ---- kernels: reduce -> coeffs -> apply, accumulating into non-zero dgamma / dbeta / dz_sum
    g0 = [_randn((C,), g) for _ in range(3)]
    dgamma, dbeta, dz_sum = (t.clone() for t in g0)
    sums = torch.zeros(2 * C, device="cuda", dtype=torch.float64)
    _abi("smaat_bn_act_bwd_reduce", _p(dy), _p(z), _p(scale), _p(shift), _p(sums), B, C, P, act, _st())
    a, b, cc = (torch.empty(C, device="cuda") for _ in range(3))
    _abi("smaat_bn_bwd_coeffs", _p(sums), float(n), _p(gamma), _p(mean), _p(invstd), int(train), _p(a), _p(b), _p(cc), _p(dgamma),
         _p(dbeta), _p(dz_sum), C, _st())
    dz = torch.empty_like(z)
    _abi("smaat_bn_act_bwd_apply", _p(dy), _p(z), _p(scale), _p(shift), _p(a), _p(b), _p(cc), _p(dz), B, C, P, act, _st())

    if mode == "offset":
        # calibrate against torch's own fp32 BatchNorm on the same data
        zf = z.clone().requires_grad_(True)
        gf, bf = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
        yf = F.batch_norm(zf, None, None, gf, bf, training=True, eps=BN_EPS)
        (torch.relu(yf) if act else yf).backward(dy)
        for got, tf, ref, nm in ((dz, zf.grad, zr.grad, "dz"), (dgamma - g0[0], gf.grad, gr.grad, "dgamma"),
                                 (dbeta - g0[1], bf.grad, br.grad, "dbeta")):
            noise = _rel(tf, ref)
            _check(got, ref, max(OFFSET_BN_FACTOR * noise, 1e-6), f"{what} {nm} (torch fp32 {noise:.2e})")
    else:
        _check(dz, zr.grad, ERR_BOUND["bn_dz"] if train else ERR_BOUND["bn_dz_eval"], f"{what} dz")
        _check(dgamma, g0[0].double() + gr.grad, ERR_BOUND["bn_param"], f"{what} dgamma")
        _check(dbeta, g0[1].double() + br.grad, ERR_BOUND["bn_param"], f"{what} dbeta")
    if train:       # with batch statistics sum dz is identically 0: the kernel leaves dz_sum untouched
        assert torch.equal(dz_sum, g0[2])
    else:
        _check(dz_sum, g0[2].double() + zr.grad.sum(dim=(0, 2, 3)), ERR_BOUND["bn_param"], f"{what} dz_sum")
    if act and not train:   # planted zero pre-activations get exactly zero gradient, like torch's relu
        assert bool((dz[(2 * z - 1) == 0] == 0).all())

    # ---- the reduce's sums against float64 (the mask is exact here: eval affine exact, train data off the threshold), and
    # the scalar variants on the same data: apply bit-equal with the same coefficients, reduce within the bound
    z64, dA = z.double(), dy.double()
    if act:
        dA = dA * ((z64 * scale.double()[:, None, None] + shift.double()[:, None, None]) > 0)
    s1_ref, s2_ref = dA.sum(dim=(0, 2, 3)), (dA * z64).sum(dim=(0, 2, 3))
    _check(sums[:C], s1_ref, ERR_BOUND["bn_stats"], f"{what} reduce S1")
    _check(sums[C:], s2_ref, ERR_BOUND["bn_stats"], f"{what} reduce S2")
    if P % 4 == 0:
        dz_s = _offset(torch.empty_like(z))
        dy_s, z_s = _offset(dy), _offset(z)
        _abi("smaat_bn_act_bwd_apply", _p(dy_s), _p(z_s), _p(scale), _p(shift), _p(a), _p(b), _p(cc), _p(dz_s), B, C, P, act, _st())
        assert torch.equal(dz_s, dz)
        sums_s = torch.zeros_like(sums)
        _abi("smaat_bn_act_bwd_reduce", _p(dy_s), _p(z_s), _p(scale), _p(shift), _p(sums_s), B, C, P, act, _st())
        _check(sums_s[:C], s1_ref, ERR_BOUND["bn_stats"], f"{what} reduce S1 scalar")
        _check(sums_s[C:], s2_ref, ERR_BOUND["bn_stats"], f"{what} reduce S2 scalar")


# =====================================================================================================================
# D: CBAM backward chain
# =====================================================================================================================
# (B, C, H, W, hidden, ks, kind)
CBAM_CASES = [
    (8, 64, 288, 288, 4, 7, "relu"),     # gate_in 128-bit path; gate weight gradient loops (B x 81 tiles = 648 > 2 x SMs)
    (4, 128, 144, 144, 8, 7, "relu"),
    (32, 256, 72, 72, 16, 7, "relu"),    # P < 8192: gate_in scalar path; dsc / dx grid.y = 2
    (32, 512, 36, 36, 32, 7, "relu"),
    (32, 512, 18, 18, 32, 7, "relu"),
    (4, 12, 40, 40, 3, 3, "relu"),       # C % 8 != 0, ks 3
    (4, 64, 96, 96, 4, 3, "negative"),   # negative inputs (the plane argmax keys of negative floats), gate_in 128-bit
    (3, 24, 37, 29, 2, 7, "relu"),       # P % 4 != 0: scalar kernels only
]


def _cbam_input(B, C, H, W, kind, g):
    if kind == "negative":
        x = _randn((B, C, H, W), g, 0.7, -1.0)
    else:
        x = torch.relu(_randn((B, C, H, W), g))          # about half exact zeros
    x[0, :, 1, 2] = 0.0                                     # dead pixels: every channel 0 (channel ties at u = 0)
    x[B - 1, :, H - 1, W - 1] = 0.0
    x[0, min(3, C - 1)] = 0.0                               # dead plane: its maximum sits at every pixel
    c = 1 % C                                               # a plane maximum at two positions
    m = x[B - 1, c].max() + 0.5
    x[B - 1, c, 0, W - 1] = m
    x[B - 1, c, H - 1, 0] = m
    return x


def _cbam_module(C, hidden, ks, g):
    mod = S.CBAM(C, reduction_ratio=C // hidden, kernel_size=ks).cuda().train()
    assert mod.channel_att.MLP[1].weight.shape == (hidden, C)
    with torch.no_grad():
        l1, l2, sp = mod.channel_att.MLP[1], mod.channel_att.MLP[3], mod.spatial_att
        l1.weight.copy_(_randn(l1.weight.shape, g, C ** -0.5))
        l1.bias.copy_(_randn(l1.bias.shape, g, 0.1, 0.2))
        l2.weight.copy_(_randn(l2.weight.shape, g, hidden ** -0.5))
        l2.bias.copy_(_randn(l2.bias.shape, g, 0.1))
        sp.conv.weight.copy_(_randn(sp.conv.weight.shape, g, 0.3 / ks))
        sp.bn.weight.fill_(1.3)
        sp.bn.bias.fill_(-0.2)
    return mod


def _cbam_reference(mod, x, sc32, gout):
    """float64 autograd of CBAM (reference models/layers.py:105-141) with the max routing fixed from the fp32 values: the
    plane argmax of x and the channel argmax of x * sc32, first index on ties."""
    B, C, H, W = x.shape
    l1, l2, sp = mod.channel_att.MLP[1], mod.channel_att.MLP[3], mod.spatial_att
    params = [t.detach().double().requires_grad_(True) for t in (l1.weight, l1.bias, l2.weight, l2.bias, sp.conv.weight, sp.bn.weight,
                                                                 sp.bn.bias)]
    w1, b1, w2, b2, wc, gam, bet = params
    pidx = _first_argmax(x.view(B, C, -1), 2)
    cidx = _first_argmax(x * sc32[:, :, None, None], 1)
    xr = x.double().requires_grad_(True)
    avg = xr.mean(dim=(2, 3))
    mx = xr.view(B, C, -1).gather(2, pidx).squeeze(2)

    def mlp(v):
        return F.linear(F.relu(F.linear(v, w1, b1)), w2, b2)

    sc = torch.sigmoid(mlp(avg) + mlp(mx))
    u = xr * sc[:, :, None, None]
    pooled = torch.cat([u.mean(dim=1, keepdim=True), u.gather(1, cidx)], dim=1)
    raw = F.conv2d(pooled, wc, None, padding=wc.shape[-1] // 2)
    pre = F.batch_norm(raw, None, None, gam, bet, training=True, eps=sp.bn.eps)
    out = u * torch.sigmoid(pre)
    for t in (avg, mx, sc, pooled, raw, pre):
        t.retain_grad()
    out.backward(gout.double())
    inner = dict(davg=avg.grad, dmx=mx.grad, dsc=sc.grad, dpooled=pooled.grad, draw=raw.grad, dpre=pre.grad)
    return xr.grad, [p.grad for p in params], inner, pidx.view(B, C), cidx.view(B, H * W)


@pytest.mark.parametrize("case", CBAM_CASES, ids=lambda c: "B{}_C{}_{}x{}_h{}_k{}_{}".format(*c))
def test_cbam_backward_chain(case):
    B, C, H, W, hidden, ks, kind = case
    P = H * W
    g = _gen(B * 7 + C * 31 + H * 3 + W + ks)
    mod = _cbam_module(C, hidden, ks, g)
    x = _cbam_input(B, C, H, W, kind, g)
    gout = _randn((B, C, H, W), g)
    out, saved = Fn.cbam_fwd(mod, x)
    sc32 = saved["sc"]
    ref_dx, ref_params, inner, pidx, cidx = _cbam_reference(mod, x, sc32, gout)
    what = f"cbam {case}"

    # ---- functional.cbam_bwd, parameter gradients accumulated into non-zero buffers (the gradient-bucket sinks)
    l1, l2, sp = mod.channel_att.MLP[1], mod.channel_att.MLP[3], mod.spatial_att
    params = [l1.weight, l1.bias, l2.weight, l2.bias, sp.conv.weight, sp.bn.weight, sp.bn.bias]
    init = [_randn(p.shape, g, r.abs().max().item() * 0.3 + 1e-3) for p, r in zip(params, ref_params)]
    views = [t.clone() for t in init]
    keys = Fn.add_grad_sinks(params, views)
    try:
        dx, grads = Fn.cbam_bwd(mod, saved, gout)
    finally:
        Fn.remove_grad_sinks(keys)
    _check(dx, ref_dx, ERR_BOUND["cbam_dx"], f"{what} dx")
    names = ["mlp.w1", "mlp.b1", "mlp.w2", "mlp.b2", "gate conv", "bn.weight", "bn.bias"]
    for got, view, i0, r, nm in zip(grads, views, init, ref_params, names):
        assert got is view
        _check(view, i0.double() + r, ERR_BOUND["cbam_param"], f"{what} d{nm}")

    # ---- the chain one entry point at a time; both variants of each |x|-sized pass on the same data
    st = _st()
    sa = saved["sa"]
    dpre = torch.empty((B, 1, H, W), device="cuda")
    amax = torch.full((B, H, W), -1, device="cuda", dtype=torch.int32)
    _abi("smaat_cbam_bwd_gate_in", _p(gout), _p(x), _p(sc32), _p(sa), _p(dpre), _p(amax), B, C, P, st)
    assert torch.equal(amax.view(B, P).long(), cidx), "channel argmax routing"
    _check(dpre, inner["dpre"], ERR_BOUND["cbam_inner"], f"{what} dpre")
    dpre_s = _offset(torch.empty_like(dpre))
    amax_s = torch.full_like(amax, -1)
    g_s, x_s = _offset(gout), _offset(x)          # kept alive: the kernels are only enqueued
    _abi("smaat_cbam_bwd_gate_in", _p(g_s), _p(x_s), _p(sc32), _p(sa), _p(dpre_s), _p(amax_s), B, C, P, st)
    assert torch.equal(amax_s, amax)
    _check(dpre_s, inner["dpre"], ERR_BOUND["cbam_inner"], f"{what} dpre scalar")

    bn = sp.bn
    dg, dbt = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    draw = Fn.bn_act_bwd(dpre, saved["raw"], saved["g_sc"], saved["g_sh"], bn.weight.detach(), saved["g_m"], saved["g_i"], B * P, True, 0,
                         dg, dbt)
    _check(draw, inner["draw"], ERR_BOUND["cbam_inner"], f"{what} draw")
    dpooled = torch.empty((B, 2, H, W), device="cuda")
    dWc0 = _randn(sp.conv.weight.shape, g)
    dWc = dWc0.clone()
    _abi("smaat_cbam_gate_bwd", _p(draw), _p(saved["pooled"]), _p(sp.conv.weight.detach()), _p(dpooled), _p(dWc), B, H, W, ks, st)
    _check(dpooled, inner["dpooled"], ERR_BOUND["cbam_inner"], f"{what} dpooled")
    _check(dWc, dWc0.double() + ref_params[4], ERR_BOUND["cbam_param"], f"{what} gate conv dW (direct)")

    dsc0 = _randn((B, C), g, inner["dsc"].abs().max().item() * 0.3)
    dsc, dsc_s = dsc0.clone(), dsc0.clone()
    pkey = torch.zeros((B, C), device="cuda", dtype=torch.int64)
    pkey_s = torch.zeros_like(pkey)
    _abi("smaat_cbam_bwd_dsc", _p(gout), _p(x), _p(sa), _p(dpooled), _p(amax), _p(dsc), _p(pkey), B, C, P, st)
    _abi("smaat_cbam_bwd_dsc", _p(g_s), _p(x_s), _p(sa), _p(dpooled), _p(amax), _p(dsc_s), _p(pkey_s), B, C, P, st)
    assert torch.equal(pkey_s, pkey)
    assert torch.equal(0xFFFFFFFF - (pkey & 0xFFFFFFFF), pidx), "plane argmax routing"
    _check(dsc, dsc0.double() + inner["dsc"], ERR_BOUND["cbam_inner"], f"{what} dsc")
    _check(dsc_s, dsc0.double() + inner["dsc"], ERR_BOUND["cbam_inner"], f"{what} dsc scalar")

    # MLP backward from the kernels' own dsc (dsc - dsc0 is exact enough at this scale: both are fp32 of similar size)
    dsc_k = torch.zeros((B, C), device="cuda")
    pk = torch.zeros_like(pkey)
    _abi("smaat_cbam_bwd_dsc", _p(gout), _p(x), _p(sa), _p(dpooled), _p(amax), _p(dsc_k), _p(pk), B, C, P, st)
    m0 = [_randn(p.shape, g, r.abs().max().item() * 0.3 + 1e-3) for p, r in zip(params[:4], ref_params[:4])]
    mg = [t.clone() for t in m0]
    davg, dmx = torch.empty((B, C), device="cuda"), torch.empty((B, C), device="cuda")
    _abi("smaat_cbam_mlp_bwd", _p(saved["avg"]), _p(saved["mx"]), _p(l1.weight.detach()), _p(l1.bias.detach()), _p(l2.weight.detach()),
         _p(sc32), _p(dsc_k), _p(mg[0]), _p(mg[1]), _p(mg[2]), _p(mg[3]), _p(davg), _p(dmx), B, C, hidden, st)
    for got, i0, r, nm in zip(mg, m0, ref_params[:4], names[:4]):
        _check(got, i0.double() + r, ERR_BOUND["cbam_param"], f"{what} d{nm} (direct)")
    _check(davg, inner["davg"], ERR_BOUND["cbam_inner"], f"{what} davg")
    _check(dmx, inner["dmx"], ERR_BOUND["cbam_inner"], f"{what} dmx")

    dx_v = torch.empty_like(x)
    _abi("smaat_cbam_bwd_dx", _p(gout), _p(sc32), _p(sa), _p(dpooled), _p(amax), _p(davg), _p(dmx), _p(pk), _p(dx_v), B, C, P, st)
    _check(dx_v, ref_dx, ERR_BOUND["cbam_dx"], f"{what} dx (direct)")
    dx_s = _offset(torch.empty_like(x))
    _abi("smaat_cbam_bwd_dx", _p(g_s), _p(sc32), _p(sa), _p(dpooled), _p(amax), _p(davg), _p(dmx), _p(pk), _p(dx_s), B, C, P, st)
    assert torch.equal(dx_s, dx_v)


# =====================================================================================================================
# E: glue backward
# =====================================================================================================================
# (B, C, H, W): the four MaxPool2d(2) inputs of the encoder, then odd edges
MP_CASES = [(32, 512, 36, 36), (32, 256, 72, 72), (8, 128, 144, 144), (2, 64, 288, 288), (3, 4, 7, 9), (2, 3, 5, 4), (1, 2, 2, 3),
            (2, 2, 3, 2)]


@pytest.mark.parametrize("case", MP_CASES, ids=lambda c: "B{}_C{}_{}x{}".format(*c))
def test_maxpool2_backward_routes_to_the_first_maximum(case):
    B, C, H, W = case
    g = _gen(B + C + H * 5 + W)
    x = torch.relu(_randn((B, C, H, W), g))                 # all-zero windows and zero ties
    Ho, Wo = H // 2, W // 2
    x[:, 0, 0:2 * Ho:2, 1:2 * Wo:2] = 2.5                  # channel 0: a positive tie at window positions 1 and 3
    x[:, 0, 1:2 * Ho:2, 1:2 * Wo:2] = 2.5
    dy = _randn((B, C, Ho, Wo), g)
    dx = Fn.maxpool2_bwd(x, dy)
    # reference: explicit first-maximum routing in row-major window order
    win = x[:, :, :2 * Ho, :2 * Wo].reshape(B, C, Ho, 2, Wo, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, Ho, Wo, 4)
    idx = _first_argmax(win, 4)
    dwin = torch.zeros_like(win).scatter_(4, idx, dy[..., None])
    ref = torch.zeros_like(x)
    ref[:, :, :2 * Ho, :2 * Wo] = dwin.view(B, C, Ho, Wo, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, 2 * Ho, 2 * Wo)
    assert torch.equal(dx, ref)
    if x.numel() <= 1 << 16:     # and torch's own CPU max_pool2d backward (the reference's path)
        xc = x.cpu().requires_grad_(True)
        F.max_pool2d(xc, 2).backward(dy.cpu())
        assert torch.equal(dx.cpu(), xc.grad)


# (B, C, H, W, Ho, Wo): the four decoder upsamplings, then odd pads
UP_CASES = [(32, 512, 18, 18, 36, 36), (32, 256, 36, 36, 72, 72), (8, 128, 72, 72, 144, 144), (2, 64, 144, 144, 288, 288),
            (3, 5, 5, 5, 11, 10), (2, 3, 1, 1, 2, 2), (2, 4, 4, 6, 9, 15), (1, 2, 70, 130, 141, 262)]


@pytest.mark.parametrize("case", UP_CASES, ids=lambda c: "B{}_C{}_{}x{}_to_{}x{}".format(*c))
@pytest.mark.parametrize("sliced", [False, True])
def test_upsample2x_pad_backward(case, sliced):
    """Adjoint of nn.Upsample(x2, bilinear, align_corners=True) + F.pad; ``sliced``: dy is a channel slice of a wider tensor
    (the Up block's concat), read through its batch stride."""
    B, C, H, W, Ho, Wo = case
    g = _gen(B + C * 3 + H + Wo)
    if sliced:
        dy = _randn((B, C + 5, Ho, Wo), g)[:, 2:2 + C]
    else:
        dy = _randn((B, C, Ho, Wo), g)
    dx = Fn.upsample2x_pad_bwd(dy, (B, C, H, W))
    xr = torch.zeros((B, C, H, W), device="cuda", dtype=torch.float64, requires_grad=True)
    up = F.interpolate(xr, scale_factor=2, mode="bilinear", align_corners=True)
    dY, dX = Ho - 2 * H, Wo - 2 * W
    F.pad(up, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2]).backward(dy.double())
    # the kernel is the exact adjoint of the fp32 forward, whose source coordinates u * (n - 1) / (2n - 1) are rounded to fp32
    # as torch's fp32 upsample rounds them: against exact coordinates both carry the same error, so calibrate on torch fp32
    xf = torch.zeros((B, C, H, W), device="cuda", requires_grad=True)
    upf = F.interpolate(xf, scale_factor=2, mode="bilinear", align_corners=True)
    F.pad(upf, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2]).backward(dy)
    noise = _rel(xf.grad, xr.grad)
    _check(dx, xr.grad, UPSAMPLE_FACTOR * noise + 1e-6, f"upsample bwd {case} sliced={sliced} (torch fp32 {noise:.2e})")


# (B, Cin, ncls, H, W)
OC_CASES = [(4, 64, 1, 288, 288), (4, 64, 5, 288, 288), (3, 16, 5, 17, 19), (2, 64, 1, 17, 19), (2, 8, 3, 8, 8)]


@pytest.mark.parametrize("case", OC_CASES, ids=lambda c: "B{}_C{}_n{}_{}x{}".format(*c))
def test_outconv_backward(case):
    B, Cin, ncls, H, W = case
    P = H * W
    g = _gen(B + Cin + ncls * 7 + H)
    x = _randn((B, Cin, H, W), g, 1.0, 0.3)
    dy = _randn((B, ncls, H, W), g)
    w = _randn((ncls, Cin), g, Cin ** -0.5)
    x64, dy64 = x.double().flatten(2), dy.double().flatten(2)
    ref_dx = torch.einsum("jc,bjp->bcp", w.double(), dy64).view(B, Cin, H, W)
    ref_dw = torch.einsum("bjp,bcp->jc", dy64, x64)
    ref_db = dy64.sum(dim=(0, 2))
    dW0, db0 = _randn((ncls, Cin), g, ref_dw.abs().max().item() * 0.3), _randn((ncls,), g, ref_db.abs().max().item() * 0.3)
    results = []
    for variant in ("vec", "scalar", "no_dx"):
        dyv, xv = (_offset(dy), _offset(x)) if variant == "scalar" else (dy, x)
        dx = None if variant == "no_dx" else (_offset(torch.empty_like(x)) if variant == "scalar" else torch.empty_like(x))
        dW, db = dW0.clone(), db0.clone()
        _abi("smaat_outconv_bwd", _p(dyv), _p(xv), _p(w), _p(dx), _p(dW), _p(db), B, Cin, ncls, P, _st())
        _check(dW, dW0.double() + ref_dw, ERR_BOUND["wgrad_fp32"], f"outconv {case} {variant} dW")
        _check(db, db0.double() + ref_db, ERR_BOUND["bias"], f"outconv {case} {variant} db")
        if dx is not None:
            _check(dx, ref_dx, ERR_BOUND["outconv_dx"], f"outconv {case} {variant} dx")
            results.append(dx.clone())
    assert torch.equal(results[0], results[1])


# (B, Cin, Cout, H, W, Ho, Wo): UpDS(bilinear=False) transposed conv + pad
CT_CASES = [(4, 1024, 512, 18, 18, 36, 36), (2, 64, 32, 9, 9, 19, 21), (3, 24, 12, 5, 7, 11, 14), (2, 16, 8, 6, 8, 12, 16)]


@pytest.mark.parametrize("case", CT_CASES, ids=lambda c: "B{}_Ci{}_Co{}_{}x{}_to_{}x{}".format(*c))
def test_convt2x2_backward(case):
    """ConvTranspose2d(k=2, s=2) + F.pad backward as the library runs it: pixel_shuffle2_pad_bwd (exact gather), the pointwise
    weight gradient on the packed (4 Cout, Cin) matrix, and convt2x2_unpack_wgrad accumulating into the (Cin, Cout, 2, 2)
    layout; against conv_transpose2d autograd in float64."""
    B, Cin, Cout, H, W, Ho, Wo = case
    g = _gen(B + Cin + Cout * 3 + Ho + Wo)
    x = _randn((B, Cin, H, W), g, 1.0, 0.2)
    wt = _randn((Cin, Cout, 2, 2), g, Cin ** -0.5)
    bias = _randn((Cout,), g, 0.1)
    wide = _randn((B, Cout + 3, Ho, Wo), g)
    gy = wide[:, 1:1 + Cout]                                  # a channel slice of the concat gradient
    dY, dX = Ho - 2 * H, Wo - 2 * W
    # float64 reference
    xr, wr, br = (t.double().requires_grad_(True) for t in (x, wt, bias))
    F.pad(F.conv_transpose2d(xr, wr, br, stride=2), [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2]).backward(gy.double())
    # the pixel-shuffle transpose: exact, against autograd of the forward shuffle
    dt = torch.full((B, 4 * Cout, H, W), float("nan"), device="cuda")
    _abi("smaat_pixel_shuffle2_pad_bwd", _p(gy), gy.stride(0), _p(dt), B, Cout, H, W, Ho, Wo, _st())
    tr = torch.zeros((B, 4 * Cout, H, W), device="cuda", requires_grad=True)
    ys = tr.view(B, 2, 2, Cout, H, W).permute(0, 3, 4, 1, 5, 2).reshape(B, Cout, 2 * H, 2 * W)
    F.pad(ys, [dX // 2, dX - dX // 2, dY // 2, dY - dY // 2]).backward(gy)
    assert torch.equal(dt, tr.grad)
    # packed weight gradient -> unpack into non-zero buffers
    dWp = torch.zeros((4 * Cout, Cin), device="cuda")
    dbp = torch.zeros(4 * Cout, device="cuda")
    _abi("smaat_pw1x1_bwd_weight", _p(dt), _p(x), _p(dWp), _p(dbp), B, Cin, 4 * Cout, H * W, _st())
    dW0, db0 = _randn((Cin, Cout, 2, 2), g, wr.grad.abs().max().item() * 0.3), _randn((Cout,), g, br.grad.abs().max().item() * 0.3)
    dW, db = dW0.clone(), db0.clone()
    _abi("smaat_convt2x2_unpack_wgrad", _p(dWp), _p(dbp), _p(dW), _p(db), Cin, Cout, _st())
    # the unpack itself is data movement plus one add: exact
    assert torch.equal(dW, dW0 + dWp.view(2, 2, Cout, Cin).permute(3, 2, 0, 1))
    assert torch.equal(db, db0 + ((dbp[:Cout] + dbp[Cout:2 * Cout]) + (dbp[2 * Cout:3 * Cout] + dbp[3 * Cout:])))
    _check(dW, dW0.double() + wr.grad, ERR_BOUND["wgrad_fp32"], f"convt {case} dW")
    _check(db, db0.double() + br.grad, ERR_BOUND["bias"], f"convt {case} db")
