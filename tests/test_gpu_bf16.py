"""The bf16 arithmetic mode ('bf16', SMAAT_PW_BF16) on the GPU: the weight pack, every bf16 instance at the 288 x 288
networks' own layer shapes, exact-integer production launches, whole networks, a training step and the caches a captured
session reads.

  A  smaat_pack_bf16 against torch's round-to-nearest-even ``.to(torch.bfloat16)`` followed by the k permutation: random
     values, ties, subnormals, +-inf and NaN, zero padding for cols not a multiple of 32
  B  every bf16 instance against float64 on bf16-rounded operands: the fused DS conv (dsconv_bf16_kernel) at the 12 fused
     layers of SmaAt_UNet(12, 1) at k = 2 (eval epilogue, train epilogue with the BatchNorm sums), at k = 1 and 4 on three
     of them, the one-class OutConv, the K-class class map and the CBAM gate-on-load and pools at up4.1 / up3.0 / inc.1;
     pw1x1 forward at the six layers the fused kernel declines and its input gradient (W^T dz); the dense 3x3 conv forward
     and input gradient at UNet(12, 1)'s layers
  C  exact-integer production launches at B = 32, 288 x 288 (inputs and weights in {-1, 0, 1}, which bf16 holds exactly):
     the fused DS conv at inc.0, up4.0 and up4.1 (+ OutConv), pw1x1 forward and input gradient, the dense 3x3 conv forward
     over the virtual concat and its input gradient; bit-equal to float64
  D  SmaAt_UNet(12, 1) (k = 2, B = 32, 288 x 288), SmaAt_UNet(3, 21) (B = 8, 224 x 224) and UNet(12, 1) (B = 32, 288 x 288)
     through InferenceSession against the float64 port; the session equals the eager serving forward bit for bit, and the
     unfused class map is torch.argmax of the bf16 logits
  E  one SmaAt_UNet(12, 1) TrainSession step (the state and batch of tests/test_gpu_train_tail.py: B = 2, 288 x 288): the
     captured step's gradients equal the eager step's up to the order of the weight-gradient kernels' fp32 atomics (no
     further from an eager step than a second eager step is, times a noise factor), and they are within a noise factor of
     float64 autograd through the port run on the same rounded operands (pointwise forward and input gradient on bf16
     operands, weight gradient on tf32 ones), the factor applied to the port's own fp32-vs-float64 movement, as the
     existing training tests calibrate
  F  a session captured in bf16 keeps returning its captured result after a mode change, train() / eval() and
     load_state_dict(assign=True), until refresh()

Once the operands are rounded the same way, part B's remaining error is fp32 accumulation, as for tf32 (whose analogue in
tests/test_gpu_ds_forward_kernels.py is 3.3e-6); a wrong permutation or pack would show as errors of order 1e-2.

Bounds were set from the worst error observed over this file on an H100 80GB HBM3 (700 W power limit), no more than 10x
above it (everything else is bit-exact and was):

  quantity                                                   worst observed      bound
  B  fused DS conv y / logits (k = 1, 2, 4), OutConv, gate   2.4e-6              1.2e-5
     its BatchNorm sums                                      7.1e-7              3.5e-6
     pw1x1 y, input gradient                                 2.2e-6              1.1e-5
     conv3x3 y, input gradient                               1.1e-5              5.5e-5
  D  SmaAt_UNet(12, 1) logits against the float64 port      8.6e-3              4e-2
     SmaAt_UNet(3, 21) logits / probabilities                2.7e-3 / 4.9e-4     1.3e-2 / 2.5e-3
     UNet(12, 1) logits                                      2.3e-3              1.2e-2
  (SmaAt_UNet(3, 21)'s bf16 class map agreed with the float64 port's argmax at every pixel of the B = 8 batch.)
  E  captured vs eager gradients, rel L2                     9.2e-7-1.6e-5 (eager   5x eager vs eager
                                                             vs eager: up to 1.6e-5)
     whole gradient bucket vs float64, rel L2                0.458 (port on bf16    1.25x the port's
                                                             operands: 0.457)
     the 5 well-conditioned parameters vs float64, rel L2    1.6e-2 (port on bf16   5x the port's (8.4e-2)
                                                             operands: 1.7e-2)

Part B's errors are those of fp32 accumulation over K (the largest, 1.1e-5, is the 9 216-term dense conv of up1), the size
tf32's analogues have: the permuted pack lines up with the fragments.  Part D is what bf16 operands cost a whole network:
the float64 port is the reference model's arithmetic in exact form.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch import nn

import smaat_unet_b200 as S
from oracle import dense_oracle as DO
from oracle import torch_port as TP
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import functional as Fn
from smaat_unet_b200 import ops
from smaat_unet_b200.engine import InferenceSession
from smaat_unet_b200.modules import cached_tensors
from smaat_unet_b200.train import TrainSession
from tests._util import load_np_state_dict
from tests.test_gpu_ds_forward_kernels import (FUSED, LAYERS, UNFUSED, _batch, _bn_affine, _check, _exact, _gen, _int_data, _lid,
                                               _randn, _seed, _split, dw_emul)

pytestmark = pytest.mark.gpu

ERR_BOUND = {
    "fused": 1.2e-5,
    "fused_stats": 3.5e-6,
    "pw": 1.1e-5,
    "conv3x3": 5.5e-5,
    "net_smaat": 4e-2,
    "net_seg_logits": 1.3e-2,
    "net_seg_probs": 2.5e-3,
    "net_unet": 1.2e-2,
}
NOISE_FACTOR = 5.0           # E: bf16 step error <= this x the port's on bf16 operands; captured-vs-eager <= this x eager-vs-eager
WELL_CONDITIONED = 0.02      # E: parameters whose gradient bf16 operands move by at most this (rel L2) in the port
BUCKET_FACTOR = 1.25         # E: the whole bucket's distance from float64 <= this x the port's on bf16 operands


def bf16(t):
    """The value the tensor core multiplies in bf16 mode: round to nearest even."""
    return t.to(torch.bfloat16).float()


def perm16():
    """Physical k of logical k l within a group of 16 (smaat_pack_bf16)."""
    return torch.tensor([(l & 8) | ((l & 1) << 2) | ((l >> 1) & 3) for l in range(16)])


def pack_ref(w):
    rows, cols = w.shape
    cp = (cols + 31) // 32 * 32
    wp = torch.zeros((rows, cp), device=w.device, dtype=torch.bfloat16)
    wp[:, :cols] = w.to(torch.bfloat16)
    idx = (torch.arange(cp) // 16 * 16 + perm16().repeat(cp // 16)).to(w.device)
    return wp[:, idx]


@pytest.fixture
def bf16_mode():
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode("bf16")
    try:
        yield
    finally:
        ops.set_pointwise_mode(old)


# ================================================================================================================ A: the pack
@pytest.mark.parametrize("rows,cols", [(64, 24), (128, 128), (256, 512), (37, 1000), (5, 1)])
def test_pack_is_torch_rounding_then_the_permutation(rows, cols):
    g = _gen(rows * 7 + cols)
    w = _randn((rows, cols), g)
    flat = w.view(-1)
    n = flat.numel()
    special = torch.tensor([0.0, -0.0, float("inf"), float("-inf"), float("nan"), 1e-40, -1e-40, 1e-45, 3e38, -3e38],
                           device="cuda")
    # ties: bf16 keeps 8 significand bits, so x.5 ulp of bf16 is bit 15 set and the bits below it clear
    ties = (torch.randint(0, 1 << 16, (n // 4,), generator=g, device="cuda", dtype=torch.int32) << 16) | (1 << 15)
    flat[: n // 4] = ties.view(torch.float32)
    flat[-min(n, special.numel()):] = special[: min(n, special.numel())]
    got = ops.pack_bf16(w)
    ref = pack_ref(w)
    assert got.shape == ref.shape and got.dtype == torch.bfloat16
    gi, ri = got.view(torch.int16), ref.view(torch.int16)
    nan = torch.isnan(ref.float())
    assert bool((torch.isnan(got.float()) == nan).all()), "NaN positions differ"
    _exact(gi[~nan], ri[~nan], f"pack {rows}x{cols}")
    if cols % 32:
        src = torch.arange(got.shape[1]) // 16 * 16 + perm16().repeat(got.shape[1] // 16)
        pad = (src >= cols).to(got.device)
        assert bool((got.view(torch.int16)[:, pad] == 0).all()), "padding columns are not zero"


# ============================================================================================== B: every instance vs float64
def pw_ref_bf16(d, w):
    """float64 Z[b] = bf16(W) . bf16(D[b])."""
    B, K, H, W_ = d.shape
    wd = bf16(w.reshape(w.shape[0], K)).double()
    out = torch.empty((B, w.shape[0], H, W_), device=d.device, dtype=torch.float64)
    for b in range(B):
        out[b] = (wd @ bf16(d[b].reshape(K, -1)).double()).view(-1, H, W_)
    return out


def _fused_case(layer, k, seed_shift=11):
    name, C0, C1, Cout, H = layer
    B, Cin = _batch(H), C0 + C1
    K = k * Cin
    g = _gen(_seed(layer) + seed_shift + k)
    x = _randn((B, Cin, H, H), g)
    w, b = _randn((K, 1, 3, 3), g, 1.0 / 3.0), _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    pb = _randn((Cout,), g, 0.3)
    return g, x, w, b, pw, sc, sh, pb


CASES_B = [(l, 2) for l in FUSED] + [(l, k) for l in FUSED if l[0] in ("inc.1", "down1.0", "up2.0") for k in (1, 4)]


@pytest.mark.parametrize("layer,k", CASES_B, ids=[f"{_lid(l)}_k{k}" for l, k in CASES_B])
def test_fused_dsconv_bf16_at_network_shapes(layer, k, bf16_mode):
    name, C0, C1, Cout, H = layer
    g, x, w, b, pw, sc, sh, pb = _fused_case(layer, k)
    x0, x1 = _split(x, C0, C1)
    what = f"bf16 fused {_lid(layer)} k={k}"
    d = dw_emul(x, w, b, k)
    z = pw_ref_bf16(d, pw)
    del d
    ref_eval = torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    wops = ops.weight_operands(pw, 3)
    assert ops.dsconv_takes(x0, x1, pw, k, "bf16")
    y = ops.dsconv(x0, w, b, k, pw, sc, sh, True, x1=x1, mode="bf16", w_split=wops)
    _check(y, ref_eval, ERR_BOUND["fused"], f"{what} eval")
    _exact(ops.dsconv(x0, w, b, k, pw, sc, sh, True, x1=x1, mode="bf16"), y, f"{what} repeat, pack made by the call")
    if Cout <= 128:
        zb = z + pb.double().view(1, -1, 1, 1)
        stats = ops.new_stats(Cout, x.device)
        y = ops.dsconv(x0, w, b, k, pw, None, pb, False, x1=x1, mode="bf16", w_split=wops, stats=stats)
        _check(y, zb, ERR_BOUND["fused"], f"{what} train")
        _check(stats[:Cout], zb.sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"], f"{what} stats sum")
        _check(stats[Cout:], (zb * zb).sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"], f"{what} stats sum of squares")
        del zb
    if name == "up4.1":
        ow, ob = _randn((1, Cout), g, Cout ** -0.5), _randn((1,), g, 0.3)
        lg = ops.dsconv(x0, w, b, k, pw, sc, sh, True, x1=x1, mode="bf16", w_split=wops, outconv=(ow, ob))
        ref = torch.einsum("c,bchw->bhw", ow.double().view(-1), ref_eval).unsqueeze(1) + ob.double()
        _check(lg, ref, ERR_BOUND["fused"], f"{what} outconv")
        ow8, ob8 = _randn((8, Cout), g, Cout ** -0.5), _randn((8,), g, 0.3)
        cls, lg8 = ops.dsconv_classify(x0, w, b, k, pw, sc, sh, True, ow8, ob8, mode="bf16", w_split=wops, want_logits=True)
        ref8 = torch.einsum("kc,bchw->bkhw", ow8.double(), ref_eval) + ob8.double().view(1, -1, 1, 1)
        _check(lg8, ref8, ERR_BOUND["fused"], f"{what} 8-class logits")
        _exact(cls, torch.argmax(lg8, dim=1), f"{what} class map = argmax of its logits")
        for j in range(8):          # class j's logits are the one-class epilogue's with OutConv row j, bit for bit
            lj = ops.dsconv(x0, w, b, k, pw, sc, sh, True, mode="bf16", w_split=wops, outconv=(ow8[j:j + 1], ob8[j:j + 1]))
            _exact(lg8[:, j:j + 1], lj, f"{what} class {j} vs one-class epilogue")
    if name in ("up3.0", "inc.1", "up4.1"):
        sc_g = torch.rand((x.shape[0], C0), generator=g, device="cuda") + 0.5
        sa_g = torch.rand((x.shape[0], 1, H, H), generator=g, device="cuda")
        pools = ops.dsconv_cbam_takes(x0, x1, pw, k, gate=True, pools=True, mode="bf16")
        out = ops.dsconv_cbam(x0, w, b, k, pw, sc, sh, True, x1=x1, mode="bf16", w_split=wops, gate=(sc_g, sa_g), pools=pools)
        yg = out[0] if pools else out
        xg = x.clone()
        xg[:, :C0] = (x0 * sc_g.view(*sc_g.shape, 1, 1)) * sa_g
        refg = torch.relu(pw_ref_bf16(dw_emul(xg, w, b, k), pw) * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
        _check(yg, refg, ERR_BOUND["fused"], f"{what} CBAM gate on load")
        if pools:
            _exact(out[3], F.max_pool2d(yg, 2), f"{what} max-pool from the staged output")


@pytest.mark.parametrize("layer", UNFUSED, ids=_lid)
def test_pointwise_bf16_forward_and_input_gradient(layer, bf16_mode):
    name, C0, C1, Cout, H = layer
    B, Cin = _batch(H), C0 + C1
    K = 2 * Cin
    g = _gen(_seed(layer) + 21)
    d = _randn((B, K, H, H), g)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    z = pw_ref_bf16(d, pw)
    y = ops.pw1x1(d, pw, sc, sh, True, mode="bf16")
    _check(y, torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)), ERR_BOUND["pw"], f"bf16 pw1x1 {_lid(layer)}")
    dz = _randn((B, Cout, H, H), g)
    dW = torch.zeros_like(pw)
    dd = Fn.pw_bwd(dz, d, pw, dW, None)
    _check(dd, pw_ref_bf16(dz, pw.t().contiguous()), ERR_BOUND["pw"], f"bf16 pw1x1 input gradient {_lid(layer)}")


DENSE = [(12, 0, 64, 288), (64, 64, 64, 288), (64, 0, 128, 144), (128, 128, 128, 144), (128, 0, 256, 72), (256, 0, 512, 36),
         (512, 512, 512, 36), (256, 0, 128, 72)]


def _conv_ref(x, w):
    """float64 conv3x3 (padding 1) on bf16-rounded operands, a few images at a time."""
    out = []
    wd = bf16(w).double()
    for i in range(0, x.shape[0], 4):
        out.append(F.conv2d(bf16(x[i:i + 4]).double(), wd, padding=1))
    return torch.cat(out)


@pytest.mark.parametrize("C0,C1,Cout,H", DENSE, ids=[f"{a}{'+' + str(b) if b else ''}to{c}_S{h}" for a, b, c, h in DENSE])
def test_conv3x3_bf16_forward_and_input_gradient(C0, C1, Cout, H, bf16_mode):
    B = {288: 4, 144: 8}.get(H, 16)
    g = _gen(C0 * 5 + C1 + Cout + H)
    x = _randn((B, C0 + C1, H, H), g)
    w = _randn((Cout, C0 + C1, 3, 3), g, (9 * (C0 + C1)) ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    x0, x1 = _split(x, C0, C1)
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    assert ops.conv3x3_takes(x0, x1, wp, Cout, "bf16")
    y = ops.conv3x3(x0, wp, Cout, sc, sh, True, x1=x1, mode="bf16")
    z = _conv_ref(x, w)
    _check(y, torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1)), ERR_BOUND["conv3x3"],
           f"bf16 conv3x3 {C0}+{C1}->{Cout} S{H}")
    dz = _randn((B, Cout, H, H), g)
    wt = ops.conv3x3_pack_weight(w, C0, C1, flip_transpose=True)
    dx = ops.conv3x3(dz, wt, C0 + C1, None, None, False, mode="bf16")
    ref = torch.cat([F.conv_transpose2d(bf16(dz[i:i + 4]).double(), bf16(w).double(), padding=1) for i in range(0, B, 4)])
    _check(dx, ref, ERR_BOUND["conv3x3"], f"bf16 conv3x3 input gradient {C0}+{C1}->{Cout} S{H}")


# ======================================================================================== C: exact-integer production launches
@pytest.mark.parametrize("name", ["inc.0", "up4.0", "up4.1"])
def test_fused_dsconv_bf16_exact_integers_at_production_size(name, bf16_mode):
    layer = next(l for l in LAYERS if l[0] == name)
    _, C0, C1, Cout, H = layer
    B, Cin = 32, C0 + C1
    K = 2 * Cin
    g = _gen(_seed(layer) + 32)
    x = _int_data((B, Cin, H, H), g)
    w = _int_data((K, 1, 3, 3), g)
    b = _int_data((K,), g, -2, 2)
    pw = _int_data((Cout, K), g)
    sc = 2.0 ** _int_data((Cout,), g)
    sh = _int_data((Cout,), g, -32, 32) / 8
    ow, ob = _int_data((1, Cout), g), _int_data((1,), g, -16, 16) / 8
    x0, x1 = _split(x, C0, C1)
    y_ref = torch.empty((B, Cout, H, H), device="cuda")
    lg_ref = torch.empty((B, 1, H, H), device="cuda")
    for i in range(B):
        d = F.conv2d(x[i:i + 1].double(), w.double(), b.double(), padding=1, groups=Cin)
        assert d.abs().max().item() <= 256, "depthwise values must stay exact in bf16"
        z = (pw.double() @ d.view(K, -1)).view(1, Cout, H, H)
        ye = torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
        y_ref[i] = ye[0].float()
        lg_ref[i] = (torch.einsum("c,chw->hw", ow.double().view(-1), ye[0]) + ob.double()).float()
    del x
    _exact(ops.dsconv(x0, w, b, 2, pw, sc, sh, True, x1=x1, mode="bf16"), y_ref, f"bf16 integers {name} B32 y")
    if name == "up4.1":
        _exact(ops.dsconv(x0, w, b, 2, pw, sc, sh, True, mode="bf16", outconv=(ow, ob)), lg_ref, f"bf16 integers {name} logits")


def _int_affine(C, g):
    return 2.0 ** _int_data((C,), g), _int_data((C,), g, -32, 32) / 8


def test_pointwise_bf16_exact_integers_at_production_size(bf16_mode):
    """pw1x1 in bf16 at B = 32, 288 x 288 on inc.1's depthwise output (K = 128 -> 64: the N_TILE 64 instance) and its input
    gradient (64 -> 128: the N_TILE 128 instance), integer data: bit-equal to float64."""
    B, K, Cout, H = 32, 128, 64, 288
    g = _gen(4242)
    d = _int_data((B, K, H, H), g)
    pw = _int_data((Cout, K), g)
    sc, sh = _int_affine(Cout, g)
    y_ref = torch.empty((B, Cout, H, H), device="cuda")
    for i in range(B):
        z = (pw.double() @ d[i].reshape(K, -1).double()).view(Cout, H, H)
        y_ref[i] = torch.relu(z * sc.double().view(-1, 1, 1) + sh.double().view(-1, 1, 1)).float()
    _exact(ops.pw1x1(d, pw, sc, sh, True, mode="bf16"), y_ref, "bf16 integers pw1x1 B32 288 y")
    del y_ref
    dz = _int_data((B, Cout, H, H), g)
    dd_ref = torch.empty((B, K, H, H), device="cuda")
    for i in range(B):
        dd_ref[i] = (pw.double().t() @ dz[i].reshape(Cout, -1).double()).view(K, H, H).float()
    dd = Fn.pw_bwd(dz, d, pw, torch.zeros_like(pw), None)
    _exact(dd, dd_ref, "bf16 integers pw1x1 input gradient B32 288")


def test_conv3x3_bf16_exact_integers_at_production_size(bf16_mode):
    """The dense 3x3 conv in bf16 at B = 32, 288 x 288: UNet up4's first conv over the virtual concat (64 + 64 -> 64) and its
    input gradient (64 -> 128), integer data: bit-equal to float64."""
    B, C0, C1, Cout, H = 32, 64, 64, 64, 288
    g = _gen(4343)
    x = _int_data((B, C0 + C1, H, H), g)
    w = _int_data((Cout, C0 + C1, 3, 3), g)
    sc, sh = _int_affine(Cout, g)
    x0, x1 = _split(x, C0, C1)
    y_ref = torch.empty((B, Cout, H, H), device="cuda")
    for i in range(B):
        z = F.conv2d(x[i:i + 1].double(), w.double(), padding=1)[0]
        y_ref[i] = torch.relu(z * sc.double().view(-1, 1, 1) + sh.double().view(-1, 1, 1)).float()
    del x
    wp = ops.conv3x3_pack_weight(w, C0, C1)
    _exact(ops.conv3x3(x0, wp, Cout, sc, sh, True, x1=x1, mode="bf16"), y_ref, "bf16 integers conv3x3 B32 288 y")
    del x0, x1, y_ref
    dz = _int_data((B, Cout, H, H), g)
    dx_ref = torch.empty((B, C0 + C1, H, H), device="cuda")
    for i in range(B):
        dx_ref[i] = F.conv_transpose2d(dz[i:i + 1].double(), w.double(), padding=1)[0].float()
    wt = ops.conv3x3_pack_weight(w, C0, C1, flip_transpose=True)
    _exact(ops.conv3x3(dz, wt, C0 + C1, None, None, False, mode="bf16"), dx_ref, "bf16 integers conv3x3 input gradient B32 288")


# ============================================================================================================ D: whole networks
def _bn_randomise(m, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for mod in m.modules():
            if isinstance(mod, nn.BatchNorm2d):
                mod.running_mean.uniform_(-0.2, 0.2, generator=g)
                mod.running_var.uniform_(0.5, 1.5, generator=g)
                mod.weight.uniform_(0.8, 1.2, generator=g)
                mod.bias.uniform_(-0.1, 0.1, generator=g)
    return m


def _port(model, x, dense=False):
    sd = {k: (v.detach() if v.dtype == torch.int64 else v.detach().double()) for k, v in model.state_dict().items()}
    out = []
    with torch.no_grad():
        for i in range(0, x.shape[0], 4):
            xd = x[i:i + 4].double()
            out.append(DO.port_unet_forward(xd, sd) if dense else TP.smaat_unet_forward(xd, sd))
    return torch.cat(out)


NETS = {
    "smaat_12_1": (lambda: S.SmaAt_UNet(12, 1, kernels_per_layer=2), 32, (12, 288, 288), "net_smaat", False),
    "smaat_3_21": (lambda: S.SmaAt_UNet(3, 21, kernels_per_layer=2), 8, (3, 224, 224), "net_seg_logits", False),
    "unet_12_1": (lambda: S.UNet(12, 1), 32, (12, 288, 288), "net_unet", True),
}


@pytest.mark.parametrize("name", list(NETS))
def test_networks_in_bf16_against_the_float64_port(name, bf16_mode):
    ctor, B, shape, bound, dense = NETS[name]
    torch.manual_seed(3)
    model = _bn_randomise(ctor(), 4).cuda().eval()
    x = torch.rand((B,) + shape, generator=_gen(5), device="cuda")
    sess = InferenceSession(model, B, shape)
    y = sess.forward(x).clone()
    with torch.no_grad():
        eager = model.forward_serving(x)
    _exact(y, eager, f"{name} session vs eager serving forward")
    ref = _port(model, x, dense)
    _check(y, ref, ERR_BOUND[bound], f"{name} bf16 logits vs float64 port")
    if name == "smaat_3_21":
        probs = InferenceSession(model, B, shape, output="probs").forward(x).clone()
        with torch.no_grad():
            _exact(probs, model.forward_probs(x), f"{name} probability session vs eager")
        _check(probs, torch.softmax(ref, dim=1), ERR_BOUND["net_seg_probs"], f"{name} bf16 probabilities vs float64 port")
        cls_unfused = InferenceSession(model, B, shape, output="classes", serving_fusions=False).forward(x).clone()
        _exact(cls_unfused, torch.argmax(eager, dim=1), f"{name} unfused class map = argmax(bf16 logits)")
        cls = InferenceSession(model, B, shape, output="classes").forward(x).clone()
        with torch.no_grad():
            _exact(cls, model.forward_classes(x), f"{name} class-map session vs eager")
        agree = float((cls == torch.argmax(ref, dim=1)).double().mean())
        print(f"ERR {name} bf16 class map agreement with the float64 port: {agree:.5f}")
        assert agree > 0.99


# ============================================================================================================ E: a training step
def _session_step(sd, x, y, mode, use_graph):
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode(mode)
    try:
        m = S.SmaAt_UNet(12, 1, kernels_per_layer=2)
        m.load_state_dict(sd)
        m = m.cuda().train()
        sess = TrainSession(m, x.shape[0], tuple(x.shape[1:]), lr=1e-3, use_graph=use_graph)
        names = [k for k, _ in m.named_parameters()]
        params = dict(m.named_parameters())
        P0 = sess.flat_param.clone()
        sess.step(x, y)
        torch.cuda.synchronize()
        G = sess.flat_grad.clone()
        spans = {k: (o, params[k].numel(), params[k].shape) for k, o in zip(names, sess._offsets)}
        sess.close()
        state = {k: P0[o:o + n].view(s).double() for k, (o, n, s) in spans.items()}
        return G, spans, state
    finally:
        ops.set_pointwise_mode(old)


def _tf32_trunc(t):
    return (t.float().contiguous().view(torch.int32) & -8192).view(torch.float32).to(t.dtype)


class _PointwiseBf16Operands(torch.autograd.Function):
    """The pointwise conv as the bf16 training step computes it, in the port's dtype: forward and input gradient on
    bf16-rounded operands (pw1x1 in 'bf16'), weight gradient on tf32-truncated operands (the tf32 weight-gradient kernel)."""

    @staticmethod
    def forward(ctx, d, w, b):
        ctx.save_for_backward(d, w)
        return F.conv2d(bf16(d).to(d.dtype), bf16(w).to(w.dtype), b)

    @staticmethod
    def backward(ctx, g):
        d, w = ctx.saved_tensors
        dd = F.conv_transpose2d(bf16(g).to(g.dtype), bf16(w).to(w.dtype))
        dw = torch.einsum("bohw,bchw->oc", _tf32_trunc(g), _tf32_trunc(d)).view_as(w)
        return dd, dw, g.sum(dim=(0, 2, 3))


def _ds_conv_bf16_operands(x, sd, p):
    """oracle.torch_port.ds_conv with its pointwise conv on the bf16 step's operands."""
    w = sd[p + ".depthwise.weight"]
    y = F.conv2d(x, w, sd[p + ".depthwise.bias"], padding=1, groups=x.shape[1])
    return _PointwiseBf16Operands.apply(y, sd[p + ".pointwise.weight"], sd[p + ".pointwise.bias"])


def test_train_session_step_in_bf16():
    """The state and batch of tests/test_gpu_train_tail.py's captured-step check (fill_schema weights, B = 2, 288 x 288, mse):
    a well-conditioned step, where the tf32x3 session is within a few times the port's own fp32 noise of float64."""
    sd = load_np_state_dict(S.SmaAt_UNet(12, 1, kernels_per_layer=2),
                            cast_sd(fill_schema(smaat_unet_schema(12, 1, 2), 12), np.float32)).state_dict()
    B, H = 2, 288
    rng = np.random.default_rng(5)
    x = torch.from_numpy(rng.uniform(0, 1, (B, 12, H, H))).float().cuda()
    y = torch.from_numpy(rng.uniform(0, 1, (B, H, H))).float().cuda()
    Gc, spans, state = _session_step(sd, x, y, "bf16", True)
    Ge, _, _ = _session_step(sd, x, y, "bf16", False)
    Ge2, _, _ = _session_step(sd, x, y, "bf16", False)
    # the weight-gradient kernels merge their partial sums with fp32 atomics: two eager steps differ in the last bits, and
    # train-mode BatchNorm carries that into every earlier layer.  The captured step must be no further from an eager step
    d_ce, d_ee = (Gc - Ge).norm().item(), (Ge2 - Ge).norm().item()
    print(f"ERR bf16 captured vs eager step gradients: rel L2 {d_ce / Ge.norm().item():.2e} "
          f"(eager vs eager {d_ee / Ge.norm().item():.2e})")
    assert d_ce <= NOISE_FACTOR * max(d_ee, 1e-7 * Ge.norm().item())

    def port_grads(dtype, bf16_operands=False):
        full = {k: (v.detach().cuda() if v.dtype == torch.int64 else v.detach().cuda().to(dtype)) for k, v in sd.items()}
        for k in spans:
            full[k] = state[k].to(dtype).clone().requires_grad_(True)
        with pytest.MonkeyPatch.context() as mp:
            if bf16_operands:
                mp.setattr(TP, "ds_conv", _ds_conv_bf16_operands)
            out = TP.smaat_unet_forward(x.to(dtype), full, True)
        loss = F.mse_loss(out.squeeze(1), y.to(dtype), reduction="sum") / B
        return dict(zip(spans, torch.autograd.grad(loss, [full[k] for k in spans])))

    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    try:
        g64 = port_grads(torch.float64)                          # the reference in exact arithmetic
        g64_ops = port_grads(torch.float64, bf16_operands=True)  # float64 on the operands the bf16 step rounds
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    gmax = max(v.abs().max().item() for v in g64.values())
    on = [k for k in spans if g64[k].abs().max().item() >= 1e-6 * gmax]   # the rest is mathematically zero (biases before
                                                                           # a train-mode BatchNorm): summation noise only

    def rel(G, ref, keys):
        """Bucket rel L2 of G against ref over ``keys``, and the per-parameter rel L2."""
        got = {k: (G[k].double() if isinstance(G, dict) else G[spans[k][0]:spans[k][0] + spans[k][1]].view(spans[k][2]).double())
               for k in keys}
        num = sum(((got[k] - ref[k]) ** 2).sum().item() for k in keys) ** 0.5
        den = sum((ref[k] ** 2).sum().item() for k in keys) ** 0.5
        return num / den, {k: (got[k] - ref[k]).norm().item() / ref[k].norm().item() for k in keys}

    # Train-mode BatchNorm over this batch makes most gradients chaotic at bf16 resolution: the port on bf16 operands moves
    # the bucket by 0.46 from float64 (fp32 operands: 4.7e-3), so no bf16 arithmetic, ours or torch's, can be held close to
    # float64 there.  Two checks that can still fail:
    #  1. over all parameters, the step is no further from float64 than BUCKET_FACTOR x the port on the same rounded
    #     operands (an all-zero gradient is 1.0 off, a sign-flipped one 2.0);
    #  2. over the parameters whose gradient bf16 operands move by at most WELL_CONDITIONED in the port, the step is within
    #     NOISE_FACTOR x the port's own distance, a bound well below 1
    o_all, moved = rel(g64_ops, g64, on)
    r_all, _ = rel(Gc, g64, on)
    sel = [k for k in on if moved[k] <= WELL_CONDITIONED]
    o, _ = rel(g64_ops, g64, sel)
    e, per = rel(Gc, g64, sel)
    tol_all, tol = BUCKET_FACTOR * o_all, NOISE_FACTOR * o
    print(f"ERR bf16 step gradients vs float64, all {len(on)} parameters: bucket rel L2 {r_all:.2e} (the port on bf16 operands "
          f"{o_all:.2e}, bound {tol_all:.2e})")
    print(f"ERR bf16 step gradients vs float64, the {len(sel)} parameters bf16 operands move by <= {WELL_CONDITIONED:.0%} "
          f"({', '.join(sel)}): bucket rel L2 {e:.2e} (the port on bf16 operands {o:.2e}, bound {tol:.2e})")
    assert tol_all < 1.0 and r_all <= tol_all
    assert len(sel) >= 3 and tol <= 0.1 and e <= tol


# ===================================================================================================== F: caches and sessions
def _disrupt(m, how):
    if how == "mode":
        ops.set_pointwise_mode("tf32x3")
    elif how == "train_eval":
        m.train()
        m.eval()
    elif how == "assign":
        torch.manual_seed(77)
        other = _bn_randomise(S.SmaAt_UNet(12, 1), 78).state_dict()
        m.load_state_dict({k: v.cuda() for k, v in other.items()}, assign=True)
        m.eval()


@pytest.mark.parametrize("how", ["mode", "train_eval", "assign"])
def test_bf16_pack_survives_what_the_split_survives(how, bf16_mode):
    torch.manual_seed(12)
    m = _bn_randomise(S.SmaAt_UNet(12, 1), 13).cuda().eval()
    x = torch.rand((2, 12, 64, 64), generator=_gen(14), device="cuda")
    sess = InferenceSession(m, 2, (12, 64, 64))
    y0 = sess.forward(x).clone()
    packs = [t for t in cached_tensors(m) if t.dtype == torch.bfloat16]
    assert packs, "the bf16 packs are cached"
    held = {t.data_ptr() for t in sess._keepalive}
    assert all(t.data_ptr() in held for t in packs), "the session holds every bf16 pack its graph reads"
    _disrupt(m, how)
    with torch.no_grad():                                           # eager work that recycles freed blocks
        m(torch.rand((2, 12, 64, 64), device="cuda"))
    junk = [torch.full((1 << 18,), float("nan"), device="cuda") for _ in range(64)]
    torch.cuda.synchronize()
    _exact(sess.forward(x).clone(), y0, f"session after {how}: its captured result")
    del junk
    ops.set_pointwise_mode("bf16")
    sess.refresh()
    fresh = S.SmaAt_UNet(12, 1)
    fresh.load_state_dict(m.state_dict())
    fresh = fresh.cuda().eval()
    with torch.no_grad():
        want = fresh.forward_serving(x)
    _exact(sess.forward(x).clone(), want, f"session after {how} and refresh(): the fresh model's bf16 output")
