"""The serving forward's CBAM fusions for levels 1-3 (smaat_dsconv_cbam_fwd, smaat_cbam_mlp_partials_fwd):
(a) the partial pools and the 2x2 max-pool a DS conv writes from its epilogue against the standalone pool kernels on that conv's
    own output: maxima and max-pool bit for bit, means within 2e-6, two launches bit for bit;
(b) an up-block DS conv that applies the CBAM gates as it loads the skip against the same conv on the materialised CBAM output,
    bit for bit, at the up2 / up3 / up4 shapes in both tensor-core modes;
(c) SmaAt_UNet.forward_serving, which applies the level 1-3 gates on load, against the plain-call forward.
The serving forward uses (b) only: pools summed in another order would move the channel gate, and with it the logits, away
from the plain forward's."""
import numpy as np
import pytest
import torch

import smaat_unet_b200 as S
from oracle.cases import cast_sd, fill_schema, smaat_unet_schema
from smaat_unet_b200 import ops
from tests._util import NET_TOL, assert_close, load_np_state_dict

pytestmark = pytest.mark.gpu


def _conv_params(g, Cin, Cout, k=2):
    K = k * Cin
    return dict(dw_weight=torch.randn(K, 1, 3, 3, device="cuda", generator=g) * 0.3,
                dw_bias=torch.randn(K, device="cuda", generator=g) * 0.1,
                pw_weight=torch.randn(Cout, K, 1, 1, device="cuda", generator=g) * (1.0 / K ** 0.5),
                scale=torch.rand(Cout, device="cuda", generator=g) + 0.5,
                shift=torch.randn(Cout, device="cuda", generator=g) * 0.1)


def _mlp(g, C, r=16):
    h = C // r
    return (torch.randn(h, C, device="cuda", generator=g) * 0.2, torch.randn(h, device="cuda", generator=g) * 0.1,
            torch.randn(C, h, device="cuda", generator=g) * 0.2, torch.randn(C, device="cuda", generator=g) * 0.1)


# (B, Cin, H, W, Cout): the second DS conv of inc / down1 / down2 (the maps CBAM levels 1-3 gate), and one odd-H shape whose
# last half-patch row lies across the image's bottom edge (odd last row: in the pools, not in the max-pool)
POOL_CASES = [(32, 64, 288, 288, 64), (32, 128, 144, 144, 128), (32, 256, 72, 72, 256), (2, 16, 101, 64, 64)]


@pytest.mark.parametrize("case", POOL_CASES, ids=lambda c: f"C{c[1]}_N{c[4]}_{c[2]}x{c[3]}")
def test_epilogue_pools_match_pool_kernels_on_the_conv_output(case):
    B, Cin, H, W, Cout = case
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.rand(B, Cin, H, W, device="cuda", generator=g)
    prm = _conv_params(g, Cin, Cout)
    assert ops.dsconv_cbam_takes(x, None, prm["pw_weight"], 2, pools=True)
    y, psum, pmax, pooled = ops.dsconv_cbam(x, prm["dw_weight"], prm["dw_bias"], 2, prm["pw_weight"], prm["scale"], prm["shift"],
                                            True, pools=True)
    w1, b1, w2, b2 = _mlp(g, Cout)
    sc, avg, mx = ops.cbam_mlp_partials(psum, pmax, H, W, w1, b1, w2, b2)
    # the reference: the standalone kernels on the very tensor the conv wrote
    avg_ref, mx_ref = ops.cbam_pool(y)
    assert torch.equal(mx, mx_ref), "channel max differs from smaat_cbam_pool_fwd"
    rel = ((avg.double() - avg_ref.double()).abs() / avg_ref.double().abs().clamp_min(1e-30)).max().item()
    assert rel <= 2e-6, f"channel mean: max rel diff {rel:.2e} vs smaat_cbam_pool_fwd"
    assert torch.equal(pooled, ops.maxpool2(y)), "epilogue max-pool differs from smaat_maxpool2_fwd"
    sc_ref = ops.cbam_mlp(avg_ref, mx_ref, w1, b1, w2, b2)
    assert_close(sc, sc_ref.double().cpu().numpy(), 1e-6, "channel gate from the partials")
    # a second launch writes the same bits (fixed partial layout and reduction order)
    y2, psum2, pmax2, pooled2 = ops.dsconv_cbam(x, prm["dw_weight"], prm["dw_bias"], 2, prm["pw_weight"], prm["scale"],
                                                prm["shift"], True, pools=True)
    sc2, avg2, mx2 = ops.cbam_mlp_partials(psum2, pmax2, H, W, w1, b1, w2, b2)
    assert torch.equal(y, y2) and torch.equal(psum, psum2) and torch.equal(pmax, pmax2) and torch.equal(pooled, pooled2)
    assert torch.equal(avg, avg2) and torch.equal(mx, mx2) and torch.equal(sc, sc2)
    # the activation itself is what the plain fused conv writes
    y_plain = ops.dsconv(x, prm["dw_weight"], prm["dw_bias"], 2, prm["pw_weight"], prm["scale"], prm["shift"], True)
    assert torch.equal(y, y_plain)


# (B, C0 = C1, S, Cout): the first DS conv of up2 (two channel passes, so it gates twice), up3 and up4
GATE_CASES = [(32, 256, 72, 256), (32, 128, 144, 128), (32, 64, 288, 64)]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32"])
@pytest.mark.parametrize("case", GATE_CASES, ids=lambda c: f"C{2 * c[1]}_N{c[3]}_{c[2]}")
def test_gated_conv_equals_conv_on_materialised_cbam_output(case, mode):
    B, C0, S_, Cout = case
    g = torch.Generator(device="cuda").manual_seed(12)
    x0 = torch.rand(B, C0, S_, S_, device="cuda", generator=g)           # the un-attended skip (post-ReLU: non-negative)
    x1 = torch.randn(B, C0, S_, S_, device="cuda", generator=g)          # the upsampled decoder map
    sc = torch.rand(B, C0, device="cuda", generator=g)
    sa = torch.rand(B, 1, S_, S_, device="cuda", generator=g)
    prm = _conv_params(g, 2 * C0, Cout)
    assert ops.dsconv_cbam_takes(x0, x1, prm["pw_weight"], 2, gate=True, mode=mode)
    y_cbam = ops.cbam_scale(x0, sc, sa)
    ref = ops.dsconv(y_cbam, prm["dw_weight"], prm["dw_bias"], 2, prm["pw_weight"], prm["scale"], prm["shift"], True, x1=x1, mode=mode)
    assert ref is not None
    got = ops.dsconv_cbam(x0, prm["dw_weight"], prm["dw_bias"], 2, prm["pw_weight"], prm["scale"], prm["shift"], True, x1=x1,
                          mode=mode, gate=(sc, sa))
    assert torch.equal(got, ref), f"gated conv differs from the conv on the CBAM output: max |diff| {(got - ref).abs().max().item():.3e}"


def test_forward_serving_matches_forward_and_takes_the_cbam_fusions():
    sd = cast_sd(fill_schema(smaat_unet_schema(12, 1, 2), 5), np.float32)
    m = load_np_state_dict(S.SmaAt_UNet(12, 1, kernels_per_layer=2), sd).cuda().eval()
    x = torch.rand(4, 12, 288, 288, device="cuda", generator=torch.Generator(device="cuda").manual_seed(13))
    with torch.no_grad():
        ref = m(x)
        with ops.profile() as prof:
            got = m.forward_serving(x)
        names = [r[0] for r in prof.records]
    assert_close(got, ref.double().cpu().numpy(), NET_TOL["tf32x3"], "forward_serving vs forward")
    # levels 1-3 never write their CBAM output (levels 4-5 still do), and the launch count stays what it was
    assert [n for n in names if n.startswith("smaat_cbam_gate_scale_fwd")] == ["smaat_cbam_gate_scale_fwd[C512_S36]"], names
    # levels 1-3 compute sa alone; level 5 (W = 18, not a multiple of 4) runs the gate and the scale as two launches
    assert sum(n.startswith("smaat_cbam_gate_fwd") for n in names) == 4
    assert sum(n.startswith("smaat_cbam_scale_fwd") for n in names) == 1
