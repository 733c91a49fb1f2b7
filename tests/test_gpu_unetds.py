"""UNetDS and UNetDSAttention4CBAMs built natively, and the fused DS conv's max-pool epilogue, on the GPU.

  A  the max-pool epilogue (smaat_dsconv_maxpool_fwd, smaat_dsconv_maxpool_bf16_fwd): y is bit for bit the plain fused conv's
     output and pooled bit for bit max_pool2d(y), at UNetDS's producing convs (288) and at partial tiles, odd H, k = 1, B = 1
     and 5, both pooled dtypes from bf16 maps; written through the C ABI into NaN-poisoned, over-allocated buffers
  B  both reference goldens through the native classes, forward and forward_serving, in tf32x3, tf32 and fp32
  C  the networks against the float64 port (TP.smaat_unet_forward(..., n_cbams=0 / 4)): (12, 1) B = 32 at 288 logits and
     (3, 21) B = 8 at 224 logits, probabilities and class maps, through the fp32 and the bf16 storage routes (the bf16 route
     also against the port with its roundings emulated), with test_gpu_bf16_activations.py's bounds
  D  UNetDS's serving launch profile: no standalone max-pool where the epilogue takes the shape
  E  sessions: output bit for bit the eager serving forward; partial batches the same rows of the full batch
  F  a TrainSession step on each model against the same step of RefOrderNet (the reference's call order)
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from oracle import torch_port as TP
from oracle.cases import CASES, case_tensors
from smaat_unet_b200 import _lib, ops
from smaat_unet_b200.engine import InferenceSession
from tests._util import NET_TOL, assert_close, dev, load_np_state_dict
from tests.test_gpu_bf16 import _bn_randomise
from tests.test_gpu_bf16_activations import MIN_CLASS_AGREEMENT, NET_BOUND, _dc_port, _sd64, _up, r16
from tests.test_gpu_ds_forward_kernels import _check, _exact, _gen, _randn

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
GOLD = os.path.join(os.path.dirname(__file__), "golden")
MODELS = {0: S.UNetDS, 4: S.UNetDSAttention4CBAMs}


# ================================================================================================= A: the max-pool epilogue
# (name, Cin, Cout, H, W, k, B): UNetDS(12, 1)'s producing convs at 288 (down3.1's 36 x 36 map is not fused: the patch waste
# rule), then partial tiles (Cout 40, W not a multiple of the patch), odd H, k = 1, B = 1 and 5
POOL_CASES = [("inc.1", 64, 64, 288, 288, 2, 2), ("down1.1", 128, 128, 144, 144, 2, 2), ("down2.1", 256, 256, 72, 72, 2, 2),
              ("down3.1_64", 512, 512, 64, 64, 2, 2), ("partial_odd", 64, 40, 37, 56, 2, 5), ("k1_b1", 32, 8, 20, 24, 1, 1),
              ("pw16_b5", 128, 128, 56, 40, 2, 5)]


def _case(name, Cin, Cout, H, W, k, B, bf16):
    g = _gen(Cin * 7 + Cout + H * 3 + W + k)
    x = _randn((B, Cin, H, W), g)
    if bf16:
        x = r16(x).float()
    K = k * Cin
    w, b = _randn((K, 1, 3, 3), g, 1.0 / 3.0), _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = torch.rand((Cout,), generator=g, device="cuda") + 0.5, _randn((Cout,), g, 0.1)
    return x, w, b, pw, sc, sh


def _poisoned(n, dtype, pad=4096):
    return torch.full((n + pad,), float("nan"), device="cuda", dtype=dtype)


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "bf16"])
@pytest.mark.parametrize("case", POOL_CASES, ids=[c[0] for c in POOL_CASES])
def test_maxpool_epilogue_fp32_maps(case, mode):
    name, Cin, Cout, H, W, k, B = case
    x, w, b, pw, sc, sh = _case(*case, bf16=False)
    assert ops.dsconv_maxpool_takes(x, None, pw, k, mode), case
    y0 = ops.dsconv(x, w, b, k, pw, sc, sh, True, mode=mode)
    y, pooled = ops.dsconv_maxpool(x, w, b, k, pw, sc, sh, True, mode=mode)
    _exact(y, y0, f"{name} {mode}: y vs the plain fused conv")
    _exact(pooled, F.max_pool2d(y, 2), f"{name} {mode}: pooled vs max_pool2d(y)")
    # through the C ABI into NaN-poisoned, over-allocated buffers: nothing is stored past either output
    m = ops.PW_MODES[mode]
    w2d, wlo = ops.weight_operands(pw, m)
    yb, pb = _poisoned(y.numel(), torch.float32), _poisoned(pooled.numel(), torch.float32)
    _lib.check(_lib.load().smaat_dsconv_maxpool_fwd(x.data_ptr(), Cin, Cin * H * W, None, 0, 0, w.data_ptr(), b.data_ptr(),
                                                    w2d.data_ptr(), ops._ptr(wlo), sc.data_ptr(), sh.data_ptr(), yb.data_ptr(),
                                                    Cout * H * W, pb.data_ptr(), B, H, W, k, Cout, 1, m,
                                                    torch.cuda.current_stream().cuda_stream), "dsconv_maxpool")
    _exact(yb[:y.numel()].view_as(y), y, f"{name} {mode}: ABI y")
    _exact(pb[:pooled.numel()].view_as(pooled), pooled, f"{name} {mode}: ABI pooled")
    assert bool(yb[y.numel():].isnan().all()) and bool(pb[pooled.numel():].isnan().all()), f"{name} {mode}: store past the output"


BF_POOL_CASES = [c for c in POOL_CASES if c[4] % 8 == 0]


@pytest.mark.parametrize("pdt", [BF, torch.float32], ids=["pooled_bf16", "pooled_fp32"])
@pytest.mark.parametrize("case", BF_POOL_CASES, ids=[c[0] for c in BF_POOL_CASES])
def test_maxpool_epilogue_bf16_maps(case, pdt):
    name, Cin, Cout, H, W, k, B = case
    x, w, b, pw, sc, sh = _case(*case, bf16=True)
    xb = x.to(BF)
    assert ops.dsconv_maxpool_bf16_takes(xb, None, pw, k), case
    y0 = ops.dsconv_bf16(xb, w, b, k, pw, sc, sh, True)
    y, pooled = ops.dsconv_maxpool_bf16(xb, w, b, k, pw, sc, sh, True, pooled_dtype=pdt)
    assert y.dtype == BF and pooled.dtype == pdt
    _exact(y, y0, f"{name} bf16: y vs the plain bf16 conv")
    _exact(pooled, F.max_pool2d(y.float(), 2).to(pdt), f"{name} bf16 -> {pdt}: pooled vs max_pool2d(y)")
    pack = ops.pack_bf16(pw)
    yb, pb = _poisoned(y.numel(), BF), _poisoned(pooled.numel(), pdt)
    _lib.check(_lib.load().smaat_dsconv_maxpool_bf16_fwd(xb.data_ptr(), Cin, Cin * H * W, None, 0, 0, w.data_ptr(), b.data_ptr(),
                                                         pack.data_ptr(), sc.data_ptr(), sh.data_ptr(), yb.data_ptr(), Cout * H * W,
                                                         pb.data_ptr(), int(pdt == BF), B, H, W, k, Cout, 1,
                                                         torch.cuda.current_stream().cuda_stream), "dsconv_maxpool_bf16")
    _exact(yb[:y.numel()].view_as(y), y, f"{name} bf16: ABI y")
    _exact(pb[:pooled.numel()].view_as(pooled), pooled, f"{name} bf16: ABI pooled")
    assert bool(yb[y.numel():].isnan().all()) and bool(pb[pooled.numel():].isnan().all()), f"{name} bf16: store past the output"


# ================================================================================================== B: the reference goldens
GOLDEN = [("lit_ds_k1_32", 0), ("lit_dsatt4_k2_48", 4)]


@pytest.mark.parametrize("mode", ["tf32x3", "tf32", "fp32"])
@pytest.mark.parametrize("name,n_cbams", GOLDEN)
def test_native_classes_match_the_reference_goldens(name, n_cbams, mode):
    c = CASES[name]
    sd, xs = case_tensors(name, np.float32)
    net = load_np_state_dict(MODELS[n_cbams](c["n_channels"], c["n_classes"], kernels_per_layer=c["k"]), sd).cuda().eval()
    ref = np.load(os.path.join(GOLD, name + ".npz"))["output"]
    S.set_pointwise_mode(mode)
    try:
        with torch.no_grad():
            assert_close(net(dev(xs[0])), ref, NET_TOL[mode], f"{name} forward [{mode}]")
            assert_close(net.forward_serving(dev(xs[0])), ref, NET_TOL[mode], f"{name} forward_serving [{mode}]")
    finally:
        S.set_pointwise_mode("tf32x3")


# ============================================================================================== C: the float64 port, both routes
def _model(n_cbams, n_ch, n_cls, seed=3):
    torch.manual_seed(seed)
    return _bn_randomise(MODELS[n_cbams](n_ch, n_cls, kernels_per_layer=2), 4).cuda().eval()


def _port(x, sd, n_cbams):
    with torch.no_grad():
        return torch.cat([TP.smaat_unet_forward(x[i:i + 4].double(), sd, n_cbams=n_cbams) for i in range(0, x.shape[0], 4)])


def _port_bf16(x, sd, n_cbams, fused_head):
    """test_gpu_bf16_activations._port_bf16 with ``n_cbams`` CBAMs (levels 1..n_cbams)."""
    def one(v):
        enc = [_dc_port(r16(v), sd, "inc", True)]
        for i in range(1, 5):
            enc.append(_dc_port(F.max_pool2d(enc[-1], 2), sd, f"down{i}.maxpool_conv.1", i < 3))
        att = [TP.cbam(e, sd, f"cbam{i + 1}") if i < n_cbams else e for i, e in enumerate(enc)]
        y = TP.up_ds(att[4], att[3], sd, "up1")
        for i in range(2, 5):
            y = _dc_port(_up(y, att[4 - i], BF), sd, f"up{i}.conv", True, round_out=not (i == 4 and fused_head))
        return r16(F.conv2d(y, sd["outc.conv.weight"], sd["outc.conv.bias"]))
    with torch.no_grad():
        return torch.cat([one(x[i:i + 4].double()) for i in range(0, x.shape[0], 4)])


@pytest.mark.parametrize("n_cbams", [0, 4])
def test_12_1_logits_against_the_float64_port(n_cbams):
    B, shape = 32, (12, 288, 288)
    model = _model(n_cbams, 12, 1)
    x = torch.rand((B,) + shape, generator=_gen(5), device="cuda")
    sd = _sd64(model)
    port = _port(x, sd, n_cbams)
    y = InferenceSession(model, B, shape).forward(x).clone()
    assert_close(y, port.cpu().numpy(), NET_TOL["tf32x3"], f"n_cbams={n_cbams} (12, 1) fp32 session vs float64 port")
    xb = x.to(BF)
    yb = InferenceSession(model, B, shape, dtype=BF).forward(xb).clone()
    assert yb.dtype == BF
    _check(yb, _port_bf16(xb, sd, n_cbams, fused_head=True), NET_BOUND["smaat_12_1_emul"],
           f"n_cbams={n_cbams} (12, 1) bf16 logits vs float64 port with the bf16 roundings")
    _check(yb, _port(xb.float(), sd, n_cbams), NET_BOUND["smaat_12_1_port"], f"n_cbams={n_cbams} (12, 1) bf16 logits vs port")


@pytest.mark.parametrize("n_cbams", [0, 4])
def test_3_21_logits_probs_and_classes_against_the_float64_port(n_cbams):
    B, shape = 8, (3, 224, 224)
    model = _model(n_cbams, 3, 21)
    x = torch.rand((B,) + shape, generator=_gen(6), device="cuda")
    sd = _sd64(model)
    port = _port(x, sd, n_cbams)
    lg = InferenceSession(model, B, shape).forward(x).clone()
    assert_close(lg, port.cpu().numpy(), NET_TOL["tf32x3"], f"n_cbams={n_cbams} (3, 21) fp32 logits vs port")
    pr = InferenceSession(model, B, shape, output="probs").forward(x).clone()
    _exact(pr, ops.softmax_channels(lg), f"n_cbams={n_cbams} (3, 21) probabilities = softmax of the served logits")
    cls = InferenceSession(model, B, shape, output="classes").forward(x).clone()
    agree = float((cls == port.argmax(dim=1)).double().mean())
    print(f"ERR n_cbams={n_cbams} (3, 21) fp32 class map agreement with the port: {agree:.6f}")
    assert agree >= 0.999
    xb = x.to(BF)
    emul = _port_bf16(xb, sd, n_cbams, fused_head=False)
    lgb = InferenceSession(model, B, shape, dtype=BF).forward(xb).clone()
    _check(lgb, emul, NET_BOUND["smaat_3_21_emul"], f"n_cbams={n_cbams} (3, 21) bf16 logits vs emulated port")
    _check(lgb, _port(xb.float(), sd, n_cbams), NET_BOUND["smaat_3_21_port"], f"n_cbams={n_cbams} (3, 21) bf16 logits vs port")
    prb = InferenceSession(model, B, shape, output="probs", dtype=BF).forward(xb).clone()
    _check(prb, torch.softmax(emul, dim=1), NET_BOUND["smaat_3_21_probs_emul"], f"n_cbams={n_cbams} (3, 21) bf16 probabilities")
    clsb = InferenceSession(model, B, shape, output="classes", dtype=BF).forward(xb).clone()
    agree = float((clsb == emul.argmax(dim=1)).double().mean())
    print(f"ERR n_cbams={n_cbams} (3, 21) bf16 class map agreement with the emulated port: {agree:.5f}")
    assert agree >= MIN_CLASS_AGREEMENT


# ======================================================================================================= D: launch profile
@pytest.mark.parametrize("S_,expect", [(256, 4), (288, 3)])
def test_unetds_serving_takes_its_max_pools_from_the_epilogue(S_, expect):
    """At 288 the level-4 map (36 x 36) is not taken by the fused conv (patch waste), so down4 pools it itself."""
    model = _model(0, 12, 1)
    x = torch.rand((2, 12, S_, S_), device="cuda")
    with torch.no_grad(), ops.profile() as prof:
        model.forward_serving(x)
    names = [r[0].split("[")[0] for r in prof.records]
    assert names.count("smaat_dsconv_maxpool_fwd") == expect, names
    assert names.count("smaat_maxpool2_fwd") == 4 - expect, names
    with torch.no_grad(), ops.profile() as prof:
        model.forward_serving(x.to(BF))
    names = [r[0].split("[")[0] for r in prof.records]
    assert names.count("smaat_dsconv_maxpool_bf16_fwd") == 3 and names.count("smaat_maxpool2_fwd") == 4 - expect, names


# ============================================================================================================= E: sessions
@pytest.mark.parametrize("dtype", [torch.float32, BF], ids=["fp32", "bf16"])
@pytest.mark.parametrize("n_cbams", [0, 4])
def test_sessions_equal_the_eager_serving_forward_and_partial_batches_their_rows(n_cbams, dtype):
    B, shape = 8, (3, 224, 224)
    model = _model(n_cbams, 3, 21, seed=11)
    x = torch.rand((B,) + shape, generator=_gen(12), device="cuda").to(dtype)
    for output, eager in (("logits", model.forward_serving), ("classes", model.forward_classes), ("probs", model.forward_probs)):
        sess = InferenceSession(model, B, shape, output=output, dtype=dtype, batch_sizes=(3,))
        full = sess.forward(x).clone()
        with torch.no_grad():
            _exact(full, eager(x), f"n_cbams={n_cbams} {output} {dtype}: session vs eager")
        _exact(sess.forward(x[:3]).clone(), full[:3], f"n_cbams={n_cbams} {output} {dtype}: 3 rows")
        _exact(sess.forward(x[:5]).clone(), full[:5], f"n_cbams={n_cbams} {output} {dtype}: 5 rows (the full graph)")


# ================================================================================================= F: training, one step
@pytest.mark.parametrize("n_cbams", [0, 4])
def test_train_session_step_matches_the_reference_order_net(n_cbams):
    from smaat_unet_b200.train import TrainSession
    from tests.test_gpu_api_paths import RefOrderNet
    torch.manual_seed(7)
    m = MODELS[n_cbams](12, 1, kernels_per_layer=2).cuda()
    m_ref = RefOrderNet(12, 1, 2, n_cbams).cuda().train()
    m_ref.load_state_dict(m.state_dict(), strict=True)
    assert [k for k, _ in m.named_parameters()] == [k for k, _ in m_ref.named_parameters()]
    sess = TrainSession(m, 2, (12, 32, 32), lr=0.0, use_graph=True)       # lr 0: weights stay comparable
    assert sess._split is None                       # UNetDS: no CBAM to split at; 4CBAMs: refused by _verify_split
    x, y = torch.rand(2, 12, 32, 32, device="cuda"), torch.rand(2, 32, 32, device="cuda")
    sess.step(x, y)
    loss = torch.nn.functional.mse_loss(m_ref(x).squeeze(1), y, reduction="sum") / 2
    loss.backward()
    torch.cuda.synchronize()
    gmax = max(float(p.grad.abs().max()) for p in m_ref.parameters())
    for (k, p), q in zip(m.named_parameters(), m_ref.parameters()):
        assert (p.grad - q.grad).abs().max().item() <= 2e-3 * gmax, (n_cbams, k)
    sess.close()
