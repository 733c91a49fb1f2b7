"""The fused DS conv's paired tiles (dsconv_pair_kernel) against the single tile and float64, at the pair's edges.

At Cout <= 64, k = 2 or 4, in tf32 / 3xTF32 with fp32 maps and the register A form, a tile is two vertically adjacent patches
(2 PH rows x PW) that share each chunk's input box and weight chunk, wherever the image has an even number of patch rows
(ceil(H / PH)); an odd number takes the single tile, which would otherwise cover one more patch row.  Each half keeps the
single tile's A layout, accumulator rows, MMA order and epilogue, so every output must be bit for bit what the single tile
computes.  The single tile is reached through the shape rule itself: an image cropped to an odd number of patch rows runs
it, and every output that does not see the crop's bottom edge (rows < Hc - 1, pooled rows < (Hc - 1) // 2, partial pools
of patch rows < PRc - 1) must equal the paired run's.

  A  which kernel runs (torch.profiler, once for the whole module in a fresh process: in one process only the first test
     module that profiles sees kernel events, and not always all of them): the pair at 288^2 and 144^2 with Cout 64 in
     tf32 / 3xTF32, k = 2 and 4; the single tile at an odd number of patch rows, at Cout 128, in bf16 mode, in the
     shared-memory A form and for 22 classes; the pair under every case of B, C and D
  B  y, paired against cropped single, and both against float64: PW 32 and 16, partial W, H = 30 (the last pair's lower
     half partly below the image), k = 2 and 4, tf32 and 3xTF32
  C  the epilogues on the lower half, pair against single: the 1-class OutConv, K-class logits and class map, the max-pool,
     and the CBAM gate on a concat with the partial pools; the BatchNorm statistics against float64 sums of y

Bounds are those of tests/test_gpu_ds_forward_kernels.py (ERR_BOUND "fused" / "fused_stats").
"""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from smaat_unet_b200 import ops
from tests.test_gpu_ds_forward_kernels import ERR_BOUND, _bn_affine, _check, _exact, _gen, _randn, dw_emul, pw_ref

gpu = pytest.mark.gpu
TC_MODES = ("tf32", "tf32x3")
PAIR = "dsconv_pair_kernel"
# (H, W, Hc): Hc crops to an odd number of patch rows (the single tile); PW = 32 unless W says 16
GEOMS = [
    (32, 64, 28),     # PW 32, PH 4: 8 patch rows -> 4 pairs; crop 7
    (32, 52, 28),     # PW 32, partial last column tile
    (30, 64, 26),     # PW 32: the last pair's lower half holds rows 28, 29 only; crop 7 patch rows
    (32, 48, 24),     # PW 16, PH 8: 4 patch rows -> 2 pairs; crop 3
    (48, 40, 40),     # PW 16, partial last column tile; crop 5 patch rows
]
EPILOGUE_GEOMS = [(32, 64, 28), (32, 48, 24), (30, 64, 26)]


def _params(Cin, Cout, k, g):
    K = k * Cin
    w = _randn((K, 1, 3, 3), g, 0.3)
    b = _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    return w, b, pw, sc, sh


def _ds(shape, Cout, k, g, **kw):
    """A call of ops.dsconv on a random (B, C, H, W) input (one fused DS conv launch)."""
    x = _randn(shape, g)
    w, b, pw, sc, sh = _params(shape[1], Cout, k, g)
    return lambda: ops.dsconv(x, w, b, k, pw, sc, sh, True, **kw)


def _smem(fn):
    def run():
        ops.set_dsconv_impl("smem")
        try:
            fn()
        finally:
            ops.set_dsconv_impl("auto")
    return run


def _classify(K, g):
    x = _randn((2, 16, 32, 64), g)
    w, b, pw, sc, sh = _params(16, 64, 2, g)
    ow, ob = _randn((K, 64), g, 0.125), _randn((K,), g, 0.3)
    return lambda: ops.dsconv_classify(x, w, b, 2, pw, sc, sh, True, ow, ob, mode="tf32x3")


def selection_cases():
    """(key, call, fused DS conv launches of the call) of every kernel-selection check below.  ``ran`` runs them in a fresh
    process: in one process only the first test module that profiles sees kernel events, and not always all of them."""
    g = _gen(11)
    cases = []
    for mode in TC_MODES:
        for k in (2, 4):
            for C, S in ((64, 288), (128, 144)):
                cases.append((f"A even {mode} k{k} {C}x{S}", _ds((2, C, S, S), 64, k, g, mode=mode), 1))
            # 28 rows at PW 32: 7 patch rows (odd), the pair would cover 32
            cases.append((f"A odd {mode} k{k}", _ds((2, 16, 28, 64), 64, k, g, mode=mode), 1))
            # Cout 128: N_TILE 128 keeps the single tile
            cases.append((f"A cout128 {mode} k{k}", _ds((2, 16, 32, 64), 128, k, g, mode=mode), 1))
            for H, W, Hc in GEOMS:
                cases.append((f"B {mode} k{k} {H}x{W}", _ds((2, 24, H, W), 40, k, g, mode=mode), 1))
                cases.append((f"B crop {mode} k{k} {H}x{W}", _ds((2, 24, Hc, W), 40, k, g, mode=mode), 1))
            for H, W, _ in EPILOGUE_GEOMS:
                run = _epilogue_case(mode, k, H, W)[0]
                cases.append((f"C {mode} k{k} {H}x{W}", lambda run=run, H=H: run(H), 4))
            cases.append((f"D {mode} k{k}", _stats_case(mode, k)[0], 1))
    cases.append(("A bf16", _ds((2, 16, 32, 64), 64, 2, g, mode="bf16"), 1))
    cases.append(("A smem", _smem(_ds((2, 16, 32, 64), 64, 2, g, mode="tf32x3")), 1))
    # 22 classes: more class weights than a paired tile keeps beside its rings
    cases.append(("A classes22", _classify(22, g), 1))
    cases.append(("A classes21", _classify(21, g), 1))
    return cases


_SELECTION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from tests.test_gpu_dsconv_pairs import selection_cases

cases = selection_cases()
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for key, fn, n in cases:
        fn()
        torch.cuda.synchronize()
ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "dsconv" in e.name),
            key=lambda e: e.time_range.start)
out, i = {}, 0
for key, fn, n in cases:
    out[key] = sorted({e.name for e in ev[i:i + n]})
    i += n
print(json.dumps({"launched": i, "seen": len(ev), "cases": out}))
"""


@pytest.fixture(scope="module")
def ran():
    """key -> the dsconv kernels its call ran, from one profiled run of selection_cases() in a fresh process."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _SELECTION, root], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    # one kernel per fused DS conv call, in order: a missing or extra one would shift every name after it
    assert got["seen"] == got["launched"], f"the profiler saw {got['seen']} dsconv kernels for {got['launched']} calls"
    return got["cases"]


def _pair(ran, key):
    """Whether the call ``key`` ran the paired tile; it must have run some fused DS conv kernel."""
    names = ran[key]
    assert names, f"{key}: no dsconv kernel seen"
    return any(PAIR in n for n in names)


# ============================================================================================================ A: selection
@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("k", (2, 4))
def test_pair_runs_where_the_patch_rows_are_even(mode, k, ran):
    for C, S in ((64, 288), (128, 144)):
        assert _pair(ran, f"A even {mode} k{k} {C}x{S}"), ran[f"A even {mode} k{k} {C}x{S}"]
    assert not _pair(ran, f"A odd {mode} k{k}"), ran[f"A odd {mode} k{k}"]
    assert not _pair(ran, f"A cout128 {mode} k{k}"), ran[f"A cout128 {mode} k{k}"]


@gpu
def test_single_tile_where_the_pair_is_not_built(ran):
    for key in ("A bf16", "A smem", "A classes22"):
        assert not _pair(ran, key), (key, ran[key])
    assert _pair(ran, "A classes21"), ran["A classes21"]


# ======================================================================================================= B: y at the edges
@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("k", (2, 4))
@pytest.mark.parametrize("H,W,Hc", GEOMS)
def test_pair_equals_single_and_float64(mode, k, H, W, Hc, ran):
    g = _gen(100 + H + W + k)
    Cin, Cout = 24, 40
    x = _randn((2, Cin, H, W), g)
    w, b, pw, sc, sh = _params(Cin, Cout, k, g)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    xc = x[:, :, :Hc].contiguous()
    assert _pair(ran, f"B {mode} k{k} {H}x{W}") and not _pair(ran, f"B crop {mode} k{k} {H}x{W}")
    y = ops.dsconv(x, w, b, k, pw, sc, sh, True, mode=mode, w_split=ws)
    yc = ops.dsconv(xc, w, b, k, pw, sc, sh, True, mode=mode, w_split=ws)
    _exact(y[:, :, :Hc - 1], yc[:, :, :Hc - 1], f"pair vs single {mode} k={k} {H}x{W}")
    z = pw_ref(dw_emul(x, w, b, k), pw, mode)
    ref = torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    _check(y, ref, ERR_BOUND["fused"][mode], f"pair {mode} k={k} {H}x{W}")
    zc = pw_ref(dw_emul(xc, w, b, k), pw, mode)
    refc = torch.relu(zc * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))
    _check(yc, refc, ERR_BOUND["fused"][mode], f"single {mode} k={k} {Hc}x{W}")


# =================================================================================================== C: epilogues, stats
def _epilogue_case(mode, k, H, W):
    """run(h): the 1-class OutConv, K-class classify, max-pool and CBAM (gate on a concat + pools) forms of one DS conv on the
    image's first h rows (one fused DS conv launch each); and Cout."""
    g = _gen(200 + H + W + k)
    C0, C1, Cout = 16, 16, 64
    x0, x1 = _randn((2, C0, H, W), g), _randn((2, C1, H, W), g)
    w, b, pw, sc, sh = _params(C0 + C1, Cout, k, g)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    ow1, ob1 = _randn((1, Cout), g, 0.125), _randn((1,), g, 0.3)
    owk, obk = _randn((5, Cout), g, 0.125), _randn((5,), g, 0.3)
    gsc = torch.rand((2, C0), generator=g, device="cuda")
    gsa = torch.rand((2, 1, H, W), generator=g, device="cuda")
    common = (w, b, k, pw, sc, sh, True)

    def run(h):
        a0, a1 = x0[:, :, :h].contiguous(), x1[:, :, :h].contiguous()
        sa = gsa[:, :, :h].contiguous()
        out = {"oc": ops.dsconv(a0, *common, x1=a1, mode=mode, w_split=ws, outconv=(ow1, ob1))}
        out["cls"], out["logits"] = ops.dsconv_classify(a0, *common, owk, obk, x1=a1, mode=mode, w_split=ws, want_logits=True)
        out["y_mp"], out["mp"] = ops.dsconv_maxpool(a0, *common, x1=a1, mode=mode, w_split=ws)
        out["y_cbam"], out["psum"], out["pmax"], out["pooled"] = ops.dsconv_cbam(a0, *common, x1=a1, mode=mode, w_split=ws,
                                                                                 gate=(gsc, sa), pools=True)
        return out

    return run, Cout


@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("k", (2, 4))
@pytest.mark.parametrize("H,W,Hc", EPILOGUE_GEOMS)
def test_pair_epilogues_equal_single(mode, k, H, W, Hc, ran):
    run, Cout = _epilogue_case(mode, k, H, W)
    assert _pair(ran, f"C {mode} k{k} {H}x{W}")
    full, crop = run(H), run(Hc)
    for key in ("oc", "logits", "y_mp", "y_cbam"):
        _exact(full[key][:, :, :Hc - 1], crop[key][:, :, :Hc - 1], f"{key} {mode} k={k} {H}x{W}")
    _exact(full["cls"][:, :Hc - 1], crop["cls"][:, :Hc - 1], f"classes {mode} k={k} {H}x{W}")
    hp = (Hc - 1) // 2
    for key in ("mp", "pooled"):
        _exact(full[key][:, :, :hp], crop[key][:, :, :hp], f"{key} {mode} k={k} {H}x{W}")
    _exact(full["mp"], F.max_pool2d(full["y_mp"], 2), f"max-pool of y {mode} k={k} {H}x{W}")
    _exact(full["pooled"], F.max_pool2d(full["y_cbam"], 2), f"CBAM max-pool of y {mode} k={k} {H}x{W}")
    _exact(full["cls"], full["logits"].argmax(dim=1), f"class map {mode} k={k} {H}x{W}")
    # partial pools: (B, patch rows, column tiles, 2 half-patches, Cout)
    pw_ = 16 if W in (48, 40) else 32
    tx, ph = -(-W // pw_), 128 // pw_
    pr, prc = -(-H // ph), -(-Hc // ph)
    for key in ("psum", "pmax"):
        a = full[key].view(2, pr, tx, 2, Cout)[:, :prc - 1]
        c = crop[key].view(2, prc, tx, 2, Cout)[:, :prc - 1]
        _exact(a, c, f"{key} {mode} k={k} {H}x{W}")
    # the lower half's last partial pools against the stored y they cover (-inf for a half-patch wholly below the image)
    y = full["y_cbam"]
    for wg in (0, 1):
        r0 = (pr - 1) * ph + wg * (ph // 2)
        got = full["pmax"].view(2, pr, tx, 2, Cout)[:, -1, -1, wg]
        want = y[:, :, r0:r0 + ph // 2, (tx - 1) * pw_:].amax(dim=(2, 3)) if r0 < H else torch.full_like(got, -float("inf"))
        _exact(got, want, f"last pmax wg={wg} {mode} k={k} {H}x{W}")


def _stats_case(mode, k):
    """A training-mode call with BatchNorm statistics (one fused DS conv launch), and its operands."""
    g = _gen(300 + k)
    x = _randn((2, 32, 30, 64), g)
    w, b, pw, _, _ = _params(32, 64, k, g)
    pb = _randn((64,), g, 0.3)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    run = lambda: ops.dsconv(x, w, b, k, pw, None, pb, False, mode=mode, w_split=ws, stats=ops.new_stats(64, x.device))
    return run, x, w, b, pw, pb, ws


@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("k", (2, 4))
def test_pair_batch_statistics(mode, k, ran):
    _, x, w, b, pw, pb, ws = _stats_case(mode, k)
    assert _pair(ran, f"D {mode} k{k}")
    stats = ops.new_stats(64, x.device)
    y = ops.dsconv(x, w, b, k, pw, None, pb, False, mode=mode, w_split=ws, stats=stats)
    zb = pw_ref(dw_emul(x, w, b, k), pw, mode) + pb.double().view(1, -1, 1, 1)
    _check(y, zb, ERR_BOUND["fused"][mode], f"pair train y {mode} k={k}")
    _check(stats[:64], zb.sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"][mode], f"pair stats sum {mode} k={k}")
    _check(stats[64:], (zb * zb).sum(dim=(0, 2, 3)), ERR_BOUND["fused_stats"][mode], f"pair stats sum of squares {mode} k={k}")
