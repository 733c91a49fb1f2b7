"""The fused DS conv's wide tiles (dsconv_wide_kernel) against the two-pass route and float64.

At 128 < Cout <= 256, k = 2, in tf32 / 3xTF32 with fp32 maps and the register A form, a tile is one patch and both 128-channel
halves: each chunk's input box and depthwise stencil are computed once and feed both halves' accumulators from the same A
fragments.  Each accumulator sees the k-steps of a single 128-channel pass in that pass's order, so every output must be bit
for bit what the two passes compute.  ``ops.set_dsconv_wide(False)`` selects the two passes, which take Cout a multiple of
128 only; Cout 136 and 200 (a partial second half) are compared against the two passes at Cout 256 with the same leading
weight rows, whose first channels are the same sums.

  A  which kernel runs (torch.profiler, in a fresh process: in one process only the first test module that profiles sees
     kernel events): the wide tile at bench.py's three 256-channel layers (72^2) in tf32 / 3xTF32; the
     two passes with the switch off, at Cout 384 / 512, in bf16 mode and in the shared-memory A form
  B  y, wide against two-pass and both against float64: Cout 256, 136, 200; PW 32 and 16, partial W and H tiles, the concat
     input; tf32 and 3xTF32
  C  the epilogues: up2.0's CBAM gate on load (concat, 72^2), the max-pool (against max_pool2d of the stored y) and the CBAM
     partial pools, wide against two-pass
  D  batch statistics stay where a kernel has them: Cout <= 128 (a request above is declined, not an error)

Bounds are those of tests/test_gpu_ds_forward_kernels.py (ERR_BOUND "fused").
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
WIDE = "dsconv_wide_kernel"
TWO_PASS = "dsconv_fused_kernel"


def _params(Cin, Cout, k, g):
    K = k * Cin
    w = _randn((K, 1, 3, 3), g, 0.3)
    b = _randn((K,), g, 0.1)
    pw = _randn((Cout, K), g, K ** -0.5)
    sc, sh = _bn_affine(Cout, g)
    return w, b, pw, sc, sh


def _two_pass(fn):
    ops.set_dsconv_wide(False)
    try:
        return fn()
    finally:
        ops.set_dsconv_wide(True)


def _ref(x, w, b, k, pw, sc, sh, mode):
    z = pw_ref(dw_emul(x, w, b, k), pw, mode)
    return torch.relu(z * sc.double().view(1, -1, 1, 1) + sh.double().view(1, -1, 1, 1))


# ============================================================================================================ A: selection
_SELECTION = r"""
import json, sys
import torch
sys.path.insert(0, sys.argv[1])
from smaat_unet_b200 import ops


def kernels(fn):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sorted({e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "dsconv" in e.name})


g = torch.Generator(device="cuda").manual_seed(21)
rnd = lambda *s: torch.randn(s, generator=g, device="cuda")
out = {}
for mode in ("tf32", "tf32x3"):
    for C0, C1 in ((128, 0), (256, 0), (256, 256)):          # down2.0, down2.1, up2.0 (concat) at 72^2
        x0, x1 = rnd(2, C0, 72, 72), (rnd(2, C1, 72, 72) if C1 else None)
        w, b, pw = rnd(2 * (C0 + C1), 1, 3, 3), rnd(2 * (C0 + C1)), rnd(256, 2 * (C0 + C1)) * 0.05
        run = lambda: ops.dsconv(x0, w, b, 2, pw, None, None, True, x1=x1, mode=mode)
        out[f"wide {mode} {C0}+{C1}"] = kernels(run)
        ops.set_dsconv_wide(False)
        out[f"two-pass {mode} {C0}+{C1}"] = kernels(run)
        ops.set_dsconv_wide(True)
x = rnd(2, 32, 32, 64)
w, b = rnd(64, 1, 3, 3), rnd(64)
for Cout in (384, 512):
    pw = rnd(Cout, 64) * 0.1
    out[f"Cout {Cout}"] = kernels(lambda: ops.dsconv(x, w, b, 2, pw, None, None, True, mode="tf32x3"))
pw = rnd(256, 64) * 0.1
out["bf16"] = kernels(lambda: ops.dsconv(x, w, b, 2, pw, None, None, True, mode="bf16"))
ops.set_dsconv_impl("smem")
out["smem"] = kernels(lambda: ops.dsconv(x, w, b, 2, pw, None, None, True, mode="tf32x3"))
print(json.dumps(out))
"""


@gpu
def test_which_kernel_runs():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _SELECTION, root], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    for key, names in got.items():
        assert names, (key, got)
        wide = any(WIDE in n for n in names)
        assert wide == key.startswith("wide "), (key, names)
        if key.startswith("wide "):
            assert not any(TWO_PASS in n for n in names), (key, names)
        if key.startswith("two-pass "):
            assert any(TWO_PASS in n for n in names), (key, names)


@gpu
def test_cout_off_a_multiple_of_128_only_as_wide_tiles():
    """Cout not a multiple of 128 is the wide tile's alone: declined with the switch off, and in bf16 mode."""
    g = _gen(22)
    x = _randn((2, 32, 32, 64), g)
    w, b, pw, sc, sh = _params(32, 200, 2, g)
    assert ops.dsconv_takes(x, None, pw, 2, mode="tf32x3")
    assert not _two_pass(lambda: ops.dsconv_takes(x, None, pw, 2, mode="tf32x3"))
    assert not ops.dsconv_takes(x, None, pw, 2, mode="bf16")


# ======================================================================================================= B: y at the edges
# (C0, C1, H, W): PW 32 unless W says 16
GEOMS = [
    (24, 0, 32, 64),      # PW 32, PH 4
    (24, 0, 30, 52),      # PW 32, partial last row and column tiles
    (16, 16, 32, 64),     # concat
    (24, 0, 40, 40),      # PW 16, PH 8
    (16, 16, 36, 40),     # PW 16, concat, partial row tile
]


@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("Cout", (256, 136, 200))
@pytest.mark.parametrize("C0,C1,H,W", GEOMS)
def test_wide_equals_two_pass_and_float64(mode, Cout, C0, C1, H, W):
    g = _gen(100 + Cout + H + W + C1)
    k = 2
    x0 = _randn((2, C0, H, W), g)
    x1 = _randn((2, C1, H, W), g) if C1 else None
    w, b, pw, sc, sh = _params(C0 + C1, 256, k, g)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    # the two passes at Cout 256; the wide tile at Cout on the leading rows
    y2 = _two_pass(lambda: ops.dsconv(x0, w, b, k, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws))
    pwc, scc, shc = pw[:Cout].contiguous(), sc[:Cout].contiguous(), sh[:Cout].contiguous()
    wsc = ops.split_tf32(pwc) if mode == "tf32x3" else None
    y = ops.dsconv(x0, w, b, k, pwc, scc, shc, True, x1=x1, mode=mode, w_split=wsc)
    _exact(y, y2[:, :Cout], f"wide vs two-pass {mode} Cout={Cout} {C0}+{C1} {H}x{W}")
    x = torch.cat([x0, x1], dim=1) if C1 else x0
    _check(y, _ref(x, w, b, k, pwc, scc, shc, mode), ERR_BOUND["fused"][mode], f"wide {mode} Cout={Cout} {H}x{W}")
    _check(y2, _ref(x, w, b, k, pw, sc, sh, mode), ERR_BOUND["fused"][mode], f"two-pass {mode} {H}x{W}")


# =========================================================================================================== C: epilogues
@gpu
@pytest.mark.parametrize("mode", TC_MODES)
def test_wide_gate_on_load_at_up2(mode):
    """up2.0: C256 + 256 -> 256 at 72^2 with the CBAM gate applied on load, wide against two-pass and float64."""
    g = _gen(31)
    C0 = C1 = 256
    x0, x1 = _randn((2, C0, 72, 72), g), _randn((2, C1, 72, 72), g)
    w, b, pw, sc, sh = _params(C0 + C1, 256, 2, g)
    ws = ops.split_tf32(pw) if mode == "tf32x3" else None
    gsc = torch.rand((2, C0), generator=g, device="cuda")
    gsa = torch.rand((2, 1, 72, 72), generator=g, device="cuda")
    run = lambda: ops.dsconv_cbam(x0, w, b, 2, pw, sc, sh, True, x1=x1, mode=mode, w_split=ws, gate=(gsc, gsa))
    y = run()
    _exact(y, _two_pass(run), f"gated wide vs two-pass {mode}")
    xg = torch.cat([(x0 * gsc.view(2, C0, 1, 1)) * gsa, x1], dim=1)
    _check(y, _ref(xg, w, b, 2, pw, sc, sh, mode), ERR_BOUND["fused"][mode], f"gated wide {mode}")


@gpu
@pytest.mark.parametrize("mode", TC_MODES)
@pytest.mark.parametrize("Cout", (256, 200))
@pytest.mark.parametrize("H,W", [(72, 72), (30, 52), (36, 40)])
def test_wide_maxpool_and_pools(mode, Cout, H, W):
    g = _gen(400 + Cout + H + W)
    C0 = 32
    x0 = _randn((2, C0, H, W), g)
    w, b, pw, sc, sh = _params(C0, 256, 2, g)
    gsc = torch.rand((2, C0), generator=g, device="cuda")
    gsa = torch.rand((2, 1, H, W), generator=g, device="cuda")

    def run(n):
        p, s, h = pw[:n].contiguous(), sc[:n].contiguous(), sh[:n].contiguous()
        ws = ops.split_tf32(p) if mode == "tf32x3" else None
        common = (w, b, 2, p, s, h, True)
        out = {}
        out["y_mp"], out["mp"] = ops.dsconv_maxpool(x0, *common, mode=mode, w_split=ws)
        out["y_cbam"], out["psum"], out["pmax"], out["pooled"] = ops.dsconv_cbam(x0, *common, mode=mode, w_split=ws, gate=(gsc, gsa),
                                                                                 pools=True)
        return out

    wide, two = run(Cout), _two_pass(lambda: run(256))
    what = f"{mode} Cout={Cout} {H}x{W}"
    for key in ("y_mp", "mp", "y_cbam", "pooled"):
        _exact(wide[key], two[key][:, :Cout], f"{key} wide vs two-pass {what}")
    for key in ("psum", "pmax"):
        _exact(wide[key], two[key][:, :, :Cout], f"{key} wide vs two-pass {what}")
    _exact(wide["mp"], F.max_pool2d(wide["y_mp"], 2), f"max-pool of y {what}")
    _exact(wide["pooled"], F.max_pool2d(wide["y_cbam"], 2), f"CBAM max-pool of y {what}")


# =================================================================================================== D: batch statistics
@gpu
def test_batch_statistics_above_128_channels_are_declined():
    """Batch statistics are taken by the fused kernel up to Cout 128; above it (wide tile or two passes) the request is
    declined, and DepthwiseSeparableConv.run(stats=...) falls back to dw3x3 + pw1x1 with the same sums."""
    g = _gen(41)
    x = _randn((2, 32, 32, 64), g)
    for Cout in (136, 256):
        w, b, pw, sc, sh = _params(32, Cout, 2, g)
        assert ops.dsconv_takes(x, None, pw, 2, mode="tf32x3")
        assert not ops.dsconv_takes(x, None, pw, 2, mode="tf32x3", stats=True)
        assert ops.dsconv(x, w, b, 2, pw, None, sh, False, mode="tf32x3", stats=ops.new_stats(Cout, x.device)) is None
