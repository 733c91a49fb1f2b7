"""The fused DS conv's staged epilogue: each consumer warpgroup stages a 32-channel x 64-pixel slice of its output in shared
memory and writes it with one TMA tensor store, which clips whatever falls outside W, H or Cout.  The shapes below put patches
across the right and bottom image edges (one with a store box wholly below the image), Cout across a 32-channel slice and
the output into a channel slice of a larger buffer; every result is checked against the numpy oracle and must repeat bit for
bit.  Outputs TMA cannot describe (a misaligned base, a batch stride that is not a multiple of 4) are declined."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import smaat_oracle as O
from smaat_unet_b200 import _lib, ops
from tests._util import PW_TOL, assert_close, dev

RNG = np.random.default_rng(2468)
SMAAT_E_UNSUPPORTED = -3


def rnd(*shape, lo=-1.0, hi=1.0):
    return RNG.uniform(lo, hi, shape).astype(np.float32)


@pytest.fixture(params=["smem", "regs"])
def ds_impl(request):
    ops.set_dsconv_impl(request.param)
    yield request.param
    ops.set_dsconv_impl("auto")


def _data(B, C, H, W, k, Cout):
    x = rnd(B, C, H, W)
    dw_w, dw_b = rnd(k * C, 1, 3, 3), rnd(k * C)
    pw_w = rnd(Cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    acc = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, dw_b, k), pw_w, None)
    ref = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    return (x, dw_w, dw_b, pw_w, scale, shift), ref


# B, C, H, W, k, Cout
EDGE_CASES = [
    (2, 16, 72, 72, 2, 64),      # PW 16: the fifth patch column is half outside the image
    (2, 16, 100, 48, 2, 64),     # PH 8: the last patch row has 4 of 8 rows inside
    (2, 16, 102, 64, 2, 128),    # PH 4: the last patch row's second half-patch lies wholly below the image
    (2, 32, 40, 64, 2, 40),      # Cout 40: the second 32-channel slice is clipped to 8 channels
    (2, 16, 48, 64, 2, 96),      # N_TILE 128, Cout 96: three slices, the fourth is skipped
    (2, 16, 40, 40, 2, 8),       # Cout 8: one slice, mostly clipped
    (1, 40, 40, 40, 1, 96),      # k = 1 (N_TILE 128 in 3xTF32 keeps the direct stores), PW 16 across the right edge
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", EDGE_CASES)
def test_dsconv_staged_store_edges_match_oracle_and_repeat(case, mode, ds_impl):
    B, C, H, W, k, Cout = case
    (x, dw_w, dw_b, pw_w, scale, shift), ref = _data(B, C, H, W, k, Cout)
    args = (dev(x), dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True)
    y = ops.dsconv(*args, mode=mode)
    y2 = ops.dsconv(*args, mode=mode)
    torch.cuda.synchronize()
    assert y is not None, f"fused kernel refused {case}"
    assert_close(y, ref, PW_TOL[mode], f"dsconv {mode} {case}")
    assert torch.equal(y, y2), "two launches differ"


def _fwd(x, d, y_ptr, y_bstride, Cout, k, mode):
    B, C, H, W = x.shape
    dw_w, dw_b, pw_w, scale, shift = d
    w2d = pw_w.view(Cout, -1)
    hi, lo = ops.split_tf32(w2d) if mode == "tf32x3" else (w2d, None)
    p = ops._ptr
    return _lib.load().smaat_dsconv_fwd(p(x), C, C * H * W, None, 0, 0, p(dw_w), p(dw_b), p(hi), p(lo), p(scale), p(shift), y_ptr,
                                        y_bstride, None, B, H, W, k, Cout, 1, ops.PW_MODES[mode], ops._stream())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cout", [64, 96])
def test_dsconv_writes_a_channel_slice_of_a_larger_buffer(cout, mode, ds_impl):
    """y is channels [c_off, c_off + Cout) of a (B, Ctot, H, W) buffer: y_bstride = Ctot * H * W > Cout * H * W.  The slice
    matches the oracle and every NaN sentinel outside it is untouched."""
    B, C, H, W, k = 3, 16, 40, 72, 2
    c_off, Ctot = 8, cout + 24
    (x, dw_w, dw_b, pw_w, scale, shift), ref = _data(B, C, H, W, k, cout)
    d = tuple(dev(a) for a in (dw_w, dw_b, pw_w, scale, shift))
    outs = []
    for _ in range(2):
        big = torch.full((B, Ctot, H, W), float("nan"), device="cuda")
        rc = _fwd(dev(x), d, big[:, c_off:].data_ptr(), Ctot * H * W, cout, k, mode)
        torch.cuda.synchronize()
        assert rc == 0, _lib.load().smaat_last_error()
        assert_close(big[:, c_off:c_off + cout], ref, PW_TOL[mode], f"channel slice {mode}")
        assert bool(torch.isnan(big[:, :c_off]).all()) and bool(torch.isnan(big[:, c_off + cout:]).all()), "wrote outside the slice"
        outs.append(big[:, c_off:c_off + cout].clone())
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
def test_dsconv_declines_outputs_tma_cannot_store():
    """A y that is not 16-byte aligned, or a batch stride that is not a multiple of 4 floats: SMAAT_E_UNSUPPORTED (the caller
    runs dw3x3 + pw1x1), nothing written."""
    B, C, H, W, k, Cout = 2, 16, 32, 32, 2, 64
    (x, dw_w, dw_b, pw_w, scale, shift), _ = _data(B, C, H, W, k, Cout)
    d = tuple(dev(a) for a in (dw_w, dw_b, pw_w, scale, shift))
    P = Cout * H * W
    big = torch.full((B * P + 64,), float("nan"), device="cuda")
    for mode in ("tf32", "tf32x3"):
        assert _fwd(dev(x), d, big.data_ptr() + 4, P, Cout, k, mode) == SMAAT_E_UNSUPPORTED     # misaligned base
        assert _fwd(dev(x), d, big.data_ptr(), P + 2, Cout, k, mode) == SMAAT_E_UNSUPPORTED     # stride % 4 != 0
        assert _fwd(dev(x), d, big.data_ptr(), P + 4, Cout, k, mode) == 0
    torch.cuda.synchronize()
    assert not bool(torch.isnan(big[:P]).any())


# (N_TILE, k, 3xTF32, A from shared memory) of the instances whose 30 KB input boxes leave no room for a staging buffer: they
# keep the direct stores
DIRECT_STORE = {(128, 1, 1, 0), (64, 1, 1, 1)}


def test_dsconv_instances_stage_their_output_through_tma_stores_without_local_memory():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "dsconv_fused_kernel" in m.group(1) else None
            if name:
                funcs[name] = False
        elif name and "UTMASTG" in line:
            funcs[name] = True
    assert len(funcs) == 32, f"expected 32 dsconv_fused_kernel instances, found {len(funcs)}"
    for n, staged in funcs.items():
        nt, kpl, _pw, x3, a_smem = map(int, re.search(r"ILi(\d+)ELi(\d+)ELi(\d+)ELb(\d)ELb(\d)E", n).groups())
        assert staged == ((nt, kpl, x3, a_smem) not in DIRECT_STORE), f"{n}: TMA store {'present' if staged else 'missing'}"
    usage = subprocess.run([exe, "--dump-resource-usage", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if "dsconv_fused_kernel" in m.group(1):
            seen += 1
            local = re.search(r"LOCAL:(\d+)", m.group(2))
            assert local and int(local.group(1)) == 0, f"{m.group(1)} uses local memory: {m.group(2)}"
    assert seen == len(funcs)
