"""The pipelined wgmma main loops of the fused DS conv and pw1x1_tc: chunk i's MMAs stay in flight while chunk i - 1 retires
and hands its shared-memory stages back.  The shapes below put the late release, the unroll-by-2 odd tail and the tile
boundaries where they are easiest to get wrong; every result is checked against the numpy oracle and must repeat bit for bit.

The CPU test reads the built library: every instance of the two kernels waits with one MMA group still in flight and uses no
local memory (no spills from the second register-A fragment set)."""
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

RNG = np.random.default_rng(4321)


def rnd(*shape, lo=-1.0, hi=1.0):
    return RNG.uniform(lo, hi, shape).astype(np.float32)


@pytest.fixture(params=["smem", "regs"])
def ds_impl(request):
    ops.set_dsconv_impl(request.param)
    yield request.param
    ops.set_dsconv_impl("auto")


# B, C0, C1, H, W, k, Cout.  k = 2: a chunk is 16 input channels
DS_CASES = [
    (8, 16, 0, 128, 128, 2, 64),       # one chunk per tile, 1024 tiles: 7-8 tiles per CTA
    (8, 16, 0, 128, 64, 2, 128),       # ... N_TILE 128
    (2, 32, 0, 32, 64, 2, 64),         # 2 chunks
    (2, 48, 0, 32, 64, 2, 128),        # 3 chunks (odd tail)
    (2, 80, 0, 48, 48, 2, 64),         # 5 chunks, 16-wide patches
    (1, 40, 0, 32, 32, 1, 96),         # k = 1: 32 channels per chunk, 2 chunks with a ragged channel tail
    (1, 256, 256, 16, 32, 2, 256),     # concat, K = 1024, two passes of 128 over each patch
    (1, 256, 256, 16, 32, 2, 512),     # ... four passes
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("case", DS_CASES)
def test_dsconv_pipelined_matches_oracle_and_repeats(case, mode, ds_impl):
    B, C0, C1, H, W, k, Cout = case
    C = C0 + C1
    x = rnd(B, C, H, W)
    dw_w, dw_b = rnd(k * C, 1, 3, 3), rnd(k * C)
    pw_w = rnd(Cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    acc = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, dw_b, k), pw_w, None)
    ref = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    x0 = dev(x[:, :C0])
    x1 = dev(x[:, C0:]) if C1 else None
    args = (x0, dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True)
    y = ops.dsconv(*args, x1=x1, mode=mode)
    y2 = ops.dsconv(*args, x1=x1, mode=mode)
    torch.cuda.synchronize()
    assert y is not None, f"fused kernel refused {case}"
    assert_close(y, ref, PW_TOL[mode], f"dsconv {mode} {case}")
    assert torch.equal(y, y2), "two launches differ"


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cout", [64, 128])
def test_dsconv_statistics_on_one_chunk_tiles(cout, mode, ds_impl):
    B, C, H, W, k = 4, 16, 64, 96, 2
    x = rnd(B, C, H, W)
    dw_w = rnd(k * C, 1, 3, 3)
    pw_w = rnd(cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    pre = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, None, k), pw_w, None)
    outs = []
    for _ in range(2):
        st = torch.zeros(2 * cout, device="cuda", dtype=torch.float64)
        y = ops.dsconv(dev(x), dev(dw_w), None, k, dev(pw_w), None, None, False, mode=mode, stats=st)
        torch.cuda.synchronize()
        assert_close(y, pre, PW_TOL[mode], f"dsconv+stats {mode}")
        assert_close(st[:cout], pre.sum(axis=(0, 2, 3)), 2e-3 if mode == "tf32" else 1e-4, "channel sums")
        assert_close(st[cout:], (pre ** 2).sum(axis=(0, 2, 3)), 2e-3 if mode == "tf32" else 1e-4, "channel sums of squares")
        outs.append(y)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tf32", "tf32x3"])
@pytest.mark.parametrize("cout", [64, 128])
def test_dsconv_outconv_on_one_chunk_tiles(cout, mode, ds_impl):
    B, C, H, W, k = 4, 16, 64, 96, 2
    x = rnd(B, C, H, W)
    dw_w, dw_b = rnd(k * C, 1, 3, 3), rnd(k * C)
    pw_w = rnd(cout, k * C, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(cout, lo=0.5, hi=1.5), rnd(cout)
    ow, ob = rnd(1, cout, 1, 1), rnd(1)
    acc = O.pointwise1x1(O.depthwise3x3(x.astype(np.float64), dw_w, dw_b, k), pw_w, None)
    ref = O.pointwise1x1(np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0), ow, ob)
    args = (dev(x), dev(dw_w), dev(dw_b), k, dev(pw_w), dev(scale), dev(shift), True)
    y = ops.dsconv(*args, mode=mode, outconv=(dev(ow), dev(ob)))
    y2 = ops.dsconv(*args, mode=mode, outconv=(dev(ow), dev(ob)))
    torch.cuda.synchronize()
    assert_close(y, ref, PW_TOL[mode], f"dsconv+outconv {mode}")
    assert torch.equal(y, y2)


# B, K, Cout, H, W: chunk counts 1, 2, 3, 64 (K / 32); 4 x 72 x 2 = 576 tiles, not a multiple of the SM count
PW_CASES = [
    (2, 32, 128, 32, 32),
    (2, 64, 64, 32, 32),
    (2, 96, 256, 16, 32),
    (1, 2048, 512, 16, 16),
    (4, 64, 256, 96, 96),
]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
@pytest.mark.parametrize("case", PW_CASES)
def test_pw1x1_chunk_counts_match_oracle_and_repeat(case, mode):
    B, K, Cout, H, W = case
    x, w = rnd(B, K, H, W), rnd(Cout, K, 1, 1, lo=-0.2, hi=0.2)
    scale, shift = rnd(Cout, lo=0.5, hi=1.5), rnd(Cout)
    acc = O.pointwise1x1(x.astype(np.float64), w, None)
    ref = np.maximum(acc * scale[None, :, None, None] + shift[None, :, None, None], 0)
    y = ops.pw1x1(dev(x), dev(w), dev(scale), dev(shift), True, mode=mode)
    y2 = ops.pw1x1(dev(x), dev(w), dev(scale), dev(shift), True, mode=mode)
    torch.cuda.synchronize()
    assert_close(y, ref, PW_TOL[mode], f"pw1x1 {mode} {case}")
    assert torch.equal(y, y2)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["fp32", "tf32", "tf32x3"])
def test_pw1x1_statistics_repeat(mode):
    B, K, Cout, H, W = 3, 96, 192, 40, 40
    x, w, bias = rnd(B, K, H, W), rnd(Cout, K, 1, 1, lo=-0.3, hi=0.3), rnd(Cout)
    pre = O.pointwise1x1(x.astype(np.float64), w, bias)
    outs = []
    for _ in range(2):
        st = torch.zeros(2 * Cout, device="cuda", dtype=torch.float64)
        y = ops.pw1x1(dev(x), dev(w), None, dev(bias), False, mode=mode, stats=st)
        torch.cuda.synchronize()
        assert_close(y, pre, PW_TOL[mode], f"pw1x1+stats {mode}")
        tol = 2e-3 if mode == "tf32" else 1e-4
        assert_close(st[:Cout], pre.sum(axis=(0, 2, 3)), tol, "channel sums")
        assert_close(st[Cout:], (pre ** 2).sum(axis=(0, 2, 3)), tol, "channel sums of squares")
        outs.append(y)
    assert torch.equal(outs[0], outs[1])


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(_lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    return exe


KERNELS = re.compile(r"(dsconv_fused_kernel|pw1x1_tc_kernel)")


def test_fused_kernel_keeps_one_group_in_flight_and_tensor_core_kernels_do_not_spill():
    exe = _cuobjdump()
    sass = subprocess.run([exe, "-sass", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs = {}
    name = None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if KERNELS.search(m.group(1)) else None
            if name:
                funcs[name] = False
        elif name and "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
            funcs[name] = True
    assert len(funcs) >= 36, f"expected every dsconv_fused_kernel / pw1x1_tc_kernel instance, found {len(funcs)}"
    serial = [n for n, ok in funcs.items() if not ok]
    assert not serial, f"MMA waits drain the pipe in: {serial}"

    usage = subprocess.run([exe, "--dump-resource-usage", _lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if KERNELS.search(m.group(1)):
            seen += 1
            local = re.search(r"LOCAL:(\d+)", m.group(2))
            assert local and int(local.group(1)) == 0, f"{m.group(1)} uses local memory: {m.group(2)}"
    assert seen == len(funcs)
