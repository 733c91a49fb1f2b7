"""CPU-side checks of kernels_per_layer = 4 in the fused DS conv: which shapes smaat_dsconv_eligible takes at k = 4 (host
logic only, fake aligned addresses that are never dereferenced), and, where the library is built, that its eight k = 4
instances exist, use no local memory and write their output with TMA tensor stores."""
import os
import re
import shutil
import subprocess

import pytest

import smaat_unet_b200 as S

A = 1 << 20      # fake, 16-byte aligned address


def _eligible(lib, k, C0, C1, S_, Cout, stats=0):
    return lib.smaat_dsconv_eligible2(A, C0, C0 * S_ * S_, A if C1 else None, C1, C1 * S_ * S_, A, S_, S_, k, Cout, stats)


# (C0, C1, S, Cout) of SmaAt_UNet(12, 1, kernels_per_layer=4)'s DS convs that the fused kernel takes at 288 x 288 (the 36 x 36
# and 18 x 18 ones run dw3x3 + pw1x1 at every k)
FUSED = [(12, 0, 288, 64), (64, 0, 288, 64), (64, 0, 144, 128), (128, 0, 144, 128), (128, 0, 72, 256), (256, 0, 72, 256),
         (256, 256, 72, 256), (256, 0, 72, 128), (128, 128, 144, 128), (128, 0, 144, 64), (64, 64, 288, 64)]


def test_eligibility_at_k4():
    lib = S._lib.load()
    for C0, C1, S_, Cout in FUSED:
        assert _eligible(lib, 4, C0, C1, S_, Cout) == 1, (C0, C1, S_, Cout)
        assert _eligible(lib, 2, C0, C1, S_, Cout) == 1
        assert _eligible(lib, 3, C0, C1, S_, Cout) == 0, "k = 3 stays unfused"
    for C0, C1, S_, Cout in [(512, 0, 36, 512), (512, 0, 18, 512), (512, 512, 36, 512)]:
        assert _eligible(lib, 4, C0, C1, S_, Cout) == _eligible(lib, 2, C0, C1, S_, Cout) == 0
    # statistics: one pass of at most 128 channels, as at k = 2
    assert _eligible(lib, 4, 64, 0, 288, 64, 1) == 1 and _eligible(lib, 4, 128, 0, 72, 256, 1) == 0
    # a virtual concat needs whole chunks of x0: 8 channels at k = 4 (16 at k = 2)
    assert _eligible(lib, 4, 8, 8, 64, 64) == 1 and _eligible(lib, 2, 8, 8, 64, 64) == 0
    assert _eligible(lib, 4, 12, 4, 64, 64) == 0 and _eligible(lib, 4, 20, 12, 64, 64) == 0
    assert _eligible(lib, 4, 12, 0, 64, 64) == 1 and _eligible(lib, 4, 3, 0, 64, 64) == 1


def test_shared_memory_a_form_keeps_k4_unfused():
    lib = S._lib.load()
    assert lib.smaat_set_dsconv_impl(1) == 0
    try:
        assert _eligible(lib, 4, 64, 0, 288, 64) == 0 and _eligible(lib, 2, 64, 0, 288, 64) == 1
        assert lib.smaat_dsconv_cbam_eligible(A, 64, 64 * 288 * 288, None, 0, 0, A, 288, 288, 4, 64, 2, 1, 0) == 0
        assert lib.smaat_dsconv_classify_eligible(A, 64, 64 * 288 * 288, None, 0, 0, A, 288, 288, 4, 64, 8, 2) == 0
    finally:
        assert lib.smaat_set_dsconv_impl(0) == 0
    assert _eligible(lib, 4, 64, 0, 288, 64) == 1
    assert lib.smaat_set_dsconv_impl(2) == 0
    try:
        assert _eligible(lib, 4, 64, 0, 288, 64) == 1
    finally:
        assert lib.smaat_set_dsconv_impl(0) == 0


def test_k4_epilogues_are_offered():
    lib = S._lib.load()
    for mode in (1, 2):     # tf32, tf32x3
        # the gate on load at every fused shape, the pools where the instance stages its output
        assert lib.smaat_dsconv_cbam_eligible(A, 64, 64 * 288 * 288, A, 64, 64 * 288 * 288, A, 288, 288, 4, 64, mode, 1, 0) == 1
        assert lib.smaat_dsconv_cbam_eligible(A, 64, 64 * 288 * 288, None, 0, 0, A, 288, 288, 4, 64, mode, 0, 1) == 1
        for K in (1, 8, 21):
            assert lib.smaat_dsconv_classify_eligible(A, 64, 64 * 288 * 288, None, 0, 0, A, 288, 288, 4, 64, K, mode) == 1
            assert lib.smaat_dsconv_classify_eligible(A, 128, 128 * 144 * 144, None, 0, 0, A, 144, 144, 4, 128, K, mode) == 1


def test_k4_instances_stage_their_output_through_tma_stores_without_local_memory():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(S._lib.LIB_PATH):
        pytest.skip("needs cuobjdump and the built library")
    sass = subprocess.run([exe, "-sass", S._lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if "dsconv_kpl4_kernel" in m.group(1) else None
            if name:
                funcs[name] = False
        elif name and "UTMASTG" in line:
            funcs[name] = True
    got = sorted(tuple(map(int, re.search(r"ILi(\d+)ELi(\d+)ELb(\d)E", n).groups())) for n in funcs)
    assert got == sorted((nt, pw, x3) for nt in (64, 128) for pw in (16, 32) for x3 in (0, 1)), got
    assert all(funcs.values()), f"TMA store missing: {[n for n, s in funcs.items() if not s]}"
    usage = subprocess.run([exe, "--dump-resource-usage", S._lib.LIB_PATH], check=True, capture_output=True, text=True).stdout
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if "dsconv_kpl4_kernel" in m.group(1):
            seen += 1
            local = re.search(r"LOCAL:(\d+)", m.group(2))
            assert local and int(local.group(1)) == 0, f"{m.group(1)} uses local memory: {m.group(2)}"
    assert seen == 8
