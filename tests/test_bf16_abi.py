"""CPU-side checks of the bf16 arithmetic mode (SMAAT_PW_BF16 = 3): the Python mode table, smaat_pack_bf16's argument checks,
which fused DS conv requests the mode-taking eligibility tests accept in bf16 (host logic only, fake aligned addresses that
are never dereferenced), that the weight-gradient entry points still refuse the mode, which weight form the ops helper gives
each mode, and, where the library is built, that the bf16 instances exist, keep one MMA group in flight, stage their output
through TMA stores where the tf32 ones do, and use no local memory."""
import functools
import os
import re
import shutil
import subprocess
import sys

import pytest

import smaat_unet_b200 as S
from smaat_unet_b200 import ops

A = 1 << 20      # fake, 16-byte aligned address
BADARG = -1


def test_mode_table_and_default():
    assert ops.PW_MODES == {"fp32": 0, "tf32": 1, "tf32x3": 2, "bf16": 3}
    old = ops.get_pointwise_mode()
    try:
        ops.set_pointwise_mode("bf16")
        assert ops.get_pointwise_mode() == "bf16"
        with pytest.raises(ValueError):
            ops.set_pointwise_mode("fp16")
        assert ops.get_pointwise_mode() == "bf16"
    finally:
        ops.set_pointwise_mode(old)


def _mode_in_fresh_process(env_value):
    env = dict(os.environ, SMAAT_PW_MODE=env_value)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return subprocess.run([sys.executable, "-c", "import smaat_unet_b200 as S; print(S.get_pointwise_mode())"], cwd=root, env=env,
                          capture_output=True, text=True)


def test_environment_presets_bf16_and_the_default_stays_tf32x3():
    r = _mode_in_fresh_process("bf16")
    assert r.returncode == 0 and r.stdout.strip() == "bf16", r.stderr
    env = {k: v for k, v in os.environ.items() if k != "SMAAT_PW_MODE"}
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", "import smaat_unet_b200 as S; print(S.get_pointwise_mode())"], cwd=root, env=env,
                       capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.strip() == "tf32x3", r.stderr
    assert _mode_in_fresh_process("fp16").returncode != 0


def test_pack_bf16_refuses_bad_arguments():
    lib = S._lib.load()
    assert lib.smaat_pack_bf16(None, A, 4, 40, 64, None) == BADARG
    assert lib.smaat_pack_bf16(A, None, 4, 40, 64, None) == BADARG
    assert lib.smaat_pack_bf16(A, A, 0, 40, 64, None) == BADARG
    assert lib.smaat_pack_bf16(A, A, 4, 0, 32, None) == BADARG
    for cols_out in (40, 32, 96, 63):          # cols_out must be cols rounded up to 32
        assert lib.smaat_pack_bf16(A, A, 4, 40, cols_out, None) == BADARG, cols_out
    assert lib.smaat_pack_bf16(A, A + 2, 4, 40, 64, None) == BADARG      # 4-byte aligned output


def _cbam(lib, k, C0, C1, S_, Cout, mode, gate=0, pools=0):
    return lib.smaat_dsconv_cbam_eligible(A, C0, C0 * S_ * S_, A if C1 else None, C1, C1 * S_ * S_, A, S_, S_, k, Cout, mode, gate, pools)


def _classify(lib, k, C0, S_, Cout, K, mode):
    return lib.smaat_dsconv_classify_eligible(A, C0, C0 * S_ * S_, None, 0, 0, A, S_, S_, k, Cout, K, mode)


# (C0, C1, S, Cout) of the DS convs the fused kernel takes in SmaAt_UNet(12, 1)'s 288 x 288 network
FUSED = [(12, 0, 288, 64), (64, 0, 288, 64), (64, 0, 144, 128), (128, 0, 144, 128), (128, 0, 72, 256), (256, 0, 72, 256),
         (256, 256, 72, 256), (256, 0, 72, 128), (128, 128, 144, 128), (128, 0, 144, 64), (64, 64, 288, 64)]


def test_mode_taking_eligibility_answers_for_bf16():
    lib = S._lib.load()
    for k in (1, 2, 4):
        for C0, C1, S_, Cout in FUSED:
            if k == 1 and C1 and C0 % 32:
                continue
            assert _cbam(lib, k, C0, C1, S_, Cout, 3, gate=1) == _cbam(lib, k, C0, C1, S_, Cout, 1, gate=1) == 1, (k, C0, C1, S_, Cout)
        # the pools where the instance stages its output: bf16's half-size B stages leave at least tf32's room for staging
        for C0, C1, S_, Cout in FUSED:
            if _cbam(lib, k, C0, C1, S_, Cout, 1, pools=1):
                assert _cbam(lib, k, C0, C1, S_, Cout, 3, pools=1) == 1, (k, C0, S_, Cout)
        for K in (1, 8, 21, 22):
            assert _classify(lib, k, 64, 288, 64, K, 3) == 1
            assert _classify(lib, k, 128, 144, 128, K, 3) == 1
        assert _classify(lib, k, 64, 288, 64, 33, 3) == 0
    # the CUDA-core mode has no fused kernel, unknown modes none either
    assert _cbam(lib, 2, 64, 0, 288, 64, 0) == 0 and _cbam(lib, 2, 64, 0, 288, 64, 4) == 0
    assert _classify(lib, 2, 64, 288, 64, 8, 0) == 0 and _classify(lib, 2, 64, 288, 64, 8, 4) == 0
    # shapes the fused kernel declines stay declined
    assert _cbam(lib, 2, 512, 0, 36, 512, 3) == 0 and _cbam(lib, 3, 64, 0, 288, 64, 3) == 0


def test_bf16_has_the_register_form_only():
    lib = S._lib.load()
    assert lib.smaat_set_dsconv_impl(1) == 0
    try:
        assert _cbam(lib, 2, 64, 0, 288, 64, 3) == 0 and _cbam(lib, 2, 64, 0, 288, 64, 2) == 1
        assert _classify(lib, 2, 64, 288, 64, 8, 3) == 0 and _classify(lib, 2, 64, 288, 64, 8, 1) == 1
    finally:
        assert lib.smaat_set_dsconv_impl(0) == 0
    assert _cbam(lib, 2, 64, 0, 288, 64, 3) == 1


def test_weight_gradient_entry_points_refuse_bf16():
    lib = S._lib.load()
    assert lib.smaat_pw1x1_bwd_weight_tc(A, A, A, A, 2, 64, 64, 1024, 3, None) == BADARG
    assert lib.smaat_conv3x3_bwd_weight(A, A, 64, 64 * 1024, None, 0, 0, A, 2, 32, 32, 64, 3, None) == BADARG
    assert ops.wgrad_mode(3) == 1 and [ops.wgrad_mode(m) for m in (0, 1, 2)] == [0, 1, 2]


def test_weight_operands_give_each_mode_its_form(monkeypatch):
    calls = []
    monkeypatch.setattr(ops, "split_tf32", lambda w: calls.append("split") or ("hi", "lo"))
    monkeypatch.setattr(ops, "pack_bf16", lambda w: calls.append("pack") or "pack")
    w = object()
    assert ops.weight_operands(w, 0) == (w, None) and ops.weight_operands(w, 1) == (w, None)
    assert calls == []
    assert ops.weight_operands(w, 2) == ("hi", "lo") and calls == ["split"]
    assert ops.weight_operands(w, 3) == ("pack", None) and calls == ["split", "pack"]
    # a cached form is returned as it is; the modes that take w as it is ignore it
    assert ops.weight_operands(w, 3, ("cached", None)) == ("cached", None)
    assert ops.weight_operands(w, 1, ("cached", None)) == (w, None)
    assert calls == ["split", "pack"]
    # what the module caches hold: nothing in the modes that take w as it is
    assert ops.derived_operands(w, 0) is None and ops.derived_operands(w, 1) is None
    assert ops.derived_operands(w, 2) == ("hi", "lo") and ops.derived_operands(w, 3) == ("pack", None)


@functools.lru_cache(maxsize=1)
def _dump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(exe) or not os.path.exists(S._lib.LIB_PATH):
        return None
    run = lambda flag: subprocess.run([exe, flag, S._lib.LIB_PATH], check=True, capture_output=True, text=True).stdout  # noqa: E731
    return run("-sass"), run("--dump-resource-usage")


def _sass_funcs(pattern):
    if _dump() is None:
        pytest.skip("needs cuobjdump and the built library")
    sass, usage = _dump()
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1) if re.search(pattern, m.group(1)) else None
            if name:
                funcs[name] = set()
        elif name:
            if "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
                funcs[name].add("pipelined")
            if "UTMASTG" in line:
                funcs[name].add("tma_store")
            if "HGMMA" in line and "BF16" in line:
                funcs[name].add("bf16_mma")
    local = {}
    for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", usage):
        if m.group(1) in funcs:
            local[m.group(1)] = int(re.search(r"LOCAL:(\d+)", m.group(2)).group(1))
    return funcs, local


def test_bf16_instances_are_pipelined_bf16_mmas_without_local_memory():
    funcs, local = _sass_funcs(r"dsconv_bf16_kernel")
    got = sorted(tuple(map(int, re.search(r"ILi(\d+)ELi(\d+)ELi(\d+)E", n).groups())) for n in funcs)
    assert got == sorted((nt, k, pw) for nt in (64, 128) for k in (1, 2, 4) for pw in (16, 32)), got
    for n, props in funcs.items():
        assert {"pipelined", "bf16_mma"} <= props, (n, props)
        # the tf32 instances without staging (k = 1 in 3xTF32) have no bf16 counterpart: every bf16 one stages
        assert "tma_store" in props, n
    assert len(local) == len(funcs) and not any(local.values()), local
    # the bf16 pw1x1 / conv3x3 instances (template argument Prec::BF16 = 2)
    pw, pw_local = _sass_funcs(r"pw1x1_tc_kernel.*ELNS_4PrecE2E")
    c3, c3_local = _sass_funcs(r"conv3x3_tc_kernel.*ELNS_4PrecE2E")
    assert len(pw) == 2 and len(c3) == 4, (list(pw), list(c3))
    for n, props in list(pw.items()) + list(c3.items()):
        assert "bf16_mma" in props, n
    assert all("pipelined" in p for p in pw.values())
    assert not any(pw_local.values()) and not any(c3_local.values())
