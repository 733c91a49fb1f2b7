"""The fused DS conv across its dispatch table (tests/test_dsconv_dispatch_abi.py CELLS) on the GPU, against float64.

Every cell is one request to a raw smaat_dsconv_*_fwd entry point with small tensors (B <= 2, at most 72 x 72, a few at
144^2 / 288^2 where the persistent grid wraps around unevenly), x0 / x1 dense or batch-strided channel slices and y dense or
a channel slice of a wider buffer.  Every output buffer (y with its unused channels and batch-stride gap, the statistics, the
max-pool, the CBAM partial pools, logits and class map) is filled with NaN (the class map with -7) past a guard tail before
the launch.

  A  which kernel runs: every taken cell once, in a fresh process under torch.profiler (in one process only the first test
     module that profiles sees kernel events), against ``expected``'s kernel, N_TILE, PW, precision and A form
  B  values: y against the float64 reference of the kernel's arithmetic (dw_emul, pw_ref / pw_ref_bf16 on bf16-rounded
     operands; the bf16 maps within one bf16 ulp), BatchNorm sums against float64 sums, the max-pool bit for bit against
     max_pool2d of the stored y, the CBAM partial pools against float64 sums and maxima of the stored y per half-patch,
     logits against float64 and the class map against its argmax outside near ties; nothing written outside the outputs
  C  tile forms bit for bit: paired tiles against single tiles (smaat_set_dsconv_pair(0)), wide tiles against the two
     128-channel passes (smaat_set_dsconv_wide(0)) at Cout 256
  D  declined cells: ops' *_takes say no, the raw entry point returns SMAAT_E_UNSUPPORTED without a launch or a write, and
     DoubleConvDS still matches a float64 port on a few of those shapes through the unfused kernels

Bounds are those of tests/test_gpu_ds_forward_kernels.py (tf32 / 3xTF32), tests/test_gpu_bf16.py (bf16 operands) and
tests/test_gpu_bf16_activations.py (bf16 maps), except the partial sums' (POOL_SUM_BOUND) and DoubleConvDS's (FALLBACK_BOUND).
Worst observed max |err| / max |ref| over all cells (H100 80GB HBM3 SXM, 700 W): y 7.8e-7 (tf32), 2.1e-6 (3xTF32),
4.2e-7 (bf16); logits 6.8e-7, 1.7e-6, 2.7e-7; BatchNorm sums of squares 8.3e-7, 2.7e-6, 2.2e-7; partial sums 1.3e-7;
bf16 maps and their logits within 0.50 bf16 ulp (+ atol); DoubleConvDS on the declined shapes 3.7e-6.  The file ran in
84 s on one H100 with 0.9 GiB of peak torch memory in the test process (1 104 tests: 936 taken cells, 162 declined ones,
the selection run and 5 fallback shapes).
"""
import json
import os
import subprocess
import sys
import zlib

import pytest
import torch
import torch.nn.functional as F

import smaat_unet_b200 as S
from smaat_unet_b200 import _lib, ops
from tests.test_dsconv_dispatch_abi import CELLS, DECLINED, expected
from tests.test_gpu_bf16 import ERR_BOUND as BF16_BOUND
from tests.test_gpu_bf16 import pw_ref_bf16
from tests.test_gpu_bf16_activations import DS_ATOL, HEAD_ATOL, _one_ulp
from tests.test_gpu_ds_forward_kernels import ERR_BOUND, _bn_affine, _check, _exact, _randn, dw_emul, pw_ref

gpu = pytest.mark.gpu
TAKEN = [c for c in CELLS if c["want"] != DECLINED]
REFUSED = [c for c in CELLS if c["want"] == DECLINED]
GUARD = 40                      # elements past each output that must stay untouched
CLS_FILL = -7
POOL_SUM_BOUND = 1e-6           # the CBAM partial sums: fp32 sums of at most 64 pixels
FALLBACK_BOUND = 2e-5           # DoubleConvDS in 3xTF32 through dw3x3 + pw1x1 against torch's layers in float64
E_UNSUPPORTED = -3
BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------ one cell
def _strided(B, C, H, W, bs, g, dtype):
    """(B, C, H, W) random values with batch stride ``bs``, the rest of the buffer NaN."""
    off = 0 if bs == C * H * W else 32 // torch.finfo(dtype).bits * 8     # a slice: start two 16-byte steps in
    buf = torch.full(((B - 1) * bs + C * H * W + off + 8,), float("nan"), device="cuda", dtype=dtype)
    v = buf[off:].as_strided((B, C, H, W), (bs, H * W, W, 1))
    v.copy_(_randn((B, C, H, W), g).to(dtype))
    return v


def _guarded(n, dtype, fill=float("nan"), head=None):
    buf = torch.full((n + GUARD,), fill, device="cuda", dtype=dtype)
    if head is not None:
        buf[:n] = head
    return buf


def make(c):
    """The cell's inputs and NaN-filled outputs (flat, guarded buffers and the views the kernel writes)."""
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c["id"].encode()))
    B, C0, C1, H, W, k, Cout = c["B"], c["C0"], c["C1"], c["H"], c["W"], c["k"], c["Cout"]
    dt = BF if c["bact"] else torch.float32
    K = k * (C0 + C1)
    t = dict(x0=_strided(B, C0, H, W, c["bs0"], g, dt), x1=_strided(B, C1, H, W, c["bs1"], g, dt) if C1 else None)
    t["w"], t["b"] = _randn((K, 1, 3, 3), g, 0.3), _randn((K,), g, 0.1)
    t["pw"] = _randn((Cout, K), g, K ** -0.5)
    t["sc"], t["sh"] = _bn_affine(Cout, g)
    if c["epilogue"] in ("linear", "stats"):
        t["sc"], t["sh"] = None, _randn((Cout,), g, 0.3)
    if c["epilogue"] == "gate":
        t["gsc"], t["gsa"] = torch.rand((B, C0), generator=g, device="cuda"), torch.rand((B, 1, H, W), generator=g, device="cuda")
    ncls = {"outconv": 1, "classify": c["ncls"]}.get(c["epilogue"], 0)
    if ncls:
        t["ow"], t["ob"] = _randn((ncls, Cout), g, 0.125), _randn((ncls,), g, 0.3)
    m = c["prec"]
    t["wa"], t["wb"] = (t["pw"], None) if m == "tf32" else ops.split_tf32(t["pw"]) if m == "tf32x3" else (ops.pack_bf16(t["pw"]), None)
    # outputs
    out = {}
    if c["epilogue"] in ("outconv", "classify"):
        out["logits"] = _guarded(B * ncls * H * W, dt)
        if c["epilogue"] == "classify":
            out["cls"] = _guarded(B * H * W, torch.int64, CLS_FILL)
    else:
        cy = Cout + 5 if c["y_slice"] else Cout
        out["ybuf"] = _guarded(B * cy * H * W, dt)
        t["ybs"] = cy * H * W
        t["y"] = out["ybuf"][:B * cy * H * W].view(B, cy, H, W)[:, 2:2 + Cout] if c["y_slice"] else out["ybuf"][:B * Cout * H * W].view(B, Cout, H, W)
    if c["epilogue"] == "stats":
        out["stats"] = _guarded(2 * Cout, torch.float64, head=0.0)
    if c["epilogue"] in ("maxpool", "pools"):
        out["pooled"] = _guarded(B * Cout * (H // 2) * (W // 2), dt)
    if c["epilogue"] == "pools":
        t["npart"] = _lib.load().smaat_dsconv_pool_parts(H, W)
        out["psum"] = _guarded(B * t["npart"] * Cout, torch.float32)
        out["pmax"] = _guarded(B * t["npart"] * Cout, torch.float32)
    t["out"] = out
    return t


def _p(x):
    return None if x is None else x.data_ptr()


def launch(c, t):
    """One call of the cell's raw entry point; its return code."""
    lib, st = _lib.load(), ops._stream()
    B, C0, C1, H, W, k, Cout = c["B"], c["C0"], c["C1"], c["H"], c["W"], c["k"], c["Cout"]
    o, e = t["out"], c["epilogue"]
    xin = (_p(t["x0"]), C0, c["bs0"], _p(t["x1"]), C1, c["bs1"], _p(t["w"]), _p(t["b"]))
    aff = (_p(t["sc"]), _p(t["sh"]))
    relu = int(e not in ("linear", "stats"))
    tail = (B, H, W, k, Cout, relu)
    gate = (_p(t.get("gsc")), _p(t.get("gsa")))
    if c["bact"]:
        if e in ("relu", "linear", "gate"):
            return lib.smaat_dsconv_bf16_fwd(*xin, _p(t["wa"]), *aff, _p(t["y"]), t["ybs"], *gate, *tail, st)
        if e == "maxpool":
            return lib.smaat_dsconv_maxpool_bf16_fwd(*xin, _p(t["wa"]), *aff, _p(t["y"]), t["ybs"], _p(o["pooled"]), 1, *tail, st)
        if e == "outconv":
            return lib.smaat_dsconv_outconv_bf16_fwd(*xin, _p(t["wa"]), *aff, _p(t["ow"]), _p(t["ob"]), _p(o["logits"]), *tail, st)
        return lib.smaat_dsconv_classify_bf16_fwd(*xin, _p(t["wa"]), *aff, _p(t["ow"]), _p(t["ob"]), c["ncls"], _p(o["logits"]),
                                                  _p(o["cls"]), *tail, st)
    wts = (_p(t["wa"]), _p(t["wb"]))
    mode = ops.PW_MODES[c["mode"]]
    if e in ("relu", "linear", "stats"):
        return lib.smaat_dsconv_fwd(*xin, *wts, *aff, _p(t["y"]), t["ybs"], _p(o.get("stats")), *tail, mode, st)
    if e == "outconv":
        return lib.smaat_dsconv_outconv_fwd(*xin, *wts, *aff, _p(t["ow"]), _p(t["ob"]), _p(o["logits"]), *tail, mode, st)
    if e == "classify":
        return lib.smaat_dsconv_classify_fwd(*xin, *wts, *aff, _p(t["ow"]), _p(t["ob"]), c["ncls"], _p(o["logits"]), _p(o["cls"]),
                                             *tail, mode, st)
    if e == "maxpool":
        return lib.smaat_dsconv_maxpool_fwd(*xin, *wts, *aff, _p(t["y"]), t["ybs"], _p(o["pooled"]), *tail, mode, st)
    return lib.smaat_dsconv_cbam_fwd(*xin, *wts, *aff, _p(t["y"]), t["ybs"], *gate, _p(o.get("psum")), _p(o.get("pmax")),
                                     _p(o.get("pooled")), *tail, mode, st)


class switches:
    """The cell's A form and wide switch (and optionally the pair switch) for the duration of a block."""

    def __init__(self, c, pair=True, wide=None):
        self.impl, self.wide, self.pair = c["impl"], c["wide_on"] if wide is None else wide, pair

    def __enter__(self):
        lib = _lib.load()
        assert lib.smaat_set_dsconv_impl({"regs": 2, "smem": 1}[self.impl]) == 0
        assert lib.smaat_set_dsconv_wide(int(self.wide)) == 0 and lib.smaat_set_dsconv_pair(int(self.pair)) == 0

    def __exit__(self, *a):
        lib = _lib.load()
        assert lib.smaat_set_dsconv_impl(0) == 0 and lib.smaat_set_dsconv_wide(1) == 0 and lib.smaat_set_dsconv_pair(1) == 0


def signature(c):
    """The kernel name and template arguments ``expected`` implies, as the profiler prints them."""
    kern, nt, pw, _ = c["want"]
    x3 = str(c["prec"] == "tf32x3").lower()
    smem = str(c["impl"] == "smem").lower()
    args = {"dsconv_fused_kernel": (nt, c["k"], pw, x3, smem), "dsconv_kpl4_kernel": (nt, pw, x3),
            "dsconv_bf16_kernel": (nt, c["k"], pw), "dsconv_bf16act_kernel": (nt, c["k"], pw),
            "dsconv_pair_kernel": (c["k"], pw, x3), "dsconv_wide_kernel": (pw, x3)}[kern]
    return f"{kern}<{', '.join(str(a) for a in args)}>"


# ============================================================================================================ A: selection
_SELECTION = r"""
import json, sys
sys.path.insert(0, sys.argv[1])
import torch
from tests.test_gpu_dsconv_dispatch import TAKEN, launch, make, switches

ran = []
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for c in TAKEN:
        t = make(c)
        torch.cuda.synchronize()
        with switches(c):
            rc = launch(c, t)
        torch.cuda.synchronize()
        ran.append(rc)
ev = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "dsconv" in e.name),
            key=lambda e: e.time_range.start)
print(json.dumps({"rc": ran, "kernels": [e.name for e in ev]}))
"""


@gpu
def test_which_kernel_runs_in_every_cell():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _SELECTION, root], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got["rc"] == [0] * len(TAKEN), [(c["id"], rc) for c, rc in zip(TAKEN, got["rc"]) if rc][:10]
    # one dsconv kernel per cell, in order: a cell that ran none, or two, shifts every name after it
    names = got["kernels"]
    assert len(names) == len(TAKEN), f"{len(names)} dsconv kernels for {len(TAKEN)} cells"
    bad = [f"{c['id']}: want {signature(c)}, ran {n[:120]}" for c, n in zip(TAKEN, names) if signature(c) not in n]
    assert not bad, f"{len(bad)} cells ran another kernel:\n" + "\n".join(bad[:20])


# =============================================================================================================== B: values
def _untouched(buf, n, what):
    tail = buf[n:]
    ok = bool(torch.isnan(tail).all()) if tail.is_floating_point() else bool((tail == CLS_FILL).all())
    assert ok, f"{what}: written past its end"


def _reference(c, t):
    """float64 of the kernel's arithmetic: the activation (or the training-mode z + bias) and, for heads, the logits."""
    x0 = t["x0"].float()
    if c["epilogue"] == "gate":
        x0 = (x0 * t["gsc"].view(*t["gsc"].shape, 1, 1)) * t["gsa"]
    x = torch.cat([x0, t["x1"].float()], dim=1) if c["C1"] else x0
    d = dw_emul(x.contiguous(), t["w"], t["b"], c["k"])
    z = pw_ref_bf16(d, t["pw"]) if c["mode"] == "bf16" else pw_ref(d, t["pw"], c["mode"])
    if t["sc"] is not None:
        z = z * t["sc"].double().view(1, -1, 1, 1)
    z = z + t["sh"].double().view(1, -1, 1, 1)
    a = torch.relu(z) if c["epilogue"] not in ("linear", "stats") else z
    lg = None
    if "ow" in t:
        lg = torch.einsum("kc,bchw->bkhw", t["ow"].double(), a) + t["ob"].double().view(1, -1, 1, 1)
    return a, lg


def _bound(c, key="fused"):
    return BF16_BOUND[key] if c["mode"] == "bf16" else ERR_BOUND[key][c["mode"]]


def _half_patch_pools(y, pw, npart):
    """float64 (sum, max) of y per half-patch: (B, patch rows, column tiles, 2 halves, C) flattened as the kernel writes them."""
    B, C, H, W = y.shape
    ph = 128 // pw
    pr, tx = -(-H // ph), -(-W // pw)
    assert npart == 2 * pr * tx
    yd = y.double()
    pad = (0, tx * pw - W, 0, pr * ph - H)
    s = F.pad(yd, pad).view(B, C, pr, 2, ph // 2, tx, pw).sum(dim=(4, 6))
    m = F.pad(yd, pad, value=-float("inf")).view(B, C, pr, 2, ph // 2, tx, pw).amax(dim=(4, 6))
    return s.permute(0, 2, 4, 3, 1).reshape(B, npart, C), m.permute(0, 2, 4, 3, 1).reshape(B, npart, C)


def check_cell(c, t):
    """Every output of a taken cell against float64, and nothing written outside them.  Returns the outputs."""
    B, H, W, Cout, e = c["B"], c["H"], c["W"], c["Cout"], c["epilogue"]
    o = t["out"]
    a, lg = _reference(c, t)
    what = c["id"]
    res = {}
    if "ybuf" in o:
        y = t["y"]
        n = B * (Cout + 5 if c["y_slice"] else Cout) * H * W
        _untouched(o["ybuf"], n, f"{what} y")
        rest = o["ybuf"][:n].clone()
        if c["y_slice"]:
            rest.view(B, Cout + 5, H, W)[:, 2:2 + Cout] = float("nan")
            assert bool(torch.isnan(rest).all()), f"{what}: y's other channels written"
        assert bool(torch.isfinite(y).all()), f"{what}: y not fully written"
        if c["bact"]:
            _one_ulp(y, a, f"{what} y", DS_ATOL)
        else:
            _check(y, a, _bound(c), f"{what} y")
        res["y"] = y.clone()
    if e == "stats":
        _untouched(o["stats"], 2 * Cout, f"{what} stats")
        _check(o["stats"][:Cout], a.sum(dim=(0, 2, 3)), _bound(c, "fused_stats"), f"{what} stats sum")
        _check(o["stats"][Cout:2 * Cout], (a * a).sum(dim=(0, 2, 3)), _bound(c, "fused_stats"), f"{what} stats sum of squares")
    if "pooled" in o:
        n = B * Cout * (H // 2) * (W // 2)
        _untouched(o["pooled"], n, f"{what} pooled")
        res["pooled"] = o["pooled"][:n].view(B, Cout, H // 2, W // 2).clone()
        _exact(res["pooled"], F.max_pool2d(t["y"], 2), f"{what} max-pool of y")
    if e == "pools":
        n = B * t["npart"] * Cout
        for key in ("psum", "pmax"):
            _untouched(o[key], n, f"{what} {key}")
            res[key] = o[key][:n].view(B, t["npart"], Cout).clone()
        s, m = _half_patch_pools(t["y"], c["want"][2], t["npart"])
        _check(res["psum"], s, POOL_SUM_BOUND, f"{what} partial sums")
        _exact(res["pmax"].double(), m, f"{what} partial maxima")
    if lg is not None:
        K = lg.shape[1]
        _untouched(o["logits"], B * K * H * W, f"{what} logits")
        got = o["logits"][:B * K * H * W].view(B, K, H, W)
        if c["bact"]:
            _one_ulp(got, lg, f"{what} logits", HEAD_ATOL)
        else:
            _check(got, lg, _bound(c), f"{what} logits")
        res["logits"] = got.clone()
    if e == "classify":
        _untouched(o["cls"], B * H * W, f"{what} classes")
        cls = o["cls"][:B * H * W].view(B, H, W)
        tol = HEAD_ATOL if c["bact"] else _bound(c)
        scale = float(lg.abs().max())
        top2 = lg.topk(2, dim=1).values if lg.shape[1] > 1 else None
        clear = (top2[:, 0] - top2[:, 1]) > 2 * tol * scale if top2 is not None else torch.ones_like(cls, dtype=torch.bool)
        bad = int(((cls != lg.argmax(1)) & clear).sum())
        assert bad == 0, f"{what}: {bad} pixels away from a tie take another class than float64's argmax"
        if not c["bact"]:
            _exact(cls, res["logits"].argmax(1), f"{what} class map vs its logits")
        res["cls"] = cls.clone()
    return res


@gpu
@pytest.mark.parametrize("c", TAKEN, ids=[c["id"] for c in TAKEN])
def test_cell_against_float64(c):
    t = make(c)
    with switches(c):
        _lib.check(launch(c, t), c["id"])
    torch.cuda.synchronize()
    res = check_cell(c, t)
    # C: the same cell through the other tile form, bit for bit (the statistics' atomics sum in no fixed order)
    other = None
    if c["want"][0] == "dsconv_pair_kernel":
        other = dict(pair=False)
    elif c["want"][0] == "dsconv_wide_kernel" and c["Cout"] == 256:
        other = dict(wide=False)
    if other is not None:
        t2 = make(c)
        with switches(c, **other):
            _lib.check(launch(c, t2), c["id"])
        torch.cuda.synchronize()
        res2 = check_cell(c, t2)
        for key in res:
            _exact(res2[key], res[key], f"{c['id']} {key}: {c['want'][0]} vs {other}")


# ========================================================================================================== D: declined
def _takes(c, t):
    x0, x1, pw, k, e, mode = t["x0"], t["x1"], t["pw"], c["k"], c["epilogue"], c["mode"]
    if c["bact"]:
        if e == "maxpool":
            return ops.dsconv_maxpool_bf16_takes(x0, x1, pw, k)
        return ops.dsconv_bf16_takes(x0, x1, pw, k, ncls={"outconv": 1, "classify": c["ncls"]}.get(e, 0))
    if e in ("relu", "linear", "stats"):
        return ops.dsconv_takes(x0, x1, pw, k, mode, stats=e == "stats")
    if e in ("outconv", "classify"):
        return ops.dsconv_classify_takes(x0, x1, pw, k, 1 if e == "outconv" else c["ncls"], mode)
    if e == "maxpool":
        return ops.dsconv_maxpool_takes(x0, x1, pw, k, mode)
    return ops.dsconv_cbam_takes(x0, x1, pw, k, gate=e == "gate", pools=e == "pools", mode=mode)


@gpu
@pytest.mark.parametrize("c", REFUSED, ids=[c["id"] for c in REFUSED])
def test_declined_cell(c):
    t = make(c)
    torch.cuda.synchronize()
    with switches(c):
        assert not _takes(c, t)
        n0 = _lib.launch_count()
        assert launch(c, t) == E_UNSUPPORTED
        assert _lib.launch_count() == n0, "a declined request launched a kernel"
    torch.cuda.synchronize()
    for key, buf in t["out"].items():
        filled = torch.isnan(buf[:-GUARD]) if buf.is_floating_point() else buf[:-GUARD] == CLS_FILL
        if key == "stats":
            filled = buf[:-GUARD] == 0
        assert bool(filled.all()) and (not buf.is_floating_point() or bool(torch.isnan(buf[-GUARD:]).all())), f"{key} written"


# (C0, Cout, H, W, k): shapes the fused kernel declines -- pick_pw refuses 36 x 36, W not a multiple of 4, k = 3, Cout 136 at
# k = 4 (only the wide tile takes Cout off a multiple of 128), Cout under 8
FALLBACK = [(24, 64, 36, 36, 2), (24, 24, 32, 50, 1), (32, 64, 32, 64, 3), (24, 136, 32, 64, 4), (24, 4, 32, 64, 2)]


def _port64(block, x):
    """DoubleConvDS in float64 with torch's own layers (eval: running statistics)."""
    seq = block.double_conv if hasattr(block, "double_conv") else None
    assert seq is not None
    h = x.double()
    for m in seq:
        if isinstance(m, S.modules.DepthwiseSeparableConv):
            h = F.conv2d(h, m.depthwise.weight.double(), m.depthwise.bias.double(), padding=1, groups=m.depthwise.groups)
            h = F.conv2d(h, m.pointwise.weight.double(), m.pointwise.bias.double())
        elif isinstance(m, torch.nn.BatchNorm2d):
            h = F.batch_norm(h, m.running_mean.double(), m.running_var.double(), m.weight.double(), m.bias.double(), False, 0.0, m.eps)
        else:
            h = torch.relu(h)
    return h


@gpu
@pytest.mark.parametrize("C0,Cout,H,W,k", FALLBACK)
def test_declined_shape_runs_unfused_in_double_conv_ds(C0, Cout, H, W, k):
    assert expected(C0, 0, C0 * H * W, 0, H, W, k, Cout, "tf32x3", "regs", True, False, "relu", 0) == DECLINED
    g = torch.Generator(device="cuda").manual_seed(C0 + Cout + H + W + k)
    torch.manual_seed(C0 + Cout + H + W + k)
    block = S.DoubleConvDS(C0, Cout, kernels_per_layer=k).cuda().eval()
    for m in block.modules():
        if isinstance(m, torch.nn.BatchNorm2d):
            m.running_mean.copy_(_randn(m.running_mean.shape, g, 0.2))
            m.running_var.copy_(torch.rand(m.running_var.shape, generator=g, device="cuda") + 0.5)
    x = _randn((2, C0, H, W), g)
    old = ops.get_pointwise_mode()
    ops.set_pointwise_mode("tf32x3")
    try:
        with torch.no_grad():
            y = block(x)
    finally:
        ops.set_pointwise_mode(old)
    _check(y, _port64(block, x), FALLBACK_BOUND, f"DoubleConvDS {C0}->{Cout} {H}x{W} k={k}")
