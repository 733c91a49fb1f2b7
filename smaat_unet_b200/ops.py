"""Functional host-side wrappers: torch tensors in, C-ABI calls on the current CUDA stream.

PyTorch is plumbing here (device memory, streams); every byte of arithmetic happens in
libsmaat_b200.so.  Tensors must be fp32 CUDA tensors, NCHW, dense in (C?, H, W) -- a
batch stride larger than C*H*W is allowed where the C ABI takes a ``bstride``.  The ops of
SmaAt-UNet's serving forward also take bf16 activations (its bf16 storage route: the
``*_bf16`` entry points of include/smaat_b200.h); each says so.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import gc
import os

import torch

from . import _lib

PW_MODES = {"fp32": 0, "tf32": 1, "tf32x3": 2, "bf16": 3}
_pw_mode = os.environ.get("SMAAT_PW_MODE", "tf32x3")
assert _pw_mode in PW_MODES, f"SMAAT_PW_MODE must be one of {list(PW_MODES)}"


def set_pointwise_mode(mode: str) -> None:
    """'tf32x3' (default; wgmma 3xTF32 split, fp32-grade), 'tf32' (wgmma single pass; what
    cuDNN's allow_tf32=True default gives the reference on a GPU), 'bf16' (wgmma on bf16-rounded operands, fp32
    accumulation: what torch.set_float32_matmul_precision('medium') allows torch's matmuls), 'fp32' (CUDA-core exact).
    The mode applies to the forward GEMMs (fused DS conv, pointwise, dense 3x3, and their input gradients); the weight
    gradients run their tf32 kernels in 'bf16'."""
    global _pw_mode
    if mode not in PW_MODES:
        raise ValueError(f"pointwise mode must be one of {list(PW_MODES)}")
    _pw_mode = mode


def get_pointwise_mode() -> str:
    return _pw_mode


# ---- generation counter of "weights written behind torch's back" (see modules._versions) ----
_weights_gen = 0


def weights_generation() -> int:
    return _weights_gen


def bump_weights_generation() -> None:
    """Call after parameters / buffers were (or may have been) written through raw pointers or a CUDA-graph replay:
    invalidates every cache derived from them (folded BatchNorm affine, tf32 hi/lo weight splits)."""
    global _weights_gen
    _weights_gen += 1


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


# ---- optional per-launch timing (bench.py roofline leg): CUDA events on the launching stream ----
_prof = None


class profile:
    """Context manager: records (kernel name, algorithmic bytes, flops, start/end CUDA events) for every
    C-ABI launch made inside it.  ``summary()`` synchronises and aggregates per kernel name."""

    def __enter__(self):
        global _prof
        self.records = []
        _prof = self
        return self

    def __exit__(self, *exc):
        global _prof
        _prof = None
        return False

    def summary(self, by_shape=False):
        torch.cuda.synchronize()
        agg = {}
        for name, nbytes, flops, e0, e1 in self.records:
            key = name if by_shape else name.split("[")[0]
            a = agg.setdefault(key, {"launches": 0, "ms": 0.0, "bytes": 0, "flops": 0})
            a["launches"] += 1
            a["ms"] += e0.elapsed_time(e1)
            a["bytes"] += nbytes
            a["flops"] += flops
        return agg


def _call(name, nbytes, flops, fn, *args):
    """Invoke one C-ABI entry point on the current stream (optionally bracketed by timing events)."""
    if _prof is None:
        _lib.check(fn(*args), name.split("[")[0])
        return
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(fn(*args), name)
    e1.record()
    _prof.records.append((name, int(nbytes), int(flops), e0, e1))


def _ptr(t):
    return None if t is None else t.data_ptr()


def _req(t, name, ndim=None, bf16=False):
    """``bf16``: a bfloat16 tensor is accepted too (the bf16 route's activations)."""
    ok = (torch.float32, torch.bfloat16) if bf16 else (torch.float32,)
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype not in ok:
        raise RuntimeError(f"smaat_unet_b200: {name} must be a float32{' or bfloat16' if bf16 else ''} CUDA tensor "
                           f"(got {type(t).__name__} {getattr(t, 'dtype', None)} {getattr(t, 'device', None)}); "
                           "there is no CPU fallback")
    if ndim is not None and t.dim() != ndim:
        raise RuntimeError(f"smaat_unet_b200: {name} must be {ndim}-D, got shape {tuple(t.shape)}")
    return t


def _dense(t, name, bf16=False):
    _req(t, name, bf16=bf16)
    return t if t.is_contiguous() else t.contiguous()


def _nchw_bstride(t, name, bf16=False):
    """Accept NCHW tensors that are dense in (C,H,W); return (tensor, batch stride in elements)."""
    _req(t, name, 4, bf16=bf16)
    B, Cc, H, W = t.shape
    st = t.stride()
    if (st[3] == 1 or W == 1) and (st[2] == W or H == 1) and (st[1] == H * W or Cc == 1) and (B == 1 or st[0] >= Cc * H * W):
        return t, (st[0] if B > 1 else Cc * H * W)
    t = t.contiguous()
    return t, Cc * H * W


def _concat_operands(x, x1, bf16=False):
    """The virtual concat [x, x1] as the C ABI reads it: (x, its batch stride, x1 or None, C1, x1's batch stride).  ``bf16``:
    both bfloat16 (the bf16 route)."""
    x, bs0 = _nchw_bstride(x, "x", bf16=bf16)
    if bf16 and x.dtype != torch.bfloat16:
        raise RuntimeError("smaat_unet_b200: the bf16 route's x must be bfloat16")
    if x1 is None:
        return x, bs0, None, 0, 0
    x1, bs1 = _nchw_bstride(x1, "x1", bf16=bf16)
    if x1.dtype != x.dtype:
        raise RuntimeError(f"smaat_unet_b200: concat inputs must have one dtype, got {x.dtype} and {x1.dtype}")
    assert x1.shape[0] == x.shape[0] and x1.shape[2:] == x.shape[2:], "concat inputs must agree in B, H, W"
    return x, bs0, x1, x1.shape[1], bs1


def _pw_matrix(pw_weight, k=None, Cin=None):
    """The pointwise weight (Cout, k Cin[, 1, 1]) as the GEMM's (Cout, k Cin) matrix, checked against k * Cin when given."""
    w2d = _dense(pw_weight, "pointwise.weight").view(pw_weight.shape[0], -1)
    assert k is None or w2d.shape[1] == k * Cin, f"pointwise weight {tuple(pw_weight.shape)} does not match k*Cin={k * Cin}"
    return w2d


_TAKES_W = (0, 1)        # mode codes whose kernels take the fp32 weight as it is ('fp32', 'tf32')


def derived_operands(w, m):
    """What the modules cache for the (rows, K) fp32 matrix w in mode code ``m``: w's tf32 (hi, lo) split in 'tf32x3', (its
    bf16 pack, None) in 'bf16' (``pack_bf16``), None in the modes whose kernels take w as it is."""
    if m in _TAKES_W:
        return None
    return split_tf32(w) if m == 2 else (pack_bf16(w), None)


def weight_operands(w, m, cached=None):
    """The weight operands a GEMM kernel takes in mode code ``m`` for the (rows, K) fp32 matrix w: (w, None) in 'fp32' /
    'tf32', else ``derived_operands`` -- the caller's ``cached`` copy of them when given, derived now when None."""
    if m in _TAKES_W:
        return w, None
    return cached if cached is not None else derived_operands(w, m)


def wgrad_mode(m):
    """The mode code the weight-gradient kernels run for forward mode code ``m``: 'bf16' runs their one-pass tf32 instance
    (their operands reach shared memory as fp32, and operand width does not limit them)."""
    return 1 if m == 3 else m


# ---------------------------------------------------------------------------------------------
def dw3x3(x, weight, bias, k, x1=None, in_scale=None, in_shift=None, loader=0):
    """Depthwise 3x3/pad 1 over the virtual concat [x, x1] (layers.py:38-44; parts_ds.py:85)."""
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    w = _dense(weight, "depthwise.weight")
    assert w.numel() == k * (C0 + C1) * 9, f"depthwise weight {tuple(w.shape)} does not match k*(C0+C1)={k * (C0 + C1)}"
    y = torch.empty((B, k * (C0 + C1), H, W), device=x.device, dtype=torch.float32)
    _call(f"smaat_dw3x3_fwd[C{C0 + C1}_S{H}]", 4 * B * H * W * (C0 + C1) * (1 + k), 18 * B * H * W * k * (C0 + C1), _lib.load().smaat_dw3x3_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(w), _ptr(bias), _ptr(in_scale), _ptr(in_shift),
                                   _ptr(y), B, H, W, k, loader, _stream())
    return y


def tc_eligible(x, w2d) -> bool:
    K, P = x.shape[1], x.shape[2] * x.shape[3]
    return bool(_lib.load().smaat_pw1x1_tc_eligible(_ptr(x), _ptr(w2d), K, w2d.shape[0], P))


def split_tf32(w):
    w = _dense(w, "w")
    hi, lo = torch.empty_like(w), torch.empty_like(w)
    _call("smaat_split_tf32", 12 * w.numel(), 0, _lib.load().smaat_split_tf32, _ptr(w), _ptr(hi), _ptr(lo), w.numel(), _stream())
    return hi, lo


def pack_bf16(w):
    """The bf16 weight operand of 'bf16' mode: (rows, K) fp32 -> (rows, K rounded up to 32) bf16, each value rounded to
    nearest even, k permuted within groups of 16 as the kernels' register fragments present the activations, zero padded
    (smaat_pack_bf16)."""
    w = _dense(w, "w")
    rows, cols = w.shape[0], w[0].numel()
    out = torch.empty((rows, _pad32(cols)), device=w.device, dtype=torch.bfloat16)
    _call("smaat_pack_bf16", 4 * w.numel() + 2 * out.numel(), 0, _lib.load().smaat_pack_bf16, _ptr(w), _ptr(out), rows, cols,
          out.shape[1], _stream())
    return out


def pw1x1(x, weight, scale, shift, relu, mode=None, w_split=None, stats=None, out=None):
    """Pointwise 1x1 + per-channel affine (+ReLU) (layers.py:45,49 + parts_ds.py:25-26).

    weight: (Cout, K[,1,1]).  mode None = module-level default.  w_split = cached weight operands of the mode
    (``weight_operands``: the tf32 (hi, lo) for 'tf32x3', (bf16 pack, None) for 'bf16').  Falls to the exact CUDA-core kernel
    for shapes the tensor-core path does not take.
    """
    x = _dense(x, "x")
    B, K, H, W = x.shape
    w2d = _pw_matrix(weight)
    Cout = w2d.shape[0]
    assert w2d.shape[1] == K, f"pointwise weight {tuple(weight.shape)} does not match K={K}"
    P = H * W
    if out is None:
        out = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.float32)
        ybs = Cout * P
    else:
        out, ybs = _nchw_bstride(out, "out")
    mode = mode or _pw_mode
    m = PW_MODES[mode]
    # the tensor-core kernel stages an epilogue affine for at most 512 output channels (SmaAt_UNet(bilinear=False)'s
    # 1024-channel bottleneck has more)
    if m != 0 and (not tc_eligible(x, w2d) or (Cout > 512 and (scale is not None or shift is not None))):
        m = 0
    w2d, wlo = weight_operands(w2d, m, w_split)
    _call(f"smaat_pw1x1_fwd[K{K}_N{Cout}_P{P}]", 4 * B * P * (K + Cout) + 4 * K * Cout, 2 * B * P * K * Cout, _lib.load().smaat_pw1x1_fwd, _ptr(x), _ptr(w2d), _ptr(wlo), _ptr(scale), _ptr(shift), _ptr(out), ybs, _ptr(stats),
                                           B, K, Cout, P, int(bool(relu)), m, _stream())
    return out


_fuse_ds = os.environ.get("SMAAT_FUSE_DS", "1") != "0"


def set_fused_dsconv(enabled: bool) -> None:
    """Enable/disable the fused depthwise->pointwise kernel (default on; off = dw3x3 + pw1x1 kernels)."""
    global _fuse_ds
    _fuse_ds = bool(enabled)


def set_dsconv_impl(impl: str) -> None:
    """How the fused DS-conv kernel feeds the depthwise result to the tensor core: 'auto', 'smem' (wgmma reads it from shared
    memory) or 'regs' (loaded into registers first)."""
    _lib.check(_lib.load().smaat_set_dsconv_impl({"auto": 0, "smem": 1, "regs": 2}[impl]), "smaat_set_dsconv_impl")


def set_dsconv_wide(enabled: bool) -> None:
    """Run the fused DS conv's 128 < Cout <= 256 layers (k = 2, 'tf32' / 'tf32x3', fp32 maps, the register A form) as wide tiles,
    both 128-channel halves from one depthwise chunk (default on), or in two 128-channel passes (off; Cout a multiple of 128
    only).  The outputs are bitwise equal.  SMAAT_DSCONV_WIDE=0 presets off.  For A/B measurements (tools/time_dsconv.py)."""
    _lib.check(_lib.load().smaat_set_dsconv_wide(int(bool(enabled))), "smaat_set_dsconv_wide")


def set_dsconv_pair(enabled: bool) -> None:
    """Run the fused DS conv's Cout <= 64 layers (k = 2 or 4, 'tf32' / 'tf32x3', fp32 maps, the register A form, an even number
    of patch rows) as paired tiles, two patches sharing each input box and weight chunk (default on), or one patch per tile
    (off).  The outputs are bitwise equal.  SMAAT_DSCONV_PAIR=0 presets off.  For A/B measurements and tests."""
    _lib.check(_lib.load().smaat_set_dsconv_pair(int(bool(enabled))), "smaat_set_dsconv_pair")


def dsconv_takes(x, x1, pw_weight, k, mode=None, stats=False) -> bool:
    """True when ``dsconv`` would run its fused kernel on these inputs (smaat_dsconv_eligible + the arithmetic mode)."""
    mode = mode or _pw_mode
    if not _fuse_ds or PW_MODES[mode] == 0:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    w2d = _pw_matrix(pw_weight)
    lib = _lib.load()
    args = (_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2], x.shape[3], k, w2d.shape[0])
    if not lib.smaat_dsconv_eligible2(*args, int(bool(stats))):
        return False
    # 'bf16' has register-A instances only: the mode-taking test also declines it under set_dsconv_impl('smem')
    return PW_MODES[mode] != 3 or bool(lib.smaat_dsconv_cbam_eligible(*args, 3, 0, 0))


def dsconv_cbam_takes(x, x1, pw_weight, k, gate=False, pools=False, mode=None) -> bool:
    """True when ``dsconv_cbam`` runs on these inputs: the fused kernel, reading x as a CBAM output (``gate``) and / or writing
    the channel gate's partial pools and the 2x2 max-pool of its output (``pools``)."""
    mode = mode or _pw_mode
    if not _fuse_ds or PW_MODES[mode] == 0:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    w2d = _pw_matrix(pw_weight)
    return bool(_lib.load().smaat_dsconv_cbam_eligible(_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2], x.shape[3], k,
                                                       w2d.shape[0], PW_MODES[mode], int(bool(gate)), int(bool(pools))))


def dsconv_cbam(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, x1=None, mode=None, w_split=None, gate=None, pools=False):
    """``dsconv`` in the serving forward's CBAM fusions (smaat_dsconv_cbam_fwd).  ``gate=(sc (B, C0), sa (B, 1, H, W))``: x is read as
    the CBAM output (x * sc) * sa.  ``pools``: also returns the channel gate's partial sums / maxima (B, npart, Cout) and
    MaxPool2d(2) of the output: (y, psum, pmax, pooled).  Raises where ``dsconv_cbam_takes`` is False."""
    mode = mode or _pw_mode
    if not dsconv_cbam_takes(x, x1, pw_weight, k, gate is not None, pools, mode):
        raise RuntimeError("smaat_unet_b200: dsconv_cbam called on a request the fused kernel does not take (check dsconv_cbam_takes)")
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    Cin = C0 + C1
    w2d = _pw_matrix(pw_weight, k, Cin)
    Cout, K = w2d.shape
    w2d, wlo = weight_operands(w2d, PW_MODES[mode], w_split)
    lib = _lib.load()
    sc = sa = None
    if gate is not None:
        sc, sa = _dense(gate[0], "gate sc"), _dense(gate[1], "gate sa")
        assert sc.numel() == B * C0 and sa.numel() == B * H * W, "CBAM gate: sc (B, C0), sa (B, 1, H, W)"
    psum = pmax = pooled = None
    if pools:
        npart = lib.smaat_dsconv_pool_parts(H, W)
        psum = torch.empty((B, npart, Cout), device=x.device, dtype=torch.float32)
        pmax = torch.empty_like(psum)
        pooled = torch.empty((B, Cout, H // 2, W // 2), device=x.device, dtype=torch.float32)
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.float32)
    extra = (4 * B * H * W * C0 if gate is not None else 0) + (4 * B * Cout * (H // 2) * (W // 2) + 8 * psum.numel() if pools else 0)
    _call(f"smaat_dsconv_fwd[C{Cin}_N{Cout}_S{H}]",
          4 * B * H * W * (Cin + Cout) + 4 * K * Cout + extra, 2 * B * H * W * K * (Cout + 9),
          lib.smaat_dsconv_cbam_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(_dense(dw_weight, "depthwise.weight")), _ptr(dw_bias),
          _ptr(w2d), _ptr(wlo), _ptr(scale), _ptr(shift), _ptr(y), Cout * H * W, _ptr(sc), _ptr(sa), _ptr(psum), _ptr(pmax), _ptr(pooled),
          B, H, W, k, Cout, int(bool(relu)), PW_MODES[mode], _stream())
    return (y, psum, pmax, pooled) if pools else y


def dsconv_maxpool_takes(x, x1, pw_weight, k, mode=None) -> bool:
    """True when ``dsconv_maxpool`` runs on these inputs: a fused instance with the staged epilogue
    (smaat_dsconv_maxpool_eligible) in the arithmetic mode, and set_fused_dsconv(True)."""
    mode = mode or _pw_mode
    if not _fuse_ds or PW_MODES[mode] == 0:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    w2d = _pw_matrix(pw_weight)
    return bool(_lib.load().smaat_dsconv_maxpool_eligible(_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2],
                                                          x.shape[3], k, w2d.shape[0], PW_MODES[mode]))


def dsconv_maxpool(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, x1=None, mode=None, w_split=None):
    """``dsconv`` that also returns MaxPool2d(2) of its output from the epilogue (smaat_dsconv_maxpool_fwd): (y, pooled), pooled
    bit for bit the max-pool of y, without a second read of y.  None where ``dsconv_maxpool_takes`` is False (the caller then
    runs ``dsconv`` and ``maxpool2``)."""
    mode = mode or _pw_mode
    if not dsconv_maxpool_takes(x, x1, pw_weight, k, mode):
        return None
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    Cin = C0 + C1
    w2d = _pw_matrix(pw_weight, k, Cin)
    Cout, K = w2d.shape
    w2d, wlo = weight_operands(w2d, PW_MODES[mode], w_split)
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.float32)
    pooled = torch.empty((B, Cout, H // 2, W // 2), device=x.device, dtype=torch.float32)
    _call(f"smaat_dsconv_maxpool_fwd[C{Cin}_N{Cout}_S{H}]", 4 * B * H * W * (Cin + Cout) + 4 * K * Cout + 4 * pooled.numel(),
          2 * B * H * W * K * (Cout + 9), _lib.load().smaat_dsconv_maxpool_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1,
          _ptr(_dense(dw_weight, "depthwise.weight")), _ptr(dw_bias), _ptr(w2d), _ptr(wlo), _ptr(scale), _ptr(shift), _ptr(y),
          Cout * H * W, _ptr(pooled), B, H, W, k, Cout, int(bool(relu)), PW_MODES[mode], _stream())
    return y, pooled


def dsconv(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, x1=None, mode=None, w_split=None, stats=None, outconv=None):
    """Fused DepthwiseSeparableConv (layers.py:47-50) + affine (+ReLU); returns None when the fused kernel
    does not take this shape/mode (caller then runs dw3x3 + pw1x1).  ``outconv=(weight (1, Cout[,1,1]), bias or None)``
    appends the 1-class OutConv in the epilogue and returns the (B, 1, H, W) logits instead of the activation."""
    mode = mode or _pw_mode
    if not dsconv_takes(x, x1, pw_weight, k, mode, stats=stats is not None):
        return None
    if outconv is not None and pw_weight.shape[0] > 128:     # the fused OutConv needs all channels in one pass (smaat_dsconv_outconv_fwd)
        return None
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    Cin = C0 + C1
    w2d = _pw_matrix(pw_weight, k, Cin)
    Cout, K = w2d.shape
    w2d, wlo = weight_operands(w2d, PW_MODES[mode], w_split)
    lib = _lib.load()
    dw_w = _dense(dw_weight, "depthwise.weight")
    if outconv is not None:
        ow, ob = outconv
        assert ow.numel() == Cout and stats is None, "fused OutConv: one class over the block's Cout channels, no batch statistics"
        logits = torch.empty((B, 1, H, W), device=x.device, dtype=torch.float32)
        _call(f"smaat_dsconv_outconv_fwd[C{Cin}_N{Cout}_S{H}]", 4 * B * H * W * (Cin + 1) + 4 * K * Cout, 2 * B * H * W * (K * (Cout + 9) + Cout),
              lib.smaat_dsconv_outconv_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(dw_w), _ptr(dw_bias), _ptr(w2d), _ptr(wlo), _ptr(scale),
              _ptr(shift), _ptr(_dense(ow, "outconv.weight")), _ptr(ob), _ptr(logits), B, H, W, k, Cout, int(bool(relu)), PW_MODES[mode], _stream())
        return logits
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.float32)
    _call(f"smaat_dsconv_fwd[C{Cin}_N{Cout}_S{H}]", 4 * B * H * W * (Cin + Cout) + 4 * K * Cout, 2 * B * H * W * K * (Cout + 9),
          lib.smaat_dsconv_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(dw_w), _ptr(dw_bias), _ptr(w2d), _ptr(wlo), _ptr(scale),
          _ptr(shift), _ptr(y), Cout * H * W, _ptr(stats), B, H, W, k, Cout, int(bool(relu)), PW_MODES[mode], _stream())
    return y


_fuse_classify = os.environ.get("SMAAT_FUSE_CLASSIFY", "1") != "0"


def set_fused_classify(enabled: bool) -> None:
    """Enable/disable the K-class OutConv + argmax in the last DS conv's epilogue (default on; off = that conv, OutConv and
    the channel argmax kernel as separate launches).  For A/B measurements (tools/bench_classes.py, tools/bench_probs.py)."""
    global _fuse_classify
    _fuse_classify = bool(enabled)


def dsconv_classify_takes(x, x1, pw_weight, k, n_classes, mode=None) -> bool:
    """True when ``dsconv_classify`` runs on these inputs: the fused kernel with a ``n_classes``-class OutConv and argmax in its
    epilogue (smaat_dsconv_classify_eligible: Cout <= 128, 1 <= n_classes <= 32 -- 22 to 32 by instance, at least 22 for Cout > 64 --
    the fused DS conv's shapes), and neither set_fused_dsconv(False) nor set_fused_classify(False)."""
    mode = mode or _pw_mode
    if not _fuse_ds or not _fuse_classify or PW_MODES[mode] == 0:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    w2d = _pw_matrix(pw_weight)
    return bool(_lib.load().smaat_dsconv_classify_eligible(_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2], x.shape[3],
                                                           k, w2d.shape[0], int(n_classes), PW_MODES[mode]))


def dsconv_classify(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, oc_weight, oc_bias, x1=None, mode=None, w_split=None,
                    want_logits=False):
    """``dsconv`` followed by OutConv(Cout -> K) and the channel argmax, all in the fused kernel's epilogue
    (smaat_dsconv_classify_fwd).  oc_weight (K, Cout[,1,1]), oc_bias (K) or None.  Returns the (B, H, W) int64 class map, or
    (classes, (B, K, H, W) logits) with ``want_logits``; class j's logits are bit for bit those of ``dsconv(..., outconv=(oc_weight[j],
    oc_bias[j]))``.  Returns None where ``dsconv_classify_takes`` is False (the caller then runs the layers apart)."""
    mode = mode or _pw_mode
    ow = _dense(oc_weight, "outconv.weight")
    K = ow.shape[0]
    if not dsconv_classify_takes(x, x1, pw_weight, k, K, mode):
        return None
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    Cin = C0 + C1
    w2d = _pw_matrix(pw_weight, k, Cin)
    Cout, Kd = w2d.shape
    assert ow.numel() == K * Cout, f"OutConv weight {tuple(oc_weight.shape)} does not match (K, Cout={Cout})"
    ob = _dense(oc_bias, "outconv.bias") if oc_bias is not None else None
    assert ob is None or ob.numel() == K, f"OutConv bias {tuple(oc_bias.shape)} does not match K={K}"
    w2d, wlo = weight_operands(w2d, PW_MODES[mode], w_split)
    classes = torch.empty((B, H, W), device=x.device, dtype=torch.int64)
    logits = torch.empty((B, K, H, W), device=x.device, dtype=torch.float32) if want_logits else None
    _call(f"smaat_dsconv_classify_fwd[C{Cin}_N{Cout}_K{K}_S{H}]",
          4 * B * H * W * (Cin + (K if want_logits else 0) + 2) + 4 * Kd * Cout, 2 * B * H * W * (Kd * (Cout + 9) + K * Cout),
          _lib.load().smaat_dsconv_classify_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(_dense(dw_weight, "depthwise.weight")),
          _ptr(dw_bias), _ptr(w2d), _ptr(wlo), _ptr(scale), _ptr(shift), _ptr(ow), _ptr(ob), K, _ptr(logits), _ptr(classes), B, H,
          W, k, Cout, int(bool(relu)), PW_MODES[mode], _stream())
    return (classes, logits) if want_logits else classes


def is_bf16(t) -> bool:
    return isinstance(t, torch.Tensor) and t.dtype == torch.bfloat16


def dsconv_bf16_takes(x, x1, pw_weight, k, ncls=0) -> bool:
    """True when the bf16-activation DS conv (smaat_dsconv_bf16_eligible) takes bf16 x [, x1]: ``ncls`` = 0 for ``dsconv_bf16``,
    else the classes of ``dsconv_head_bf16``'s OutConv.  set_fused_dsconv(False) declines it too: it has no unfused form."""
    if not _fuse_ds:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1, bf16=True)
    w2d = _pw_matrix(pw_weight)
    return bool(_lib.load().smaat_dsconv_bf16_eligible(_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2], x.shape[3], k,
                                                       w2d.shape[0], int(ncls)))


def _ds_bf16_args(x, x1, dw_weight, k, pw_weight, w_split):
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1, bf16=True)
    B, C0, H, W = x.shape
    Cin = C0 + C1
    w2d = _pw_matrix(pw_weight, k, Cin)
    pack, _ = weight_operands(w2d, PW_MODES["bf16"], w_split)
    return x, bs0, x1, C1, bs1, B, C0, H, W, Cin, w2d.shape[0], pack, _dense(dw_weight, "depthwise.weight")


def dsconv_bf16(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, x1=None, w_split=None, gate=None):
    """``dsconv`` / ``dsconv_cbam`` (gate only) on bf16 activations (smaat_dsconv_bf16_fwd): bf16 x [, x1] -> bf16 y, bf16 GEMM
    operands whatever the pointwise mode (``w_split``: the cached 'bf16' operands), fp32 arithmetic, each output rounded once.
    Raises where ``dsconv_bf16_takes`` is False: the bf16 route has no unfused DS conv."""
    if not dsconv_bf16_takes(x, x1, pw_weight, k):
        raise RuntimeError("smaat_unet_b200: the bf16 DS conv does not take this request (k = 1 or 2, W a multiple of 8, the "
                           "register A form, set_fused_dsconv(True))")
    x, bs0, x1, C1, bs1, B, C0, H, W, Cin, Cout, pack, dw_w = _ds_bf16_args(x, x1, dw_weight, k, pw_weight, w_split)
    sc = sa = None
    if gate is not None:
        sc, sa = _dense(gate[0], "gate sc"), _dense(gate[1], "gate sa")
        assert sc.numel() == B * C0 and sa.numel() == B * H * W, "CBAM gate: sc (B, C0), sa (B, 1, H, W)"
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.bfloat16)
    _call(f"smaat_dsconv_bf16_fwd[C{Cin}_N{Cout}_S{H}]", 2 * B * H * W * (Cin + Cout) + 2 * k * Cin * Cout + (4 * B * H * W if gate else 0),
          2 * B * H * W * k * Cin * (Cout + 9), _lib.load().smaat_dsconv_bf16_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(dw_w),
          _ptr(dw_bias), _ptr(pack), _ptr(scale), _ptr(shift), _ptr(y), Cout * H * W, _ptr(sc), _ptr(sa), B, H, W, k, Cout,
          int(bool(relu)), _stream())
    return y


def dsconv_maxpool_bf16_takes(x, x1, pw_weight, k) -> bool:
    """True when ``dsconv_maxpool_bf16`` takes bf16 x [, x1] (smaat_dsconv_maxpool_bf16_eligible); set_fused_dsconv(False)
    declines it too."""
    if not _fuse_ds:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1, bf16=True)
    w2d = _pw_matrix(pw_weight)
    return bool(_lib.load().smaat_dsconv_maxpool_bf16_eligible(_ptr(x), x.shape[1], bs0, _ptr(x1), C1, bs1, _ptr(w2d), x.shape[2],
                                                               x.shape[3], k, w2d.shape[0]))


def dsconv_maxpool_bf16(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, x1=None, w_split=None, pooled_dtype=torch.bfloat16):
    """``dsconv_bf16`` that also returns MaxPool2d(2) of its bf16 output (smaat_dsconv_maxpool_bf16_fwd): (y, pooled), pooled in
    ``pooled_dtype`` (bfloat16 or float32, the dtype of the level it feeds), bit for bit the max-pool of y.  Raises where
    ``dsconv_maxpool_bf16_takes`` is False."""
    if pooled_dtype not in (torch.bfloat16, torch.float32):
        raise ValueError(f"smaat_unet_b200: pooled_dtype must be torch.bfloat16 or torch.float32, got {pooled_dtype}")
    if not dsconv_maxpool_bf16_takes(x, x1, pw_weight, k):
        raise RuntimeError("smaat_unet_b200: the bf16 DS conv with the max-pool epilogue does not take this request (k = 1 or 2, W "
                           "a multiple of 8, the register A form, set_fused_dsconv(True))")
    x, bs0, x1, C1, bs1, B, C0, H, W, Cin, Cout, pack, dw_w = _ds_bf16_args(x, x1, dw_weight, k, pw_weight, w_split)
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.bfloat16)
    pooled = torch.empty((B, Cout, H // 2, W // 2), device=x.device, dtype=pooled_dtype)
    _call(f"smaat_dsconv_maxpool_bf16_fwd[C{Cin}_N{Cout}_S{H}]",
          2 * B * H * W * (Cin + Cout) + 2 * k * Cin * Cout + pooled.element_size() * pooled.numel(), 2 * B * H * W * k * Cin * (Cout + 9),
          _lib.load().smaat_dsconv_maxpool_bf16_fwd, _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(dw_w), _ptr(dw_bias), _ptr(pack),
          _ptr(scale), _ptr(shift), _ptr(y), Cout * H * W, _ptr(pooled), int(pooled_dtype == torch.bfloat16), B, H, W, k, Cout,
          int(bool(relu)), _stream())
    return y, pooled


def dsconv_head_bf16(x, dw_weight, dw_bias, k, pw_weight, scale, shift, relu, oc_weight, oc_bias, head, w_split=None):
    """The last DS conv of the bf16 route with the OutConv in its epilogue: ``head="logits"`` (one class: the (B, 1, H, W) bf16
    logits, smaat_dsconv_outconv_bf16_fwd) or ``"classes"`` (the (B, H, W) int64 class map, smaat_dsconv_classify_bf16_fwd).
    None where the kernel does not take it (the caller runs the conv and the OutConv apart)."""
    ow = _dense(oc_weight, "outconv.weight")
    K = ow.shape[0]
    if (head == "logits" and K != 1) or not dsconv_bf16_takes(x, None, pw_weight, k, ncls=K):
        return None
    x, bs0, _, _, _, B, C0, H, W, Cin, Cout, pack, dw_w = _ds_bf16_args(x, None, dw_weight, k, pw_weight, w_split)
    assert ow.numel() == K * Cout, f"OutConv weight {tuple(oc_weight.shape)} does not match (K, Cout={Cout})"
    ob = _dense(oc_bias, "outconv.bias") if oc_bias is not None else None
    lib = _lib.load()
    flops = 2 * B * H * W * (k * Cin * (Cout + 9) + K * Cout)
    if head == "logits":
        out = torch.empty((B, 1, H, W), device=x.device, dtype=torch.bfloat16)
        _call(f"smaat_dsconv_outconv_bf16_fwd[C{Cin}_N{Cout}_S{H}]", 2 * B * H * W * (Cin + 1), flops, lib.smaat_dsconv_outconv_bf16_fwd,
              _ptr(x), C0, bs0, None, 0, 0, _ptr(dw_w), _ptr(dw_bias), _ptr(pack), _ptr(scale), _ptr(shift), _ptr(ow), _ptr(ob),
              _ptr(out), B, H, W, k, Cout, int(bool(relu)), _stream())
        return out
    out = torch.empty((B, H, W), device=x.device, dtype=torch.int64)
    _call(f"smaat_dsconv_classify_bf16_fwd[C{Cin}_N{Cout}_K{K}_S{H}]", 2 * B * H * W * Cin + 8 * B * H * W, flops,
          lib.smaat_dsconv_classify_bf16_fwd, _ptr(x), C0, bs0, None, 0, 0, _ptr(dw_w), _ptr(dw_bias), _ptr(pack), _ptr(scale),
          _ptr(shift), _ptr(ow), _ptr(ob), K, None, _ptr(out), B, H, W, k, Cout, int(bool(relu)), _stream())
    return out


def softmax_channels(x):
    """The class probabilities of (B, K, ...) logits: fp32 of the same shape, torch.softmax(x, 1) within fp32 rounding, with
    torch's NaN / 0 / 1 pattern on non-finite logits (smaat_softmax_channels_fwd, 1 <= K <= 1024).  Inference only: no
    gradient."""
    x = _dense(x, "logits", bf16=True)
    if x.dim() < 2:
        raise RuntimeError(f"smaat_unet_b200: logits must be (B, K, ...), got shape {tuple(x.shape)}")
    B, K = x.shape[0], x.shape[1]
    P = x[0, 0].numel()
    probs = torch.empty_like(x)
    if is_bf16(x):      # bf16 logits -> bf16 probabilities (the bf16 route)
        _call(f"smaat_softmax_channels_bf16_fwd[K{K}]", 4 * B * K * P, 0, _lib.load().smaat_softmax_channels_bf16_fwd, _ptr(x),
              _ptr(probs), B, K, P, _stream())
        return probs
    _call(f"smaat_softmax_channels_fwd[K{K}]", 8 * B * K * P, 0, _lib.load().smaat_softmax_channels_fwd, _ptr(x), _ptr(probs),
          B, K, P, _stream())
    return probs


def argmax_channels(x):
    """The class map of (B, K, H, W) logits: int64 (B, H, W), torch.argmax(x, 1) exactly -- ties to the first index, a NaN
    wins (smaat_argmax_channels_fwd, 1 <= K <= 1024)."""
    x = _dense(x, "logits", bf16=True)
    if x.dim() < 2:
        raise RuntimeError(f"smaat_unet_b200: logits must be (B, K, ...), got shape {tuple(x.shape)}")
    B, K = x.shape[0], x.shape[1]
    P = x[0, 0].numel()
    classes = torch.empty((B,) + tuple(x.shape[2:]), device=x.device, dtype=torch.int64)
    if is_bf16(x):
        _call(f"smaat_argmax_channels_bf16_fwd[K{K}]", 2 * B * K * P + 8 * B * P, 0, _lib.load().smaat_argmax_channels_bf16_fwd,
              _ptr(x), _ptr(classes), B, K, P, _stream())
        return classes
    _call(f"smaat_argmax_channels_fwd[K{K}]", 4 * B * K * P + 8 * B * P, 0, _lib.load().smaat_argmax_channels_fwd, _ptr(x), _ptr(classes),
          B, K, P, _stream())
    return classes


def _pad32(c):
    return (c + 31) // 32 * 32


def conv3x3_pack_weight(w, C0, C1=0, flip_transpose=False):
    """nn.Conv2d 3x3 weight (Cout, C0 + C1, 3, 3) -> the packed K-major GEMM matrix of smaat_conv3x3_fwd: (Cout, 9 (C0p + C1p)),
    or with ``flip_transpose`` the input-gradient matrix (C0 + C1, 9 Coutp) (csrc/conv3x3_simt.cu)."""
    w = _dense(w, "conv.weight")
    Cout = w.shape[0]
    assert tuple(w.shape) == (Cout, C0 + C1, 3, 3), f"conv weight {tuple(w.shape)} does not match Cin={C0 + C1}"
    shape = (C0 + C1, 9 * _pad32(Cout)) if flip_transpose else (Cout, 9 * (_pad32(C0) + _pad32(C1)))
    wp = torch.empty(shape, device=w.device, dtype=torch.float32)
    _call("smaat_conv3x3_pack_weight", 8 * wp.numel(), 0, _lib.load().smaat_conv3x3_pack_weight, _ptr(w), _ptr(wp), Cout, C0, C1,
          int(bool(flip_transpose)), _stream())
    return wp


def conv3x3_takes(x, x1, wp, Cout, mode=None) -> bool:
    """True when ``conv3x3`` runs the tensor-core kernel for these inputs in ``mode`` (else the CUDA-core one)."""
    mode = mode or _pw_mode
    if PW_MODES[mode] == 0:
        return False
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    return bool(_lib.load().smaat_conv3x3_tc_eligible(_ptr(x), bs0, _ptr(x1), C1, bs1, _ptr(wp), x.shape[3], Cout))


def conv3x3(x, wp, Cout, scale, shift, relu, x1=None, mode=None, w_split=None, stats=None):
    """nn.Conv2d(Cin, Cout, 3, padding=1) over the virtual concat [x, x1] + per-channel affine (+ReLU) (unet_parts.py:16-21,63).

    wp: ``conv3x3_pack_weight`` of the weight; w_split: its cached operands for the mode (``weight_operands``).  Shapes the tensor-core kernel
    does not take (W % 4 != 0, Cout < 8) run on the exact CUDA-core kernel."""
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    assert wp.shape == (Cout, 9 * (_pad32(C0) + _pad32(C1))), f"packed weight {tuple(wp.shape)} does not match Cin={C0}+{C1}"
    mode = mode or _pw_mode
    m = PW_MODES[mode]
    lib = _lib.load()
    if m != 0 and not lib.smaat_conv3x3_tc_eligible(_ptr(x), bs0, _ptr(x1), C1, bs1, _ptr(wp), W, Cout):
        m = 0
    wp, wlo = weight_operands(wp, m, w_split)
    y = torch.empty((B, Cout, H, W), device=x.device, dtype=torch.float32)
    name = "smaat_conv3x3_fwd" if m else "smaat_conv3x3_fwd_simt"
    Cin = C0 + C1
    _call(f"{name}[C{Cin}_N{Cout}_S{H}x{W}]", 4 * B * H * W * (Cin + Cout) + 36 * Cin * Cout, 18 * B * H * W * Cin * Cout, lib.smaat_conv3x3_fwd,
          _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(wp), _ptr(wlo), _ptr(scale), _ptr(shift), _ptr(y), Cout * H * W, _ptr(stats),
          B, H, W, Cout, int(bool(relu)), m, _stream())
    return y


def conv3x3_bwd_weight(dz, x, x1, dW, mode=None):
    """dW (Cout, Cin, 3, 3) += the weight gradient of ``conv3x3`` over [x, x1] for output gradient dz (unet_parts.py:16,19).
    Tensor cores in 'tf32' / 'tf32x3' (and in 'bf16', which runs the tf32 kernel: ``wgrad_mode``) where the shape allows
    (W % 4 == 0, aligned), else the exact CUDA-core kernel."""
    dz = _dense(dz, "dz")
    x, bs0, x1, C1, bs1 = _concat_operands(x, x1)
    B, C0, H, W = x.shape
    Cout = dz.shape[1]
    assert tuple(dW.shape) == (Cout, C0 + C1, 3, 3) and dW.is_contiguous()
    m = wgrad_mode(PW_MODES[mode or _pw_mode])
    tc_ok = W % 4 == 0 and bs0 % 4 == 0 and bs1 % 4 == 0 and all(t.data_ptr() % 16 == 0 for t in (dz, x) + ((x1,) if C1 else ()))
    if not tc_ok:
        m = 0
    Cin = C0 + C1
    name = "smaat_conv3x3_bwd_weight" if m else "smaat_conv3x3_bwd_weight_simt"
    _call(f"{name}[C{Cin}_N{Cout}_S{H}x{W}]", 4 * B * H * W * (Cin + Cout), 18 * B * H * W * Cin * Cout,
          _lib.load().smaat_conv3x3_bwd_weight, _ptr(dz), _ptr(x), C0, bs0, _ptr(x1), C1, bs1, _ptr(dW), B, H, W, Cout, m, _stream())
    return dW


def bn_fold(gamma, beta, running_mean, running_var, conv_bias, eps):
    """Eval BatchNorm2d -> (scale, shift) for the pw epilogue (parts_ds.py:25,34)."""
    Cn = gamma.numel()
    scale = torch.empty(Cn, device=gamma.device, dtype=torch.float32)
    shift = torch.empty_like(scale)
    _call("smaat_bn_fold", 28 * Cn, 0, _lib.load().smaat_bn_fold, _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), _ptr(conv_bias),
                                         float(eps), _ptr(scale), _ptr(shift), Cn, _stream())
    return scale, shift


def new_stats(C, device):
    """Zeroed fp64 accumulators [sum(C) | sum of squares(C)] for the train-mode BN epilogues."""
    return torch.zeros(2 * C, device=device, dtype=torch.float64)


def channel_stats(x, stats=None):
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    if stats is None:
        stats = new_stats(Cc, x.device)
    _call("smaat_channel_stats", 4 * B * Cc * H * W, 0, _lib.load().smaat_channel_stats, _ptr(x), _ptr(stats), B, Cc, H * W, _stream())
    return stats


def bn_finalize(stats, count, bn, save=False):
    """Batch statistics -> (scale, shift) [, mean, invstd]; updates bn.running_mean/var in place (torch semantics)."""
    Cn = bn.num_features
    dev = stats.device
    scale = torch.empty(Cn, device=dev, dtype=torch.float32)
    shift = torch.empty_like(scale)
    mean = torch.empty_like(scale) if save else None
    invstd = torch.empty_like(scale) if save else None
    track = bn.track_running_stats and bn.running_mean is not None
    if track and bn.momentum is None:
        raise NotImplementedError("BatchNorm2d(momentum=None) (cumulative average) is not supported")
    if track:
        bump_weights_generation()      # running statistics are written by raw pointer: no _version bump
    _call("smaat_bn_finalize", 40 * Cn, 0, _lib.load().smaat_bn_finalize, _ptr(stats), float(count),
          _ptr(bn.weight.detach() if bn.weight is not None else None), _ptr(bn.bias.detach() if bn.bias is not None else None),
          float(bn.eps), float(bn.momentum if bn.momentum is not None else 0.1),
          _ptr(bn.running_mean if track else None), _ptr(bn.running_var if track else None),
          _ptr(scale), _ptr(shift), _ptr(mean), _ptr(invstd),
          _ptr(bn.num_batches_tracked if (track and bn.num_batches_tracked is not None) else None), Cn, _stream())
    return (scale, shift, mean, invstd) if save else (scale, shift)


def affine_act(x, scale, shift, act):
    """y = act(scale[c]*x + shift[c]); act in {'none','relu','sigmoid'}."""
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    y = torch.empty_like(x)
    code = {"none": 0, "relu": 1, "sigmoid": 2}[act]
    _call("smaat_affine_act_fwd", 8 * B * Cc * H * W, 0, _lib.load().smaat_affine_act_fwd, _ptr(x), _ptr(scale), _ptr(shift), _ptr(y),
          B, Cc, H * W, code, _stream())
    return y


def maxpool2(x):
    """nn.MaxPool2d(2) (parts_ds.py:48)."""
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    y = torch.empty((B, Cc, H // 2, W // 2), device=x.device, dtype=torch.float32)
    _call("smaat_maxpool2_fwd", 4 * B * Cc * (H * W + (H // 2) * (W // 2)), 0, _lib.load().smaat_maxpool2_fwd, _ptr(x), _ptr(y), B * Cc, H, W, _stream())
    return y


def upsample2x_pad(x, Ho, Wo, out_dtype=torch.float32):
    """nn.Upsample(x2, bilinear, align_corners=True) + F.pad to (Ho, Wo) (parts_ds.py:64,78-81).  ``out_dtype=torch.bfloat16``
    (the bf16 route): a bf16 output from an fp32 or bf16 x."""
    if out_dtype == torch.bfloat16:
        x = _dense(x, "x", bf16=True)
        B, Cc, H, W = x.shape
        y = torch.empty((B, Cc, Ho, Wo), device=x.device, dtype=torch.bfloat16)
        _call(f"smaat_upsample2x_pad_bf16_fwd[C{Cc}_S{H}]", B * Cc * (x.element_size() * H * W + 2 * Ho * Wo), 0,
              _lib.load().smaat_upsample2x_pad_bf16_fwd, _ptr(x), int(is_bf16(x)), _ptr(y), Cc * Ho * Wo, B, Cc, H, W, Ho, Wo, _stream())
        return y
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    y = torch.empty((B, Cc, Ho, Wo), device=x.device, dtype=torch.float32)
    _call(f"smaat_upsample2x_pad_fwd[C{Cc}_S{H}]", 4 * B * Cc * (H * W + Ho * Wo), 0, _lib.load().smaat_upsample2x_pad_fwd, _ptr(x), _ptr(y), Cc * Ho * Wo, B, Cc, H, W, Ho, Wo, _stream())
    return y


def convt2x2_pack_weight(w):
    """ConvTranspose2d(k=2, s=2) weight (Cin, Cout, 2, 2) -> the pointwise GEMM's (4 Cout, Cin) matrix (csrc/convt.cu)."""
    w = _dense(w, "up.weight")
    Cin, Cout = w.shape[0], w.shape[1]
    wp = torch.empty((4 * Cout, Cin), device=w.device, dtype=torch.float32)
    _call("smaat_convt2x2_pack_weight", 8 * w.numel(), 0, _lib.load().smaat_convt2x2_pack_weight, _ptr(w), _ptr(wp), Cin, Cout, _stream())
    return wp


def pixel_shuffle2_pad(t, bias, Cout, Ho, Wo):
    """(B, 4 Cout, H, W) packed taps -> (B, Cout, Ho, Wo): 2x2 pixel shuffle + bias + F.pad frame (parts_ds.py:76-81)."""
    t = _dense(t, "t")
    B, C4, H, W = t.shape
    assert C4 == 4 * Cout
    y = torch.empty((B, Cout, Ho, Wo), device=t.device, dtype=torch.float32)
    _call("smaat_pixel_shuffle2_pad_fwd", 4 * B * Cout * (4 * H * W + Ho * Wo), 0, _lib.load().smaat_pixel_shuffle2_pad_fwd, _ptr(t), _ptr(bias), _ptr(y),
          Cout * Ho * Wo, B, Cout, H, W, Ho, Wo, _stream())
    return y


def cbam_pool(x):
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    avg = torch.empty((B, Cc), device=x.device, dtype=torch.float32)
    mx = torch.empty_like(avg)
    _call("smaat_cbam_pool_fwd", 4 * B * Cc * H * W, 0, _lib.load().smaat_cbam_pool_fwd, _ptr(x), _ptr(avg), _ptr(mx), B * Cc, H * W, _stream())
    return avg, mx


def _pool_bf16(x, pooled_dtype):
    """bf16 x: (its batch of planes, the (B, C, H / 2, W / 2) max-pool buffer in ``pooled_dtype``), or None where the bf16 kernel
    does not take the shape."""
    B, Cc, H, W = x.shape
    if W % 4 != 0 or H % 2 != 0:
        return None
    return torch.empty((B, Cc, H // 2, W // 2), device=x.device, dtype=pooled_dtype)


def cbam_pool_maxpool(x, pooled_dtype=torch.float32):
    """(avg, mx, maxpool2(x)) from one read of x, or None when the shape is not taken (odd H, W % 4 != 0).  A bf16 x (the bf16
    route) writes its max-pool in ``pooled_dtype`` (bf16 or fp32: the dtype of the level it feeds)."""
    x = _dense(x, "x", bf16=True)
    B, Cc, H, W = x.shape
    if is_bf16(x):
        pooled = _pool_bf16(x, pooled_dtype)
        if pooled is None:
            return None
        avg = torch.empty((B, Cc), device=x.device, dtype=torch.float32)
        mx = torch.empty_like(avg)
        _call("smaat_cbam_pool_maxpool_bf16_fwd", 2 * B * Cc * H * W + pooled.numel() * pooled.element_size(), 0,
              _lib.load().smaat_cbam_pool_maxpool_bf16_fwd, _ptr(x), _ptr(avg), _ptr(mx), _ptr(pooled), int(is_bf16(pooled)), B * Cc,
              H, W, _stream())
        return avg, mx, pooled
    if W % 4 != 0 or H % 2 != 0:
        return None
    avg = torch.empty((B, Cc), device=x.device, dtype=torch.float32)
    mx = torch.empty_like(avg)
    pooled = torch.empty((B, Cc, H // 2, W // 2), device=x.device, dtype=torch.float32)
    _call("smaat_cbam_pool_maxpool_fwd", 5 * B * Cc * H * W, 0, _lib.load().smaat_cbam_pool_maxpool_fwd, _ptr(x), _ptr(avg), _ptr(mx),
          _ptr(pooled), B * Cc, H, W, _stream())
    return avg, mx, pooled


@contextlib.contextmanager
def gc_paused():
    """Keep Python's cyclic garbage collector out of a CUDA-graph capture.  A collection may free unreachable objects that
    own CUDA resources (pinned host buffers, events, graphs of an earlier session); releasing them calls into the driver,
    which invalidates the capture in progress.  They are collected after it instead."""
    was = gc.isenabled()
    gc.disable()
    try:
        yield
    finally:
        if was:
            gc.enable()


_cbam_counters = {}
_retired_counters = []       # superseded buffers: a captured graph may still hand them to its kernels


def _counters(device, n):
    """Zeroed int32 scratch (>= n entries) for the last-arriving-CTA hand-off of smaat_cbam_pool_mlp_fwd: the kernel returns
    it at zero, so one buffer per device serves every call (stream-ordered; allocated outside any graph capture).  A larger
    batch gets a larger buffer; the old one is kept, never freed, because graphs captured earlier have its address."""
    t = _cbam_counters.get(device)
    if t is None or t.numel() < n:
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError("smaat_unet_b200: run one eager forward before capturing a CUDA graph (CBAM scratch allocation)")
        if t is not None:
            _retired_counters.append(t)
        t = torch.zeros(max(n, 256), device=device, dtype=torch.int32)
        _cbam_counters[device] = t
    return t


def cbam_pool_mlp(x, w1, b1, w2, b2, with_maxpool=False, pooled_dtype=torch.float32):
    """ChannelAttention gate in ONE launch: (sc, avg, mx, pooled or None); None when the shape is not taken
    (C % 8, C > 512, hidden > 64) -- callers then use cbam_pool / cbam_pool_maxpool + cbam_mlp.  A bf16 x (the bf16 route) is
    taken with the max-pool only, written in ``pooled_dtype``."""
    x = _dense(x, "x", bf16=True)
    B, Cc, H, W = x.shape
    hidden = w1.shape[0]
    if Cc % 8 != 0 or Cc > 512 or hidden > 64:
        return None
    if is_bf16(x):
        pooled = _pool_bf16(x, pooled_dtype) if with_maxpool else None
        if pooled is None:
            return None
        avg = torch.empty((B, Cc), device=x.device, dtype=torch.float32)
        mx = torch.empty_like(avg)
        sc = torch.empty_like(avg)
        cnt = _counters(x.device, B)
        _call(f"smaat_cbam_pool_mlp_bf16_fwd[C{Cc}_S{H}]", 2 * B * Cc * H * W + pooled.numel() * pooled.element_size(), 0,
              _lib.load().smaat_cbam_pool_mlp_bf16_fwd, _ptr(x), _ptr(avg), _ptr(mx), _ptr(pooled), int(is_bf16(pooled)),
              _ptr(_dense(w1, "w1")), _ptr(b1), _ptr(_dense(w2, "w2")), _ptr(b2), _ptr(sc), _ptr(cnt), B, Cc, H, W, hidden, _stream())
        return sc, avg, mx, pooled
    want_pool = with_maxpool and W % 4 == 0 and H % 2 == 0
    avg = torch.empty((B, Cc), device=x.device, dtype=torch.float32)
    mx = torch.empty_like(avg)
    sc = torch.empty_like(avg)
    pooled = torch.empty((B, Cc, H // 2, W // 2), device=x.device, dtype=torch.float32) if want_pool else None
    cnt = _counters(x.device, B)
    _call(f"smaat_cbam_pool_mlp_fwd[C{Cc}_S{H}]", (5 if want_pool else 4) * B * Cc * H * W, 0, _lib.load().smaat_cbam_pool_mlp_fwd, _ptr(x), _ptr(avg), _ptr(mx),
          _ptr(pooled), _ptr(_dense(w1, "w1")), _ptr(b1), _ptr(_dense(w2, "w2")), _ptr(b2), _ptr(sc), _ptr(cnt), B, Cc, H, W, hidden, _stream())
    return sc, avg, mx, pooled


def cbam_mlp_partials(psum, pmax, H, W, w1, b1, w2, b2):
    """ChannelAttention gate from the partial pools ``dsconv_cbam(..., pools=True)`` wrote for an (H, W) map, in one launch:
    (sc, avg, mx), each (B, C); None when the shape is not taken (C % 16, C > 512, hidden > 64) -- callers then pool the map
    itself (``cbam_pool_mlp``)."""
    B, npart, Cc = psum.shape
    hidden = w1.shape[0]
    if Cc % 16 != 0 or Cc > 512 or hidden > 64:
        return None
    avg = torch.empty((B, Cc), device=psum.device, dtype=torch.float32)
    mx = torch.empty_like(avg)
    sc = torch.empty_like(avg)
    cnt = _counters(psum.device, B)
    _call(f"smaat_cbam_mlp_partials_fwd[C{Cc}_S{H}]", 8 * psum.numel() + 12 * B * Cc, 0, _lib.load().smaat_cbam_mlp_partials_fwd,
          _ptr(_dense(psum, "psum")), _ptr(_dense(pmax, "pmax")), npart, _ptr(avg), _ptr(mx), _ptr(_dense(w1, "w1")), _ptr(b1),
          _ptr(_dense(w2, "w2")), _ptr(b2), _ptr(sc), _ptr(cnt), B, Cc, H, W, hidden, _stream())
    return sc, avg, mx


def cbam_gate_scale(x, sc, pooled, wsp, bn_affine, out=None):
    """y = (x * sc) * sigmoid(bn(conv(pooled))) in one launch (layers.py:126-128, :110); None when the shape is not taken."""
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    if W % 4 != 0:
        return None
    if out is None:
        out = torch.empty_like(x)
        ybs = Cc * H * W
    else:
        out, ybs = _nchw_bstride(out, "out")
    if ybs % 4 != 0 or out.data_ptr() % 16 or x.data_ptr() % 16:
        return None
    ks = wsp.shape[-1]
    _call(f"smaat_cbam_gate_scale_fwd[C{Cc}_S{H}]", 4 * B * (2 * Cc + 2) * H * W, 0, _lib.load().smaat_cbam_gate_scale_fwd, _ptr(pooled), _ptr(_dense(wsp, "wsp")),
          _ptr(bn_affine), _ptr(x), _ptr(sc), _ptr(out), ybs, B, Cc, H, W, ks, _stream())
    return out


def cbam_mlp(avg, mx, w1, b1, w2, b2):
    B, Cc = avg.shape
    sc = torch.empty_like(avg)
    _call("smaat_cbam_mlp_fwd", 12 * B * Cc, 0, _lib.load().smaat_cbam_mlp_fwd, _ptr(avg), _ptr(mx), _ptr(_dense(w1, "w1")), _ptr(b1), _ptr(_dense(w2, "w2")), _ptr(b2),
                                              _ptr(sc), B, Cc, w1.shape[0], _stream())
    return sc


def cbam_reduce(x, sc):
    """Per-pixel channel mean / max of x * sc: (B, 2, H, W) fp32, from an fp32 or (the bf16 route) a bf16 x."""
    x = _dense(x, "x", bf16=True)
    B, Cc, H, W = x.shape
    pooled = torch.empty((B, 2, H, W), device=x.device, dtype=torch.float32)
    if is_bf16(x):
        _call(f"smaat_cbam_reduce_bf16_fwd[C{Cc}_S{H}]", 2 * B * Cc * H * W + 8 * B * H * W, 0, _lib.load().smaat_cbam_reduce_bf16_fwd,
              _ptr(x), _ptr(sc), _ptr(pooled), B, Cc, H * W, _stream())
        return pooled
    _call(f"smaat_cbam_reduce_fwd[C{Cc}_S{H}]", 4 * B * (Cc + 2) * H * W, 0, _lib.load().smaat_cbam_reduce_fwd, _ptr(x), _ptr(sc), _ptr(pooled), B, Cc, H * W, _stream())
    return pooled


def cbam_gate(pooled, wsp, bn_affine, want_raw=False):
    B, _, H, W = pooled.shape
    sa = torch.empty((B, 1, H, W), device=pooled.device, dtype=torch.float32)
    raw = torch.empty_like(sa) if want_raw else None
    ks = wsp.shape[-1]
    _call("smaat_cbam_gate_fwd", 12 * B * H * W, 0, _lib.load().smaat_cbam_gate_fwd, _ptr(pooled), _ptr(_dense(wsp, "wsp")), _ptr(bn_affine), _ptr(sa), _ptr(raw), B, H, W, ks,
                                               _stream())
    return (sa, raw) if want_raw else sa


def cbam_scale(x, sc, sa, out=None):
    x = _dense(x, "x")
    B, Cc, H, W = x.shape
    if out is None:
        out = torch.empty_like(x)
        ybs = Cc * H * W
    else:
        out, ybs = _nchw_bstride(out, "out")
    _call("smaat_cbam_scale_fwd", 4 * B * (2 * Cc + 1) * H * W, 0, _lib.load().smaat_cbam_scale_fwd, _ptr(x), _ptr(sc), _ptr(sa), _ptr(out), ybs, B, Cc, H * W, _stream())
    return out


def outconv(x, weight, bias):
    """OutConv 1x1 (unet_parts.py:70).  A bf16 x (the bf16 route) gives bf16 logits, accumulated in fp32."""
    x = _dense(x, "x", bf16=True)
    B, Cin, H, W = x.shape
    w = _dense(weight, "weight")
    ncls = w.shape[0]
    if is_bf16(x):
        y = torch.empty((B, ncls, H, W), device=x.device, dtype=torch.bfloat16)
        _call("smaat_outconv_bf16_fwd", 2 * B * (Cin + ncls) * H * W, 2 * B * Cin * ncls * H * W, _lib.load().smaat_outconv_bf16_fwd,
              _ptr(x), _ptr(w), _ptr(bias), _ptr(y), B, Cin, ncls, H * W, _stream())
        return y
    y = torch.empty((B, ncls, H, W), device=x.device, dtype=torch.float32)
    _call("smaat_outconv_fwd", 4 * B * (Cin + ncls) * H * W, 2 * B * Cin * ncls * H * W, _lib.load().smaat_outconv_fwd, _ptr(x), _ptr(w), _ptr(bias), _ptr(y), B, Cin, ncls, H * W, _stream())
    return y


# ---- VOC training input (reference utils/dataset_VOC.py:139-168) ----
IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


def _sample_bstride(t, name, dtype, shape):
    """Batch stride of an output that must be written in place: ``dtype`` CUDA, ``shape``, dense within each sample."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != dtype or tuple(t.shape) != tuple(shape):
        raise ValueError(f"smaat_unet_b200: {name} must be a {dtype} CUDA tensor of shape {tuple(shape)}, got "
                         f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))} on {getattr(t, 'device', None)}")
    if not t[0].is_contiguous():
        raise ValueError(f"smaat_unet_b200: {name} must be dense within each sample, got strides {t.stride()}")
    return t.stride(0) if shape[0] > 1 else t[0].numel()


def voc_augment(x_u8, y_u8, aug=None, mean=IMAGENET_MEAN, std=IMAGENET_STD, out_x=None, out_y=None):
    """The VOC sample pipeline after Resize(256) + CenterCrop(224), on the device, bit for bit (smaat_voc_augment_fwd):
    ``x_u8`` (B, H, W, 3) and ``y_u8`` (B, H, W) uint8 CUDA tensors (the shards of ``data.convert_voc``), ``aug`` (B, 3) int8
    rows (flip, rot, bright) from ``voc_segmentation_shard.draw_augmentation`` or None for no augmentation (the reference's
    validation set).  Returns ``(x, y)``: (B, 3, H, W) fp32 ``Normalize(mean, std)(ToTensor(img))`` and (B, H, W) int64 with
    255 -> 0.  ``out_x`` / ``out_y`` receive the result in place (e.g. the leading rows of a session's static inputs); they
    may have any batch stride."""
    for t, name, nd in ((x_u8, "x_u8", 4), (y_u8, "y_u8", 3)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8 or t.dim() != nd:
            raise ValueError(f"smaat_unet_b200: {name} must be a {nd}-D uint8 CUDA tensor, got "
                             f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))}")
    B, H, W, C3 = x_u8.shape
    if B < 1 or C3 != 3 or tuple(y_u8.shape) != (B, H, W):
        raise ValueError(f"smaat_unet_b200: voc_augment needs x_u8 (B, H, W, 3) and y_u8 (B, H, W), got {tuple(x_u8.shape)} "
                         f"and {tuple(y_u8.shape)}")
    x_u8, y_u8 = x_u8.contiguous(), y_u8.contiguous()
    if aug is not None:
        if aug.dtype != torch.int8 or tuple(aug.shape) != (B, 3):
            raise ValueError(f"smaat_unet_b200: aug must be (B, 3) = ({B}, 3) int8, got {aug.dtype} {tuple(aug.shape)}")
        aug = aug.to(x_u8.device).contiguous()
    if out_x is None:
        out_x = torch.empty((B, 3, H, W), device=x_u8.device, dtype=torch.float32)
    if out_y is None:
        out_y = torch.empty((B, H, W), device=x_u8.device, dtype=torch.int64)
    xbs = _sample_bstride(out_x, "out_x", torch.float32, (B, 3, H, W))
    ybs = _sample_bstride(out_y, "out_y", torch.int64, (B, H, W))
    m, s = (C.c_float * 3)(*[float(v) for v in mean]), (C.c_float * 3)(*[float(v) for v in std])
    _call("smaat_voc_augment_fwd", 24 * B * H * W, 0, _lib.load().smaat_voc_augment_fwd, _ptr(x_u8), _ptr(y_u8), _ptr(aug), m, s,
          _ptr(out_x), xbs, _ptr(out_y), ybs, B, H, W, _stream())
    return out_x, out_y


class VOCNormalize:
    """The input transform of a ``TrainSession`` fed uint8 VOC batches: ``sess.step(x_u8, y_u8, aug=aug)`` runs
    ``voc_augment`` straight into the session's static inputs.  ``mean`` / ``std``: the reference's Normalize arguments."""

    def __init__(self, mean=IMAGENET_MEAN, std=IMAGENET_STD):
        self.mean, self.std = tuple(float(v) for v in mean), tuple(float(v) for v in std)
        if len(self.mean) != 3 or len(self.std) != 3:
            raise ValueError("VOCNormalize: mean and std need three values (RGB)")

    def __call__(self, x_u8, y_u8, aug=None, out_x=None, out_y=None):
        return voc_augment(x_u8, y_u8, aug, self.mean, self.std, out_x=out_x, out_y=out_y)

    def __repr__(self):
        return f"VOCNormalize(mean={self.mean}, std={self.std})"


# ---- precipitation dataset builder (reference create_datasets.py:79-82) ----
def rain_pixel_counts(frames, out=None):
    """The number of rain pixels (``v > 0``, NaN never) of every frame of a CUDA float32 ``(N, H, W)`` tensor, as ``(N,)``
    int32: ``np.sum(frame > 0)`` per frame, exact (smaat_rain_pixels_fwd).  ``out``: a dense (N,) int32 CUDA tensor to write
    into (e.g. a slice of a larger count buffer)."""
    _req(frames, "frames", 3)
    frames = frames.contiguous()
    N, H, W = frames.shape
    if out is None:
        out = torch.empty((N,), device=frames.device, dtype=torch.int32)
    elif (not isinstance(out, torch.Tensor) or not out.is_cuda or out.dtype != torch.int32 or tuple(out.shape) != (N,)
          or not out.is_contiguous()):
        raise ValueError(f"smaat_unet_b200: out must be a dense ({N},) int32 CUDA tensor, got "
                         f"{getattr(out, 'dtype', type(out).__name__)} {tuple(getattr(out, 'shape', ()))}")
    if N == 0:
        return out
    _call("smaat_rain_pixels_fwd", 4 * N * H * W + 4 * N, 0, _lib.load().smaat_rain_pixels_fwd, _ptr(frames), N, H * W,
          _ptr(out), _stream())
    return out
