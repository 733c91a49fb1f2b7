"""ctypes binding of libsmaat_b200.so (the C ABI in include/smaat_b200.h).

There is no CPU fallback and no pure-PyTorch fallback: if the shared library is
missing or a call fails, a RuntimeError is raised (the product path must fail
loudly when the CUDA extension is absent).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmaat_b200.so")

_p = C.c_void_p
_i = C.c_int
_l = C.c_int64
_f = C.c_float

# name -> argtypes; every function returns int (0 = ok) unless listed in _SPECIAL
SIGNATURES = {
    "smaat_dw3x3_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "smaat_pw1x1_fwd": [_p, _p, _p, _p, _p, _p, _l, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_pw1x1_tc_eligible": [_p, _p, _i, _i, _i],
    "smaat_dsconv_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i],
    "smaat_dsconv_eligible2": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i],
    "smaat_set_dsconv_impl": [_i],
    "smaat_set_dsconv_wide": [_i],
    "smaat_set_dsconv_pair": [_i],
    "smaat_dsconv_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _l, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_outconv_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_classify_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i, _i],
    "smaat_dsconv_classify_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_cbam_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i, _i, _i],
    "smaat_dsconv_pool_parts": [_i, _i],
    "smaat_dsconv_maxpool_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i],
    "smaat_dsconv_maxpool_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _l, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_cbam_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _l, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_split_tf32": [_p, _p, _p, _l, _p],
    "smaat_pack_bf16": [_p, _p, _i, _i, _i, _p],
    "smaat_bn_fold": [_p, _p, _p, _p, _p, _f, _p, _p, _i, _p],
    "smaat_channel_stats": [_p, _p, _i, _i, _i, _p],
    "smaat_bn_finalize": [_p, C.c_double, _p, _p, _f, _f, _p, _p, _p, _p, _p, _p, _p, _i, _p],
    "smaat_affine_act_fwd": [_p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_maxpool2_fwd": [_p, _p, _l, _i, _i, _p],
    "smaat_upsample2x_pad_fwd": [_p, _p, _l, _i, _i, _i, _i, _i, _i, _p],
    "smaat_cbam_pool_fwd": [_p, _p, _p, _l, _i, _p],
    "smaat_cbam_pool_maxpool_fwd": [_p, _p, _p, _p, _l, _i, _i, _p],
    "smaat_cbam_mlp_fwd": [_p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "smaat_cbam_reduce_fwd": [_p, _p, _p, _i, _i, _i, _p],
    "smaat_cbam_gate_fwd": [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_cbam_scale_fwd": [_p, _p, _p, _p, _l, _i, _i, _i, _p],
    "smaat_cbam_pool_mlp_fwd": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "smaat_cbam_gate_scale_fwd": [_p, _p, _p, _p, _p, _p, _l, _i, _i, _i, _i, _i, _p],
    "smaat_cbam_mlp_partials_fwd": [_p, _p, _i, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "smaat_outconv_fwd": [_p, _p, _p, _p, _i, _i, _i, _i, _p],
    # ---- backward
    "smaat_bn_act_bwd_reduce": [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_bn_bwd_coeffs": [_p, C.c_double, _p, _p, _p, _i, _p, _p, _p, _p, _p, _p, _i, _p],
    "smaat_bn_act_bwd_apply": [_p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_dw3x3_bwd_input": [_p, _p, _p, _i, _l, _p, _i, _l, _i, _i, _i, _i, _p],
    "smaat_dw3x3_bwd_weight": [_p, _p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_pw1x1_bwd_weight": [_p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_pw1x1_bwd_weight_tc": [_p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "smaat_transpose": [_p, _p, _i, _i, _p],
    "smaat_maxpool2_bwd": [_p, _p, _p, _l, _i, _i, _p],
    "smaat_upsample2x_pad_bwd": [_p, _l, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_outconv_bwd": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_cbam_bwd_gate_in": [_p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "smaat_cbam_gate_bwd": [_p, _p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_cbam_bwd_dsc": [_p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "smaat_cbam_bwd_dx": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "smaat_cbam_mlp_bwd": [_p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _p],
    "smaat_mse_metrics_fwd": [_p, _p, _l, _f, _f, _i, _p, _p, _f, _p],
    "smaat_metrics_commit": [_p, _p, _i, _i, _p],
    "smaat_precip_sweep_fwd": [_p, _l, _p, _i, _l, _f, _p, _i, _i, _p, _p, _p],
    "smaat_precip_sweep_commit": [_p, _p, _i, _l, _i, _i, _p, _p],
    "smaat_ce_fwd": [_p, _p, _i, _i, _l, _l, _i, _p, _p, _p, _p],
    "smaat_confusion_add": [_p, _p, _l, _i, _p, _p, _p],
    "smaat_cross_entropy_fwd": [_p, _p, _p, _p, _i, _i, _l, _f, _l, _i, _p, _p, _p, _p, _p],
    "smaat_onehot_classes": [_p, _p, _i, _i, _l, _p],
    "smaat_argmax_channels_fwd": [_p, _p, _i, _i, _l, _p],
    "smaat_softmax_channels_fwd": [_p, _p, _i, _i, _l, _p],
    "smaat_convt2x2_pack_weight": [_p, _p, _i, _i, _p],
    "smaat_convt2x2_unpack_wgrad": [_p, _p, _p, _p, _i, _i, _p],
    "smaat_pixel_shuffle2_pad_fwd": [_p, _p, _p, _l, _i, _i, _i, _i, _i, _i, _p],
    "smaat_pixel_shuffle2_pad_bwd": [_p, _l, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_adam_step": [_p, _p, _p, _p, _l, _p, _p, C.c_double, C.c_double, C.c_double, _p],
    "smaat_conv3x3_pack_weight": [_p, _p, _i, _i, _i, _i, _p],
    "smaat_conv3x3_tc_eligible": [_p, _l, _p, _i, _l, _p, _i, _i],
    "smaat_conv3x3_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _l, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_conv3x3_bwd_weight": [_p, _p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i, _p],
    "smaat_voc_augment_fwd": [_p, _p, _p, _p, _p, _p, _l, _p, _l, _i, _i, _i, _p],
    "smaat_rain_pixels_fwd": [_p, _l, _l, _p, _p],
    # ---- bf16 activations (the serving forward's bf16 route)
    "smaat_dsconv_bf16_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i, _i],
    "smaat_dsconv_bf16_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _l, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_outconv_bf16_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_classify_bf16_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _p, _i, _p, _p, _i, _i, _i, _i, _i, _i, _p],
    "smaat_dsconv_maxpool_bf16_eligible": [_p, _i, _l, _p, _i, _l, _p, _i, _i, _i, _i],
    "smaat_dsconv_maxpool_bf16_fwd": [_p, _i, _l, _p, _i, _l, _p, _p, _p, _p, _p, _p, _l, _p, _i, _i, _i, _i, _i, _i, _i, _p],
    "smaat_cbam_pool_mlp_bf16_fwd": [_p, _p, _p, _p, _i, _p, _p, _p, _p, _p, _p, _i, _i, _i, _i, _i, _p],
    "smaat_cbam_pool_maxpool_bf16_fwd": [_p, _p, _p, _p, _i, _l, _i, _i, _p],
    "smaat_cbam_reduce_bf16_fwd": [_p, _p, _p, _i, _i, _i, _p],
    "smaat_upsample2x_pad_bf16_fwd": [_p, _i, _p, _l, _i, _i, _i, _i, _i, _i, _p],
    "smaat_outconv_bf16_fwd": [_p, _p, _p, _p, _i, _i, _i, _i, _p],
    "smaat_argmax_channels_bf16_fwd": [_p, _p, _i, _i, _l, _p],
    "smaat_softmax_channels_bf16_fwd": [_p, _p, _i, _i, _l, _p],
}
_SPECIAL = {
    "smaat_abi_version": ([], _i),
    "smaat_last_error": ([], C.c_char_p),
    "smaat_launch_count": ([], C.c_uint64),
}
EXPORTED = sorted(list(SIGNATURES) + list(_SPECIAL))

_lib = None


def load():
    """Load (once) and return the ctypes handle; raises RuntimeError if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"smaat_unet_b200: {LIB_PATH} is not built. Run `python -c 'import __graft_entry__ as g; g.build()'` "
            "or smaat_unet_b200/csrc/build.sh. There is no CPU / PyTorch fallback for this path.")
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = _i
    for name, (argtypes, restype) in _SPECIAL.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = restype
    if lib.smaat_abi_version() != 3:
        raise RuntimeError("smaat_unet_b200: ABI version mismatch between _lib.py and libsmaat_b200.so")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().smaat_last_error()
        raise RuntimeError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")


def launch_count() -> int:
    return int(load().smaat_launch_count())
