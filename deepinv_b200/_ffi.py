"""ctypes declarations of the C ABI in include/dinvk.h (one place, used by the product loader
`deepinv_b200._lib` and by the kernel-logic tests)."""
from __future__ import annotations

import ctypes as C

c_void_p, c_int, c_float, c_size_t, c_int64 = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_int64

# DINVK_G_* multiplier modes
G_NONE, G_MASK, G_SQ, G_INV_SQ_PLUS_C, G_PINV, G_CMUL, G_CMUL_CONJ = range(7)
PAD_VALID, PAD_CIRCULAR, PAD_REPLICATE, PAD_REFLECT, PAD_CONSTANT = range(5)
PADDING_CODES = {"valid": PAD_VALID, "circular": PAD_CIRCULAR, "replicate": PAD_REPLICATE, "reflect": PAD_REFLECT,
                 "constant": PAD_CONSTANT}


class SpectralArgs(C.Structure):
    """mirror of `dinvk_spectral_args`"""

    _fields_ = [
        ("B", C.c_int32), ("H", C.c_int32), ("W", C.c_int32),
        ("fwd", C.c_int32), ("inv", C.c_int32), ("centered", C.c_int32), ("gmode", C.c_int32),
        ("p0", c_void_p), ("p1", c_void_p), ("a0", c_float), ("a1", c_float),
        ("mask", c_void_p), ("mask_sb", c_int64), ("mask_sc", c_int64), ("mask_sh", c_int64),
        ("c", c_float), ("c_batch", c_void_p),
        ("q0", c_void_p), ("q1", c_void_p), ("e0", c_float), ("e1", c_float), ("e2", c_float),
        ("out", c_void_p),
        ("ncoil", C.c_int32), ("coil_mode", C.c_int32), ("coil_maps", c_void_p), ("coil_sb", c_int64),
    ]


_SIGNATURES = {
    # name: (restype, argtypes)
    "dinvk_version": (c_int, []),
    "dinvk_last_error": (C.c_char_p, []),
    "dinvk_launch_count": (C.c_uint64, []),
    "dinvk_spectral_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "dinvk_spectral": (c_int, [C.POINTER(SpectralArgs), c_void_p, c_size_t, c_void_p]),
    "dinvk_fft_prepare": (c_int, [c_int, c_int]),
    "dinvk_spectral3d_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "dinvk_spectral3d": (c_int, [C.POINTER(SpectralArgs), c_int, c_void_p, c_size_t, c_void_p]),
    "dinvk_ramp_filter_workspace_bytes": (c_size_t, [c_int, c_int]),
    "dinvk_ramp_filter": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "dinvk_axpbypcz": (c_int, [c_void_p, c_void_p, c_float, c_void_p, c_float, c_void_p, c_float, c_int64, c_void_p]),
    "dinvk_interleaved_to_planar": (c_int, [c_void_p, c_void_p, c_int, c_int64, c_void_p]),
    "dinvk_batched_axpy": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_int, c_int64, c_void_p]),
    "dinvk_batched_dot": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_size_t, c_void_p]),
    "dinvk_batched_dot_workspace_bytes": (c_size_t, [c_int, c_int64]),
    "dinvk_cg_scalars": (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_float, c_void_p, c_int, c_void_p]),
    "dinvk_ddrm_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int64,
                                  c_float, c_float, c_float, c_float, c_float, c_float, c_float, c_int, c_void_p]),
    "dinvk_radon_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p]),
    "dinvk_radon_adj": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p]),
    "dinvk_iradon_bp": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_void_p]),
    "dinvk_fanbeam": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_float, c_float,
                              c_float, c_float, c_int, c_void_p]),
    "dinvk_blur_fwd": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 9 + [c_void_p]),
    "dinvk_blur_adj_workspace_bytes": (c_size_t, [c_int] * 7),
    "dinvk_blur_adj": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 9 + [c_void_p, c_size_t, c_void_p]),
    "dinvk_blur3d_fwd": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 11 + [c_void_p]),
    "dinvk_blur3d_adj_workspace_bytes": (c_size_t, [c_int] * 9),
    "dinvk_blur3d_adj": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 11 + [c_void_p, c_size_t, c_void_p]),
    "dinvk_svblur_fwd": (c_int, [c_void_p] * 4 + [c_int] * 12 + [c_void_p]),
    "dinvk_svblur_adj_workspace_bytes": (c_size_t, [c_int] * 7),
    "dinvk_svblur_adj": (c_int, [c_void_p] * 4 + [c_int] * 12 + [c_void_p, c_size_t, c_void_p]),
    "dinvk_tiled_svblur_fwd": (c_int, [c_void_p] * 4 + [c_int] * 13 + [c_void_p]),
    "dinvk_tiled_svblur_adj": (c_int, [c_void_p] * 4 + [c_int] * 13 + [c_void_p]),
    "dinvk_resize_fwd": (c_int, [c_void_p] * 2 + [c_int] * 5 + [c_void_p] * 2 + [c_int] + [c_void_p] * 2 + [c_int, C.c_double,
                                                                                                      c_void_p]),
    "dinvk_resize_adj": (c_int, [c_void_p] * 2 + [c_int] * 5 + [c_void_p] * 6 + [c_int, C.c_double, c_void_p]),
    "dinvk_conv_f32": (c_int, [c_void_p] * 6 + [c_int] * 7 + [c_void_p]),
    "dinvk_conv_f32_wgrad": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_void_p]),
    "dinvk_relu_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "dinvk_conv3x3_bf16": (c_int, [c_void_p] * 6 + [c_int] * 6 + [c_void_p]),
    "dinvk_conv3x3_bf16_tail": (c_int, [c_void_p] * 5 + [c_int] * 5 + [c_void_p]),
    "dinvk_conv3x3_head_bf16": (c_int, [c_void_p] * 4 + [c_int] * 4 + [c_float, c_void_p, c_int, c_int, c_void_p]),
    "dinvk_nchw_f32_to_nhwc_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int, c_void_p]),
    "dinvk_nhwc_bf16_to_nchw_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dinvk_conv2x2_down_bf16": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_void_p]),
    "dinvk_conv2x2_up_bf16": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_void_p]),
    "dinvk_conv_tc32": (c_int, [c_void_p] * 6 + [c_int] * 9 + [c_void_p, c_void_p]),
    "dinvk_conv_tc32_slab": (c_int, [c_void_p] * 6 + [c_int] * 8 + [c_void_p, c_void_p]),
    "dinvk_conv_tc32_head": (c_int, [c_void_p] * 4 + [c_int] * 5 + [c_float, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dinvk_conv_tc32_tail": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_void_p, c_void_p]),
    "dinvk_split16_to_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dinvk_nchw_to_split16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "dinvk_conv3d_f32": (c_int, [c_void_p] * 6 + [c_int] * 8 + [c_void_p]),
    "dinvk_conv3d_tc32": (c_int, [c_void_p] * 6 + [c_int] * 10 + [c_void_p, c_void_p]),
    "dinvk_conv3d_tc32_head": (c_int, [c_void_p] * 4 + [c_int] * 6 + [c_float, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "dinvk_conv3d_tc32_tail": (c_int, [c_void_p] * 5 + [c_int] * 7 + [c_void_p, c_void_p]),
    "dinvk_tv_prox": (c_int, [c_void_p] * 6 + [c_int] * 5 + [c_float, C.c_double, C.c_double, c_int, c_int, c_int,
                                                               c_void_p, c_size_t, c_void_p]),
    "dinvk_tv_prox_workspace_bytes": (c_size_t, [c_int] * 4),
    "dinvk_tv_block": (c_int, [C.POINTER(c_int), C.POINTER(c_int)]),
    "dinvk_tv_stencil": (c_int, [c_int, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "dinvk_tv_fn": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_size_t, c_void_p]),
    "dinvk_tv_fn_workspace_bytes": (c_size_t, [c_int] * 4),
    "dinvk_tgv_prox": (c_int, [c_void_p] * 9 + [c_int] * 5 + [c_float, C.c_double, C.c_double, c_int, c_int,
                                                               c_void_p, c_size_t, c_void_p]),
    "dinvk_tgv_prox_workspace_bytes": (c_size_t, [c_int] * 4),
    "dinvk_tgv_block": (c_int, [C.POINTER(c_int), C.POINTER(c_int)]),
}


def declared_symbols() -> list[str]:
    return sorted(_SIGNATURES)


def bind(lib: C.CDLL, required: bool = True) -> C.CDLL:
    """attach restype/argtypes; with required=False missing symbols are skipped (partial test builds)"""
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            if required:
                raise
            continue
        fn.restype = res
        fn.argtypes = args
    return lib
