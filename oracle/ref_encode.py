"""
oracle/ref_encode.py -- TEST INFRASTRUCTURE ONLY (ctypes access to oracle/_ref/liboracle_encode.so, see ref_encode.cc).

The unmodified reference's conversion of RGB input to YCbCr as heif_context_encode_image() runs it, on any of the input
layouts libheif accepts there, and the operation chain its planner picked.
"""
import ctypes as C
import os

import numpy as np

from . import bindings as ob

_lib = None

DOWNSAMPLING_NEAREST, DOWNSAMPLING_AVERAGE, DOWNSAMPLING_SHARP_YUV = 1, 2, 3    # heif_chroma_downsampling_algorithm


def lib():
    """liboracle_encode.so, or None where it was not built (reference sources absent)."""
    global _lib
    if _lib is None:
        p = os.path.join(ob.REF, "liboracle_encode.so")
        if not os.path.exists(p) or not os.path.exists(os.path.join(ob.REF, "libheif_ref.so")):
            return None
        _lib = C.CDLL(p)      # RTLD_LOCAL: libheif_ref.so's C++ symbols must not interpose on torch
        _lib.ref_rgb_to_ycbcr_ex.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_void_p)] + [C.c_int] * 7 + [C.c_void_p] * 4 + [
            C.POINTER(C.c_int), C.c_char_p, C.c_int]
    return _lib


def ycc_shapes(w, h, out_chroma):
    sh, sv = (2 if out_chroma in (1, 2) else 1), (2 if out_chroma == 1 else 1)
    return (h, w), ((h + sv - 1) // sv, (w + sh - 1) // sh)


def ref_rgb_to_ycbcr_ex(rgb, in_chroma, bit_depth, out_chroma, nclx, downsampling=DOWNSAMPLING_AVERAGE, only_preferred=0,
                        alpha_bit_depth=None):
    """UNMODIFIED reference: convert_colorspace(RGB input -> YCbCr out_chroma at the input depth, target nclx = (cp, tc, mc, full)).

    rgb: interleaved (in_chroma 10..15) -> uint8 array [H, W * bytes per pixel] in the layout's byte order;
         planar (in_chroma 3) -> tuple (R, G, B[, A]) of uint8 / uint16 [H, W] arrays.
    Returns (y, cb, cr, alpha or None, pipeline), pipeline = list of the reference operation names; None when
    convert_colorspace fails."""
    l = lib()
    has_alpha = 0
    if in_chroma == 3:
        planes = [np.ascontiguousarray(p) for p in rgb]
        h, w = planes[0].shape
        has_alpha = int(len(planes) == 4)
    else:
        planes = [np.ascontiguousarray(rgb)]
        bpp = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}[in_chroma]
        h, w = planes[0].shape[0], planes[0].shape[1] // bpp
    abd = alpha_bit_depth if alpha_bit_depth is not None else bit_depth
    ptrs = (C.c_void_p * 4)(*[p.ctypes.data for p in planes] + [None] * (4 - len(planes)))
    dt = np.uint16 if bit_depth > 8 else np.uint8
    ys, cs = ycc_shapes(w, h, out_chroma)
    y, cb, cr, a = np.empty(ys, dt), np.empty(cs, dt), np.empty(cs, dt), np.empty(ys, dt)    # alpha leaves at the colour depth
    oha = C.c_int(0)
    buf = C.create_string_buffer(1024)
    cp, tc, mc, fr = nclx
    rc = l.ref_rgb_to_ycbcr_ex(in_chroma, bit_depth, abd, has_alpha, w, h, ptrs, out_chroma, cp, tc, mc, int(fr), downsampling,
                               int(only_preferred), y.ctypes.data, cb.ctypes.data, cr.ctypes.data, a.ctypes.data, C.byref(oha), buf, len(buf))
    if rc == -4:
        return None
    if rc != 0:
        raise RuntimeError(f"ref_rgb_to_ycbcr_ex rc={rc}")
    return y, cb, cr, (a if oha.value else None), buf.value.decode().split(";")


_ex = None


def oracle_rgb_to_ycbcr_ex(rgb, in_chroma, bit_depth, out_chroma, nclx, downsampling=DOWNSAMPLING_AVERAGE, only_preferred=0):
    """C restatement (oracle/color_oracle_ex.c: co_rgb_to_ycbcr_ex); arguments as ref_rgb_to_ycbcr_ex.
    Returns (y, cb, cr, alpha or None, B200_YCC_PIPE_* mask), or None where it refuses (-2)."""
    global _ex
    if _ex is None:
        p = os.path.join(ob.REF, "liboracle_ex.so")
        if not os.path.exists(p):
            raise RuntimeError("oracle/_ref/liboracle_ex.so missing: run `make -C oracle -f encode.mk`")
        _ex = C.CDLL(p)
        _ex.co_rgb_to_ycbcr_ex.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_void_p)] + [C.c_int] * 6 + [C.c_void_p] * 4 + [C.POINTER(C.c_int)]
    if in_chroma == 3:
        planes = [np.ascontiguousarray(p) for p in rgb]
        h, w = planes[0].shape
        has_alpha = len(planes) == 4
    else:
        planes = [np.ascontiguousarray(rgb)]
        nb = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}[in_chroma]
        h, w = planes[0].shape[0], planes[0].shape[1] // nb
        has_alpha = in_chroma in (11, 13, 15)
    ptrs = (C.c_void_p * 4)(*[p.ctypes.data for p in planes] + [None] * (4 - len(planes)))
    dt = np.uint16 if bit_depth > 8 else np.uint8
    ys, cs = ycc_shapes(w, h, out_chroma)
    y, cb, cr = np.empty(ys, dt), np.empty(cs, dt), np.empty(cs, dt)
    a = np.empty(ys, dt) if has_alpha else None
    pipe = C.c_int(0)
    cp, _, mc, fr = nclx
    rc = _ex.co_rgb_to_ycbcr_ex(in_chroma, bit_depth, int(has_alpha), w, h, ptrs, out_chroma, cp, mc, int(fr), downsampling, int(only_preferred),
                                y.ctypes.data, cb.ctypes.data, cr.ctypes.data, None if a is None else a.ctypes.data, C.byref(pipe))
    if rc == -2:
        return None
    if rc != 0:
        raise RuntimeError(f"co_rgb_to_ycbcr_ex rc={rc}")
    return y, cb, cr, a, pipe.value
