"""
oracle/refheif.py -- TEST INFRASTRUCTURE ONLY: ctypes access to the C API of the UNMODIFIED reference libheif
(oracle/_ref/libheif_ref.so, built by oracle/Makefile from /root/reference) for end-to-end tests of the drop-in
boundary (heif_register_decoder_plugin / heif_register_encoder_plugin, heif_context_encode_grid, heif_decode_image).

IMPORTANT: load() opens libheif_ref.so with RTLD_GLOBAL so that plugins can find the heif_* entry points; its C++
symbols would then interpose on torch's libraries, so only use this module in processes that never import torch
(the tests run it in a subprocess).
"""
import ctypes as C
import os

import numpy as np

from . import bindings as ob

COLORSPACE_YCBCR, COLORSPACE_RGB, COLORSPACE_MONO = 0, 1, 2
CHROMA_420, CHROMA_INTERLEAVED_RGB, CHROMA_INTERLEAVED_RGBA = 1, 10, 11
CHANNEL_Y, CHANNEL_CB, CHANNEL_CR, CHANNEL_INTERLEAVED = 0, 1, 2, 10
COMPRESSION_HEVC = 1


class Err(C.Structure):
    _fields_ = [("code", C.c_int), ("sub", C.c_int), ("msg", C.c_char_p)]


class DecodingOptionsHead(C.Structure):     # leading members of heif_decoding_options (heif_decoding.h:63-97)
    _fields_ = [("version", C.c_uint8), ("ignore_transformations", C.c_uint8), ("start_progress", C.c_void_p),
                ("on_progress", C.c_void_p), ("end_progress", C.c_void_p), ("progress_user_data", C.c_void_p),
                ("convert_hdr_to_8bit", C.c_uint8), ("strict_decoding", C.c_uint8), ("decoder_id", C.c_char_p)]


class Nclx(C.Structure):                    # heif_color_profile_nclx (heif_color.h)
    _fields_ = [("version", C.c_uint8), ("color_primaries", C.c_int), ("transfer_characteristics", C.c_int),
                ("matrix_coefficients", C.c_int), ("full_range_flag", C.c_uint8)]


_h = None


def load():
    global _h
    if _h is None:
        # B200_REF_LIB=libheif_ref_b200.so selects the second build with the GPU colour operation (SURVEY 8f N2, oracle/Makefile n2)
        p = os.path.join(ob.REF, os.environ.get("B200_REF_LIB", "libheif_ref.so"))
        if not os.path.exists(p):
            raise RuntimeError(f"{p} missing")
        h = C.CDLL(p, mode=C.RTLD_GLOBAL)
        h.heif_context_alloc.restype = C.c_void_p
        for name in ["heif_context_read_from_file", "heif_context_get_primary_image_handle", "heif_decode_image", "heif_image_create",
                     "heif_image_add_plane", "heif_context_get_encoder_for_format", "heif_encoder_set_lossy_quality",
                     "heif_context_encode_image", "heif_context_encode_grid", "heif_context_write_to_file", "heif_register_decoder_plugin",
                     "heif_register_encoder_plugin", "heif_image_set_nclx_color_profile", "heif_encoder_set_parameter_integer",
                     "heif_context_read_from_memory_without_copy"]:
            getattr(h, name).restype = Err
        h.heif_context_read_from_file.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p]
        h.heif_context_get_primary_image_handle.argtypes = [C.c_void_p, C.POINTER(C.c_void_p)]
        h.heif_decode_image.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_void_p]
        h.heif_image_get_plane_readonly.restype = C.POINTER(C.c_uint8)
        h.heif_image_get_plane_readonly.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        h.heif_image_get_plane.restype = C.POINTER(C.c_uint8)
        h.heif_image_get_plane.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int)]
        h.heif_image_get_width.argtypes = [C.c_void_p, C.c_int]
        h.heif_image_get_height.argtypes = [C.c_void_p, C.c_int]
        h.heif_image_release.argtypes = [C.c_void_p]
        h.heif_image_handle_release.argtypes = [C.c_void_p]
        h.heif_context_free.argtypes = [C.c_void_p]
        h.heif_image_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p)]
        h.heif_image_add_plane.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
        h.heif_image_set_nclx_color_profile.argtypes = [C.c_void_p, C.POINTER(Nclx)]
        h.heif_context_get_encoder_for_format.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
        h.heif_encoder_set_lossy_quality.argtypes = [C.c_void_p, C.c_int]
        h.heif_encoder_set_parameter_integer.argtypes = [C.c_void_p, C.c_char_p, C.c_int]
        h.heif_encoder_release.argtypes = [C.c_void_p]
        h.heif_context_encode_image.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        h.heif_context_encode_grid.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint16, C.c_uint16, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
        h.heif_context_write_to_file.argtypes = [C.c_void_p, C.c_char_p]
        h.heif_context_set_max_decoding_threads.argtypes = [C.c_void_p, C.c_int]
        h.heif_register_decoder_plugin.argtypes = [C.c_void_p]
        h.heif_register_encoder_plugin.argtypes = [C.c_void_p]
        h.heif_decoding_options_alloc.restype = C.POINTER(DecodingOptionsHead)
        h.heif_decoding_options_free.argtypes = [C.POINTER(DecodingOptionsHead)]
        h.heif_image_handle_has_alpha_channel.argtypes = [C.c_void_p]
        h.heif_encoder_get_name.restype = C.c_char_p
        h.heif_encoder_get_name.argtypes = [C.c_void_p]
        _h = h
    return _h


def check(e, what=""):
    if e.code != 0:
        raise RuntimeError(f"libheif error {e.code}/{e.sub} {what}: {(e.msg or b'').decode(errors='replace')}")


def register_cpu_decoder():
    """The CPU decoder plugin of the oracle (FFmpeg in the libde265 role), id 'b200-oracle'."""
    load()
    # the plugin variant linked against the reference build in use (one copy of libheif per process)
    name = "liboracle_plugin_b200.so" if os.environ.get("B200_REF_LIB", "libheif_ref.so") == "libheif_ref_b200.so" else "liboracle_plugin.so"
    plug = C.CDLL(os.path.join(ob.REF, name))
    rc = plug.b200_oracle_register(ob.avcodec_dir().encode())
    if rc != 0:
        raise RuntimeError("b200_oracle_register failed")
    return plug


def make_ycbcr_image(y, cb, cr, bit_depth=8, nclx=None):
    h = load()
    img = C.c_void_p()
    hh, ww = y.shape
    mono = cb is None
    check(h.heif_image_create(ww, hh, COLORSPACE_MONO if mono else COLORSPACE_YCBCR, 0 if mono else CHROMA_420, C.byref(img)))
    for ch, pl in ((CHANNEL_Y, y), (CHANNEL_CB, cb), (CHANNEL_CR, cr)):
        if pl is None:
            continue
        ph, pw = pl.shape
        check(h.heif_image_add_plane(img, ch, pw, ph, bit_depth))
        st = C.c_int()
        p = h.heif_image_get_plane(img, ch, C.byref(st))
        bps = 2 if bit_depth > 8 else 1
        dst = np.ctypeslib.as_array(p, shape=(ph, st.value))
        src = np.ascontiguousarray(pl.astype(np.uint16 if bps == 2 else np.uint8)).view(np.uint8).reshape(ph, pw * bps)
        dst[:, :pw * bps] = src
    if nclx is not None:
        n = Nclx(1, nclx[0], nclx[1], nclx[2], nclx[3])
        check(h.heif_image_set_nclx_color_profile(img, C.byref(n)))
    return img


def rgb_image(rgb):
    """heif_image of an interleaved 8-bit RGB / RGBA array [H, W, 3|4]."""
    h = load()
    hh, ww, ch = rgb.shape
    img = C.c_void_p()
    check(h.heif_image_create(ww, hh, COLORSPACE_RGB, CHROMA_INTERLEAVED_RGBA if ch == 4 else CHROMA_INTERLEAVED_RGB, C.byref(img)))
    check(h.heif_image_add_plane(img, CHANNEL_INTERLEAVED, ww, hh, 8))
    st = C.c_int()
    p = h.heif_image_get_plane(img, CHANNEL_INTERLEAVED, C.byref(st))
    np.ctypeslib.as_array(p, shape=(hh, st.value))[:, :ww * ch] = rgb.reshape(hh, ww * ch)
    return img


def encode_file(path, images, columns=1, rows=1, quality=60, params=None):
    """heif_context_encode_image / heif_context_encode_grid with whatever HEVC encoder plugin is registered."""
    h = load()
    ctx = h.heif_context_alloc()
    enc = C.c_void_p()
    check(h.heif_context_get_encoder_for_format(ctx, COMPRESSION_HEVC, C.byref(enc)), "get_encoder_for_format")
    check(h.heif_encoder_set_lossy_quality(enc, quality))
    for k, v in (params or {}).items():
        check(h.heif_encoder_set_parameter_integer(enc, k.encode(), int(v)), k)
    out = C.c_void_p()
    if len(images) == 1:
        check(h.heif_context_encode_image(ctx, images[0], enc, None, C.byref(out)), "encode_image")
    else:
        arr = (C.c_void_p * len(images))(*images)
        # NOTE: the header names the parameters (rows, columns) but the implementation takes (columns, rows)
        # (api/libheif/heif_tiling.h:109-115 vs heif_tiling.cc:138-141; flagged in the reference's tests/encode_grid.cc:164-166)
        check(h.heif_context_encode_grid(ctx, arr, columns, rows, enc, None, C.byref(out)), "encode_grid")
    check(h.heif_context_write_to_file(ctx, path.encode()), "write")
    h.heif_image_handle_release(out)
    h.heif_encoder_release(enc)
    h.heif_context_free(ctx)


last_timing = {}


def decode_file(path, chroma=CHROMA_INTERLEAVED_RGB, decoder_id=None, threads=None):
    """heif_decode_image(primary image) -> (uint8 array [H, W*channels]).  last_timing["api_s"]: seconds spent in the libheif
    calls that produce the picture (heif_context_read_from_file .. heif_decode_image), without this wrapper's copy into numpy."""
    import time
    h = load()
    t0 = time.perf_counter()
    ctx = h.heif_context_alloc()
    check(h.heif_context_read_from_file(ctx, path.encode(), None), "read")
    if threads is not None:
        h.heif_context_set_max_decoding_threads(ctx, threads)
    hd = C.c_void_p()
    check(h.heif_context_get_primary_image_handle(ctx, C.byref(hd)))
    opts = h.heif_decoding_options_alloc()
    keep = decoder_id.encode() if decoder_id else None
    if keep:
        opts.contents.decoder_id = keep
    img = C.c_void_p()
    try:
        check(h.heif_decode_image(hd, C.byref(img), COLORSPACE_RGB, chroma, opts), "decode_image")
    finally:
        h.heif_decoding_options_free(opts)
    last_timing["api_s"] = time.perf_counter() - t0
    st = C.c_int()
    p = h.heif_image_get_plane_readonly(img, CHANNEL_INTERLEAVED, C.byref(st))
    w, hh = h.heif_image_get_width(img, CHANNEL_INTERLEAVED), h.heif_image_get_height(img, CHANNEL_INTERLEAVED)
    nch = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}[chroma]        # bytes per pixel of the interleaved formats
    out = np.ctypeslib.as_array(p, shape=(hh, st.value))[:, :w * nch].copy()
    h.heif_image_release(img)
    h.heif_image_handle_release(hd)
    h.heif_context_free(ctx)
    return out
