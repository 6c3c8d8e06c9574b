"""ctypes loader for libb200heif.so: the one place that opens the library, the ctypes mirrors of the structs of
include/b200_heif.h and the signature of every entry point (tests/test_python_abi.py pins both against the headers).

Fails loudly: there is no CPU or PyTorch fallback for any operation of this package.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("B200_LIB", os.path.join(HERE, "libb200heif.so"))   # B200_LIB: development override (kernel variants)


class Planes(C.Structure):
    _fields_ = [("y", C.c_void_p), ("cb", C.c_void_p), ("cr", C.c_void_p), ("alpha", C.c_void_p),
                ("y_stride", C.c_size_t), ("c_stride", C.c_size_t), ("alpha_stride", C.c_size_t),
                ("width", C.c_int), ("height", C.c_int), ("chroma", C.c_int), ("bit_depth", C.c_int),
                ("colour_primaries", C.c_int), ("transfer_characteristics", C.c_int),
                ("matrix_coefficients", C.c_int), ("full_range", C.c_int)]


class Geometry(C.Structure):
    _fields_ = [("m", C.c_int * 6), ("out_w", C.c_int), ("out_h", C.c_int), ("chroma", C.c_int), ("detour", C.c_int),
                ("pre", C.c_int * 6), ("pre_w", C.c_int), ("pre_h", C.c_int)]


class RgbImage(C.Structure):
    _fields_ = [("rgb", C.c_void_p), ("rgb_stride", C.c_size_t), ("r", C.c_void_p), ("g", C.c_void_p), ("b", C.c_void_p),
                ("alpha", C.c_void_p), ("r_stride", C.c_size_t), ("g_stride", C.c_size_t), ("b_stride", C.c_size_t),
                ("alpha_stride", C.c_size_t), ("width", C.c_int), ("height", C.c_int), ("chroma", C.c_int), ("bit_depth", C.c_int),
                ("alpha_bit_depth", C.c_int)]


class RgbToYCbCrOptions(C.Structure):
    _fields_ = [("chroma_downsampling", C.c_int), ("only_use_preferred", C.c_int)]


class ColorOptions(C.Structure):
    _fields_ = [("out_chroma", C.c_int), ("out_bit_depth", C.c_int), ("chroma_upsampling", C.c_int)]


class EncParams(C.Structure):
    _fields_ = [(n, C.c_int) for n in (
        "width", "height", "bit_depth", "chroma_format_idc", "log2_ctb_size", "qp", "init_qp",
        "max_transform_hierarchy_depth_intra", "sao", "sign_data_hiding", "transform_skip", "strong_intra_smoothing",
        "cu_qp_delta", "diff_cu_qp_delta_depth", "dqp_range", "cb_qp_offset", "cr_qp_offset", "slice_chroma_qp_offsets",
        "slice_cb_qp_offset", "slice_cr_qp_offset", "wpp", "slice_ctb_rows", "dependent_slice_segments",
        "loop_filter_across_slices", "slice_loop_filter_across_slices", "deblocking_disabled", "beta_offset_div2",
        "tc_offset_div2", "slice_deblocking_override", "slice_deblocking_disabled", "slice_beta_offset_div2",
        "slice_tc_offset_div2", "mode_decision", "split_threshold", "still_picture", "vui_present",
        "colour_description_present", "colour_primaries", "transfer_characteristics", "matrix_coefficients", "full_range")] + \
        [("seed", C.c_uint32), ("scaling_lists", C.c_int), ("pcm", C.c_int), ("transquant_bypass", C.c_int), ("tile_cols", C.c_int), ("tile_rows", C.c_int), ("tiles_uniform", C.c_int),
         ("loop_filter_across_tiles", C.c_int), ("slice_per_tile", C.c_int), ("speed", C.c_int)]


class GpuEncodeStats(C.Structure):
    _fields_ = [("analyse_ms", C.c_double), ("entropy_ms", C.c_double), ("framing_ms", C.c_double), ("total_ms", C.c_double),
                ("bytes", C.c_uint64), ("ctus", C.c_uint64), ("pictures", C.c_uint64),
                ("mode_evaluations", C.c_uint64), ("cu_evaluations", C.c_uint64)]


class GridEncodeInfo(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("cols", "rows", "tile_w", "tile_h", "width", "height", "has_alpha", "pipeline")] + \
        [("colour_ms", C.c_double), ("upload_ms", C.c_double)]


class ImageInfo(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("width", "height", "tile_width", "tile_height", "chroma", "bit_depth", "colour_primaries",
                                       "transfer_characteristics", "matrix_coefficients", "full_range")]


class DecodeStats(C.Structure):
    _fields_ = [(n, C.c_double) for n in ("parse_ms", "pack_ms", "h2d_ms", "gpu_ms", "total_ms", "entropy_ms", "recon_ms", "deblock_ms", "sao_ms")] + \
               [(n, C.c_uint64) for n in ("bitstream_bytes", "command_bytes", "coefficient_entries", "transform_units", "ctus", "h2d_bytes", "pixels")] + \
               [("kernel_launches", C.c_int), ("front_end", C.c_int), ("bands", C.c_int)]


_P, _vp, _int, _sz = C.POINTER, C.c_void_p, C.c_int, C.c_size_t
_u8pp = _P(_P(C.c_uint8))
_decode_to_rgb = (_int, [_vp, _int, _int, _P(C.c_char_p), _P(_sz), C.c_uint64, _int, _int, _P(Geometry), _P(ColorOptions), _vp, _sz,
                         _P(ImageInfo)])

# name -> (restype, argtypes) of every function of include/b200_heif.h and of the b200_* functions of
# include/b200_heif_plugin_abi.h.  Opaque handles (b200_decoder*, b200_gpu_encoder*) and cudaStream_t are c_void_p.
FUNCTIONS = {
    "b200_last_error": (C.c_char_p, []),
    "b200_version": (_int, []),
    "b200_geometry_identity": (None, [_int, _int, _P(Geometry)]),
    "b200_geometry_init": (None, [_int, _int, _int, _P(Geometry)]),
    "b200_geometry_rotate_ccw": (_int, [_P(Geometry), _int]),
    "b200_geometry_mirror": (_int, [_P(Geometry), _int]),
    "b200_geometry_crop": (_int, [_P(Geometry), _int, _int, _int, _int]),
    "b200_color_convert_device": (_int, [_P(Planes), _P(Geometry), _P(ColorOptions), _vp, _vp, _vp, _sz, _vp, _P(_int)]),
    "b200_color_convert_scaled_device": (_int, [_P(Planes), _P(Geometry), _P(ColorOptions), _int, _int, _vp, _vp, _vp, _sz, _vp, _P(_int)]),
    "b200_color_convert_host": (_int, [_P(Planes), _P(Geometry), _P(ColorOptions), _vp, _vp, _vp, _sz, _P(_int)]),
    "b200_rgb_to_ycbcr_device": (_int, [_vp, _sz, _int, _P(Planes), _vp]),
    "b200_rgb_to_ycbcr_host": (_int, [_vp, _sz, _int, _P(Planes)]),
    "b200_rgb_to_ycbcr_plan": (_int, [_P(RgbImage), _P(Planes), _P(RgbToYCbCrOptions), _P(_int)]),
    "b200_rgb_to_ycbcr_ex_device": (_int, [_P(RgbImage), _P(Planes), _P(RgbToYCbCrOptions), _vp, _P(_int)]),
    "b200_rgb_to_ycbcr_ex_host": (_int, [_P(RgbImage), _P(Planes), _P(RgbToYCbCrOptions), _P(_int)]),
    "b200_ycbcr_to_rgb_coefficients": (None, [_int, _int, _P(C.c_float)]),
    "b200_overlay_fill_device": (_int, [_P(_vp), _P(_sz), _int, _int, _P(C.c_uint16), _vp]),
    "b200_overlay_device": (_int, [_P(_vp), _P(_sz), _int, _int, _P(_vp), _P(_sz), _int, _int, C.c_int32, C.c_int32, _vp]),
    "b200_scale_nearest_device": (_int, [_vp, _sz, _vp, _sz] + [C.c_uint32] * 6 + [_int, _vp]),
    "b200_hevc_enc_params_default": (None, [_P(EncParams)]),
    "b200_hevc_encode_intra": (_int, [_P(EncParams), _vp, _vp, _vp, _sz, _sz, _u8pp, _P(_sz)]),
    "b200_free": (None, [_vp]),
    "b200_gpu_encode_check": (_int, [_P(EncParams), _int, _P(Planes)]),
    "b200_gpu_encoder_create": (_int, [_P(_vp)]),
    "b200_gpu_encoder_destroy": (None, [_vp]),
    "b200_gpu_encode_intra_device": (_int, [_vp, _P(EncParams), _int, _P(Planes), _vp]),
    "b200_gpu_encode_intra_host": (_int, [_vp, _P(EncParams), _int, _P(Planes)]),
    "b200_gpu_encoder_output": (_int, [_vp, _int, _u8pp, _P(_sz)]),
    "b200_gpu_encoder_read_recon": (_int, [_vp, _int, _vp, _vp, _vp, _sz, _sz]),
    "b200_gpu_encoder_get_stats": (_int, [_vp, _P(GpuEncodeStats)]),
    "b200_gpu_encoder_substream_capacity": (_sz, [_int, _int, _int]),
    "b200_gpu_encoder_e1_warps_per_sm": (_int, [_int, _P(_int)]),
    "b200_gpu_encode_rgb_grid_check": (_int, [_P(RgbImage), _int, _int, _P(EncParams), _P(RgbToYCbCrOptions)]),
    "b200_gpu_encode_rgb_grid_device": (_int, [_vp, _P(RgbImage), _int, _int, _P(EncParams), _P(RgbToYCbCrOptions), _vp, _P(GridEncodeInfo)]),
    "b200_gpu_encode_rgb_grid_host": (_int, [_vp, _P(RgbImage), _int, _int, _P(EncParams), _P(RgbToYCbCrOptions), _P(GridEncodeInfo)]),
    "b200_decoder_create": (_int, [_P(_vp), _int]),
    "b200_decoder_destroy": (None, [_vp]),
    "b200_decoder_decode_grid": (_int, [_vp, _int, _int, _P(C.c_char_p), _P(_sz), C.c_uint64, _int, _int, _P(ImageInfo), _vp]),
    "b200_decoder_get_planes": (_int, [_vp, _P(Planes)]),
    "b200_decoder_read_planes": (_int, [_vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "b200_decoder_debug_read_tile": (_int, [_vp, _int, _int, _vp, _vp, _vp]),
    "b200_decoder_set_front_end": (_int, [_vp, _int]),
    "b200_decoder_set_debug_stage": (_int, [_vp, _int]),
    "b200_decoder_get_stats": (_int, [_vp, _P(DecodeStats)]),
    "b200_decoder_rerun_device": (_int, [_vp, _vp]),
    "b200_probe_access_unit": (_int, [C.c_char_p, _sz, C.c_uint64, _P(ImageInfo)]),
    "b200_decode_grid_to_rgb_host": _decode_to_rgb,
    "b200_decode_grid_to_rgb_host_async": _decode_to_rgb,
    "b200_decode_grid_to_rgb_scaled_host": (_int, _decode_to_rgb[1][:10] + [_int, _int] + _decode_to_rgb[1][10:]),
    "b200_decoder_wait": (_int, [_vp]),
    "b200_host_alloc": (_int, [_sz, _P(_vp)]),
    "b200_host_free": (None, [_vp]),
    "b200_host_register": (_int, [_vp, _sz]),
    "b200_host_unregister": (_int, [_vp]),
    "b200_get_decoder_plugin": (_vp, []),
    "b200_get_encoder_plugin": (_vp, []),
    "b200_get_gpu_encoder_plugin": (_vp, []),
    "b200_plugin_bind_libheif": (_int, [_vp]),
    "b200_plugin_queue_stats": (None, [_P(C.c_uint64)]),
    "b200_plugin_encoder_stats": (None, [_P(C.c_uint64)]),
}

# Test-only entry points the library exports outside the headers (stage harnesses of the tests and probes of scripts/).
# Their buffers are c_void_p, so callers pass numpy addresses or ctypes arrays alike.
DEBUG_FUNCTIONS = {
    "b200_debug_parse": (_int, [C.c_char_p, _sz, _vp, _vp, _vp, _vp, _vp]),
    "b200_debug_parse_filters": (_int, [C.c_char_p, _sz, _vp, _vp, _int, _vp, _int]),
    "b200_debug_parse_many": (_int, [_P(C.c_char_p), _P(_sz), _int, _int, _int, _P(C.c_double)]),
    "b200_debug_unescape": (_int, [C.c_char_p, _sz, _vp, _vp, _sz, _P(_sz)]),
    "b200_debug_k1_residual": (_int, [_int, _vp, _vp, _vp, _vp]),
    "b200_debug_chroma_qp": (_int, [_int, _vp, _vp]),
    "b200_debug_k1_predict": (_int, [_int] + [_vp] * 7),
    "b200_debug_k1_descriptors": (_int, [C.c_char_p, _sz, _vp, _vp, _int, _vp, _int]),
    "b200_debug_loop_filters": (_int, [_int, _int] + [_vp] * 8 + [_int]),
    "b200_debug_enc_transform_host": (_int, [_int, _vp, _vp, _vp]),
    "b200_debug_enc_transform_device": (_int, [_int, _vp, _vp, _vp]),
    "b200_debug_enc_predict_host": (_int, [_int, _vp, _vp, _vp, _vp]),
    "b200_debug_enc_predict_device": (_int, [_int, _vp, _vp, _vp, _vp]),
    "b200_debug_hevc_encode_forced_levels": (_int, [_P(EncParams), _vp, _vp, _vp, _sz, _sz, _vp, _int, _u8pp, _P(_sz), _vp, _vp, _vp]),
}

# Exported only by the B200_ENTROPY_TRACE build of the library that scripts/k0_trace_probe.py loads through B200_LIB.
TRACE_FUNCTIONS = {
    "b200_debug_entropy_trace": (_int, [_vp, _int]),
}

_lib = None


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"libb200heif error {code}: {msg}")
        self.code = code


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ImportError(f"{SO_PATH} is missing: build it with `python -m libheif_b200.build` "
                              "(or __graft_entry__.build()); there is no fallback path")
        l = C.CDLL(SO_PATH)
        for name, (res, args) in {**FUNCTIONS, **DEBUG_FUNCTIONS, **TRACE_FUNCTIONS}.items():
            if name in TRACE_FUNCTIONS and not hasattr(l, name):
                continue
            f = getattr(l, name)
            f.restype, f.argtypes = res, args
        _lib = l
    return _lib


def check(rc):
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))
