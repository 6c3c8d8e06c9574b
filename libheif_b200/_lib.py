"""ctypes loader for libb200heif.so (the C ABI declared in include/b200_heif.h).

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
        _lib = C.CDLL(SO_PATH)
        _lib.b200_last_error.restype = C.c_char_p
        _lib.b200_geometry_identity.argtypes = [C.c_int, C.c_int, C.POINTER(Geometry)]
        _lib.b200_geometry_identity.restype = None
        _lib.b200_geometry_init.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(Geometry)]
        _lib.b200_geometry_init.restype = None
        _lib.b200_geometry_rotate_ccw.argtypes = [C.POINTER(Geometry), C.c_int]
        _lib.b200_geometry_mirror.argtypes = [C.POINTER(Geometry), C.c_int]
        _lib.b200_geometry_crop.argtypes = [C.POINTER(Geometry)] + [C.c_int] * 4
        _lib.b200_color_convert_device.argtypes = [C.POINTER(Planes), C.POINTER(Geometry), C.POINTER(ColorOptions),
                                                   C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p,
                                                   C.POINTER(C.c_int)]
        _lib.b200_color_convert_host.argtypes = [C.POINTER(Planes), C.POINTER(Geometry), C.POINTER(ColorOptions),
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_int)]
        _lib.b200_ycbcr_to_rgb_coefficients.argtypes = [C.c_int, C.c_int, C.POINTER(C.c_float)]
        _lib.b200_ycbcr_to_rgb_coefficients.restype = None
        _lib.b200_rgb_to_ycbcr_device.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(Planes), C.c_void_p]
        _lib.b200_rgb_to_ycbcr_host.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.POINTER(Planes)]
        _lib.b200_rgb_to_ycbcr_plan.argtypes = [C.POINTER(RgbImage), C.POINTER(Planes), C.POINTER(RgbToYCbCrOptions), C.POINTER(C.c_int)]
        _lib.b200_rgb_to_ycbcr_ex_device.argtypes = [C.POINTER(RgbImage), C.POINTER(Planes), C.POINTER(RgbToYCbCrOptions), C.c_void_p,
                                                     C.POINTER(C.c_int)]
        _lib.b200_rgb_to_ycbcr_ex_host.argtypes = [C.POINTER(RgbImage), C.POINTER(Planes), C.POINTER(RgbToYCbCrOptions), C.POINTER(C.c_int)]
    return _lib


def check(rc):
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))
