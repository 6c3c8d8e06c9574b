"""Colour post-stage: host mirror of libheif's convert_colorspace()/rotate_ccw()/mirror_inplace()/crop().

Reference interfaces mirrored (argument meaning and order of application):
  convert_colorspace(img, colorspace, chroma, ...)        libheif/color-conversion/colorconversion.cc:490-623
  HeifPixelImage::rotate_ccw / mirror_inplace / crop      libheif/image/pixelimage.cc:1175-1546
  ImageItem::decode_image transform loop                  libheif/image-items/image_item.cc:947-1020
"""
import ctypes as C
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import _lib

CHROMA_MONO, CHROMA_420, CHROMA_422, CHROMA_444 = 0, 1, 2, 3
CHROMA_INTERLEAVED_RGB, CHROMA_INTERLEAVED_RGBA = 10, 11
CHROMA_INTERLEAVED_RRGGBB_BE, CHROMA_INTERLEAVED_RRGGBBAA_BE = 12, 13
CHROMA_INTERLEAVED_RRGGBB_LE, CHROMA_INTERLEAVED_RRGGBBAA_LE = 14, 15

_BYTES_PER_PIXEL = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}


class Geometry:
    """Chain of irot / imir / clap transforms, composed in the order libheif applies them."""

    def __init__(self, width: int, height: int, chroma: int = 1):
        """chroma: B200_CHROMA_* of the picture the chain applies to (decides where the reference converts to 4:4:4 first)."""
        self.g = _lib.Geometry()
        _lib.lib().b200_geometry_init(width, height, chroma, C.byref(self.g))

    def rotate_ccw(self, degrees: int) -> "Geometry":
        _lib.check(_lib.lib().b200_geometry_rotate_ccw(C.byref(self.g), degrees))
        return self

    def mirror(self, direction: int) -> "Geometry":
        """direction: heif_transform_mirror_direction (0 = vertical: top<->bottom, 1 = horizontal: left<->right)."""
        _lib.check(_lib.lib().b200_geometry_mirror(C.byref(self.g), direction))
        return self

    def crop(self, left: int, right: int, top: int, bottom: int) -> "Geometry":
        _lib.check(_lib.lib().b200_geometry_crop(C.byref(self.g), left, right, top, bottom))
        return self

    @property
    def size(self):
        return self.g.out_w, self.g.out_h


@dataclass
class YCbCrImage:
    """Decoded picture as the decoder plugin hands it over (decoder_libde265.cc:97-171): planes + nclx."""
    y: object
    cb: Optional[object] = None
    cr: Optional[object] = None
    alpha: Optional[object] = None
    chroma: int = CHROMA_420
    bit_depth: int = 8
    colour_primaries: int = 2
    transfer_characteristics: int = 2
    matrix_coefficients: int = 2
    full_range: bool = False
    _keep: list = field(default_factory=list, repr=False)


class _Host:
    """numpy arrays, converted by the _host entry points (which stage them through the GPU inside the call)."""
    u8, u16, rgb16 = np.uint8, np.uint16, np.uint16     # rgb16: convert_colorspace_host's 16-bit planar RGB

    ptr = staticmethod(lambda a: a.ctypes.data)
    stride = staticmethod(lambda a: a.strides[0])

    @staticmethod
    def is16(a):
        if a.dtype not in (np.uint8, np.uint16):
            raise ValueError("uint8 / uint16 arrays only")
        return a.dtype == np.uint16

    @staticmethod
    def packed(a):
        return a.strides[-1] == a.itemsize and (a.ndim == 2 or a.strides[1] == a.shape[2] * a.itemsize)

    @staticmethod
    def empty(shape, dtype):
        return np.empty(shape, dtype)

    @staticmethod
    def call(name, *args, pipeline=True):
        """name + "_host"(*args[, &pipeline]); returns the pipeline mask"""
        pipe = C.c_int(0)
        _lib.check(getattr(_lib.lib(), name + "_host")(*args, *((C.byref(pipe),) if pipeline else ())))
        return pipe.value


class _Cuda:
    """CUDA tensors on `device`, converted by the _device entry points on `stream` (default: the device's current stream)."""

    def __init__(self, device, stream=None):
        import torch
        self.torch, self.device, self.stream = torch, device, stream
        self.u8, self.u16, self.rgb16 = torch.uint8, torch.uint16, torch.int16   # rgb16: convert_colorspace's 16-bit planar RGB

    ptr = staticmethod(lambda t: t.data_ptr())
    stride = staticmethod(lambda t: t.stride(0) * t.element_size())
    is16 = staticmethod(lambda t: t.element_size() == 2)
    packed = staticmethod(lambda t: t.stride(-1) == 1 and (t.dim() == 2 or t.stride(1) == t.shape[2]))

    def empty(self, shape, dtype):
        return self.torch.empty(shape, dtype=dtype, device=self.device)

    def call(self, name, *args, pipeline=True):
        """name + "_device"(*args, stream[, &pipeline]); returns the pipeline mask"""
        s = self.stream if self.stream is not None else self.torch.cuda.current_stream(self.device)
        pipe = C.c_int(0)
        with self.torch.cuda.device(self.device):
            _lib.check(getattr(_lib.lib(), name + "_device")(*args, C.c_void_p(s.cuda_stream), *((C.byref(pipe),) if pipeline else ())))
        return pipe.value


_HOST = _Host()


def _fill_planes(img: YCbCrImage, mem):
    p = _lib.Planes()
    h, w = img.y.shape
    p.y = mem.ptr(img.y); p.y_stride = mem.stride(img.y)
    if img.chroma != CHROMA_MONO:
        p.cb = mem.ptr(img.cb); p.cr = mem.ptr(img.cr); p.c_stride = mem.stride(img.cb)
        assert mem.stride(img.cb) == mem.stride(img.cr)
    if img.alpha is not None:
        p.alpha = mem.ptr(img.alpha); p.alpha_stride = mem.stride(img.alpha)
    p.width, p.height, p.chroma, p.bit_depth = w, h, img.chroma, img.bit_depth
    p.colour_primaries, p.transfer_characteristics = img.colour_primaries, img.transfer_characteristics
    p.matrix_coefficients, p.full_range = img.matrix_coefficients, int(bool(img.full_range))
    return p


def _out_shape(out_chroma, w, h, bit_depth):
    """(shape, whether the samples are 16 bit) of the conversion's output"""
    if out_chroma == CHROMA_444:
        return (3, h, w), bit_depth > 8
    return (h, w * _BYTES_PER_PIXEL[out_chroma]), False


def _convert(mem, img: YCbCrImage, out_chroma: int, geometry: Optional[Geometry], out=None, bilinear: bool = False, scale=None):
    h, w = img.y.shape
    geom = geometry or Geometry(w, h)
    if out is None:
        shape, wide = _out_shape(out_chroma, *(scale or geom.size), img.bit_depth)
        out = mem.empty(shape, mem.rgb16 if wide else mem.u8)
    if out_chroma == CHROMA_444:
        o, og, ob = mem.ptr(out[0]), mem.ptr(out[1]), mem.ptr(out[2])
    else:
        o, og, ob = mem.ptr(out), None, None
    opt = _lib.ColorOptions(out_chroma, 0, 1 if bilinear else 0)
    head = (C.byref(_fill_planes(img, mem)), C.byref(geom.g), C.byref(opt))
    stride = mem.stride(out[0] if out_chroma == CHROMA_444 else out)
    if scale is None:
        pipe = mem.call("b200_color_convert", *head, o, og, ob, stride)
    else:
        pipe = mem.call("b200_color_convert_scaled", *head, int(scale[0]), int(scale[1]), o, og, ob, stride)
    return out, pipe


def convert_colorspace(img: YCbCrImage, out_chroma: int, geometry: Optional[Geometry] = None, out=None, stream=None, bilinear: bool = False,
                       scale=None):
    """Device -> device. `img` planes are CUDA torch tensors (uint8, or int16/uint16 for >8 bit).

    scale=(w, h): the result scaled to w x h as heif_image_scale_image (HeifPixelImage::scale_nearest_neighbor) would scale
    the unscaled one, converting only the pixels it keeps (b200_color_convert_scaled_device).
    Returns a CUDA uint8 tensor [H, W*bytes_per_pixel] (interleaved) or [3, H, W] (planar RGB 4:4:4), H x W = the scaled size
    when scale is given."""
    return _convert(_Cuda(img.y.device, stream), img, out_chroma, geometry, out, bilinear, scale)[0]


def convert_colorspace_host(img: YCbCrImage, out_chroma: int, geometry: Optional[Geometry] = None):
    """Host -> host through the C ABI (H2D + kernel + D2H inside the call). Planes are numpy arrays."""
    return _convert(_HOST, img, out_chroma, geometry)


def _ycc_out_planes(w, h, out_chroma, want_alpha, alloc):
    sh = 0 if out_chroma == CHROMA_444 else 1
    sv = 1 if out_chroma == CHROMA_420 else 0
    y = alloc((h, w))
    cb = alloc(((h + sv) >> sv, (w + sh) >> sh))
    cr = alloc(((h + sv) >> sv, (w + sh) >> sh))
    a = alloc((h, w)) if want_alpha else None
    return y, cb, cr, a


def _rgb_to_ycbcr(mem, rgb, out_chroma, matrix_coefficients, colour_primaries, full_range, want_alpha) -> YCbCrImage:
    assert rgb.dtype == mem.u8 and rgb.ndim == 3 and rgb.shape[2] in (3, 4) and mem.packed(rgb)
    h, w, bpp = rgb.shape
    if want_alpha is None:
        want_alpha = bpp == 4
    y, cb, cr, a = _ycc_out_planes(w, h, out_chroma, want_alpha, lambda s: mem.empty(s, mem.u8))
    img = YCbCrImage(y, cb, cr, a, chroma=out_chroma, bit_depth=8, colour_primaries=colour_primaries,
                     matrix_coefficients=matrix_coefficients, full_range=full_range)
    mem.call("b200_rgb_to_ycbcr", C.c_void_p(mem.ptr(rgb)), C.c_size_t(mem.stride(rgb)), int(bpp == 4), C.byref(_fill_planes(img, mem)),
             pipeline=False)
    return img


def rgb_to_ycbcr(rgb, out_chroma: int = CHROMA_420, matrix_coefficients: int = 6, colour_primaries: int = 1, full_range: bool = True,
                 want_alpha: Optional[bool] = None, stream=None) -> YCbCrImage:
    """Encoder-side direction, device -> device: interleaved RGB / RGBA (CUDA uint8 tensor [H, W, 3 or 4]) -> YCbCrImage of
    CUDA uint8 planes, as Op_RGB24_32_to_YCbCr does (libheif/color-conversion/rgb2yuv.cc:575-808).
    want_alpha: None = an alpha plane iff the source has one (what the reference's planner targets for has_alpha)."""
    return _rgb_to_ycbcr(_Cuda(rgb.device, stream), rgb, out_chroma, matrix_coefficients, colour_primaries, full_range, want_alpha)


def rgb_to_ycbcr_host(rgb: np.ndarray, out_chroma: int = CHROMA_420, matrix_coefficients: int = 6, colour_primaries: int = 1,
                      full_range: bool = True, want_alpha: Optional[bool] = None) -> YCbCrImage:
    """Host -> host through the C ABI (H2D + kernel + D2H inside the call). rgb: uint8 [H, W, 3 or 4], rows may be strided."""
    return _rgb_to_ycbcr(_HOST, rgb, out_chroma, matrix_coefficients, colour_primaries, full_range, want_alpha)


# ---- every RGB layout heif_context_encode_image accepts (b200_rgb_to_ycbcr_ex_*) ----------------------------------------
# names of the reference operations behind the B200_YCC_PIPE_* bits, in chain order
YCC_PIPE_NAMES = ((32, "Op_RRGGBBaa_swap_endianness"), (16, "Op_RRGGBBaa_BE_to_RGB_HDR / Op_RGB24_32_to_RGB"),
                  (1, "Op_RGB24_32_to_YCbCr"), (2, "Op_RGB24_32_to_YCbCr444_GBR"), (4, "Op_RRGGBBxx_HDR_to_YCbCr420"),
                  (8, "Op_RGB_to_YCbCr"))


def _rgb_image(rgb, bit_depth, endianness, alpha_bit_depth, ptr, stride, is16, packed):
    """b200_rgb_image for an interleaved [H, W, 3|4] array / tensor or a tuple (R, G, B[, A]) of [H, W] planes.
    packed(a): the samples of a row (and the components of a pixel) are adjacent in memory."""
    d = _lib.RgbImage()
    if isinstance(rgb, (tuple, list)):
        if len(rgb) not in (3, 4) or any(p.ndim != 2 or p.shape != rgb[0].shape or not packed(p) for p in rgb):
            raise ValueError("planar input: 3 or 4 [H, W] planes of one size, samples adjacent within a row")
        if is16(rgb[0]) and bit_depth is None:
            raise ValueError("16-bit planes need bit_depth (9..16)")
        depth, adepth = bit_depth or 8, alpha_bit_depth or bit_depth or 8
        if any(is16(p) != (depth > 8) for p in rgb[:3]) or (len(rgb) == 4 and is16(rgb[3]) != (adepth > 8)):
            raise ValueError("planar input: uint8 planes at 8 bit, uint16 above (alpha at alpha_bit_depth)")
        d.r, d.g, d.b = ptr(rgb[0]), ptr(rgb[1]), ptr(rgb[2])
        d.r_stride, d.g_stride, d.b_stride = stride(rgb[0]), stride(rgb[1]), stride(rgb[2])
        if len(rgb) == 4:
            d.alpha, d.alpha_stride = ptr(rgb[3]), stride(rgb[3])
        d.height, d.width = rgb[0].shape
        d.chroma = CHROMA_444
        d.bit_depth = bit_depth or 8
        d.alpha_bit_depth = alpha_bit_depth or 0
        return d, len(rgb) == 4
    if rgb.ndim != 3 or rgb.shape[2] not in (3, 4) or not packed(rgb):
        raise ValueError("interleaved input: [H, W, 3 or 4], pixels and their components adjacent within a row")
    h, w, nch = rgb.shape
    if is16(rgb):
        if endianness not in ("little", "big") or bit_depth is None:
            raise ValueError("16-bit interleaved input needs endianness ('little' / 'big': the byte order of the samples as stored) and bit_depth")
        d.chroma = {(3, "big"): CHROMA_INTERLEAVED_RRGGBB_BE, (4, "big"): CHROMA_INTERLEAVED_RRGGBBAA_BE,
                    (3, "little"): CHROMA_INTERLEAVED_RRGGBB_LE, (4, "little"): CHROMA_INTERLEAVED_RRGGBBAA_LE}[(nch, endianness)]
        d.bit_depth = bit_depth
    else:
        if bit_depth not in (None, 8):
            raise ValueError("uint8 interleaved input is RGB / RGBA at 8 bit")
        d.chroma = CHROMA_INTERLEAVED_RGB if nch == 3 else CHROMA_INTERLEAVED_RGBA
        d.bit_depth = 8
    d.rgb, d.rgb_stride = ptr(rgb), stride(rgb)
    d.width, d.height = w, h
    return d, nch == 4


def _ycc_target(img_planes, w, h, out_chroma, bit_depth, mc, cp, full):
    p = _lib.Planes()
    if img_planes is not None:
        y, cb, cr, a, ptr, stride = img_planes
        p.y, p.cb, p.cr = ptr(y), ptr(cb), ptr(cr)
        p.y_stride, p.c_stride = stride(y), stride(cb)
        if a is not None:
            p.alpha, p.alpha_stride = ptr(a), stride(a)
    p.width, p.height, p.chroma, p.bit_depth = w, h, out_chroma, bit_depth
    p.colour_primaries, p.transfer_characteristics, p.matrix_coefficients, p.full_range = cp, 2, mc, int(bool(full))
    return p


def rgb_to_ycbcr_plan(rgb, out_chroma: int = CHROMA_420, bit_depth: Optional[int] = None, endianness: Optional[str] = None,
                      matrix_coefficients: int = 6, colour_primaries: int = 1, full_range: bool = True, chroma_downsampling: int = 2,
                      only_use_preferred: bool = False, alpha_bit_depth: Optional[int] = None) -> int:
    """Host only: the B200_YCC_PIPE_* mask of the reference chain for this input (numpy arrays, arguments as for
    rgb_to_ycbcr_ex; no pixel is read); raises B200Error (code -2) where the conversion is refused."""
    d, _ = _rgb_image(rgb, bit_depth, endianness, alpha_bit_depth, _HOST.ptr, _HOST.stride, _HOST.is16, _HOST.packed)
    t = _ycc_target(None, d.width, d.height, out_chroma, d.bit_depth, matrix_coefficients, colour_primaries, full_range)
    opt = _lib.RgbToYCbCrOptions(chroma_downsampling, int(bool(only_use_preferred)))
    pipe = C.c_int(0)
    _lib.check(_lib.lib().b200_rgb_to_ycbcr_plan(C.byref(d), C.byref(t), C.byref(opt), C.byref(pipe)))
    return pipe.value


def _rgb_to_ycbcr_ex(mem, rgb, out_chroma, bit_depth, endianness, matrix_coefficients, colour_primaries, full_range, chroma_downsampling,
                     only_use_preferred, alpha_bit_depth):
    d, has_alpha = _rgb_image(rgb, bit_depth, endianness, alpha_bit_depth, mem.ptr, mem.stride, mem.is16, mem.packed)
    dt = mem.u16 if d.bit_depth > 8 else mem.u8
    y, cb, cr, a = _ycc_out_planes(d.width, d.height, out_chroma, has_alpha, lambda s: mem.empty(s, dt))
    img = YCbCrImage(y, cb, cr, a, chroma=out_chroma, bit_depth=d.bit_depth, colour_primaries=colour_primaries,
                     matrix_coefficients=matrix_coefficients, full_range=full_range)
    t = _ycc_target((y, cb, cr, a, mem.ptr, mem.stride), d.width, d.height, out_chroma, d.bit_depth, matrix_coefficients,
                    colour_primaries, full_range)
    opt = _lib.RgbToYCbCrOptions(chroma_downsampling, int(bool(only_use_preferred)))
    return img, mem.call("b200_rgb_to_ycbcr_ex", C.byref(d), C.byref(t), C.byref(opt))


def rgb_to_ycbcr_ex(rgb, out_chroma: int = CHROMA_420, bit_depth: Optional[int] = None, endianness: Optional[str] = None,
                    matrix_coefficients: int = 6, colour_primaries: int = 1, full_range: bool = True, chroma_downsampling: int = 2,
                    only_use_preferred: bool = False, alpha_bit_depth: Optional[int] = None, stream=None):
    """Encoder-side direction for every RGB layout, device -> device (b200_rgb_to_ycbcr_ex_device): what convert_colorspace
    does before heif_context_encode_image hands the picture to an encoder (libheif/codecs/encoder.cc:116-175).

    rgb: CUDA tensor [H, W, 3|4] (uint8: RGB / RGBA 8 bit; uint16: RRGGBB[AA], with `endianness` naming the byte order the
    samples are stored in and `bit_depth` 9..16), or a tuple (R, G, B[, A]) of [H, W] planes (uint8, or uint16 with bit_depth).
    Returns (YCbCrImage at the input depth -- uint16 planes above 8 bit, an alpha plane when the input has one --,
    B200_YCC_PIPE_* mask of the reference chain that was mirrored)."""
    import torch
    first = rgb[0] if isinstance(rgb, (tuple, list)) else rgb
    for t in (rgb if isinstance(rgb, (tuple, list)) else (rgb,)):
        if t.device != first.device or t.device.type != "cuda" or t.dtype not in (torch.uint8, torch.uint16):
            raise ValueError("rgb_to_ycbcr_ex: uint8 / uint16 CUDA tensors on one device")
    return _rgb_to_ycbcr_ex(_Cuda(first.device, stream), rgb, out_chroma, bit_depth, endianness, matrix_coefficients, colour_primaries,
                            full_range, chroma_downsampling, only_use_preferred, alpha_bit_depth)


def rgb_to_ycbcr_ex_host(rgb, out_chroma: int = CHROMA_420, bit_depth: Optional[int] = None, endianness: Optional[str] = None,
                         matrix_coefficients: int = 6, colour_primaries: int = 1, full_range: bool = True, chroma_downsampling: int = 2,
                         only_use_preferred: bool = False, alpha_bit_depth: Optional[int] = None):
    """Host -> host form of rgb_to_ycbcr_ex (b200_rgb_to_ycbcr_ex_host: H2D + kernel + D2H inside the call); numpy input,
    rows may be strided."""
    return _rgb_to_ycbcr_ex(_HOST, rgb, out_chroma, bit_depth, endianness, matrix_coefficients, colour_primaries, full_range,
                            chroma_downsampling, only_use_preferred, alpha_bit_depth)
