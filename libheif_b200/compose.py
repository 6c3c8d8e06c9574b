"""Overlay compositing and nearest-neighbour scaling on the GPU (ctypes mirror of include/b200_heif.h, section a11/a12).

Reference: HeifPixelImage::fill_RGB_16bit / overlay / scale_nearest_neighbor (libheif/image/pixelimage.cc:1549-1972),
driven by ImageItem_Overlay::decode_overlay_image (libheif/image-items/overlay.cc:290-393).
"""
import ctypes as C
from ._lib import lib, check


def _stream():
    import torch   # deferred: the package must stay importable in processes that only use the host-side C ABI
    return torch.cuda.current_stream().cuda_stream


def _planes(ts, n):
    ptrs = (C.c_void_p * n)(*[t.data_ptr() if t is not None else None for t in ts])
    strides = (C.c_size_t * n)(*[t.stride(0) * t.element_size() if t is not None else 0 for t in ts])
    return ptrs, strides


def overlay_canvas(width, height, background_rgba, device="cuda:0"):
    """8-bit planar RGB canvas (3, H, W) filled with background >> 8 (fill_RGB_16bit)."""
    import torch
    canvas = torch.empty((3, height, width), dtype=torch.uint8, device=device)
    ptrs, strides = _planes([canvas[0], canvas[1], canvas[2]], 3)
    bkg = (C.c_uint16 * 4)(*[int(v) & 0xffff for v in background_rgba])
    check(lib().b200_overlay_fill_device(ptrs, strides, width, height, bkg, _stream()))
    return canvas


def overlay(canvas, child_rgb, dx, dy, child_alpha=None):
    """Composite child_rgb (3, h, w) uint8 [+ alpha (h, w)] onto canvas (3, H, W) at (dx, dy), in place (HeifPixelImage::overlay)."""
    import torch
    assert canvas.dtype == torch.uint8 and child_rgb.dtype == torch.uint8 and canvas.is_cuda and child_rgb.is_cuda
    cp, cs = _planes([canvas[0], canvas[1], canvas[2]], 3)
    op, os_ = _planes([child_rgb[0], child_rgb[1], child_rgb[2], child_alpha], 4)
    check(lib().b200_overlay_device(cp, cs, canvas.shape[2], canvas.shape[1], op, os_, child_rgb.shape[2], child_rgb.shape[1],
                                    dx, dy, _stream()))
    return canvas


def scale_nearest_plane(plane, out_w, out_h, image_in, image_out, components=1):
    """One plane (h, w*components) of uint8 / uint16 scaled with the reference's index arithmetic; image_in / image_out = (W, H) of the IMAGE."""
    import torch
    assert plane.is_cuda and plane.dim() == 2
    out = torch.empty((out_h, out_w * components), dtype=plane.dtype, device=plane.device)
    bpp = components * plane.element_size()
    check(lib().b200_scale_nearest_device(plane.data_ptr(), plane.stride(0) * plane.element_size(), out.data_ptr(), out.stride(0) * out.element_size(),
                                          out_w, out_h, image_in[0], image_in[1], image_out[0], image_out[1], bpp, _stream()))
    return out


def thumbnail_size(width, height, size):
    """(w, h) heif-thumbnailer scales a width x height picture to for a thumbnail of `size` (examples/heif_thumbnailer.cc:169-191):
    the long side becomes `size`, the other side other * size // long; a picture that fits is left as it is.  Raises
    ValueError where the reference gives up with "Zero thumbnail output size"."""
    if width <= size and height <= size:
        return width, height
    if width > height:
        w, h = size, height * size // width
    else:
        w, h = width * size // height, size
    if w == 0 or h == 0:
        raise ValueError(f"{width} x {height} at size {size}: zero thumbnail output size")
    return w, h
