"""rgb_to_ycbcr_ex / rgb_to_ycbcr_ex_host (b200_rgb_to_ycbcr_ex_device / _host) against the unmodified reference's
convert_colorspace on the same RGB input (oracle/ref_encode.cc), byte for byte, with the chain it reports."""
import itertools

import numpy as np
import pytest

import libheif_b200 as lb
from oracle import ref_encode
from rgb_ex_cases import LAYOUTS, MATRICES, make_input, ref_mask

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(ref_encode.lib() is None, reason="oracle/_ref/liboracle_encode.so not built")]


def to_dev(a, cuda):
    import torch
    if a.dtype == np.uint16:
        return torch.from_numpy(np.ascontiguousarray(a).view(np.int16)).to(cuda).view(torch.uint16)
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def to_np(t):
    import torch
    if t.dtype == torch.uint16:
        return t.view(torch.int16).cpu().numpy().view(np.uint16)
    return t.cpu().numpy()


def dev_input(ex_in, cuda):
    return tuple(to_dev(p, cuda) for p in ex_in) if isinstance(ex_in, tuple) else to_dev(ex_in, cuda)


def check(img, ref, what, host=False):
    got = [img.y, img.cb, img.cr, img.alpha]
    if not host:
        got = [None if g is None else to_np(g) for g in got]
    for name, g, r in zip(("Y", "Cb", "Cr", "alpha"), got, ref[:4]):
        assert (g is None) == (r is None), f"{what}: {name} presence"
        if r is not None:
            assert g.dtype == r.dtype and np.array_equal(g, r), f"{what}: {name} differs ({np.count_nonzero(g != r)} samples)"


def img_from(planes):
    return lb.YCbCrImage(planes[0], planes[1], planes[2], planes[3])


def run_case(cuda, ref_in, ex_in, endian, chroma, depth, out_chroma, mc, full, ds=2, only=0, host=True):
    ref = ref_encode.ref_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full), ds, only)
    want = None if ref is None else ref_mask(ref[4])
    what = f"chroma={chroma} depth={depth} -> {out_chroma} mc={mc} full={full} opt={(ds, only)} ref={None if ref is None else ref[4]}"
    kw = dict(out_chroma=out_chroma, bit_depth=depth, endianness=endian, matrix_coefficients=mc, colour_primaries=1,
              full_range=bool(full), chroma_downsampling=ds, only_use_preferred=bool(only))
    if want is None:
        with pytest.raises(lb.B200Error) as e:
            lb.rgb_to_ycbcr_ex(dev_input(ex_in, cuda), **kw)
        assert e.value.code == -2, what
        return
    co = ref_encode.oracle_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full), ds, only)
    assert co is not None and co[4] == want, what
    check(img_from(co), ref, what + " (C restatement)", host=True)
    img, pipe = lb.rgb_to_ycbcr_ex(dev_input(ex_in, cuda), **kw)
    assert pipe == want, what
    check(img, ref, what)
    if host:
        himg, hpipe = lb.rgb_to_ycbcr_ex_host(ex_in, **kw)
        assert hpipe == want, what
        check(himg, ref, what + " (host)", host=True)


@pytest.mark.parametrize("label,chroma,depth,alpha", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_matches_reference(cuda, label, chroma, depth, alpha):
    for k, (w, h) in enumerate(((1, 1), (1, 6), (7, 1), (17, 9))):
        ref_in, ex_in, endian = make_input(100 + k, w, h, chroma, depth, alpha)
        for out_chroma, mc, full in itertools.product((1, 2, 3), MATRICES, (0, 1)):
            run_case(cuda, ref_in, ex_in, endian, chroma, depth, out_chroma, mc, full)


@pytest.mark.parametrize("chroma,depth,alpha,out_chroma,mc,full", [
    (14, 10, False, 1, 9, 1),     # Op_RRGGBBxx_HDR_to_YCbCr420
    (14, 10, False, 1, 9, 0),     # swap + unpack + Op_RGB_to_YCbCr<uint16_t>
    (13, 12, True, 2, 1, 1),
    (3, 16, True, 2, 6, 0),
    (3, 8, False, 1, 0, 0),
    (11, 8, True, 1, 8, 1),
    (10, 8, False, 3, 0, 1),      # Op_RGB24_32_to_YCbCr444_GBR
    (10, 8, False, 1, 6, 0),      # Op_RGB24_32_to_YCbCr
])
def test_large_picture(cuda, chroma, depth, alpha, out_chroma, mc, full):
    ref_in, ex_in, endian = make_input(7, 4097, 2051, chroma, depth, alpha)
    run_case(cuda, ref_in, ex_in, endian, chroma, depth, out_chroma, mc, full)


@pytest.mark.parametrize("label,chroma,depth,alpha", [l for l in LAYOUTS if l[0] in ("rgba8", "rrggbb_le10", "rrggbbaa_be16", "planar10", "planara8")])
def test_unaligned_rows_and_pointers(cuda, label, chroma, depth, alpha):
    import torch
    w, h = 45, 13
    ref_in, ex_in, endian = make_input(11, w, h, chroma, depth, alpha)
    for out_chroma, mc, full in ((1, 6, 1), (1, 9, 0), (2, 0, 0), (3, 8, 1)):
        ref = ref_encode.ref_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full))
        kw = dict(out_chroma=out_chroma, bit_depth=depth, endianness=endian, matrix_coefficients=mc, colour_primaries=1, full_range=bool(full))
        # rows padded by 3 samples and starting one sample (one pixel) into the allocation
        if isinstance(ex_in, tuple):
            pads = [np.zeros((h, w + 3), p.dtype) for p in ex_in]
            for q, p in zip(pads, ex_in):
                q[:, 1:w + 1] = p
            host_in = tuple(q[:, 1:w + 1] for q in pads)
            dev_in = tuple(to_dev(q, cuda)[:, 1:w + 1] for q in pads)
        else:
            q = np.zeros((h, w + 3, ex_in.shape[2]), ex_in.dtype)
            q[:, 1:w + 1] = ex_in
            host_in = q[:, 1:w + 1]
            dev_in = to_dev(q, cuda)[:, 1:w + 1]
        img, pipe = lb.rgb_to_ycbcr_ex(dev_in, **kw)
        assert pipe == ref_mask(ref[4])
        check(img, ref, f"{label} -> {out_chroma} mc={mc} (device, unaligned)")
        himg, _ = lb.rgb_to_ycbcr_ex_host(host_in, **kw)
        check(himg, ref, f"{label} -> {out_chroma} mc={mc} (host, unaligned)", host=True)
        torch.cuda.synchronize()


def test_host_rows_longer_than_a_bounce_slot(cuda):
    # 8 bytes per pixel: an input row of 32 MiB + 40 bytes, more than one 32 MiB slot of the staging bounce buffer
    w, h = (32 << 20) // 8 + 5, 3
    ref_in, ex_in, endian = make_input(5, w, h, 15, 12, True)
    ref = ref_encode.ref_rgb_to_ycbcr_ex(ref_in, 15, 12, 1, (9, 16, 9, 0))
    himg, pipe = lb.rgb_to_ycbcr_ex_host(ex_in, 1, 12, endian, matrix_coefficients=9, colour_primaries=9, full_range=False)
    assert pipe == ref_mask(ref[4]) == 32 | 16 | 8
    check(himg, ref, "long rows (host)", host=True)


@pytest.mark.parametrize("case", ["mc11", "mc14", "alpha_depth", "average_420", "sharp_422", "alpha_plane_missing"])
def test_refusals(cuda, case):
    ref_in, ex_in, endian = make_input(3, 8, 6, 3, 10, True)
    kw = dict(out_chroma=1, bit_depth=10, matrix_coefficients=6)
    if case in ("mc11", "mc14"):
        kw["matrix_coefficients"] = int(case[2:])
        assert ref_encode.ref_rgb_to_ycbcr_ex(ref_in, 3, 10, 1, (1, 13, kw["matrix_coefficients"], 1)) is None
    elif case == "alpha_depth":
        ex_in = ex_in[:3] + ((ex_in[3] >> 2).astype(np.uint8),)
        kw["alpha_bit_depth"] = 8
    elif case == "average_420":
        kw.update(chroma_downsampling=2, only_use_preferred=True)
    elif case == "sharp_422":
        kw.update(out_chroma=2, chroma_downsampling=3, only_use_preferred=True)
        assert ref_encode.ref_rgb_to_ycbcr_ex(ref_in, 3, 10, 2, (1, 13, 6, 1), 3, 1) is None
    if case == "alpha_plane_missing":
        # the result has an alpha plane whenever the input has one: the device call needs somewhere to put it
        import ctypes as C
        from libheif_b200 import _lib
        d, _ = lb.color._rgb_image(dev_input(ex_in, cuda), 10, None, None, lambda t: t.data_ptr(), lambda t: t.stride(0) * t.element_size(),
                                   lambda t: t.element_size() == 2, lambda t: True)
        y = to_dev(np.zeros((6, 8), np.uint16), cuda)
        c = to_dev(np.zeros((3, 4), np.uint16), cuda)
        t = lb.color._ycc_target((y, c, c.clone(), None, lambda x: x.data_ptr(), lambda x: x.stride(0) * 2), 8, 6, 1, 10, 6, 1, True)
        rc = _lib.lib().b200_rgb_to_ycbcr_ex_device(C.byref(d), C.byref(t), None, None, None)
        assert rc == -1
        return
    with pytest.raises(lb.B200Error) as e:
        lb.rgb_to_ycbcr_ex(dev_input(ex_in, cuda), **kw)
    assert e.value.code == -2
    with pytest.raises(lb.B200Error) as e:
        lb.rgb_to_ycbcr_ex_host(ex_in, **kw)
    assert e.value.code == -2
