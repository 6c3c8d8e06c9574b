"""Scaled decode: the colour stage fused with the reference's nearest-neighbour scaler (heif_decode_image followed by
heif_image_scale_image, as heif-thumbnailer runs them; HeifPixelImage::scale_nearest_neighbor, libheif/image/pixelimage.cc:1783-1972).

CPU: thumbnail_size (examples/heif_thumbnailer.cc:169-191) and the argument checks of the two scaled entry points, which
refuse before any CUDA call.
GPU: b200_color_convert_scaled_device against the unmodified reference (geometry + convert_colorspace, then
scale_nearest_neighbor; skipped without oracle/_ref), against the unscaled call at the identity size, and against the
two-step device route (b200_color_convert_device + b200_scale_nearest_device); b200_decode_grid_to_rgb_scaled_host on
single pictures and grids into pageable and page-locked memory.
"""
import ctypes as C
import hashlib

import numpy as np
import pytest

import libheif_b200 as lb
from libheif_b200 import _lib
from oracle import bindings as ob
from util import random_ycbcr, ref_plugin, ref_postprocess

needs_ref = pytest.mark.skipif(ref_plugin() is None, reason="oracle/_ref reference build not present")

BPP = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}


# ---------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("size,want", [
    ((1280, 854, 256), (256, 170)),          # example.heic's primary item
    ((4000, 3000, 512), (512, 384)),         # wide
    ((3000, 4000, 512), (384, 512)),         # tall
    ((1000, 1000, 300), (300, 300)),         # square
    ((200, 100, 256), (200, 100)),           # fits: unchanged
    ((256, 256, 256), (256, 256)),           # fits exactly
    ((1000, 4, 256), (256, 1)),              # 1-pixel result
    ((3, 999, 333), (1, 333)),
])
def test_thumbnail_size(size, want):
    assert lb.thumbnail_size(*size) == want


def test_thumbnail_size_zero_side_is_refused():
    with pytest.raises(ValueError):           # heif-thumbnailer: "Zero thumbnail output size"
        lb.thumbnail_size(1000, 3, 256)


def _refusal(rc):
    """(code, message) of a call that must have returned before touching CUDA: without a device any CUDA call gives -4."""
    return rc, _lib.lib().b200_last_error().decode()


@pytest.mark.parametrize("sw,sh,name", [(0, 5, "scale_w"), (-3, 5, "scale_w"), (5, 0, "scale_h"), (5, -1, "scale_h")])
def test_color_scaled_refuses_bad_sizes(sw, sh, name):
    p, g, o = _lib.Planes(), _lib.Geometry(), _lib.ColorOptions(10, 0, 0)
    p.width, p.height, p.chroma, p.bit_depth = 4, 4, 1, 8
    g.out_w = g.out_h = 4
    rc, msg = _refusal(_lib.lib().b200_color_convert_scaled_device(C.byref(p), C.byref(g), C.byref(o), sw, sh, C.c_void_p(16), None, None, 12,
                                                                   None, None))
    assert rc == -1 and name in msg, (rc, msg)


@pytest.mark.parametrize("missing", ["in", "geom", "opt", "out"])
def test_color_scaled_refuses_null(missing):
    p, g, o = _lib.Planes(), _lib.Geometry(), _lib.ColorOptions(10, 0, 0)
    args = {"in": C.byref(p), "geom": C.byref(g), "opt": C.byref(o), "out": C.c_void_p(16)}
    args[missing] = None
    rc, msg = _refusal(_lib.lib().b200_color_convert_scaled_device(args["in"], args["geom"], args["opt"], 2, 2, args["out"], None, None, 12,
                                                                   None, None))
    assert rc == -1 and msg.startswith(missing + " "), (rc, msg)


@pytest.mark.parametrize("sw,sh,missing,name", [(0, 2, None, "scale_w"), (2, -1, None, "scale_h"), (2, 2, "dec", "dec"), (2, 2, "au", "au"),
                                                (2, 2, "au_size", "au_size"), (2, 2, "opt", "opt"), (2, 2, "out", "out")])
def test_fused_scaled_refuses_before_any_cuda_call(sw, sh, missing, name):
    au = (C.c_char_p * 1)(b"\x00\x00\x00\x01\x40")
    size = (C.c_size_t * 1)(5)
    o = _lib.ColorOptions(10, 0, 0)
    out = np.empty(64, np.uint8)
    args = {"dec": C.c_void_p(16), "au": au, "au_size": size, "opt": C.byref(o), "out": out.ctypes.data}
    if missing:
        args[missing] = None
    else:
        args["dec"] = None                    # the size checks come first: nothing else is looked at
    rc, msg = _refusal(_lib.lib().b200_decode_grid_to_rgb_scaled_host(args["dec"], 1, 1, args["au"], args["au_size"], 0, 0, 0, None, args["opt"],
                                                                      sw, sh, args["out"], 6, None))
    assert rc == -1 and name in msg, (rc, msg)
    if missing:
        assert msg.startswith(name + " ")


# ---------------------------------------------------------------------------------------------------------------- cases
# Geometry chains (ops as in test_color_oracle: (1, deg) rotate, (2, dir) mirror, (3, l, r, t, b) crop) on a 34 x 18 picture:
# rotations and mirrors keep 4:2:0 / 4:2:2 planes aligned; the odd crop is the reference's 4:4:4 conversion point there.
W0, H0 = 34, 18
GEOMS = [("identity", []), ("rot90", [(1, 90)]), ("rot180", [(1, 180)]), ("rot270", [(1, 270)]), ("mirror", [(2, 1)]),
         ("oddcrop", [(3, 3, 30, 1, 16)])]
# scaled sizes, as functions of the unscaled size (Wg, Hg): odd sizes, non-integer down factors, up-scaling, 1 x 1, w = 1, h > Hg
SCALES = [lambda w, h: (w * 2 // 3 | 1, h * 3 // 5 | 1), lambda w, h: (w * 5 // 2 + 1, h * 7 // 3), lambda w, h: (1, 1),
          lambda w, h: (1, h // 2 + 1), lambda w, h: (w // 3 + 1, h + 13), lambda w, h: (w - 1, h - 1)]


def _cases():
    """(id, chroma, bpp, nclx, out_chroma, alpha, ops, bilinear, scale index): every input format at every depth, range and
    matrix, every target, every geometry and every kind of scaled size, cycled so that each appears with several others."""
    out = []
    k = 0
    for chroma in (1, 2, 3, 0):
        for bpp in (8, 10, 12):
            for full in (0, 1):
                targets = [10, 11, 3] if bpp == 8 else [14, 12, 15, 13, 3, 10, 11]
                if chroma == 0 and bpp > 8:
                    targets = [14, 12, 15, 13, 3]
                for outc in targets:
                    mc = (1, 6, 0, 8, 16)[k % 5]
                    gname, ops = GEOMS[k % len(GEOMS)]
                    # the reference's 4:4:4 conversion point: the odd crop, and 4:2:2 under a quarter turn
                    detour = (gname == "oddcrop" and chroma in (1, 2)) or (gname in ("rot90", "rot270") and chroma == 2)
                    if detour and mc in (0, 8, 16):
                        mc = 6                                  # limited range is refused there; the special matrices stay off it
                    bilinear = chroma == 1 and k % 7 == 3 and mc in (1, 6)
                    alpha = outc in (13, 15) or (outc == 11 and k % 2 == 0)
                    nclx = (1, 13, mc, full)
                    out.append((f"c{chroma}_b{bpp}_f{full}_m{mc}_o{outc}{'_a' if alpha else ''}_{gname}{'_bil' if bilinear else ''}_s{k % len(SCALES)}",
                                chroma, bpp, nclx, outc, alpha, ops, bilinear, k % len(SCALES)))
                    k += 1
    return out


CASES = _cases()


def _img(y, cb, cr, a, chroma, bpp, nclx, dev):
    import torch
    dt = np.uint8 if bpp == 8 else np.uint16

    def cv(p):
        if p is None:
            return None
        arr = np.ascontiguousarray(p.astype(dt))
        return torch.from_numpy(arr.view(np.int16) if bpp > 8 else arr).to(dev)
    cp, tc, mc, fr = nclx
    return lb.YCbCrImage(cv(y), cv(cb), cv(cr), cv(a), chroma=chroma, bit_depth=bpp, colour_primaries=cp,
                         transfer_characteristics=tc, matrix_coefficients=mc, full_range=bool(fr))


def _geom(chroma, ops):
    g = lb.Geometry(W0, H0, chroma)
    for o in ops:
        if o[0] == 1:
            g.rotate_ccw(o[1])
        elif o[0] == 2:
            g.mirror(o[1])
        else:
            g.crop(*o[1:5])
    return g


def _setup(case, dev):
    _, chroma, bpp, nclx, outc, alpha, ops, bilinear, si = case
    y, cb, cr, a = random_ycbcr(0x5CA1 + chroma * 31 + bpp, W0, H0, chroma, bpp, alpha=alpha)
    g = _geom(chroma, ops)
    return (y, cb, cr, a), _img(y, cb, cr, a, chroma, bpp, nclx, dev), g, SCALES[si](*g.size)


def _bytes(t):
    return t.cpu().numpy().view(np.uint8).reshape(-1)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_scaled_colour_matches_reference(cuda, case):
    """convert_colorspace(scale=) == the reference's geometry + convert_colorspace, then its scale_nearest_neighbor."""
    _, chroma, bpp, nclx, outc, alpha, ops, bilinear, _ = case
    (y, cb, cr, a), img, g, (sw, sh) = _setup(case, cuda)
    hdr8 = 1 if bpp > 8 and outc in (10, 11) else 0
    ref, rw, rh, npl = ref_postprocess(y, cb, cr, a, chroma, bpp, nclx, ops, outc, only_preferred=int(bilinear), upsampling=2, hdr_to_8bit=hdr8)
    assert (rw, rh) == g.size
    if outc == 3:
        depth = 8 if bpp == 8 else bpp
        planes = np.frombuffer(ref.tobytes(), np.uint8 if bpp == 8 else np.uint16).reshape(3, rh, rw)
        want = ob.ref_scale_nn(1, 3, depth, list(planes), rw, rh, sw, sh)
    else:
        wide = BPP[outc] > 4
        plane = np.frombuffer(ref.tobytes(), np.uint16 if wide else np.uint8).reshape(rh, -1)
        want = ob.ref_scale_nn(3, outc, 16 if wide else 8, [plane], rw, rh, sw, sh)
    got = lb.convert_colorspace(img, outc, g, bilinear=bilinear, scale=(sw, sh))
    assert tuple(got.shape[-2:]) == ((sh, sw) if outc == 3 else (sh, sw * BPP[outc]))
    got = _bytes(got)
    assert np.array_equal(got, want), f"first diffs at byte {np.argwhere(got != want)[:4].ravel().tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_identity_size_equals_unscaled(cuda, case):
    """scale = the geometry's size gives the unscaled call's bytes."""
    import torch
    _, chroma, bpp, nclx, outc, alpha, ops, bilinear, _ = case
    _, img, g, _ = _setup(case, cuda)
    full = lb.convert_colorspace(img, outc, g, bilinear=bilinear)
    same = lb.convert_colorspace(img, outc, g, bilinear=bilinear, scale=g.size)
    assert torch.equal(full, same)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_scaled_equals_two_step_device_route(cuda, case):
    """== b200_color_convert_device, then b200_scale_nearest_device on every plane (the same device buffers)."""
    import torch
    _, chroma, bpp, nclx, outc, alpha, ops, bilinear, _ = case
    _, img, g, (sw, sh) = _setup(case, cuda)
    full = lb.convert_colorspace(img, outc, g, bilinear=bilinear)
    if outc == 3:
        two = torch.stack([lb.compose.scale_nearest_plane(full[c], sw, sh, g.size, (sw, sh)) for c in range(3)])
    else:
        two = lb.compose.scale_nearest_plane(full, sw, sh, g.size, (sw, sh), BPP[outc])
    pipe_full, pipe_scaled = C.c_int(-1), C.c_int(-2)
    assert torch.equal(lb.convert_colorspace(img, outc, g, bilinear=bilinear, scale=(sw, sh)), two)
    # *pipeline reports the unscaled call's chain
    p = lb.color._fill_planes(img, lb.color._Cuda(cuda))
    o = _lib.ColorOptions(outc, 0, int(bilinear))
    scratch = torch.empty((3, sh + H0 * 3, (sw + W0 * 3) * 8), dtype=torch.uint8, device=cuda)
    s = torch.cuda.current_stream().cuda_stream
    planes = [scratch[c].data_ptr() for c in range(3)] if outc == 3 else [scratch.data_ptr(), None, None]
    _lib.check(_lib.lib().b200_color_convert_device(C.byref(p), C.byref(g.g), C.byref(o), *planes, scratch.stride(1), C.c_void_p(s), C.byref(pipe_full)))
    _lib.check(_lib.lib().b200_color_convert_scaled_device(C.byref(p), C.byref(g.g), C.byref(o), sw, sh, *planes, scratch.stride(1), C.c_void_p(s),
                                                           C.byref(pipe_scaled)))
    torch.cuda.synchronize()
    assert pipe_scaled.value == pipe_full.value


# ---------------------------------------------------------------------------------------------------------------- fused
def _nn(rgb, bpp, w, h):
    """scale_nearest_neighbor of an interleaved picture [H, W * bpp]: the reference's when it is built, else its index rule."""
    H, W = rgb.shape[0], rgb.shape[1] // bpp
    if ref_plugin() is not None:
        wide = bpp > 4
        plane = rgb.view(np.uint16) if wide else rgb
        outc = {3: 10, 4: 11, 6: 14, 8: 15}[bpp]
        return ob.ref_scale_nn(3, outc, 16 if wide else 8, [plane], W, H, w, h).reshape(h, w * bpp)
    iy = (np.arange(h, dtype=np.uint64) * H // h).astype(np.int64)
    ix = (np.arange(w, dtype=np.uint64) * W // w).astype(np.int64)
    return rgb.reshape(H, W, bpp)[iy][:, ix].reshape(h, w * bpp)


def _outs(h, row_bytes):
    """a pageable and a page-locked (b200_host_alloc) destination of h rows"""
    ptr = C.c_void_p()
    _lib.check(_lib.lib().b200_host_alloc(h * row_bytes, C.byref(ptr)))
    pinned = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(h, row_bytes))
    return [("pageable", np.zeros((h, row_bytes), np.uint8), None), ("page-locked", pinned, ptr)]


def _scaled_both_ways(dec, aus, cols, rows, outc, w, h, **kw):
    """the scaled fused call into pageable and page-locked memory: both results, which must agree"""
    res = []
    for _, out, ptr in _outs(h, w * BPP[outc]):
        try:
            out[:] = 0
            dec.decode_grid_to_rgb_host(aus, cols, rows, outc, out=out, scale=(w, h), **kw)
            res.append(out.copy())
        finally:
            if ptr is not None:
                _lib.lib().b200_host_free(ptr)
    assert np.array_equal(res[0], res[1])
    return res[0]


@pytest.fixture(scope="module")
def dec(cuda):
    d = lb.Decoder(host_threads=8)
    yield d
    d.close()


@pytest.mark.gpu
def test_fused_example_heic_thumbnail(dec):
    """example.heic's primary item -> 256 x 170: == scale_nearest_neighbor of the full-size fused RGB, whose md5 is the
    reference's heif_decode_image result."""
    from hevc_cases import all_streams
    au = dict(all_streams())["example_primary_1280x854.au"]
    full = np.empty((854, 1280 * 3), np.uint8)
    dec.decode_grid_to_rgb_host([au], 1, 1, lb.CHROMA_INTERLEAVED_RGB, out=full)
    assert hashlib.md5(full.tobytes()).hexdigest() == "01672ec0cdf97b977628957cd6533dc2"
    w, h = lb.thumbnail_size(1280, 854, 256)
    assert (w, h) == (256, 170)
    got = _scaled_both_ways(dec, [au], 1, 1, lb.CHROMA_INTERLEAVED_RGB, w, h)
    assert np.array_equal(got, _nn(full, 3, w, h))


def _grid_tiles(seed, n, tw, th, bit_depth=8, chroma=1, **kw):
    tiles = []
    for k in range(n):
        y, cb, cr = lb.hevc_enc.synthetic_image(seed + k, tw, th, bit_depth, chroma)
        tiles.append(lb.hevc_enc.encode_intra(y, cb, cr, bit_depth=bit_depth, log2_ctb_size=4 + k % 2, wpp=k % 2, seed=seed + k, vui_present=1,
                                              colour_description_present=1, colour_primaries=1, transfer_characteristics=13,
                                              matrix_coefficients=6, full_range=0, **kw))
    return tiles


GRID_CASES = [
    # (id, bit depth, chroma, target, canvas, geometry ops, scaled sizes)
    ("8bit_420_rgb_crop", 8, 1, lb.CHROMA_INTERLEAVED_RGB, (350, 100), [], [(117, 33), (700, 211), (1, 1)]),
    ("10bit_420_rrggbb_le", 10, 1, lb.CHROMA_INTERLEAVED_RRGGBB_LE, (350, 100), [], [(117, 33), (351, 101)]),
    ("10bit_420_rgb_hdr_to_8bit", 10, 1, lb.CHROMA_INTERLEAVED_RGB, (350, 100), [], [(117, 33), (1, 90)]),
    ("8bit_422_rgba", 8, 2, lb.CHROMA_INTERLEAVED_RGBA, (0, 0), [], [(129, 41), (400, 300)]),
    ("8bit_420_rot90_oddcrop", 8, 1, lb.CHROMA_INTERLEAVED_RGB, (350, 100), [(1, 90), (3, 3, 96, 1, 340)], [(31, 107), (200, 700)]),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", GRID_CASES, ids=[c[0] for c in GRID_CASES])
def test_fused_grid(dec, case):
    """3 x 2 grids of host-encoder tiles (canvas cropping the overhang where given): scaled fused call == scale_nearest_neighbor
    of the unscaled fused call, into pageable and page-locked memory."""
    _, bd, chroma, outc, canvas, ops, sizes = case
    tiles = _grid_tiles(0x5CA1 + bd + chroma, 6, 128, 64, bd, chroma)
    W, H = canvas if canvas != (0, 0) else (384, 128)
    geom = None
    if ops:
        geom = lb.Geometry(W, H, chroma)
        for o in ops:
            geom.rotate_ccw(o[1]) if o[0] == 1 else geom.crop(*o[1:5])
        W, H = geom.size
    bpp = BPP[outc]
    full = np.empty((H, W * bpp), np.uint8)
    dec.decode_grid_to_rgb_host(tiles, 3, 2, outc, canvas=canvas, geometry=geom, out=full)
    for w, h in sizes:
        got = _scaled_both_ways(dec, tiles, 3, 2, outc, w, h, canvas=canvas, geometry=geom)
        assert np.array_equal(got, _nn(full, bpp, w, h)), (w, h)


@pytest.mark.gpu
@pytest.mark.parametrize("chunks", [None, "0"])
def test_fused_grid_past_the_band_threshold(cuda, chunks, monkeypatch):
    """A grid with more CABAC sub-streams than one wave of the entropy kernel: the unscaled call into page-locked memory runs
    in bands, the scaled call converts the finished canvas once; B200_CHUNKS unset or 0 gives the same scaled bytes, equal to
    scale_nearest_neighbor of the unscaled result."""
    y, cb, cr = lb.hevc_enc.synthetic_image(0xBA4D, 256, 256, 8, True)
    tile = lb.hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=4, wpp=1, seed=0xBA4D, vui_present=1, colour_description_present=1,
                                    colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=0)
    cols = rows = 14                          # 196 tiles x 16 WPP rows = 3136 sub-streams
    W = H = 256 * cols
    monkeypatch.delenv("B200_CHUNKS", raising=False)
    d = lb.Decoder(host_threads=8)
    try:
        ptr = C.c_void_p()
        _lib.check(_lib.lib().b200_host_alloc(H * W * 3, C.byref(ptr)))
        try:
            full = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint8)), shape=(H, W * 3))
            d.decode_grid_to_rgb_host([tile] * (cols * rows), cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=full)
            assert d.stats().front_end == 3 and d.stats().bands > 1
            full = full.copy()
        finally:
            _lib.lib().b200_host_free(ptr)
        if chunks is not None:
            monkeypatch.setenv("B200_CHUNKS", chunks)
        for w, h in [lb.thumbnail_size(W, H, 512), (1001, 333)]:
            got = _scaled_both_ways(d, [tile] * (cols * rows), cols, rows, lb.CHROMA_INTERLEAVED_RGB, w, h)
            assert np.array_equal(got, _nn(full, 3, w, h)), (w, h)
    finally:
        d.close()


@pytest.mark.gpu
def test_scaled_unscaled_scaled_on_one_decoder(cuda):
    """The decoder's buffers serve a scaled call, an unscaled one and a scaled one of another size in turn."""
    tiles = _grid_tiles(0xEE, 4, 128, 64)
    d = lb.Decoder(host_threads=4)
    try:
        full = np.empty((128, 256 * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, 2, 2, lb.CHROMA_INTERLEAVED_RGB, out=full)
        want = full.copy()
        a = np.empty((50, 99 * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, 2, 2, lb.CHROMA_INTERLEAVED_RGB, out=a, scale=(99, 50))
        full[:] = 0
        d.decode_grid_to_rgb_host(tiles, 2, 2, lb.CHROMA_INTERLEAVED_RGB, out=full)
        b = np.empty((300, 513 * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, 2, 2, lb.CHROMA_INTERLEAVED_RGB, out=b, scale=(513, 300))
        assert np.array_equal(full, want)
        assert np.array_equal(a, _nn(want, 3, 99, 50))
        assert np.array_equal(b, _nn(want, 3, 513, 300))
        dev = d.to_rgb_device(lb.CHROMA_INTERLEAVED_RGB, scale=(77, 31))
        assert np.array_equal(dev.cpu().numpy(), _nn(want, 3, 77, 31))
    finally:
        d.close()
