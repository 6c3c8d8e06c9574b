"""GPU parity: the fused sm_90a colour kernel (K6) through the C ABI vs the C restatement of the reference
(oracle/color_oracle.c, itself pinned on the unmodified reference by test_color_oracle.py). Bit-exact."""
import hashlib

import numpy as np
import pytest

import libheif_b200 as lb
from test_color_oracle import CASES, GEOM
from util import oracle_postprocess, random_ycbcr

pytestmark = pytest.mark.gpu


def _img(y, cb, cr, a, chroma, bpp, nclx, dev=None):
    import torch
    dt = np.uint8 if bpp == 8 else np.uint16

    def cv(p):
        if p is None:
            return None
        arr = np.ascontiguousarray(p.astype(dt))
        if dev is None:
            return arr
        t = torch.from_numpy(arr.view(np.int16) if bpp > 8 else arr).to(dev)
        return t
    cp, tc, mc, fr = nclx if nclx else (2, 2, 2, 1)
    return lb.YCbCrImage(cv(y), cv(cb), cv(cr), cv(a), chroma=chroma, bit_depth=bpp, colour_primaries=cp,
                         transfer_characteristics=tc, matrix_coefficients=mc, full_range=bool(fr))


def _geom(w, h, ops, chroma=1):
    g = lb.Geometry(w, h, chroma)
    for o in ops:
        if o[0] == 1:
            g.rotate_ccw(o[1])
        elif o[0] == 2:
            g.mirror(o[1])
        else:
            g.crop(*o[1:5])
    return g


def _as_bytes(t):
    return t.cpu().numpy().view(np.uint8).reshape(-1) if hasattr(t, "cpu") else np.ascontiguousarray(t).view(np.uint8).reshape(-1)


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("size", [(2, 2), (34, 18), (64, 64), (130, 70), (517, 259)])
def test_device_matches_oracle(cuda, case, size):
    chroma, bpp, nclx, outc = case
    w, h = size
    y, cb, cr, _ = random_ycbcr(0xB200 + w * 131 + h, w, h, chroma, bpp)
    want, ow, oh = oracle_postprocess(y, cb, cr, None, chroma, bpp, nclx, [], outc)
    got = lb.convert_colorspace(_img(y, cb, cr, None, chroma, bpp, nclx, cuda), outc)
    assert np.array_equal(_as_bytes(got), want)


@pytest.mark.parametrize("ops", GEOM + [[(1, 90), (3, 2, 17, 4, 27)], [(2, 1), (1, 270), (2, 0)]])
@pytest.mark.parametrize("fmt", [(1, 8, (1, 13, 6, 0), 10), (1, 8, (1, 13, 6, 1), 10), (1, 10, (9, 16, 9, 0), 14), (3, 8, (1, 13, 6, 1), 11)])
@pytest.mark.parametrize("size", [(32, 24), (200, 136)])
def test_geometry_fused(cuda, ops, fmt, size):
    chroma, bpp, nclx, outc = fmt
    w, h = size
    y, cb, cr, _ = random_ycbcr(1234, w, h, chroma, bpp)
    # (even sizes and crop origins: no 4:4:4 conversion point of the reference in these chains; see test_444_detour)
    want, ow, oh = oracle_postprocess(y, cb, cr, None, chroma, bpp, nclx, ops, outc)
    got = lb.convert_colorspace(_img(y, cb, cr, None, chroma, bpp, nclx, cuda), outc, _geom(w, h, ops, chroma))
    assert np.array_equal(_as_bytes(got), want)


@pytest.mark.parametrize("outc", [10, 11])
def test_alpha(cuda, outc):
    y, cb, cr, a = random_ycbcr(77, 100, 52, 1, 8, alpha=True)
    for nclx in [(1, 13, 6, 1), (1, 13, 6, 0)]:
        want, _, _ = oracle_postprocess(y, cb, cr, a if outc == 11 else None, 1, 8, nclx, [], outc)
        got = lb.convert_colorspace(_img(y, cb, cr, a if outc == 11 else None, 1, 8, nclx, cuda), outc)
        assert np.array_equal(_as_bytes(got), want)


def test_host_entry_point(cuda):
    """b200_color_convert_host: host buffers in, host buffer out (H2D/D2H inside the C-ABI call)."""
    y, cb, cr, _ = random_ycbcr(5, 300, 200, 1, 8)
    want, _, _ = oracle_postprocess(y, cb, cr, None, 1, 8, (1, 13, 6, 0), [(1, 90)], 10)
    out, pipe = lb.convert_colorspace_host(_img(y, cb, cr, None, 1, 8, (1, 13, 6, 0)), 10, _geom(300, 200, [(1, 90)]))
    assert pipe & 2
    assert np.array_equal(out.reshape(-1), want)


def test_full_size_properties(cuda):
    """BASELINE config 2 size (4096x4096 8-bit 4:2:0 -> RGB24): size-independent properties.
    (a) rotating four times by 90 degrees is the identity; (b) a tile of the big result equals the oracle on that
    tile's planes (NN chroma makes conversion local); (c) checksum of row-checksums is stable across both entry points."""
    import torch
    w = h = 4096
    y, cb, cr, _ = random_ycbcr(0xB200, w, h, 1, 8)
    img = _img(y, cb, cr, None, 1, 8, (1, 13, 6, 0), cuda)
    base = lb.convert_colorspace(img, 10)
    rot4 = lb.convert_colorspace(img, 10, lb.Geometry(w, h).rotate_ccw(90).rotate_ccw(90).rotate_ccw(90).rotate_ccw(90))
    assert torch.equal(base, rot4)
    r90 = lb.convert_colorspace(img, 10, lb.Geometry(w, h).rotate_ccw(90))
    back = r90.view(h, w, 3).flip(0).transpose(0, 1).contiguous().view(h, w * 3)   # undo: rot90ccw -> rotate clockwise
    assert torch.equal(base, back)
    ty, tx = 1024, 2048
    want, _, _ = oracle_postprocess(y[ty:ty + 128, tx:tx + 128], cb[ty // 2:ty // 2 + 64, tx // 2:tx // 2 + 64],
                                    cr[ty // 2:ty // 2 + 64, tx // 2:tx // 2 + 64], None, 1, 8, (1, 13, 6, 0), [], 10)
    tile = base.view(h, w, 3)[ty:ty + 128, tx:tx + 128].contiguous()
    assert np.array_equal(_as_bytes(tile), want)
    host, _ = lb.convert_colorspace_host(_img(y, cb, cr, None, 1, 8, (1, 13, 6, 0)), 10)
    assert hashlib.md5(host.tobytes()).hexdigest() == hashlib.md5(base.cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("case", [(1, 8, (1, 13, 6, 0), 10), (1, 8, (1, 13, 6, 1), 10), (1, 8, (1, 13, 1, 0), 11), (1, 10, (9, 16, 9, 0), 14), (1, 12, (9, 16, 9, 1), 14)])
@pytest.mark.parametrize("size", [(4, 4), (34, 18), (33, 17), (130, 70), (512, 256)])
def test_bilinear_chroma_upsampling(cuda, case, size):
    """only_use_preferred_chroma_algorithm + bilinear (heif-dec -C bilinear): Op_YCbCr420_bilinear_to_YCbCr444 + float op."""
    chroma, bpp, nclx, outc = case
    w, h = size
    y, cb, cr, _ = random_ycbcr(0xB200 + w * 7 + h, w, h, chroma, bpp)
    want, ow, oh = oracle_postprocess(y, cb, cr, None, chroma, bpp, nclx, [], outc, bilinear=1)
    got = lb.convert_colorspace(_img(y, cb, cr, None, chroma, bpp, nclx, cuda), outc, bilinear=True)
    assert np.array_equal(_as_bytes(got), want)


from test_color_oracle import DETOUR  # noqa: E402


@pytest.mark.parametrize("case", DETOUR)
@pytest.mark.parametrize("fmt", [(8, (1, 13, 6, 1), 10, False), (8, (1, 13, 6, 1), 11, True), (10, (9, 16, 9, 1), 14, False)])
def test_444_detour(cuda, case, fmt):
    """4:2:0 pictures whose transform chain makes the reference convert to 4:4:4 first (odd crop origin, odd sizes under
    rotate / mirror): plane-wise pre-pass + bilinear upsampling + the rest of the chain, against the restatement."""
    w, h, ops = case
    bpp, nclx, outc, alpha = fmt
    y, cb, cr, a = random_ycbcr(77, w, h, 1, bpp, alpha=alpha)
    want, ow, oh = oracle_postprocess(y, cb, cr, a, 1, bpp, nclx, ops, outc)
    out = lb.convert_colorspace(_img(y, cb, cr, a, 1, bpp, nclx, cuda), outc, _geom(w, h, ops, 1))
    assert np.array_equal(_as_bytes(out), want)


@pytest.mark.parametrize("case", DETOUR)
@pytest.mark.parametrize("fmt", [(8, (1, 13, 6, 0), 10, False), (8, (2, 2, 2, 0), 11, True), (10, (9, 16, 9, 0), 14, False), (12, (1, 13, 1, 0), 3, False)])
def test_444_detour_limited_range(cuda, case, fmt):
    """Limited-range 4:2:0 pictures at the reference's 4:4:4 conversion point: bilinear upsampling, then the range conversion
    through RGB (Op_YCbCr_to_RGB -> Op_RGB_to_YCbCr to full range, pixelimage.cc:1187-1215), then the rest of the chain."""
    w, h, ops = case
    bpp, nclx, outc, alpha = fmt
    y, cb, cr, a = random_ycbcr(77, w, h, 1, bpp, alpha=alpha)
    want, ow, oh = oracle_postprocess(y, cb, cr, a, 1, bpp, nclx, ops, outc)
    out = lb.convert_colorspace(_img(y, cb, cr, a, 1, bpp, nclx, cuda), outc, _geom(w, h, ops, 1))
    got = np.concatenate([_as_bytes(t) for t in out]) if isinstance(out, (list, tuple)) else _as_bytes(out)
    assert np.array_equal(got, want)


from test_color_oracle import DETOUR_422  # noqa: E402


@pytest.mark.parametrize("case", DETOUR_422)
@pytest.mark.parametrize("fmt", [(8, (1, 13, 6, 1), 10, False), (8, (1, 13, 6, 0), 11, True), (10, (9, 16, 9, 0), 14, False), (12, (1, 13, 1, 1), 3, False)])
def test_444_detour_422(cuda, case, fmt):
    """4:2:2 pictures: rotate 90 / 270, 180 with odd height, horizontal mirror with odd width, crop with odd left convert to
    4:4:4 first with Op_YCbCr422_bilinear_to_YCbCr444 (chroma_sampling.cc:784-905)."""
    w, h, ops = case
    bpp, nclx, outc, alpha = fmt
    y, cb, cr, a = random_ycbcr(78, w, h, 2, bpp, alpha=alpha)
    want, ow, oh = oracle_postprocess(y, cb, cr, a, 2, bpp, nclx, ops, outc)
    out = lb.convert_colorspace(_img(y, cb, cr, a, 2, bpp, nclx, cuda), outc, _geom(w, h, ops, 2))
    got = np.concatenate([_as_bytes(t) for t in out]) if isinstance(out, (list, tuple)) else _as_bytes(out)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("mc", [0, 8, 16])
@pytest.mark.parametrize("chroma", [1, 2, 3])
@pytest.mark.parametrize("bpp,outc", [(8, 10), (8, 11), (8, 3), (10, 10), (10, 14), (10, 3), (12, 15)])
@pytest.mark.parametrize("full", [0, 1])
def test_special_matrices(cuda, mc, chroma, bpp, outc, full):
    """matrix_coefficients 0 (GBR), 8 (YCgCo), 16 (YCgCo-Re): the special branches of Op_YCbCr_to_RGB (yuv2rgb.cc:222-262),
    including which cases the dedicated 4:2:0 ops take instead -- 126 cases, the same the oracle is pinned on."""
    for size in ((34, 18), (130, 70)):
        w, h = size
        y, cb, cr, a = random_ycbcr(4242 + mc + w, w, h, chroma, bpp, alpha=outc in (11, 15))
        want, ow, oh = oracle_postprocess(y, cb, cr, a, chroma, bpp, (1, 13, mc, full), [], outc)
        out = lb.convert_colorspace(_img(y, cb, cr, a, chroma, bpp, (1, 13, mc, full), cuda), outc)
        got = np.concatenate([_as_bytes(t) for t in out]) if isinstance(out, (list, tuple)) else _as_bytes(out)
        assert np.array_equal(got, want)


@pytest.mark.parametrize("ops", GEOM[:6])
def test_bilinear_after_geometry(cuda, ops):
    y, cb, cr, _ = random_ycbcr(99, 32, 24, 1, 8)
    want, ow, oh = oracle_postprocess(y, cb, cr, None, 1, 8, (1, 13, 6, 0), ops, 10, bilinear=1)
    out = lb.convert_colorspace(_img(y, cb, cr, None, 1, 8, (1, 13, 6, 0), cuda), 10, _geom(32, 24, ops, 1), bilinear=True)
    assert np.array_equal(_as_bytes(out), want)


# ---- encoder-side direction: RGB / RGBA 8 bit -> YCbCr (b200_rgb_to_ycbcr_device / _host vs oracle/color_oracle.c) ----
from test_color_oracle import RGB2YCC_NCLX, RGB2YCC_SIZES, rgb_pattern  # noqa: E402


def _check_ycc(img, ref, what):
    for name, g, r in zip("Y Cb Cr A".split(), (img.y, img.cb, img.cr, img.alpha), ref):
        if r is None:
            assert g is None
            continue
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        assert g.shape == r.shape, (what, name, g.shape, r.shape)
        assert np.array_equal(g, r), f"{what}: {name} differs, first at {np.argwhere(g != r)[:3].tolist()}"


@pytest.mark.parametrize("size", RGB2YCC_SIZES + [(517, 259), (1024, 512), (1030, 77)])
@pytest.mark.parametrize("alpha", [0, 1])
@pytest.mark.parametrize("out_chroma", [1, 2, 3])
def test_rgb_to_ycbcr_device_matches_oracle(cuda, size, alpha, out_chroma):
    import torch
    from oracle.bindings import oracle_rgb_to_ycbcr
    w, h = size
    bpp = 4 if alpha else 3
    rgb = rgb_pattern(0xC0DE + w * 13 + h, w, h, bpp)
    t = torch.from_numpy(rgb.reshape(h, w, bpp)).cuda()
    for nclx in RGB2YCC_NCLX:
        cp, _, mc, fr = nclx
        img = lb.rgb_to_ycbcr(t, out_chroma, matrix_coefficients=mc, colour_primaries=cp, full_range=bool(fr))
        torch.cuda.synchronize()
        _check_ycc(img, oracle_rgb_to_ycbcr(rgb, alpha, out_chroma, nclx), f"{size} alpha={alpha} chroma={out_chroma} nclx={nclx}")


@pytest.mark.parametrize("out_chroma", [1, 2, 3])
def test_rgb_to_ycbcr_unaligned_rows_and_host_call(cuda, out_chroma):
    """Odd row pitch / odd base address take the byte-wise load path; RGB without alpha into an alpha plane gives 0xff."""
    import torch
    from oracle.bindings import oracle_rgb_to_ycbcr
    w, h = 203, 61
    for bpp in (3, 4):
        rgb = rgb_pattern(77 + bpp, w, h, bpp)
        pitch = w * bpp + 5
        buf = torch.zeros(h * pitch + 1, dtype=torch.uint8, device="cuda")
        view = buf[1:].as_strided((h, w, bpp), (pitch, bpp, 1))
        view.copy_(torch.from_numpy(rgb.reshape(h, w, bpp)).cuda())
        nclx = (1, 13, 6, 0)
        img = lb.rgb_to_ycbcr(view, out_chroma, matrix_coefficients=6, colour_primaries=1, full_range=False, want_alpha=True)
        torch.cuda.synchronize()
        ref = list(oracle_rgb_to_ycbcr(rgb, bpp == 4, out_chroma, nclx))
        if bpp == 3:
            ref[3] = np.full((h, w), 255, np.uint8)
        _check_ycc(img, ref, f"strided bpp={bpp}")
        himg = lb.rgb_to_ycbcr_host(rgb.reshape(h, w, bpp), out_chroma, matrix_coefficients=6, colour_primaries=1, full_range=False, want_alpha=True)
        _check_ycc(himg, ref, f"host bpp={bpp}")


@pytest.mark.parametrize("mc", [0, 8, 11, 14])
def test_rgb_to_ycbcr_refuses_what_the_reference_op_refuses(cuda, mc):
    import torch
    t = torch.zeros((4, 4, 3), dtype=torch.uint8, device="cuda")
    with pytest.raises(lb.B200Error) as e:
        lb.rgb_to_ycbcr(t, 1, matrix_coefficients=mc)
    assert e.value.code == -2            # B200_E_UNSUPPORTED


def test_rgb_to_ycbcr_then_back_is_close(cuda):
    """Size-independent property at a full-size picture: RGB -> YCbCr 4:4:4 full range -> RGB (K6) is within rounding of identity."""
    import torch
    w, h = 4096, 2048
    g = torch.Generator(device="cuda").manual_seed(5)
    rgb = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda", generator=g)
    img = lb.rgb_to_ycbcr(rgb, 3, matrix_coefficients=6, colour_primaries=1, full_range=True)
    back = lb.convert_colorspace(img, lb.CHROMA_INTERLEAVED_RGB).reshape(h, w, 3)
    assert (back.int() - rgb.int()).abs().max().item() <= 2
