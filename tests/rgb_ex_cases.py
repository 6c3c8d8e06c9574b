"""RGB inputs of the encoder-side conversion in every layout (shared by the planner and GPU tests of rgb_to_ycbcr_ex)."""
import numpy as np

# (label, heif_chroma of the input, bit depth, alpha) -- interleaved RGB / RGBA 8 bit, RRGGBB(AA) BE / LE, planar 4:4:4
LAYOUTS = [("rgb8", 10, 8, False), ("rgba8", 11, 8, True)]
LAYOUTS += [(f"rrggbb{'aa' if a else ''}_{e}{d}", c, d, a) for (c, e, a) in ((12, "be", False), (13, "be", True), (14, "le", False), (15, "le", True))
            for d in (10, 12, 16)]
LAYOUTS += [(f"planar{'a' if a else ''}{d}", 3, d, a) for d in (8, 10, 12, 16) for a in (False, True)]
MATRICES = (0, 1, 5, 6, 8, 9, 10, 12)
PIPE = {"Op_RGB24_32_to_YCbCr": 1, "Op_RGB24_32_to_YCbCr444_GBR": 2, "Op_RRGGBBxx_HDR_to_YCbCr420": 4, "Op_RGB_to_YCbCr<unsigned char>": 8,
        "Op_RGB_to_YCbCr<unsigned short>": 8, "Op_RGB24_32_to_RGB": 16, "Op_RRGGBBaa_BE_to_RGB_HDR": 16, "Op_RRGGBBaa_swap_endianness": 32}


def make_input(seed, w, h, chroma, depth, alpha):
    """Returns (reference form, rgb_to_ycbcr_ex form, endianness): interleaved as the layout's bytes (uint8 [H, W*bytes]) for
    the reference and as [H, W, C] (uint8, or uint16 holding those same bytes) for this library; planar as a tuple of planes."""
    rng = np.random.default_rng(seed)
    maxv = (1 << depth) - 1
    if chroma == 3:
        dt = np.uint8 if depth == 8 else np.uint16
        planes = tuple(rng.integers(0, maxv + 1, (h, w)).astype(dt) for _ in range(4 if alpha else 3))
        return planes, planes, None
    nch = 4 if alpha else 3
    if depth == 8:
        a = rng.integers(0, 256, (h, w, nch)).astype(np.uint8)
        return a.reshape(h, w * nch), a, None
    vals = rng.integers(0, maxv + 1, (h, w, nch)).astype(np.uint16)
    big = chroma in (12, 13)
    raw = vals.astype(">u2" if big else "<u2").view(np.uint8).reshape(h, w * nch * 2)
    return raw, raw.view(np.uint16).reshape(h, w, nch), "big" if big else "little"


def ref_mask(pipeline):
    """B200_YCC_PIPE_* mask of a reference chain, or None when it holds an operation the GPU path does not mirror."""
    m = 0
    for op in pipeline:
        if op not in PIPE:
            return None
        m |= PIPE[op]
    return m
