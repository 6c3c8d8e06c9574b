"""b200_rgb_to_ycbcr_plan (host only) against the unmodified reference planner: for every RGB layout, depth, target chroma,
matrix, range and option set the GPU conversion must mirror exactly the chain convert_colorspace runs, and refuse where
that chain fails or holds an operation it does not mirror."""
import itertools

import numpy as np
import pytest

import libheif_b200 as lb
from oracle import ref_encode
from rgb_ex_cases import LAYOUTS, MATRICES, make_input, ref_mask

pytestmark = pytest.mark.skipif(ref_encode.lib() is None, reason="oracle/_ref/liboracle_encode.so not built (reference sources absent)")

OPTIONS = [(2, 0), (1, 1), (2, 1), (3, 1)]     # (heif_chroma_downsampling_algorithm, only_use_preferred): default, NN, average, sharp YUV


@pytest.mark.parametrize("label,chroma,depth,alpha", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_plan_matches_reference_planner(label, chroma, depth, alpha):
    ref_in, ex_in, endian = make_input(1, 3, 3, chroma, depth, alpha)
    for out_chroma, mc, full, (ds, only) in itertools.product((1, 2, 3), MATRICES + (2, 11, 14), (0, 1), OPTIONS):
        ref = ref_encode.ref_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full), ds, only)
        want = None if ref is None else ref_mask(ref[4])
        what = f"{label} chroma={out_chroma} mc={mc} full={full} opt={(ds, only)} ref={None if ref is None else ref[4]}"
        if want is None:
            with pytest.raises(lb.B200Error) as e:
                lb.rgb_to_ycbcr_plan(ex_in, out_chroma, depth, endian, mc, 1, bool(full), ds, only)
            assert e.value.code == -2, what
        else:
            assert lb.rgb_to_ycbcr_plan(ex_in, out_chroma, depth, endian, mc, 1, bool(full), ds, only) == want, what


@pytest.mark.parametrize("depth,alpha_depth", [(8, 10), (10, 8), (10, 12)])
def test_mismatched_alpha_depth_is_refused(depth, alpha_depth):
    # the reference inserts Op_adjust_alpha_bit_depth; the GPU path does not mirror it
    dt = lambda d: np.uint8 if d == 8 else np.uint16   # noqa: E731
    planes = tuple(np.zeros((3, 5), dt(depth)) for _ in range(3)) + (np.zeros((3, 5), dt(alpha_depth)),)
    ref = ref_encode.ref_rgb_to_ycbcr_ex(planes, 3, depth, 1, (1, 13, 6, 1), alpha_bit_depth=alpha_depth)
    assert ref is not None and ref_mask(ref[4]) is None
    with pytest.raises(lb.B200Error) as e:
        lb.rgb_to_ycbcr_plan(planes, 1, depth, alpha_bit_depth=alpha_depth)
    assert e.value.code == -2
