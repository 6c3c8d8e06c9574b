"""The C restatement of the encoder-side colour stage (oracle/color_oracle_ex.c) against the unmodified reference's
convert_colorspace, byte for byte and chain for chain, on every RGB layout x depth x target chroma x matrix x range x alpha,
at tiny odd sizes: settles the float order of the arithmetic the GPU kernel mirrors, without a GPU."""
import itertools

import numpy as np
import pytest

from oracle import ref_encode
from rgb_ex_cases import LAYOUTS, MATRICES, make_input, ref_mask

pytestmark = pytest.mark.skipif(ref_encode.lib() is None, reason="oracle/_ref/liboracle_encode.so not built (reference sources absent)")

SIZES = ((1, 1), (1, 5), (5, 1), (17, 9))


@pytest.mark.parametrize("label,chroma,depth,alpha", LAYOUTS, ids=[l[0] for l in LAYOUTS])
def test_restatement_matches_reference(label, chroma, depth, alpha):
    for k, (w, h) in enumerate(SIZES):
        ref_in, _, _ = make_input(200 + k, w, h, chroma, depth, alpha)
        for out_chroma, mc, full, (ds, only) in itertools.product((1, 2, 3), MATRICES + (2, 11, 14), (0, 1), ((2, 0), (1, 1), (2, 1))):
            ref = ref_encode.ref_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full), ds, only)
            co = ref_encode.oracle_rgb_to_ycbcr_ex(ref_in, chroma, depth, out_chroma, (1, 13, mc, full), ds, only)
            what = f"{label} {w}x{h} -> {out_chroma} mc={mc} full={full} opt={(ds, only)} ref={None if ref is None else ref[4]}"
            want = None if ref is None else ref_mask(ref[4])
            if want is None:
                assert co is None, what
                continue
            assert co is not None and co[4] == want, what
            for name, g, r in zip(("Y", "Cb", "Cr", "alpha"), co[:4], ref[:4]):
                assert (g is None) == (r is None), f"{what}: {name} presence"
                if r is not None:
                    assert np.array_equal(g, r), f"{what}: {name} differs ({np.count_nonzero(g != r)} samples)"
