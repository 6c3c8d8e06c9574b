"""The HEVC access units the reference pushes into a decoder plugin while decoding its own fuzzing corpus
(tests/golden/corpus, extracted by tests/golden/make_corpus.py): every decoder of this repo must answer each one with an
error code or with the oracle's planes -- never a crash, a hang or different pixels."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

from libheif_b200 import _lib
from oracle import bindings as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "corpus", "*.au")))


def oracle_planes(au):
    try:
        return ob.restatement_decode(au)[0]
    except Exception:  # noqa: BLE001
        return None


@pytest.mark.timeout(120)
@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f) for f in FILES])
def test_host_front_end_on_corpus(path):
    au = open(path, "rb").read()
    l = _lib.lib()
    n8 = 4096 * 4096 // 64
    qp8 = np.zeros(n8, np.int8); edge8 = np.zeros(n8, np.uint8); lm = np.zeros(n8 * 4, np.uint8); cm = np.zeros(n8 * 4, np.uint8)
    out5 = (C.c_ulonglong * 5)()
    info = _lib.ImageInfo()
    if l.b200_probe_access_unit(au, len(au), 4096 * 4096, info) != 0:
        return                                            # rejected by the header parser: fine
    rc = l.b200_debug_parse(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out5)
    if rc == 0:                                           # decodable: then the oracle must decode it too, to the same size
        want = oracle_planes(au)
        assert want is not None
        assert (out5[3], out5[4]) >= (want[0].shape[1], want[0].shape[0])


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("path", FILES, ids=[os.path.basename(f) for f in FILES])
def test_gpu_decoder_on_corpus(cuda, path):
    import libheif_b200 as lb
    au = open(path, "rb").read()
    dec = lb.Decoder(host_threads=2)
    try:
        try:
            dec.decode_image(au, max_image_size_pixels=4096 * 4096)
            got = dec.planes_host()
        except lb.B200Error:
            return                                        # an error code: fine
        want = oracle_planes(au)
        assert want is not None, "the CUDA decoder produced a picture the oracle rejects"
        for c in range(len(want)):
            assert np.array_equal(got[c], want[c]), f"plane {c}"
    finally:
        dec.close()
