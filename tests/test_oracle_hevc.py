"""CPU: pin the C restatement of HEVC intra decoding (oracle/hevc_oracle.c) on an independent conforming decoder
(FFmpeg libavcodec, oracle/ffhevc.c) for the reference's fixtures and for every synthetic stream; plus the golden md5s
of SURVEY.md Appendix C for the reference fixtures (planes of examples/example.heic)."""
import hashlib
import os

import numpy as np
import pytest

from hevc_cases import all_streams, cpu_extra_streams, synth_params, synth_source, synth_stream
from oracle import bindings as ob

have_ffmpeg = ob.avcodec_dir() is not None

# FFmpeg 62's chroma SAO reads neighbours whose horizontal-edge deblocking is still deferred when log2_ctb_size == 4
# (its deblocking defers chroma horizontal edges by 16 luma samples = one whole 16x16 CTB), so it deviates from H.265
# 8.7.3 ("deblocked sample array") at a handful of CTB-corner chroma samples.  Those streams are pinned on luma +
# the no-SAO / no-deblocking variants instead.
FFMPEG_CTB16_CHROMA_SAO = {"ctb16_basic"}


def ffmpeg_planes(name, nplanes):
    """Planes of stream `name` FFmpeg 62 decodes per H.265.  Two more deviations of that build, both established on LOSSLESS
    streams (every coding unit cu_transquant_bypass: the decoded picture must equal the encoder's input, which the
    restatement reproduces on all planes and FFmpeg only on luma, test_lossless_streams_reproduce_their_source):
      * with SAO enabled, FFmpeg's chroma SAO does not leave the samples of cu_transquant_bypass units / of PCM units under
        pcm_loop_filter_disabled_flag unchanged (8.7.3 requires SaoTypeIdx to be treated as 0 there): luma only, the
        chroma path is pinned by the sao=0 variants of the same streams (x_*_nosao);
      * 4:0:0 streams with PCM units lose CABAC synchronisation in FFmpeg ("cu_qp_delta ... outside the valid range"): not compared."""
    if name in FFMPEG_CTB16_CHROMA_SAO:
        return [0]
    p = synth_params(name)
    if p is not None:
        o = p[5]
        if o.get("pcm") and not p[4]:
            return []
        if p[4] == 2 and o.get("log2_ctb_size") == 4 and o.get("sao", 1):
            return [0]                                     # the CTB-16 chroma SAO deviation above, 4:2:2
        if o.get("sao", 1) and (o.get("transquant_bypass") or o.get("pcm") == 2):
            return [0]
    return list(range(nplanes))


@pytest.mark.skipif(not have_ffmpeg, reason="FFmpeg (cv2 wheel) not present")
@pytest.mark.parametrize("name,au", all_streams() + cpu_extra_streams(), ids=[s[0] for s in all_streams() + cpu_extra_streams()])
def test_restatement_matches_ffmpeg(name, au):
    ff, bd, ch = ob.ffmpeg_decode(au)
    rs, info = ob.restatement_decode(au)
    assert info["bit_depth"] == bd and info["chroma"] == ch
    for c in ffmpeg_planes(name, len(ff)):
        assert np.array_equal(ff[c], rs[c]), f"plane {c} differs at {np.argwhere(ff[c] != rs[c])[:3].tolist()}"


LOSSLESS = [s[0] for s in __import__("hevc_cases").SYNTH + __import__("hevc_cases").SYNTH_CPU_EXTRA if s[5].get("transquant_bypass") == 2]


@pytest.mark.parametrize("name", LOSSLESS)
def test_lossless_streams_reproduce_their_source(name):
    """cu_transquant_bypass on every coding unit: scaling, transform and all in-loop filters are bypassed (8.6.2, 8.7.2.5.7,
    8.7.3), so the decoded picture IS the picture that was encoded -- a pin of the bypass path that needs no second decoder."""
    rs, info = ob.restatement_decode(synth_stream(name))
    src = synth_source(name)
    for c in range(len(rs)):
        assert np.array_equal(rs[c], src[c]), f"plane {c}"


def test_example_heic_golden_md5():
    """SURVEY.md Appendix C: FFmpeg planes of examples/example.heic item 20004."""
    au = dict(all_streams())["example_primary_1280x854.au"]
    rs, _ = ob.restatement_decode(au)
    md5 = [hashlib.md5(p.astype(np.uint8).tobytes()).hexdigest() for p in rs]
    assert md5 == ["5a0423057f3fede64a297243982465c7", "8a2344a26a2347f045842be7f731085c", "29ad6bcbe5dd90a536d0abe36777a1b5"]


@pytest.mark.skipif(not (ob.ref_plugin() is not None and have_ffmpeg), reason="oracle/_ref not present")
def test_golden_streams_are_what_the_reference_pushes_into_a_decoder_plugin():
    """tests/golden/streams/*.au regenerate byte-for-byte from the reference's fixture files stored under
    tests/golden/fixtures/ through the unmodified reference libheif (tests/golden/make_streams.py --check)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tests", "golden", "make_streams.py"), "--check"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    assert r.stdout.count("ok   ") == 5, r.stdout
