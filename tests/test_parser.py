"""CPU: the product's host HEVC front-end (CABAC + syntax -> command stream, libheif_b200/csrc/b200_hevc_parse.cc)
against the C restatement's syntax-level state (oracle/hevc_oracle.c: hevc_oracle_debug_maps), which is itself pinned
on FFmpeg's pixels by test_oracle_hevc.py.  Compared: QpY and filterEdgeFlag maps (8x8), luma/chroma intra modes (4x4),
TU count and an order-independent digest of every coefficient level with its position."""
import ctypes as C

import numpy as np
import pytest

from hevc_cases import all_streams, cpu_extra_streams
from libheif_b200 import _lib
from oracle import bindings as ob


def product_digest(au):
    l = _lib.lib()
    n8 = 2048 * 2048 // 64
    qp8 = np.zeros(n8, np.int8); edge8 = np.zeros(n8, np.uint8); lm = np.zeros(n8 * 4, np.uint8); cm = np.zeros(n8 * 4, np.uint8)
    out5 = (C.c_ulonglong * 5)()
    _lib.check(l.b200_debug_parse(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out5))
    w, h = out5[3], out5[4]
    return dict(hash=out5[0], ncoef=out5[1], ntu=out5[2], w=w, h=h, qp8=qp8[:w * h // 64].copy(), edge8=edge8[:w * h // 64].copy(),
                lm=lm[:w * h // 16].copy(), cm=cm[:w * h // 16].copy())


def oracle_digest(au):
    l = ob.lib()
    n8 = 2048 * 2048 // 64
    qp8 = np.zeros(n8, np.int8); edge8 = np.zeros(n8, np.uint8); lm = np.zeros(n8 * 4, np.uint8); cm = np.zeros(n8 * 4, np.uint8)
    out3 = (C.c_ulonglong * 3)(); dims = (C.c_int * 2)()
    l.hevc_oracle_debug_maps.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_ulonglong), C.POINTER(C.c_int)]
    rc = l.hevc_oracle_debug_maps(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out3, dims)
    assert rc == 0
    w, h = dims[0], dims[1]
    return dict(hash=out3[0], ncoef=out3[1], ntu=out3[2], w=w, h=h, qp8=qp8[:w * h // 64].copy(), edge8=edge8[:w * h // 64].copy(),
                lm=lm[:w * h // 16].copy(), cm=cm[:w * h // 16].copy())


@pytest.mark.parametrize("name,au", all_streams() + cpu_extra_streams(), ids=[s[0] for s in all_streams() + cpu_extra_streams()])
def test_front_end_matches_restatement(name, au):
    p, o = product_digest(au), oracle_digest(au)
    assert (p["w"], p["h"]) == (o["w"], o["h"])
    assert p["ntu"] == o["ntu"]
    assert p["ncoef"] == o["ncoef"]
    assert np.array_equal(p["lm"], o["lm"]), "luma intra modes differ"
    assert np.array_equal(p["cm"], o["cm"]), "chroma intra modes differ"
    assert np.array_equal(p["qp8"], o["qp8"]), "QpY map differs"
    assert np.array_equal(p["edge8"], o["edge8"]), "deblocking edge flags differ"
    assert p["hash"] == o["hash"], "coefficient digest differs"


def test_rejects_garbage():
    l = _lib.lib()
    out5 = (C.c_ulonglong * 5)()
    buf = np.zeros(1 << 16, np.uint8)
    rc = l.b200_debug_parse(b"\x00\x00\x00\x05\x40\x01\x0c\x01\xff", 9, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, out5)
    assert rc != 0


def test_mutated_streams_never_crash_the_front_end():
    """Bit flips / byte substitutions / deletions in every fixture: the host front-end (the syntax decoder the GPU kernel
    shares) must either decode or fail with an error code.  (The same loop ran 20 000 mutations under ASan + UBSan while
    this round was developed; two findings in the header parser -- ue(v) with 32 leading zeros, an unchecked
    log2_sao_offset_scale -- were fixed.)"""
    import random
    from hevc_cases import cpu_extra_streams
    l = _lib.lib()
    n8 = 2048 * 2048 // 64
    qp8 = np.zeros(n8, np.int8); edge8 = np.zeros(n8, np.uint8); lm = np.zeros(n8 * 4, np.uint8); cm = np.zeros(n8 * 4, np.uint8)
    out5 = (C.c_ulonglong * 5)()
    streams = [a for _, a in all_streams() + cpu_extra_streams() if len(a) < 100000]
    rng = random.Random(0xB200)
    decoded = 0
    for _ in range(400):
        b = bytearray(rng.choice(streams))
        mode = rng.random()
        for _ in range(rng.choice([1, 1, 2, 4, 16])):
            p = rng.randrange(len(b))
            if mode < 0.7:
                b[p] ^= 1 << rng.randrange(8)
            elif mode < 0.85:
                b[p] = rng.randrange(256)
            else:
                del b[p:p + rng.randrange(1, 8)]
        rc = l.b200_debug_parse(bytes(b), len(b), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out5)
        decoded += rc == 0
    assert decoded < 400          # most mutations must be rejected (sanity of the test itself)


# ---------------------------------------------------------------------------------------------------------------------
# Syntax-element-level injection (ADVICE round 1): every ue(v)/se(v) field of the SPS, PPS and slice-segment header is
# replaced, one at a time, by extreme Exp-Golomb codes -- 33 leading zeros (saturating code), 2^32 - 2, 65535, 1000 and
# a handful of small out-of-range values.  The front-end must return (error or success) without crashing, hanging or
# touching memory outside its maps; bit-flip fuzzing cannot reach these values (31+ leading zero bits).
class _Bits:
    def __init__(self, data):
        self.bits = "".join(f"{b:08b}" for b in data); self.pos = 0; self.fields = []

    def u(self, n):
        v = int(self.bits[self.pos:self.pos + n] or "0", 2); self.pos += n; return v

    def ue(self, name):
        start = self.pos; z = 0
        while self.pos < len(self.bits) and self.bits[self.pos] == "0":
            z += 1; self.pos += 1
        self.pos += 1
        v = (1 << z) - 1 + (self.u(z) if z else 0)
        self.fields.append((name, start, self.pos - start)); return v

    def se(self, name):
        k = self.ue(name); return (k + 1) >> 1 if k & 1 else -(k >> 1)


def _unescape(nal):
    out = bytearray(); z = 0
    for b in nal:
        if z >= 2 and b == 3:
            z = 0; continue
        out.append(b); z = z + 1 if b == 0 else 0
    return bytes(out)


def _escape(rbsp):
    out = bytearray(); z = 0
    for b in rbsp:
        if z >= 2 and b <= 3:
            out.append(3); z = 0
        out.append(b); z = z + 1 if b == 0 else 0
    return bytes(out)


def _split_nals(au):
    nals = []; p = 0
    while p + 4 <= len(au):
        n = int.from_bytes(au[p:p + 4], "big"); nals.append(au[p + 4:p + 4 + n]); p += 4 + n
    return nals


def _join_nals(nals):
    return b"".join(len(n).to_bytes(4, "big") + n for n in nals)


def _walk_sps(r):
    b = _Bits(r); b.u(16); b.u(4); msl = b.u(3); b.u(1); b.u(96)
    assert msl == 0
    b.ue("sps_id"); cf = b.ue("chroma_format_idc")
    if cf == 3:
        b.u(1)
    b.ue("width"); b.ue("height")
    if b.u(1):
        for n in ("conf_l", "conf_r", "conf_t", "conf_b"):
            b.ue(n)
    b.ue("bit_depth_luma"); b.ue("bit_depth_chroma"); b.ue("log2_max_poc_lsb"); b.u(1)
    b.ue("max_dec_pic_buffering"); b.ue("max_num_reorder"); b.ue("max_latency")
    b.ue("log2_min_cb"); b.ue("log2_diff_cb"); b.ue("log2_min_tb"); b.ue("log2_diff_tb"); b.ue("max_th_depth_inter"); b.ue("max_th_depth_intra")
    b.u(1); b.u(1); b.u(1); b.u(1)            # scaling_list, amp, sao, pcm (all as our encoder writes them: scaling/pcm 0)
    b.ue("num_st_rps")
    return b


def _walk_pps(r):
    b = _Bits(r); b.u(16)
    b.ue("pps_id"); b.ue("pps_sps_id"); b.u(1); b.u(1); b.u(3); b.u(1); b.u(1); b.ue("num_ref_idx_l0"); b.ue("num_ref_idx_l1")
    b.se("init_qp"); b.u(1); b.u(1)
    if b.u(1):
        b.ue("diff_cu_qp_delta_depth")
    b.se("cb_qp_offset"); b.se("cr_qp_offset")
    return b


def _walk_slice(r, nal_type):
    b = _Bits(r); b.u(16); first = b.u(1)
    if 16 <= nal_type <= 23:
        b.u(1)
    b.ue("slice_pps_id")
    if first:
        b.ue("slice_type")
    return b


_EXTREME = ["0" * 33, "0" * 31 + "1" + "1" * 30 + "0", "0" * 16 + "1" + "0" * 16, "0" * 9 + "1111101001",
            "1", "010", "011", "00100", "00101", "00111", "0001000", "0001111", "000010000"]


def _inject(au, which):
    """Yields (description, mutated access unit) for every (field, extreme code) of the chosen header."""
    nals = _split_nals(au)
    for i, nal in enumerate(nals):
        t = (nal[0] >> 1) & 0x3f
        if which == "sps" and t == 33:
            walk = _walk_sps
        elif which == "pps" and t == 34:
            walk = _walk_pps
        elif which == "slice" and 16 <= t <= 21:
            walk = lambda r, t=t: _walk_slice(r, t)
        else:
            continue
        rbsp = _unescape(nal)
        b = walk(rbsp)
        for name, start, ln in b.fields:
            for code in _EXTREME:
                bits = b.bits[:start] + code + b.bits[start + ln:]
                bits += "0" * (-len(bits) % 8)
                out = bytes(int(bits[k:k + 8], 2) for k in range(0, len(bits), 8))
                m = list(nals); m[i] = out[:2] + _escape(out[2:])
                yield f"{name}<-{code[:12]}({len(code)})", _join_nals(m)
        return


@pytest.mark.timeout(120)
@pytest.mark.parametrize("which", ["sps", "pps", "slice"])
def test_extreme_exp_golomb_values_in_every_header_field(which):
    l = _lib.lib()
    n8 = 2048 * 2048 // 64
    qp8 = np.zeros(n8, np.int8); edge8 = np.zeros(n8, np.uint8); lm = np.zeros(n8 * 4, np.uint8); cm = np.zeros(n8 * 4, np.uint8)
    guard = [a.copy() for a in (qp8, edge8, lm, cm)]
    out5 = (C.c_ulonglong * 5)()
    streams = dict(all_streams() + cpu_extra_streams())
    base = [streams[k] for k in sorted(streams) if len(streams[k]) < 60000][:6]
    ran = rejected = 0
    for au in base:
        assert l.b200_debug_parse(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out5) == 0
        for desc, m in _inject(au, which):
            rc = l.b200_debug_parse(m, len(m), qp8.ctypes.data, edge8.ctypes.data, lm.ctypes.data, cm.ctypes.data, out5)
            ran += 1; rejected += rc != 0
            if rc == 0:       # a mutation that still decodes must describe a picture that fits the maps
                assert out5[3] * out5[4] <= 2048 * 2048, desc
    assert ran > 50 and rejected > ran // 3


def test_advice_r1_reproducer_min_cb_wraps():
    """ADVICE round 1 (high): log2_min_luma_coding_block_size_minus3 coded with 33 zero bits on a 12x12 picture used to
    pass the block-size check and overrun the ipm4/cd8/qp8/edge8 maps."""
    l = _lib.lib()
    streams = dict(all_streams() + cpu_extra_streams())
    au = streams[sorted(k for k in streams if len(streams[k]) < 60000)[0]]
    nals = _split_nals(au)
    i = next(k for k, n in enumerate(nals) if (n[0] >> 1) & 0x3f == 33)
    rb = _unescape(nals[i]); b = _walk_sps(rb)
    f = {n: (s, ln) for n, s, ln in b.fields}
    bits = b.bits
    for name, code in sorted((("log2_min_cb", "0" * 33), ("height", "0001101"), ("width", "0001101")), key=lambda t: -f[t[0]][0]):
        s, ln = f[name]; bits = bits[:s] + code + bits[s + ln:]
    bits += "0" * (-len(bits) % 8)
    out = bytes(int(bits[k:k + 8], 2) for k in range(0, len(bits), 8))
    nals[i] = out[:2] + _escape(out[2:])
    m = _join_nals(nals)
    buf = np.zeros(1 << 20, np.uint8); out5 = (C.c_ulonglong * 5)()
    assert l.b200_debug_parse(m, len(m), buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, out5) != 0


def test_emulation_prevention_removal_matches_the_byte_serial_rule():
    """7.4.2: the header stage strips emulation_prevention_three_byte with memchr + block copies; the result (RBSP bytes and the
    NAL offsets of the removed bytes, which the entry points are corrected by) must equal the byte-serial rule of the
    specification -- "0x03 after two zero bytes since the last removal" -- on strings made of little else than 0x00 / 0x03."""
    import ctypes as C
    from libheif_b200 import _lib
    l = _lib.lib()
    rng = np.random.default_rng(7)

    def serial(b):
        out, epb, zeros = bytearray(), [], 0
        for i, v in enumerate(b):
            if zeros >= 2 and v == 3:
                zeros = 0
                epb.append(i)
                continue
            out.append(v)
            zeros = zeros + 1 if v == 0 else 0
        return bytes(out), epb

    cases = [b"", b"\x00", b"\x00\x00\x03", b"\x00\x00\x03\x00\x00\x03", b"\x00\x00\x00\x03\x03", b"\x03\x00\x00\x03\x01", b"\x00\x00\x03\x00\x03"]
    for k in range(400):
        n = int(rng.integers(0, 300))
        alphabet = [np.array([0, 3], np.uint8), np.array([0, 0, 3, 1], np.uint8), np.arange(256, dtype=np.uint8)][k % 3]
        cases.append(bytes(alphabet[rng.integers(0, len(alphabet), n)]))
    cases.append(bytes(rng.integers(0, 4, 200000, dtype=np.uint8)))        # long: many block copies
    for b in cases:
        want, want_epb = serial(b)
        out = np.zeros(len(b) + 16, np.uint8)
        epb = np.zeros(len(b) + 1, np.uint32)
        cnt = C.c_size_t(0)
        n = l.b200_debug_unescape(b, len(b), out.ctypes.data, epb.ctypes.data, len(epb), C.byref(cnt))
        assert n == len(want) and bytes(out[:n]) == want, b[:40]
        assert cnt.value == len(want_epb) and epb[:cnt.value].tolist() == want_epb, b[:40]
