"""Transform stage, block by block: the decoder's scaling and inverse transforms (K1's residual4_lane / residual_big), its
chroma QP mapping, and the transform, (de)quantisation and intra-prediction primitives the host and GPU encoders share
(b200_hevc_enc_recon.h), each against a plain int64 numpy restatement of H.265, exactly.  Every legal extreme is reached by
choosing the input: dequantised coefficients of +-32767 with signs lined up with the transform matrix drive the residual of
8x8 and larger blocks past 16 bits at 10 and 12 bits (8.6.4.2 leaves it unbounded; only pred + res is clipped, 8.6.7).
One targeted stream per format then checks the same limits end to end."""
import ctypes as C
import math

import numpy as np
import pytest

from libheif_b200 import _lib
from libheif_b200 import hevc_enc
from intra_ref import filtered, predict, substitute

I32, I16, U8, U16 = np.int32, np.int16, np.uint8, np.uint16
E_INVALID = -1

# ------------------------------------------------------------------------------------------ restatement (numpy, int64)
# 8.6.4.2: the 32 magnitudes transMatrix lists for column 0 (coefficient rows 0..31 of the 32-point DCT)
MAGS = [64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67, 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4]
DST4 = np.array([[29, 55, 74, 84], [74, 74, 0, -74], [84, -29, -74, 55], [55, -84, 74, -29]], np.int64)
LEVEL_SCALE = [40, 45, 51, 57, 64, 72]
QUANT_SCALE = [26214, 23302, 20560, 18396, 16384, 14564]


def _dct32():
    # Entry [k][x] is the magnitude of phase k (2x + 1) (in units of pi / 64) folded into 0..32, with the sign of the cosine:
    # the spec's symmetry rule (columns 16..31 mirror 0..15 with sign (-1)^k) follows from it.
    m = np.zeros((32, 32), np.int64)
    for k in range(32):
        for x in range(32):
            c = math.cos(math.pi * k * (2 * x + 1) / 64)
            j = round(math.acos(abs(c)) * 64 / math.pi)
            m[k, x] = MAGS[j] if c > 0 else -MAGS[j]
    for k in range(32):                                 # the listed symmetry
        for x in range(16, 32):
            assert m[k, x] == (-1) ** k * m[k, 31 - x]
    return m


M32 = _dct32()


def tmat(lg, dst=False):
    """transMatrix of an n x n block: rows k << (5 - log2 n) of the 32-point matrix (8.6.4.2), or the 4x4 DST."""
    if dst:
        return DST4
    n = 1 << lg
    return M32[::32 // n, :n].copy()


def sf_of(factors, lg, y, x):
    """Scaling factor m[x][y] (7.4.5 / 8.6.4.2) from a 65-entry row: 8x8 raster (4x4 raster in the first 16), DC last."""
    if factors is None:
        return 16
    if lg == 2:
        return int(factors[y * 4 + x])
    if lg >= 4 and x == 0 and y == 0:
        return int(factors[64])
    return int(factors[((y >> (lg - 3)) << 3) + (x >> (lg - 3))])


def scale(levels, lg, bd, qp, factors=None):
    """8.6.2 / 8.6.3: d[y][x] = Clip3(-32768, 32767, (level * m * levelScale << qp / 6 + (1 << bdShift - 1)) >> bdShift)."""
    n = 1 << lg
    m = np.array([[sf_of(factors, lg, y, x) for x in range(n)] for y in range(n)], np.int64)
    bs = bd + lg - 5
    t = (levels.astype(np.int64) * m * (LEVEL_SCALE[qp % 6] << (qp // 6)) + (1 << (bs - 1))) >> bs
    return np.clip(t, -32768, 32767)


def inv_first(d, lg, dst=False):
    """First (vertical) stage with its 16-bit clip: g[y][x] = Clip3(-32768, 32767, (sum_k M[k][y] d[k][x] + 64) >> 7)."""
    return np.clip((tmat(lg, dst).T @ d.astype(np.int64) + 64) >> 7, -32768, 32767)


def inv_second(g, lg, bd, dst=False):
    """Second (horizontal) stage and the final shift, unclipped: r[y][x] = (sum_k g[y][k] M[k][x] + rnd) >> (20 - bd)."""
    bs = 20 - bd
    return (g.astype(np.int64) @ tmat(lg, dst) + (1 << (bs - 1))) >> bs


def residual(levels, lg, bd, qp, dst=False, tskip=False, raw=False, factors=None):
    """8.6.2: the residual block of TransCoeffLevel `levels` (n x n raster), int64 and unbounded."""
    if raw:
        return levels.astype(np.int64)
    d = scale(levels, lg, bd, qp, factors)
    if tskip:
        bs = 20 - bd
        return ((d << 7) + (1 << (bs - 1))) >> bs
    return inv_second(inv_first(d, lg, dst), lg, bd, dst)


def sat16(a):
    return np.clip(a, -32768, 32767)


def worst_case(lg, y0, x0, dst=False, neg=False, mag=32767):
    """Dequantised coefficients whose signs line up with the matrix for output (x0, y0): every first-stage value of row y0
    saturates with the sign of M[l][x0], so the residual there is the largest the block can give."""
    m = tmat(lg, dst)
    s = np.where(m[:, y0] >= 0, 1, -1)[:, None] * np.where(m[:, x0] >= 0, 1, -1)[None, :]
    return (-s if neg else s) * mag


# ------------------------------------------------------------------------------------------ restatement self-checks (CPU)
def test_matrices_near_orthogonal():
    for lg in (2, 3, 4, 5):
        n = 1 << lg
        for dst in ((False, True) if lg == 2 else (False,)):
            m = tmat(lg, dst)
            g = m @ m.T
            want = 64 * 64 * n
            assert np.all(np.abs(np.diag(g) - want) <= want // 100), (lg, dst)
            assert np.all(np.abs(g - np.diag(np.diag(g))) <= want // 100), (lg, dst)
    for lg in (2, 3, 4):                               # the smaller DCTs are the even rows of the next larger one
        assert np.array_equal(tmat(lg), tmat(lg + 1)[::2, :1 << lg])


def max_abs_residual(lg, bd, dst=False, low=-32767):
    """Largest |residual| over every output position of the sign-aligned blocks of dequantised coefficients 32767 / low."""
    n = 1 << lg
    best = 0
    for y0 in range(n):
        for x0 in range(n):
            for neg in (False, True):
                d = np.where(worst_case(lg, y0, x0, dst, neg) > 0, 32767, low)
                best = max(best, int(np.abs(inv_second(inv_first(d, lg, dst), lg, bd, dst)).max()))
    return best


@pytest.mark.parametrize("lg,dst,want", [(2, False, (1976, 7904, 31616)), (2, True, (1936, 7744, 30976)), (3, False, (3832, 15328, 61312)),
                                         (4, False, (7520, 30080, 120320)), (5, False, (14896, 59584, 238336))])
def test_worst_case_residuals(lg, dst, want):
    """Largest |residual| of dequantised coefficients of +-32767, per size and bit depth 8 / 10 / 12: past 16 bits for 8x8 ..
    32x32 at 12 bits and for 32x32 at 10 bits; a 4x4 block stays inside 16 bits even with -32768 in the mix."""
    for bd, w in zip((8, 10, 12), want):
        assert max_abs_residual(lg, bd, dst) == w, (lg, bd)
    if lg == 2:
        assert max_abs_residual(lg, 12, dst, -32768) <= 32767


# ------------------------------------------------------------------------------------------ K1 harness
class Block:
    """One block of the K1 harness: parameters, optional scaling factors, (pos, level) list."""

    def __init__(self, lg, bd, qp, levels=None, coefs=None, dst=False, tskip=False, raw=False, factors=None):
        n = 1 << lg
        if coefs is None:
            coefs = [(int(p), int(levels.flat[p])) for p in np.flatnonzero(levels)]
        self.lg, self.bd, self.qp, self.dst, self.tskip, self.raw, self.factors = lg, bd, qp, dst, tskip, raw, factors
        self.coefs = coefs
        self.levels = np.zeros((n, n), np.int64)
        for p, v in coefs:
            self.levels.flat[p] = v

    def want(self):
        return residual(self.levels, self.lg, self.bd, self.qp, self.dst, self.tskip, self.raw, self.factors)


def k1_pack(blocks):
    prm = np.array([[b.lg, b.bd, b.qp, int(b.dst), int(b.tskip), int(b.raw), int(b.factors is not None), len(b.coefs)] for b in blocks], I32)
    fac = np.zeros((len(blocks), 65), U8)
    for i, b in enumerate(blocks):
        if b.factors is not None:
            fac[i] = b.factors
    co = np.array([(p & 0xffff) | ((v & 0xffff) << 16) for b in blocks for (p, v) in b.coefs] or [0], np.uint32)
    return prm, fac, co


def k1_run(blocks):
    prm, fac, co = k1_pack(blocks)
    out = np.zeros((len(blocks), 1024), I16)
    _lib.check(_lib.lib().b200_debug_k1_residual(len(blocks), prm.ctypes.data, fac.ctypes.data, co.ctypes.data, out.ctypes.data))
    return [out[i, :1 << (2 * b.lg)].reshape(1 << b.lg, 1 << b.lg).astype(np.int64) for i, b in enumerate(blocks)]


# ------------------------------------------------------------------------------------------ K1 inputs
def qp_top(bd):
    return 51 + 6 * (bd - 8)


def factor_rows(rng):
    flat1, flat255 = np.full(65, 1, U8), np.full(65, 255, U8)
    mixed = rng.integers(1, 256, 65).astype(U8)
    mixed[64] = 255
    dc1 = np.full(65, 16, U8)
    dc1[64] = 1
    return [None, flat1, np.full(65, 16, U8), flat255, mixed, dc1]


def k1_blocks(lg, bd):
    rng = np.random.default_rng(1000 * lg + bd)
    n, top = 1 << lg, qp_top(bd)
    qps = sorted({0, 1, 5, 6, top // 2, top - 6, top - 1, top})
    kinds = [dict(dst=True), dict()] if lg == 2 else [dict()]
    out = []
    for kw in kinds:
        # sign-aligned worst cases: levels of 32767 dequantise to 32767 / -32768 at the top qp
        for y0, x0 in {(0, 0), (n - 1, n - 1), (0, n - 1), (n - 1, 0), (n // 2, 1)}:
            for neg in (False, True):
                lev = worst_case(lg, y0, x0, kw.get("dst", False), neg)
                out.append(Block(lg, bd, top, lev, **kw))
                out.append(Block(lg, bd, top, np.where(lev < 0, -32768, lev), **kw))
        # single extreme coefficients at the corners and on the last row / column only (maxrow / maxcol pruning, ncol rounded to 4)
        pos = [0, n - 1, (n - 1) * n, n * n - 1, (n - 1) * n + int(rng.integers(0, n)), int(rng.integers(0, n)) * n + n - 1,
               (n - 1) * n + 1, 1 * n + n - 1, (n - 1) * n + n // 2]
        for p in pos:
            for v in (32767, -32768, -32767, 1, -1):
                for qp in (0, top // 2, top):
                    out.append(Block(lg, bd, qp, coefs=[(p, v)], **kw))
        for f in factor_rows(rng):
            for qp in (0, top // 2, top):
                out.append(Block(lg, bd, qp, coefs=[(0, 32767), (n * n - 1, -32768), (n - 1, 1000)], factors=f, **kw))
                out.append(Block(lg, bd, qp, worst_case(lg, 0, 0, kw.get("dst", False)), factors=f, **kw))
        # nnz 1, 31, 32, 33 and n * n at random positions, random order
        for nnz in sorted({1, min(31, n * n), min(32, n * n), min(33, n * n), n * n}):
            for big in (False, True):
                ps = rng.permutation(n * n)[:nnz]
                vs = rng.integers(-32768, 32768, nnz) if big else rng.integers(-40, 41, nnz)
                vs = np.where(vs == 0, 1, vs)
                qp = int(rng.choice(qps))
                out.append(Block(lg, bd, qp, coefs=list(zip(ps.tolist(), vs.tolist())), factors=factor_rows(rng)[int(rng.integers(0, 6))], **kw))
        # seeded random dense blocks over the qp range
        for qp in qps:
            lev = rng.integers(-32768, 32768, (n, n)) if qp % 2 else rng.integers(-300, 301, (n, n))
            out.append(Block(lg, bd, qp, lev, **kw))
    # transform skip (4x4) and raw (cu_transquant_bypass / PCM) at the extremes
    for qp in (0, top // 2, top):
        ext = np.array([[32767, -32768] * (n // 2)] * n)
        if lg == 2:
            out.append(Block(lg, bd, qp, ext, tskip=True))
            out.append(Block(lg, bd, qp, ext, tskip=True, dst=True))
            out.append(Block(lg, bd, qp, ext, tskip=True, factors=factor_rows(rng)[3]))
        out.append(Block(lg, bd, qp, ext, raw=True))
        out.append(Block(lg, bd, qp, rng.integers(-32768, 32768, (n, n)), raw=True, dst=lg == 2))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("lg", [2, 3, 4, 5])
def test_k1_residual(cuda, lg, bd):
    """K1's scaling + inverse transform of every block == the restatement saturated to 16 bits; where the restatement fits
    in int16 (always for 4x4, transform skip, raw and 8-bit blocks) that is the restatement itself."""
    blocks = k1_blocks(lg, bd)
    got = k1_run(blocks)
    over = 0
    for i, (b, g) in enumerate(zip(blocks, got)):
        w = b.want()
        fits = w.min() >= -32768 and w.max() <= 32767
        over += not fits
        assert np.array_equal(g, sat16(w)), f"block {i}: lg {b.lg} bd {b.bd} qp {b.qp} dst {b.dst} ts {b.tskip} raw {b.raw} sf {b.factors is not None} nnz {len(b.coefs)}"
    overflows = lg >= 3 and bd == 12 or lg == 5 and bd >= 10
    assert (over > 0) == overflows, f"{over} blocks past 16 bits"


# ------------------------------------------------------------------------------------------ chroma QP (8.6.1, Table 8-10)
QPC_TABLE = {30: 29, 31: 30, 32: 31, 33: 32, 34: 33, 35: 33, 36: 34, 37: 34, 38: 35, 39: 35, 40: 36, 41: 36, 42: 37, 43: 37}


def chroma_qp_ref(qpy, off, bd, cat):
    qbd = 6 * (bd - 8)
    qpi = min(max(qpy + off, -qbd), 57)
    if cat == 1:
        qpc = qpi if qpi < 30 else (QPC_TABLE[qpi] if qpi <= 43 else qpi - 6)
    else:
        qpc = min(qpi, 51)
    return qpc + qbd


@pytest.mark.gpu
def test_chroma_qp(cuda):
    q = np.array([(qpy, off, bd, cat) for bd in range(8, 13) for cat in (1, 2, 3) for qpy in range(-6 * (bd - 8), 52) for off in range(-12, 13)], I32)
    # the domain reaches both ends of the qPi clip
    assert {-6 * (bd - 8) for bd in range(8, 13)} <= {max(a + b, -6 * (c - 8)) for a, b, c, _ in q.tolist()}
    assert (q[:, 0] + q[:, 1]).max() > 57
    out = np.zeros(len(q), I32)
    _lib.check(_lib.lib().b200_debug_chroma_qp(len(q), q.ctypes.data, out.ctypes.data))
    want = np.array([chroma_qp_ref(*r) for r in q.tolist()], I32)
    assert np.array_equal(out, want)


# ------------------------------------------------------------------------------------------ encoder transform primitives
def enc_ref(p, a):
    """The six stages of b200_debug_enc_transform_* on input a (n x n): fwd_col, fwd_row, quant_level, dequant, inv_col,
    inv_row, each applied to a itself."""
    lg, dst, bd, qp, m = p
    n = 1 << lg
    M = tmat(lg, bool(dst))
    a = a.astype(np.int64)
    s1 = lg + bd - 9
    fc = (M @ a + (1 << (s1 - 1))) >> s1                       # out[k][x] = sum_y M[k][y] a[y][x]
    fr = (a @ M.T + (1 << (lg + 5))) >> (lg + 6)              # out[y][k] = sum_x M[k][x] a[y][x]
    qb = 14 + qp // 6 + 15 - bd - lg
    ql = np.minimum((np.abs(a) * QUANT_SCALE[qp % 6] + (171 << (qb - 9))) >> qb, 32767) * np.where(a < 0, -1, 1)
    dq = scale(a, lg, bd, qp, np.full(65, m, U8) if m != 16 else None)
    ic = inv_first(a, lg, bool(dst))
    ir = inv_second(a, lg, bd, bool(dst))
    return [x.reshape(n, n) for x in (fc, fr, ql, dq, ic, ir)]


def enc_cases(bds):
    rng = np.random.default_rng(77)
    prm, ins = [], []
    for bd in bds:
        for lg in (2, 3, 4, 5):
            n = 1 << lg
            for dst in ((0, 1) if lg == 2 else (0,)):
                for qp in (0, 1, 27, qp_top(bd)):
                    for kind in range(5):
                        if kind == 0:
                            a = rng.integers(-(1 << bd) + 1, 1 << bd, (n, n))            # residual range
                        elif kind == 1:
                            a = rng.integers(-32768, 32768, (n, n))
                        elif kind == 2:
                            a = worst_case(lg, 0, 0, bool(dst))
                        elif kind == 3:
                            a = np.where(worst_case(lg, n - 1, 0, bool(dst)) < 0, -32768, 32767)
                        else:
                            a = np.zeros((n, n), np.int64)
                            a[0, 0], a[-1, -1], a[0, -1] = -32768, 32767, 1
                        prm.append((lg, dst, bd, qp, int(rng.choice([1, 16, 255]))))
                        buf = np.zeros(1024, I32)
                        buf[:n * n] = a.reshape(-1)
                        ins.append(buf)
    return np.array(prm, I32), np.array(ins, I32)


def enc_transform(side, prm, ins):
    out = np.zeros((len(prm), 6, 1024), I32)
    f = _lib.lib().b200_debug_enc_transform_host if side == "host" else _lib.lib().b200_debug_enc_transform_device
    _lib.check(f(len(prm), prm.ctypes.data, ins.ctypes.data, out.ctypes.data))
    return out


def check_enc_transform(prm, ins, got):
    names = ("fwd_col", "fwd_row", "quant_level", "dequant", "inv_col", "inv_row")
    for i, p in enumerate(prm.tolist()):
        n = 1 << p[0]
        want = enc_ref(p, ins[i, :n * n].reshape(n, n))
        for st in range(6):
            assert np.array_equal(got[i, st, :n * n].reshape(n, n), want[st]), f"{names[st]}: block {i} (log2n, dst, bd, qp, m) = {p}"


def test_enc_transform_host():
    """The host encoder's transform primitives at 8, 10 and 12 bits == the restatement."""
    prm, ins = enc_cases((8, 10, 12))
    check_enc_transform(prm, ins, enc_transform("host", prm, ins))


@pytest.mark.gpu
def test_enc_transform_device(cuda):
    """The GPU encoder's device code (dct_coef() matrices) == the host code (kDctPhase) == the restatement, at 8 bits: the
    GPU encoder's only bit depth."""
    prm, ins = enc_cases((8,))
    dev = enc_transform("device", prm, ins)
    check_enc_transform(prm, ins, dev)
    host = enc_transform("host", prm, ins)
    for i, p in enumerate(prm.tolist()):
        n2 = 1 << (2 * p[0])
        assert np.array_equal(dev[i, :, :n2], host[i, :, :n2])


# ------------------------------------------------------------------------------------------ intra prediction (8.4.4.2.2 - 8.4.4.2.6)
def pred_cases(bds):
    """(log2n, bd, luma, plane filtered, strong) x neighbours: random, all 0, all maxv, a smooth ramp (strong smoothing),
    and partly unavailable (-1) runs."""
    rng = np.random.default_rng(5)
    prm, refs = [], []
    for bd in bds:
        maxv = (1 << bd) - 1
        for lg in (2, 3, 4, 5):
            n = 1 << lg
            for luma, plane in ((1, 1), (0, 0), (0, 1)):
                for strong in ((0, 1) if luma else (0,)):
                    for kind in range(6):
                        r = np.zeros(129, I16)
                        if kind == 0:
                            r[:4 * n + 1] = rng.integers(0, maxv + 1, 4 * n + 1)
                        elif kind == 1:
                            r[:4 * n + 1] = 0
                        elif kind == 2:
                            r[:4 * n + 1] = maxv
                        elif kind == 3:
                            r[:4 * n + 1] = (np.arange(4 * n + 1) * (maxv // 8) // (4 * n)) + maxv // 3
                        else:
                            r[:4 * n + 1] = rng.integers(0, maxv + 1, 4 * n + 1)
                            cut = sorted(rng.integers(0, 4 * n + 2, 2))
                            r[cut[0]:cut[1]] = -1
                            if kind == 5:
                                r[:2 * n + 1] = -1
                        prm.append((lg, bd, luma, plane, strong))
                        refs.append(r)
    refs.append(np.full(129, -1, I16))                    # nothing available
    prm.append((5, bds[0], 1, 1, 1))
    return np.array(prm, I32), np.array(refs, I16)


def enc_predict(side, prm, refs):
    rf = np.zeros((len(prm), 258), I16)
    pred = np.zeros((len(prm), 35, 1024), I32)
    f = _lib.lib().b200_debug_enc_predict_host if side == "host" else _lib.lib().b200_debug_enc_predict_device
    _lib.check(f(len(prm), prm.ctypes.data, refs.ctypes.data, rf.ctypes.data, pred.ctypes.data))
    return rf, pred


def check_predict(prm, refs, rf, pred):
    for i, (lg, bd, luma, plane, strong) in enumerate(prm.tolist()):
        n = 1 << lg
        r = substitute([int(v) for v in refs[i, :4 * n + 1]], n, bd)
        f = filtered(r, n, bd, strong)
        assert rf[i, :4 * n + 1].tolist() == r, f"substitute_refs: block {i}"
        assert rf[i, 129:129 + 4 * n + 1].tolist() == f, f"filter_refs: block {i}"
        for mode in range(35):
            want = predict(r, f, n, mode, luma, plane, bd)
            assert np.array_equal(pred[i, mode, :n * n].reshape(n, n), want), f"block {i} (log2n, bd, luma, plane, strong) = {(lg, bd, luma, plane, strong)} mode {mode}"


def test_enc_predict_host():
    """The host encoder's neighbour substitution, filtering and prediction of all 35 modes at 8, 10 and 12 bits == 8.4.4.2."""
    prm, refs = pred_cases((8, 10, 12))
    check_predict(prm, refs, *enc_predict("host", prm, refs))


@pytest.mark.gpu
def test_enc_predict_device(cuda):
    prm, refs = pred_cases((8,))
    rf, pred = enc_predict("device", prm, refs)
    check_predict(prm, refs, rf, pred)
    hrf, hpred = enc_predict("host", prm, refs)
    for i, p in enumerate(prm.tolist()):
        n = 1 << p[0]
        assert np.array_equal(rf[i, :4 * n + 1], hrf[i, :4 * n + 1]) and np.array_equal(rf[i, 129:130 + 4 * n], hrf[i, 129:130 + 4 * n])
        assert np.array_equal(pred[i, :, :n * n], hpred[i, :, :n * n])


# ------------------------------------------------------------------------------------------ argument refusals (CPU)
def _k1_call(blocks_prm, coefs, factors=None, n=None):
    prm = np.array(blocks_prm, I32).reshape(-1, 8)
    co = np.array(coefs or [0], np.uint32)
    out = np.zeros((max(len(prm), 1), 1024), I16)
    return _lib.lib().b200_debug_k1_residual(len(prm) if n is None else n, prm.ctypes.data, None if factors is None else factors.ctypes.data,
                                             co.ctypes.data, out.ctypes.data)


@pytest.mark.parametrize("prm,coefs,why", [
    ([1, 8, 0, 0, 0, 0, 0, 0], [], "log2 size 1"), ([6, 8, 0, 0, 0, 0, 0, 0], [], "log2 size 6"),
    ([3, 7, 0, 0, 0, 0, 0, 0], [], "bit depth 7"), ([3, 13, 0, 0, 0, 0, 0, 0], [], "bit depth 13"),
    ([3, 8, -1, 0, 0, 0, 0, 0], [], "qp -1"), ([3, 8, 52, 0, 0, 0, 0, 0], [], "qp 52 at 8 bits"), ([3, 12, 76, 0, 0, 0, 0, 0], [], "qp 76 at 12 bits"),
    ([3, 8, 0, 1, 0, 0, 0, 0], [], "DST on 8x8"), ([3, 8, 0, 0, 1, 0, 0, 0], [], "transform skip on 8x8"),
    ([2, 8, 0, 0, 1, 1, 0, 0], [], "transform skip and raw"), ([2, 8, 0, 2, 0, 0, 0, 0], [], "flag 2"),
    ([2, 8, 0, 0, 0, 0, 0, 17], list(range(17)), "nnz 17 on 4x4"), ([2, 8, 0, 0, 0, 0, 0, -1], [], "nnz -1"),
    ([2, 8, 0, 0, 0, 0, 0, 1], [16 | (5 << 16)], "position 16 on 4x4"), ([5, 8, 0, 0, 0, 0, 0, 1], [1024], "position 1024 on 32x32"),
    ([3, 8, 0, 0, 0, 0, 0, 2], [3 | (1 << 16), 3 | (2 << 16)], "position twice"),
    ([3, 8, 0, 0, 0, 0, 1, 0], [], "factors used, none given"),
    ([3, 8, 0, 0, 0, 0, 0, 0, 3, 8, 0, 1, 0, 0, 0, 0], [], "second block bad"),
])
def test_k1_residual_refusals(prm, coefs, why):
    assert _k1_call(prm, coefs) == E_INVALID, why


def test_k1_residual_refusals_counts():
    assert _k1_call([3, 8, 0, 0, 0, 0, 0, 0], [], n=0) == E_INVALID
    assert _k1_call([3, 8, 0, 0, 0, 0, 0, 0], [], n=-3) == E_INVALID
    assert _lib.lib().b200_debug_k1_residual(1, None, None, None, None) == E_INVALID


@pytest.mark.parametrize("q", [(-1, 0, 8, 1), (52, 0, 8, 1), (-13, 0, 10, 1), (0, 13, 8, 1), (0, -13, 8, 1), (0, 0, 7, 1), (0, 0, 13, 1), (0, 0, 8, 0), (0, 0, 8, 4)])
def test_chroma_qp_refusals(q):
    qq = np.array([(20, 0, 8, 1), q], I32)
    out = np.zeros(2, I32)
    assert _lib.lib().b200_debug_chroma_qp(2, qq.ctypes.data, out.ctypes.data) == E_INVALID


@pytest.mark.parametrize("side", ["host", "device"])
@pytest.mark.parametrize("p,bad", [((1, 0, 8, 0, 16), None), ((6, 0, 8, 0, 16), None), ((3, 1, 8, 0, 16), None), ((2, 2, 8, 0, 16), None),
                                   ((2, 0, 7, 0, 16), None), ((2, 0, 13, 0, 16), None), ((2, 0, 8, 52, 16), None), ((2, 0, 8, -1, 16), None),
                                   ((2, 0, 8, 0, 0), None), ((2, 0, 8, 0, 256), None), ((2, 0, 8, 0, 16), 32768), ((2, 0, 8, 0, 16), -32769)])
def test_enc_transform_refusals(side, p, bad):
    prm = np.array([p], I32)
    ins = np.zeros((1, 1024), I32)
    if bad is not None:
        ins[0, 15] = bad
    out = np.zeros((1, 6, 1024), I32)
    f = _lib.lib().b200_debug_enc_transform_host if side == "host" else _lib.lib().b200_debug_enc_transform_device
    assert f(1, prm.ctypes.data, ins.ctypes.data, out.ctypes.data) == E_INVALID


@pytest.mark.parametrize("side", ["host", "device"])
@pytest.mark.parametrize("p,bad", [((1, 8, 1, 1, 0), None), ((6, 8, 1, 1, 0), None), ((2, 7, 1, 1, 0), None), ((2, 13, 1, 1, 0), None),
                                   ((2, 8, 1, 0, 0), None), ((2, 8, 2, 1, 0), None), ((2, 8, 1, 1, 2), None), ((2, 8, 1, 1, 0), 256), ((2, 8, 1, 1, 0), -2)])
def test_enc_predict_refusals(side, p, bad):
    prm = np.array([p], I32)
    refs = np.zeros((1, 129), I16)
    if bad is not None:
        refs[0, 16] = bad
    rf = np.zeros((1, 258), I16)
    pred = np.zeros((1, 35, 1024), I32)
    f = _lib.lib().b200_debug_enc_predict_host if side == "host" else _lib.lib().b200_debug_enc_predict_device
    assert f(1, prm.ctypes.data, refs.ctypes.data, rf.ctypes.data, pred.ctypes.data) == E_INVALID


# ------------------------------------------------------------------------------------------ forced-level streams
def forced_encode(bd, cfmt, log2ctb, pattern, count=64, sdh=0, seed=0x7A11):
    w, h = 128, 64
    y, cb, cr = hevc_enc.synthetic_image(seed, w, h, bd, cfmt)
    p = hevc_enc.default_params(width=w, height=h, bit_depth=bd, chroma_format_idc=cfmt, log2_ctb_size=log2ctb, sign_data_hiding=sdh,
                                seed=seed, still_picture=0)
    sx, sy = (1, 1) if cfmt == 1 else (0, 0)
    rec = [np.zeros((h, w), U16), np.zeros((h >> sy, w >> sx), U16), np.zeros((h >> sy, w >> sx), U16)]
    pat = np.ascontiguousarray(pattern, I16)
    data, size = C.POINTER(C.c_uint8)(), C.c_size_t()
    l = _lib.lib()
    rc = l.b200_debug_hevc_encode_forced_levels(C.byref(p), y.ctypes.data, cb.ctypes.data, cr.ctypes.data, y.strides[0], cb.strides[0],
                                                 pat.ctypes.data, count, C.byref(data), C.byref(size), rec[0].ctypes.data, rec[1].ctypes.data,
                                                 rec[2].ctypes.data)
    if rc:
        return rc, None, None
    au = C.string_at(data, size.value)
    l.b200_free(data)
    return 0, au, rec


def test_forced_levels_refusals():
    pat = np.full((32, 32), 32767, I16)
    assert forced_encode(8, 1, 5, pat, sdh=1)[0] == E_INVALID            # sign-data hiding would drop signs of the pattern
    assert forced_encode(8, 1, 5, pat, count=-1)[0] == E_INVALID


def test_forced_levels_zero_count_is_the_normal_encoder():
    pat = np.full((32, 32), 32767, I16)
    rc, au, _ = forced_encode(10, 1, 5, pat, count=0)
    assert rc == 0
    y, cb, cr = hevc_enc.synthetic_image(0x7A11, 128, 64, 10, True)
    assert au == hevc_enc.encode_intra(y, cb, cr, bit_depth=10, log2_ctb_size=5, sign_data_hiding=0, seed=0x7A11, still_picture=0)


FORCED = [(8, 1, 5), (8, 1, 6), (10, 1, 5), (10, 1, 6), (12, 1, 5), (12, 1, 6), (12, 3, 5)]


@pytest.mark.gpu
@pytest.mark.parametrize("neg", [False, True], ids=["pos", "neg"])
@pytest.mark.parametrize("bd,cfmt,log2ctb", FORCED, ids=[f"{b}bit-{'420' if c == 1 else '444'}-ctb{1 << l}" for b, c, l in FORCED])
def test_forced_level_stream(cuda, bd, cfmt, log2ctb, neg):
    """A conforming stream whose transform blocks of 8x8 and up hold the sign-aligned worst case: the C restatement, FFmpeg
    (8 and 12 bits), both decoder front-ends, and the decoder's stage 1 (before deblocking) against the encoder's own
    reconstruction."""
    import libheif_b200 as lb
    from oracle import bindings as ob
    pattern = worst_case(5, 0, 0)
    pattern = np.where(pattern < 0, -32768, 32767) if not neg else np.where(pattern < 0, 32767, -32768)
    rc, au, rec = forced_encode(bd, cfmt, log2ctb, pattern)
    assert rc == 0
    want0, info = ob.restatement_decode(au, 0)
    want1, _ = ob.restatement_decode(au, 1)
    assert info["bit_depth"] == bd
    for c in range(3):
        assert np.array_equal(want1[c], rec[c]), f"restatement stage 1 != encoder reconstruction, plane {c}"
    # FFmpeg's 10-bit output differs from the restatement (and from this decoder) on these streams, in the samples of the
    # blocks past 16 bits; it is not a reference at that depth
    if bd != 10:
        ff, ffbd, _ = ob.ffmpeg_decode(au)
        assert ffbd == bd
        for c in range(3):
            assert np.array_equal(ff[c], want0[c]), f"FFmpeg != restatement, plane {c}"
    dec = lb.Decoder(host_threads=4)
    try:
        for device in (True, False):
            dec.set_front_end(device)
            for stage, want in ((1, want1), (0, want0)):
                dec.set_debug_stage(stage)
                dec.decode_image(au)
                got = dec.debug_tile(0, 128, 64) if stage else dec.planes_host()
                for c in range(3):
                    assert np.array_equal(got[c].astype(U16), want[c]), f"{'device' if device else 'host'} front-end, stage {stage}, plane {c}"
    finally:
        dec.close()
