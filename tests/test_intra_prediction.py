"""Intra prediction in the decoder's reconstruction kernel K1, against the restatement of tests/intra_ref.py, exactly:
- constructed blocks through K1's own make_desc + predict_tb (b200_debug_k1_predict), in K1's lane and shared-memory layout for
  each kind of work item (luma; the 4:2:0 Cb + Cr pair on two half-warps; a 4:2:2 or 4:4:4 chroma plane): every mode at every
  size, every aligned position in CTBs of 16, 32 and 64, all CTB-neighbour combinations, right / bottom edge CTBs of every legal
  remaining size, thresholds of the smoothing decisions, clipping edge filters and residuals, PCM.  Samples that must not be
  read (unavailable, outside the picture) hold random values, and the whole tile is compared after the call;
- the descriptors phase A builds for every stream of hevc_cases and every fixture (b200_debug_k1_descriptors, host only),
  against 6.4.1 evaluated on the slices and tiles the headers define."""
from collections import Counter

import numpy as np
import pytest

from libheif_b200 import _lib
from hevc_cases import SYNTH, SYNTH_CPU_EXTRA, fixture_streams, synth_stream
from intra_ref import ANGLE, PicCtx, filter_flag, filtered, mark_neighbours, neighbour_offsets, predict, substitute, tile_boundaries_from_ids

E_INVALID = -1
PAD, TILE, TOP, RES, REF = 16, 64 * 80, 256, 1024, 129
LUMA, PAIR, P422, P444 = 0, 1, 2, 3
SUB = {LUMA: (1, 1), PAIR: (2, 2), P422: (2, 1), P444: (1, 1)}       # SubWidthC, SubHeightC of the kind's component
SENT = -32768


def comp_size(kind, lc):
    sw, sh = SUB[kind]
    return (1 << lc) // sw, (1 << lc) // sh


def max_lg(kind):
    return 5 if kind in (LUMA, P444) else 4


# ------------------------------------------------------------------------------------------ constructed cases
class Case:
    """One block of b200_debug_k1_predict: the make_desc inputs, the shared-memory images of its component(s), the residuals."""

    def __init__(self, rng, bd, kind, lc, lg, bx, by, mode, cx0, cy0, cw, ch, nb, strong=1, coded=(1, 1), pcm=0, content="random"):
        self.bd, self.kind, self.lc, self.lg, self.bx, self.by, self.mode = bd, kind, lc, lg, bx, by, mode
        self.cx0, self.cy0, self.cw, self.ch, self.nb, self.strong, self.pcm = cx0, cy0, cw, ch, tuple(nb), strong, pcm
        self.ncomp = 2 if kind == PAIR else 1
        self.coded = (coded[0], coded[1] if kind == PAIR else 0)
        self.tw, self.th = comp_size(kind, lc)
        n, maxv, S = 1 << lg, (1 << bd) - 1, self.tw + PAD
        self.tiles = np.zeros((self.ncomp, self.th, S), np.int64)
        self.tops = np.zeros((self.ncomp, TOP), np.int64)
        self.res = np.zeros((self.ncomp, n, n), np.int64)
        ntop = PAD + 2 * self.tw + 16
        for c in range(self.ncomp):
            if content == "zero":
                v = 0
            elif content == "max":
                v = maxv
            else:
                v = None
            self.tiles[c] = rng.integers(0, maxv + 1, (self.th, S)) if v is None else v
            self.tops[c, :ntop] = rng.integers(0, maxv + 1, ntop) if v is None else v
            if pcm:
                self.res[c] = rng.integers(0, maxv + 1, (n, n))
            elif content in ("res_clip", "zero", "max"):
                self.res[c] = rng.choice([-32768, 32767, -maxv, maxv, 0, 1, -1], (n, n))
            else:
                self.res[c] = rng.integers(-maxv, maxv + 1, (n, n))
        self.content = content

    @property
    def n(self):
        return 1 << self.lg

    def record(self):
        return [self.kind, self.lc, self.bd, self.strong, self.bx, self.by, self.lg, self.mode, self.coded[0], self.coded[1], self.pcm,
                self.cx0, self.cy0, self.cw, self.ch, *self.nb]

    def slots(self, i):
        """(image, index) of r[i] in the component images, or None where the sample lies outside them"""
        n = self.n
        x, y = (-1, 2 * n - 1 - i) if i < 2 * n else (i - 2 * n - 1, -1)
        if y >= 0:
            return ("tile", self.by + y, PAD + self.bx - 1) if self.by + y < self.th else None
        if self.by > 0:
            return ("tile", self.by - 1, PAD + self.bx + x) if PAD + self.bx + x < self.tw + PAD else None
        return ("top", PAD + self.bx + x)

    def get_r(self, c, i):
        s = self.slots(i)
        if s is None:
            return None
        return int(self.tiles[c, s[1], s[2]]) if s[0] == "tile" else int(self.tops[c, s[1]])

    def set_r(self, c, vals):
        for i, v in enumerate(vals):
            s = self.slots(i)
            if s is None:
                continue
            if s[0] == "tile":
                self.tiles[c, s[1], s[2]] = v
            else:
                self.tops[c, s[1]] = v

    def ctx(self):
        """A picture in which the CTB-neighbour flags hold: CTBs carry distinct slices except the current one and the
        neighbours whose flag is set (one tile, raster order)."""
        sw, sh = SUB[self.kind]
        w, h = self.cw * sw, self.ch * sh
        ctb = 1 << self.lc
        wctb, hctb = -(-w // ctb), -(-h // ctb)
        rx, ry = self.cx0 * sw // ctb, self.cy0 * sh // ctb
        lab = 1000 + np.arange(wctb * hctb)
        lab[ry * wctb + rx] = 0
        for (dx, dy), f in zip(((-1, 0), (-1, -1), (0, -1), (1, -1)), self.nb):
            if f:
                lab[(ry + dy) * wctb + rx + dx] = 0
        return PicCtx(w, h, self.lc, lab)


def desc_mask(d, n):
    """the availability of r[0 .. 4n] a descriptor word states"""
    fL, fC, fT = (d >> 18) & 1, (d >> 19) & 1, (d >> 20) & 1
    blc, trc = ((d >> 21) & 15) * 4, ((d >> 25) & 15) * 4
    i = np.arange(4 * n + 1)
    return (((i >= n - blc) & (i < n)) | (fL & (i >= n) & (i < 2 * n)).astype(bool) | ((i == 2 * n) & bool(fC)) |
            (bool(fT) & (i > 2 * n) & (i <= 3 * n)) | ((i > 3 * n) & (i <= 3 * n + trc)))


def expected(case, cov=None):
    """(availability, per component: raw r, substituted r, filtered r or None, block) of the restatement"""
    n, bd, kind, mode = case.n, case.bd, case.kind, case.mode
    sw, sh = SUB[kind]
    avail = mark_neighbours(case.ctx(), sw, sh, [case.cx0 + case.bx], [case.cy0 + case.by], n)[0]
    luma, plane = kind == LUMA, kind in (LUMA, P444)
    strong = case.strong if luma else 0
    maxv = (1 << bd) - 1
    out = []
    for c in range(case.ncomp):
        raw = [case.get_r(c, i) if avail[i] else -1 for i in range(4 * n + 1)]
        assert all(v is not None for v in raw), "an available neighbour outside the images"
        r = substitute(raw, n, bd)
        flag = filter_flag(plane, mode, n)
        f = filtered(r, n, bd, strong)
        pred = predict(r, f, n, mode, luma, plane, bd)
        res = case.res[c]
        if case.pcm:
            blk = res.copy()
        elif case.coded[c]:
            blk = np.clip(pred + res, 0, maxv)
        else:
            blk = pred
        out.append((raw, r, f if flag else None, blk))
        if cov is not None:
            branches(cov, case, avail, r, flag, strong, pred, res, c)
    return avail, out


def branches(cov, case, avail, r, flag, strong, pred, res, c):
    """Branch counters of the restatement for one component of a case"""
    n, bd, mode = case.n, case.bd, case.mode
    maxv, thr = (1 << bd) - 1, 1 << (bd - 5)
    if not avail.any():
        cov["sub"]["none"] += 1
    else:
        k = int(np.argmax(avail))
        cov["sub"]["first_" + ("bl" if k < n else "l" if k < 2 * n else "c" if k == 2 * n else "t" if k <= 3 * n else "tr")] += 1
    blc, trc = int(avail[:n].sum()), int(avail[3 * n + 1:].sum())
    if 0 < blc < n:
        cov["sub"]["bl_partial"] += 1
    if 0 < trc < n:
        cov["sub"]["tr_partial"] += 1
    if flag:
        left_c = abs(r[2 * n] + r[0] - 2 * r[n])
        top_c = abs(r[2 * n] + r[4 * n] - 2 * r[3 * n])
        if strong and n == 32:
            c1, c2 = top_c < thr, left_c < thr
            cov["filter"]["strong" if c1 and c2 else "121"] += 1
            if not c1 and c2 and top_c == thr:
                cov["filter"]["strong_top_fails_at_thr"] += 1
            if c1 and not c2 and left_c == thr:
                cov["filter"]["strong_left_fails_at_thr"] += 1
            if c1 and c2 and (top_c == thr - 1 or left_c == thr - 1):
                cov["filter"]["strong_at_thr_minus_1"] += 1
        else:
            cov["filter"]["121"] += 1
    else:
        cov["filter"]["none"] += 1
    if case.kind in (LUMA, P444) and n in (8, 16) and mode != 1:
        dist, t = min(abs(mode - 26), abs(mode - 10)), {8: 7, 16: 1}[n]
        if dist in (t, t + 1):
            cov["thres"][f"n{n}_{'eq' if dist == t else 'plus1'}"] += 1
    luma = case.kind == LUMA
    if mode == 1 and luma and n < 32:
        cov["mode"]["dc_edge"] += 1
    if mode in (10, 26) and luma and n < 32:
        lf, cn, tp = [r[2 * n - 1 - y] for y in range(n)], r[2 * n], [r[2 * n + 1 + x] for x in range(n)]
        edge = [tp[0] + ((lf[y] - cn) >> 1) for y in range(n)] if mode == 26 else [lf[0] + ((tp[x] - cn) >> 1) for x in range(n)]
        if min(edge) < 0:
            cov["mode"][f"m{mode}_clip0"] += 1
        if max(edge) > maxv:
            cov["mode"][f"m{mode}_clipmax"] += 1
    if 11 <= mode <= 25 and (n * ANGLE[mode]) >> 5 < -1:
        cov["mode"]["neg_projection"] += 1
    if mode >= 2 and any(((k + 1) * ANGLE[mode]) & 31 == 0 for k in range(n)):
        cov["mode"]["ifact0"] += 1
    if case.pcm:
        cov["res"]["pcm"] += 1
    elif case.coded[c]:
        s = pred + res
        if s.min() < 0:
            cov["res"]["clip0"] += 1
        if s.max() > maxv:
            cov["res"]["clipmax"] += 1
    else:
        cov["res"]["uncoded"] += 1


def _pick_nb(kind, lc, cx0, cy0, cw, k):
    tw, th = comp_size(kind, lc)
    nb = [(k >> b) & 1 for b in range(4)]
    return [nb[0] and cx0 > 0, nb[1] and cx0 > 0 and cy0 > 0, nb[2] and cy0 > 0, nb[3] and cy0 > 0 and cx0 + tw < cw]


def strong_ramp(case, d_top, d_left):
    """neighbours of a 32x32 block, smooth, with |corner + top[63] - 2 top[31]| = |d_top| and the left one = |d_left|"""
    maxv = (1 << case.bd) - 1
    c = maxv // 2
    step = max(1, maxv // 256)
    for comp in range(case.ncomp):
        tr, bl = c + 64 * step + (abs(d_top) & 1), c - 64 * step - (abs(d_left) & 1)
        r = [0] * 129
        r[64] = c
        for x in range(64):
            r[65 + x] = c + (tr - c) * (x + 1) // 64
        for y in range(64):
            r[63 - y] = c + (bl - c) * (y + 1) // 64
        r[128], r[0] = tr, bl
        r[96] = (c + tr - d_top) // 2
        r[32] = (c + bl - d_left) // 2
        assert abs(c + tr - 2 * r[96]) == abs(d_top) and abs(c + bl - 2 * r[32]) == abs(d_left)
        case.set_r(comp, r)


def edge_clip(case, low):
    """neighbours that push the mode-10 / mode-26 boundary filters below 0 (low) or above maxv"""
    maxv = (1 << case.bd) - 1
    n = case.n
    a, b = (0, maxv) if low else (maxv, 0)
    case.set_r(0, [a] * (2 * n) + [b] + [a] * (2 * n))


def cases_for(bd):
    rng = np.random.default_rng(1234 + bd)
    out = []
    k = 0
    contents = ["random", "random", "zero", "max", "res_clip", "random"]
    for kind in (LUMA, PAIR, P422, P444):
        for lc in (4, 5, 6):
            tw, th = comp_size(kind, lc)
            for lg in range(2, max_lg(kind) + 1):
                n = 1 << lg
                if n > tw or n > th:
                    continue
                # every aligned position, in an interior CTB and in the top-left one
                for by in range(0, th - n + 1, n):
                    for bx in range(0, tw - n + 1, n):
                        k += 1
                        corner = k % 4 == 0
                        cx0, cy0 = (0, 0) if corner else (tw, th)
                        cw, ch = 3 * tw, 2 * th
                        out.append(Case(rng, bd, kind, lc, lg, bx, by, (k * 7 + lg) % 35, cx0, cy0, cw, ch, _pick_nb(kind, lc, cx0, cy0, cw, k),
                                        strong=k % 5 != 0, coded=(k % 3 != 0, k % 4 != 1), pcm=int(k % 13 == 6), content=contents[k % len(contents)]))
                # every mode
                for mode in range(35):
                    k += 1
                    bx, by = int(rng.integers(0, tw // n)) * n, int(rng.integers(0, th // n)) * n
                    out.append(Case(rng, bd, kind, lc, lg, bx, by, mode, tw, th, 3 * tw, 2 * th, _pick_nb(kind, lc, tw, th, 3 * tw, k | 5),
                                    strong=1, coded=(k % 2, (k + 1) % 2), content=contents[k % len(contents)]))
                # right / bottom edge CTBs of every legal remaining size: above-right and below-left cut by the picture
                stepx = 4 if SUB[kind][0] == 2 else 8
                stepy = 4 if SUB[kind][1] == 2 else 8
                for rem in range(stepx, tw + 1, stepx):
                    for bx in range(0, rem - n + 1, n):
                        if bx + 2 * n <= rem and bx + n < tw:
                            continue
                        for by in sorted({0, th - n, n if n < th else 0}):
                            k += 1
                            out.append(Case(rng, bd, kind, lc, lg, bx, by, k % 35, tw, th, tw + rem, 2 * th, _pick_nb(kind, lc, tw, th, tw + rem, 15),
                                            content=contents[k % len(contents)]))
                for rem in range(stepy, th + 1, stepy):
                    for by in range(0, rem - n + 1, n):
                        if by + 2 * n <= rem and by + n < th:
                            continue
                        for bx in sorted({b for b in (0, n, 2 * n, tw - n) if 0 <= b <= tw - n}):
                            k += 1
                            out.append(Case(rng, bd, kind, lc, lg, bx, by, k % 35, tw, th, 3 * tw, th + rem, _pick_nb(kind, lc, tw, th, 3 * tw, 15),
                                            content=contents[k % len(contents)]))
    # all 16 CTB-neighbour combinations at the CTB's corner blocks
    for kind in (LUMA, PAIR, P422, P444):
        for f in range(16):
            for lc in (4, 6):
                tw, th = comp_size(kind, lc)
                for bx, by in ((0, 0), (tw - 4, 0), (0, th - 4), (4, 0), (0, 4)):
                    k += 1
                    out.append(Case(rng, bd, kind, lc, 2, bx, by, k % 35, tw, th, 3 * tw, 2 * th, [(f >> b) & 1 for b in range(4)]))
            # a block as wide as the CTB at its top-left corner: with only nbAR set, the above-right run is all there is
            for lc in (4, 5):
                tw, th = comp_size(kind, lc)
                lg = tw.bit_length() - 1
                if lg <= max_lg(kind) and tw <= th:
                    k += 1
                    out.append(Case(rng, bd, kind, lc, lg, 0, 0, k % 35, tw, th, 3 * tw, 2 * th, [(f >> b) & 1 for b in range(4)]))
    # strong smoothing: each condition at its threshold and one below, alone and together, in both signs
    t = 1 << (bd - 5)
    for lc in (5, 6):
        for mode in (0, 2, 18, 34, 9, 27):
            for dt, dl in ((t - 1, t - 1), (t, t - 1), (t - 1, t), (t, t), (-(t - 1), -(t - 1)), (-t, t - 1), (t - 1, -t), (0, 0)):
                for strong in (1, 0):
                    c = Case(rng, bd, LUMA, lc, 5, 0, 0, mode, 32, 32, 128, 128, [1, 1, 1, 1], strong=strong)
                    c.cx0, c.cy0 = (1 << lc), (1 << lc)
                    c.cw, c.ch = 3 << lc, 2 << lc
                    strong_ramp(c, dt, dl)
                    out.append(c)
    # the boundary filters of modes 10 and 26 clipping at both ends; DC edges
    for lg in (2, 3, 4):
        for mode in (10, 26, 1):
            for low in (True, False):
                c = Case(rng, bd, LUMA, 5, lg, 8 if lg < 4 else 16, 8 if lg < 4 else 16, mode, 32, 32, 96, 64, [1, 1, 1, 1], coded=(0, 0))
                edge_clip(c, low)
                out.append(c)
    # PCM and uncoded blocks of every kind and size
    for kind in (LUMA, PAIR, P422, P444):
        for lg in range(2, max_lg(kind) + 1):
            tw, th = comp_size(kind, 6)
            for pcm, coded in ((1, (1, 1)), (0, (0, 0)), (0, (1, 0)), (0, (0, 1))):
                k += 1
                out.append(Case(rng, bd, kind, 6, lg, 0, 0, k % 35, tw, th, 3 * tw, 2 * th, [1, 1, 1, 1], coded=coded, pcm=pcm))
    return out


def coverage(cases):
    cov = {"sub": Counter(), "filter": Counter(), "thres": Counter(), "mode": Counter(), "res": Counter()}
    for c in cases:
        expected(c, cov)
    return cov


WANT = {"sub": ["none", "first_bl", "first_l", "first_c", "first_t", "first_tr", "bl_partial", "tr_partial"],
        "filter": ["none", "121", "strong", "strong_top_fails_at_thr", "strong_left_fails_at_thr", "strong_at_thr_minus_1"],
        "thres": ["n8_eq", "n8_plus1", "n16_eq", "n16_plus1"],
        "mode": ["dc_edge", "m10_clip0", "m10_clipmax", "m26_clip0", "m26_clipmax", "neg_projection", "ifact0"],
        "res": ["clip0", "clipmax", "pcm", "uncoded"]}

_CASES = {}


def cached_cases(bd):
    if bd not in _CASES:
        cs = cases_for(bd)
        _CASES[bd] = (cs, coverage(cs))
    return _CASES[bd]


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_cases_reach_every_branch(bd):
    """the constructed cases of each bit depth reach every branch counter of the restatement, every mode at every size of
    every kind, every CTB-neighbour combination and every clamp of the above-right / below-left counts"""
    cases, cov = cached_cases(bd)
    for group, names in WANT.items():
        for nm in names:
            assert cov[group][nm] > 0, f"{bd} bits: {group}/{nm} never reached ({dict(cov[group])})"
    seen = {(c.kind, c.lg, c.mode) for c in cases}
    for kind in (LUMA, PAIR, P422, P444):
        for lg in range(2, max_lg(kind) + 1):
            assert all((kind, lg, m) in seen for m in range(35)), (kind, lg)
    assert {(c.kind, c.nb) for c in cases} >= {(kd, tuple((f >> b) & 1 for b in range(4))) for kd in range(4) for f in range(16)}
    clamps = Counter()
    for c in cases:
        avail, _ = expected(c)
        n = c.n
        trc, blc = int(avail[3 * n + 1:].sum()), int(avail[:n].sum())
        clamps[("tr", c.kind, n, trc)] += 1
        clamps[("bl", c.kind, n, blc)] += 1
    for kind in (LUMA, PAIR, P422, P444):
        stepx = 4 if SUB[kind][0] == 2 else 8
        stepy = 4 if SUB[kind][1] == 2 else 8
        for lg in range(2, max_lg(kind) + 1):
            n = 1 << lg
            for v in range(0, n, stepx):
                assert clamps[("tr", kind, n, v)] > 0, ("above-right", kind, n, v)
            for v in range(0, n, stepy):
                assert clamps[("bl", kind, n, v)] > 0, ("below-left", kind, n, v)


def k1_predict(cases):
    m = len(cases)
    prm = np.array([c.record() for c in cases], np.int32)
    tiles = np.zeros((m, 2, TILE), np.uint16)
    tops = np.zeros((m, 2, TOP), np.uint16)
    res = np.zeros((m, 2, RES), np.int16)
    for i, c in enumerate(cases):
        for comp in range(c.ncomp):
            t = c.tiles[comp].reshape(-1)
            tiles[i, comp, :t.size] = t
            tops[i, comp] = c.tops[comp]
            res[i, comp, :c.n * c.n] = c.res[comp].reshape(-1)
    desc = np.zeros(m, np.uint32)
    refs = np.zeros((m, 2, 2, REF), np.int16)
    tout = np.zeros((m, 2, TILE), np.uint16)
    _lib.check(_lib.lib().b200_debug_k1_predict(m, prm.ctypes.data, tiles.ctypes.data, tops.ctypes.data, res.ctypes.data, desc.ctypes.data,
                                                 refs.ctypes.data, tout.ctypes.data))
    return desc, refs, tout


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_k1_predict(cuda, bd):
    """K1's descriptor, neighbour array, filtered array and the whole tile after predict_tb == the restatement"""
    cases, _ = cached_cases(bd)
    desc, refs, tout = k1_predict(cases)
    for i, c in enumerate(cases):
        what = f"case {i}: kind {c.kind} ctb {1 << c.lc} n {c.n} at ({c.bx}, {c.by}) mode {c.mode} CTB ({c.cx0}, {c.cy0}) of {c.cw}x{c.ch} nb {c.nb} {c.content}"
        avail, comps = expected(c)
        d, n = int(desc[i]), c.n
        assert [d & 15, (d >> 4) & 15, (d >> 8) & 3, (d >> 10) & 63, (d >> 16) & 1, (d >> 17) & 1, (d >> 29) & 1] == \
            [c.bx >> 2, c.by >> 2, c.lg - 2, c.mode, int(c.coded[0]), int(c.coded[1]), c.pcm], what
        assert np.array_equal(desc_mask(d, n), avail), f"{what}: availability {desc_mask(d, n).astype(int).tolist()} != {avail.astype(int).tolist()}"
        for comp, (raw, r, f, blk) in enumerate(comps):
            assert refs[i, comp, 0, :4 * n + 1].tolist() == r, f"{what}: component {comp}: substituted neighbours"
            if c.kind != PAIR:
                got_f = refs[i, comp, 1, :4 * n + 1].tolist()
                assert got_f == (f if f is not None else [SENT] * (4 * n + 1)), f"{what}: filtered neighbours"
            want = c.tiles[comp].copy()
            want[c.by:c.by + n, PAD + c.bx:PAD + c.bx + n] = blk
            got = tout[i, comp, :want.size].reshape(want.shape).astype(np.int64)
            bad = np.argwhere(got != want)
            assert not len(bad), f"{what}: component {comp}: tile differs at (row, col - 16) {[(a, b - PAD) for a, b in bad[:6].tolist()]}"


def _one(**kw):
    """a legal 8x8 luma case, then the attributes of kw set as given"""
    c = Case(np.random.default_rng(0), 8, LUMA, 5, 3, 8, 8, 5, 32, 32, 96, 64, [1, 1, 1, 1])
    for a, v in kw.items():
        setattr(c, a, v)
    return c


@pytest.mark.parametrize("change", [dict(kind=4), dict(lc=3), dict(lc=7), dict(bd=7), dict(bd=13), dict(lg=1), dict(lg=6),
                                    dict(kind=PAIR, lg=5, bx=0, by=0, cx0=16, cy0=16, cw=48, ch=32), dict(bx=4), dict(bx=32), dict(by=-8),
                                    dict(mode=35), dict(mode=-1), dict(pcm=2), dict(strong=2), dict(coded=(1, 1)), dict(nb=(1, 1, 1, 2)),
                                    dict(cx0=0, nb=(1, 0, 0, 0)), dict(cy0=0, nb=(0, 0, 1, 0)), dict(cw=64, nb=(0, 0, 0, 1)),
                                    dict(cx0=16), dict(cw=38), dict(cw=40), dict(ch=0)])
def test_k1_predict_refusals(change):
    c = _one(**change)
    assert _refused([c])


def _refused(cases):
    m = len(cases)
    prm = np.array([c.record() for c in cases], np.int32)
    tiles = np.zeros((m, 2, TILE), np.uint16)
    for i, c in enumerate(cases):
        t = c.tiles[0].reshape(-1)
        tiles[i, 0, :t.size] = t
    tops = np.zeros((m, 2, TOP), np.uint16)
    res = np.zeros((m, 2, RES), np.int16)
    desc, refs, tout = np.zeros(m, np.uint32), np.zeros((m, 2, 2, REF), np.int16), np.zeros((m, 2, TILE), np.uint16)
    return _lib.lib().b200_debug_k1_predict(m, prm.ctypes.data, tiles.ctypes.data, tops.ctypes.data, res.ctypes.data, desc.ctypes.data,
                                            refs.ctypes.data, tout.ctypes.data) == E_INVALID


def test_k1_predict_refuses_samples_and_mixed_depths():
    c = _one()
    c.tiles[0, 3, 20] = 256
    assert _refused([c])
    assert _refused([_one(), _one(bd=10)])
    c = _one(pcm=1)
    c.res[0, 1, 1] = -1
    m = 1
    prm = np.array([c.record()], np.int32)
    res = np.zeros((m, 2, RES), np.int16)
    res[0, 0, :64] = c.res[0].reshape(-1)
    z = np.zeros((m, 2, TILE), np.uint16)
    assert _lib.lib().b200_debug_k1_predict(1, prm.ctypes.data, z.ctypes.data, np.zeros((m, 2, TOP), np.uint16).ctypes.data, res.ctypes.data,
                                            np.zeros(1, np.uint32).ctypes.data, np.zeros((1, 2, 2, REF), np.int16).ctypes.data, z.ctypes.data) == E_INVALID
    assert _lib.lib().b200_debug_k1_predict(0, prm.ctypes.data, None, None, None, None, None, None) == E_INVALID


# ------------------------------------------------------------------------------------------ descriptors of real streams (CPU)
def k1_descriptors(au):
    l = _lib.lib()
    hdr = np.zeros(6, np.int32)
    _lib.check(l.b200_debug_k1_descriptors(au, len(au), hdr.ctypes.data, None, 0, None, 0))
    w, h, lg, chroma, ng, nd = hdr.tolist()
    nctb = (-(-w >> lg)) * (-(-h >> lg))
    desc = np.zeros(max(nd, 1), np.uint32)
    counts = np.zeros(nctb * ng, np.int32)
    _lib.check(l.b200_debug_k1_descriptors(au, len(au), hdr.ctypes.data, desc.ctypes.data, nd, counts.ctypes.data, nctb * ng))
    return (w, h, lg, chroma, ng), desc[:nd], counts.reshape(nctb, ng)


def stream_ctx(au):
    """PicCtx of a stream from b200_debug_parse_filters: SliceAddrRs from each CTB's slice, TileId and the tile grid from the
    TileId map (never the region index itself); and the luma / chroma modes per 4x4 of b200_debug_parse"""
    l = _lib.lib()
    hdr = np.zeros(13, np.int32)
    _lib.check(l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, None, 0, None, 0))
    w, h, lg, bd, chroma = hdr[:5].tolist()
    ns = int(hdr[8])
    wctb, hctb = -(-w >> lg), -(-h >> lg)
    ctbs = np.zeros((wctb * hctb, 19), np.int32)
    regs = np.zeros((ns, 6), np.int32)
    _lib.check(l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, ctbs.ctypes.data, wctb * hctb, regs.ctypes.data, ns))
    slice_id = regs[ctbs[:, 0], 3].astype(np.int64)
    tile_id = regs[ctbs[:, 0], 4].astype(np.int64)
    cols, rows = tile_boundaries_from_ids(tile_id.reshape(hctb, wctb))
    ctx = PicCtx(w, h, lg, slice_id, tile_id, cols, rows)
    assert np.array_equal(ctx.tile_id, tile_id)
    qp8 = np.zeros((h >> 3) * (w >> 3), np.int8)
    edge8 = np.zeros_like(qp8, np.uint8)
    lm4, cm4 = np.zeros((h >> 2) * (w >> 2), np.uint8), np.zeros((h >> 2) * (w >> 2), np.uint8)
    out5 = np.zeros(5, np.uint64)
    _lib.check(l.b200_debug_parse(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm4.ctypes.data, cm4.ctypes.data, out5.ctypes.data))
    return ctx, bd, lm4.reshape(h >> 2, w >> 2), cm4.reshape(h >> 2, w >> 2)


def group_sub(chroma, gi):
    """(SubWidthC, SubHeightC, cIdx) of component group gi as K1 orders them"""
    if gi == 0:
        return 1, 1, 0
    if chroma == 1:
        return 2, 2, 1
    return (2 if chroma == 2 else 1), 1, gi


def check_stream_descriptors(name, au, reach):
    """every descriptor of the stream against 6.4.1 / 8.4.4.2.2; the blocks of each component tile their plane once, in z-order"""
    (w, h, lg, chroma, ng), desc, counts = k1_descriptors(au)
    ctx, bd, lm4, cm4 = stream_ctx(au)
    wctb = ctx.wctb
    ctb = 1 << lg
    starts = np.concatenate([[0], np.cumsum(counts.reshape(-1))])
    recs = {gi: [] for gi in range(ng)}
    for a in range(counts.shape[0]):
        rx, ry = a % wctb, a // wctb
        for gi in range(ng):
            sw, sh, cidx = group_sub(chroma, gi)
            d = desc[starts[a * ng + gi]:starts[a * ng + gi + 1]].astype(np.int64)
            bx, by, n = (d & 15) * 4, ((d >> 4) & 15) * 4, 1 << (((d >> 8) & 3) + 2)
            cx0, cy0 = (rx * ctb) // sw, (ry * ctb) // sh
            # tiling, in z-order of the luma locations
            cov = np.zeros((ctb // sh, ctb // sw), np.int64)
            for x, y, nn in zip(bx.tolist(), by.tolist(), n.tolist()):
                cov[y:y + nn, x:x + nn] += 1
            cw, ch = min(ctb // sw, w // sw - cx0), min(ctb // sh, h // sh - cy0)
            assert (cov[:ch, :cw] == 1).all() and (cov[ch:, :] == 0).all() and (cov[:, cw:] == 0).all(), f"{name}: CTB {a} group {gi}: blocks do not tile the plane"
            zs = ctx.zs[((cy0 + by) * sh) >> 2, ((cx0 + bx) * sw) >> 2]
            assert (np.diff(zs) > 0).all(), f"{name}: CTB {a} group {gi}: blocks out of z-order"
            recs[gi].append(np.stack([d, cx0 + bx, cy0 + by, n], 1))
    for gi in range(ng):
        sw, sh, cidx = group_sub(chroma, gi)
        allr = np.concatenate(recs[gi])
        modes = (allr[:, 0] >> 10) & 63
        want_mode = (lm4 if gi == 0 else cm4)[(allr[:, 2] * sh) >> 2, (allr[:, 1] * sw) >> 2]
        assert np.array_equal(modes, want_mode), f"{name}: group {gi}: modes differ from b200_debug_parse"
        for n in (4, 8, 16, 32):
            sel = allr[allr[:, 3] == n]
            if not len(sel):
                continue
            want = mark_neighbours(ctx, sw, sh, sel[:, 1], sel[:, 2], n)
            got = np.stack([desc_mask(int(d), n) for d in sel[:, 0]])
            bad = np.argwhere((got != want).any(1))
            assert not len(bad), f"{name}: group {gi}: n {n}: block at {sel[bad[0][0], 1:3].tolist()}: {got[bad[0][0]].astype(int).tolist()} != {want[bad[0][0]].astype(int).tolist()}"
            reach_counts(reach, ctx, sw, sh, sel, n, want, chroma, gi)


def reach_counts(reach, ctx, sw, sh, sel, n, avail, chroma, gi):
    """what the stream set reaches: neighbours across tile boundaries inside one slice, across slice-segment boundaries inside one
    slice, clamped counts, and 4:2:2 lower blocks"""
    ox, oy = neighbour_offsets(n)
    xc, yc = sel[:, 1:2] * sw, sel[:, 2:3] * sh
    xn, yn = (sel[:, 1:2] + ox[None]) * sw, (sel[:, 2:3] + oy[None]) * sh
    inside = (xn >= 0) & (yn >= 0) & (xn < ctx.w) & (yn < ctx.h)
    cn = np.where(inside, (np.clip(yn, 0, ctx.h - 1) >> ctx.lg) * ctx.wctb + (np.clip(xn, 0, ctx.w - 1) >> ctx.lg), 0)
    cc = (yc >> ctx.lg) * ctx.wctb + (xc >> ctx.lg)
    cross_tile = inside & (ctx.tile_id[cn] != ctx.tile_id[cc]) & (ctx.slice_addr[cn] == ctx.slice_addr[cc])
    reach["tile_boundary_same_slice"] += int(cross_tile.any(1).sum())
    d = sel[:, 0]
    blc, trc = ((d >> 21) & 15) * 4, ((d >> 25) & 15) * 4
    reach["trc_clamped"] += int(((trc > 0) & (trc < n)).sum())
    reach["blc_clamped"] += int(((blc > 0) & (blc < n)).sum())
    if chroma == 2 and gi > 0:
        lower = (sel[:, 2] // n) % 2 == 1
        for j in np.flatnonzero(lower):
            key = "".join(str(int(avail[j, i])) for i in (0, n, 2 * n, 2 * n + 1, 3 * n + 1))
            reach["422_lower_" + key] += 1


STREAM_NAMES = [s[0] for s in SYNTH + SYNTH_CPU_EXTRA]


def _all_streams():
    out = [(nm, synth_stream(nm)) for nm in STREAM_NAMES] + fixture_streams()
    return out


def test_stream_descriptors():
    """K1's phase-A descriptors of every stream of hevc_cases and every fixture == 6.4.1 / 8.4.4.2.2 on the stream's own
    slices and tiles; the stream set reaches tile boundaries inside a slice, dependent slice segments, clamped counts and
    4:2:2 lower blocks with each neighbour outcome"""
    reach = Counter()
    for name, au in _all_streams():
        check_stream_descriptors(name, au, reach)
    assert reach["tile_boundary_same_slice"] > 0
    assert reach["trc_clamped"] > 0 and reach["blc_clamped"] > 0
    lower = {k: v for k, v in reach.items() if k.startswith("422_lower_")}
    # below-left, left and corner of a lower block both available and not; its top (the upper block) always available, its
    # above-right (the next unit, or outside the picture) never
    outcomes = [{k[-5:][pos] for k in lower} for pos in range(5)]
    assert outcomes == [{"0", "1"}, {"0", "1"}, {"0", "1"}, {"1"}, {"0"}], lower


def _vcl_nal_units(au):
    """number of slice segment NAL units (nal_unit_type < 32) of an access unit of 4-byte length-prefixed NAL units"""
    n, i = 0, 0
    while i + 4 < len(au):
        size = int.from_bytes(au[i:i + 4], "big")
        n += ((au[i + 4] >> 1) & 63) < 32
        i += 4 + size
    return n


def test_dependent_slice_segments_stay_available():
    """dependent slice segments belong to the slice of the segment before them (6.4.1 compares SliceAddrRs): the top row of
    every CTB row that continues a slice sees the row above, the first row of a new slice does not"""
    au = synth_stream("dependent_slices")
    ctx, *_ = stream_ctx(au)
    nslices = len(set(ctx.slice_addr.tolist()))
    assert _vcl_nal_units(au) > nslices > 1, "the stream has no dependent slice segment"
    (w, h, lg, chroma, ng), desc, counts = k1_descriptors(au)
    wctb = ctx.wctb
    top_avail = Counter()
    starts = np.concatenate([[0], np.cumsum(counts.reshape(-1))])
    for a in range(counts.shape[0]):
        d = desc[starts[a * ng]:starts[a * ng + 1]].astype(np.int64)
        top_avail[a // wctb] += int(((d >> 20) & 1)[((d >> 4) & 15) == 0].sum())
    for ry in range(1, ctx.hctb):
        same = ctx.slice_addr[ry * wctb] == ctx.slice_addr[(ry - 1) * wctb]
        assert (top_avail[ry] > 0) == same, (ry, same, top_avail)
    assert sum(ctx.slice_addr[ry * wctb] == ctx.slice_addr[(ry - 1) * wctb] for ry in range(1, ctx.hctb)) >= nslices


# ------------------------------------------------------------------------------------------ intra-edge streams
def smooth_image(seed, w, h, bd, chroma):
    """A picture whose left half is made of gentle linear ramps (strong smoothing fires on its 32x32 blocks) and whose right
    half is the encoder's synthetic texture (it does not), with chroma of the same kind"""
    from libheif_b200 import hevc_enc
    rng = np.random.default_rng(seed)
    planes = list(hevc_enc.synthetic_image(seed, w, h, bd, chroma))
    maxv = (1 << bd) - 1
    for c, p in enumerate(planes):
        if p is None:
            continue
        ph, pw = p.shape
        yy, xx = np.mgrid[0:ph, 0:pw]
        gx, gy = rng.uniform(-0.5, 0.5, 2) * (maxv / 255.0)
        ramp = np.clip(maxv // 2 + gx * xx + gy * yy, 0, maxv)
        half = pw // 2
        p[:, :half] = ramp[:, :half].astype(p.dtype)
        planes[c] = np.ascontiguousarray(p)
    return planes


# (name, width, height, bit depth, chroma_format_idc, smooth content, encoder options): random modes and deep transform trees,
# picture sizes that cut CTBs, CTB 16 / 32 / 64, tiles together with slices, strong intra smoothing on and off
EDGE_STREAMS = [
    ("e_420_8_ctb64_tiles_slices", 200, 136, 8, 1, False, dict(log2_ctb_size=6, mode_decision=0, max_transform_hierarchy_depth_intra=3,
                                                              tile_cols=2, tile_rows=2, slice_per_tile=1)),
    ("e_422_10_ctb16_tiles", 136, 72, 10, 2, False, dict(log2_ctb_size=4, mode_decision=0, max_transform_hierarchy_depth_intra=2,
                                                        tile_cols=3, tile_rows=2, strong_intra_smoothing=0)),
    ("e_444_12_ctb32_slices", 168, 104, 12, 3, False, dict(log2_ctb_size=5, mode_decision=0, max_transform_hierarchy_depth_intra=3,
                                                          slice_ctb_rows=1)),
    ("e_420_12_ctb16_nostrong", 120, 88, 12, 1, False, dict(log2_ctb_size=4, mode_decision=0, max_transform_hierarchy_depth_intra=1,
                                                           strong_intra_smoothing=0, tile_cols=2, tile_rows=2, slice_per_tile=1)),
    ("e_420_8_ctb64_smooth", 256, 128, 8, 1, True, dict(log2_ctb_size=6, qp=32)),
    ("e_420_10_ctb64_smooth_tiles", 256, 128, 10, 1, True, dict(log2_ctb_size=6, qp=32, tile_cols=2, tile_rows=1)),
    ("e_444_10_ctb32_smooth_random", 192, 96, 10, 3, True, dict(log2_ctb_size=5, qp=30, mode_decision=0)),
]
_EDGE = {}


def edge_stream(name):
    if name not in _EDGE:
        from libheif_b200 import hevc_enc
        (_, w, h, bd, chroma, smooth, opts) = next(s for s in EDGE_STREAMS if s[0] == name)
        seed = 0x1E + w + h + bd
        y, cb, cr = smooth_image(seed, w, h, bd, chroma) if smooth else hevc_enc.synthetic_image(seed, w, h, bd, chroma)
        _EDGE[name] = hevc_enc.encode_intra(y, cb, cr, bit_depth=bd, seed=seed, **opts)
    return _EDGE[name]


EDGE_NAMES = [s[0] for s in EDGE_STREAMS]


def strong_outcomes(au):
    """For every 32x32 luma block whose neighbours are filtered: whether 8.4.4.2.3's strong-smoothing condition holds, evaluated
    on the C restatement's picture before deblocking with the availability of K1's descriptors"""
    from oracle import bindings as ob
    (w, h, lg, chroma, ng), desc, counts = k1_descriptors(au)
    ctx, bd, lm4, cm4 = stream_ctx(au)
    luma = ob.restatement_decode(au, 1)[0][0].astype(np.int64)
    starts = np.concatenate([[0], np.cumsum(counts.reshape(-1))])
    out = Counter()
    ctb = 1 << lg
    ox, oy = neighbour_offsets(32)
    for a in range(counts.shape[0]):
        x0, y0 = (a % ctx.wctb) * ctb, (a // ctx.wctb) * ctb
        for d in desc[starts[a * ng]:starts[a * ng + 1]].tolist():
            mode = (d >> 10) & 63
            if ((d >> 8) & 3) != 3 or not filter_flag(True, mode, 32):
                continue
            bx, by = x0 + (d & 15) * 4, y0 + ((d >> 4) & 15) * 4
            m = desc_mask(d, 32)
            raw = [int(luma[by + oy[i], bx + ox[i]]) if m[i] else -1 for i in range(129)]
            r = substitute(raw, 32, bd)
            thr = 1 << (bd - 5)
            out[abs(r[64] + r[128] - 2 * r[96]) < thr and abs(r[64] + r[0] - 2 * r[32]) < thr] += 1
    return bd, out


def test_edge_streams_reach_both_strong_smoothing_outcomes():
    """real 32x32 luma blocks take both outcomes of the strong-smoothing condition, at 8 bits and at a higher bit depth; the
    descriptors of the intra-edge streams pass the same checks as those of hevc_cases"""
    seen = {}
    reach = Counter()
    for name in EDGE_NAMES:
        au = edge_stream(name)
        check_stream_descriptors(name, au, reach)
        params = next(s for s in EDGE_STREAMS if s[0] == name)[6]
        if params.get("strong_intra_smoothing", 1):
            bd, out = strong_outcomes(au)
            seen.setdefault(bd > 8, Counter()).update(out)
    for deep in (False, True):
        assert seen[deep][True] > 0 and seen[deep][False] > 0, (deep, seen)
    assert reach["tile_boundary_same_slice"] > 0 and reach["trc_clamped"] > 0


@pytest.mark.gpu
def test_edge_streams_on_the_gpu(cuda):
    """the decoder's picture before deblocking, with either front-end, == the C restatement's, for every intra-edge stream"""
    import libheif_b200 as lb
    from oracle import bindings as ob
    dec = lb.Decoder(host_threads=4)
    try:
        dec.set_debug_stage(1)
        for name in EDGE_NAMES:
            au = edge_stream(name)
            want, info = ob.restatement_decode(au, 1)
            w, h = want[0].shape[1], want[0].shape[0]
            for device in (True, False):
                dec.set_front_end(device)
                dec.decode_image(au)
                got = dec.debug_tile(0, w, h)
                for c in range(3 if info["chroma"] else 1):
                    bad = np.argwhere(got[c].astype(np.int64) != want[c].astype(np.int64))
                    assert not len(bad), f"{name}: {'device' if device else 'host'} front-end, plane {c}: first diffs {bad[:4].tolist()}"
    finally:
        dec.set_debug_stage(0)
        dec.close()
