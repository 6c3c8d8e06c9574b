"""In-loop filters, stage by stage: the decoder's deblocking (K3, deblock_kernel) and SAO with the conformance crop and the
paste into the destination (K4, sao_rows_kernel) against a plain int64 numpy restatement of H.265 8.7.2 and 8.7.3, exactly.

The restatement is written from the text of the standard (8.7.2.5.3 - 8.7.2.5.8, 8.7.3, Tables 8-10 and 8-12) and counts
which branch every edge segment and every sample takes, so that the tests can assert what they reached:
- constructed edges put each deblocking decision at its threshold and one below it, at 8, 10 and 12 bits, over the whole
  tC' / beta' tables, with keep bits (bypass / PCM) on either side and two regions with different offsets;
- constructed pictures reach every SAO band slot and edgeIdx, both saturation ends, partial units, warps that load their
  own outer neighbours, slice and tile boundaries, conformance windows on all four sides and misaligned destinations;
- every stream of hevc_cases is chained through the restatement: stage 1 -> deblocking -> stage 2 -> SAO -> stage 0, on the
  C restatement's stages here and on the decoder's own stages on the GPU, with the conformance window removed so that the
  filters' reads near the right and bottom edges are compared too;
- conformance windows with left and top offsets, written into real streams by an SPS rewriter, decode to the window of the
  window-free decode."""
import os
from collections import Counter, defaultdict

import numpy as np
import pytest

import libheif_b200 as lb
from libheif_b200 import _lib
from libheif_b200 import hevc_enc
from hevc_cases import SYNTH, SYNTH_CPU_EXTRA, fixture_streams, synth_stream

E_INVALID, E_UNSUPPORTED, E_BITSTREAM = -1, -2, -3
SENTINEL = 0xA5

# ------------------------------------------------------------------------------------------ tables typed from H.265
# Table 8-12: tC' for Q = 0 .. 53 and beta' for Q = 0 .. 51
TC_PRIME = [0] * 18 + [1] * 9 + [2] * 4 + [3] * 4 + [4] * 3 + [5, 5, 6, 6, 7, 8, 9, 10, 11, 13, 14, 16, 18, 20, 22, 24]
BETA_PRIME = [0] * 16 + list(range(6, 19)) + list(range(20, 65, 2))
# Table 8-10: QpC as a function of qPi for ChromaArrayType == 1 (qPi < 30: QpC = qPi; qPi > 43: QpC = qPi - 6)
QPC_TABLE = {30: 29, 31: 30, 32: 31, 33: 32, 34: 33, 35: 33, 36: 34, 37: 34, 38: 35, 39: 35, 40: 36, 41: 36, 42: 37, 43: 37}
assert len(TC_PRIME) == 54 and len(BETA_PRIME) == 52 and BETA_PRIME[28] == 18 and BETA_PRIME[29] == 20 and BETA_PRIME[51] == 64


def sub_wh(chroma):
    """SubWidthC, SubHeightC (Table 6-1) as shifts"""
    return (1 if chroma in (1, 2) else 0), (1 if chroma == 1 else 0)


def qpc_of(qpi, chroma):
    if chroma != 1:
        return min(qpi, 51)
    if qpi < 30:
        return qpi
    return QPC_TABLE[qpi] if qpi <= 43 else qpi - 6


class Cov:
    """Branch counters of the restatement: cov[name][value] = how often"""

    def __init__(self):
        self.c = defaultdict(Counter)

    def add(self, name, values):
        v, n = np.unique(np.asarray(values).reshape(-1), return_counts=True)
        for a, b in zip(v.tolist(), n.tolist()):
            self.c[name][a] += b

    def margins(self, name, value, thr):
        """value - threshold, clipped to [-3, 3]: -1 and 0 are the tight cases of a `value < thr` decision"""
        self.add(name, np.clip(np.asarray(value) - np.asarray(thr), -3, 3))

    def __getitem__(self, k):
        return self.c[k]


# ------------------------------------------------------------------------------------------ picture description
class Pic:
    """One picture as K3 / K4 see it: coded planes, the 8x8 maps, per-CTB region and SAO parameters, the region table, the
    conformance window and the destination it is pasted into."""

    def __init__(self, w, h, lg, bd, chroma, planes=None, qp8=None, edge8=None, ctb_region=None, sao=None, regions=None,
                 cb_off=0, cr_off=0, sao_enabled=1, window=None, dst=None):
        self.w, self.h, self.lg, self.bd, self.chroma = w, h, lg, bd, chroma
        self.sx, self.sy = sub_wh(chroma)
        self.w8, self.h8 = w >> 3, h >> 3
        self.wctb, self.hctb = -(-w >> lg), -(-h >> lg)
        self.planes = planes
        self.qp8 = qp8 if qp8 is not None else np.full((self.h8, self.w8), 30, np.int64)
        self.edge8 = edge8 if edge8 is not None else np.zeros((self.h8, self.w8), np.int64)
        self.ctb_region = ctb_region if ctb_region is not None else np.zeros((self.hctb, self.wctb), np.int64)
        self.sao = sao if sao is not None else np.zeros((self.hctb, self.wctb, 3, 6), np.int64)   # type, band / class, 4 offsets
        self.regions = regions if regions is not None else [dict(beta=0, tc=0, across_slices=1, slice_id=0, tile_id=0, across_tiles=1)]
        self.cb_off, self.cr_off, self.sao_enabled = cb_off, cr_off, sao_enabled
        self.window = window if window is not None else (0, 0, w, h)      # crop_x, crop_y, out_w, out_h (luma samples)
        cx, cy, ow, oh = self.window
        # destination: (width, height, luma pitch, chroma pitch, paste x, paste y)
        self.dst = dst if dst is not None else (ow, oh, ow, (ow + self.sx) >> self.sx, 0, 0)

    @property
    def ncomp(self):
        return 3 if self.chroma else 1

    @property
    def maxv(self):
        return (1 << self.bd) - 1

    def comp_size(self, c):
        return (self.w >> self.sx, self.h >> self.sy) if c else (self.w, self.h)

    def dst_shapes(self):
        dw, dh, dp, dcp, px, py = self.dst
        out = [(dh, dp)]
        if self.chroma:
            out += [((dh + self.sy) >> self.sy, dcp)] * 2
        return out


# ------------------------------------------------------------------------------------------ restatement: deblocking (8.7.2)
def _tables():
    return np.array(TC_PRIME, np.int64), np.array(BETA_PRIME, np.int64)


def _deblock_dir(pic, planes, vertical, cov):
    """One direction of 8.7.2 over the whole picture: every edge of that direction at once (edges of one direction are 8
    samples apart and touch at most 4 samples on each side, so they are independent).  `planes` are modified in place."""
    tc_t, beta_t = _tables()
    bd, maxv = pic.bd, pic.maxv
    # work on the transpose for horizontal edges: the edge is then vertical, its segments run down the rows
    e8 = pic.edge8 if vertical else pic.edge8.T
    qp8 = pic.qp8 if vertical else pic.qp8.T
    creg = pic.ctb_region if vertical else pic.ctb_region.T
    bit = 1 if vertical else 2
    beta_off = np.array([r["beta"] for r in pic.regions], np.int64)
    tc_off = np.array([r["tc"] for r in pic.regions], np.int64)
    by, bx = np.nonzero(e8 & bit)                        # 8x8 cells (in the oriented picture) whose left edge is filtered
    keep = bx > 0
    by, bx = by[keep], bx[keep]
    qpq, qpp = qp8[by, bx], qp8[by, bx - 1]
    kq, kp = (e8[by, bx] & 4) != 0, (e8[by, bx - 1] & 4) != 0   # pcm + pcm_loop_filter_disabled_flag / cu_transquant_bypass_flag
    qpl = (qpq + qpp + 1) >> 1                           # QpL (8-275)
    cov.add("qp_odd_sum", (qpq + qpp) & 1)
    cov.add("qpl_sign", np.sign(qpl))
    cov.add("keep", kp * 1 + kq * 2)
    # ---- luma: two 4-line segments per 8x8 cell edge
    P = planes[0] if vertical else planes[0].T
    seg_y = np.concatenate([by * 8, by * 8 + 4])
    seg_x = np.concatenate([bx * 8, bx * 8])
    sq = np.concatenate([qpl, qpl])
    skp, skq = np.concatenate([kp, kp]), np.concatenate([kq, kq])
    reg = creg[seg_y >> pic.lg, seg_x >> pic.lg]          # the region (slice) that contains q0,0
    Qb = np.clip(sq + beta_off[reg], 0, 51)
    Qt = np.clip(sq + 2 * (2 - 1) + tc_off[reg], 0, 53)   # bS = 2
    beta = beta_t[Qb] * (1 << (bd - 8))
    tc = tc_t[Qt] * (1 << (bd - 8))
    cov.add(f"Qbeta", Qb)
    cov.add(f"Qtc", Qt)
    cov.add("Qbeta_raw_clamp", np.sign(sq + beta_off[reg] - np.clip(sq + beta_off[reg], 0, 51)))
    cov.add("Qtc_raw_clamp", np.sign(sq + 2 + tc_off[reg] - np.clip(sq + 2 + tc_off[reg], 0, 53)))
    rows = seg_y[:, None] + np.arange(4)[None, :]                       # [seg, line]
    cols = seg_x[:, None] + np.arange(-4, 4)[None, :]                   # [seg, k]: p3 p2 p1 p0 q0 q1 q2 q3
    S = P[rows[:, :, None], cols[:, None, :]].astype(np.int64)          # [seg, line, 8]
    p = [S[:, :, 3 - i] for i in range(4)]
    q = [S[:, :, 4 + i] for i in range(4)]
    dpl = np.abs(p[2] - 2 * p[1] + p[0])
    dql = np.abs(q[2] - 2 * q[1] + q[0])
    dpq0, dpq3 = dpl[:, 0] + dql[:, 0], dpl[:, 3] + dql[:, 3]
    dp, dq = dpl[:, 0] + dpl[:, 3], dql[:, 0] + dql[:, 3]
    d = dpq0 + dpq3
    on = d < beta                                                        # 8.7.2.5.3
    cov.margins("d_vs_beta", d, beta)

    def dsam(l, dpq):                                                    # 8.7.2.5.6
        c1 = 2 * dpq < (beta >> 2)
        c2 = np.abs(p[3][:, l] - p[0][:, l]) + np.abs(q[0][:, l] - q[3][:, l]) < (beta >> 3)
        c3 = np.abs(p[0][:, l] - q[0][:, l]) < ((5 * tc + 1) >> 1)
        cov.margins(f"strong1_l{l}", 2 * dpq[on], (beta >> 2)[on])
        cov.margins(f"strong2_l{l}", (np.abs(p[3][:, l] - p[0][:, l]) + np.abs(q[0][:, l] - q[3][:, l]))[on], (beta >> 3)[on])
        cov.margins(f"strong3_l{l}", np.abs(p[0][:, l] - q[0][:, l])[on], ((5 * tc + 1) >> 1)[on])
        return c1 & c2 & c3

    strong = on & dsam(0, dpq0) & dsam(3, dpq3)                           # dE = 2
    side = (beta + (beta >> 1)) >> 3
    dEp, dEq = dp < side, dq < side
    normal = on & ~strong
    cov.margins("dEp", dp[normal], side[normal])
    cov.margins("dEq", dq[normal], side[normal])
    cov.add("decision", np.where(~on, 0, np.where(strong, 2, 1)))
    out = S.copy()
    t2 = (2 * tc)[:, None]
    # strong filter (8.7.2.5.7, nDp = nDq = 3)
    sp = [np.clip((p[2] + 2 * p[1] + 2 * p[0] + 2 * q[0] + q[1] + 4) >> 3, p[0] - t2, p[0] + t2),
          np.clip((p[2] + p[1] + p[0] + q[0] + 2) >> 2, p[1] - t2, p[1] + t2),
          np.clip((2 * p[3] + 3 * p[2] + p[1] + p[0] + q[0] + 4) >> 3, p[2] - t2, p[2] + t2)]
    sq_ = [np.clip((p[1] + 2 * p[0] + 2 * q[0] + 2 * q[1] + q[2] + 4) >> 3, q[0] - t2, q[0] + t2),
           np.clip((p[0] + q[0] + q[1] + q[2] + 2) >> 2, q[1] - t2, q[1] + t2),
           np.clip((p[0] + q[0] + q[1] + 3 * q[2] + 2 * q[3] + 4) >> 3, q[2] - t2, q[2] + t2)]
    # normal filter
    tcb = tc[:, None]
    delta = (9 * (q[0] - p[0]) - 3 * (q[1] - p[1]) + 8) >> 4
    act = np.abs(delta) < tcb * 10
    cov.margins("delta_vs_10tc", np.abs(delta)[normal], (tcb * 10 * np.ones_like(delta))[normal])
    dl = np.clip(delta, -tcb, tcb)
    cov.add("delta_clipped", np.sign(delta - dl)[normal[:, None] & act])
    np0, nq0 = p[0] + dl, q[0] - dl
    hp = tcb >> 1
    dpp = np.clip((((p[2] + p[0] + 1) >> 1) - p[1] + dl) >> 1, -hp, hp)
    dqq = np.clip((((q[2] + q[0] + 1) >> 1) - q[1] - dl) >> 1, -hp, hp)
    np1, nq1 = p[1] + dpp, q[1] + dqq
    m_n = (normal[:, None] & act)
    for name, v in (("clip_p0", np0), ("clip_q0", nq0), ("clip_p1", np1), ("clip_q1", nq1)):
        cov.add(name + f"_bd{bd}", np.where(v < 0, -1, np.where(v > maxv, 1, 0))[m_n])
    np0, nq0, np1, nq1 = [np.clip(v, 0, maxv) for v in (np0, nq0, np1, nq1)]
    wp, wq = ~skp[:, None], ~skq[:, None]
    st_ = strong[:, None]
    for i in range(3):
        out[:, :, 3 - i] = np.where(st_ & wp, sp[i], out[:, :, 3 - i])
        out[:, :, 4 + i] = np.where(st_ & wq, sq_[i], out[:, :, 4 + i])
    out[:, :, 3] = np.where(m_n & wp, np0, out[:, :, 3])
    out[:, :, 4] = np.where(m_n & wq, nq0, out[:, :, 4])
    out[:, :, 2] = np.where(m_n & wp & dEp[:, None], np1, out[:, :, 2])
    out[:, :, 5] = np.where(m_n & wq & dEq[:, None], nq1, out[:, :, 5])
    cov.add("keep_active", (skp * 1 + skq * 2)[on])
    P[rows[:, :, None], cols[:, None, :]] = out
    # ---- chroma (8.7.2.5.5): edges on the chroma 8-sample grid, bS = 2
    if pic.chroma:
        ex, ey = (pic.sx, pic.sy) if vertical else (pic.sy, pic.sx)      # sub-sampling across / along the oriented edge
        sel = (bx * 8) % (8 << ex) == 0
        cby, cbx = by[sel], bx[sel]
        cq = qpl[sel]
        ckp, ckq = kp[sel], kq[sel]
        for c, off in ((1, pic.cb_off), (2, pic.cr_off)):
            Pc = planes[c] if vertical else planes[c].T
            qpi = cq + off                                               # cQpPicOffset = pps_cb_qp_offset / pps_cr_qp_offset
            qpc = np.array([qpc_of(int(v), pic.chroma) for v in qpi], np.int64)
            if pic.chroma == 1:
                cov.add("qpi_range", np.where(qpi < 30, 0, np.where(qpi <= 42, 1, 2)))
            # two luma segments per 8x8 cell -> 8 >> ey chroma lines per cell edge
            yc0 = (cby * 8) >> ey
            xc = (cbx * 8) >> ex
            n = 8 >> ey
            regc = creg[(cby * 8) >> pic.lg, (cbx * 8) >> pic.lg]
            Qc = np.clip(qpc + 2 + tc_off[regc], 0, 53)
            cov.add("Qtc_chroma", Qc)
            tcc = (tc_t[Qc] * (1 << (bd - 8)))[:, None]
            rr = yc0[:, None] + np.arange(n)[None, :]
            p0 = Pc[rr, (xc - 1)[:, None]].astype(np.int64)
            p1 = Pc[rr, (xc - 2)[:, None]].astype(np.int64)
            q0 = Pc[rr, xc[:, None]].astype(np.int64)
            q1 = Pc[rr, (xc + 1)[:, None]].astype(np.int64)
            dlt = np.clip((((q0 - p0) << 2) + p1 - q1 + 4) >> 3, -tcc, tcc)
            a, b = p0 + dlt, q0 - dlt
            cov.add(f"clip_chroma_bd{bd}", np.where((a < 0) | (b < 0), -1, np.where((a > maxv) | (b > maxv), 1, 0)))
            Pc[rr, (xc - 1)[:, None]] = np.where(ckp[:, None], p0, np.clip(a, 0, maxv))
            Pc[rr, xc[:, None]] = np.where(ckq[:, None], q0, np.clip(b, 0, maxv))
            cov.add("chroma_edges_fmt", np.full(len(cby), pic.chroma))


def deblock(pic, planes, cov):
    """8.7.2: all vertical edges of the picture, then all horizontal edges, on int64 copies of `planes`"""
    out = [np.array(a, np.int64) for a in planes]
    _deblock_dir(pic, out, True, cov)
    _deblock_dir(pic, out, False, cov)
    return out


# ------------------------------------------------------------------------------------------ restatement: SAO (8.7.3) + crop / paste
H_POS = [(-1, 1), (0, 0), (-1, 1), (1, -1)]        # hPos / vPos of the four SaoEoClass values (Table 8-13)
V_POS = [(0, 0), (-1, 1), (-1, 1), (-1, 1)]


def sao(pic, planes, cov):
    """8.7.3 on the deblocked planes; returns the SAO output planes (int64, coded size)"""
    out = []
    sid = np.array([r["slice_id"] for r in pic.regions], np.int64)
    tid = np.array([r["tile_id"] for r in pic.regions], np.int64)
    across = np.array([r["across_slices"] for r in pic.regions], np.int64)
    tiles_across = pic.regions[0]["across_tiles"]       # loop_filter_across_tiles_enabled_flag is a PPS flag: one value per picture
    for c in range(pic.ncomp):
        rec = np.array(planes[c], np.int64)
        h, w = rec.shape
        sx, sy = (pic.sx, pic.sy) if c else (0, 0)
        ctw, cth = (1 << pic.lg) >> sx, (1 << pic.lg) >> sy
        yy, xx = np.mgrid[0:h, 0:w]
        ry, rx = yy // cth, xx // ctw
        prm = pic.sao[ry, rx, c]                         # [h, w, 6]
        typ = prm[..., 0] * (1 if pic.sao_enabled else 0)
        # SaoTypeIdx is treated as 0 for samples of bypass / pcm-without-loop-filter coding units (8.7.3)
        keep = (pic.edge8[(yy << sy) >> 3, (xx << sx) >> 3] & 4) != 0
        typ = np.where(keep, 0, typ)
        reg = pic.ctb_region[ry, rx]
        offval = np.concatenate([np.zeros((h, w, 1), np.int64), prm[..., 2:6]], axis=2)   # SaoOffsetVal[0..4]
        bd = pic.bd
        idx = np.zeros((h, w), np.int64)
        # band offset: bandTable[(k + sao_band_position) & 31] = k + 1, bandIdx = bandTable[sample >> bandShift]
        bshift = bd - 5
        band = rec >> bshift
        bidx = np.zeros((h, w), np.int64)
        for k in range(4):
            bidx = np.where(((k + prm[..., 1]) & 31) == band, k + 1, bidx)
        isb = typ == 1
        idx = np.where(isb, bidx, idx)
        cov.add(f"band_slot_bd{bd}", bidx[isb])
        cov.add(f"band_pos_bd{bd}", prm[..., 1][isb])
        cov.add(f"band_wrap_bd{bd}", ((prm[..., 1] + 3 > 31) & (bidx > 0) & (band < 4))[isb])
        # edge offset
        ise = typ == 2
        cls = np.where(ise, prm[..., 1], 0)
        ok = np.ones((h, w), bool)
        sgn = np.zeros((h, w), np.int64)
        for k in range(2):
            hx = np.choose(cls, [H_POS[e][k] for e in range(4)])
            vy = np.choose(cls, [V_POS[e][k] for e in range(4)])
            nx, ny = xx + hx, yy + vy
            inside = (nx >= 0) & (nx < w) & (ny >= 0) & (ny < h)
            ok &= inside
            nxc, nyc = np.clip(nx, 0, w - 1), np.clip(ny, 0, h - 1)
            nreg = pic.ctb_region[nyc // cth, nxc // ctw]
            other = sid[nreg] != sid[reg]
            # the sample of the earlier slice sees the later slice's flag decide, and vice versa (8.7.3.2)
            later_flag = np.where(sid[nreg] < sid[reg], across[reg], across[nreg])
            blocked = (other & (later_flag == 0)) | ((tid[nreg] != tid[reg]) & (tiles_across == 0))
            cov.add("eo_blocked", (blocked & inside)[ise])
            ok &= ~blocked
            sgn = sgn + np.sign(rec - rec[nyc, nxc])
        cov.add("eo_outside", (~ok)[ise])
        eidx = 2 + sgn
        eidx = np.where(eidx <= 2, np.where(eidx == 2, 0, eidx + 1), eidx)
        eidx = np.where(ok, eidx, 0)
        idx = np.where(ise, eidx, idx)
        cov.add(f"edge_idx_bd{bd}", (cls * 5 + eidx)[ise & ok])
        off = np.take_along_axis(offval, idx[..., None], axis=2)[..., 0]
        off = np.where(typ > 0, off, 0)
        v = rec + off
        cov.add(f"sao_sat_bd{bd}", np.where(v < 0, -1, np.where(v > pic.maxv, 1, 0))[typ > 0])
        out.append(np.clip(v, 0, pic.maxv))
    return out


def crop_paste(pic, planes, cov):
    """the conformance window of the SAO output pasted into a sentinel-filled destination"""
    cx, cy, ow, oh = pic.window
    dw, dh, dp, dcp, px, py = pic.dst
    for side, cut in (("left", cx > 0), ("right", cx + ow < pic.w), ("top", cy > 0), ("bottom", cy + oh < pic.h)):
        cov.add(f"crop_side_bd{pic.bd}", [side] if cut else [])
    cov.add(f"crop_chroma_off_grid_bd{pic.bd}", [bool(pic.chroma) and ((cx >> pic.sx) & 7) != 0])
    cov.add(f"paste_misaligned_bd{pic.bd}", [(px & 7) != 0 or (dp & 7) != 0])
    fill = SENTINEL if pic.bd == 8 else SENTINEL * 257
    res = []
    for c, (rows, pitch) in enumerate(pic.dst_shapes()):
        sx, sy = (pic.sx, pic.sy) if c else (0, 0)
        d = np.full((rows, pitch), fill, np.int64)
        x0, y0, w, h = cx >> sx, cy >> sy, (ow + sx) >> sx, (oh + sy) >> sy
        d[py >> sy:(py >> sy) + h, px >> sx:(px >> sx) + w] = planes[c][y0:y0 + h, x0:x0 + w]
        res.append(d)
    return res


# ------------------------------------------------------------------------------------------ the exports
def _records(pics):
    rec = np.array([[p.w, p.h, p.lg, p.bd, p.chroma, p.cb_off, p.cr_off, p.sao_enabled, len(p.regions), *p.window, *p.dst] for p in pics], np.int32)
    qp8 = np.concatenate([p.qp8.reshape(-1) for p in pics]).astype(np.int8)
    edge8 = np.concatenate([p.edge8.reshape(-1) for p in pics]).astype(np.uint8)
    ctbs = np.concatenate([np.concatenate([p.ctb_region.reshape(-1, 1), p.sao.reshape(-1, 18)], axis=1) for p in pics]).astype(np.int32)
    regs = np.array([[r["beta"], r["tc"], r["across_slices"], r["slice_id"], r["tile_id"], r["across_tiles"]] for p in pics for r in p.regions], np.int32)
    planes = b"".join(np.ascontiguousarray(a, np.uint8 if p.bd == 8 else np.uint16).tobytes() for p in pics for a in p.planes[:p.ncomp])
    return rec, qp8, edge8, ctbs, regs, planes


def run_filters(pics, stages):
    """b200_debug_loop_filters: (rc, deblocked planes per picture, destination planes per picture)"""
    rec, qp8, edge8, ctbs, regs, planes = _records(pics)
    pin = np.frombuffer(planes, np.uint8).copy()
    rout = np.zeros_like(pin)
    dsz = sum(rows * pitch * (1 if p.bd == 8 else 2) for p in pics for rows, pitch in p.dst_shapes())
    dout = np.zeros(max(dsz, 1), np.uint8)
    rc = _lib.lib().b200_debug_loop_filters(stages, len(pics), rec.ctypes.data, qp8.ctypes.data, edge8.ctypes.data, ctbs.ctypes.data, regs.ctypes.data,
                                            pin.ctypes.data, rout.ctypes.data, dout.ctypes.data, SENTINEL)
    if rc:
        return rc, None, None
    recs, dsts, a, b = [], [], 0, 0
    for p in pics:
        dt = np.uint8 if p.bd == 8 else np.uint16
        bps = np.dtype(dt).itemsize
        r = []
        for c in range(p.ncomp):
            w, h = p.comp_size(c)
            r.append(rout[a:a + w * h * bps].view(dt).reshape(h, w).astype(np.int64)); a += w * h * bps
        recs.append(r)
        d = []
        for rows, pitch in p.dst_shapes():
            d.append(dout[b:b + rows * pitch * bps].view(dt).reshape(rows, pitch).astype(np.int64)); b += rows * pitch * bps
        dsts.append(d)
    return 0, recs, dsts


def parse_filters(au):
    """b200_debug_parse_filters + b200_debug_parse: the Pic (without planes) the host front-end parses from `au`"""
    l = _lib.lib()
    hdr = np.zeros(13, np.int32)
    _lib.check(l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, None, 0, None, 0))
    w, h, lg, bd, chroma, cb, cr, sao_en, ns, cx, cy, ow, oh = hdr.tolist()
    nctb = (-(-w >> lg)) * (-(-h >> lg))
    ctbs = np.zeros((nctb, 19), np.int32)
    regs = np.zeros((ns, 6), np.int32)
    _lib.check(l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, ctbs.ctypes.data, nctb, regs.ctypes.data, ns))
    qp8 = np.zeros((h >> 3) * (w >> 3), np.int8)
    edge8 = np.zeros_like(qp8, np.uint8)
    lm4, cm4 = np.zeros((h >> 2) * (w >> 2), np.uint8), np.zeros((h >> 2) * (w >> 2), np.uint8)
    out5 = np.zeros(5, np.uint64)
    _lib.check(l.b200_debug_parse(au, len(au), qp8.ctypes.data, edge8.ctypes.data, lm4.ctypes.data, cm4.ctypes.data, out5.ctypes.data))
    wctb, hctb = -(-w >> lg), -(-h >> lg)
    regions = [dict(beta=int(r[0]), tc=int(r[1]), across_slices=int(r[2]), slice_id=int(r[3]), tile_id=int(r[4]), across_tiles=int(r[5])) for r in regs]
    return Pic(w, h, lg, bd, chroma, qp8=qp8.astype(np.int64).reshape(h >> 3, w >> 3), edge8=edge8.astype(np.int64).reshape(h >> 3, w >> 3),
               ctb_region=ctbs[:, 0].astype(np.int64).reshape(hctb, wctb), sao=ctbs[:, 1:].astype(np.int64).reshape(hctb, wctb, 3, 6),
               regions=regions, cb_off=cb, cr_off=cr, sao_enabled=sao_en, window=(cx, cy, ow, oh))


# ------------------------------------------------------------------------------------------ SPS rewriter (conformance window)
class _Bits:
    def __init__(self, data):
        self.b = np.unpackbits(np.frombuffer(data, np.uint8)).tolist()
        self.i = 0

    def u(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | self.b[self.i]; self.i += 1
        return v

    def ue(self):
        z = 0
        while self.b[self.i] == 0:
            z += 1; self.i += 1
        self.i += 1
        return (1 << z) - 1 + self.u(z)


def _ue_bits(v):
    v += 1
    n = v.bit_length()
    return [0] * (n - 1) + [(v >> (n - 1 - i)) & 1 for i in range(n)]


def _unescape(b):
    out, z = bytearray(), 0
    for x in b:
        if z >= 2 and x == 3:
            z = 0
            continue
        out.append(x)
        z = z + 1 if x == 0 else 0
    return bytes(out)


def _escape(b):
    out, z = bytearray(), 0
    for x in b:
        if z >= 2 and x <= 3:
            out.append(3); z = 0
        out.append(x)
        z = z + 1 if x == 0 else 0
    return bytes(out)


def _nals(au):
    i, out = 0, []
    while i < len(au):
        n = int.from_bytes(au[i:i + 4], "big")
        out.append(au[i + 4:i + 4 + n]); i += 4 + n
    return out


def set_conformance_window(au, left, right, top, bottom):
    """The access unit with the SPS's conformance window replaced (offsets in chroma units; all zero: no window).  Only the
    fields up to the window are parsed (7.3.2.2): everything after it is copied bit for bit, then the stop bit is set anew
    and the emulation prevention put back."""
    out = bytearray()
    for nal in _nals(au):
        if (nal[0] >> 1) & 63 == 33:
            r = _unescape(nal[2:])
            bits = np.unpackbits(np.frombuffer(r, np.uint8)).tolist()
            last = len(bits) - 1 - bits[::-1].index(1)                     # rbsp_stop_one_bit
            b = _Bits(r)
            b.u(4); msl = b.u(3); b.u(1)
            b.u(88); b.u(8)                                                # general profile / level (profile_tier_level)
            flags = [(b.u(1), b.u(1)) for _ in range(msl)]
            if msl:
                b.u(2 * (8 - msl))
            for pp, lp in flags:
                b.u(88 * pp + 8 * lp)
            b.ue()
            chroma = b.ue()
            if chroma == 3:
                b.u(1)
            b.ue(); b.ue()
            head = bits[:b.i]
            if b.u(1):
                for _ in range(4):
                    b.ue()
            tail = bits[b.i:last]
            win = [1] + sum((_ue_bits(v) for v in (left, right, top, bottom)), []) if (left or right or top or bottom) else [0]
            nb = head + win + tail + [1]
            nb += [0] * (-len(nb) % 8)
            nal = nal[:2] + _escape(np.packbits(np.array(nb, np.uint8)).tobytes())
        out += len(nal).to_bytes(4, "big") + nal
    return bytes(out)


def sps_window(au):
    """(chroma_format_idc, W, H, conformance window offsets or None) as written in the SPS"""
    for nal in _nals(au):
        if (nal[0] >> 1) & 63 == 33:
            b = _Bits(_unescape(nal[2:]))
            b.u(4); msl = b.u(3); b.u(1); b.u(96)
            flags = [(b.u(1), b.u(1)) for _ in range(msl)]
            if msl:
                b.u(2 * (8 - msl))
            for pp, lp in flags:
                b.u(88 * pp + 8 * lp)
            b.ue()
            chroma = b.ue()
            if chroma == 3:
                b.u(1)
            w, h = b.ue(), b.ue()
            return chroma, w, h, (tuple(b.ue() for _ in range(4)) if b.u(1) else None)
    raise ValueError("no SPS")


# ------------------------------------------------------------------------------------------ restatement self-checks (CPU)
def test_tables_against_the_spec_rows():
    """spot values of Tables 8-10 and 8-12 as printed, and the monotonicity the tables have"""
    assert [TC_PRIME[q] for q in (17, 18, 26, 27, 31, 35, 38, 40, 42, 47, 53)] == [0, 1, 1, 2, 3, 4, 5, 6, 7, 13, 24]
    assert [BETA_PRIME[q] for q in (15, 16, 20, 28, 29, 40, 51)] == [0, 6, 10, 18, 20, 42, 64]
    assert all(a <= b for a, b in zip(TC_PRIME, TC_PRIME[1:])) and all(a <= b for a, b in zip(BETA_PRIME, BETA_PRIME[1:]))
    assert [qpc_of(q, 1) for q in (29, 30, 34, 35, 42, 43, 44, 57)] == [29, 29, 33, 33, 37, 37, 38, 51]
    assert [qpc_of(q, 2) for q in (-10, 40, 51, 60)] == [-10, 40, 51, 51]


def test_sps_rewriter_round_trip():
    au = synth_stream("odd_size_random")                 # 130x70: coded 136x72 with a right / bottom window
    chroma, w, h, win = sps_window(au)
    assert (chroma, w, h, win) == (1, 136, 72, (0, 3, 0, 1))
    assert set_conformance_window(au, *win) == au
    au2 = set_conformance_window(au, 2, 1, 3, 0)
    assert sps_window(au2) == (1, 136, 72, (2, 1, 3, 0))
    assert sps_window(set_conformance_window(au2, 0, 0, 0, 0)) == (1, 136, 72, None)


# ------------------------------------------------------------------------------------------ constructed edges (K3)
def _segment(rng, beta, tc, maxv):
    """4 lines x (p3 p2 p1 p0 q0 q1 q2 q3) of one edge segment, built so that one decision of 8.7.2.5.3 / 8.7.2.5.6 /
    8.7.2.5.7 lands at its threshold or one below it (or a clip at 0 / maxv is reached)"""
    mode = int(rng.integers(0, 8))
    k = int(rng.integers(-1, 1))
    dp, dq, tp, tq, g, u = (np.zeros(4, np.int64) for _ in range(6))
    L = int(rng.choice([0, 3]))
    side = (beta + (beta >> 1)) >> 3
    m = None
    if mode == 0:                                       # dpq0 + dpq3 against beta
        dp[0], dq[0], dp[3], dq[3] = rng.multinomial(max(beta + k, 0), [0.25] * 4)
    elif mode == 1:                                     # 2 * dpq against beta >> 2, on line 0 or 3
        t = max(((beta >> 2) + k + int(rng.integers(0, 2))) // 2, 0)
        dp[L] = int(rng.integers(0, t + 1)); dq[L] = t - dp[L]
    elif mode == 2:                                     # |p3 - p0| + |q0 - q3| against beta >> 3
        t = max((beta >> 3) + k, 0)
        tp[L] = int(rng.integers(0, t + 1)); tq[L] = t - tp[L]
    elif mode == 3:                                     # |p0 - q0| against (5 tc + 1) >> 1
        g[L] = max(((5 * tc + 1) >> 1) + k, 0) * int(rng.choice([-1, 1]))
    elif mode == 4:                                     # dEp / dEq (normal filter: flatness fails)
        tp[0] = tp[3] = (beta >> 3) + 1
        a, b = max(side + k, 0), max(side + int(rng.integers(-1, 1)), 0)
        if rng.integers(0, 2):
            a, b = b, a
        dp[0] = int(rng.integers(0, a + 1)); dp[3] = a - dp[0]
        dq[0] = int(rng.integers(0, b + 1)); dq[3] = b - dq[0]
    elif mode == 5:                                     # |delta| against 10 tc
        tp[:] = (beta >> 3) + 1
        T = max(10 * tc + k, 0)
        sgn = int(rng.choice([-1, 1]))
        gg = np.arange(-maxv, maxv + 1)[:, None]
        uu = np.arange(-maxv, maxv + 1, max(1, maxv // 64))[None, :]
        dl = (6 * gg - 3 * uu + 8) >> 4
        span = np.maximum(np.abs(gg) + np.abs(2 * uu), 0)
        ok = (dl == sgn * T) & (span <= maxv)
        if ok.any():
            i, j = np.argwhere(ok)[int(rng.integers(0, ok.sum()))]
            g[:] = gg[i, 0]; u[:] = uu[0, j]
    elif mode == 6:                                     # clips at 0 (mirrored: at maxv) in the normal filter
        tp[:] = (beta >> 3) + 1
        m = int(rng.integers(0, 3))
        g[:] = rng.integers(0, 3)
        u[:] = rng.integers(tc, 4 * tc + 12)
        dp[:] = rng.integers(0, 2); dq[:] = rng.integers(0, 2)
    else:                                               # anything near the thresholds
        r = beta // 2 + 2
        dp[:], dq[:], tp[:], tq[:] = (rng.integers(-r, r + 1, 4) for _ in range(4))
        g[:] = rng.integers(-3 * tc - 2, 3 * tc + 3, 4); u[:] = rng.integers(-tc - 2, tc + 3, 4)
    for l in (1, 2):                                    # lines 1 and 2: like line 0 or 3
        s = int(rng.choice([0, 3]))
        for a in (dp, dq, tp, tq, g, u):
            a[l] = a[s]
    sgn = lambda a: a * rng.choice([-1, 1], 4)
    dpv, dqv, tpv, tqv = sgn(dp), sgn(dq), sgn(tp), sgn(tq)
    if mode == 6:
        dpv, dqv, tpv = dp, dq, tp
    rel = np.stack([tpv, dpv, np.zeros(4, np.int64), np.zeros(4, np.int64), g, g + u, g + 2 * u + dqv, g + tqv], axis=1)
    if m is None:
        lo, hi = rel.min(), rel.max()
        m = int(rng.integers(-lo, max(maxv - hi, -lo) + 1)) if hi - lo <= maxv else -lo
    v = np.clip(rel + m, 0, maxv)
    if mode == 6 and rng.integers(0, 2):
        v = maxv - v
    if mode == 6 and rng.integers(0, 2):                # the same on the Q side
        v = v[:, ::-1]
    return v


def _extreme_plane(rng, shape, maxv):
    """samples piled up at 0 and maxv and spread in between"""
    pick = rng.integers(0, 4, shape)
    return np.select([pick == 0, pick == 1], [rng.integers(0, 3, shape), maxv - rng.integers(0, 3, shape)], rng.integers(0, maxv + 1, shape)).astype(np.int64)


def k3_picture(rng, w, h, lg, bd, chroma, vertical):
    """A picture whose edges of one direction are constructed segment by segment (_segment); built as a picture with
    vertical edges and transposed for horizontal ones.  Two regions with different beta / tc offsets meet inside it."""
    W, H = (w, h) if vertical else (h, w)                 # oriented size
    w8, h8 = W >> 3, H >> 3
    maxv = (1 << bd) - 1
    minqp = -6 * (bd - 8)
    qp8 = rng.integers(minqp, 52, (h8, w8))
    qp8[rng.random((h8, w8)) < 0.1] = 51
    qp8[rng.random((h8, w8)) < 0.1] = minqp
    e8 = np.where(rng.random((h8, w8)) < 0.9, 1, 0) | np.where(rng.random((h8, w8)) < 0.9, 2, 0) | np.where(rng.random((h8, w8)) < 0.12, 4, 0)
    wc, hc = -(-W >> lg), -(-H >> lg)
    creg = np.zeros((hc, wc), np.int64)
    creg[:, wc // 2:] = 1
    offs = rng.choice(np.arange(-12, 13, 2), 4)
    offs[int(rng.integers(0, 4))] = int(rng.choice([-12, 12]))
    regions = [dict(beta=int(offs[0]), tc=int(offs[1]), across_slices=1, slice_id=0, tile_id=0, across_tiles=1),
               dict(beta=int(offs[2]), tc=int(offs[3]), across_slices=1, slice_id=1, tile_id=0, across_tiles=1)]
    Y = _extreme_plane(rng, (H, W), maxv)
    for by in range(h8):
        for bx in range(1, w8):
            qpl = (int(qp8[by, bx]) + int(qp8[by, bx - 1]) + 1) >> 1
            for half in (0, 1):
                y, x = by * 8 + 4 * half, bx * 8
                r = regions[creg[y >> lg, x >> lg]]
                beta = BETA_PRIME[min(max(qpl + r["beta"], 0), 51)] << (bd - 8)
                tc = TC_PRIME[min(max(qpl + 2 + r["tc"], 0), 53)] << (bd - 8)
                Y[y:y + 4, x - 4:x + 4] = _segment(rng, beta, tc, maxv)
    sx, sy = sub_wh(chroma)
    planes = [Y if vertical else Y.T.copy()]
    if chroma:
        planes += [_extreme_plane(rng, (h >> sy, w >> sx), maxv) for _ in range(2)]
    if not vertical:
        qp8, creg = qp8.T.copy(), creg.T.copy()
        e8 = ((e8 & 1) << 1 | (e8 & 2) >> 1 | (e8 & 4)).T.copy()
    co = rng.choice([-12, -5, 0, 3, 12], 2)
    return Pic(w, h, lg, bd, chroma, planes=planes, qp8=qp8, edge8=e8, ctb_region=creg, regions=regions, cb_off=int(co[0]), cr_off=int(co[1]))


# (w, h, log2 CTB, chroma, edges constructed vertical) of the pictures of one batch: sizes and CTB sizes differ, so that the
# kernel's max_w8 / max_seg indexing is exercised
K3_BATCH = [(264, 136, 4, 1, True), (200, 264, 5, 2, False), (520, 72, 6, 3, True), (128, 128, 4, 0, False), (136, 200, 5, 1, False),
            (96, 320, 6, 2, True), (72, 48, 4, 3, False), (256, 96, 5, 1, True)]


def k3_batch(bd):
    rng = np.random.default_rng(0x3D + bd)
    return [k3_picture(rng, w, h, lg, bd, ch, v) for (w, h, lg, ch, v) in K3_BATCH]


_k3_cache = {}


def k3_expected(bd):
    if bd not in _k3_cache:
        pics = k3_batch(bd)
        cov = Cov()
        _k3_cache[bd] = (pics, [deblock(p, p.planes, cov) for p in pics], cov)
    return _k3_cache[bd]


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_k3_constructed_edges_reach_every_branch(bd):
    """the constructed batch reaches every deblocking decision at its threshold and one below it, both clips, every entry of
    tC' and beta' with the clamps, odd P / Q QP sums, keep bits on either side, and every chroma QP range"""
    _, _, cov = k3_expected(bd)
    for name in ["d_vs_beta", "dEp", "dEq", "delta_vs_10tc"] + [f"strong{i}_l{l}" for i in (2, 3) for l in (0, 3)]:
        assert {-1, 0} <= set(cov[name]), (name, dict(cov[name]))
    for l in (0, 3):                                      # 2 * dpq is even: tight below is -2 or -1, tight at is 0 or 1
        assert set(cov[f"strong1_l{l}"]) & {-2, -1} and set(cov[f"strong1_l{l}"]) & {0, 1}, dict(cov[f"strong1_l{l}"])
    assert set(cov["decision"]) == {0, 1, 2}
    for name in ("clip_p0", "clip_q0", "clip_p1", "clip_q1", "clip_chroma"):
        assert {-1, 0, 1} <= set(cov[f"{name}_bd{bd}"]), (name, dict(cov[f"{name}_bd{bd}"]))
    assert {-1, 1} <= set(cov["delta_clipped"])
    assert set(cov["Qbeta"]) == set(range(52)) and set(cov["Qtc"]) == set(range(54))
    assert {-1, 0, 1} <= set(cov["Qbeta_raw_clamp"]) and {-1, 0, 1} <= set(cov["Qtc_raw_clamp"])
    assert {0, 1, 2, 3} <= set(cov["keep_active"]) and 1 in cov["qp_odd_sum"]
    assert set(cov["qpi_range"]) == {0, 1, 2} and set(cov["chroma_edges_fmt"]) == {1, 2, 3}
    if bd > 8:
        assert -1 in cov["qpl_sign"]


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_k3_constructed_edges(cuda, bd):
    pics, want, _ = k3_expected(bd)
    rc, got, _ = run_filters(pics, 1)
    assert rc == 0
    for i, (p, g, wnt) in enumerate(zip(pics, got, want)):
        for c in range(p.ncomp):
            bad = np.argwhere(g[c] != wnt[c])
            assert not len(bad), f"picture {i} ({p.w}x{p.h} chroma {p.chroma}) plane {c}: first diffs {bad[:4].tolist()}"


# ------------------------------------------------------------------------------------------ constructed pictures (K4)
def _cmax(bd):
    return ((1 << (min(bd, 10) - 5)) - 1) << max(0, bd - 10)


def k4_picture(rng, w, h, lg, bd, chroma, band_base=0, regions=None, ctb_region=None, window=None, dst=None, sao_enabled=1, off_comp=None):
    """A picture for SAO: every CTB of every component gets its own type, band position (consecutive positions from
    `band_base`, so a batch covers all 32) or EO class and offsets with +-cmax often; samples are spread over every band
    with runs of equal values (edgeIdx ties) and piles at 0 and maxv; the keep bit is set on some 8x8 cells."""
    p = Pic(w, h, lg, bd, chroma, regions=regions, ctb_region=ctb_region, window=window, dst=dst, sao_enabled=sao_enabled)
    maxv, cm = p.maxv, _cmax(bd)
    sao = np.zeros((p.hctb, p.wctb, 3, 6), np.int64)
    n = p.hctb * p.wctb
    for c in range(3):
        t = rng.choice([0, 1, 1, 2, 2, 2], n)
        pos = (band_base + 7 * c + np.arange(n)) % 32
        cls = rng.integers(0, 4, n)
        offs = rng.integers(-cm, cm + 1, (n, 4))
        offs[rng.random((n, 4)) < 0.35] = cm
        offs[rng.random((n, 4)) < 0.35] = -cm
        sao[..., c, 0] = 0 if c == off_comp else t.reshape(p.hctb, p.wctb)      # off_comp: slice_sao_luma / chroma_flag = 0
        sao[..., c, 1] = np.where(t == 2, cls, pos).reshape(p.hctb, p.wctb)
        sao[..., c, 2:] = offs.reshape(p.hctb, p.wctb, 4)
    p.sao = sao
    planes = []
    for c in range(p.ncomp):
        cw, chh = p.comp_size(c)
        base = rng.integers(0, maxv + 1, (chh, cw))
        level = np.repeat(np.repeat(rng.integers(0, maxv + 1, (-(-chh // 4), -(-cw // 4))), 4, 0), 4, 1)[:chh, :cw]
        level[rng.random(level.shape) < 0.05] = 0
        level[rng.random(level.shape) < 0.05] = maxv
        tie = np.clip(level + rng.integers(-1, 2, (chh, cw)), 0, maxv)
        planes.append(np.where(rng.random((chh, cw)) < 0.4, base, tie).astype(np.int64))
    p.planes = planes
    p.edge8 = np.where(rng.random((p.h8, p.w8)) < 0.15, 4, 0) | rng.integers(0, 4, (p.h8, p.w8))
    p.qp8 = rng.integers(-6 * (bd - 8), 52, (p.h8, p.w8))
    return p


def _window_dst(p, rng, kind):
    """conformance window and destination of kind 0: none, 1: all four sides with chroma offsets off the 8-sample grid and a
    misaligned paste / pitch, 2: left and top only, 3: right and bottom only, in a larger canvas"""
    sx, sy = p.sx, p.sy
    if kind == 0:
        return
    ux, uy = 1 << sx, 1 << sy
    l = 0 if kind == 3 else ux * int(rng.integers(1, 6)) + (ux if kind == 1 else 0)
    t = 0 if kind == 3 else uy * int(rng.integers(1, 6))
    r = 0 if kind == 2 else ux * int(rng.integers(1, 6))
    b = 0 if kind == 2 else uy * int(rng.integers(1, 6))
    ow, oh = p.w - l - r, p.h - t - b
    px, py = ux * int(rng.integers(0, 6)) + ux, uy * int(rng.integers(0, 4))
    dw, dh = px + ow + int(rng.integers(0, 9)), py + oh + int(rng.integers(0, 3))
    dp = dw + int(rng.integers(0, 5))
    dcp = ((dw + sx) >> sx) + int(rng.integers(0, 3))
    p.window, p.dst = (l, t, ow, oh), (dw, dh, dp, dcp, px, py)


# (w, h, log2 CTB, chroma): chroma widths = 4 mod 8 (partial units), widths above 256 (lane 0 / 31 load their own outer
# neighbours), 512 luma samples = exactly two warps, 4:0:0 to 4:4:4, CTB 16 / 32 / 64
K4_BATCH = [(264, 72, 4, 1), (512, 40, 5, 0), (776, 48, 6, 2), (136, 56, 4, 3), (1032, 24, 5, 1), (520, 64, 6, 1), (256, 32, 4, 3), (72, 40, 5, 2)]


def k4_batch(bd):
    rng = np.random.default_rng(0x4D + bd)
    pics = []
    for i, (w, h, lg, ch) in enumerate(K4_BATCH):
        p = k4_picture(rng, w, h, lg, bd, ch, band_base=5 * i, sao_enabled=0 if i == 7 else 1, off_comp=(1 if i == 3 else (0 if i == 6 else None)))
        _window_dst(p, rng, i % 4)
        pics.append(p)
    return pics


def k4_regions_batch(bd):
    """multi-region pictures: slices by CTB rows with slice_loop_filter_across_slices_enabled_flag 0 / 1 in both orders, tiles
    with loop_filter_across_tiles_enabled_flag 0 / 1, one slice over several tiles"""
    rng = np.random.default_rng(0x5D + bd)
    pics = []
    lay = [  # (w, h, lg, chroma, kind)
        (264, 128, 4, 1, "slices01"), (200, 96, 5, 3, "slices10"), (320, 128, 5, 2, "tiles0"), (264, 144, 4, 0, "tiles1"), (384, 128, 6, 1, "slice_over_tiles")]
    for i, (w, h, lg, ch, kind) in enumerate(lay):
        wc, hc = -(-w >> lg), -(-h >> lg)
        cr = np.zeros((hc, wc), np.int64)
        R = lambda **k: dict(dict(beta=0, tc=0, across_slices=1, slice_id=0, tile_id=0, across_tiles=1), **k)
        if kind.startswith("slices"):
            f = [0, 1, 0, 1] if kind == "slices01" else [1, 0, 1, 0]
            cr[:] = np.minimum(np.arange(hc) * 4 // hc, 3)[:, None]
            cr[hc // 2, wc // 3:] = 3                                   # a slice that starts mid row
            regions = [R(slice_id=k, across_slices=f[k]) for k in range(4)]
        elif kind.startswith("tiles"):
            a = 1 if kind == "tiles1" else 0
            cr[:, wc // 2:] = 1; cr[hc // 2:, :] += 2
            regions = [R(slice_id=k, tile_id=k, across_tiles=a, across_slices=k % 2) for k in range(4)]
        else:
            cr[:, wc // 3:] = 1; cr[:, 2 * wc // 3:] = 2
            regions = [R(slice_id=0, tile_id=k, across_tiles=0) for k in range(3)]
        p = k4_picture(rng, w, h, lg, bd, ch, band_base=3 * i, regions=regions, ctb_region=cr)
        _window_dst(p, rng, (i + 1) % 4)
        pics.append(p)
    return pics


def expected_k4(pics, cov, with_deblock=False):
    out = []
    for p in pics:
        pl = deblock(p, p.planes, cov) if with_deblock else p.planes
        out.append(crop_paste(p, sao(p, pl, cov), cov))
    return out


@pytest.mark.parametrize("bd", [8, 10, 12])
def test_k4_constructed_pictures_reach_every_branch(bd):
    cov = Cov()
    expected_k4(k4_batch(bd) + k4_regions_batch(bd), cov)
    assert set(cov[f"band_slot_bd{bd}"]) == {0, 1, 2, 3, 4}
    assert set(cov[f"band_pos_bd{bd}"]) == set(range(32)) and True in cov[f"band_wrap_bd{bd}"]
    assert set(cov[f"edge_idx_bd{bd}"]) == set(range(20))          # every EO class with every edgeIdx
    assert {-1, 0, 1} <= set(cov[f"sao_sat_bd{bd}"])
    assert True in cov["eo_outside"] and True in cov["eo_blocked"]
    assert set(cov[f"crop_side_bd{bd}"]) == {"left", "right", "top", "bottom"}    # conformance window sides
    assert True in cov[f"crop_chroma_off_grid_bd{bd}"] and True in cov[f"paste_misaligned_bd{bd}"]


def _compare(pics, got, want, what):
    for i, (p, g, wnt) in enumerate(zip(pics, got, want)):
        for c in range(len(wnt)):
            bad = np.argwhere(g[c] != wnt[c])
            assert not len(bad), f"{what}: picture {i} ({p.w}x{p.h} chroma {p.chroma} window {p.window} dst {p.dst}) plane {c}: first diffs {bad[:4].tolist()}"


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
@pytest.mark.parametrize("batch", ["single_region", "regions"])
def test_k4_constructed_pictures(cuda, bd, batch):
    """K4 alone on the given planes; the whole destination, sentinel included, must match"""
    pics = k4_batch(bd) if batch == "single_region" else k4_regions_batch(bd)
    rc, _, got = run_filters(pics, 2)
    assert rc == 0
    _compare(pics, got, expected_k4(pics, Cov()), "K4")


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10, 12])
def test_k3_then_k4(cuda, bd):
    pics = k4_batch(bd)[:4] + k4_regions_batch(bd)[:2]
    rc, rec, got = run_filters(pics, 3)
    assert rc == 0
    cov = Cov()
    _compare(pics, rec, [deblock(p, p.planes, cov) for p in pics], "K3")
    _compare(pics, got, expected_k4(pics, cov, with_deblock=True), "K3 + K4")


@pytest.mark.gpu
@pytest.mark.parametrize("bd", [8, 10])
def test_k4_fast_path_equals_general_path(cuda, bd):
    """one region (the single-slice path) and the same picture as two slices that both filter across (the multi-region
    path) give the same bytes"""
    rng = np.random.default_rng(0x6D + bd)
    one = k4_picture(rng, 776, 96, 5, bd, 1)
    two = Pic(one.w, one.h, one.lg, bd, 1, planes=one.planes, qp8=one.qp8, edge8=one.edge8, sao=one.sao,
              ctb_region=(np.arange(one.hctb)[:, None] * one.wctb + np.arange(one.wctb)[None, :] >= one.wctb + 5).astype(np.int64),
              regions=[dict(beta=0, tc=0, across_slices=1, slice_id=0, tile_id=0, across_tiles=1), dict(beta=0, tc=0, across_slices=1, slice_id=1, tile_id=0, across_tiles=1)])
    rc1, _, a = run_filters([one], 2)
    rc2, _, b = run_filters([two], 2)
    assert rc1 == rc2 == 0
    for c in range(3):
        assert np.array_equal(a[0][c], b[0][c]), f"plane {c}"
    _compare([one], a, expected_k4([one], Cov()), "K4")


# ------------------------------------------------------------------------------------------ refusals (host checks)
def _good():
    rng = np.random.default_rng(1)
    return [k4_picture(rng, 64, 32, 4, 8, 1)]


BAD = {
    "none": lambda p, a: None,                  # the unmodified call passes the checks (and fails only without a device)
    "stages": lambda p, a: a.__setitem__("stages", 4),
    "npics": lambda p, a: a.__setitem__("npics", 0),
    "size": lambda p, a: setattr(p, "w", 60),
    "log2_ctb": lambda p, a: setattr(p, "lg", 7),
    "bit_depth": lambda p, a: setattr(p, "bd", 13),
    "chroma": lambda p, a: setattr(p, "chroma", 4),
    "qp_offset": lambda p, a: setattr(p, "cb_off", 13),
    "sao_flag": lambda p, a: setattr(p, "sao_enabled", 2),
    "qp8_low": lambda p, a: p.qp8.__setitem__((0, 0), -1),
    "qp8_high": lambda p, a: p.qp8.__setitem__((0, 0), 52),
    "edge8_bits": lambda p, a: p.edge8.__setitem__((0, 0), 8),
    "region_index": lambda p, a: p.ctb_region.__setitem__((0, 0), 1),
    "sao_type": lambda p, a: p.sao.__setitem__((0, 0, 0, 0), 3),
    "eo_class": lambda p, a: (p.sao.__setitem__((0, 0, 0, 0), 2), p.sao.__setitem__((0, 0, 0, 1), 4)),
    "sao_offset": lambda p, a: p.sao.__setitem__((0, 0, 1, 2), 8),
    "beta_odd": lambda p, a: p.regions[0].__setitem__("beta", 1),
    "tc_range": lambda p, a: p.regions[0].__setitem__("tc", 14),
    "window_x": lambda p, a: setattr(p, "window", (1, 0, 62, 32)),
    "window_size": lambda p, a: setattr(p, "window", (2, 0, 64, 32)),
    "paste": lambda p, a: setattr(p, "dst", (64, 32, 64, 32, 2, 0)),
    "pitch": lambda p, a: setattr(p, "dst", (64, 32, 63, 32, 0, 0)),
    "null_dst": lambda p, a: a.__setitem__("dst", None),
    "sentinel": lambda p, a: a.__setitem__("sentinel", 256),
    "npics_high": lambda p, a: a.__setitem__("npics", 257),
    "size_large": lambda p, a: setattr(p, "h", 4104),
    "regions_none": lambda p, a: a.__setitem__("nslices", 0),
    "regions_many": lambda p, a: a.__setitem__("nslices", 4097),
    "window_y_odd": lambda p, a: setattr(p, "window", (0, 1, 64, 30)),
    "paste_y_odd": lambda p, a: setattr(p, "dst", (64, 40, 64, 32, 0, 3)),
    "chroma_pitch": lambda p, a: setattr(p, "dst", (64, 32, 64, 31, 0, 0)),
    "across_slices_flag": lambda p, a: p.regions[0].__setitem__("across_slices", 2),
    "across_tiles_flag": lambda p, a: p.regions[0].__setitem__("across_tiles", 2),
    "slice_id": lambda p, a: p.regions[0].__setitem__("slice_id", 65536),
    "tile_id": lambda p, a: p.regions[0].__setitem__("tile_id", -1),
    "across_tiles_differ": lambda p, a: (p.regions.append(dict(p.regions[0], slice_id=1, across_tiles=0)), p.ctb_region.__setitem__((0, 0), 1)),
}


@pytest.mark.parametrize("what", sorted(BAD))
def test_loop_filters_refuses_bad_arguments(what):
    """every refusal happens on the host, before any CUDA call: these run without a device"""
    pics = _good()
    args = dict(stages=2, npics=1, dst=True, sentinel=SENTINEL)
    BAD[what](pics[0], args)
    rec, qp8, edge8, ctbs, regs, planes = _records(pics)
    if "nslices" in args:
        rec[0, 8] = args["nslices"]
    pin = np.frombuffer(planes, np.uint8).copy()
    out = np.zeros(1 << 16, np.uint8)
    rc = _lib.lib().b200_debug_loop_filters(args["stages"], args["npics"], rec.ctypes.data, qp8.ctypes.data, edge8.ctypes.data, ctbs.ctypes.data, regs.ctypes.data,
                                            pin.ctypes.data, out.ctypes.data, out.ctypes.data if args["dst"] else None, args["sentinel"])
    assert (rc != E_INVALID) if what == "none" else (rc == E_INVALID)


def test_loop_filters_refuses_samples_above_maxv():
    rng = np.random.default_rng(2)
    p = k4_picture(rng, 64, 32, 4, 10, 1)
    p.planes[0][3, 3] = 1024
    rc, _, _ = run_filters([p], 2)
    assert rc == E_INVALID


@pytest.mark.gpu
@pytest.mark.parametrize("stages", [1, 2, 3])
def test_mixed_bit_depths_are_refused(cuda, stages):
    """launch_deblock's own check refuses a batch of 8-bit and wider pictures before launching anything; K4 alone is refused
    the same way by the export"""
    rng = np.random.default_rng(3)
    rc, _, _ = run_filters([k4_picture(rng, 64, 32, 4, 8, 1), k4_picture(rng, 64, 32, 4, 10, 1)], stages)
    assert rc == E_UNSUPPORTED


# ------------------------------------------------------------------------------------------ stage chaining on real streams
STREAMS = [s[0] for s in SYNTH + SYNTH_CPU_EXTRA]
FIXTURES = [n for n, _ in fixture_streams()]


def _stream(name):
    return dict(fixture_streams())[name] if name in FIXTURES else synth_stream(name)


def windowless(au):
    """the stream with its conformance window removed: the decode is then the whole coded picture, so the filters' reads
    and writes right of and below the window are compared too"""
    return set_conformance_window(au, 0, 0, 0, 0)


def _oracle(au, stage):
    from oracle import bindings as ob
    return [a.astype(np.int64) for a in ob.restatement_decode(au, stage)[0]]


def _check_chain(pic, s1, s2, s0, what):
    cov = Cov()
    d = deblock(pic, s1, cov)
    for c in range(pic.ncomp):
        bad = np.argwhere(d[c] != s2[c])
        assert not len(bad), f"{what}: deblocking, plane {c}: first diffs {bad[:4].tolist()}"
    s = sao(pic, s2, cov)
    for c in range(pic.ncomp):
        bad = np.argwhere(s[c] != s0[c])
        assert not len(bad), f"{what}: SAO, plane {c}: first diffs {bad[:4].tolist()}"


@pytest.mark.parametrize("name", STREAMS + FIXTURES)
def test_chain_on_the_c_restatement(name):
    """restatement(stage 1) == stage 2 and restatement(stage 2) == stage 0 of the C restatement, for every stream: an
    independent pin of the filters where FFmpeg deviates (chroma SAO at CTB 16, beside bypass / PCM units)"""
    au = windowless(_stream(name))
    pic = parse_filters(au)
    assert pic.window == (0, 0, pic.w, pic.h)
    _check_chain(pic, _oracle(au, 1), _oracle(au, 2), _oracle(au, 0), name)


@pytest.mark.gpu
@pytest.mark.parametrize("front_end", ["device", "host"])
def test_chain_on_the_decoder_stages(cuda, front_end):
    """the same two equalities on the decoder's own stage 1 / stage 2 / final planes, every stream, both front-ends"""
    d = lb.Decoder(host_threads=8)
    d.set_front_end(front_end == "device")
    try:
        for name in STREAMS + FIXTURES:
            au = windowless(_stream(name))
            pic = parse_filters(au)
            st = {}
            for stage in (1, 2, 0):
                d.set_debug_stage(stage)
                d.decode_image(au)
                pl = d.planes_host() if stage == 0 else d.debug_tile(0, pic.w, pic.h)
                st[stage] = [a.astype(np.int64) for a in pl]
            _check_chain(pic, st[1], st[2], st[0], f"{name} ({front_end} front-end)")
    finally:
        d.set_debug_stage(0)
        d.close()


# ------------------------------------------------------------------------------------------ conformance windows in real streams
# (stream, window in chroma units: left, right, top, bottom).  Every window is cut from the window-free coded picture.
def _crop_cases():
    cases = []
    for name in ("mono8", "ctb32", "x_422_basic", "x_444_basic", "main10", "mono10_ctb16_wpp", "x_422_main10_random_tskip", "x_444_main10_ctb16_random_tskip"):
        _, w, h, bd, chroma, _ = next(c for c in SYNTH + SYNTH_CPU_EXTRA if c[0] == name)
        ch = 1 if chroma is True else (0 if chroma is False else chroma)
        sx, sy = sub_wh(ch)
        W, H = (w + 7) & ~7, (h + 7) & ~7
        uw, uh = W >> sx, H >> sy                          # the picture in window units
        cases += [(name, "left", (3, 0, 0, 0)), (name, "top", (0, 0, 5, 0)), (name, "all", (1, 2, 3, 1))]
        if name in ("ctb32", "x_422_basic", "mono10_ctb16_wpp", "x_444_main10_ctb16_random_tskip"):
            cases += [(name, "one_unit", (uw // 2, uw - uw // 2 - 1, uh - 1, 0)), (name, "all_but_one_unit", (1, 0, 0, 1))]
    return cases


CROP_CASES = _crop_cases()


def _cropped(name, win):
    au = windowless(synth_stream(name))
    return au, set_conformance_window(au, *win)


def _expected_window(full, chroma, win):
    sx, sy = sub_wh(chroma)
    l, r, t, b = win
    H, W = full[0].shape
    x0, y0, x1, y1 = l << sx, t << sy, W - (r << sx), H - (b << sy)
    return [a[(y0 >> (sy if c else 0)):(y1 >> (sy if c else 0)), (x0 >> (sx if c else 0)):(x1 >> (sx if c else 0))] for c, a in enumerate(full)]


@pytest.mark.parametrize("name,kind,win", CROP_CASES, ids=[f"{c[0]}-{c[1]}" for c in CROP_CASES])
def test_cropped_stream_on_the_cpu(name, kind, win):
    """the rewritten SPS parses to the new window (host front-end and restatement), and the C restatement's decode of the
    cropped stream is the window of the window-free decode.  FFmpeg is compared only without a left offset: without
    AV_CODEC_FLAG_UNALIGNED it may round a left crop down to keep its planes aligned."""
    from oracle import bindings as ob
    base, au = _cropped(name, win)
    pic = parse_filters(au)
    sx, sy = sub_wh(pic.chroma)
    l, r, t, b = win
    assert pic.window == (l << sx, t << sy, pic.w - ((l + r) << sx), pic.h - ((t + b) << sy))
    full = _oracle(base, 0)
    want = _expected_window(full, pic.chroma, win)
    got = _oracle(au, 0)
    assert [g.shape for g in got] == [w.shape for w in want]
    for c in range(len(want)):
        assert np.array_equal(got[c], want[c]), f"plane {c}"
    if l == 0:
        ff = ob.ffmpeg_decode(au)[0]
        for c in range(len(want)):
            assert np.array_equal(ff[c].astype(np.int64), want[c]), f"FFmpeg plane {c}"


def test_too_large_window_is_refused():
    base = windowless(synth_stream("ctb32"))
    _, w, h, _ = sps_window(base)
    l = _lib.lib()
    hdr = np.zeros(13, np.int32)
    for win in [(w // 4, w // 4, 0, 0), (0, 0, h // 2, 0), (w // 2, 0, 0, 0)]:
        au = set_conformance_window(base, *win)
        assert l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, None, 0, None, 0) == E_BITSTREAM, win
    au = set_conformance_window(base, w // 2 - 1, 0, 0, h // 2 - 1)
    assert l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, None, 0, None, 0) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("front_end", ["device", "host"])
def test_too_large_window_fails_to_decode(cuda, front_end):
    """a window as wide or as high as the picture is a corrupt stream for decode_image too, with either front-end; the
    decoder stays usable"""
    base = windowless(synth_stream("ctb32"))
    _, w, h, _ = sps_window(base)
    d = lb.Decoder(host_threads=4)
    d.set_front_end(front_end == "device")
    try:
        for win in [(w // 4, w // 4, 0, 0), (0, 0, 0, h // 2)]:
            with pytest.raises(lb.B200Error) as e:
                d.decode_image(set_conformance_window(base, *win))
            assert e.value.code == E_BITSTREAM, win
        d.decode_image(base)
        assert np.array_equal(d.planes_host()[0].astype(np.int64), _oracle(base, 0)[0])
    finally:
        d.close()


def test_parse_filters_refuses_bad_arguments():
    au = synth_stream("ctb32")
    l = _lib.lib()
    hdr = np.zeros(13, np.int32)
    small = np.zeros(19, np.int32)
    assert l.b200_debug_parse_filters(None, 0, hdr.ctypes.data, None, 0, None, 0) == E_INVALID
    assert l.b200_debug_parse_filters(au, len(au), None, None, 0, None, 0) == E_INVALID
    assert l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, small.ctypes.data, 1, None, 0) == E_INVALID
    assert l.b200_debug_parse_filters(au, len(au), hdr.ctypes.data, None, 0, small.ctypes.data, 0) == E_INVALID


def test_crop_cases_cover_every_side():
    """left, right, top and bottom offsets at 8 and 10 bits in every chroma format"""
    seen = set()
    for name, _, win in CROP_CASES:
        _, _, _, bd, chroma, _ = next(c for c in SYNTH + SYNTH_CPU_EXTRA if c[0] == name)
        ch = 1 if chroma is True else (0 if chroma is False else chroma)
        for side, v in zip("lrtb", win):
            if v:
                seen.add((side, bd, ch))
    assert {(s, bd, ch) for s in "lrtb" for bd in (8, 10) for ch in range(4)} <= seen


@pytest.mark.gpu
@pytest.mark.parametrize("front_end", ["device", "host"])
def test_cropped_streams_decode(cuda, front_end):
    d = lb.Decoder(host_threads=8)
    d.set_front_end(front_end == "device")
    try:
        for name, kind, win in CROP_CASES:
            base, au = _cropped(name, win)
            d.decode_image(base)
            full = [a.astype(np.int64) for a in d.planes_host()]
            want = _expected_window(full, parse_filters(au).chroma, win)
            d.decode_image(au)
            got = d.planes_host()
            for c in range(len(want)):
                assert np.array_equal(got[c].astype(np.int64), want[c]), f"{name} {kind}: plane {c}"
            ref = _oracle(au, 0)
            for c in range(len(want)):
                assert np.array_equal(ref[c], want[c]), f"{name} {kind}: restatement plane {c}"
    finally:
        d.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name,win", [("ctb32", (3, 1, 2, 3)), ("x_444_basic", (5, 0, 3, 2)), ("main10", (1, 2, 0, 3))])
def test_grid_of_cropped_tiles(cuda, name, win):
    """a 2x2 grid of cropped tiles on a canvas smaller than the grid, to planes and through the fused RGB entry point"""
    from oracle import bindings as ob
    from util import oracle_postprocess
    base, au = _cropped(name, win)
    tile = _oracle(au, 0)
    th, tw = tile[0].shape
    pic = parse_filters(au)
    sx, sy = sub_wh(pic.chroma)
    cw, chh = 2 * tw - (3 << sx), 2 * th - (5 << sy)
    d = lb.Decoder(host_threads=8)
    try:
        d.decode_grid([au] * 4, cols=2, rows=2, canvas=(cw, chh))
        got = d.planes_host()
        want = []
        for c in range(len(tile)):
            ssx, ssy = (sx, sy) if c else (0, 0)
            g = np.tile(tile[c], (2, 2))
            want.append(g[:(chh + ssy) >> ssy, :(cw + ssx) >> ssx])
        for c in range(len(want)):
            assert np.array_equal(got[c].astype(np.int64), want[c]), f"plane {c}"
        bd = pic.bd
        oc = lb.CHROMA_INTERLEAVED_RGB if bd == 8 else lb.CHROMA_INTERLEAVED_RRGGBB_LE
        info = ob.restatement_decode(au)[1]
        rgb, ow, oh = oracle_postprocess(*[a.astype(np.uint16) for a in want], None, pic.chroma, bd, (info["cp"], info["tc"], info["mc"], info["full_range"]), [], oc)
        out = np.empty((oh, ow * (3 if bd == 8 else 6)), np.uint8)
        d.decode_grid_to_rgb_host([au] * 4, 2, 2, oc, canvas=(cw, chh), out=out)
        assert np.array_equal(out.reshape(-1), rgb)
    finally:
        d.close()
