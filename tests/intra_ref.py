"""Intra prediction restated from the text of H.265, in plain Python / numpy, for the tests of the encoders' prediction
primitives (test_transform_stage.py) and of the decoder's reconstruction kernel K1 (test_intra_prediction.py):
- 8.4.4.2.2 - 8.4.4.2.6: reference substitution, filtering of the neighbours and the 35 prediction modes;
- 6.5.1 / 6.5.2 / 6.4.1: CTB raster-to-tile scan, the z-scan order of minimum blocks and the availability of a neighbour;
- 8.4.4.2.2's marking of the 4n + 1 neighbouring samples of a block, vectorised over blocks and samples.
Nothing here follows the kernel's shortcuts (morton codes, runs of available samples, lane layouts)."""
import numpy as np

# ------------------------------------------------------------------------------------------ prediction (8.4.4.2.2 - 8.4.4.2.6)
ANGLE = [0, 0, 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32, -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32]
INV_ANGLE = {11: -4096, 12: -1638, 13: -910, 14: -630, 15: -482, 16: -390, 17: -315, 18: -256, 19: -315, 20: -390, 21: -482, 22: -630,
             23: -910, 24: -1638, 25: -4096}


def to_xy(r, n):
    """r[0 .. 4n] (r[2n - 1 - y] = p[-1][y], r[2n] = p[-1][-1], r[2n + 1 + x] = p[x][-1]) -> (left[y], corner, top[x])."""
    r = [int(v) for v in r]
    return [r[2 * n - 1 - y] for y in range(2 * n)], r[2 * n], [r[2 * n + 1 + x] for x in range(2 * n)]


def to_r(left, corner, top):
    return list(reversed(left)) + [corner] + list(top)


def substitute(r, n, bd):
    """8.4.4.2.2, walking p[-1][2n - 1] up to p[-1][-1], then p[0][-1] .. p[2n - 1][-1]."""
    seq = list(r)                     # already in that order
    if all(v < 0 for v in seq):
        return [1 << (bd - 1)] * len(seq)
    if seq[0] < 0:
        seq[0] = next(v for v in seq if v >= 0)
    for i in range(1, len(seq)):
        if seq[i] < 0:
            seq[i] = seq[i - 1]
    return seq


def filtered(r, n, bd, strong):
    """8.4.4.2.3 filtering process of the neighbours (both filters, regardless of filterFlag)."""
    left, c, top = to_xy(r, n)
    if strong and n == 32 and abs(c + top[2 * n - 1] - 2 * top[n - 1]) < (1 << (bd - 5)) and abs(c + left[2 * n - 1] - 2 * left[n - 1]) < (1 << (bd - 5)):
        fl = [((63 - y) * c + (y + 1) * left[63] + 32) >> 6 for y in range(63)] + [left[63]]
        ft = [((63 - x) * c + (x + 1) * top[63] + 32) >> 6 for x in range(63)] + [top[63]]
        return to_r(fl, c, ft)
    fc = (left[0] + 2 * c + top[0] + 2) >> 2
    fl = [(left[y + 1] + 2 * left[y] + (left[y - 1] if y else c) + 2) >> 2 for y in range(2 * n - 1)] + [left[2 * n - 1]]
    ft = [((top[x - 1] if x else c) + 2 * top[x] + top[x + 1] + 2) >> 2 for x in range(2 * n - 1)] + [top[2 * n - 1]]
    return to_r(fl, fc, ft)


def filter_flag(plane, mode, n):
    if not plane or mode == 1 or n == 4:
        return False
    return min(abs(mode - 26), abs(mode - 10)) > {8: 7, 16: 1, 32: 0}[n]


def predict(r, f, n, mode, luma, plane, bd):
    """8.4.4.2.4 - 8.4.4.2.6: the n x n prediction [y][x] from the substituted neighbours r (f: filtered)."""
    lg = n.bit_length() - 1
    left, c, top = to_xy(f if filter_flag(plane, mode, n) else r, n)
    P = lambda x, y: c if x < 0 and y < 0 else (left[y] if x < 0 else top[x])   # noqa: E731
    maxv = (1 << bd) - 1
    out = np.zeros((n, n), np.int64)
    if mode == 0:
        for y in range(n):
            for x in range(n):
                out[y, x] = ((n - 1 - x) * P(-1, y) + (x + 1) * P(n, -1) + (n - 1 - y) * P(x, -1) + (y + 1) * P(-1, n) + n) >> (lg + 1)
        return out
    if mode == 1:
        dc = (sum(P(x, -1) for x in range(n)) + sum(P(-1, y) for y in range(n)) + n) >> (lg + 1)
        out[:] = dc
        if luma and n < 32:
            out[0, 0] = (P(-1, 0) + 2 * dc + P(0, -1) + 2) >> 2
            for x in range(1, n):
                out[0, x] = (P(x, -1) + 3 * dc + 2) >> 2
            for y in range(1, n):
                out[y, 0] = (P(-1, y) + 3 * dc + 2) >> 2
        return out
    ang = ANGLE[mode]
    ref = {}
    if mode >= 18:
        for x in range(n + 1):
            ref[x] = P(-1 + x, -1)
        if ang < 0:
            if (n * ang) >> 5 < -1:
                for x in range((n * ang) >> 5, 0):
                    ref[x] = P(-1, -1 + ((x * INV_ANGLE[mode] + 128) >> 8))
        else:
            for x in range(n + 1, 2 * n + 1):
                ref[x] = P(-1 + x, -1)
        for y in range(n):
            idx, fact = ((y + 1) * ang) >> 5, ((y + 1) * ang) & 31
            for x in range(n):
                out[y, x] = ((32 - fact) * ref[x + idx + 1] + fact * ref[x + idx + 2] + 16) >> 5 if fact else ref[x + idx + 1]
        if mode == 26 and luma and n < 32:
            for y in range(n):
                out[y, 0] = min(max(P(0, -1) + ((P(-1, y) - P(-1, -1)) >> 1), 0), maxv)
    else:
        for x in range(n + 1):
            ref[x] = P(-1, -1 + x)
        if ang < 0:
            if (n * ang) >> 5 < -1:
                for x in range((n * ang) >> 5, 0):
                    ref[x] = P(-1 + ((x * INV_ANGLE[mode] + 128) >> 8), -1)
        else:
            for x in range(n + 1, 2 * n + 1):
                ref[x] = P(-1, -1 + x)
        for x in range(n):
            idx, fact = ((x + 1) * ang) >> 5, ((x + 1) * ang) & 31
            for y in range(n):
                out[y, x] = ((32 - fact) * ref[y + idx + 1] + fact * ref[y + idx + 2] + 16) >> 5 if fact else ref[y + idx + 1]
        if mode == 10 and luma and n < 32:
            for x in range(n):
                out[0, x] = min(max(P(-1, 0) + ((P(x, -1) - P(-1, -1)) >> 1), 0), maxv)
    return out


# ------------------------------------------------------------------------------------------ scan orders (6.5.1, 6.5.2)
def tile_boundaries_from_ids(tile_id):
    """colBd / rowBd (6.5.1) of a picture from its TileId per CTB (raster, hctb x wctb): a new tile column starts wherever
    the TileId of the first CTB row changes, a new tile row wherever that of the first CTB column does."""
    t = np.asarray(tile_id)
    cols = [0] + [x for x in range(1, t.shape[1]) if t[0, x] != t[0, x - 1]] + [t.shape[1]]
    rows = [0] + [y for y in range(1, t.shape[0]) if t[y, 0] != t[y - 1, 0]] + [t.shape[0]]
    return cols, rows


def ctb_addr_rs_to_ts(wctb, hctb, col_bd=None, row_bd=None):
    """CtbAddrRsToTs[] and TileId[] (indexed by raster address) of 6.5.1 for tile column / row boundaries colBd / rowBd
    (each list starts with 0 and ends with the picture size in CTBs; None: one tile)."""
    col_bd = col_bd or [0, wctb]
    row_bd = row_bd or [0, hctb]
    rs2ts = np.zeros(wctb * hctb, np.int64)
    tile = np.zeros(wctb * hctb, np.int64)
    for rs in range(wctb * hctb):
        tbx, tby = rs % wctb, rs // wctb
        tx = max(i for i in range(len(col_bd) - 1) if tbx >= col_bd[i])
        ty = max(j for j in range(len(row_bd) - 1) if tby >= row_bd[j])
        v = 0
        for i in range(tx):
            v += (row_bd[ty + 1] - row_bd[ty]) * (col_bd[i + 1] - col_bd[i])
        for j in range(ty):
            v += wctb * (row_bd[j + 1] - row_bd[j])
        v += (tby - row_bd[ty]) * (col_bd[tx + 1] - col_bd[tx]) + tbx - col_bd[tx]
        rs2ts[rs] = v
        tile[rs] = ty * (len(col_bd) - 1) + tx
    assert sorted(rs2ts.tolist()) == list(range(wctb * hctb))
    return rs2ts, tile


def min_tb_addr_zs(w, h, log2ctb, rs2ts):
    """MinTbAddrZs[y][x] of 6.5.2 over the luma picture (w x h samples), for minimum blocks of 4 x 4 luma samples.

    4 x 4 is exact whatever log2_min_luma_transform_block_size a stream uses: every transform block (and every chroma block,
    scaled to luma) starts on a multiple of 4 luma samples, so two locations share a 4 x 4 address only inside one 4 x 4
    square, which never holds both a block's first sample and one of its neighbours.  Where the spec's coarser array gives
    two such locations the same address (availability TRUE), the 4 x 4 one orders them as their blocks are decoded."""
    wctb = -(-w >> log2ctb)
    w4, h4 = -(-w >> 2), -(-h >> 2)
    y, x = np.mgrid[0:h4, 0:w4]
    ctb_rs = (y >> (log2ctb - 2)) * wctb + (x >> (log2ctb - 2))
    a = np.asarray(rs2ts)[ctb_rs] << (2 * (log2ctb - 2))
    for i in range(log2ctb - 2):
        m = 1 << i
        a = a + np.where(x & m, m * m, 0) + np.where(y & m, 2 * m * m, 0)
    return a


class PicCtx:
    """What 6.4.1 needs of a picture: its luma size, CTB size, and per CTB (raster) SliceAddrRs and TileId."""

    def __init__(self, w, h, log2ctb, slice_addr, tile_id=None, col_bd=None, row_bd=None):
        self.w, self.h, self.lg = w, h, log2ctb
        self.wctb, self.hctb = -(-w >> log2ctb), -(-h >> log2ctb)
        self.rs2ts, tid = ctb_addr_rs_to_ts(self.wctb, self.hctb, col_bd, row_bd)
        self.slice_addr = np.asarray(slice_addr, np.int64).reshape(-1)
        self.tile_id = tid if tile_id is None else np.asarray(tile_id, np.int64).reshape(-1)
        self.zs = min_tb_addr_zs(w, h, log2ctb, self.rs2ts)

    def available(self, xc, yc, xn, yn):
        """6.4.1 for current luma locations (xc, yc) and neighbouring luma locations (xn, yn) (broadcast arrays)."""
        xc, yc, xn, yn = np.broadcast_arrays(*(np.asarray(v, np.int64) for v in (xc, yc, xn, yn)))
        inside = (xn >= 0) & (yn >= 0) & (xn < self.w) & (yn < self.h)
        xs, ys = np.where(inside, xn, 0), np.where(inside, yn, 0)
        later = self.zs[ys >> 2, xs >> 2] > self.zs[yc >> 2, xc >> 2]
        cn = (ys >> self.lg) * self.wctb + (xs >> self.lg)
        cc = (yc >> self.lg) * self.wctb + (xc >> self.lg)
        same = (self.slice_addr[cn] == self.slice_addr[cc]) & (self.tile_id[cn] == self.tile_id[cc])
        return inside & ~later & same


def neighbour_offsets(n):
    """(x, y) of r[0 .. 4n] relative to the block: r[2n - 1 - y] = p[-1][y], r[2n] = p[-1][-1], r[2n + 1 + x] = p[x][-1]."""
    i = np.arange(4 * n + 1)
    x = np.where(i < 2 * n, -1, i - 2 * n - 1)
    y = np.where(i < 2 * n, 2 * n - 1 - i, -1)
    return x, y


def mark_neighbours(ctx, sub_w, sub_h, xc, yc, n):
    """8.4.4.2.2: availability of the 4n + 1 neighbouring samples of blocks of one size n in a component with
    SubWidthC = sub_w, SubHeightC = sub_h at component locations (xc[k], yc[k]): a (len(xc), 4n + 1) bool array in r order.
    The current location is the luma location (xTbCmp * SubWidthC, yTbCmp * SubHeightC), the neighbour that of each
    sample the same way -- so the chroma block of a 4 x 4 luma unit, which sits at the parent 8 x 8 origin, and the lower
    block of a 4:2:2 chroma unit are judged from their own position."""
    xc, yc = np.asarray(xc, np.int64)[:, None], np.asarray(yc, np.int64)[:, None]
    ox, oy = neighbour_offsets(n)
    return ctx.available(xc * sub_w, yc * sub_h, (xc + ox[None, :]) * sub_w, (yc + oy[None, :]) * sub_h)
