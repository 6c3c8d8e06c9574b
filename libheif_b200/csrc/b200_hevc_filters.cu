// b200_hevc_filters.cu -- K3 deblocking (H.265 8.7.2) and K4 SAO (8.7.3) + K5 conformance crop / tile paste.
//
// The in-loop filters libde265 applies before libheif/plugins/decoder_libde265.cc:97-171 copies the planes out.
// Intra pictures: bS = 2 on every transform edge of the 8x8 grid (host supplies the filterEdgeFlag map and the
// QpY map, one byte per 8x8 block each).  Deblocking runs in place on the reconstruction planes: one pass over all
// vertical edges of all pictures of the batch, then one over all horizontal edges (8.7.2 orders them picture-wide;
// edges of one direction are independent because they are 8 samples apart and touch at most 3 samples per side).
// SAO reads the deblocked planes and writes the final samples straight into the destination (conformance window
// applied, destination pointer already offset to the tile's paste position: K5 folded into K4's store).
#include <algorithm>
#include <cstdlib>
#include "b200_hevc.h"
#include "b200_staging.h"

namespace b200 {

__constant__ uint8_t c_tc[54] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,1,1,1,1,1,1,1,1,1,2,2,2,2,3,3,3,3,4,4,4,5,5,6,6,7,8,9,10,11,13,14,16,18,20,22,24};
__constant__ uint8_t c_beta[52] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,6,7,8,9,10,11,12,13,14,15,16,17,18,20,22,24,26,28,30,32,34,36,38,40,42,44,46,48,50,52,54,56,58,60,62,64};
__constant__ uint8_t c_qpc2[14] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37};

__device__ __forceinline__ int clip3d(int lo, int hi, int v) { return min(max(v, lo), hi); }

// one thread = one 4-sample luma edge segment (+ the 2-sample chroma segments lying on it)
template <typename T, int VERT>
__global__ void __launch_bounds__(256) deblock_kernel(const DeviceBatch b, int max_w8, int max_seg) {
  const PicDesc& pic = b.pics[blockIdx.y];
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  // VERT: edges at x = 8*e, segments along y (4 rows each); else edges at y = 8*e, segments along x
  const int nedge = VERT ? pic.w8 : pic.h8, nseg = (VERT ? pic.height : pic.width) >> 2;
  // consecutive threads walk along the contiguous image direction: edges for the vertical pass, segments for the horizontal one
  const int e = VERT ? idx % max_w8 : idx / max_seg, sg = VERT ? idx / max_w8 : idx % max_seg;
  if (e >= nedge || sg >= nseg || e == 0) return;
  const int x = VERT ? e * 8 : sg * 4, y = VERT ? sg * 4 : e * 8;
  const uint8_t* edge8 = b.edge8 + pic.map8_base;
  const int8_t* qp8 = b.qp8 + pic.map8_base;
  const int bi = (y >> 3) * pic.w8 + (x >> 3);
  if (!(edge8[bi] & (VERT ? 1 : 2))) return;
  const int bj = VERT ? bi - 1 : bi - pic.w8;
  const bool keep_q = edge8[bi] & 4, keep_p = edge8[bj] & 4;       // cu_transquant_bypass, pcm + pcm_loop_filter_disabled: nDq / nDp = 0 (8.7.2.5.7)
  const CtuInfo& ci = b.ctus[pic.ctu_base + (y >> pic.log2_ctb) * pic.wctb + (x >> pic.log2_ctb)];
  const SliceInfo sl = b.slices[pic.slice_base + ci.slice_idx];
  const int bd = pic.bit_depth, maxv = (1 << bd) - 1;
  const int qpl = (qp8[bi] + qp8[bj] + 1) >> 1;
  {
    const int beta = c_beta[clip3d(0, 51, qpl + sl.beta_offset)] * (1 << (bd - 8));
    const int tc = c_tc[clip3d(0, 53, qpl + 2 + sl.tc_offset)] * (1 << (bd - 8));
    T* pl = static_cast<T*>(pic.rec[0]);
    const int st = pic.rec_stride[0];
    const int xs = VERT ? 1 : st, ls = VERT ? st : 1;
    T* q = pl + (size_t)y * st + x;
    int s[4][8];                                        // [line][p3 p2 p1 p0 q0 q1 q2 q3]
#pragma unroll
    for (int l = 0; l < 4; l++)
#pragma unroll
      for (int k = 0; k < 8; k++) s[l][k] = q[(ptrdiff_t)(k - 4) * xs + (ptrdiff_t)l * ls];
#define P_(k, l) s[l][3 - (k)]
#define Q_(k, l) s[l][4 + (k)]
    const int dp0 = abs(P_(2, 0) - 2 * P_(1, 0) + P_(0, 0)), dp3 = abs(P_(2, 3) - 2 * P_(1, 3) + P_(0, 3));
    const int dq0 = abs(Q_(2, 0) - 2 * Q_(1, 0) + Q_(0, 0)), dq3 = abs(Q_(2, 3) - 2 * Q_(1, 3) + Q_(0, 3));
    const int dpq0 = dp0 + dq0, dpq3 = dp3 + dq3, dp = dp0 + dp3, dq = dq0 + dq3;
    if (dpq0 + dpq3 < beta) {                            // 8.7.2.5.3
      const bool s0 = 2 * dpq0 < (beta >> 2) && abs(P_(3, 0) - P_(0, 0)) + abs(Q_(0, 0) - Q_(3, 0)) < (beta >> 3) && abs(P_(0, 0) - Q_(0, 0)) < ((5 * tc + 1) >> 1);
      const bool s3 = 2 * dpq3 < (beta >> 2) && abs(P_(3, 3) - P_(0, 3)) + abs(Q_(0, 3) - Q_(3, 3)) < (beta >> 3) && abs(P_(0, 3) - Q_(0, 3)) < ((5 * tc + 1) >> 1);
      const bool strong = s0 && s3;
      const bool dep = dp < ((beta + (beta >> 1)) >> 3), deq = dq < ((beta + (beta >> 1)) >> 3);
#pragma unroll
      for (int l = 0; l < 4; l++) {                       // 8.7.2.5.7
        const int p0 = P_(0, l), p1 = P_(1, l), p2 = P_(2, l), p3 = P_(3, l), q0 = Q_(0, l), q1 = Q_(1, l), q2 = Q_(2, l), q3 = Q_(3, l);
        T* ql = q + (ptrdiff_t)l * ls;
        if (strong) {
          if (!keep_p) {
            ql[-1 * (ptrdiff_t)xs] = (T)clip3d(p0 - 2 * tc, p0 + 2 * tc, (p2 + 2 * p1 + 2 * p0 + 2 * q0 + q1 + 4) >> 3);
            ql[-2 * (ptrdiff_t)xs] = (T)clip3d(p1 - 2 * tc, p1 + 2 * tc, (p2 + p1 + p0 + q0 + 2) >> 2);
            ql[-3 * (ptrdiff_t)xs] = (T)clip3d(p2 - 2 * tc, p2 + 2 * tc, (2 * p3 + 3 * p2 + p1 + p0 + q0 + 4) >> 3);
          }
          if (!keep_q) {
            ql[0] = (T)clip3d(q0 - 2 * tc, q0 + 2 * tc, (p1 + 2 * p0 + 2 * q0 + 2 * q1 + q2 + 4) >> 3);
            ql[xs] = (T)clip3d(q1 - 2 * tc, q1 + 2 * tc, (p0 + q0 + q1 + q2 + 2) >> 2);
            ql[2 * (ptrdiff_t)xs] = (T)clip3d(q2 - 2 * tc, q2 + 2 * tc, (p0 + q0 + q1 + 3 * q2 + 2 * q3 + 4) >> 3);
          }
        } else {
          int delta = (9 * (q0 - p0) - 3 * (q1 - p1) + 8) >> 4;
          if (abs(delta) < tc * 10) {
            delta = clip3d(-tc, tc, delta);
            if (!keep_p) ql[-1 * (ptrdiff_t)xs] = (T)clip3d(0, maxv, p0 + delta);
            if (!keep_q) ql[0] = (T)clip3d(0, maxv, q0 - delta);
            if (dep && !keep_p) ql[-2 * (ptrdiff_t)xs] = (T)clip3d(0, maxv, p1 + clip3d(-(tc >> 1), tc >> 1, (((p2 + p0 + 1) >> 1) - p1 + delta) >> 1));
            if (deq && !keep_q) ql[xs] = (T)clip3d(0, maxv, q1 + clip3d(-(tc >> 1), tc >> 1, (((q2 + q0 + 1) >> 1) - q1 - delta) >> 1));
          }
        }
      }
    }
#undef P_
#undef Q_
  }
  // chroma: edges on the 8-sample CHROMA grid (every 16 luma samples where the chroma is sub-sampled across the edge), bS == 2 only
  // (8.7.2.5.5 / 8.7.2.5.8); a 4-luma-sample segment covers 4 >> (sub-sampling along the edge) chroma samples
  const int fsx = (pic.chroma == 1 || pic.chroma == 2) ? 1 : 0, fsy = pic.chroma == 1 ? 1 : 0;
  if (pic.chroma && ((VERT ? x : y) & ((8 << (VERT ? fsx : fsy)) - 1)) == 0) {
    const int len = 4 >> (VERT ? fsy : fsx);
    for (int c = 1; c <= 2; c++) {
      const int qpi = qpl + (c == 1 ? pic.pps_cb_qp_offset : pic.pps_cr_qp_offset);
      const int qpc = pic.chroma != 1 ? min(qpi, 51) : (qpi < 30 ? qpi : (qpi >= 43 ? qpi - 6 : c_qpc2[qpi - 30]));   // Table 8-10 only when ChromaArrayType == 1
      const int tc = c_tc[clip3d(0, 53, qpc + 2 + sl.tc_offset)] * (1 << (bd - 8));
      T* pl = static_cast<T*>(pic.rec[c]);
      const int st = pic.rec_stride[c];
      const int xs = VERT ? 1 : st, ls = VERT ? st : 1;
      T* q = pl + (size_t)(y >> fsy) * st + (x >> fsx);
#pragma unroll
      for (int l = 0; l < 4; l++) {
        if (l >= len) break;
        T* ql = q + (ptrdiff_t)l * ls;
        const int p0 = ql[-(ptrdiff_t)xs], p1 = ql[-2 * (ptrdiff_t)xs], q0 = ql[0], q1 = ql[xs];
        const int delta = clip3d(-tc, tc, ((((q0 - p0) << 2) + p1 - q1 + 4) >> 3));
        if (!keep_p) ql[-(ptrdiff_t)xs] = (T)clip3d(0, maxv, p0 + delta);
        if (!keep_q) ql[0] = (T)clip3d(0, maxv, q0 - delta);
      }
    }
  }
}

// SAO offset of ONE sample with every rule of 8.7.3 (picture bounds, slice boundaries with
// slice_loop_filter_across_slices_enabled_flag): the path for pictures with more than one slice.
template <typename T>
__device__ __noinline__ int sao_sample_generic(const DeviceBatch& b, const PicDesc& pic, const CtuInfo* ctus, const T* src, int st, int c, int x, int y, int w, int h, int lg, int lgy) {   // lg / lgy: log2 of the component's CTB width / height
  int v = src[(size_t)y * st + x];
  const CtuInfo& ci = ctus[(y >> lgy) * pic.wctb + (x >> lg)];
  const SaoComp sp = ci.sao[c];
  if (!pic.sao_enabled || !sp.type) return v;
  const int bd = pic.bit_depth, maxv = (1 << bd) - 1;
  int off = 0;
  if (sp.type == 1) {
    const int k = ((v >> (bd - 5)) - sp.band_or_class) & 31;
    if (k < 4) off = sp.offset[k];
  } else {
    const int e = sp.band_or_class;
    const int hx = e == 1 ? 0 : (e == 3 ? 1 : -1), vy = e == 0 ? 0 : -1;      // first neighbour; second is the opposite
    const int xa = x + hx, ya = y + vy, xb = x - hx, yb = y - vy;
    if (xa >= 0 && xb >= 0 && ya >= 0 && yb >= 0 && xa < w && xb < w && ya < h && yb < h) {
      bool skip = false;
      const SliceInfo* sls = b.slices + pic.slice_base;
      const int cur = ci.slice_idx;
      const int sa = ctus[(ya >> lgy) * pic.wctb + (xa >> lg)].slice_idx, sb = ctus[(yb >> lgy) * pic.wctb + (xb >> lg)].slice_idx;
      // 8.7.3.2: a neighbour in another slice counts only if the later of the two slices filters across its boundary; one in another
      // tile only with loop_filter_across_tiles_enabled_flag (regions = slice x tile, compared through their slice / tile ids)
      const SliceInfo c0 = sls[cur];
      if (sa != cur) { const SliceInfo o = sls[sa]; if ((o.slice_id != c0.slice_id && !(o.slice_id < c0.slice_id ? c0.lf_across_slices : o.lf_across_slices)) || (o.tile_id != c0.tile_id && !c0.lf_across_tiles)) skip = true; }
      if (sb != cur) { const SliceInfo o = sls[sb]; if ((o.slice_id != c0.slice_id && !(o.slice_id < c0.slice_id ? c0.lf_across_slices : o.lf_across_slices)) || (o.tile_id != c0.tile_id && !c0.lf_across_tiles)) skip = true; }
      if (!skip) {
        const int a = src[(size_t)ya * st + xa], bb = src[(size_t)yb * st + xb];
        const int ei = 2 + (v > a) - (v < a) + (v > bb) - (v < bb);
        if (ei != 2) off = sp.offset[ei < 2 ? ei : ei - 1];           // edgeIdx 0,1,3,4 -> SaoOffsetVal[1..4]
      }
    }
  }
  return clip3d(0, maxv, v + off);
}

// ---- K4: one thread = 8 horizontally adjacent samples (one SAO unit: always inside one CTB) of FOUR consecutive rows (a
// 4-aligned row group never straddles a CTB either).  All six source rows a thread needs (the row above its group .. the row
// below) are requested up front with 8- / 16-byte loads -- six independent loads in flight per thread instead of a dependent
// chain of three -- and the horizontal neighbours come from the adjacent lanes by shuffle (one warp = 256 consecutive samples
// of a row; only lanes 0 and 31 load their outer neighbour).  The CTB's parameters, the bypass / PCM cell and the picture
// descriptor are fetched once per 32 samples.
// (One row per thread was bound by block turnover and load latency, with 393 K blocks of 2 KB; walking four rows one after
// the other in a rolled loop was slower still.)
template <typename T> struct SaoPack;
template <> struct SaoPack<uint8_t> {
  uint2 q;
  __device__ __forceinline__ void zero() { q = make_uint2(0, 0); }
  __device__ __forceinline__ void load_vec(const uint8_t* p) { q = *reinterpret_cast<const uint2*>(p); }
  __device__ __forceinline__ void load_n(const uint8_t* p, int n) { unsigned long long v = 0; for (int k = 0; k < 8; k++) if (k < n) v |= (unsigned long long)p[k] << (8 * k); q.x = (unsigned)v; q.y = (unsigned)(v >> 32); }
  __device__ __forceinline__ int first() const { return (int)(q.x & 0xffu); }
  __device__ __forceinline__ int last() const { return (int)(q.y >> 24); }
  __device__ __forceinline__ void unpack(int* d) const {
#pragma unroll
    for (int k = 0; k < 4; k++) { d[k] = (int)((q.x >> (8 * k)) & 0xffu); d[4 + k] = (int)((q.y >> (8 * k)) & 0xffu); }
  }
  __device__ __forceinline__ static void store_vec(uint8_t* p, const int* r) {
    uint2 o; o.x = (unsigned)r[0] | ((unsigned)r[1] << 8) | ((unsigned)r[2] << 16) | ((unsigned)r[3] << 24); o.y = (unsigned)r[4] | ((unsigned)r[5] << 8) | ((unsigned)r[6] << 16) | ((unsigned)r[7] << 24);
    *reinterpret_cast<uint2*>(p) = o;
  }
};
template <> struct SaoPack<uint16_t> {
  uint4 q;
  __device__ __forceinline__ void zero() { q = make_uint4(0, 0, 0, 0); }
  __device__ __forceinline__ void load_vec(const uint16_t* p) { q = *reinterpret_cast<const uint4*>(p); }
  __device__ __forceinline__ void load_n(const uint16_t* p, int n) {
    unsigned u[4] = {0, 0, 0, 0};
    for (int k = 0; k < 8; k++) if (k < n) u[k >> 1] |= (unsigned)p[k] << (16 * (k & 1));
    q = make_uint4(u[0], u[1], u[2], u[3]);
  }
  __device__ __forceinline__ int first() const { return (int)(q.x & 0xffffu); }
  __device__ __forceinline__ int last() const { return (int)(q.w >> 16); }
  __device__ __forceinline__ void unpack(int* d) const {
    const unsigned u[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < 4; k++) { d[2 * k] = (int)(u[k] & 0xffffu); d[2 * k + 1] = (int)(u[k] >> 16); }
  }
  __device__ __forceinline__ static void store_vec(uint16_t* p, const int* r) {
    uint4 o; o.x = (unsigned)r[0] | ((unsigned)r[1] << 16); o.y = (unsigned)r[2] | ((unsigned)r[3] << 16); o.z = (unsigned)r[4] | ((unsigned)r[5] << 16); o.w = (unsigned)r[6] | ((unsigned)r[7] << 16);
    *reinterpret_cast<uint4*>(p) = o;
  }
};

// 8-bit samples, four per register (SIMD video instructions): one row of one SAO unit = two words.
// tab_pos / tab_neg: magnitudes of the positive / negative offsets by table index (bytes 0..4; index 2 of the edge table and
// index 4 of the band table are zero), looked up for four samples at once with PRMT.
struct SaoTab8 { unsigned pos_lo, pos_hi, neg_lo, neg_hi; };
__device__ __forceinline__ unsigned sao_apply4(unsigned v, unsigned idx, const SaoTab8& t) {
  // idx: one table index (0..4) per byte -> PRMT selector nibbles
  const unsigned u = idx | (idx >> 4), sel = __byte_perm(u, 0, 0x4420);
  const unsigned pos = __byte_perm(t.pos_lo, t.pos_hi, sel), neg = __byte_perm(t.neg_lo, t.neg_hi, sel);
  return __vsubus4(__vaddus4(v, pos), neg);                     // clip to [0, 255]
}
__device__ __forceinline__ unsigned sao_edge_idx4(unsigned v, unsigned a, unsigned bb) {
  // edgeIdx = 2 + sign(v - a) + sign(v - b) per byte (8.7.3.2); the comparison masks are 0xff = -1
  unsigned ei = __vsub4(0x02020202u, __vcmpgtu4(v, a));
  ei = __vadd4(ei, __vcmpltu4(v, a));
  ei = __vsub4(ei, __vcmpgtu4(v, bb));
  return __vadd4(ei, __vcmpltu4(v, bb));
}

constexpr int SAO_ROWS = 4;
template <typename T>
__global__ void __launch_bounds__(256, 3) sao_rows_kernel(const DeviceBatch b, int c_first, int ncomp) {
  // grid.z = picture x component (c_first .. c_first + ncomp - 1): luma and the two chroma planes are launched apart, each with a
  // grid of its own size (one grid sized for luma left half of all blocks empty: 0.2 ms on the bench grid)
  const int pi = blockIdx.z / ncomp, c = c_first + blockIdx.z % ncomp;
  const PicDesc& pic = b.pics[pi];
  if (c > 0 && !pic.chroma) return;                                                     // (uniform per block)
  const int sh = (c && (pic.chroma == 1 || pic.chroma == 2)) ? 1 : 0, shy = (c && pic.chroma == 1) ? 1 : 0;
  const int w = pic.width >> sh, h = pic.height >> shy;
  const int lane = threadIdx.x;                                                           // blockDim.x == 32: one warp per row group
  const int x0 = (blockIdx.x * 32 + lane) * 8, yb = (blockIdx.y * blockDim.y + threadIdx.y) * SAO_ROWS;
  if (blockIdx.x * 256 >= w || yb >= h) return;                                          // (uniform per warp: every lane stays for the shuffles)
  const bool in = x0 < w;
  const int n = in ? min(8, w - x0) : 0;
  const int cx = pic.crop_x >> sh, cy = pic.crop_y >> shy, ow = (pic.out_w + sh) >> sh, oh = (pic.out_h + shy) >> shy;
  const T* src = static_cast<const T*>(pic.rec[c]);
  const int st = pic.rec_stride[c];
  const int lg = pic.log2_ctb - sh, lgy = pic.log2_ctb - shy;
  const CtuInfo* ctus = b.ctus + pic.ctu_base;
  const int bd = pic.bit_depth, maxv = (1 << bd) - 1;
  T* const dplane = static_cast<T*>(pic.dst[c]);
  const int dst_st = pic.dst_stride[c];
  const int ox0 = x0 - cx;
  if (pic.nslices > 1) {
    // several slices: every sample through the rule-complete path (slice-boundary conditions of 8.7.3.2)
    if (!in) return;
    for (int r = 0; r < SAO_ROWS; r++) {
      const int y = yb + r, oy = y - cy;
      if (y >= h || oy < 0 || oy >= oh) continue;
      const uint8_t* cell = b.edge8 + pic.map8_base + ((y << shy) >> 3) * pic.w8 + ((x0 << sh) >> 3);
      const bool k0 = cell[0] & 4, k1 = sh ? (((x0 + 4) << 1) < pic.width && (cell[1] & 4)) : k0;
      T* drow = dplane + (size_t)oy * dst_st;
      for (int k = 0; k < n; k++) {
        const int v = (k < 4 ? k0 : k1) ? (int)src[(size_t)y * st + x0 + k] : sao_sample_generic<T>(b, pic, ctus, src, st, c, x0 + k, y, w, h, lg, lgy);
        const int ox = ox0 + k;
        if (ox >= 0 && ox < ow) drow[ox] = (T)v;
      }
    }
    return;
  }
  // ---- the six source rows (yb - 1 .. yb + 4), all requested before anything is used
  SaoPack<T> row[SAO_ROWS + 2];
  int hl[SAO_ROWS + 2], hr[SAO_ROWS + 2];                                                // outer neighbours (x0 - 1, x0 + 8) of every row
  const bool has_l = in && x0 > 0, has_r = in && x0 + 8 < w;
#pragma unroll
  for (int j = 0; j < SAO_ROWS + 2; j++) {
    const int y = yb - 1 + j;
    row[j].zero(); hl[j] = 0; hr[j] = 0;
    if (in && y >= 0 && y < h) {
      const T* p = src + (size_t)y * st + x0;
      if (n == 8) row[j].load_vec(p); else row[j].load_n(p, n);
      if (lane == 0 && has_l) hl[j] = (int)p[-1];
      if (lane == 31 && has_r) hr[j] = (int)p[8];
    }
  }
  SaoComp sp{}; bool keep0 = false, keep1 = false;
  if (in) {
    sp = ctus[(yb >> lgy) * pic.wctb + (x0 >> lg)].sao[c];
    // cu_transquant_bypass / pcm + pcm_loop_filter_disabled (8.7.3: SaoTypeIdx is treated as 0 there): bit 2 of the 8x8 luma cells
    // (the four rows of the group lie in one row of cells: 4 rows of luma, or 4 chroma rows = 8 luma rows, 4-aligned)
    const uint8_t* cell = b.edge8 + pic.map8_base + ((yb << shy) >> 3) * pic.w8 + ((x0 << sh) >> 3);
    keep0 = cell[0] & 4; keep1 = sh ? (((x0 + 4) << 1) < pic.width && (cell[1] & 4)) : keep0;
  }
#pragma unroll
  for (int j = 0; j < SAO_ROWS + 2; j++) {
    const int fl = __shfl_up_sync(0xffffffffu, row[j].last(), 1), fr = __shfl_down_sync(0xffffffffu, row[j].first(), 1);
    if (lane != 0) hl[j] = fl;
    if (lane != 31) hr[j] = fr;
  }
  if (!in) return;
  const unsigned offs = (unsigned)(uint8_t)sp.offset[0] | ((unsigned)(uint8_t)sp.offset[1] << 8) | ((unsigned)(uint8_t)sp.offset[2] << 16) | ((unsigned)(uint8_t)sp.offset[3] << 24);
  auto offset = [&](int i) { return (int)(int8_t)(offs >> (8 * i)); };                   // register-resident SaoOffsetVal[1..4]
  const int type = (pic.sao_enabled && sp.type) ? (int)sp.type : 0;
  const int e = sp.band_or_class;
  const int hx = e == 1 ? 0 : (e == 3 ? 1 : -1);
  const bool vert = e != 0;
  // packed tables of the 8-bit SIMD path: |offset| of the positive and of the negative offsets by table index
  SaoTab8 edge_tab{0, 0, 0, 0}, band_tab{0, 0, 0, 0};
  if constexpr (sizeof(T) == 1) {
    unsigned pos = 0, neg = 0;                                                          // byte i: max(offset(i), 0) / max(-offset(i), 0)
#pragma unroll
    for (int i = 0; i < 4; i++) { const int o = offset(i); pos |= (unsigned)(o > 0 ? o : 0) << (8 * i); neg |= (unsigned)(o < 0 ? -o : 0) << (8 * i); }
    band_tab.pos_lo = pos; band_tab.neg_lo = neg;                                        // [o0 o1 o2 o3 | 0]
    edge_tab.pos_lo = (pos & 0xffffu) | ((pos & 0xff0000u) << 8); edge_tab.pos_hi = pos >> 24;   // [o0 o1 0 o2 | o3]
    edge_tab.neg_lo = (neg & 0xffffu) | ((neg & 0xff0000u) << 8); edge_tab.neg_hi = neg >> 24;
  }
#pragma unroll
  for (int r = 0; r < SAO_ROWS; r++) {
    const int y = yb + r, oy = y - cy;
    if (y >= h || oy < 0 || oy >= oh) continue;                                           // outside the picture / the conformance window: never output
    if constexpr (sizeof(T) == 1) {
      {
        // 8-bit samples: four per instruction (a partial unit at the right picture edge is zero-filled beyond its n samples)
        const uint2 cv = row[r + 1].q;
        uint2 out = cv;
        if (type == 1) {
          const unsigned bnd = (unsigned)e * 0x01010101u;
          unsigned k0 = __vsub4((cv.x >> 3) & 0x1f1f1f1fu, bnd) & 0x1f1f1f1fu, k1 = __vsub4((cv.y >> 3) & 0x1f1f1f1fu, bnd) & 0x1f1f1f1fu;
          const unsigned m0 = __vcmpltu4(k0, 0x04040404u), m1 = __vcmpltu4(k1, 0x04040404u);
          k0 = (k0 & m0) | (~m0 & 0x04040404u); k1 = (k1 & m1) | (~m1 & 0x04040404u);
          out.x = sao_apply4(cv.x, k0, band_tab); out.y = sao_apply4(cv.y, k1, band_tab);
        } else if (type == 2 && (!vert || (y > 0 && y + 1 < h))) {
          // neighbour vectors: L = the sample to the left at every position, R = the one to the right
          const uint2 uv = row[r].q, dv = row[r + 2].q;
          uint2 a, bb;
          if (e == 0) {
            a.x = (cv.x << 8) | (unsigned)hl[r + 1]; a.y = __funnelshift_l(cv.x, cv.y, 8);
            bb.x = __funnelshift_r(cv.x, cv.y, 8); bb.y = (cv.y >> 8) | ((unsigned)hr[r + 1] << 24);
          } else if (e == 1) { a = uv; bb = dv; }
          else if (e == 2) {
            a.x = (uv.x << 8) | (unsigned)hl[r]; a.y = __funnelshift_l(uv.x, uv.y, 8);
            bb.x = __funnelshift_r(dv.x, dv.y, 8); bb.y = (dv.y >> 8) | ((unsigned)hr[r + 2] << 24);
          } else {
            a.x = __funnelshift_r(uv.x, uv.y, 8); a.y = (uv.y >> 8) | ((unsigned)hr[r] << 24);
            bb.x = (dv.x << 8) | (unsigned)hl[r + 2]; bb.y = __funnelshift_l(dv.x, dv.y, 8);
          }
          unsigned e0 = sao_edge_idx4(cv.x, a.x, bb.x), e1 = sao_edge_idx4(cv.y, a.y, bb.y);
          if (e != 1) {                                                                   // first / last column of the picture: a neighbour is missing
            if (!has_l) e0 = (e0 & 0xffffff00u) | 0x02u;
            if (!has_r) {                                                                 // the unit's last sample (n - 1) is the picture's last column
              const unsigned sft = 8u * (unsigned)((n - 1) & 3), clr = ~(0xffu << sft), two = 0x02u << sft;
              if (n > 4) e1 = (e1 & clr) | two; else e0 = (e0 & clr) | two;
            }
          }
          out.x = sao_apply4(cv.x, e0, edge_tab); out.y = sao_apply4(cv.y, e1, edge_tab);
        }
        if (keep0) out.x = cv.x;
        if (keep1) out.y = cv.y;
        T* drow8 = dplane + (size_t)oy * dst_st;
        if (n == 8 && ox0 >= 0 && ox0 + 8 <= ow && ((reinterpret_cast<uintptr_t>(drow8 + ox0) & 7) == 0)) *reinterpret_cast<uint2*>(drow8 + ox0) = out;
        else {
#pragma unroll
          for (int k = 0; k < 8; k++) { const int ox = ox0 + k; if (k < n && ox >= 0 && ox < ow) drow8[ox] = (T)(((k < 4 ? out.x : out.y) >> (8 * (k & 3))) & 0xffu); }
        }
      }
    } else {
    int cur[10], res[8];
    row[r + 1].unpack(cur + 1); cur[0] = hl[r + 1]; cur[9] = hr[r + 1];
    if (type == 0) {
#pragma unroll
      for (int k = 0; k < 8; k++) res[k] = cur[1 + k];
    } else if (type == 1) {
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int v = cur[1 + k], kk = ((v >> (bd - 5)) - e) & 31;
        res[k] = clip3d(0, maxv, v + (kk < 4 ? offset(kk) : 0));
      }
    } else {
      int up[10], dn[10];
      if (vert) { row[r].unpack(up + 1); up[0] = hl[r]; up[9] = hr[r]; row[r + 2].unpack(dn + 1); dn[0] = hl[r + 2]; dn[9] = hr[r + 2]; }
      else {
#pragma unroll
        for (int k = 0; k < 10; k++) up[k] = dn[k] = 0;
      }
      const bool rows_ok = !vert || (y > 0 && y + 1 < h);
#pragma unroll
      for (int k = 0; k < 8; k++) {
        const int v = cur[1 + k];
        int off = 0;
        const int xa = x0 + k + hx, xb = x0 + k - hx;
        if (rows_ok && xa >= 0 && xb >= 0 && xa < w && xb < w) {
          const int a_l = vert ? up[k] : cur[k], a_m = up[1 + k], a_r = vert ? up[2 + k] : cur[2 + k];
          const int b_l = vert ? dn[k] : cur[k], b_m = dn[1 + k], b_r = vert ? dn[2 + k] : cur[2 + k];
          const int a = hx < 0 ? a_l : (hx > 0 ? a_r : a_m), bb = hx < 0 ? b_r : (hx > 0 ? b_l : b_m);
          const int ei = 2 + (v > a) - (v < a) + (v > bb) - (v < bb);
          if (ei != 2) off = offset(ei < 2 ? ei : ei - 1);              // edgeIdx 0,1,3,4 -> SaoOffsetVal[1..4]
        }
        res[k] = clip3d(0, maxv, v + off);
      }
    }
    if (keep0 | keep1) {
#pragma unroll
      for (int k = 0; k < 8; k++) if (k < 4 ? keep0 : keep1) res[k] = cur[1 + k];
    }
    // store (conformance window applied; destination already offset to the tile's paste position)
    T* drow = dplane + (size_t)oy * dst_st;
    if (n == 8 && ox0 >= 0 && ox0 + 8 <= ow && ((reinterpret_cast<uintptr_t>(drow + ox0) & (8 * sizeof(T) - 1)) == 0)) SaoPack<T>::store_vec(drow + ox0, res);
    else {
#pragma unroll
      for (int k = 0; k < 8; k++) { const int ox = ox0 + k; if (k < n && ox >= 0 && ox < ow) drow[ox] = (T)res[k]; }
    }
    }   // (samples wider than 8 bits: scalar arithmetic)
  }
}

int launch_deblock(const DeviceBatch& b, const PicDesc* hp, cudaStream_t s) {
  int max_w8 = 0, max_h8 = 0, max_w = 0, max_h = 0; bool any16 = false, any8 = false;
  for (int i = 0; i < b.npics; i++) {
    max_w8 = max(max_w8, hp[i].w8); max_h8 = max(max_h8, hp[i].h8); max_w = max(max_w, hp[i].width); max_h = max(max_h, hp[i].height);
    if (hp[i].bit_depth > 8) any16 = true; else any8 = true;
  }
  if (any16 && any8) return set_error(B200_E_UNSUPPORTED, "a batch must not mix 8-bit and >8-bit pictures");
  if (!b.npics) return B200_OK;
  {
    const int m = max_w8, total = m * (max_h >> 2);
    dim3 grid((total + 255) / 256, b.npics);
    if (any16) deblock_kernel<uint16_t, 1><<<grid, 256, 0, s>>>(b, m, max_h >> 2); else deblock_kernel<uint8_t, 1><<<grid, 256, 0, s>>>(b, m, max_h >> 2);
  }
  {
    const int total = max_h8 * (max_w >> 2);
    dim3 grid((total + 255) / 256, b.npics);
    if (any16) deblock_kernel<uint16_t, 0><<<grid, 256, 0, s>>>(b, max_w8, max_w >> 2); else deblock_kernel<uint8_t, 0><<<grid, 256, 0, s>>>(b, max_w8, max_w >> 2);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "deblock launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

int launch_sao(const DeviceBatch& b, const PicDesc* hp, cudaStream_t s, int* launches) {
  int max_w = 0, max_h = 0, max_cw = 0, max_ch = 0; bool any16 = false;
  for (int i = 0; i < b.npics; i++) {
    max_w = max(max_w, hp[i].width); max_h = max(max_h, hp[i].height); if (hp[i].bit_depth > 8) any16 = true;
    if (hp[i].chroma) { max_cw = max(max_cw, hp[i].width >> (hp[i].chroma != 3 ? 1 : 0)); max_ch = max(max_ch, hp[i].height >> (hp[i].chroma == 1 ? 1 : 0)); }
  }
  if (launches) *launches = 0;
  if (!b.npics) return B200_OK;
  const dim3 block(32, 8);
  const dim3 grid_y((max_w + 255) / 256, (max_h + 8 * SAO_ROWS - 1) / (8 * SAO_ROWS), b.npics);
  if (any16) sao_rows_kernel<uint16_t><<<grid_y, block, 0, s>>>(b, 0, 1); else sao_rows_kernel<uint8_t><<<grid_y, block, 0, s>>>(b, 0, 1);
  if (launches) *launches = 1;
  if (max_cw > 0 && max_ch > 0) {
    const dim3 grid_c((max_cw + 255) / 256, (max_ch + 8 * SAO_ROWS - 1) / (8 * SAO_ROWS), b.npics * 2);
    if (any16) sao_rows_kernel<uint16_t><<<grid_c, block, 0, s>>>(b, 1, 2); else sao_rows_kernel<uint8_t><<<grid_c, block, 0, s>>>(b, 1, 2);
    if (launches) *launches = 2;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "sao launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

}  // namespace b200

// ---- test-only: K3 and K4 on pictures the caller describes (b200_debug_loop_filters)
namespace {
enum { LFP_W, LFP_H, LFP_LOG2_CTB, LFP_BD, LFP_CHROMA, LFP_CB_OFF, LFP_CR_OFF, LFP_SAO, LFP_NSLICES, LFP_CROP_X, LFP_CROP_Y, LFP_OUT_W, LFP_OUT_H,
       LFP_DST_W, LFP_DST_H, LFP_DST_PITCH, LFP_DST_CPITCH, LFP_PASTE_X, LFP_PASTE_Y, LFP_FIELDS };
enum { LFC_SLICE, LFC_SAO, LFC_FIELDS = LFC_SAO + 3 * 6 };
enum { LFS_BETA, LFS_TC, LFS_ACROSS_SLICES, LFS_SLICE_ID, LFS_TILE_ID, LFS_ACROSS_TILES, LFS_FIELDS };
}  // namespace

// b200_debug_loop_filters: the decoder's own launch_deblock (stages bit 0) and launch_sao (bit 1) on a batch of `npics`
// pictures.  Per picture, in batch order:
//   pics[i * 19 ..]: coded width, height (multiples of 8, at most 4096), log2 CTB size (4..6), bit depth (8..12),
//     chroma_format_idc (0..3), pps Cb / Cr QP offsets (-12..12), sample_adaptive_offset_enabled_flag, number of regions,
//     conformance window (crop_x, crop_y, out_w, out_h: luma samples, crop_x / crop_y multiples of SubWidthC / SubHeightC),
//     destination (width, height, luma and chroma pitch in samples) and the paste position of the window in it (multiples
//     of SubWidthC / SubHeightC; the window must fit);
//   qp8 / edge8: the w8 x h8 maps (QpY from -6 * (bit depth - 8) to 51; filterEdgeFlags in bits 0..2 only);
//   ctbs[k * 19 ..]: region index, then type (0..2), band position (0..31) or EO class (0..3) and the four SaoOffsetVal of
//     Y, Cb, Cr (|offset| <= (1 << (Min(bit depth, 10) - 5)) - 1, shifted by bit depth - 10 above 10 bits);
//   regions[k * 6 ..]: beta offset, tc offset (even, -12..12), slice_loop_filter_across_slices_enabled_flag, slice index in
//     decoding order, TileId, loop_filter_across_tiles_enabled_flag (a PPS flag: the same in every region of a picture);
//   planes_in / rec_out: the Y, Cb, Cr planes of the coded size, rows back to back (1 byte per sample at 8 bits, else 2);
//   dst_out: the destination planes, pitch x rows (read only with bit 1).
// The reconstruction planes are laid out as the decoder lays them out (stride (w + 63) & ~63 samples, 256-byte aligned
// planes): K4's vector loads rely on it.  The destination is filled with `sentinel` bytes before K4 runs and returned whole.
// rec_out receives the reconstruction planes after the run (deblocked with bit 0).
extern "C" int b200_debug_loop_filters(int stages, int npics, const int32_t* pics, const int8_t* qp8, const uint8_t* edge8, const int32_t* ctbs,
                                       const int32_t* regions, const void* planes_in, void* rec_out, void* dst_out, int sentinel) {
  using namespace b200;
  if (stages < 1 || stages > 3 || npics < 1 || npics > 256 || !pics || !qp8 || !edge8 || !ctbs || !regions || !planes_in || !rec_out || ((stages & 2) && !dst_out) ||
      sentinel < 0 || sentinel > 255)
    return set_error(B200_E_INVALID, "loop_filters: stages %d, %d pictures, null argument or sentinel %d", stages, npics, sentinel);
  std::vector<PicDesc> hp((size_t)npics);
  std::vector<CtuInfo> ctu;
  std::vector<SliceInfo> sli;
  size_t nmap = 0, in_bytes = 0, rec_bytes = 0, dst_bytes = 0;
  std::vector<size_t> rec_off((size_t)npics * 3), dst_off((size_t)npics * 3);
  bool any8 = false, any16 = false;
  for (int i = 0; i < npics; i++) {
    const int32_t* f = pics + (size_t)i * LFP_FIELDS;
    PicDesc& p = hp[(size_t)i];
    memset(&p, 0, sizeof p);
    const int W = f[LFP_W], H = f[LFP_H], lg = f[LFP_LOG2_CTB], bd = f[LFP_BD], ch = f[LFP_CHROMA];
    if (W < 8 || H < 8 || W > 4096 || H > 4096 || (W & 7) || (H & 7)) return set_error(B200_E_INVALID, "loop_filters: picture %d: size %dx%d", i, W, H);
    if (lg < 4 || lg > 6 || bd < 8 || bd > 12 || ch < 0 || ch > 3) return set_error(B200_E_INVALID, "loop_filters: picture %d: log2 CTB %d, bit depth %d, chroma %d", i, lg, bd, ch);
    if (f[LFP_CB_OFF] < -12 || f[LFP_CB_OFF] > 12 || f[LFP_CR_OFF] < -12 || f[LFP_CR_OFF] > 12 || (f[LFP_SAO] != 0 && f[LFP_SAO] != 1))
      return set_error(B200_E_INVALID, "loop_filters: picture %d: qp offsets %d %d, sao %d", i, f[LFP_CB_OFF], f[LFP_CR_OFF], f[LFP_SAO]);
    const int sx = (ch == 1 || ch == 2) ? 1 : 0, sy = ch == 1 ? 1 : 0;
    const int cx = f[LFP_CROP_X], cy = f[LFP_CROP_Y], ow = f[LFP_OUT_W], oh = f[LFP_OUT_H];
    if (cx < 0 || cy < 0 || ow < 1 || oh < 1 || (cx & sx) || (cy & sy) || (int64_t)cx + ow > W || (int64_t)cy + oh > H)
      return set_error(B200_E_INVALID, "loop_filters: picture %d: conformance window %d,%d %dx%d in %dx%d", i, cx, cy, ow, oh, W, H);
    const int dw = f[LFP_DST_W], dh = f[LFP_DST_H], dp = f[LFP_DST_PITCH], dcp = f[LFP_DST_CPITCH], px = f[LFP_PASTE_X], py = f[LFP_PASTE_Y];
    const int dcw = ch ? (dw + sx) >> sx : 0, dch = ch ? (dh + sy) >> sy : 0;
    if (dw < 1 || dh < 1 || dw > 8192 || dh > 8192 || dp < dw || dp > 8192 || (ch && (dcp < dcw || dcp > 8192)) || px < 0 || py < 0 || (px & sx) || (py & sy) ||
        (int64_t)px + ow > dw || (int64_t)py + oh > dh)
      return set_error(B200_E_INVALID, "loop_filters: picture %d: destination %dx%d pitch %d / %d, paste at %d,%d", i, dw, dh, dp, dcp, px, py);
    const int ns = f[LFP_NSLICES];
    if (ns < 1 || ns > 4096) return set_error(B200_E_INVALID, "loop_filters: picture %d: %d regions", i, ns);
    (bd > 8 ? any16 : any8) = true;
    p.width = W; p.height = H; p.log2_ctb = lg; p.wctb = (W + (1 << lg) - 1) >> lg; p.hctb = (H + (1 << lg) - 1) >> lg;
    p.bit_depth = bd; p.chroma = ch; p.crop_x = cx; p.crop_y = cy; p.out_w = ow; p.out_h = oh;
    p.pps_cb_qp_offset = f[LFP_CB_OFF]; p.pps_cr_qp_offset = f[LFP_CR_OFF]; p.sao_enabled = f[LFP_SAO]; p.nslices = ns;
    p.w8 = W >> 3; p.h8 = H >> 3; p.scaling_idx = -1;
    p.map8_base = (uint32_t)nmap; p.ctu_base = (uint32_t)ctu.size(); p.slice_base = (uint32_t)sli.size();
    const int minqp = -6 * (bd - 8);
    for (size_t k = 0; k < (size_t)p.w8 * p.h8; k++) {
      if (qp8[nmap + k] < minqp || qp8[nmap + k] > 51) return set_error(B200_E_INVALID, "loop_filters: picture %d: QpY %d", i, qp8[nmap + k]);
      if (edge8[nmap + k] & ~7) return set_error(B200_E_INVALID, "loop_filters: picture %d: edge flags %#x", i, edge8[nmap + k]);
    }
    nmap += (size_t)p.w8 * p.h8;
    const int cmax = ((1 << (std::min(bd, 10) - 5)) - 1) << std::max(0, bd - 10);
    for (int k = 0; k < p.wctb * p.hctb; k++) {
      const int32_t* c = ctbs + (ctu.size()) * LFC_FIELDS;
      CtuInfo ci; memset(&ci, 0, sizeof ci);
      if (c[LFC_SLICE] < 0 || c[LFC_SLICE] >= ns) return set_error(B200_E_INVALID, "loop_filters: picture %d: CTB %d: region %d", i, k, c[LFC_SLICE]);
      ci.slice_idx = (uint16_t)c[LFC_SLICE];
      for (int comp = 0; comp < 3; comp++) {
        const int32_t* s = c + LFC_SAO + 6 * comp;
        if (s[0] < 0 || s[0] > 2 || s[1] < 0 || s[1] > (s[0] == 2 ? 3 : 31)) return set_error(B200_E_INVALID, "loop_filters: picture %d: CTB %d: SAO type %d / %d", i, k, s[0], s[1]);
        ci.sao[comp].type = (uint8_t)s[0]; ci.sao[comp].band_or_class = (uint8_t)s[1];
        for (int o = 0; o < 4; o++) {
          if (s[2 + o] < -cmax || s[2 + o] > cmax) return set_error(B200_E_INVALID, "loop_filters: picture %d: CTB %d: SAO offset %d", i, k, s[2 + o]);
          ci.sao[comp].offset[o] = (int8_t)s[2 + o];
        }
      }
      ctu.push_back(ci);
    }
    for (int k = 0; k < ns; k++) {
      const int32_t* r = regions + sli.size() * LFS_FIELDS;
      if (r[LFS_BETA] < -12 || r[LFS_BETA] > 12 || (r[LFS_BETA] & 1) || r[LFS_TC] < -12 || r[LFS_TC] > 12 || (r[LFS_TC] & 1) || (r[LFS_ACROSS_SLICES] & ~1) ||
          r[LFS_SLICE_ID] < 0 || r[LFS_SLICE_ID] > 65535 || r[LFS_TILE_ID] < 0 || r[LFS_TILE_ID] > 65535 || (r[LFS_ACROSS_TILES] & ~1))
        return set_error(B200_E_INVALID, "loop_filters: picture %d: region %d", i, k);
      if (r[LFS_ACROSS_TILES] != regions[(size_t)p.slice_base * LFS_FIELDS + LFS_ACROSS_TILES])   // a PPS flag: one value per picture
        return set_error(B200_E_INVALID, "loop_filters: picture %d: region %d: loop_filter_across_tiles_enabled_flag differs", i, k);
      SliceInfo si; memset(&si, 0, sizeof si);
      si.beta_offset = (int8_t)r[LFS_BETA]; si.tc_offset = (int8_t)r[LFS_TC]; si.lf_across_slices = (uint8_t)r[LFS_ACROSS_SLICES];
      si.slice_id = (uint16_t)r[LFS_SLICE_ID]; si.tile_id = (uint16_t)r[LFS_TILE_ID]; si.lf_across_tiles = (uint8_t)r[LFS_ACROSS_TILES];
      sli.push_back(si);
    }
    const int bps = bd > 8 ? 2 : 1, maxv = (1 << bd) - 1;
    for (int c = 0; c < (ch ? 3 : 1); c++) {
      const int w = c ? W >> sx : W, h = c ? H >> sy : H, st = (w + 63) & ~63;
      if (bps == 2) {
        const uint16_t* s = reinterpret_cast<const uint16_t*>(static_cast<const uint8_t*>(planes_in) + in_bytes);
        for (size_t k = 0; k < (size_t)w * h; k++) if (s[k] > maxv) return set_error(B200_E_INVALID, "loop_filters: picture %d: sample %u above %d", i, s[k], maxv);
      }
      in_bytes += (size_t)w * h * bps;
      p.rec_stride[c] = st; rec_off[(size_t)i * 3 + c] = rec_bytes;
      rec_bytes = (rec_bytes + (size_t)st * h * bps + 255) & ~(size_t)255;
      const int rows = c ? dch : dh, pitch = c ? dcp : dp;
      dst_off[(size_t)i * 3 + c] = dst_bytes;
      p.dst_stride[c] = pitch;
      dst_bytes += (size_t)pitch * rows * bps;
    }
  }
  if (any8 && any16 && !(stages & 1)) return set_error(B200_E_UNSUPPORTED, "a batch must not mix 8-bit and >8-bit pictures");
  DevBuf<PicDesc> d_pics; DevBuf<CtuInfo> d_ctu; DevBuf<SliceInfo> d_sli; DevBuf<int8_t> d_qp; DevBuf<uint8_t> d_edge, d_rec, d_dst;
  int rc = 0;
  if ((rc = d_pics.reserve((size_t)npics, false)) || (rc = d_ctu.reserve(ctu.size(), false)) || (rc = d_sli.reserve(sli.size(), false)) || (rc = d_qp.reserve(nmap, false)) ||
      (rc = d_edge.reserve(nmap, false)) || (rc = d_rec.reserve(rec_bytes, false)) || (rc = d_dst.reserve(dst_bytes + 1, false)))
    return rc;
  for (int i = 0; i < npics; i++) {
    PicDesc& p = hp[(size_t)i];
    const int sx = (p.chroma == 1 || p.chroma == 2) ? 1 : 0, sy = p.chroma == 1 ? 1 : 0, bps = p.bit_depth > 8 ? 2 : 1;
    const int32_t* f = pics + (size_t)i * LFP_FIELDS;
    for (int c = 0; c < (p.chroma ? 3 : 1); c++) {
      p.rec[c] = d_rec.d + rec_off[(size_t)i * 3 + c];
      const int px = c ? f[LFP_PASTE_X] >> sx : f[LFP_PASTE_X], py = c ? f[LFP_PASTE_Y] >> sy : f[LFP_PASTE_Y];
      p.dst[c] = d_dst.d + dst_off[(size_t)i * 3 + c] + ((size_t)py * p.dst_stride[c] + px) * bps;
    }
  }
  size_t in_pos = 0;
  for (int i = 0; i < npics; i++) {
    const PicDesc& p = hp[(size_t)i];
    const int sx = (p.chroma == 1 || p.chroma == 2) ? 1 : 0, sy = p.chroma == 1 ? 1 : 0, bps = p.bit_depth > 8 ? 2 : 1;
    for (int c = 0; c < (p.chroma ? 3 : 1); c++) {
      const int w = c ? p.width >> sx : p.width, h = c ? p.height >> sy : p.height;
      B200_CUDA_CHECK(cudaMemcpy2D(p.rec[c], (size_t)p.rec_stride[c] * bps, static_cast<const uint8_t*>(planes_in) + in_pos, (size_t)w * bps, (size_t)w * bps, h, cudaMemcpyHostToDevice));
      in_pos += (size_t)w * h * bps;
    }
  }
  B200_CUDA_CHECK(cudaMemcpy(d_pics.d, hp.data(), hp.size() * sizeof(PicDesc), cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_ctu.d, ctu.data(), ctu.size() * sizeof(CtuInfo), cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_sli.d, sli.data(), sli.size() * sizeof(SliceInfo), cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_qp.d, qp8, nmap, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_edge.d, edge8, nmap, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemset(d_dst.d, sentinel, dst_bytes + 1));
  DeviceBatch b{};
  b.pics = d_pics.d; b.npics = npics; b.ctus = d_ctu.d; b.slices = d_sli.d; b.qp8 = d_qp.d; b.edge8 = d_edge.d;
  b.wide_samples = any16 ? 1 : 0;
  if ((stages & 1) && (rc = launch_deblock(b, hp.data(), nullptr))) return rc;
  if ((stages & 2) && (rc = launch_sao(b, hp.data(), nullptr))) return rc;
  B200_CUDA_CHECK(cudaDeviceSynchronize());
  size_t out_pos = 0;
  for (int i = 0; i < npics; i++) {
    const PicDesc& p = hp[(size_t)i];
    const int sx = (p.chroma == 1 || p.chroma == 2) ? 1 : 0, sy = p.chroma == 1 ? 1 : 0, bps = p.bit_depth > 8 ? 2 : 1;
    for (int c = 0; c < (p.chroma ? 3 : 1); c++) {
      const int w = c ? p.width >> sx : p.width, h = c ? p.height >> sy : p.height;
      B200_CUDA_CHECK(cudaMemcpy2D(static_cast<uint8_t*>(rec_out) + out_pos, (size_t)w * bps, p.rec[c], (size_t)p.rec_stride[c] * bps, (size_t)w * bps, h, cudaMemcpyDeviceToHost));
      out_pos += (size_t)w * h * bps;
    }
  }
  if (stages & 2) B200_CUDA_CHECK(cudaMemcpy(dst_out, d_dst.d, dst_bytes, cudaMemcpyDeviceToHost));
  return B200_OK;
}
