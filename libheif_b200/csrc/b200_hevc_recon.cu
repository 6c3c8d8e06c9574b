// b200_hevc_recon.cu -- K1 + K2: scaling, inverse DCT/DST, intra prediction and reconstruction on sm_90a.
//
// Does the per-sample half of what libde265 does inside de265_decode() (reached from
// libheif/plugins/decoder_libde265.cc:386-457): H.265 8.6.2-8.6.4 (scaling, transforms), 8.4.4.2 (intra sample
// prediction incl. reference substitution and smoothing), 8.6.6 (reconstruction), driven by the command stream
// of the entropy stage (b200_hevc_types.h).
//
// Work item = (picture, CTB row, component group): luma, or the Cb + Cr pair.  Chroma prediction never reads luma, so the
// two groups are independent wavefronts; Cb and Cr share position, size, mode and availability, so one warp does both at
// once on its two half-warps.  ONE WARP walks the CTBs of its row left to right; rows advance as a wavefront with a lag
// of two CTBs (above-right dependency) through per-(row, group) progress counters.  A global ticket hands items out in
// "row k of every picture" order, so a dependency always holds a smaller ticket (no co-residency requirement).
//
// Per CTB the warp works in two phases:
//   A. residual phase, lane-parallel over the CTB's transform units (no dependency between them): every lane decodes
//      one TuCmd, derives the neighbour availability of its block (6.4.1, z-scan order) into a packed descriptor, and
//      -- 4x4 blocks being 80 % of all blocks of a typical intra picture -- dequantises and inverse-transforms its own
//      4x4 block entirely in registers (32 blocks per pass).  Larger blocks (8..32) are done by the whole warp, one at a
//      time, with zero-row/column skipping.  Residuals land in shared memory, block-contiguous in z-order.
//   B. prediction phase, block after block (the intra dependency chain): one gather of the 4n+1 neighbours with the
//      substitution process (8.4.4.2.2) folded into the index computation, optional smoothing, prediction, residual
//      add, store into the CTB tile in shared memory.  ~100 warp instructions per block instead of ~900.
// The finished CTB leaves shared memory with one cp.async.bulk (TMA) row copy per lane; the halo (row above incl.
// above-right, column to the left) is kept in shared memory next to the tile.  Integer work: no tensor cores.
#include "b200_hevc.h"
#include "b200_staging.h"

namespace b200 {

#ifndef B200_RECON_MIN_BLOCKS
#define B200_RECON_MIN_BLOCKS 5
#endif
constexpr int WARPS = 4;                       // warps (= work items in flight) per CTA
constexpr int PAD = 16;                        // samples left of the tile / halo row: column PAD - 1 is the left halo
// Transposed DCT matrices MT_n[y][k] = transMatrix_n[k][y] for n = 32, 16, 8 (rows padded by 4 bytes: lanes that read different
// rows hit different banks), shared by the CTA: 32 x 36 + 16 x 20 + 8 x 12 bytes
constexpr int MT32_OFF = 0, MT16_OFF = 32 * 36, MT8_OFF = MT16_OFF + 16 * 20;
constexpr int MAT_BYTES = MT8_OFF + 8 * 12;
constexpr int REF_STRIDE = 136;                // int16 entries per neighbour array (4 * 32 + 1 rounded up)

struct WarpLayout { int tile, top, res, tmp, desc, total; };     // byte offsets inside the warp's shared-memory slice
__host__ __device__ inline WarpLayout warp_layout(int log2ctb, int bps) {
  const int ctb = 1 << log2ctb, tb = ctb < 32 ? ctb : 32;
  WarpLayout L; int o = 0;
  L.tile = o; o += ctb * (ctb + PAD) * bps;                      // luma tile; the Cb + Cr tiles of a chroma item fit inside
  L.top = o; o += (2 * PAD + 2 * ctb + 32) * bps;                // halo row(s)
  o = (o + 15) & ~15;
  L.res = o; o += ctb * ctb * 2;                                 // residuals, int16, z-order block-contiguous
  L.tmp = o; o += (tb * (tb + 2) * 2 > 1024 ? tb * (tb + 2) * 2 : 1024);   // first-stage output (rows padded by 2) / 4x4 scratch / neighbour arrays
  L.desc = o; o += (ctb / 4) * (ctb / 4) * 8;                    // one descriptor per transform block of the CTB
  L.total = (o + 15) & ~15;
  return L;
}

__constant__ int8_t c_dct[32] = {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67,
                                 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4};
__constant__ int8_t c_angle[35] = {0, 0, 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                   -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32};
__constant__ int16_t c_inv_angle[35] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, -4096, -1638, -910, -630, -482, -390, -315, -256,
                                        -315, -390, -482, -630, -910, -1638, -4096, 0, 0, 0, 0, 0, 0, 0, 0, 0};
__constant__ uint8_t c_qpc[14] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37};
__constant__ uint8_t c_level_scale[6] = {40, 45, 51, 57, 64, 72};

__host__ __device__ __forceinline__ int clip3i(int lo, int hi, int v) { return min(max(v, lo), hi); }
__host__ __device__ __forceinline__ unsigned morton4(unsigned x, unsigned y) {   // z-order index of a 4x4 block inside a CTB
  unsigned sx = (x & 1) | ((x & 2) << 1) | ((x & 4) << 2) | ((x & 8) << 3);
  unsigned sy = (y & 1) | ((y & 2) << 1) | ((y & 4) << 2) | ((y & 8) << 3);
  return sx | (sy << 1);
}
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// TMA (bulk asynchronous copy) of one finished tile row: shared -> global.  Source and destination 16-byte aligned, size a
// multiple of 16.
__device__ __forceinline__ void bulk_store(void* g, const void* s, unsigned bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(g), "r"((unsigned)__cvta_generic_to_shared(s)), "r"(bytes) : "memory");
}

// Command-stream reads.  LIVE = K0 is running concurrently: a neighbouring, not yet written entry may share a cache
// line with one read earlier and L1 is not coherent, so everything goes to L2 (ld.global.cg).  Otherwise the command
// stream is complete and plain loads let consecutive entries hit the L1 line the first one brought in.
template <bool LIVE, class T> __device__ __forceinline__ T ld_cmd(const T* p) { return LIVE ? __ldcg(p) : *p; }
template <bool LIVE> __device__ __forceinline__ TuCmd ld_tu(const TuCmd* p) { const uint4 v = ld_cmd<LIVE>(reinterpret_cast<const uint4*>(p)); return TuCmd{v.x, v.y, v.z, v.w}; }
template <bool LIVE> __device__ __forceinline__ CoefEntry ld_coef(const CoefEntry* p) { const unsigned v = ld_cmd<LIVE>(reinterpret_cast<const unsigned*>(p)); CoefEntry e; e.pos = (uint16_t)(v & 0xffff); e.level = (int16_t)(v >> 16); return e; }
template <bool LIVE> __device__ __forceinline__ CtuInfo ld_ctu(const CtuInfo* p) {
  CtuInfo c; const uint2* s = reinterpret_cast<const uint2*>(p); uint2* d = reinterpret_cast<uint2*>(&c);
#pragma unroll
  for (int i = 0; i < (int)(sizeof(CtuInfo) / 8); i++) d[i] = ld_cmd<LIVE>(s + i);
  return c;
}

__host__ __device__ __forceinline__ int chroma_qp(int qpy, int off, int bd, int cfmt = 1) {       // 8.6.1: Table 8-10 when ChromaArrayType == 1, else Min(qPi, 51)
#ifndef __CUDA_ARCH__
  static const uint8_t c_qpc[14] = {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37};   // the host's copy of the table
#endif
  const int qbd = 6 * (bd - 8);
  const int qpi = clip3i(-qbd, 57, qpy + off);
  const int qpc = cfmt != 1 ? min(qpi, 51) : (qpi < 30 ? qpi : (qpi >= 43 ? qpi - 6 : c_qpc[qpi - 30]));
  return qpc + qbd;
}

// 8.6.3 / 8.6.4.2 scaling: TransCoeffLevel -> d, clipped to 16 bits; m = 16 (flat) or the scaling factor of the position
__device__ __forceinline__ int dequant(int level, int qp, int bd_shift, int m) {
  const long long scale = (long long)(c_level_scale[qp % 6] << (qp / 6)) * m;
  const long long t = ((long long)level * scale + (1LL << (bd_shift - 1))) >> bd_shift;
  return (int)(t < -32768 ? -32768 : (t > 32767 ? 32767 : t));
}

// Descriptor of one transform block, built in phase A, consumed in phase B (uint2):
//  x: bx/4 [0:4) by/4 [4:8) log2n-2 [8:10) mode [10:16) coded [16] (Cr: [17]) availL [18] availCorner [19] availTop [20]
//     available below-left samples / 4 [21:25)  available above-right samples / 4 [25:29)  pcm [29]: the "residuals" are the samples
//  y: offset of the block's residuals inside the component's residual area (samples)
// (tw, th: the component's CTB size; shx: its horizontal sub-sampling when the decoding order inside the CTB has to be judged in
//  LUMA units -- the 4:2:2 chroma planes, whose blocks follow the z-order of the luma quadtree, not of their own coordinates)
__host__ __device__ __forceinline__ unsigned make_desc(int bx, int by, int lg, int mode, int coded0, int coded1, int tw, int th, int shx, int cx0, int cy0, int cw, int ch,
                                              bool nbL, bool nbAL, bool nbA, bool nbAR) {
  const int n = 1 << lg;
  const bool fL = bx > 0 || nbL, fT = by > 0 || nbA;
  const bool fC = (bx > 0 && by > 0) ? true : (bx > 0 ? nbA : (by > 0 ? nbL : nbAL));
  const unsigned me = morton4((unsigned)(bx << shx) >> 2, (unsigned)by >> 2);
  bool tr = false, bl = false;
  if (cx0 + bx + n < cw) {
    if (by > 0) { if (bx + n < tw) tr = morton4((unsigned)((bx + n) << shx) >> 2, (unsigned)(by - 1) >> 2) < me; }
    else tr = (bx + n < tw) ? nbA : nbAR;
  }
  if (cy0 + by + n < ch && by + n < th) {
    if (bx > 0) bl = morton4((unsigned)((bx - 1) << shx) >> 2, (unsigned)(by + n) >> 2) < me; else bl = nbL;
  }
  const int trc = tr ? min(n, cw - (cx0 + bx + n)) : 0, blc = bl ? min(n, ch - (cy0 + by + n)) : 0;
  return (unsigned)(bx >> 2) | ((unsigned)(by >> 2) << 4) | ((unsigned)(lg - 2) << 8) | ((unsigned)mode << 10) | ((unsigned)coded0 << 16) | ((unsigned)coded1 << 17) |
         ((unsigned)fL << 18) | ((unsigned)fC << 19) | ((unsigned)fT << 20) | ((unsigned)(blc >> 2) << 21) | ((unsigned)(trc >> 2) << 25);
}

// Phase A's derivation, shared by K1 and the host descriptor export (b200_debug_k1_descriptors), so that the export runs K1's own
// code.  Macros rather than functions: every function form of this code, even a one-line inline helper, changed ptxas's register
// allocation of K1 (more spills); the expansions are token for token the code K1 had inline.
//
// B200_K1_CTB_NEIGHBOURS(REGION): the CTB-level availability nbL / nbAL / nbA / nbAR -- the left / above-left / above / above-right
// CTB holds the current CTB's region (one slice inside one tile, b200_hevc_types.h).  Expands where rx, ry, addr (raster address),
// wctb and cur (the CTB's region index) are defined; REGION(a) is the region index of the CTB at raster address a.
#define B200_K1_CTB_NEIGHBOURS(REGION)                                                  \
  const bool nbL = rx > 0 && REGION(addr - 1) == cur;                                   \
  const bool nbAL = rx > 0 && ry > 0 && REGION(addr - wctb - 1) == cur;                 \
  const bool nbA = ry > 0 && REGION(addr - wctb) == cur;                                \
  const bool nbAR = ry > 0 && rx + 1 < wctb && REGION(addr - wctb + 1) == cur;
// B200_K1_TB_OF_CMD: one lane's TuCmd `cmd` (valid: the lane holds one) in component group g of the CTB at luma (x0, y0) -> has, the
// block's position bx, by in the component's CTB, log2 size lg, mode, coded0 / coded1 (Cb / Cr in the pair), pcm, and what the
// residual needs (qp0 / qp1, ts0 / ts1, ce / ce1, n0 / n1, raw).  Not paired: a luma block, or (4:2:2 / 4:4:4) the block of plane
// `pl`, the commands of the other planes skipped; paired: the 4:2:0 Cb + Cr blocks (those of a 4x4 luma unit at the parent 8x8
// origin).  A lane without a block gets an uncoded 4x4 block at (0, 0).  Expands where cmd, valid, paired, pl, shx, x0, y0, bd,
// cfmt, sl (SliceInfo) and coefs are defined.
#define B200_K1_TB_OF_CMD                                                                                                                  \
  const int log2n = 2 + (int)((cmd.w0 >> 24) & 3);                                                                                         \
  const int lx = (int)((cmd.w0 & 0xfff) << 2) - x0, ly = (int)(((cmd.w0 >> 12) & 0xfff) << 2) - y0;                                        \
  const int qpy = (int)((cmd.w1 >> 12) & 0xff) - 64;                                                                                       \
  const bool pcm = (cmd.w1 >> 21) & 1, raw = ((cmd.w1 >> 21) & 3) != 0;                                                                    \
  const int nl = (int)(cmd.w3 & 0x7ff), ncb = (int)((cmd.w3 >> 11) & 0x3ff), ncr = (int)((cmd.w3 >> 21) & 0x3ff);                          \
  const CoefEntry* ce = coefs + cmd.w2;                                                                                                    \
  bool has; int bx, by, lg, mode, coded0, coded1, qp0, qp1 = 0, ts0, ts1 = 0, n0, n1 = 0; const CoefEntry* ce1 = ce;                       \
  if (!paired) {                                                                                                                           \
    has = valid && (int)((cmd.w1 >> 23) & 3) == pl;                                                                                        \
    bx = lx >> shx; by = ly; lg = log2n; mode = (int)(cmd.w1 & 63); coded0 = (int)((cmd.w0 >> 26) & 1); coded1 = 0;                        \
    qp0 = pl == 0 ? qpy + 6 * (bd - 8) : chroma_qp(qpy, pl == 1 ? sl.cb_qp_offset : sl.cr_qp_offset, bd, cfmt);                           \
    ts0 = (int)((cmd.w0 >> 30) & 1); n0 = nl;                                                                                              \
  } else {                                                                                                                                 \
    has = valid && ((cmd.w0 >> 29) & 1);                                                                                                   \
    if (log2n > 2) { bx = lx >> 1; by = ly >> 1; lg = log2n - 1; } else { bx = (lx - 4) >> 1; by = (ly - 4) >> 1; lg = 2; }               \
    mode = (int)((cmd.w1 >> 6) & 63); coded0 = (int)((cmd.w0 >> 27) & 1); coded1 = (int)((cmd.w0 >> 28) & 1);                             \
    qp0 = chroma_qp(qpy, sl.cb_qp_offset, bd); qp1 = chroma_qp(qpy, sl.cr_qp_offset, bd);                                                  \
    ts0 = (int)((cmd.w0 >> 31) & 1); ts1 = (int)((cmd.w1 >> 20) & 1);                                                                      \
    ce = ce + nl; n0 = ncb; ce1 = ce + ncb; n1 = ncr;                                                                                      \
  }                                                                                                                                        \
  if (!has) { coded0 = coded1 = 0; bx = by = 0; lg = 2; }                                                                                  \
  coded0 = coded0 && n0 > 0; coded1 = coded1 && n1 > 0;
// B200_K1_DESC: the descriptor word of that block (after B200_K1_TB_OF_CMD and B200_K1_CTB_NEIGHBOURS; tw, th, cx0, cy0, cw, ch: the
// component's CTB size, CTB origin and plane size).  The 4:2:0 pair is judged in its own coordinates (shx 0), a 4:2:2 plane in luma
// units.
#define B200_K1_DESC (make_desc(bx, by, lg, mode, coded0, coded1, tw, th, paired ? 0 : shx, cx0, cy0, cw, ch, nbL, nbAL, nbA, nbAR) | ((unsigned)pcm << 29))

// ---- phase A, 4x4 blocks: the calling lane owns the block.  scr: the warp's [16][32] int16 scratch (column = lane).
template <bool LIVE>
__device__ __forceinline__ void residual4_lane(int16_t* scr, int lane, const CoefEntry* __restrict__ ce, int nnz, int qp, int bd, bool dst, bool tskip, bool raw, int16_t* out,
                                               const uint8_t* __restrict__ sf) {      // raw: cu_transquant_bypass / pcm, the levels ARE the residuals (8.6.2)      // sf: the 16 scaling factors of this component (raster), or nullptr
  int16_t* my = scr + lane;
#pragma unroll
  for (int p = 0; p < 16; p++) my[p * 32] = 0;
  const int bd_shift = bd - 3;                        // bd + log2(4) - 5
#pragma unroll 1
  for (int i = 0; i < nnz; i++) {
    const CoefEntry e = ld_coef<LIVE>(&ce[i]);
    my[(e.pos & 15) * 32] = raw ? e.level : (int16_t)dequant(e.level, qp, bd_shift, sf ? (int)__ldg(sf + (e.pos & 15)) : 16);
  }
  int c[16];
#pragma unroll
  for (int p = 0; p < 16; p++) c[p] = my[p * 32];
  const int bs2 = 20 - bd, rnd = 1 << (bs2 - 1);
  unsigned* o32 = reinterpret_cast<unsigned*>(out);
  if (raw) {
#pragma unroll
    for (int p = 0; p < 16; p += 2) o32[p >> 1] = (unsigned)(c[p] & 0xffff) | ((unsigned)c[p + 1] << 16);
    return;
  }
  if (tskip) {                                        // 8.6.4.2, transform_skip_flag: r = d << 7
#pragma unroll
    for (int p = 0; p < 16; p += 2) {
      const int r0 = ((c[p] << 7) + rnd) >> bs2, r1 = ((c[p + 1] << 7) + rnd) >> bs2;
      o32[p >> 1] = (unsigned)(r0 & 0xffff) | ((unsigned)r1 << 16);
    }
    return;
  }
  // coefficient c[k * 4 + x] (k: vertical frequency).  First stage (columns): t[x][y] = clip16((sum_k c[k][x] * M[k][y] + 64) >> 7)
  int t[16];
#pragma unroll
  for (int x = 0; x < 4; x++) {
    const int c0 = c[x], c1 = c[4 + x], c2 = c[8 + x], c3 = c[12 + x];
    int e0, e1, e2, e3;
    if (dst) {                                        // DST-VII (8.6.4.2): M = {29 55 74 84; 74 74 0 -74; 84 -29 -74 55; 55 -84 74 -29}
      e0 = 29 * c0 + 74 * c1 + 84 * c2 + 55 * c3; e1 = 55 * c0 + 74 * c1 - 29 * c2 - 84 * c3;
      e2 = 74 * c0 - 74 * c2 + 74 * c3;           e3 = 84 * c0 - 74 * c1 + 55 * c2 - 29 * c3;
    } else {                                          // DCT-II: M = {64 64 64 64; 83 36 -36 -83; 64 -64 -64 64; 36 -83 83 -36}
      const int a = 64 * (c0 + c2), b = 64 * (c0 - c2), o0 = 83 * c1 + 36 * c3, o1 = 36 * c1 - 83 * c3;
      e0 = a + o0; e1 = b + o1; e2 = b - o1; e3 = a - o0;
    }
    t[x * 4 + 0] = clip3i(-32768, 32767, (e0 + 64) >> 7); t[x * 4 + 1] = clip3i(-32768, 32767, (e1 + 64) >> 7);
    t[x * 4 + 2] = clip3i(-32768, 32767, (e2 + 64) >> 7); t[x * 4 + 3] = clip3i(-32768, 32767, (e3 + 64) >> 7);
  }
  // second stage (rows): r[y][x] = (sum_k t[k][y] * M[k][x] + rnd) >> bs2
#pragma unroll
  for (int y = 0; y < 4; y++) {
    const int c0 = t[y], c1 = t[4 + y], c2 = t[8 + y], c3 = t[12 + y];
    int e0, e1, e2, e3;
    if (dst) {
      e0 = 29 * c0 + 74 * c1 + 84 * c2 + 55 * c3; e1 = 55 * c0 + 74 * c1 - 29 * c2 - 84 * c3;
      e2 = 74 * c0 - 74 * c2 + 74 * c3;           e3 = 84 * c0 - 74 * c1 + 55 * c2 - 29 * c3;
    } else {
      const int a = 64 * (c0 + c2), b = 64 * (c0 - c2), o0 = 83 * c1 + 36 * c3, o1 = 36 * c1 - 83 * c3;
      e0 = a + o0; e1 = b + o1; e2 = b - o1; e3 = a - o0;
    }
    const int r0 = (e0 + rnd) >> bs2, r1 = (e1 + rnd) >> bs2, r2 = (e2 + rnd) >> bs2, r3 = (e3 + rnd) >> bs2;
    o32[y * 2] = (unsigned)(r0 & 0xffff) | ((unsigned)r1 << 16);
    o32[y * 2 + 1] = (unsigned)(r2 & 0xffff) | ((unsigned)r3 << 16);
  }
}

// ---- phase A, 8x8 .. 32x32 blocks: the whole warp, in place in the block's residual slot (coefficients -> residuals).
// COPY: the same code in an out-of-line function of its own for the test harness (k1_residual_kernel): a second caller of K1's
// copy changes how ptxas allocates K1's registers around the call.
template <bool LIVE, int COPY = 0>
__device__ __noinline__ void residual_big(int16_t* rs, int16_t* tmp, const int8_t* __restrict__ mat, const CoefEntry* __restrict__ ce, int nnz, int lg, int qp, int bd, int lane,
                                          const uint8_t* __restrict__ sf, int sf_dc, bool raw) {   // sf: 8x8 raster scaling factors of (component, size) or nullptr; sf_dc: factor of position (0, 0) for 16x16 / 32x32
  const int n = 1 << lg;
  unsigned* z = reinterpret_cast<unsigned*>(rs);
#pragma unroll 1
  for (int i = lane; i < n * n / 2; i += 32) z[i] = 0;
  __syncwarp();
  const int bd_shift = bd + lg - 5;
  int maxrow = 0, maxcol = 0;
  // coefficients are scattered TRANSPOSED (column x of the block = row x of the buffer): the first transform stage runs down the
  // columns, and with the vertical frequencies k of a column adjacent in memory two of them ride in one register (dp2a)
#pragma unroll 1
  for (int i = lane; i < nnz; i += 32) {
    const CoefEntry e = ld_coef<LIVE>(&ce[i]);
    const int pos = e.pos & (n * n - 1);
    const int x = pos & (n - 1), y = pos >> lg;
    int m = 16;
    if (sf) m = (pos == 0 && lg >= 4) ? sf_dc : (int)__ldg(sf + ((y >> (lg - 3)) << 3) + (x >> (lg - 3)));
    rs[raw ? pos : x * n + y] = raw ? e.level : (int16_t)dequant(e.level, qp, bd_shift, m);
    maxrow = max(maxrow, y); maxcol = max(maxcol, x);
  }
  maxrow = __reduce_max_sync(0xffffffffu, maxrow); maxcol = __reduce_max_sync(0xffffffffu, maxcol);
  __syncwarp();
  if (raw) return;                                    // cu_transquant_bypass / pcm (warp-uniform): no scaling, no transform
  const int8_t* mt = mat + (lg == 5 ? MT32_OFF : (lg == 4 ? MT16_OFF : MT8_OFF));
  const int ms = n + 4, P2 = n + 2;                   // row strides: matrix (bytes), intermediate (int16)
  const int kq1 = (maxrow >> 2) + 1, ncol = ((maxcol >> 2) + 1) << 2;     // groups of 4 vertical frequencies; columns, rounded up to 4 (the extra ones are zero)
  // first stage (columns): u[y][x] = clip16((sum_k coef[k][x] * M[k][y] + 64) >> 7), only columns that hold coefficients
#pragma unroll 1
  for (int i = lane; i < n * ncol; i += 32) {
    const int y = i & (n - 1), x = i >> lg;
    const int2* c = reinterpret_cast<const int2*>(rs + x * n);
    const int* mq = reinterpret_cast<const int*>(mt + y * ms);
    int e = 0;
#pragma unroll 2
    for (int q = 0; q < kq1; q++) { const int2 a = c[q]; const int bq = mq[q]; e = __dp2a_lo(a.x, bq, e); e = __dp2a_hi(a.y, bq, e); }
    tmp[y * P2 + x] = (int16_t)clip3i(-32768, 32767, (e + 64) >> 7);
  }
  __syncwarp();
  // second stage (rows): residual r[y][x] = (sum_k u[y][k] * M[k][x] + rnd) >> bs2
  const int bs2 = 20 - bd, rnd = 1 << (bs2 - 1), kq2 = ncol >> 2;
#pragma unroll 1
  for (int p = lane; p < n * n; p += 32) {
    const int x = p & (n - 1), y = p >> lg;
    const int* u = reinterpret_cast<const int*>(tmp + y * P2);
    const int* mq = reinterpret_cast<const int*>(mt + x * ms);
    int e = 0;
#pragma unroll 2
    for (int q = 0; q < kq2; q++) { const int bq = mq[q]; e = __dp2a_lo(u[2 * q], bq, e); e = __dp2a_hi(u[2 * q + 1], bq, e); }
    // the residual itself is unbounded (8.6.4.2) and reaches 61312 at 12 bits / 8x8 and 59584 at 10 bits / 32x32; any value
    // past 16 bits is beyond maxv, so saturating it leaves Clip1(pred + r) of 8.6.7 exact
    rs[p] = (int16_t)clip3i(-32768, 32767, (e + rnd) >> bs2);
  }
  __syncwarp();
}

// The transposed DCT matrices of the CTA (MT32_OFF, MT16_OFF, MT8_OFF), built by threads tid = 0, stride, 2 * stride, ...;
// the caller synchronises before reading them
__device__ void build_dct_matrices(int8_t* mat, int tid, int stride) {
  for (int i = tid; i < 1024 + 256 + 64; i += stride) {
    const int lg = i < 1024 ? 5 : (i < 1280 ? 4 : 3), j0 = i < 1024 ? i : (i < 1280 ? i - 1024 : i - 1280);
    const int n = 1 << lg, y = j0 >> lg, kn = j0 & (n - 1), k = kn << (5 - lg);     // row kn of the n-point matrix = row kn << (5 - log2 n) of the 32-point one
    int v;
    if (k == 0) v = 64;
    else { int j = (k * (2 * y + 1)) & 127, sgn = 1; if (j > 64) j = 128 - j; if (j > 32) { j = 64 - j; sgn = -1; } v = sgn * c_dct[j]; }
    mat[(lg == 5 ? MT32_OFF : (lg == 4 ? MT16_OFF : MT8_OFF)) + y * (n + 4) + kn] = (int8_t)v;
  }
}

// ---- phase B: one transform block (of one component, or of Cb and Cr on the two half-warps).
//  tl: the lane's component tile (row stride S, sample (x, y) at tl[y * S + PAD + x]), tp: its halo row (sample x at
//  tp[PAD + x]), rs: its residual area, rf: its neighbour array(s), l / lpc: lane index inside / lanes per component,
//  gmask: the lanes working on this component.
template <typename P>
__device__ __forceinline__ void predict_tb(const uint2 d, P* tl, const P* tp, const int16_t* rs, int16_t* rf, int S, int l, int lpc, unsigned gmask, int cidx, bool luma, bool smooth, int bd, int strong_en) {   // luma: boundary filters of DC / horizontal / vertical (cIdx == 0); smooth: 8.4.4.2.3 applies (luma; chroma in 4:4:4)
  const int bx = (int)(d.x & 15) << 2, by = (int)((d.x >> 4) & 15) << 2, lg = 2 + (int)((d.x >> 8) & 3), mode = (int)((d.x >> 10) & 63);
  const int n = 1 << lg, n2 = 2 * n, n4 = 4 * n;
  const bool coded = (d.x >> (16 + cidx)) & 1, pcm = (d.x >> 29) & 1;
  const bool fL = (d.x >> 18) & 1, fC = (d.x >> 19) & 1, fT = (d.x >> 20) & 1;
  const int blc = (int)((d.x >> 21) & 15) << 2, trc = (int)((d.x >> 25) & 15) << 2;
  // ---- neighbour array rf[0 .. 4n]: index 0 = bottom of the below-left column ... 2n = corner ... 4n = end of above-right.
  // Substitution (8.4.4.2.2) = every unavailable index reads the nearest available index below it, or the first available
  // one; the available indices form up to five intervals known per block, so the source index is a handful of min / compare.
  const int first = blc ? n - blc : (fL ? n : (fC ? n2 : (fT ? n2 + 1 : (trc ? 3 * n + 1 : -1))));
  const P* colL = tl + by * S + PAD + bx - 1;                          // left column: sample y at colL[y * S]
  const P* rowA = (by > 0 ? tl + (by - 1) * S : tp) + PAD + bx;        // row above: sample x at rowA[x] (x = -1: corner)
  int dcs = 0;
  const bool small = n4 < lpc;                                         // 4x4 on a full warp: the corner rides in the same pass
  const int jn = small ? n4 + 1 : n4;
#pragma unroll 1
  for (int j = l; j < jn; j += lpc) {
    const int i = j == n4 ? n2 : (j < n2 ? j : j + 1);
    int v = 1 << (bd - 1);
    if (first >= 0) {
      int s = first;
      if (blc && i >= n - blc) s = min(i, n - 1);
      if (fL && i >= n) s = min(i, n2 - 1);
      if (fC && i >= n2) s = n2;
      if (fT && i > n2) s = min(i, 3 * n);
      if (trc && i > 3 * n) s = min(i, 3 * n + trc);
      v = s < n2 ? (int)colL[(n2 - 1 - s) * S] : (int)rowA[s - n2 - 1];
    }
    rf[i] = (int16_t)v;
    if ((i >= n && i < n2) || (i > n2 && i <= 3 * n)) dcs += v;
  }
  if (!small && l == 0) {                                               // corner (index 2n) for blocks that fill every lane
    int v = 1 << (bd - 1);
    if (first >= 0) {
      int s = first;
      if (blc) s = n - 1;
      if (fL) s = n2 - 1;
      if (fC) s = n2;
      v = s < n2 ? (int)colL[(n2 - 1 - s) * S] : (int)rowA[s - n2 - 1];
    }
    rf[n2] = (int16_t)v;
  }
  __syncwarp();
  // ---- smoothing of the neighbours (8.4.4.2.3): luma only in 4:2:0
  const int16_t* ref = rf;
  if (smooth && mode != 1 && n != 4) {
    const int dist = min(abs(mode - 26), abs(mode - 10));
    const int thr = n == 8 ? 7 : (n == 16 ? 1 : 0);
    if (dist > thr) {
      const int corner = rf[n2], bl = rf[0], tr = rf[n4];
      const bool strong = strong_en && n == 32 && abs(corner + tr - 2 * rf[3 * n]) < (1 << (bd - 5)) && abs(corner + bl - 2 * rf[n]) < (1 << (bd - 5));
      int16_t* rb = rf + REF_STRIDE;
#pragma unroll 1
      for (int i = l; i <= n4; i += lpc) {
        int v;
        if (i == 0 || i == n4) v = rf[i];
        else if (strong) {
          if (i == n2) v = corner;
          else if (i < n2) { const int y = n2 - 1 - i; v = ((63 - y) * corner + (y + 1) * bl + 32) >> 6; }
          else { const int x = i - n2 - 1; v = ((63 - x) * corner + (x + 1) * tr + 32) >> 6; }
        } else v = (rf[i - 1] + 2 * rf[i] + rf[i + 1] + 2) >> 2;
        rb[i] = (int16_t)v;
      }
      __syncwarp();
      ref = rb;
    }
  }
  // ---- prediction (8.4.4.2.4 - 8.4.4.2.6) + residual (8.6.6), written straight into the tile
  const int maxv = (1 << bd) - 1;
#define LEFT(y) ((int)ref[n2 - 1 - (y)])
#define TOP(x) ((int)ref[n2 + 1 + (x)])
  int dc = 0;
  if (mode == 1) dc = (__reduce_add_sync(gmask, dcs) + n) >> (lg + 1);
  const int ang = c_angle[mode], ia = c_inv_angle[mode];
  const bool edge = luma && n < 32;
  const int16_t* rsb = rs + d.y;
  P* out = tl + by * S + PAD + bx;
#pragma unroll 1
  for (int e = l; e < n * n; e += lpc) {
    const int x = e & (n - 1), y = e >> lg;
    int v;
    if (pcm) { out[y * S + x] = (P)rsb[e]; continue; }                   // 8.4.4.1: no prediction
    if (mode == 0) v = ((n - 1 - x) * LEFT(y) + (x + 1) * TOP(n) + (n - 1 - y) * TOP(x) + (y + 1) * LEFT(n) + n) >> (lg + 1);
    else if (mode == 1) {
      v = dc;
      if (edge) {
        if (x == 0 && y == 0) v = (LEFT(0) + 2 * dc + TOP(0) + 2) >> 2;
        else if (y == 0) v = (TOP(x) + 3 * dc + 2) >> 2;
        else if (x == 0) v = (LEFT(y) + 3 * dc + 2) >> 2;
      }
    } else if (mode >= 18) {
      const int idx = ((y + 1) * ang) >> 5, f = ((y + 1) * ang) & 31;
      const int k0 = x + idx + 1, k1 = k0 + 1;      // r[k] = p[-1 + k][-1] for k >= 0, projected left column for k < 0
      const int a = k0 >= 0 ? TOP(k0 - 1) : LEFT(-1 + ((k0 * ia + 128) >> 8));
      if (f) { const int b = k1 >= 0 ? TOP(k1 - 1) : LEFT(-1 + ((k1 * ia + 128) >> 8)); v = ((32 - f) * a + f * b + 16) >> 5; } else v = a;
      if (mode == 26 && edge && x == 0) v = clip3i(0, maxv, TOP(0) + ((LEFT(y) - LEFT(-1)) >> 1));
    } else {
      const int idx = ((x + 1) * ang) >> 5, f = ((x + 1) * ang) & 31;
      const int k0 = y + idx + 1, k1 = k0 + 1;
      const int a = k0 >= 0 ? LEFT(k0 - 1) : TOP(-1 + ((k0 * ia + 128) >> 8));
      if (f) { const int b = k1 >= 0 ? LEFT(k1 - 1) : TOP(-1 + ((k1 * ia + 128) >> 8)); v = ((32 - f) * a + f * b + 16) >> 5; } else v = a;
      if (mode == 10 && edge && y == 0) v = clip3i(0, maxv, LEFT(0) + ((TOP(x) - TOP(-1)) >> 1));
    }
    if (coded) v = clip3i(0, maxv, v + (int)rsb[e]);
    out[y * S + x] = (P)v;
  }
#undef LEFT
#undef TOP
  __syncwarp();
}

template <typename P, bool LIVE>
__global__ void __launch_bounds__(WARPS * 32, B200_RECON_MIN_BLOCKS) hevc_recon_kernel(const DeviceBatch b) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  int8_t* mat = reinterpret_cast<int8_t*>(smem_raw);                       // the transposed DCT matrices, shared by the CTA
  build_dct_matrices(mat, threadIdx.x, blockDim.x);
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const WarpLayout L = warp_layout(b.max_log2_ctb, (int)sizeof(P));
  unsigned char* wb = smem_raw + MAT_BYTES + (threadIdx.x >> 5) * L.total;
  P* const tile0 = reinterpret_cast<P*>(wb + L.tile);
  P* const top0 = reinterpret_cast<P*>(wb + L.top);
  int16_t* const res0 = reinterpret_cast<int16_t*>(wb + L.res);
  int16_t* const tmp = reinterpret_cast<int16_t*>(wb + L.tmp);
  uint2* const desc = reinterpret_cast<uint2*>(wb + L.desc);
  const unsigned lt_mask = (1u << lane) - 1u;

  for (;;) {
    unsigned t = 0;
    if (lane == 0) t = atomicAdd(b.ticket, 1u);
    t = __shfl_sync(0xffffffffu, t, 0);
    if (t >= (unsigned)b.nrows) break;
    const uint2 pr = b.row_list[t];
    const PicDesc* pic = &b.pics[pr.x];
    // g = 0: luma; 1: Cb + Cr of a 4:2:0 picture on the two half-warps; 2 / 3: the Cb / Cr plane of a 4:2:2 or 4:4:4 picture, handled
    // like luma (full warp, its own commands: b200_hevc_syntax.h transform_unit_x)
    const int g = (int)(pr.y >> 30), ry = (int)(pr.y & 0x3fffffffu);
    const int pl = g >= 2 ? g - 1 : 0;                                      // plane of a luma-like item
    const int cfmt = pic->chroma;
    const int shx = g == 0 ? 0 : (g == 1 ? 1 : (cfmt == 2 ? 1 : 0)), shy = g == 1 ? 1 : 0;
    const bool paired = g == 1;
    const CtuInfo* ctus = b.ctus + pic->ctu_base;
    const SliceInfo* slices = b.slices + pic->slice_base;
    const int log2ctb = pic->log2_ctb, wctb = pic->wctb, bd = pic->bit_depth, strong_en = pic->strong_intra;
    const int tw = (1 << log2ctb) >> shx, th = (1 << log2ctb) >> shy, S = tw + PAD;   // component CTB size, tile row stride
    const int cw = pic->width >> shx, ch = pic->height >> shy;
    const int y0 = ry << log2ctb, cy0 = y0 >> shy;
    const uint8_t* sfac = pic->scaling_idx >= 0 ? b.scaling + (size_t)pic->scaling_idx * 784 : nullptr;      // sl::Factors: m[3][4][64], dc[3][4]
    const TuCmd* tus = b.tus + pic->tu_base;
    const CoefEntry* coefs = b.coefs + pic->coef_base;
    unsigned* prog = b.progress + 3 * pic->progress_base + (g == 3 ? 2 : (g ? 1 : 0));   // counter of (row r, item kind) at prog[3 * r]
    const unsigned* eprog = b.entropy_progress ? b.entropy_progress + pic->progress_base : nullptr;
    // lane roles in phase B
    const int lpc = paired ? 16 : 32, l = lane & (lpc - 1), cidx = paired ? lane >> 4 : 0;
    const unsigned gmask = paired ? (0xffffu << (16 * cidx)) : 0xffffffffu;
    P* const tl = tile0 + cidx * (th * S);
    P* const tp = top0 + cidx * (PAD + 2 * tw + 16);
    int16_t* const rs = res0 + cidx * (tw * th);
    int16_t* const rf = tmp + cidx * REF_STRIDE;
    const int plane = paired ? 1 + cidx : pl;
    P* const recp = static_cast<P*>(pic->rec[plane]);
    const int rst = pic->rec_stride[plane];

    for (int rx = 0; rx < wctb; rx++) {
      const int x0 = rx << log2ctb, cx0 = x0 >> shx;
      // (1) with K0 running concurrently: this CTB's commands must have been published.  Relaxed polling loads (no L1
      // invalidation) with microsecond back-off: waiting rows must not flood L2 with polls.
      if (eprog) {
        int abort = 0;
        if (lane == 0) {
          unsigned spins = 0, ns = 250;
          while (ld_acquire(&eprog[ry]) < (unsigned)(rx + 1)) {
            __nanosleep(ns); if (ns < 8000) ns <<= 1;
            if ((++spins & 31u) == 0 && ld_acquire(b.error_flag)) break;            // K0 failed (corrupt stream): its progress will never come
            if (spins > (1u << 23)) { atomicExch(b.error_flag, 1u); break; }       // ~1 min; turns a would-be hang into an error
          }
          abort = ld_acquire(b.error_flag) != 0u;
        }
        if (__shfl_sync(0xffffffffu, abort, 0)) return;
      }
      const int addr = ry * wctb + rx;
      const CtuInfo ci = ld_ctu<LIVE>(&ctus[addr]);
      const int cur = ci.slice_idx;
#define B200_K1_REGION(a) (int)ld_cmd<LIVE>(&ctus[a].slice_idx)
      B200_K1_CTB_NEIGHBOURS(B200_K1_REGION)
#undef B200_K1_REGION
      const SliceInfo sl = slices[cur];
      // ---- phase A: descriptors + residuals, lane-parallel over the CTB's transform units
      int ntb = 0;
#pragma unroll 1
      for (unsigned base = 0; base < ci.tu_count; base += 32) {
        const bool valid = base + lane < ci.tu_count;
        TuCmd cmd{0, 0, 0, 0};
        if (valid) cmd = ld_tu<LIVE>(&tus[ci.tu_start + base + lane]);
        B200_K1_TB_OF_CMD
        const unsigned hb = __ballot_sync(0xffffffffu, has);
        const int idx = ntb + __popc(hb & lt_mask);
        const unsigned roff = morton4((unsigned)bx >> 2, (unsigned)by >> 2) * 16;
        if (has) desc[idx] = make_uint2(B200_K1_DESC, roff);
        ntb += __popc(hb);
        // 4x4 blocks: one lane each, in registers
        if (lg == 2) {
#pragma unroll 1
          for (int c2 = 0; c2 < 2; c2++)
            if (c2 ? coded1 : coded0)
              residual4_lane<LIVE>(tmp, lane, c2 ? ce1 : ce, c2 ? n1 : n0, c2 ? qp1 : qp0, bd, g == 0, c2 ? ts1 : ts0, raw, res0 + (c2 ? tw * th : 0) + roff,
                                   sfac ? sfac + (paired ? 1 + c2 : pl) * 256 : nullptr);
        }
        __syncwarp();
        // larger blocks: the whole warp, one block at a time
        unsigned big0 = __ballot_sync(0xffffffffu, lg > 2 && coded0), big1 = __ballot_sync(0xffffffffu, lg > 2 && coded1);
#pragma unroll 1
        for (int c2 = 0; c2 < 2; c2++) {
          unsigned m = c2 ? big1 : big0;
          while (m) {
            const int src = __ffs(m) - 1; m &= m - 1;
            const unsigned long long cp = __shfl_sync(0xffffffffu, (unsigned long long)(c2 ? ce1 : ce), src);
            const int nn = __shfl_sync(0xffffffffu, c2 ? n1 : n0, src), lgg = __shfl_sync(0xffffffffu, lg, src), qq = __shfl_sync(0xffffffffu, c2 ? qp1 : qp0, src);
            const unsigned ro = __shfl_sync(0xffffffffu, roff, src); const bool rw = __shfl_sync(0xffffffffu, (int)raw, src) != 0;
            residual_big<LIVE>(res0 + (c2 ? tw * th : 0) + ro, tmp, mat, reinterpret_cast<const CoefEntry*>(cp), nn, lgg, qq, bd, lane,
                               sfac ? sfac + (paired ? 1 + c2 : pl) * 256 + (lgg - 2) * 64 : nullptr, sfac ? (int)sfac[768 + (paired ? 1 + c2 : pl) * 4 + (lgg - 2)] : 16, rw);
          }
        }
      }
      __syncwarp();
      // (2) wavefront: the above-right CTB of this component group must be reconstructed (lag 2)
      if (ry > 0) {
        int abort = 0;
        if (lane == 0) {
          const unsigned need = (unsigned)min(rx + 2, wctb);
          unsigned spins = 0, ns = 250;
          while (ld_acquire(&prog[3 * (ry - 1)]) < need) {
            __nanosleep(ns); if (ns < 8000) ns <<= 1;
            if ((++spins & 31u) == 0 && ld_acquire(b.error_flag)) break;
            if (spins > (1u << 23)) { atomicExch(b.error_flag, 1u); break; }
          }
          abort = ld_acquire(b.error_flag) != 0u;
        }
        if (__shfl_sync(0xffffffffu, abort, 0)) return;                      // the batch is reported as failed; nothing it produced is used
        // halo row above (corner .. above-right) from HBM/L2: written by another SM during this kernel -> L1-bypassing loads
        const int cnt = 1 + 2 * tw;
        const P* grow = recp + (size_t)(cy0 - 1) * rst;
#pragma unroll 1
        for (int i = l; i < cnt; i += lpc) {
          const int gx = cx0 - 1 + i;
          int v = 0;
          if (gx >= 0 && gx < cw) v = (int)__ldcg(grow + gx);
          tp[PAD - 1 + i] = (P)v;
        }
      }
      __syncwarp();
      // ---- phase B: prediction + reconstruction, block after block
#pragma unroll 1
      for (int k = 0; k < ntb; k++) predict_tb<P>(desc[k], tl, tp, rs, rf, S, l, lpc, gmask, cidx, g == 0, g == 0 || (g >= 2 && cfmt == 3), bd, g == 0 ? strong_en : 0);
      // ---- the finished CTB goes to HBM; its last column becomes the next CTB's left halo
      {
        const int w = min(tw, cw - cx0), h = min(th, ch - cy0);
        const unsigned rowb = (unsigned)(w * (int)sizeof(P));
        P* gdst = recp + (size_t)cy0 * rst + cx0;
        if ((rowb & 15u) == 0) {
          // TMA: one bulk row copy per lane (generic-proxy writes of the tile made visible to the async proxy first)
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
#pragma unroll 1
          for (int y = l; y < h; y += lpc) bulk_store(gdst + (size_t)y * rst, tl + y * S + PAD, rowb);
          asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        } else {
          const int wq = (int)(rowb >> 2);                                     // 4-byte words per row (widths are multiples of 4 samples)
#pragma unroll 1
          for (int i = l; i < h * wq; i += lpc) {
            const int y = i / wq, q = i - y * wq;
            reinterpret_cast<unsigned*>(gdst + (size_t)y * rst)[q] = reinterpret_cast<const unsigned*>(tl + y * S + PAD)[q];
          }
        }
        // last column -> left halo of the next CTB (read before, written after the rows have left the tile)
        P keep0 = 0, keep1 = 0;
        if (l < th) keep0 = tl[l * S + PAD + tw - 1];
        if (l + lpc < th) keep1 = tl[(l + lpc) * S + PAD + tw - 1];
        if ((rowb & 15u) == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");     // rows are in global memory; the tile may be overwritten
        __syncwarp();
        if (l < th) tl[l * S + PAD - 1] = keep0;
        if (l + lpc < th) tl[(l + lpc) * S + PAD - 1] = keep1;
        __threadfence();
        __syncwarp();                                         // all lanes' stores precede lane 0's release store (cumulativity)
        if (lane == 0) st_release(&prog[3 * ry], (unsigned)(rx + 1));
      }
    }
  }
}

int launch_recon(const DeviceBatch& b, cudaStream_t s) {
  if (b.nrows <= 0) return B200_OK;
  const bool live = b.entropy_progress != nullptr;
  const int bps = b.wide_samples ? 2 : 1;
  const size_t smem = MAT_BYTES + (size_t)warp_layout(b.max_log2_ctb, bps).total * WARPS;
  const void* kern = bps == 2 ? (live ? (const void*)hevc_recon_kernel<uint16_t, true> : (const void*)hevc_recon_kernel<uint16_t, false>)
                              : (live ? (const void*)hevc_recon_kernel<uint8_t, true> : (const void*)hevc_recon_kernel<uint8_t, false>);
  B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(MAT_BYTES + (size_t)warp_layout(6, 2).total * WARPS)));
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int occ = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, WARPS * 32, smem);
  if (occ < 1) occ = 1;
  if (b.blocks_per_sm > 0 && b.blocks_per_sm < occ) occ = b.blocks_per_sm;
  const int want = (b.nrows + WARPS - 1) / WARPS;
  const int grid = want < sms * occ ? want : sms * occ;
  void* args[] = {const_cast<DeviceBatch*>(&b)};
  cudaError_t e = cudaLaunchKernel(kern, dim3((unsigned)grid), dim3(WARPS * 32), args, smem, s);
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "recon launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

// ---- test-only: the scaling and inverse transform of phase A on single blocks (b200_debug_k1_residual)
enum { K1B_LOG2N, K1B_BD, K1B_QP, K1B_DST, K1B_TSKIP, K1B_RAW, K1B_SF, K1B_NNZ, K1B_FIELDS };
constexpr int K1H_RES = (MAT_BYTES + 15) & ~15, K1H_TMP = K1H_RES + 32 * 32 * 2, K1H_SMEM = K1H_TMP + 32 * 34 * 2;   // K1's 16-byte aligned res / tmp

// One warp (CTA) per block: K1's residual4_lane (on lane 0, as a 4x4 block's owner lane) or residual_big, then the residual
// in raster order to out[block][0 .. n * n)
__global__ void __launch_bounds__(32) k1_residual_kernel(const int* __restrict__ prm, const uint8_t* __restrict__ sf, const CoefEntry* __restrict__ coefs,
                                                         const int* __restrict__ coef_off, int16_t* __restrict__ out) {
  __shared__ __align__(16) unsigned char sm[K1H_SMEM];
  int8_t* mat = reinterpret_cast<int8_t*>(sm);
  int16_t* rs = reinterpret_cast<int16_t*>(sm + K1H_RES);
  int16_t* tmp = reinterpret_cast<int16_t*>(sm + K1H_TMP);
  const int b = blockIdx.x, lane = threadIdx.x;
  const int* p = prm + b * K1B_FIELDS;
  const int lg = p[K1B_LOG2N], n = 1 << lg;
  const uint8_t* f = p[K1B_SF] ? sf + (size_t)b * 65 : nullptr;
  const CoefEntry* ce = coefs + coef_off[b];
  build_dct_matrices(mat, lane, 32);
  __syncwarp();
  if (lg == 2) {
    if (lane == 0) residual4_lane<false>(tmp, 0, ce, p[K1B_NNZ], p[K1B_QP], p[K1B_BD], p[K1B_DST] != 0, p[K1B_TSKIP] != 0, p[K1B_RAW] != 0, rs, f);
  } else {
    residual_big<false, 1>(rs, tmp, mat, ce, p[K1B_NNZ], lg, p[K1B_QP], p[K1B_BD], lane, f, f ? (int)f[64] : 16, p[K1B_RAW] != 0);
  }
  __syncwarp();
  for (int i = lane; i < n * n; i += 32) out[(size_t)b * 1024 + i] = rs[i];
}

__global__ void chroma_qp_kernel(const int* __restrict__ q, int n, int* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = chroma_qp(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]);
}

// ---- test-only: K1's make_desc + predict_tb on one constructed block per warp (b200_debug_k1_predict)
enum { K1P_KIND, K1P_LOG2CTB, K1P_BD, K1P_STRONG, K1P_BX, K1P_BY, K1P_LG, K1P_MODE, K1P_CODED0, K1P_CODED1, K1P_PCM, K1P_CX0, K1P_CY0, K1P_CW, K1P_CH,
       K1P_NBL, K1P_NBAL, K1P_NBA, K1P_NBAR, K1P_FIELDS };
enum { K1P_LUMA, K1P_PAIR420, K1P_PLANE422, K1P_PLANE444 };
constexpr int K1P_TILE = 64 * (64 + PAD), K1P_TOP = 256, K1P_RES = 1024, K1P_REF = 129;   // per-component slots of the buffers
constexpr int K1P_SENTINEL = -32768;                                                     // neighbour-array entries nobody wrote

// One warp (CTA) per case in K1's configuration for the case's kind: the warp's shared-memory slice of warp_layout(log2ctb,
// sizeof(P)) at K1's offset, the per-component tl / tp / rs / rf, and lpc / gmask / cidx / luma / smooth / strong_en as at K1's
// predict_tb call (kind 0: g = 0; 1: g = 1; 2 / 3: g = 2 of a 4:2:2 / 4:4:4 picture).
template <typename P>
__global__ void __launch_bounds__(32) k1_predict_kernel(const int* __restrict__ prm, const uint16_t* __restrict__ tiles, const uint16_t* __restrict__ tops,
                                                        const int16_t* __restrict__ res, uint32_t* __restrict__ desc_out, int16_t* __restrict__ ref_out,
                                                        uint16_t* __restrict__ tile_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x, lane = threadIdx.x;
  const int* p = prm + (size_t)b * K1P_FIELDS;
  const int kind = p[K1P_KIND], log2ctb = p[K1P_LOG2CTB], bd = p[K1P_BD];
  const WarpLayout L = warp_layout(log2ctb, (int)sizeof(P));
  unsigned char* wb = smem_raw + MAT_BYTES;
  P* const tile0 = reinterpret_cast<P*>(wb + L.tile);
  P* const top0 = reinterpret_cast<P*>(wb + L.top);
  int16_t* const res0 = reinterpret_cast<int16_t*>(wb + L.res);
  int16_t* const tmp = reinterpret_cast<int16_t*>(wb + L.tmp);
  const bool paired = kind == K1P_PAIR420;
  const int shx = kind == K1P_PAIR420 || kind == K1P_PLANE422 ? 1 : 0, shy = paired ? 1 : 0;
  const int tw = (1 << log2ctb) >> shx, th = (1 << log2ctb) >> shy, S = tw + PAD, ntop = PAD + 2 * tw + 16;
  const int ncomp = paired ? 2 : 1;
  const int bx = p[K1P_BX], by = p[K1P_BY], lg = p[K1P_LG], n = 1 << lg;
  const unsigned roff = morton4((unsigned)bx >> 2, (unsigned)by >> 2) * 16;
  for (int c = 0; c < ncomp; c++) {
    const size_t slot = (size_t)b * 2 + c;
    for (int i = lane; i < th * S; i += 32) tile0[c * (th * S) + i] = (P)tiles[slot * K1P_TILE + i];
    for (int i = lane; i < ntop; i += 32) top0[c * ntop + i] = (P)tops[slot * K1P_TOP + i];
    for (int i = lane; i < tw * th; i += 32) res0[c * (tw * th) + i] = 0;
  }
  for (int i = lane; i < 2 * REF_STRIDE; i += 32) tmp[i] = (int16_t)K1P_SENTINEL;
  __syncwarp();
  for (int c = 0; c < ncomp; c++)
    for (int i = lane; i < n * n; i += 32) res0[c * (tw * th) + roff + i] = res[((size_t)b * 2 + c) * K1P_RES + i];
  __syncwarp();
  // lane roles as in K1
  const int lpc = paired ? 16 : 32, l = lane & (lpc - 1), cidx = paired ? lane >> 4 : 0;
  const unsigned gmask = paired ? (0xffffu << (16 * cidx)) : 0xffffffffu;
  P* const tl = tile0 + cidx * (th * S);
  P* const tp = top0 + cidx * (PAD + 2 * tw + 16);
  int16_t* const rs = res0 + cidx * (tw * th);
  int16_t* const rf = tmp + cidx * REF_STRIDE;
  const uint2 d = make_uint2(make_desc(bx, by, lg, p[K1P_MODE], p[K1P_CODED0], p[K1P_CODED1], tw, th, paired ? 0 : shx, p[K1P_CX0], p[K1P_CY0], p[K1P_CW], p[K1P_CH],
                                       p[K1P_NBL] != 0, p[K1P_NBAL] != 0, p[K1P_NBA] != 0, p[K1P_NBAR] != 0) | ((unsigned)p[K1P_PCM] << 29), roff);
  const bool luma = kind == K1P_LUMA, smooth = kind == K1P_LUMA || kind == K1P_PLANE444;
  predict_tb<P>(d, tl, tp, rs, rf, S, l, lpc, gmask, cidx, luma, smooth, bd, luma ? p[K1P_STRONG] : 0);
  __syncwarp();
  if (lane == 0) desc_out[b] = d.x;
  for (int c = 0; c < ncomp; c++) {
    const size_t slot = (size_t)b * 2 + c;
    for (int i = lane; i < th * S; i += 32) tile_out[slot * K1P_TILE + i] = (uint16_t)tile0[c * (th * S) + i];
    for (int i = lane; i <= 4 * n; i += 32) {
      ref_out[(slot * 2) * K1P_REF + i] = tmp[c * REF_STRIDE + i];
      if (!paired) ref_out[(slot * 2 + 1) * K1P_REF + i] = tmp[REF_STRIDE + i];     // the filtered array (in the pair, Cr's rf is there)
    }
  }
}

}  // namespace b200

// Test-only entry points (declared by the tests, not in include/b200_heif.h).  Every argument is checked here, on the host:
// a call the checks refuse never reaches the device.
//
// b200_debug_k1_residual: K1's dequantisation and inverse transform of `n` blocks.  blocks[i * 8 ..]: log2 size (2..5), bit
// depth (8..12), qp (Qp'Y or Qp'C as K1 passes it: 0 .. 51 + 6 * (bd - 8)), DST (4x4 only), transform skip (4x4 only), raw
// (cu_transquant_bypass / PCM: the levels are the residuals), use scaling factors, nnz.  factors[i * 65 ..]: the block's
// factors in sl::Factors layout (8x8 raster, or 4x4 raster in the first 16 entries) and the DC factor of 16x16 / 32x32; read
// only for blocks that use them.  coefs: the blocks' CoefEntry lists back to back (pos = y * n + x, distinct within a block).
// out[i * 1024 ..]: the int16 residual in raster order.
extern "C" int b200_debug_k1_residual(int n, const int32_t* blocks, const uint8_t* factors, const uint32_t* coefs, int16_t* out) {
  using namespace b200;
  if (n < 1 || n > 65536 || !blocks || !out) return set_error(B200_E_INVALID, "k1_residual: %d blocks, null argument", n);
  std::vector<int> off((size_t)n + 1, 0);
  bool any_sf = false;
  for (int i = 0; i < n; i++) {
    const int32_t* p = blocks + (size_t)i * K1B_FIELDS;
    const int lg = p[K1B_LOG2N], bd = p[K1B_BD], nn = 1 << (lg >= 2 && lg <= 5 ? lg : 2);
    if (lg < 2 || lg > 5) return set_error(B200_E_INVALID, "k1_residual: block %d: log2 size %d", i, lg);
    if (bd < 8 || bd > 12) return set_error(B200_E_INVALID, "k1_residual: block %d: bit depth %d", i, bd);
    if (p[K1B_QP] < 0 || p[K1B_QP] > 51 + 6 * (bd - 8)) return set_error(B200_E_INVALID, "k1_residual: block %d: qp %d", i, p[K1B_QP]);
    for (int f = K1B_DST; f <= K1B_SF; f++)
      if (p[f] != 0 && p[f] != 1) return set_error(B200_E_INVALID, "k1_residual: block %d: flag %d = %d", i, f, p[f]);
    if (lg > 2 && (p[K1B_DST] || p[K1B_TSKIP])) return set_error(B200_E_INVALID, "k1_residual: block %d: DST / transform skip on %dx%d", i, nn, nn);
    if (p[K1B_TSKIP] && p[K1B_RAW]) return set_error(B200_E_INVALID, "k1_residual: block %d: transform skip and raw", i);
    if (p[K1B_NNZ] < 0 || p[K1B_NNZ] > nn * nn) return set_error(B200_E_INVALID, "k1_residual: block %d: nnz %d", i, p[K1B_NNZ]);
    if (p[K1B_NNZ] && !coefs) return set_error(B200_E_INVALID, "k1_residual: null coefficients");
    any_sf |= p[K1B_SF] != 0;
    uint32_t seen[32] = {};
    for (int k = 0; k < p[K1B_NNZ]; k++) {
      const unsigned pos = coefs[off[i] + k] & 0xffffu;
      if (pos >= (unsigned)(nn * nn)) return set_error(B200_E_INVALID, "k1_residual: block %d: position %u", i, pos);
      if (seen[pos >> 5] & (1u << (pos & 31))) return set_error(B200_E_INVALID, "k1_residual: block %d: position %u twice", i, pos);
      seen[pos >> 5] |= 1u << (pos & 31);
    }
    off[(size_t)i + 1] = off[i] + p[K1B_NNZ];
  }
  if (any_sf && !factors) return set_error(B200_E_INVALID, "k1_residual: null factors");
  DevBuf<int> d_prm, d_off; DevBuf<uint8_t> d_sf; DevBuf<uint32_t> d_ce; DevBuf<int16_t> d_out;
  const size_t nsf = any_sf ? (size_t)n * 65 : 1, nce = off[n] ? (size_t)off[n] : 1;
  int rc = 0;
  if ((rc = d_prm.reserve((size_t)n * K1B_FIELDS, false)) || (rc = d_off.reserve(off.size(), false)) || (rc = d_sf.reserve(nsf, false)) ||
      (rc = d_ce.reserve(nce, false)) || (rc = d_out.reserve((size_t)n * 1024, false))) return rc;
  B200_CUDA_CHECK(cudaMemcpy(d_prm.d, blocks, (size_t)n * K1B_FIELDS * 4, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_off.d, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
  if (any_sf) B200_CUDA_CHECK(cudaMemcpy(d_sf.d, factors, nsf, cudaMemcpyHostToDevice));
  if (off[n]) B200_CUDA_CHECK(cudaMemcpy(d_ce.d, coefs, nce * 4, cudaMemcpyHostToDevice));
  k1_residual_kernel<<<n, 32>>>(d_prm.d, d_sf.d, reinterpret_cast<const CoefEntry*>(d_ce.d), d_off.d, d_out.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpy(out, d_out.d, (size_t)n * 1024 * 2, cudaMemcpyDeviceToHost));
  return B200_OK;
}

// b200_debug_chroma_qp: K1's Qp'C (8.6.1) for n queries q[i * 4 ..] = (QpY, qp offset, bit depth, ChromaArrayType)
extern "C" int b200_debug_chroma_qp(int n, const int32_t* q, int32_t* out) {
  using namespace b200;
  if (n < 1 || n > (1 << 20) || !q || !out) return set_error(B200_E_INVALID, "chroma_qp: %d queries, null argument", n);
  for (int i = 0; i < n; i++) {
    const int qpy = q[4 * i], off = q[4 * i + 1], bd = q[4 * i + 2], cat = q[4 * i + 3];
    if (bd < 8 || bd > 12 || cat < 1 || cat > 3 || qpy < -6 * (bd - 8) || qpy > 51 || off < -12 || off > 12)
      return set_error(B200_E_INVALID, "chroma_qp: query %d: QpY %d offset %d bit depth %d ChromaArrayType %d", i, qpy, off, bd, cat);
  }
  DevBuf<int> d_q, d_out;
  int rc = 0;
  if ((rc = d_q.reserve((size_t)n * 4, false)) || (rc = d_out.reserve((size_t)n, false))) return rc;
  B200_CUDA_CHECK(cudaMemcpy(d_q.d, q, (size_t)n * 16, cudaMemcpyHostToDevice));
  chroma_qp_kernel<<<(n + 127) / 128, 128>>>(d_q.d, n, d_out.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpy(out, d_out.d, (size_t)n * 4, cudaMemcpyDeviceToHost));
  return B200_OK;
}

// b200_debug_k1_predict: K1's make_desc and predict_tb on n constructed blocks, one warp each.  cases[i * 19 ..]: kind (0: luma,
// 1: 4:2:0 Cb + Cr pair on the two half-warps, 2: a 4:2:2 chroma plane, 3: a 4:4:4 chroma plane), log2 CTB size (4..6), bit depth
// (8..12), strong_intra_smoothing_enabled_flag, then make_desc's inputs: bx, by (component samples inside the component's CTB),
// log2 size, mode, coded (Cb / first component), coded (Cr, pair only), pcm, cx0, cy0 (the CTB's component origin), cw, ch (the
// component plane's size), nbL, nbAL, nbA, nbAR.  Per case and component c (one, two for the pair), at slot s = i * 2 + c:
// tiles[s * 5120 ..]: the component's tile as K1 keeps it in shared memory (th rows of tw + 16 samples; sample (x, y) at
// [y * (tw + 16) + 16 + x], column 15 the left halo); tops[s * 256 ..]: its halo row (sample x at [16 + x]); res[s * 1024 ..]: the
// block's residual (raster), for pcm the samples.  Outputs: desc[i], the descriptor word; refs[(s * 2) * 129 ..]: rf after
// substitution, refs[(s * 2 + 1) * 129 ..]: the filtered array (-32768 where nothing was written; not for the pair);
// tiles_out[s * 5120 ..]: the whole tile after the call.
extern "C" int b200_debug_k1_predict(int n, const int32_t* cases, const uint16_t* tiles, const uint16_t* tops, const int16_t* res, uint32_t* desc,
                                     int16_t* refs, uint16_t* tiles_out) {
  using namespace b200;
  if (n < 1 || n > 65536 || !cases || !tiles || !tops || !res || !desc || !refs || !tiles_out) return set_error(B200_E_INVALID, "k1_predict: %d cases, null argument", n);
  bool wide = false, narrow = false;
  for (int i = 0; i < n; i++) {
    const int32_t* p = cases + (size_t)i * K1P_FIELDS;
    const int kind = p[K1P_KIND], lc = p[K1P_LOG2CTB], bd = p[K1P_BD], lg = p[K1P_LG];
    if (kind < 0 || kind > 3 || lc < 4 || lc > 6 || bd < 8 || bd > 12) return set_error(B200_E_INVALID, "k1_predict: case %d: kind %d log2 CTB %d bit depth %d", i, kind, lc, bd);
    (bd > 8 ? wide : narrow) = true;
    const int shx = kind == K1P_PAIR420 || kind == K1P_PLANE422 ? 1 : 0, shy = kind == K1P_PAIR420 ? 1 : 0;
    const int tw = (1 << lc) >> shx, th = (1 << lc) >> shy, nmax = kind == K1P_LUMA || kind == K1P_PLANE444 ? 5 : 4;
    if (lg < 2 || lg > nmax || (1 << lg) > tw || (1 << lg) > th) return set_error(B200_E_INVALID, "k1_predict: case %d: log2 size %d", i, lg);
    const int nn = 1 << lg, bx = p[K1P_BX], by = p[K1P_BY];
    if (bx < 0 || by < 0 || bx % nn || by % nn || bx + nn > tw || by + nn > th) return set_error(B200_E_INVALID, "k1_predict: case %d: block at (%d, %d)", i, bx, by);
    if (p[K1P_MODE] < 0 || p[K1P_MODE] > 34) return set_error(B200_E_INVALID, "k1_predict: case %d: mode %d", i, p[K1P_MODE]);
    for (int f : {K1P_STRONG, K1P_CODED0, K1P_CODED1, K1P_PCM, K1P_NBL, K1P_NBAL, K1P_NBA, K1P_NBAR})
      if (p[f] != 0 && p[f] != 1) return set_error(B200_E_INVALID, "k1_predict: case %d: flag %d = %d", i, f, p[f]);
    if (p[K1P_CODED1] && kind != K1P_PAIR420) return set_error(B200_E_INVALID, "k1_predict: case %d: second coded flag outside the pair", i);
    const int cx0 = p[K1P_CX0], cy0 = p[K1P_CY0], cw = p[K1P_CW], ch = p[K1P_CH];
    if (cw < 4 || ch < 4 || cw > 8192 || ch > 8192 || cw % 4 || ch % 4 || cx0 < 0 || cy0 < 0 || cx0 % tw || cy0 % th || cx0 + bx + nn > cw || cy0 + by + nn > ch)
      return set_error(B200_E_INVALID, "k1_predict: case %d: CTB at (%d, %d) of a %dx%d plane", i, cx0, cy0, cw, ch);
    if ((p[K1P_NBL] && cx0 == 0) || (p[K1P_NBAL] && (cx0 == 0 || cy0 == 0)) || (p[K1P_NBA] && cy0 == 0) || (p[K1P_NBAR] && (cy0 == 0 || cx0 + tw >= cw)))
      return set_error(B200_E_INVALID, "k1_predict: case %d: a neighbouring CTB outside the picture is available", i);
    const int maxv = (1 << bd) - 1, S = tw + PAD, ntop = PAD + 2 * tw + 16;
    for (int c = 0; c < (kind == K1P_PAIR420 ? 2 : 1); c++) {
      const size_t s = (size_t)i * 2 + c;
      for (int k = 0; k < th * S; k++) if (tiles[s * K1P_TILE + k] > maxv) return set_error(B200_E_INVALID, "k1_predict: case %d: tile sample above %d", i, maxv);
      for (int k = 0; k < ntop; k++) if (tops[s * K1P_TOP + k] > maxv) return set_error(B200_E_INVALID, "k1_predict: case %d: halo sample above %d", i, maxv);
      if (p[K1P_PCM])
        for (int k = 0; k < nn * nn; k++) if (res[s * K1P_RES + k] < 0 || res[s * K1P_RES + k] > maxv) return set_error(B200_E_INVALID, "k1_predict: case %d: pcm sample outside [0, %d]", i, maxv);
    }
  }
  if (wide && narrow) return set_error(B200_E_INVALID, "k1_predict: 8-bit and deeper cases in one call");
  DevBuf<int> d_prm; DevBuf<uint16_t> d_tiles, d_tops, d_tout; DevBuf<int16_t> d_res, d_refs; DevBuf<uint32_t> d_desc;
  const size_t nt = (size_t)n * 2 * K1P_TILE;
  int rc = 0;
  if ((rc = d_prm.reserve((size_t)n * K1P_FIELDS, false)) || (rc = d_tiles.reserve(nt, false)) || (rc = d_tops.reserve((size_t)n * 2 * K1P_TOP, false)) ||
      (rc = d_res.reserve((size_t)n * 2 * K1P_RES, false)) || (rc = d_desc.reserve((size_t)n, false)) || (rc = d_refs.reserve((size_t)n * 4 * K1P_REF, false)) ||
      (rc = d_tout.reserve(nt, false))) return rc;
  B200_CUDA_CHECK(cudaMemcpy(d_prm.d, cases, (size_t)n * K1P_FIELDS * 4, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_tiles.d, tiles, nt * 2, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_tops.d, tops, (size_t)n * 2 * K1P_TOP * 2, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_res.d, res, (size_t)n * 2 * K1P_RES * 2, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemset(d_refs.d, 0, (size_t)n * 4 * K1P_REF * 2));
  B200_CUDA_CHECK(cudaMemset(d_tout.d, 0, nt * 2));
  const int smem = MAT_BYTES + warp_layout(6, wide ? 2 : 1).total;
  const void* kern = wide ? (const void*)k1_predict_kernel<uint16_t> : (const void*)k1_predict_kernel<uint8_t>;
  B200_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  if (wide) k1_predict_kernel<uint16_t><<<n, 32, smem>>>(d_prm.d, d_tiles.d, d_tops.d, d_res.d, d_desc.d, d_refs.d, d_tout.d);
  else k1_predict_kernel<uint8_t><<<n, 32, smem>>>(d_prm.d, d_tiles.d, d_tops.d, d_res.d, d_desc.d, d_refs.d, d_tout.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpy(desc, d_desc.d, (size_t)n * 4, cudaMemcpyDeviceToHost));
  B200_CUDA_CHECK(cudaMemcpy(refs, d_refs.d, (size_t)n * 4 * K1P_REF * 2, cudaMemcpyDeviceToHost));
  B200_CUDA_CHECK(cudaMemcpy(tiles_out, d_tout.d, nt * 2, cudaMemcpyDeviceToHost));
  return B200_OK;
}

// Host-only: the descriptors phase A of K1 builds for one access unit parsed by the host front-end.  hdr[6]: coded width, height,
// log2 CTB size, chroma_format_idc, number of component groups G (1 for 4:0:0; 2 for 4:2:0: luma, Cb + Cr; 3 otherwise: luma, Cb, Cr),
// number of descriptors.  desc (room for max_desc): the descriptor words (make_desc's layout, pcm in bit 29) per CTB in raster order,
// per group, in the order of the CTB's commands; counts[ctb * G + group] (room for max_counts): how many of them.  With desc / counts
// NULL only hdr is filled.
extern "C" int b200_debug_k1_descriptors(const uint8_t* au, size_t size, int32_t* hdr, uint32_t* desc, int max_desc, int32_t* counts, int max_counts) {
  using namespace b200;
  if (!au || !hdr) return set_error(B200_E_INVALID, "k1_descriptors: null argument");
  ParsedPicture pp; ParseLimits lim;
  int rc = parse_access_unit(au, size, lim, pp);
  if (rc) return rc;
  const PicDesc& p = pp.desc;
  const int cfmt = p.chroma, ng = cfmt == 0 ? 1 : (cfmt == 1 ? 2 : 3), wctb = p.wctb, nctb = p.wctb * p.hctb;
  std::vector<uint32_t> all;
  std::vector<int32_t> cnt((size_t)nctb * ng, 0);
  const int bd = p.bit_depth;
  const CoefEntry* coefs = pp.coefs.data();
  for (int addr = 0; addr < nctb; addr++) {
    const int rx = addr % wctb, ry = addr / wctb;
    const CtuInfo& ci = pp.ctus[(size_t)addr];
    const int cur = ci.slice_idx;
#define B200_HOST_REGION(a) (int)pp.ctus[(size_t)(a)].slice_idx
    B200_K1_CTB_NEIGHBOURS(B200_HOST_REGION)
#undef B200_HOST_REGION
    const SliceInfo sl = pp.slices[(size_t)cur];
    for (int gi = 0; gi < ng; gi++) {
      // the work item's group as K1 sees it: 0 luma, 1 the 4:2:0 pair, 2 / 3 the Cb / Cr plane of 4:2:2 / 4:4:4
      const int g = gi == 0 ? 0 : (cfmt == 1 ? 1 : gi + 1);
      const int pl = g >= 2 ? g - 1 : 0;
      const int shx = g == 0 ? 0 : (g == 1 ? 1 : (cfmt == 2 ? 1 : 0)), shy = g == 1 ? 1 : 0;
      const bool paired = g == 1;
      const int tw = (1 << p.log2_ctb) >> shx, th = (1 << p.log2_ctb) >> shy, cw = p.width >> shx, ch = p.height >> shy;
      const int x0 = rx << p.log2_ctb, y0 = ry << p.log2_ctb, cx0 = x0 >> shx, cy0 = y0 >> shy;
      for (unsigned k = 0; k < ci.tu_count; k++) {
        const TuCmd cmd = pp.tus[ci.tu_start + k];
        const bool valid = true;
        B200_K1_TB_OF_CMD
        if (has) { all.push_back(B200_K1_DESC); cnt[(size_t)addr * ng + gi]++; }
      }
    }
  }
  const int32_t h[6] = {p.width, p.height, p.log2_ctb, cfmt, ng, (int32_t)all.size()};
  memcpy(hdr, h, sizeof h);
  if (desc) {
    if (max_desc < 0 || (size_t)max_desc < all.size()) return set_error(B200_E_INVALID, "k1_descriptors: room for %d descriptors, %zu needed", max_desc, all.size());
    memcpy(desc, all.data(), all.size() * 4);
  }
  if (counts) {
    if (max_counts < 0 || (size_t)max_counts < cnt.size()) return set_error(B200_E_INVALID, "k1_descriptors: room for %d counts, %zu needed", max_counts, cnt.size());
    memcpy(counts, cnt.data(), cnt.size() * 4);
  }
  return B200_OK;
}
