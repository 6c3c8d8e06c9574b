// b200_hevc_gpu_enc.cu -- HEVC intra encoder on the GPU: N same-sized 8-bit 4:2:0 / 4:0:0 pictures per call.
//
//   E1 (analyse + reconstruct), one warp per (picture, CTB row): CU quadtree from the CTB down to 8x8 (NxN at 8x8), decided
//      bottom-up on J = SATD(prediction residual) + lambda(QP) * estimated mode bits; chroma = DM; TU = CU (implicit splits:
//      NxN, > 32).  The decision pass has three speeds, each an instantiation of its own (b200_hevc_enc_params::speed):
//        0: all 35 luma modes at every PU, closed loop (neighbours from the encoder's own reconstruction);
//        1: a coarse-to-fine search of at most 18 modes (search_mode), closed loop;
//        2: as 1, open loop: neighbours from the source, no transform round trip before the final pass.
//      forward DST 4x4 / DCT 4..32, uniform quantisation with the intra rounding offset 171/512, reconstruction with the
//      inverse path of 8.6.  Writes the reconstruction (HBM plane: the neighbours of the next row), the luma modes per 4x4,
//      the CU size / partition per 8x8 and the quantised levels (a coefficient plane: every TB's levels at its position).
//      Rows trail the row above by two CTBs through per-row progress counters.  The prediction, transform and
//      (de)quantisation arithmetic is the host encoder's (b200_hevc_enc_recon.h), at bit depth 8.
//   E2 (CABAC), one warp per WPP sub-stream (= CTB row): the syntax of 7.3.8 from E1's records, context hand-over after
//      the 2nd CTB of the row above (9.3.2.2), end_of_slice_segment_flag per CTB and end_of_subset_one_bit + byte
//      alignment per row, into a per-row buffer sized for the worst case.  The arithmetic coder, residual_coding() and the
//      intra mode signalling are the host encoder's (b200_hevc_enc_cabac.h).
//   Framing (host): parameter sets and slice header (b200_hevc_enc_headers.h, shared with the host encoder), entry points
//      over the escaped sub-stream sizes, emulation prevention, length prefixes.
//
// Prediction, transforms and dequantisation are shared with the host encoder rather than taken from the reconstruction
// kernel (b200_hevc_recon.cu): its predict_tb reconstructs one TB of a known mode inside K1's per-lane padded tile, from a packed
// descriptor whose neighbour availability is precomputed as index intervals, and residual4_lane / residual_big consume sparse
// CoefEntry lists.  The mode search needs the predicted sample of any of the 35 modes at any position as a pure function,
// many modes per block without reconstructing, and dense residual blocks; both files are separate translation units built
// without relocatable device code.  The tests pin the result bit-exact against that decoder, the C restatement and FFmpeg.
#include "b200_internal.h"
#include "b200_staging.h"
#include "b200_hevc_enc_headers.h"
#include "b200_hevc_enc_cabac.h"
#include "b200_hevc_enc_recon.h"
#include <algorithm>
#include <climits>
#include <chrono>
#include <memory>
#include <vector>

#define GE_LANES 32
#define GE_SYNC() __syncwarp()
#define GE_ATOMIC_ADD(p, v) atomicAdd((p), (v))
#define GE_LD(p) __ldcg(p)          // planes written by other rows' warps (other SMs): bypass the non-coherent L1

namespace b200 {
namespace genc {

using syn::clip3;

enum { CU_NXN = 0x80 };

// Worst case of one sub-stream, in bytes per sample of the CTB row, plus a fixed allowance per CTB.  Per coefficient:
// sig / gt1 / gt2 context bins (at most 6 renormalisation shifts = output bits each, rangeTabLps >= 6) + a sign bypass bin
// + coeff_abs_level_remaining of a level <= 32767 (at most 32 bypass bins) = 51 bits; 8x8 CUs coded as NxN add per 96
// samples six TBs of last-position / cbf / csbf bins and the CU header: below 64 bits = 8 bytes per sample in total.
constexpr int kBytesPerSample = 8, kBytesPerCtb = 64;
inline size_t substream_capacity(int width, int log2ctb, int cfmt) {
  const int ctb = 1 << log2ctb, wctb = (((width + 7) & ~7) + ctb - 1) >> log2ctb;
  const size_t samples = (size_t)ctb * ctb * (cfmt ? 3 : 2) / 2;
  return (size_t)wctb * (samples * kBytesPerSample + kBytesPerCtb);
}

struct Pic { const uint8_t* src[3]; size_t stride[3]; };

struct Args {
  const Pic* pics; int n;
  int W, H, Wc, Hc, sw, sh;          // coded (multiples of 8) and source sizes (luma)
  int cfmt, log2ctb, wctb, hctb, max_th_depth, strong, slice_qp, qp[3], lambda16;
  uint8_t* rec; int16_t* coef; size_t pic_samples;          // per picture: Y (W x H), Cb, Cr (Wc x Hc)
  uint8_t* ipm4; uint8_t* dec4; size_t map4;                 // per 4x4 luma: intra mode, reconstructed flag
  uint8_t* cu8; size_t map8;                                 // per 8x8: log2 CU size | CU_NXN
  unsigned* progress; unsigned* progress2; unsigned* ticket; unsigned* error;   // rows, rows, 2, 1
  uint8_t* wpp_ctx;                                          // per row: CTX_COUNT context bytes after its 2nd CTB
  uint8_t* ss; size_t ss_cap; unsigned* ss_len;              // per row sub-stream
  unsigned long long* work;                                  // E1's work counters: [0] mode evaluations, [1] eval_cu calls
                                                             // (lane 0 adds to them per PU search / eval_cu: a reduction
                                                             // without a result, and no counter register kept across the
                                                             // quadtree calls)
};

// ---------------------------------------------------------------------------------------------------- E1 workspace
struct Work {
  int res[1024], tmp[1024], coef[1024];
  int16_t lev[1024];
  uint8_t pred[1024];
  int16_t ref[2][132];               // neighbours (8.4.4.2.2): [0] substituted, [1] filtered
  int satd[36];
  int dc, any, acc, mode;
};
// E1's shared memory at speed S: Work, then per quadtree depth the state of the no-split alternative that the split
// alternative overwrites -- luma reconstruction and modes (closed loop), or the modes alone (speed 2, which reconstructs in
// the final pass only); speeds 1 and 2 add the candidate list of the coarse-to-fine search.
template <int S> struct E1Work : Work {
  uint8_t save[4][(S == 2 ? 0 : 4096) + 256];
  uint8_t list[20];                  // candidate modes of the coarse-to-fine search
};
template <> struct E1Work<0> : Work { uint8_t save[4][4096 + 256]; };

struct Ctx2 { const Args& a; int p; int lane; Work& w;
  __device__ uint8_t* plane(int c) const { return a.rec + (size_t)p * a.pic_samples + (c == 0 ? 0 : (size_t)a.W * a.H + (size_t)(c - 1) * a.Wc * a.Hc); }
  __device__ int16_t* cplane(int c) const { return a.coef + (size_t)p * a.pic_samples + (c == 0 ? 0 : (size_t)a.W * a.H + (size_t)(c - 1) * a.Wc * a.Hc); }
  __device__ uint8_t* ipm() const { return a.ipm4 + (size_t)p * a.map4; }
  __device__ uint8_t* dec() const { return a.dec4 + (size_t)p * a.map4; }
  __device__ uint8_t* cu() const { return a.cu8 + (size_t)p * a.map8; }
  __device__ int org(int c, int x, int y) const {                // edge padding of the source to the coded size
    const int sw = c ? (a.sw + 1) >> 1 : a.sw, sh = c ? (a.sh + 1) >> 1 : a.sh;
    return a.pics[p].src[c][(size_t)(y < sh ? y : sh - 1) * a.pics[p].stride[c] + (x < sw ? x : sw - 1)];
  }
  __device__ bool avail(int x, int y) const {                    // luma position reconstructed already (z-scan availability, one slice)
    if (x < 0 || y < 0 || x >= a.W || y >= a.H) return false;
    return GE_LD(dec() + (size_t)(y >> 2) * (a.W >> 2) + (x >> 2)) != 0;
  }
};

// 8.4.2: the three most probable modes of the PU at luma (x, y)
__device__ inline void mpm_cand(const uint8_t* ipm, int w4, int log2ctb, int x, int y, int cand[3]) {
  int ca = 1, cb = 1;
  if (x > 0) ca = GE_LD(ipm + (size_t)(y >> 2) * w4 + ((x - 1) >> 2));
  if (y > 0 && (y - 1) >= ((y >> log2ctb) << log2ctb)) cb = GE_LD(ipm + (size_t)((y - 1) >> 2) * w4 + (x >> 2));
  enc::mpm_candidates(ca, cb, cand);
}
__device__ inline int mode_bits(int mode, const int cand[3]) { return mode == cand[0] ? 2 : (mode == cand[1] || mode == cand[2]) ? 3 : 6; }

// neighbours of the n x n block of component c at (x0, y0): availability, substitution, filtering (8.4.4.2.2 / .3).
// Src: the sample values from the edge-padded source instead of the reconstruction (open-loop decisions), with the same
// availability.
template <bool Src = false>
__device__ void gather_refs(Ctx2& e, int c, int x0, int y0, int log2n) {
  Work& w = e.w;
  const int n = 1 << log2n, sh = c ? 1 : 0, st = c ? e.a.Wc : e.a.W;
  const uint8_t* pl = e.plane(c);
  for (int i = e.lane; i <= 4 * n; i += GE_LANES) {
    int px, py;
    if (i < 2 * n) { px = x0 - 1; py = y0 + 2 * n - 1 - i; } else if (i == 2 * n) { px = x0 - 1; py = y0 - 1; } else { px = x0 + (i - 2 * n - 1); py = y0 - 1; }
    if constexpr (Src) w.ref[0][i] = e.avail(px << sh, py << sh) ? (int16_t)e.org(c, px, py) : (int16_t)-1;
    else w.ref[0][i] = e.avail(px << sh, py << sh) ? (int16_t)GE_LD(pl + (size_t)py * st + px) : (int16_t)-1;
  }
  GE_SYNC();
  if (e.lane == 0) {
    enc::substitute_refs(w.ref[0], n, 8);
    if (c == 0 && n != 4) enc::filter_refs(w.ref[0], w.ref[1], log2n, e.a.strong, 8);
    w.dc = enc::dc_value(w.ref[0], log2n);
  }
  GE_SYNC();
}

// predicted sample (x, y) of mode `mode` from the neighbours gathered above
__device__ inline int predicted(const Work& w, int c, int log2n, int mode, int x, int y) {
  return enc::pred_sample(w.ref[enc::refs_filtered(c == 0, mode, log2n) ? 1 : 0], w.dc, log2n, mode, x, y, c == 0, 255);
}

__device__ inline int satd4(const int d[16]) {                   // 4x4 Hadamard
  int m[16], s = 0;
  for (int i = 0; i < 4; i++) {
    const int a0 = d[i * 4] + d[i * 4 + 3], a1 = d[i * 4 + 1] + d[i * 4 + 2], a2 = d[i * 4 + 1] - d[i * 4 + 2], a3 = d[i * 4] - d[i * 4 + 3];
    m[i * 4] = a0 + a1; m[i * 4 + 2] = a0 - a1; m[i * 4 + 1] = a3 + a2; m[i * 4 + 3] = a3 - a2;
  }
  for (int i = 0; i < 4; i++) {
    const int a0 = m[i] + m[12 + i], a1 = m[4 + i] + m[8 + i], a2 = m[4 + i] - m[8 + i], a3 = m[i] - m[12 + i];
    s += abs(a0 + a1) + abs(a0 - a1) + abs(a3 + a2) + abs(a3 - a2);
  }
  return (s + 1) >> 1;
}

// SATD of the n x n block at (x0, y0) for the `cnt` modes mode_at(0 .. cnt - 1), added to w.satd[mode]: one (mode, 4x4
// sub-block) pair per lane and step (the full search's loop)
template <typename ModeAt>
__device__ inline void add_satd(Ctx2& e, int x0, int y0, int log2n, int cnt, ModeAt mode_at) {
  Work& w = e.w;
  const int n = 1 << log2n, nsb = (n * n) >> 4;
  for (int it = e.lane; it < cnt * nsb; it += GE_LANES) {
    const int mode = mode_at(it % cnt), sb = it / cnt, bx = (sb % (n >> 2)) << 2, by = (sb / (n >> 2)) << 2;
    int d[16];
    for (int k = 0; k < 16; k++) d[k] = e.org(0, x0 + bx + (k & 3), y0 + by + (k >> 2)) - predicted(w, 0, log2n, mode, bx + (k & 3), by + (k >> 2));
    GE_ATOMIC_ADD(&w.satd[mode], satd4(d));
  }
}

// The same sums for the modes list[0 .. cnt) in mode-major order: the lanes of a step share a mode on consecutive 4x4
// sub-blocks (a whole warp from 16x16 up), so the prediction does not diverge, and the indices are a shift and a mask.
__device__ inline void add_satd_list(Ctx2& e, int x0, int y0, int log2n, int cnt, const uint8_t* list) {
  Work& w = e.w;
  const int lsb = 2 * log2n - 4, lw = log2n - 2;               // log2 of the sub-blocks per block / per row
  for (int it = e.lane; it < (cnt << lsb); it += GE_LANES) {
    const int mode = list[it >> lsb], sb = it & ((1 << lsb) - 1), bx = (sb & ((1 << lw) - 1)) << 2, by = (sb >> lw) << 2;
    int d[16];
    for (int k = 0; k < 16; k++) d[k] = e.org(0, x0 + bx + (k & 3), y0 + by + (k >> 2)) - predicted(w, 0, log2n, mode, bx + (k & 3), by + (k >> 2));
    GE_ATOMIC_ADD(&w.satd[mode], satd4(d));
  }
}

// the lowest J x 16 over the modes of `set`, shifted left by 6 with the mode in the low bits (ties: the lower mode); every
// lane gets it
__device__ inline long long best_mode(const Ctx2& e, unsigned long long set, const int cand[3]) {
  long long k = LLONG_MAX;
  for (int m = e.lane; m < 35; m += GE_LANES)
    if ((set >> m) & 1) k = min(k, ((((long long)e.w.satd[m] << 4) + (long long)e.a.lambda16 * mode_bits(m, cand)) << 6) | m);
  for (int o = 16; o; o >>= 1) k = min(k, (long long)__shfl_xor_sync(0xffffffffu, k, o));
  return k;
}

// best luma mode of the n x n PU at (x0, y0) on SATD + lambda * mode bits; returns the mode, *cost = its J (x16).
// S = 0: all 35 modes.  S >= 1, coarse to fine: round 1 planar, DC, the angular modes 2, 6, .., 34 and the three MPM
// candidates; round 2 the angular modes within 2 of round 1's best angular mode a* (clamped to 2..34), those not evaluated
// yet.  Ties go to the lower mode number in both rounds.  S = 2 predicts from the source (open loop).
template <int S>
__device__ int search_mode(Ctx2& e, int x0, int y0, int log2n, long long* cost) {
  Work& w = e.w;
  gather_refs<S == 2>(e, 0, x0, y0, log2n);
  unsigned long long done = (1ull << 35) - 1;                 // the modes evaluated
  if constexpr (S == 0) {
    for (int i = e.lane; i < 35; i += GE_LANES) w.satd[i] = 0;
    GE_SYNC();
    add_satd(e, x0, y0, log2n, 35, [](int m) { return m; });
  } else {
    // The candidate sets are bit masks held alike by every lane (no per-candidate serial work, nothing in local memory); each
    // round's modes are listed in shared memory in mode order, one lane per mode, behind those of the rounds before.
    uint8_t* list = static_cast<E1Work<S>&>(w).list;
    int org[16];                                               // a 4x4 PU: its source samples, loaded once for both rounds
    if (log2n == 2)
      for (int k = 0; k < 16; k++) org[k] = e.org(0, x0 + (k & 3), y0 + (k >> 2));
    int cand[3]; mpm_cand(e.ipm(), e.a.W >> 2, e.a.log2ctb, x0, y0, cand);
    constexpr unsigned long long kCoarse = 0x444444447ull;     // planar, DC, angular 2, 6, .., 34
    unsigned long long round = kCoarse | (1ull << cand[0]) | (1ull << cand[1]) | (1ull << cand[2]);
    done = 0;
    for (int i = e.lane; i < 35; i += GE_LANES) w.satd[i] = 0;
    for (int r = 0; r < 2; r++) {
      const int first = __popcll(done), cnt = __popcll(round);
      for (int m = e.lane; m < 35; m += GE_LANES)
        if ((round >> m) & 1) list[first + __popcll(round & ((1ull << m) - 1))] = (uint8_t)m;
      done |= round;
      GE_SYNC();
      if (log2n == 2) {                                        // at most 14 modes a round: one lane each
        if (e.lane < cnt) {
          const int mode = list[first + e.lane];
          int d[16];
          for (int k = 0; k < 16; k++) d[k] = org[k] - predicted(w, 0, 2, mode, k & 3, k >> 2);
          w.satd[mode] = satd4(d);
        }
      } else add_satd_list(e, x0, y0, log2n, cnt, list + first);
      GE_SYNC();
      if (r == 0) {                                            // round 2: the angular modes within 2 of round 1's best one
        const int a = (int)(best_mode(e, done & ~3ull, cand) & 63);
        round = 0;
        for (int d = -2; d <= 2; d++) round |= 1ull << clip3(2, 34, a + d);
        round &= ~done;
      }
    }
    if (e.lane == 0) atomicAdd(e.a.work, (unsigned long long)__popcll(done));
    const long long best = best_mode(e, done, cand);
    *cost = best >> 6;
    return (int)(best & 63);
  }
  if (e.lane == 0) atomicAdd(e.a.work, (unsigned long long)__popcll(done));
  GE_SYNC();
  if (e.lane == 0) {
    int cand[3]; mpm_cand(e.ipm(), e.a.W >> 2, e.a.log2ctb, x0, y0, cand);
    long long best = -1; int bm = 0;
    for (int m = 0; m < 35; m++) {
      if (!((done >> m) & 1)) continue;
      const long long j = ((long long)w.satd[m] << 4) + (long long)e.a.lambda16 * mode_bits(m, cand);
      if (best < 0 || j < best) { best = j; bm = m; }
    }
    w.mode = bm; w.satd[35] = (int)best;                      // J x 16 of a 32x32 PU stays far below 2^31
  }
  GE_SYNC();
  *cost = w.satd[35];
  return w.mode;
}

// Predict, transform, quantise, reconstruct one TB of component c (component coordinates).  `final`: store the levels in the
// coefficient plane.  Returns the SATD of the prediction residual (luma only, else 0).
__device__ int code_tb(Ctx2& e, int c, int x0, int y0, int log2n, int mode, bool final) {
  Work& w = e.w;
  const int n = 1 << log2n, nn = n * n, st = c ? e.a.Wc : e.a.W, qp = e.a.qp[c];
  const bool dst4 = c == 0 && log2n == 2;
  gather_refs(e, c, x0, y0, log2n);
  if (e.lane == 0) { w.any = 0; w.acc = 0; }
  for (int i = e.lane; i < nn; i += GE_LANES) {
    const int x = i & (n - 1), y = i >> log2n, pv = predicted(w, c, log2n, mode, x, y);
    w.pred[i] = (uint8_t)pv; w.res[i] = e.org(c, x0 + x, y0 + y) - pv;
  }
  GE_SYNC();
  if (c == 0) {
    for (int sb = e.lane; sb < (nn >> 4); sb += GE_LANES) {
      const int bx = (sb % (n >> 2)) << 2, by = (sb / (n >> 2)) << 2;
      int d[16]; for (int k = 0; k < 16; k++) d[k] = w.res[(by + (k >> 2)) * n + bx + (k & 3)];
      GE_ATOMIC_ADD(&w.acc, satd4(d));
    }
  }
  // forward transform: columns, then rows and quantisation
  for (int i = e.lane; i < nn; i += GE_LANES) w.tmp[i] = enc::fwd_col(w.res, dst4, log2n, i >> log2n, i & (n - 1), 8);
  GE_SYNC();
  for (int i = e.lane; i < nn; i += GE_LANES) {
    const int l = enc::quant_level(enc::fwd_row(w.tmp, dst4, log2n, i >> log2n, i & (n - 1)), qp, log2n, 8);
    w.lev[i] = (int16_t)l;
    if (l) w.any = 1;
  }
  GE_SYNC();
  if (final) { int16_t* cp = e.cplane(c); for (int i = e.lane; i < nn; i += GE_LANES) cp[(size_t)(y0 + (i >> log2n)) * st + x0 + (i & (n - 1))] = w.lev[i]; }
  uint8_t* rp = e.plane(c);
  if (w.any) {
    for (int i = e.lane; i < nn; i += GE_LANES) w.coef[i] = enc::dequant(w.lev[i], 16, qp, log2n, 8);
    GE_SYNC();
    for (int i = e.lane; i < nn; i += GE_LANES) w.tmp[i] = enc::inv_col(w.coef, dst4, log2n, i >> log2n, i & (n - 1));
    GE_SYNC();
    for (int i = e.lane; i < nn; i += GE_LANES) {
      const int y = i >> log2n, x = i & (n - 1);
      rp[(size_t)(y0 + y) * st + x0 + x] = (uint8_t)clip3(0, 255, w.pred[i] + enc::inv_row(w.tmp, dst4, log2n, y, x, 8));
    }
  } else {
    for (int i = e.lane; i < nn; i += GE_LANES) rp[(size_t)(y0 + (i >> log2n)) * st + x0 + (i & (n - 1))] = w.pred[i];
  }
  if (c == 0) {
    const int n4 = n >> 2; uint8_t* d = e.dec();
    for (int i = e.lane; i < n4 * n4; i += GE_LANES) d[(size_t)((y0 >> 2) + i / n4) * (e.a.W >> 2) + (x0 >> 2) + i % n4] = 1;
  }
  GE_SYNC();
  return w.acc;
}

__device__ void set_modes(Ctx2& e, int x0, int y0, int n, int mode) {
  const int n4 = n >> 2; uint8_t* m = e.ipm();
  for (int i = e.lane; i < n4 * n4; i += GE_LANES) m[(size_t)((y0 >> 2) + i / n4) * (e.a.W >> 2) + (x0 >> 2) + i % n4] = (uint8_t)mode;
  GE_SYNC();
}
__device__ void set_cu(Ctx2& e, int x0, int y0, int n, int v) {
  const int n8 = n >> 3; uint8_t* m = e.cu();
  for (int i = e.lane; i < n8 * n8; i += GE_LANES) m[(size_t)((y0 >> 3) + i / n8) * (e.a.W >> 3) + (x0 >> 3) + i % n8] = (uint8_t)v;
  GE_SYNC();
}
// save / restore / invalidate the luma reconstruction (Samples) and modes of an n x n region (decision pass)
template <bool Samples>
__device__ void region(Ctx2& e, int x0, int y0, int n, uint8_t* buf, int op /* 0 save, 1 restore, 2 mark not reconstructed */) {
  const int W = e.a.W, n4 = n >> 2; uint8_t* pl = e.plane(0); uint8_t* m = e.ipm(); uint8_t* d = e.dec();
  const int nm = Samples ? n * n : 0;                         // where the modes start in buf
  if constexpr (Samples)
    for (int i = e.lane; i < n * n; i += GE_LANES) {
      uint8_t* p = pl + (size_t)(y0 + i / n) * W + x0 + i % n;
      if (op == 0) buf[i] = *p; else if (op == 1) *p = buf[i];
    }
  for (int i = e.lane; i < n4 * n4; i += GE_LANES) {
    const size_t k = (size_t)((y0 >> 2) + i / n4) * (W >> 2) + (x0 >> 2) + i % n4;
    if (op == 0) buf[nm + i] = m[k]; else if (op == 1) m[k] = buf[nm + i]; else d[k] = 0;
  }
  GE_SYNC();
}

// open-loop decisions: the n x n luma block at (x0, y0) counts as reconstructed from here on (z-scan availability of the
// PUs that follow), as code_tb marks it in closed loop
__device__ void mark_coded(Ctx2& e, int x0, int y0, int n) {
  const int n4 = n >> 2; uint8_t* d = e.dec();
  for (int i = e.lane; i < n4 * n4; i += GE_LANES) d[(size_t)((y0 >> 2) + i / n4) * (e.a.W >> 2) + (x0 >> 2) + i % n4] = 1;
  GE_SYNC();
}

// open-loop SATD of the 32x32 luma block at (x0, y0) predicted with `mode` from the source; marks it coded
__device__ int satd_open(Ctx2& e, int x0, int y0, int mode) {
  Work& w = e.w;
  gather_refs<true>(e, 0, x0, y0, 5);
  if (e.lane == 0) w.satd[mode] = 0;
  GE_SYNC();
  add_satd(e, x0, y0, 5, 1, [mode](int) { return mode; });
  mark_coded(e, x0, y0, 32);
  return w.satd[mode];
}

// luma of one CU: closed loop (S < 2: the CU's TBs reconstructed), or open loop (S = 2: the J of the mode search alone);
// returns J x 16
template <int S>
__device__ long long eval_cu(Ctx2& e, int x0, int y0, int log2cb, bool nxn) {
  long long j = 0, jm;
  if (e.lane == 0) atomicAdd(e.a.work + 1, 1ull);
  if (nxn) {
    for (int k = 0; k < 4; k++) {
      const int px = x0 + (k & 1) * 4, py = y0 + (k >> 1) * 4;
      const int m = search_mode<S>(e, px, py, 2, &jm);
      set_modes(e, px, py, 4, m);
      if constexpr (S == 2) mark_coded(e, px, py, 4);
      else code_tb(e, 0, px, py, 2, m, false);
      j += jm;
    }
    return j + e.a.lambda16;                                  // part_mode bin
  }
  const int lg = log2cb < 5 ? log2cb : 5;
  const int m = search_mode<S>(e, x0, y0, lg, &jm);           // a 64x64 CU: chosen on its first 32x32 block
  set_modes(e, x0, y0, 1 << log2cb, m);
  if constexpr (S == 2) {
    mark_coded(e, x0, y0, 1 << lg);
    if (log2cb == 6)                                           // + the open-loop SATDs of the other three 32x32 blocks
      for (int k = 1; k < 4; k++) j += (long long)satd_open(e, x0 + (k & 1) * 32, y0 + (k >> 1) * 32, m) << 4;
    return jm + j;
  } else {
    if (log2cb < 6) { code_tb(e, 0, x0, y0, log2cb, m, false); return jm; }
    j = jm - ((long long)e.w.satd[m] << 4);
    for (int k = 0; k < 4; k++) j += (long long)code_tb(e, 0, x0 + (k & 1) * 32, y0 + (k >> 1) * 32, 5, m, false) << 4;
    return j;
  }
}

// decision pass: bottom-up quadtree, leaves the chosen luma reconstruction (closed loop) / modes / CU sizes; returns J x 16
// (The quadtree walks are templates on the block size: no run-time recursion, so the stack size is known at compile time.)
template <int S, int L>
__device__ long long decide(Ctx2& e, int x0, int y0, int depth) {
  const int n = 1 << L, log2cb = L;
  if (x0 + n > e.a.W || y0 + n > e.a.H) {                     // crosses the picture border: split implied
    long long j = 0;
    if constexpr (L > 3)
      for (int k = 0; k < 4; k++) { const int x1 = x0 + (k & 1) * (n >> 1), y1 = y0 + (k >> 1) * (n >> 1); if (x1 < e.a.W && y1 < e.a.H) j += decide<S, L - 1>(e, x1, y1, depth + 1); }
    return j;
  }
  const long long j0 = eval_cu<S>(e, x0, y0, log2cb, false);
  uint8_t* buf = static_cast<E1Work<S>&>(e.w).save[depth];
  region<S != 2>(e, x0, y0, n, buf, 0);
  region<S != 2>(e, x0, y0, n, buf, 2);
  long long j1;
  if constexpr (L == 3) j1 = eval_cu<S>(e, x0, y0, 3, true);
  else {
    j1 = e.a.lambda16;                                         // split_cu_flag
    for (int k = 0; k < 4; k++) j1 += decide<S, L - 1>(e, x0 + (k & 1) * (n >> 1), y0 + (k >> 1) * (n >> 1), depth + 1);
  }
  if (j0 <= j1) { region<S != 2>(e, x0, y0, n, buf, 1); set_cu(e, x0, y0, n, log2cb); return j0; }
  if (log2cb == 3) set_cu(e, x0, y0, 8, 3 | CU_NXN);
  return j1;
}

// final pass: the chosen CUs again, luma and chroma in decoding order, levels into the coefficient plane
template <int L>
__device__ void finalize(Ctx2& e, int x0, int y0) {
  if (x0 >= e.a.W || y0 >= e.a.H) return;
  const int n = 1 << L, W = e.a.W, log2cb = L;
  const int cell = GE_LD(e.cu() + (size_t)(y0 >> 3) * (W >> 3) + (x0 >> 3));
  if constexpr (L > 3)
    if ((cell & 7) < log2cb) { for (int k = 0; k < 4; k++) finalize<L - 1>(e, x0 + (k & 1) * (n >> 1), y0 + (k >> 1) * (n >> 1)); return; }
  const int mode = GE_LD(e.ipm() + (size_t)(y0 >> 2) * (W >> 2) + (x0 >> 2));
  const bool chroma = e.a.cfmt != 0;
  if (cell & CU_NXN) {
    for (int k = 0; k < 4; k++) {
      const int px = x0 + (k & 1) * 4, py = y0 + (k >> 1) * 4;
      code_tb(e, 0, px, py, 2, GE_LD(e.ipm() + (size_t)(py >> 2) * (W >> 2) + (px >> 2)), true);
    }
    if (chroma) { code_tb(e, 1, x0 >> 1, y0 >> 1, 2, mode, true); code_tb(e, 2, x0 >> 1, y0 >> 1, 2, mode, true); }
    return;
  }
  const int lt = log2cb < 5 ? log2cb : 5, nt = 1 << lt;
  for (int k = 0; k < (log2cb == 6 ? 4 : 1); k++) {
    const int tx = x0 + (k & 1) * nt, ty = y0 + (k >> 1) * nt;
    code_tb(e, 0, tx, ty, lt, mode, true);
    if (chroma) { code_tb(e, 1, tx >> 1, ty >> 1, lt - 1, mode, true); code_tb(e, 2, tx >> 1, ty >> 1, lt - 1, mode, true); }
  }
}

__device__ inline unsigned ld_relaxed(const unsigned* p) {
  unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
// lane 0 polls with back-off (relaxed loads), then one fence orders the reads that follow (DESIGN 4 (i) / (iii))
__device__ inline void wait_for(const unsigned* p, unsigned v, int lane) {
  if (lane == 0) {
    unsigned ns = 64;
    while (ld_relaxed(p) < v) { __nanosleep(ns); if (ns < 4096) ns <<= 1; }
    __threadfence();
  }
  __syncwarp();
}
__device__ inline void publish(unsigned* p, unsigned v, int lane) {
  __syncwarp();
  if (lane == 0) { __threadfence(); atomicExch(p, v); }
}

template <int S>
__device__ void e1_row(const Args& a, Work& w, int p, int ry, int lane) {
  Ctx2 e{a, p, lane, w};
  const size_t row = (size_t)p * a.hctb + ry;
  for (int rx = 0; rx < a.wctb; rx++) {
    if (ry > 0) wait_for(a.progress + row - 1, (unsigned)min(rx + 2, a.wctb), lane);
    const int x0 = rx << a.log2ctb, y0 = ry << a.log2ctb;
    if (a.log2ctb == 6) decide<S, 6>(e, x0, y0, 0); else decide<S, 5>(e, x0, y0, 0);
    {                                                          // the final pass sees the CTB's blocks appear in decoding order again
      const int w4 = min(1 << a.log2ctb, a.W - x0) >> 2, h4 = min(1 << a.log2ctb, a.H - y0) >> 2;
      for (int i = lane; i < w4 * h4; i += GE_LANES) e.dec()[(size_t)((y0 >> 2) + i / w4) * (a.W >> 2) + (x0 >> 2) + i % w4] = 0;
      GE_SYNC();
    }
    if (a.log2ctb == 6) finalize<6>(e, x0, y0); else finalize<5>(e, x0, y0);
    publish(a.progress + row, (unsigned)(rx + 1), lane);
  }
}

// ---------------------------------------------------------------------------------------------------- E2
// E2's bit sink: the row's buffer of `cap` bytes; a sub-stream that would pass it sets `overflow` instead of writing
struct RowSink {
  uint8_t* out; size_t cap, pos; unsigned cur; int nbits; bool overflow;
  B200_HD void put1(unsigned b) {
    cur = (cur << 1) | b;
    if (++nbits == 8) { if (pos < cap) out[pos++] = (uint8_t)cur; else overflow = true; cur = 0; nbits = 0; }
  }
  B200_HD void put(unsigned v, int n) { for (int i = n - 1; i >= 0; i--) put1((v >> i) & 1); }
  B200_HD void align_zero() { while (nbits) put1(0); }
};
using Cabac = enc::CabacWriter<RowSink>;

struct Writer {
  const Args& a; int p; Cabac& cb;
  __device__ int cu_at(int x, int y) const { return a.cu8[(size_t)p * a.map8 + (size_t)(y >> 3) * (a.W >> 3) + (x >> 3)]; }
  __device__ const int16_t* cplane(int c) const { return a.coef + (size_t)p * a.pic_samples + (c == 0 ? 0 : (size_t)a.W * a.H + (size_t)(c - 1) * a.Wc * a.Hc); }
  __device__ bool nonzero(int c, int x0, int y0, int n) const {
    const int st = c ? a.Wc : a.W; const int16_t* pl = cplane(c);
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) if (pl[(size_t)(y0 + y) * st + x0 + x]) return true;
    return false;
  }

  __device__ void residual(int c, int x0, int y0, int log2n, int scan) {
    const int st = c ? a.Wc : a.W;
    enc::residual_coding(cb, cplane(c) + (size_t)y0 * st + x0, st, log2n, c, scan, false, false, false);
  }

  // transform tree (7.3.8.8 / 7.3.8.10): TU = CU apart from the implied splits
  template <int L>
  __device__ void tree(int x0, int y0, int depth, int blk, bool nxn, int max_depth, const int lmode[4], int cmode, bool pcb, bool pcr, int cux, int cuy) {
    using namespace syn;
    const int log2n = L;
    const bool chroma = a.cfmt != 0;
    const bool can_split = log2n <= 5 && log2n > 2 && depth < max_depth && !(nxn && depth == 0);
    const bool split = !can_split && (log2n > 5 || (nxn && depth == 0));
    if (can_split) cb.bin(CTX_SPLIT_TR + 5 - log2n, 0);
    bool ccb = false, ccr = false;
    if (chroma) {
      if (log2n > 2) {
        const int nc = 1 << (log2n - 1);
        if (depth == 0 || pcb) { ccb = nonzero(1, x0 >> 1, y0 >> 1, nc); cb.bin(CTX_CBF_CHROMA + depth, ccb); }
        if (depth == 0 || pcr) { ccr = nonzero(2, x0 >> 1, y0 >> 1, nc); cb.bin(CTX_CBF_CHROMA + depth, ccr); }
      } else { ccb = pcb; ccr = pcr; }
    }
    if constexpr (L > 2)
      if (split) {
        const int h = 1 << (log2n - 1);
        for (int k = 0; k < 4; k++) tree<L - 1>(x0 + (k & 1) * h, y0 + (k >> 1) * h, depth + 1, k, nxn, max_depth, lmode, cmode, ccb, ccr, cux, cuy);
        return;
      }
    const int pu = nxn ? ((y0 > cuy) ? 2 : 0) + ((x0 > cux) ? 1 : 0) : 0;
    const bool cbf_l = nonzero(0, x0, y0, 1 << log2n);
    cb.bin(CTX_CBF_LUMA + (depth == 0 ? 1 : 0), cbf_l);
    if (cbf_l) residual(0, x0, y0, log2n, log2n <= 3 ? enc::scan_idx(lmode[pu]) : 0);
    if (chroma) {
      if (log2n > 2) {
        if (ccb) residual(1, x0 >> 1, y0 >> 1, log2n - 1, log2n - 1 == 2 ? enc::scan_idx(cmode) : 0);
        if (ccr) residual(2, x0 >> 1, y0 >> 1, log2n - 1, log2n - 1 == 2 ? enc::scan_idx(cmode) : 0);
      } else if (blk == 3) {
        if (pcb) residual(1, cux >> 1, cuy >> 1, 2, enc::scan_idx(cmode));
        if (pcr) residual(2, cux >> 1, cuy >> 1, 2, enc::scan_idx(cmode));
      }
    }
  }

  template <int L>
  __device__ void quadtree(int x0, int y0, int depth) {
    using namespace syn;
    const int n = 1 << L, W = a.W, H = a.H, log2cb = L;
    const int cell = cu_at(x0, y0);
    bool split;
    if (x0 + n <= W && y0 + n <= H && log2cb > 3) {
      split = (cell & 7) < log2cb;
      int inc = 0;
      if (x0 > 0 && a.log2ctb - (cu_at(x0 - 1, y0) & 7) > depth) inc++;
      if (y0 > 0 && a.log2ctb - (cu_at(x0, y0 - 1) & 7) > depth) inc++;
      cb.bin(CTX_SPLIT_CU + inc, split);
    } else split = log2cb > 3;
    if constexpr (L > 3)
      if (split) {
        const int h = n >> 1;
        for (int k = 0; k < 4; k++) { const int x1 = x0 + (k & 1) * h, y1 = y0 + (k >> 1) * h; if (x1 < W && y1 < H) quadtree<L - 1>(x1, y1, depth + 1); }
        return;
      }
    // coding_unit (7.3.8.5)
    const bool nxn = log2cb == 3 && (cell & CU_NXN);
    if (log2cb == 3) cb.bin(CTX_PART_MODE, !nxn);
    const int np = nxn ? 4 : 1, pb = nxn ? n / 2 : n;
    const uint8_t* ipm = a.ipm4 + (size_t)p * a.map4;
    int lmode[4] = {0, 0, 0, 0}, code[4];
    for (int i = 0; i < np; i++) {
      const int px = x0 + (i & 1) * pb, py = y0 + (i >> 1) * pb;
      int cand[3]; mpm_cand(ipm, W >> 2, a.log2ctb, px, py, cand);
      const int mode = ipm[(size_t)(py >> 2) * (W >> 2) + (px >> 2)];
      lmode[i] = mode; code[i] = enc::mpm_code(mode, cand);
    }
    enc::write_luma_modes(cb, np, code);
    if (a.cfmt) cb.bin(CTX_CHROMA_PRED, 0);                    // intra_chroma_pred_mode = 4 (DM)
    tree<L>(x0, y0, 0, 0, nxn, a.max_th_depth + (nxn ? 1 : 0), lmode, lmode[0], false, false, x0, y0);
  }
};

__device__ void e2_row(const Args& a, uint8_t* ctx, int p, int ry, int lane) {
  const size_t row = (size_t)p * a.hctb + ry;
  if (lane == 0) {
    Cabac cb{RowSink{a.ss + row * a.ss_cap, a.ss_cap, 0, 0, 0, false}, ctx};
    Writer wr{a, p, cb};
    if (ry > 0 && a.wctb >= 2) {
      const uint8_t* src = a.wpp_ctx + (row - 1) * syn::CTX_COUNT;
      for (int i = 0; i < syn::CTX_COUNT; i++) ctx[i] = GE_LD(src + i);
    } else enc::init_contexts(ctx, a.slice_qp);
    for (int rx = 0; rx < a.wctb; rx++) {
      if (a.log2ctb == 6) wr.quadtree<6>(rx << a.log2ctb, ry << a.log2ctb, 0); else wr.quadtree<5>(rx << a.log2ctb, ry << a.log2ctb, 0);
      if (rx == 1) {
        uint8_t* dst = a.wpp_ctx + row * syn::CTX_COUNT;
        for (int i = 0; i < syn::CTX_COUNT; i++) dst[i] = ctx[i];
        __threadfence(); atomicExch(a.progress2 + row, 1u);
      }
      const bool last = ry == a.hctb - 1 && rx == a.wctb - 1;
      cb.terminate(last ? 1 : 0);                              // end_of_slice_segment_flag
      if (!last && rx == a.wctb - 1) cb.terminate(1);          // end_of_subset_one_bit + byte_alignment()
    }
    a.ss_len[row] = (unsigned)cb.bits.pos;
    if (cb.bits.overflow) atomicOr(a.error, 1u);
  }
}

template <int S>
__global__ void __launch_bounds__(32) e1_kernel(Args a) {
  __shared__ E1Work<S> w;
  __shared__ unsigned t;
  if (threadIdx.x == 0) t = atomicAdd(a.ticket, 1u);
  __syncwarp();
  const unsigned row = t;
  __syncwarp();
  e1_row<S>(a, w, (int)(row / a.hctb), (int)(row % a.hctb), threadIdx.x);
}

__global__ void __launch_bounds__(32) e2_kernel(Args a) {
  __shared__ uint8_t ctx[syn::CTX_COUNT];
  __shared__ unsigned t;
  if (threadIdx.x == 0) t = atomicAdd(a.ticket + 1, 1u);
  __syncwarp();
  const unsigned row = t;
  const int p = (int)(row / a.hctb), ry = (int)(row % a.hctb);
  if (ry > 0 && a.wctb >= 2) wait_for(a.progress2 + row - 1, 1u, threadIdx.x);
  e2_row(a, ctx, p, ry, threadIdx.x);
}

// gathers the sub-streams of all rows into one packed buffer (offsets from the host's prefix sum)
__global__ void pack_kernel(const uint8_t* ss, size_t cap, const unsigned* len, const unsigned long long* off, uint8_t* out) {
  const size_t row = blockIdx.x;
  const uint8_t* s = ss + row * cap; uint8_t* d = out + off[row];
  for (unsigned i = threadIdx.x; i < len[row]; i += blockDim.x) d[i] = s[i];
}

// test-only (b200_debug_enc_transform_device): CTA (block i, stage st), one thread per output element
__global__ void debug_transform_kernel(const int* prm, const int* in, int* out) {
  const int i = blockIdx.x, st = blockIdx.y;
  const int* p = prm + i * enc::DT_FIELDS;
  const int lg = p[enc::DT_LOG2N], n = 1 << lg;
  for (int e = threadIdx.x; e < n * n; e += blockDim.x)
    out[((size_t)i * enc::DT_STAGES + st) * 1024 + e] = enc::debug_transform_stage(st, p, in + (size_t)i * 1024, e >> lg, e & (n - 1));
}

// test-only (b200_debug_enc_predict_device): one CTA per block; thread 0 substitutes and filters the neighbours, every
// thread predicts samples of all 35 modes
__global__ void debug_predict_kernel(const int* prm, const int16_t* refs, int16_t* rf, int* pred) {
  __shared__ int16_t r[129], f[129];
  __shared__ int dc;
  const int i = blockIdx.x;
  const int* p = prm + i * enc::DP_FIELDS;
  const int lg = p[enc::DP_LOG2N], bd = p[enc::DP_BD], n = 1 << lg;
  if (threadIdx.x == 0) {
    for (int k = 0; k < 129; k++) r[k] = refs[(size_t)i * 129 + k];
    enc::substitute_refs(r, n, bd);
    enc::filter_refs(r, f, lg, p[enc::DP_STRONG] != 0, bd);
    dc = enc::dc_value(r, lg);
  }
  __syncthreads();
  for (int k = threadIdx.x; k < 129; k += blockDim.x) { rf[(size_t)i * 258 + k] = r[k]; rf[(size_t)i * 258 + 129 + k] = f[k]; }
  for (int e = threadIdx.x; e < 35 * n * n; e += blockDim.x) {
    const int mode = e >> (2 * lg), s = e & (n * n - 1);
    const bool filt = enc::refs_filtered(p[enc::DP_PLANE] != 0, mode, lg);
    pred[((size_t)i * 35 + mode) * 1024 + s] = enc::pred_sample(filt ? f : r, dc, lg, mode, s & (n - 1), s >> lg, p[enc::DP_LUMA] != 0, (1 << bd) - 1);
  }
}

}  // namespace genc
}  // namespace b200

// ---------------------------------------------------------------------------------------------------- host side
struct b200_gpu_encoder {
  b200::Pool pool{std::max(1, std::min(16, (int)std::thread::hardware_concurrency()))};
  b200::Bounce bounce;
  b200::Stream stream;
  b200::Stream work;                  // colour stage + encode of b200_gpu_encode_rgb_grid_host (`stream` carries its uploads)
  b200::Event ev[3];
  b200::DevBuf<uint8_t> rgb;          // b200_gpu_encode_rgb_grid_host: the uploaded RGB
  b200::DevBuf<uint8_t> src, rec, ipm4, dec4, cu8, wpp_ctx, ss, packed;
  b200::DevBuf<int16_t> coef;
  b200::DevBuf<unsigned> sync, ss_len;
  b200::DevBuf<unsigned long long> off, counters;
  b200::DevBuf<b200::genc::Pic> pics;
  std::vector<std::vector<uint8_t>> out;
  b200_hevc_enc_params params{};
  int n = 0, W = 0, H = 0, cfmt = 1;
  int rec_first = 0;                  // output index of the first picture whose reconstruction `rec` holds
  b200_gpu_encode_stats stats{};
  bool ready = false;
};

namespace b200 {
namespace genc {

int validate(const b200_hevc_enc_params* p, int n, const b200_planes* pics) {
  if (!p || !pics) return set_error(B200_E_INVALID, "null argument");
  if (n <= 0) return set_error(B200_E_INVALID, "picture count %d", n);
  if (p->width < 8 || p->height < 8 || p->width > 16384 || p->height > 16384) return set_error(B200_E_INVALID, "size %dx%d", p->width, p->height);
  if (p->speed < 0 || p->speed > 2) return set_error(B200_E_INVALID, "speed %d: 0, 1 or 2", p->speed);
  if (p->bit_depth != 8) return set_error(B200_E_UNSUPPORTED, "bit_depth %d: the GPU encoder codes 8-bit pictures", p->bit_depth);
  if (p->chroma_format_idc != 0 && p->chroma_format_idc != 1) return set_error(B200_E_UNSUPPORTED, "chroma_format_idc %d: 4:2:0 and 4:0:0 only", p->chroma_format_idc);
  if (p->log2_ctb_size != 5 && p->log2_ctb_size != 6) return set_error(B200_E_UNSUPPORTED, "log2_ctb_size %d: 5 or 6", p->log2_ctb_size);
  if (p->qp < 0 || p->qp > 51 || p->init_qp < 0 || p->init_qp > 51) return set_error(B200_E_INVALID, "qp %d / init_qp %d", p->qp, p->init_qp);
  if (p->max_transform_hierarchy_depth_intra < 0 || p->max_transform_hierarchy_depth_intra > 4) return set_error(B200_E_INVALID, "max_transform_hierarchy_depth_intra %d", p->max_transform_hierarchy_depth_intra);
  if (abs(p->cb_qp_offset) > 12 || abs(p->cr_qp_offset) > 12 || abs(p->slice_cb_qp_offset) > 12 || abs(p->slice_cr_qp_offset) > 12 ||
      abs(p->cb_qp_offset + p->slice_cb_qp_offset) > 12 || abs(p->cr_qp_offset + p->slice_cr_qp_offset) > 12)
    return set_error(B200_E_INVALID, "chroma QP offsets");
  if (abs(p->beta_offset_div2) > 6 || abs(p->tc_offset_div2) > 6 || abs(p->slice_beta_offset_div2) > 6 || abs(p->slice_tc_offset_div2) > 6)
    return set_error(B200_E_INVALID, "deblocking offsets");
  static const struct { const char* name; int off; } refused[] = {
    {"sao", offsetof(b200_hevc_enc_params, sao)}, {"sign_data_hiding", offsetof(b200_hevc_enc_params, sign_data_hiding)},
    {"transform_skip", offsetof(b200_hevc_enc_params, transform_skip)}, {"cu_qp_delta", offsetof(b200_hevc_enc_params, cu_qp_delta)},
    {"scaling_lists", offsetof(b200_hevc_enc_params, scaling_lists)}, {"pcm", offsetof(b200_hevc_enc_params, pcm)},
    {"transquant_bypass", offsetof(b200_hevc_enc_params, transquant_bypass)}, {"slice_ctb_rows", offsetof(b200_hevc_enc_params, slice_ctb_rows)},
    {"dependent_slice_segments", offsetof(b200_hevc_enc_params, dependent_slice_segments)}};
  for (const auto& r : refused)
    if (*(const int*)((const char*)p + r.off)) return set_error(B200_E_UNSUPPORTED, "%s: not supported by the GPU encoder", r.name);
  if (p->tile_cols > 1 || p->tile_rows > 1) return set_error(B200_E_UNSUPPORTED, "tile_cols / tile_rows: tiles are not supported by the GPU encoder");
  if (!p->wpp) return set_error(B200_E_UNSUPPORTED, "wpp = 0: the GPU encoder codes one WPP sub-stream per CTB row");
  const int want_chroma = p->chroma_format_idc ? B200_CHROMA_420 : B200_CHROMA_MONO;
  for (int i = 0; i < n; i++) {
    const b200_planes& q = pics[i];
    if (!q.y || (p->chroma_format_idc && (!q.cb || !q.cr))) return set_error(B200_E_INVALID, "picture %d: missing plane", i);
    if (q.width != p->width || q.height != p->height) return set_error(B200_E_INVALID, "picture %d: %dx%d, the call codes %dx%d", i, q.width, q.height, p->width, p->height);
    if (q.chroma != want_chroma) return set_error(B200_E_INVALID, "picture %d: chroma %d, the call codes chroma_format_idc %d", i, q.chroma, p->chroma_format_idc);
    if (q.bit_depth != 8) return set_error(B200_E_UNSUPPORTED, "picture %d: bit depth %d", i, q.bit_depth);
    if (q.y_stride < (size_t)q.width || (p->chroma_format_idc && q.c_stride < (size_t)((q.width + 1) >> 1))) return set_error(B200_E_INVALID, "picture %d: stride", i);
  }
  return B200_OK;
}

// SATD-domain Lagrangian: lambda = sqrt(0.57 * 2^((QP - 12) / 3)), in 1/16 units
inline int lambda16(int qp) { return (int)(16.0 * std::sqrt(0.57 * std::pow(2.0, (qp - 12) / 3.0)) + 0.5); }

int encode(b200_gpu_encoder* e, const b200_hevc_enc_params* p, int n, const Pic* host_pics, cudaStream_t s) {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  e->ready = false;
  const int W = (p->width + 7) & ~7, H = (p->height + 7) & ~7, cfmt = p->chroma_format_idc, log2ctb = p->log2_ctb_size;
  const int Wc = cfmt ? W / 2 : 0, Hc = cfmt ? H / 2 : 0, ctb = 1 << log2ctb;
  const int wctb = (W + ctb - 1) >> log2ctb, hctb = (H + ctb - 1) >> log2ctb;
  const size_t rows = (size_t)n * hctb, pic_samples = (size_t)W * H + 2 * (size_t)Wc * Hc;
  const size_t map4 = (size_t)(W / 4) * (H / 4), map8 = (size_t)(W / 8) * (H / 8);
  const size_t cap = substream_capacity(p->width, log2ctb, cfmt);
  int rc;
  if ((rc = e->rec.reserve(n * pic_samples, false)) || (rc = e->coef.reserve(n * pic_samples, false)) || (rc = e->ipm4.reserve(n * map4, false)) ||
      (rc = e->dec4.reserve(n * map4, false)) || (rc = e->cu8.reserve(n * map8, false)) || (rc = e->wpp_ctx.reserve(rows * syn::CTX_COUNT, false)) ||
      (rc = e->ss.reserve(rows * cap, false)) || (rc = e->sync.reserve(2 * rows + 3, false)) || (rc = e->ss_len.reserve(rows)) ||
      (rc = e->off.reserve(rows)) || (rc = e->pics.reserve(n)) || (rc = e->counters.reserve(2)))
    return rc;
  for (int i = 0; i < n; i++) e->pics.h[i] = host_pics[i];
  B200_CUDA_CHECK(cudaMemcpyAsync(e->pics.d, e->pics.h, n * sizeof(Pic), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemsetAsync(e->dec4.d, 0, n * map4, s));
  B200_CUDA_CHECK(cudaMemsetAsync(e->sync.d, 0, (2 * rows + 3) * sizeof(unsigned), s));
  B200_CUDA_CHECK(cudaMemsetAsync(e->counters.d, 0, 2 * sizeof(unsigned long long), s));
  Args a{};
  a.pics = e->pics.d; a.n = n; a.W = W; a.H = H; a.Wc = Wc; a.Hc = Hc; a.sw = p->width; a.sh = p->height;
  a.cfmt = cfmt; a.log2ctb = log2ctb; a.wctb = wctb; a.hctb = hctb; a.max_th_depth = p->max_transform_hierarchy_depth_intra;
  a.strong = p->strong_intra_smoothing != 0; a.slice_qp = p->qp;
  a.qp[0] = p->qp; a.qp[1] = enc::chroma_qp(p->qp + p->cb_qp_offset + p->slice_cb_qp_offset * (p->slice_chroma_qp_offsets != 0), cfmt, 8);
  a.qp[2] = enc::chroma_qp(p->qp + p->cr_qp_offset + p->slice_cr_qp_offset * (p->slice_chroma_qp_offsets != 0), cfmt, 8);
  a.lambda16 = lambda16(p->qp);
  a.rec = e->rec.d; a.coef = e->coef.d; a.pic_samples = pic_samples; a.ipm4 = e->ipm4.d; a.dec4 = e->dec4.d; a.map4 = map4;
  a.cu8 = e->cu8.d; a.map8 = map8;
  a.progress = e->sync.d; a.progress2 = e->sync.d + rows; a.ticket = e->sync.d + 2 * rows; a.error = e->sync.d + 2 * rows + 2;
  a.wpp_ctx = e->wpp_ctx.d; a.ss = e->ss.d; a.ss_cap = cap; a.ss_len = e->ss_len.d; a.work = e->counters.d;
  B200_CUDA_CHECK(cudaEventRecord(e->ev[0], s));
  switch (p->speed) {
    case 0: e1_kernel<0><<<(unsigned)rows, 32, 0, s>>>(a); break;
    case 1: e1_kernel<1><<<(unsigned)rows, 32, 0, s>>>(a); break;
    default: e1_kernel<2><<<(unsigned)rows, 32, 0, s>>>(a); break;
  }
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(e->ev[1], s));
  e2_kernel<<<(unsigned)rows, 32, 0, s>>>(a);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaEventRecord(e->ev[2], s));
  B200_CUDA_CHECK(cudaMemcpyAsync(e->ss_len.h, e->ss_len.d, rows * sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(e->counters.h, e->counters.d, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
  unsigned err = 0;
  B200_CUDA_CHECK(cudaMemcpyAsync(&err, a.error, sizeof(unsigned), cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  const auto t1 = clk::now();
  if (err) return set_error(B200_E_LIMIT, "a sub-stream exceeded its worst-case buffer of %zu bytes", cap);
  size_t total = 0;
  for (size_t r = 0; r < rows; r++) { e->off.h[r] = total; total += e->ss_len.h[r]; }
  if ((rc = e->packed.reserve(total + 1))) return rc;
  B200_CUDA_CHECK(cudaMemcpyAsync(e->off.d, e->off.h, rows * sizeof(unsigned long long), cudaMemcpyHostToDevice, s));
  pack_kernel<<<(unsigned)rows, 256, 0, s>>>(e->ss.d, cap, e->ss_len.d, e->off.d, e->packed.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpyAsync(e->packed.h, e->packed.d, total, cudaMemcpyDeviceToHost, s));
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  // framing: one access unit per picture
  const std::vector<int> none;
  const enc::SeqHeader sh{p, W, H, cfmt, cfmt ? 1 : 0, 1, 1, 8, log2ctb, 2, std::min(5, log2ctb), p->max_transform_hierarchy_depth_intra, log2ctb, 8, 8,
                          false, nullptr, nullptr, false, &none, &none};
  std::vector<uint8_t> ps;
  enc::write_vps(ps, sh); enc::write_sps(ps, sh); enc::write_pps(ps, sh);
  e->out.resize(n);
  e->pool.parallel_for(n, [&](int i) {
    std::vector<size_t> esc(hctb);
    const uint8_t* base = e->packed.h + e->off.h[(size_t)i * hctb];
    size_t bytes = 0;
    for (int r = 0; r < hctb; r++) {
      const size_t row = (size_t)i * hctb + r;
      esc[r] = enc::escaped_size(e->packed.h + e->off.h[row], e->ss_len.h[row]);
      bytes += e->ss_len.h[row];
    }
    enc::BitWriter b;
    enc::write_slice_header(b, sh, 0, false, p->qp, esc);
    b.buf.insert(b.buf.end(), base, base + bytes);
    std::vector<uint8_t>& o = e->out[i];
    o.assign(ps.begin(), ps.end());
    enc::append_nal(o, 19 /* IDR_W_RADL */, b.buf);
  });
  const auto t2 = clk::now();
  float ms1 = 0, ms2 = 0;
  cudaEventElapsedTime(&ms1, e->ev[0], e->ev[1]);
  cudaEventElapsedTime(&ms2, e->ev[1], e->ev[2]);
  b200_gpu_encode_stats& st = e->stats;
  st.analyse_ms = ms1; st.entropy_ms = ms2;
  st.framing_ms = std::chrono::duration<double, std::milli>(t2 - t1).count();
  st.total_ms = std::chrono::duration<double, std::milli>(t2 - t0).count();
  st.bytes = 0; for (auto& o : e->out) st.bytes += o.size();
  st.ctus = (uint64_t)rows * wctb; st.pictures = (uint64_t)n;
  st.mode_evaluations = e->counters.h[0]; st.cu_evaluations = e->counters.h[1];
  e->params = *p; e->n = n; e->W = W; e->H = H; e->cfmt = cfmt; e->rec_first = 0; e->ready = true;
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------------- RGB grid in one call
struct GridPlan {
  int cols, rows, pw, ph, pipeline;
  bool alpha, interleaved;
  b200_hevc_enc_params q;             // the colour tiles' parameters (tile size, 4:2:0)
};

int grid_check(const b200_rgb_image* in, int tw, int th, const b200_hevc_enc_params* p, const b200_rgb_to_ycbcr_options* opt, GridPlan* g) {
  if (!in || !p) return set_error(B200_E_INVALID, "null argument");
  if (in->bit_depth > 8) return set_error(B200_E_UNSUPPORTED, "bit depth %d: the grid encoder takes 8-bit RGB (the GPU encoder codes 8-bit pictures)", in->bit_depth);
  g->interleaved = in->chroma == B200_CHROMA_INTERLEAVED_RGB || in->chroma == B200_CHROMA_INTERLEAVED_RGBA;
  if (!g->interleaved && in->chroma != B200_CHROMA_444)
    return set_error(B200_E_UNSUPPORTED, "RGB input chroma %d: the grid encoder takes RGB24, RGBA32 or planar 8-bit RGB", in->chroma);
  if (in->chroma == B200_CHROMA_444 && in->alpha && in->alpha_bit_depth > 8)
    return set_error(B200_E_UNSUPPORTED, "alpha bit depth %d: the grid encoder takes 8-bit alpha", in->alpha_bit_depth);
  if ((tw | th) & 1 || tw < 8 || th < 8 || tw > 16384 || th > 16384)
    return set_error(B200_E_INVALID, "tile size %dx%d: even sizes from 8 to 16384", tw, th);
  if (in->width <= 0 || in->height <= 0) return set_error(B200_E_INVALID, "picture size %dx%d", in->width, in->height);
  b200_planes t{};                    // the conversion target: what the SPS signals
  t.width = in->width; t.height = in->height; t.chroma = B200_CHROMA_420; t.bit_depth = 8;
  t.colour_primaries = p->colour_primaries; t.transfer_characteristics = p->transfer_characteristics;
  t.matrix_coefficients = p->matrix_coefficients; t.full_range = p->full_range;
  if (int rc = plan_rgb_to_ycbcr(in, &t, opt, &g->pipeline)) return rc;
  g->alpha = in->chroma == B200_CHROMA_INTERLEAVED_RGBA || (in->chroma == B200_CHROMA_444 && in->alpha);
  if (g->interleaved) {
    if (!in->rgb) return set_error(B200_E_INVALID, "RGB input plane missing");
    if (in->rgb_stride < (size_t)in->width * (g->alpha ? 4 : 3)) return set_error(B200_E_INVALID, "RGB stride %zu < row of %d pixels", in->rgb_stride, in->width);
  } else {
    if (!in->r || !in->g || !in->b) return set_error(B200_E_INVALID, "RGB input planes missing");
    const size_t st[4] = {in->r_stride, in->g_stride, in->b_stride, in->alpha_stride};
    for (int c = 0; c < (g->alpha ? 4 : 3); c++)
      if (st[c] < (size_t)in->width) return set_error(B200_E_INVALID, "plane %d stride %zu < row of %d samples", c, st[c], in->width);
  }
  g->q = *p;
  g->q.width = tw; g->q.height = th;
  b200_planes d{};                    // stands for every tile: only checked for NULL, size, chroma and depth
  d.y = d.cb = d.cr = in; d.y_stride = (size_t)tw; d.c_stride = (size_t)tw / 2; d.width = tw; d.height = th; d.bit_depth = 8;
  d.chroma = p->chroma_format_idc ? B200_CHROMA_420 : B200_CHROMA_MONO;
  if (int rc = validate(&g->q, 1, &d)) return rc;
  if (p->chroma_format_idc != 1) return set_error(B200_E_UNSUPPORTED, "chroma_format_idc %d: the colour tiles are coded 4:2:0", p->chroma_format_idc);
  g->cols = (int)(((long long)in->width + tw - 1) / tw); g->rows = (int)(((long long)in->height + th - 1) / th);
  if ((long long)g->cols * tw > (1 << 30) || (long long)g->rows * th > (1 << 30) || (long long)g->cols * g->rows > (1 << 24))
    return set_error(B200_E_INVALID, "grid of %dx%d tiles of %dx%d", g->cols, g->rows, tw, th);
  g->pw = g->cols * tw; g->ph = g->rows * th;
  return B200_OK;
}

int grid_encode(b200_gpu_encoder* e, const b200_rgb_image* in, int tw, int th, const b200_hevc_enc_params* p, const b200_rgb_to_ycbcr_options* opt,
                bool host, cudaStream_t s, b200_grid_encode_info* info) {
  using clk = std::chrono::steady_clock;
  const auto t0 = clk::now();
  if (!e) return set_error(B200_E_INVALID, "null encoder");
  GridPlan g;
  if (int rc = grid_check(in, tw, th, p, opt, &g)) return rc;
  e->ready = false;
  // the padded picture: Y, Cb, Cr (and alpha) planes of pw x ph, the tiles are windows of it
  const size_t ys = ((size_t)g.pw + 63) & ~(size_t)63, cs = ((size_t)g.pw / 2 + 63) & ~(size_t)63, ph = (size_t)g.ph;
  if (int rc = e->src.reserve(ys * ph + cs * ph + (g.alpha ? ys * ph : 0), false)) return rc;
  uint8_t* const Y = e->src.d; uint8_t* const Cb = Y + ys * ph; uint8_t* const Cr = Cb + cs * (ph / 2); uint8_t* const A = Cr + cs * (ph / 2);
  b200_planes out{};
  out.y = Y; out.cb = Cb; out.cr = Cr; out.alpha = g.alpha ? A : nullptr; out.y_stride = out.alpha_stride = ys; out.c_stride = cs;
  out.width = g.pw; out.height = g.ph; out.chroma = B200_CHROMA_420; out.bit_depth = 8;
  out.colour_primaries = p->colour_primaries; out.transfer_characteristics = p->transfer_characteristics;
  out.matrix_coefficients = p->matrix_coefficients; out.full_range = p->full_range;
  const int W = in->width, H = in->height;
  int nb = 1;                         // row bands of the host form
  size_t band = (size_t)H;
  b200_rgb_image d = *in;             // the input as the colour stage reads it
  const int nplanes = g.interleaved ? 1 : (g.alpha ? 4 : 3);
  const size_t wb = g.interleaved ? (size_t)W * (g.alpha ? 4 : 3) : (size_t)W;
  if (host) {
    band = std::max<size_t>(2, (((size_t)32 << 20) / (wb * nplanes)) & ~(size_t)1);
    nb = (int)((H + band - 1) / band);
    if (!e->work.h) B200_CUDA_CHECK(cudaStreamCreateWithFlags(&e->work.h, cudaStreamNonBlocking));
    if (int rc = e->rgb.reserve(wb * nplanes * (size_t)H, false)) return rc;
    if (g.interleaved) { d.rgb = e->rgb.d; d.rgb_stride = wb; }
    else {
      d.r = e->rgb.d; d.g = e->rgb.d + wb * H; d.b = e->rgb.d + 2 * wb * H; d.alpha = g.alpha ? e->rgb.d + 3 * wb * H : nullptr;
      d.r_stride = d.g_stride = d.b_stride = d.alpha_stride = wb;
    }
  }
  cudaStream_t ws = host ? (cudaStream_t)e->work : s;
  // events: [0] upload start, [1] band arrived, [2] upload end, then the start / end of each band's colour kernel
  std::unique_ptr<Event[]> ev(new Event[3 + 2 * (size_t)nb]);
  for (int k = 0; k < 3 + 2 * nb; k++) B200_CUDA_CHECK(cudaEventCreate(&ev[k].h));
  if (host) B200_CUDA_CHECK(cudaEventRecord(ev[0], e->stream));
  for (int k = 0, oy = 0; k < nb; k++) {
    const size_t y0 = (size_t)k * band, y1 = std::min((size_t)H, y0 + band);
    if (host) {
      const void* srcs[4] = {in->rgb, nullptr, nullptr, nullptr};
      size_t sst[4] = {in->rgb_stride, 0, 0, 0};
      if (!g.interleaved) {
        srcs[0] = in->r; srcs[1] = in->g; srcs[2] = in->b; srcs[3] = in->alpha;
        sst[0] = in->r_stride; sst[1] = in->g_stride; sst[2] = in->b_stride; sst[3] = in->alpha_stride;
      }
      for (int c = 0; c < nplanes; c++)
        if (int rc = e->bounce.upload(e->rgb.d + c * wb * H + y0 * wb, wb, (const uint8_t*)srcs[c] + y0 * sst[c], sst[c], wb, y1 - y0, e->stream, e->pool)) return rc;
      B200_CUDA_CHECK(cudaEventRecord(ev[1], e->stream));
      B200_CUDA_CHECK(cudaStreamWaitEvent(ws, ev[1], 0));
    }
    // output rows that need source rows < y1 only (all of them after the last band: the padding below the picture)
    const int oy1 = k == nb - 1 ? g.ph : (int)y1;
    B200_CUDA_CHECK(cudaEventRecord(ev[3 + 2 * k], ws));
    if (int rc = launch_rgb_to_ycbcr_grid(&d, &out, g.pipeline, oy, oy1, ws)) return rc;
    B200_CUDA_CHECK(cudaEventRecord(ev[4 + 2 * k], ws));
    oy = oy1;
  }
  if (host) B200_CUDA_CHECK(cudaEventRecord(ev[2], e->stream));
  // colour tiles, then alpha tiles, as windows of the padded picture
  const int n = g.cols * g.rows;
  std::vector<Pic> hp(n);
  for (int i = 0; i < n; i++) {
    const size_t r = (size_t)(i / g.cols), c = (size_t)(i % g.cols);
    hp[i].src[0] = Y + r * th * ys + c * tw; hp[i].stride[0] = ys;
    hp[i].src[1] = Cb + r * (th / 2) * cs + c * (tw / 2); hp[i].src[2] = Cr + r * (th / 2) * cs + c * (tw / 2); hp[i].stride[1] = hp[i].stride[2] = cs;
  }
  if (int rc = encode(e, &g.q, n, hp.data(), ws)) return rc;
  if (g.alpha) {
    std::vector<std::vector<uint8_t>> colour = std::move(e->out);
    const b200_gpu_encode_stats st = e->stats;
    for (int i = 0; i < n; i++) {
      const size_t r = (size_t)(i / g.cols), c = (size_t)(i % g.cols);
      hp[i].src[0] = A + r * th * ys + c * tw; hp[i].src[1] = hp[i].src[2] = nullptr;
    }
    b200_hevc_enc_params qa = g.q;
    qa.chroma_format_idc = 0;
    if (int rc = encode(e, &qa, n, hp.data(), ws)) return rc;
    for (auto& o : e->out) colour.push_back(std::move(o));
    e->out = std::move(colour);
    e->n = 2 * n; e->rec_first = n;
    b200_gpu_encode_stats& t = e->stats;
    t.analyse_ms += st.analyse_ms; t.entropy_ms += st.entropy_ms; t.framing_ms += st.framing_ms;
    t.bytes += st.bytes; t.ctus += st.ctus; t.pictures += st.pictures;
    t.mode_evaluations += st.mode_evaluations; t.cu_evaluations += st.cu_evaluations;
  }
  e->stats.total_ms = std::chrono::duration<double, std::milli>(clk::now() - t0).count();
  if (info) {
    float ms = 0;
    info->cols = g.cols; info->rows = g.rows; info->tile_w = tw; info->tile_h = th; info->width = W; info->height = H;
    info->has_alpha = g.alpha ? 1 : 0; info->pipeline = g.pipeline;
    info->colour_ms = 0;
    for (int k = 0; k < nb; k++) { cudaEventElapsedTime(&ms, ev[3 + 2 * k], ev[4 + 2 * k]); info->colour_ms += ms; }
    info->upload_ms = 0;
    if (host && cudaEventSynchronize(ev[2]) == cudaSuccess) { cudaEventElapsedTime(&ms, ev[0], ev[2]); info->upload_ms = ms; }
  }
  return B200_OK;
}

}  // namespace genc
}  // namespace b200

extern "C" {

int b200_gpu_encoder_create(b200_gpu_encoder** enc) {
  using namespace b200;
  if (!enc) return set_error(B200_E_INVALID, "null argument");
  std::unique_ptr<b200_gpu_encoder> e(new b200_gpu_encoder());
  B200_CUDA_CHECK(cudaStreamCreateWithFlags(&e->stream.h, cudaStreamNonBlocking));
  for (auto& ev : e->ev) B200_CUDA_CHECK(cudaEventCreate(&ev.h));
  *enc = e.release();
  return B200_OK;
}

void b200_gpu_encoder_destroy(b200_gpu_encoder* enc) { delete enc; }

int b200_gpu_encode_check(const b200_hevc_enc_params* p, int n, const b200_planes* pics) { return b200::genc::validate(p, n, pics); }

size_t b200_gpu_encoder_substream_capacity(int width, int log2_ctb_size, int chroma_format_idc) {
  return b200::genc::substream_capacity(width, log2_ctb_size, chroma_format_idc);
}

int b200_gpu_encoder_e1_warps_per_sm(int speed, int* warps) {
  using namespace b200;
  if (!warps) return set_error(B200_E_INVALID, "null argument");
  if (speed < 0 || speed > 2) return set_error(B200_E_INVALID, "speed %d: 0, 1 or 2", speed);
  const void* k = speed == 0 ? (const void*)genc::e1_kernel<0> : speed == 1 ? (const void*)genc::e1_kernel<1> : (const void*)genc::e1_kernel<2>;
  B200_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(warps, k, 32, 0));
  return B200_OK;
}

int b200_gpu_encode_intra_device(b200_gpu_encoder* enc, const b200_hevc_enc_params* p, int n, const b200_planes* pics, void* stream) {
  using namespace b200;
  if (!enc) return set_error(B200_E_INVALID, "null encoder");
  if (int rc = genc::validate(p, n, pics)) return rc;
  std::vector<genc::Pic> hp(n);
  for (int i = 0; i < n; i++) {
    hp[i].src[0] = (const uint8_t*)pics[i].y; hp[i].src[1] = (const uint8_t*)pics[i].cb; hp[i].src[2] = (const uint8_t*)pics[i].cr;
    hp[i].stride[0] = pics[i].y_stride; hp[i].stride[1] = hp[i].stride[2] = pics[i].c_stride;
  }
  cudaStream_t s = (cudaStream_t)stream;
  return genc::encode(enc, p, n, hp.data(), s);
}

int b200_gpu_encode_intra_host(b200_gpu_encoder* enc, const b200_hevc_enc_params* p, int n, const b200_planes* pics) {
  using namespace b200;
  if (!enc) return set_error(B200_E_INVALID, "null encoder");
  if (int rc = genc::validate(p, n, pics)) return rc;
  const int w = p->width, h = p->height, cw = (w + 1) >> 1, ch = (h + 1) >> 1, cfmt = p->chroma_format_idc;
  const size_t per = (size_t)w * h + (cfmt ? 2 * (size_t)cw * ch : 0);
  if (int rc = enc->src.reserve(n * per, false)) return rc;
  std::vector<genc::Pic> hp(n);
  for (int i = 0; i < n; i++) {
    uint8_t* d = enc->src.d + i * per;
    hp[i].src[0] = d; hp[i].stride[0] = w;
    if (int rc = enc->bounce.upload(d, w, pics[i].y, pics[i].y_stride, w, h, enc->stream, enc->pool)) return rc;
    if (cfmt) {
      hp[i].src[1] = d + (size_t)w * h; hp[i].src[2] = d + (size_t)w * h + (size_t)cw * ch; hp[i].stride[1] = hp[i].stride[2] = cw;
      if (int rc = enc->bounce.upload((void*)hp[i].src[1], cw, pics[i].cb, pics[i].c_stride, cw, ch, enc->stream, enc->pool)) return rc;
      if (int rc = enc->bounce.upload((void*)hp[i].src[2], cw, pics[i].cr, pics[i].c_stride, cw, ch, enc->stream, enc->pool)) return rc;
    }
  }
  return genc::encode(enc, p, n, hp.data(), enc->stream);
}

int b200_gpu_encode_rgb_grid_check(const b200_rgb_image* in, int tile_w, int tile_h, const b200_hevc_enc_params* p,
                                   const b200_rgb_to_ycbcr_options* opt) {
  b200::genc::GridPlan g;
  return b200::genc::grid_check(in, tile_w, tile_h, p, opt, &g);
}

int b200_gpu_encode_rgb_grid_device(b200_gpu_encoder* enc, const b200_rgb_image* in, int tile_w, int tile_h, const b200_hevc_enc_params* p,
                                    const b200_rgb_to_ycbcr_options* opt, void* stream, b200_grid_encode_info* info) {
  return b200::genc::grid_encode(enc, in, tile_w, tile_h, p, opt, false, (cudaStream_t)stream, info);
}

int b200_gpu_encode_rgb_grid_host(b200_gpu_encoder* enc, const b200_rgb_image* in, int tile_w, int tile_h, const b200_hevc_enc_params* p,
                                  const b200_rgb_to_ycbcr_options* opt, b200_grid_encode_info* info) {
  return b200::genc::grid_encode(enc, in, tile_w, tile_h, p, opt, true, nullptr, info);
}

int b200_gpu_encoder_output(b200_gpu_encoder* enc, int i, const uint8_t** data, size_t* size) {
  using namespace b200;
  if (!enc || !data || !size) return set_error(B200_E_INVALID, "null argument");
  if (!enc->ready || i < 0 || i >= enc->n) return set_error(B200_E_INVALID, "no picture %d in the last call", i);
  *data = enc->out[i].data(); *size = enc->out[i].size();
  return B200_OK;
}

int b200_gpu_encoder_read_recon(b200_gpu_encoder* enc, int i, void* y, void* cb, void* cr, size_t y_stride, size_t c_stride) {
  using namespace b200;
  if (!enc || !y) return set_error(B200_E_INVALID, "null argument");
  if (!enc->ready || i < enc->rec_first || i >= enc->n) return set_error(B200_E_INVALID, "no picture %d in the last call", i);
  const int w = enc->params.width, h = enc->params.height, W = enc->W, H = enc->H;
  const size_t ps = (size_t)W * H + (enc->cfmt ? 2 * (size_t)(W / 2) * (H / 2) : 0);
  const uint8_t* base = enc->rec.d + (size_t)(i - enc->rec_first) * ps;
  B200_CUDA_CHECK(cudaMemcpy2D(y, y_stride, base, W, w, h, cudaMemcpyDeviceToHost));
  if (enc->cfmt && cb && cr) {
    const int cw = (w + 1) >> 1, ch = (h + 1) >> 1;
    B200_CUDA_CHECK(cudaMemcpy2D(cb, c_stride, base + (size_t)W * H, W / 2, cw, ch, cudaMemcpyDeviceToHost));
    B200_CUDA_CHECK(cudaMemcpy2D(cr, c_stride, base + (size_t)W * H + (size_t)(W / 2) * (H / 2), W / 2, cw, ch, cudaMemcpyDeviceToHost));
  }
  return B200_OK;
}

int b200_gpu_encoder_get_stats(b200_gpu_encoder* enc, b200_gpu_encode_stats* out) {
  using namespace b200;
  if (!enc || !out) return set_error(B200_E_INVALID, "null argument");
  *out = enc->stats;
  return B200_OK;
}

// Test-only entry points (declared by the tests, not in include/b200_heif.h): b200_debug_enc_transform_host and
// b200_debug_enc_predict_host (b200_hevc_enc.cc) with the same arguments, run by the device code of the GPU encoder
int b200_debug_enc_transform_device(int n, const int32_t* prm, const int32_t* in, int32_t* out) {
  using namespace b200;
  if (n < 1 || n > 65536 || !prm || !in || !out) return set_error(B200_E_INVALID, "enc_transform: %d blocks, null argument", n);
  for (int i = 0; i < n; i++)
    if (const char* why = enc::debug_transform_args(prm + (size_t)i * enc::DT_FIELDS, in + (size_t)i * 1024)) return set_error(B200_E_INVALID, "enc_transform: block %d: %s", i, why);
  DevBuf<int> d_prm, d_in, d_out;
  int rc = 0;
  if ((rc = d_prm.reserve((size_t)n * enc::DT_FIELDS, false)) || (rc = d_in.reserve((size_t)n * 1024, false)) ||
      (rc = d_out.reserve((size_t)n * enc::DT_STAGES * 1024, false))) return rc;
  B200_CUDA_CHECK(cudaMemcpy(d_prm.d, prm, (size_t)n * enc::DT_FIELDS * 4, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_in.d, in, (size_t)n * 1024 * 4, cudaMemcpyHostToDevice));
  genc::debug_transform_kernel<<<dim3((unsigned)n, enc::DT_STAGES), 256>>>(d_prm.d, d_in.d, d_out.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpy(out, d_out.d, (size_t)n * enc::DT_STAGES * 1024 * 4, cudaMemcpyDeviceToHost));
  return B200_OK;
}

int b200_debug_enc_predict_device(int n, const int32_t* prm, const int16_t* refs, int16_t* rf, int32_t* pred) {
  using namespace b200;
  if (n < 1 || n > 65536 || !prm || !refs || !rf || !pred) return set_error(B200_E_INVALID, "enc_predict: %d blocks, null argument", n);
  for (int i = 0; i < n; i++)
    if (const char* why = enc::debug_predict_args(prm + (size_t)i * enc::DP_FIELDS, refs + (size_t)i * 129)) return set_error(B200_E_INVALID, "enc_predict: block %d: %s", i, why);
  DevBuf<int> d_prm, d_pred; DevBuf<int16_t> d_refs, d_rf;
  int rc = 0;
  if ((rc = d_prm.reserve((size_t)n * enc::DP_FIELDS, false)) || (rc = d_refs.reserve((size_t)n * 129, false)) ||
      (rc = d_rf.reserve((size_t)n * 258, false)) || (rc = d_pred.reserve((size_t)n * 35 * 1024, false))) return rc;
  B200_CUDA_CHECK(cudaMemcpy(d_prm.d, prm, (size_t)n * enc::DP_FIELDS * 4, cudaMemcpyHostToDevice));
  B200_CUDA_CHECK(cudaMemcpy(d_refs.d, refs, (size_t)n * 129 * 2, cudaMemcpyHostToDevice));
  genc::debug_predict_kernel<<<n, 256>>>(d_prm.d, d_refs.d, d_rf.d, d_pred.d);
  B200_CUDA_CHECK(cudaGetLastError());
  B200_CUDA_CHECK(cudaMemcpy(rf, d_rf.d, (size_t)n * 258 * 2, cudaMemcpyDeviceToHost));
  B200_CUDA_CHECK(cudaMemcpy(pred, d_pred.d, (size_t)n * 35 * 1024 * 4, cudaMemcpyDeviceToHost));
  return B200_OK;
}

}  // extern "C"
