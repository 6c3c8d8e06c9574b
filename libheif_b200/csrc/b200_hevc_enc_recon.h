// b200_hevc_enc_recon.h -- the reconstruction half both HEVC intra encoders share, as one piece of host + device source:
// intra prediction (8.4.4.2: reference substitution, neighbour filtering, planar / DC / angular with the edge filters), the
// forward DST 4x4 / DCT 4..32, quantisation, scaling (8.6.2-3) and the inverse transform (8.6.4), and their constant tables.
// Every function takes the bit depth; the GPU encoder (b200_hevc_gpu_enc.cu) passes 8.  The transforms and the
// (de)quantisation are "one output element" functions: the host encoder (b200_hevc_enc.cc, B200_SYNTAX_HOST_ONLY) loops
// over the elements, the GPU encoder over the lanes of a warp.  Both must match the decoder bit for bit.
#pragma once
#include "b200_hevc_syntax.h"

namespace b200 {
namespace enc {

B200_TABLE(int8_t, kDctT, [32], {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67,
                                 64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4})
B200_TABLE(int8_t, kDst4, [4][4], {{29, 55, 74, 84}, {74, 74, 0, -74}, {84, -29, -74, 55}, {55, -84, 74, -29}})
B200_TABLE(int8_t, kAngle, [35], {0, 0, 32, 26, 21, 17, 13, 9, 5, 2, 0, -2, -5, -9, -13, -17, -21, -26, -32,
                                  -26, -21, -17, -13, -9, -5, -2, 0, 2, 5, 9, 13, 17, 21, 26, 32})
B200_TABLE(int16_t, kInvAngle, [35], {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, -4096, -1638, -910, -630, -482, -390, -315, -256,
                                      -315, -390, -482, -630, -910, -1638, -4096, 0, 0, 0, 0, 0, 0, 0, 0, 0})
B200_TABLE(int32_t, kQuantScale, [6], {26214, 23302, 20560, 18396, 16384, 14564})
B200_TABLE(uint8_t, kLevelScale, [6], {40, 45, 51, 57, 64, 72})

// ------------------------------------------------------------------------------------------ intra prediction (8.4.4.2)
// The neighbours of an n x n block are r[0..4n]: r[2n - 1 - y] = p[-1][y] (left column, bottom-up from p[-1][2n - 1]),
// r[2n] = p[-1][-1], r[2n + 1 + x] = p[x][-1] (top row).

// 8.4.4.2.2: unavailable samples (marked -1) take the value of the nearest available one before them in r[] (after
// it for those before the first available one), or 1 << (bd - 1) when none is available
B200_HD inline void substitute_refs(int16_t* r, int n, int bd) {
  int first = 0; while (first <= 4 * n && r[first] < 0) first++;
  if (first > 4 * n) { for (int i = 0; i <= 4 * n; i++) r[i] = (int16_t)(1 << (bd - 1)); return; }
  for (int i = 0; i < first; i++) r[i] = r[first];
  for (int i = first + 1; i <= 4 * n; i++) if (r[i] < 0) r[i] = r[i - 1];
}

// 8.4.4.2.3: whether `mode` predicts from the filtered neighbours.  plane: the plane is filtered at all (luma; chroma only
// in 4:4:4)
B200_HD inline bool refs_filtered(bool plane, int mode, int log2n) {
  if (!plane || mode == 1 || log2n == 2) return false;
  const int dist = syn::imin(abs(mode - 26), abs(mode - 10));
  return dist > (log2n == 3 ? 7 : (log2n == 4 ? 1 : 0));
}

// 8.4.4.2.3: f = the filtered r; strong: strong_intra_smoothing_enabled_flag and luma (applies to 32 x 32 blocks only)
B200_HD inline void filter_refs(const int16_t* r, int16_t* f, int log2n, bool strong, int bd) {
  const int n = 1 << log2n, corner = r[2 * n], bl = r[0], tr = r[4 * n];
  if (strong && log2n == 5 && abs(corner + tr - 2 * r[3 * n]) < (1 << (bd - 5)) && abs(corner + bl - 2 * r[n]) < (1 << (bd - 5))) {
    f[2 * n] = (int16_t)corner; f[0] = (int16_t)bl; f[4 * n] = (int16_t)tr;
    for (int y = 0; y < 63; y++) f[2 * n - 1 - y] = (int16_t)(((63 - y) * corner + (y + 1) * bl + 32) >> 6);
    for (int x = 0; x < 63; x++) f[2 * n + 1 + x] = (int16_t)(((63 - x) * corner + (x + 1) * tr + 32) >> 6);
  } else {
    f[0] = r[0]; f[4 * n] = r[4 * n];
    for (int i = 1; i < 4 * n; i++) f[i] = (int16_t)((r[i - 1] + 2 * r[i] + r[i + 1] + 2) >> 2);
  }
}

// dcVal of 8.4.4.2.5 from the (unfiltered) neighbours
B200_HD inline int dc_value(const int16_t* r, int log2n) {
  const int n = 1 << log2n;
  int sum = n; for (int i = 0; i < n; i++) sum += r[2 * n - 1 - i] + r[2 * n + 1 + i];
  return sum >> (log2n + 1);
}

// 8.4.4.2.4-6: predicted sample (x, y) of `mode` from the neighbours ref (filtered where refs_filtered() says so) and
// dc = dc_value().  luma: the DC and mode 10 / 26 edge filters apply below 32 x 32, the latter clipped to 0..maxv.
// dc is a reference so that only the DC mode reads it: the GPU encoder keeps it in shared memory, and a load of it for
// every sample of every mode slows its mode search down.
B200_HD inline int pred_sample(const int16_t* ref, const int& dc, int log2n, int mode, int x, int y, bool luma, int maxv) {
  const int n = 1 << log2n;
#define LEFT(i) ((int)ref[2 * n - 1 - (i)])
#define TOP(i) ((int)ref[2 * n + 1 + (i)])
  if (mode == 0) return ((n - 1 - x) * LEFT(y) + (x + 1) * TOP(n) + (n - 1 - y) * TOP(x) + (y + 1) * LEFT(n) + n) >> (log2n + 1);
  if (mode == 1) {
    if (luma && n < 32) {
      if (x == 0 && y == 0) return (LEFT(0) + 2 * dc + TOP(0) + 2) >> 2;
      if (y == 0) return (TOP(x) + 3 * dc + 2) >> 2;
      if (x == 0) return (LEFT(y) + 3 * dc + 2) >> 2;
    }
    return dc;
  }
  const int ang = B200_T(kAngle)[mode], ia = B200_T(kInvAngle)[mode];
  if (mode >= 18) {
    if (mode == 26 && luma && n < 32 && x == 0) return syn::clip3(0, maxv, TOP(0) + ((LEFT(y) - LEFT(-1)) >> 1));
    const int idx = ((y + 1) * ang) >> 5, f = ((y + 1) * ang) & 31, k1 = x + idx + 1, k2 = k1 + 1;
    const int r1 = k1 >= 0 ? TOP(k1 - 1) : LEFT(-1 + ((k1 * ia + 128) >> 8));
    if (!f) return r1;
    const int r2 = k2 >= 0 ? TOP(k2 - 1) : LEFT(-1 + ((k2 * ia + 128) >> 8));
    return ((32 - f) * r1 + f * r2 + 16) >> 5;
  }
  if (mode == 10 && luma && n < 32 && y == 0) return syn::clip3(0, maxv, LEFT(0) + ((TOP(x) - TOP(-1)) >> 1));
  const int idx = ((x + 1) * ang) >> 5, f = ((x + 1) * ang) & 31, k1 = y + idx + 1, k2 = k1 + 1;
  const int r1 = k1 >= 0 ? LEFT(k1 - 1) : TOP(-1 + ((k1 * ia + 128) >> 8));
  if (!f) return r1;
  const int r2 = k2 >= 0 ? LEFT(k2 - 1) : TOP(-1 + ((k2 * ia + 128) >> 8));
  return ((32 - f) * r1 + f * r2 + 16) >> 5;
#undef LEFT
#undef TOP
}

// ------------------------------------------------------------------------------------------ transforms (8.6.4.2)
// DCT matrix entry [k][x] of an n x n transform
B200_HD inline int dct_coef(int log2n, int k, int x) {
  if (k == 0) return 64;
  int j = ((k << (5 - log2n)) * (2 * x + 1)) & 127, sgn = 1;
  if (j > 64) j = 128 - j;
  if (j > 32) { j = 64 - j; sgn = -1; }
  return sgn * B200_T(kDctT)[j];
}

// The DCT's cosines by phase j (in units of pi / 64): entry [k][x] of the n x n matrix is the one at phase
// (k << (5 - log2n)) * (2x + 1) mod 128 (32 and 96 never occur).  tmat() reads it on the host, where a lookup per
// multiply is cheaper than dct_coef(); the GPU encoder computes dct_coef() instead.
B200_TABLE(int8_t, kDctPhase, [128], {64, 90, 90, 90, 89, 88, 87, 85, 83, 82, 80, 78, 75, 73, 70, 67,
                                      64, 61, 57, 54, 50, 46, 43, 38, 36, 31, 25, 22, 18, 13, 9, 4,
                                      0, -4, -9, -13, -18, -22, -25, -31, -36, -38, -43, -46, -50, -54, -57, -61,
                                      -64, -67, -70, -73, -75, -78, -80, -82, -83, -85, -87, -88, -89, -90, -90, -90,
                                      -64, -90, -90, -90, -89, -88, -87, -85, -83, -82, -80, -78, -75, -73, -70, -67,
                                      -64, -61, -57, -54, -50, -46, -43, -38, -36, -31, -25, -22, -18, -13, -9, -4,
                                      0, 4, 9, 13, 18, 22, 25, 31, 36, 38, 43, 46, 50, 54, 57, 61,
                                      64, 67, 70, 73, 75, 78, 80, 82, 83, 85, 87, 88, 89, 90, 90, 90})

// transMatrix[k][x]: the DST of 4x4 luma blocks, else the DCT
B200_HD inline int tmat(bool dst4, int log2n, int k, int x) {
  if (dst4) return B200_T(kDst4)[k][x];
#ifdef __CUDA_ARCH__
  return dct_coef(log2n, k, x);
#else
  return B200_T(kDctPhase)[((k << (5 - log2n)) * (2 * x + 1)) & 127];
#endif
}

// The four stages, each one element (row, col) of its n x n output from the n x n input a[] (row-major).
// Forward, columns: out[k][x] = sum_y M[k][y] a[y][x], rounded and shifted by log2n + bd - 9
B200_HD inline int fwd_col(const int* a, bool dst4, int log2n, int k, int x, int bd) {
  const int n = 1 << log2n, sh = log2n + bd - 9;
  int s = 0; for (int y = 0; y < n; y++) s += tmat(dst4, log2n, k, y) * a[y * n + x];
  return (s + (1 << (sh - 1))) >> sh;
}
// Forward, rows: out[y][k] = sum_x M[k][x] a[y][x], shifted by log2n + 6
B200_HD inline int fwd_row(const int* a, bool dst4, int log2n, int y, int k) {
  const int n = 1 << log2n, sh = log2n + 6;
  int s = 0; for (int x = 0; x < n; x++) s += tmat(dst4, log2n, k, x) * a[y * n + x];
  return (s + (1 << (sh - 1))) >> sh;
}
// Inverse, columns: out[y][x] = sum_k a[k][x] M[k][y], shifted by 7 and clipped to 16 bits
B200_HD inline int inv_col(const int* a, bool dst4, int log2n, int y, int x) {
  const int n = 1 << log2n;
  int s = 0; for (int k = 0; k < n; k++) s += a[k * n + x] * tmat(dst4, log2n, k, y);
  return syn::clip3(-32768, 32767, (s + 64) >> 7);
}
// Inverse, rows: out[y][x] = sum_k a[y][k] M[k][x], shifted by 20 - bd: the residual
B200_HD inline int inv_row(const int* a, bool dst4, int log2n, int y, int x, int bd) {
  const int n = 1 << log2n, sh = 20 - bd;
  int s = 0; for (int k = 0; k < n; k++) s += a[y * n + k] * tmat(dst4, log2n, k, x);
  return (s + (1 << (sh - 1))) >> sh;
}

// ------------------------------------------------------------------------------------------ (de)quantisation
// Level of transform coefficient cf at qp (Qp'Y or Qp'C): uniform, rounding offset 171/512 (intra), |level| <= 32767
B200_HD inline int quant_level(int cf, int qp, int log2n, int bd) {
  const int qbits = 14 + qp / 6 + 15 - bd - log2n;
  const int l = syn::imin((int)(((long long)abs(cf) * B200_T(kQuantScale)[qp % 6] + (171LL << (qbits - 9))) >> qbits), 32767);
  return cf < 0 ? -l : l;
}

// 8.6.3 scaling of `level` with scaling factor m (16: flat), clipped to 16 bits
B200_HD inline int dequant(int level, int m, int qp, int log2n, int bd) {
  const int bs = bd + log2n - 5;
  const long long t = ((long long)level * m * (B200_T(kLevelScale)[qp % 6] << (qp / 6)) + (1LL << (bs - 1))) >> bs;
  return (int)(t < -32768 ? -32768 : (t > 32767 ? 32767 : t));
}

// ------------------------------------------------------------------------------------------ test-only entry points
// b200_debug_enc_transform_{host,device} and b200_debug_enc_predict_{host,device} run the functions above on given blocks
// (b200_hevc_enc.cc on the host, b200_hevc_gpu_enc.cu on the device).  These check one block's arguments: nullptr when they
// are in the functions' domain, else what is wrong.
enum { DT_LOG2N, DT_DST4, DT_BD, DT_QP, DT_M, DT_FIELDS };       // transform block: [DT_FIELDS] parameters + 1024 inputs
enum { DP_LOG2N, DP_BD, DP_LUMA, DP_PLANE, DP_STRONG, DP_FIELDS };   // prediction block: [DP_FIELDS] parameters + 129 neighbours
enum { DT_STAGES = 6 };                                           // fwd_col, fwd_row, quant_level, dequant, inv_col, inv_row
inline const char* debug_transform_args(const int32_t* p, const int32_t* in) {
  const int lg = p[DT_LOG2N], bd = p[DT_BD];
  if (lg < 2 || lg > 5) return "log2 size";
  if (bd < 8 || bd > 12) return "bit depth";
  if (p[DT_DST4] != 0 && !(p[DT_DST4] == 1 && lg == 2)) return "DST (4x4 only)";
  if (p[DT_QP] < 0 || p[DT_QP] > 51 + 6 * (bd - 8)) return "qp";
  if (p[DT_M] < 1 || p[DT_M] > 255) return "scaling factor";
  for (int i = 0; i < (1 << (2 * lg)); i++) if (in[i] < -32768 || in[i] > 32767) return "input outside int16";
  return nullptr;
}
inline const char* debug_predict_args(const int32_t* p, const int16_t* refs) {
  const int lg = p[DP_LOG2N], bd = p[DP_BD];
  if (lg < 2 || lg > 5) return "log2 size";
  if (bd < 8 || bd > 12) return "bit depth";
  for (int f = DP_LUMA; f <= DP_STRONG; f++) if (p[f] != 0 && p[f] != 1) return "flag";
  if (p[DP_LUMA] && !p[DP_PLANE]) return "luma without neighbour filtering";
  for (int i = 0; i <= 4 << lg; i++) if (refs[i] < -1 || refs[i] >= (1 << bd)) return "neighbour outside -1 .. maxv";
  return nullptr;
}
// element (row r, column c) of stage st on the n x n block a with the parameters p
B200_HD inline int debug_transform_stage(int st, const int32_t* p, const int* a, int r, int c) {
  const int lg = p[DT_LOG2N], bd = p[DT_BD], qp = p[DT_QP];
  const bool dst4 = p[DT_DST4] != 0;
  switch (st) {
    case 0: return fwd_col(a, dst4, lg, r, c, bd);
    case 1: return fwd_row(a, dst4, lg, r, c);
    case 2: return quant_level(a[(r << lg) + c], qp, lg, bd);
    case 3: return dequant(a[(r << lg) + c], p[DT_M], qp, lg, bd);
    case 4: return inv_col(a, dst4, lg, r, c);
    default: return inv_row(a, dst4, lg, r, c, bd);
  }
}

}  // namespace enc
}  // namespace b200
