// b200_hevc_enc_cabac.h -- the entropy-coding half both HEVC intra encoders share, as one piece of host + device source:
// the arithmetic encoder of 9.3.4.5 over a caller's bit sink, context initialisation (9.3.2.2), the residual_coding()
// writer (7.3.8.11), intra luma mode signalling (8.4.2 / 7.3.8.5), the tables of the last-position prefix and the
// chroma QP mapping (Table 8-10).  The host encoder (b200_hevc_enc.cc) compiles it for the host only
// (B200_SYNTAX_HOST_ONLY), the GPU encoder (b200_hevc_gpu_enc.cu) for both sides.  The context, state-transition, scan
// and sig-map tables are the decoder's (b200_hevc_syntax.h); the reconstruction half is b200_hevc_enc_recon.h.
#pragma once
#include "b200_hevc_syntax.h"

namespace b200 {
namespace enc {

B200_TABLE(uint8_t, kQpcTab, [14], {29, 30, 31, 32, 33, 33, 34, 34, 35, 35, 36, 36, 37, 37})        // Table 8-10, qPi 30..43
B200_TABLE(uint8_t, kLastGroup, [32], {0, 1, 2, 3, 4, 4, 5, 5, 6, 6, 6, 6, 7, 7, 7, 7, 8, 8, 8, 8, 8, 8, 8, 8, 9, 9, 9, 9, 9, 9, 9, 9})
B200_TABLE(uint8_t, kLastGroupMin, [10], {0, 1, 2, 3, 4, 6, 8, 12, 16, 24})

// Qp'Cb / Qp'Cr (8.6.1): qPi = Clip3(-QpBdOffsetC, 57, QpY + the chroma offsets), mapped by Table 8-10 when
// ChromaArrayType is 1 and capped at 51 otherwise, plus QpBdOffsetC
B200_HD inline int chroma_qp(int qpy_plus_offset, int chroma_format, int bit_depth) {
  const int qbd = 6 * (bit_depth - 8), qpi = syn::clip3(-qbd, 57, qpy_plus_offset);
  const int qpc = chroma_format != 1 ? syn::imin(qpi, 51) : (qpi < 30 ? qpi : (qpi >= 43 ? qpi - 6 : B200_T(kQpcTab)[qpi - 30]));
  return qpc + qbd;
}

// scanIdx of a 4x4 / 8x8 intra block (8.4.4.2.6 / 7.4.9.11): vertical scan for near-horizontal modes and vice versa
B200_HD inline int scan_idx(int mode) { return (mode >= 6 && mode <= 14) ? 2 : (mode >= 22 && mode <= 30) ? 1 : 0; }

// 8.4.2: candModeList from the modes of the left (a) and above (b) neighbours, INTRA_DC (1) where one is unavailable
B200_HD inline void mpm_candidates(int a, int b, int cand[3]) {
  if (a == b) {
    if (a < 2) { cand[0] = 0; cand[1] = 1; cand[2] = 26; }
    else { cand[0] = a; cand[1] = 2 + ((a + 29) % 32); cand[2] = 2 + ((a - 2 + 1) % 32); }
  } else {
    cand[0] = a; cand[1] = b;
    if (a != 0 && b != 0) cand[2] = 0; else if (a != 1 && b != 1) cand[2] = 1; else cand[2] = 26;
  }
}

// How `mode` is signalled against its candidates: mpm_idx (0..2) when it is one of them, else 3 + rem_intra_luma_pred_mode
B200_HD inline int mpm_code(int mode, const int cand[3]) {
  for (int k = 0; k < 3; k++) if (cand[k] == mode) return k;
  int s0 = cand[0], s1 = cand[1], s2 = cand[2], t;
  if (s0 > s1) { t = s0; s0 = s1; s1 = t; }
  if (s1 > s2) { t = s1; s1 = s2; s2 = t; }
  if (s0 > s1) { t = s0; s0 = s1; s1 = t; }
  int r = mode; if (r > s2) r--; if (r > s1) r--; if (r > s0) r--;
  return 3 + r;
}

// Arithmetic encoder of 9.3.4.5.  Sink: put1(b) writes one bit, put(v, n) the n low bits of v, align_zero() pads to a
// byte with zeros.
// Contexts are bytes pStateIdx << 1 | valMps, CTX_COUNT of them at `ctx`.
template <class Sink>
struct CabacWriter {
  Sink bits; uint8_t* ctx;
  unsigned low = 0, range = 510; int outstanding = 0; bool first = true;

  B200_HD void restart() { low = 0; range = 510; outstanding = 0; first = true; }     // 9.3.2.5, also after pcm_sample()
  B200_HD void put_bit(unsigned b) {
    if (first) first = false; else bits.put1(b);
    while (outstanding > 0) { bits.put1(1 - b); outstanding--; }
  }
  B200_HD void renorm() {
    while (range < 256) {
      if (low < 256) put_bit(0);
      else if (low >= 512) { low -= 512; put_bit(1); }
      else { low -= 256; outstanding++; }
      range <<= 1; low <<= 1;
    }
  }
  B200_HD void bin(int ci, int b) {
    const unsigned s = ctx[ci], state = s >> 1, mps = s & 1;
    const unsigned lps = (syn::B200_T(kLps4)[state] >> (8 * ((range >> 6) & 3))) & 0xff;
    range -= lps;
    if ((unsigned)b != mps) {
      low += range; range = lps;
      ctx[ci] = (uint8_t)((syn::B200_T(kTransLps)[state] << 1) | (state == 0 ? 1 - mps : mps));
    } else if (state < 62) ctx[ci] = (uint8_t)(((state + 1) << 1) | mps);
    renorm();
  }
  B200_HD void bypass(int b) {
    low <<= 1;
    if (b) low += range;
    if (low >= 1024) { put_bit(1); low -= 1024; }
    else if (low < 512) put_bit(0);
    else { low -= 512; outstanding++; }
  }
  B200_HD void bypass_bits(unsigned v, int n) { for (int i = n - 1; i >= 0; i--) bypass((v >> i) & 1); }
  // b = 1: flush (9.3.4.5.5), whose last bit is the stop bit, then zero bits up to the byte boundary
  B200_HD void terminate(int b) {
    range -= 2;
    if (b) { low += range; range = 2; renorm(); put_bit((low >> 9) & 1); bits.put(((low >> 7) & 3) | 1, 2); bits.align_zero(); }
    else renorm();
  }
};

// 9.3.2.2 for an I slice at slice_qp (0..51)
B200_HD inline void init_contexts(uint8_t* ctx, int slice_qp) {
  for (int i = 0; i < syn::CTX_COUNT; i++) {
    const int iv = syn::B200_T(kInitI)[i], m = (iv >> 4) * 5 - 45, nn = ((iv & 15) << 3) - 16;
    const int pre = syn::clip3(1, 126, ((m * slice_qp) >> 4) + nn), mps = pre > 63;
    ctx[i] = (uint8_t)(((mps ? pre - 64 : 63 - pre) << 1) | mps);
  }
}

// prev_intra_luma_pred_flag of each of the np prediction units, then each one's mpm_idx or rem_intra_luma_pred_mode
// (7.3.8.5); code[i] = mpm_code() of PU i
template <class C>
B200_HD void write_luma_modes(C& cb, int np, const int code[4]) {
  for (int i = 0; i < np; i++) cb.bin(syn::CTX_PREV_INTRA, code[i] < 3);
  for (int i = 0; i < np; i++) {
    if (code[i] < 3) { cb.bypass(code[i] > 0); if (code[i] > 0) cb.bypass(code[i] > 1); }
    else cb.bypass_bits(code[i] - 3, 5);
  }
}

// residual_coding() (7.3.8.11) of the n x n levels at lev[y * stride + x] (at least one non-zero) of component c.
// tskip_present: transform_skip_flag is coded (transform_skip_enabled_flag, 4x4, no bypass), with value tskip;
// sign_hiding: sign_data_hiding_enabled_flag and no bypass.
template <class C>
B200_HD void residual_coding(C& cb, const int16_t* lev, int stride, int log2n, int c, int scan, bool tskip_present, bool tskip,
                             bool sign_hiding) {
  using namespace syn;
  const int l2sb = log2n - 2;
  if (tskip_present && log2n == 2) cb.bin(CTX_TSKIP + (c ? 1 : 0), tskip);
  const uint8_t *sbx = B200_T(kScanX)[l2sb][scan], *sby = B200_T(kScanY)[l2sb][scan], *px = B200_T(kScanX)[2][scan], *py = B200_T(kScanY)[2][scan];
#define LEV(xx, yy) ((int)lev[(size_t)(yy) * stride + (xx)])
  int last_sb = -1, last_pos = -1;
  for (int i = (1 << (2 * l2sb)) - 1; i >= 0 && last_sb < 0; i--) for (int k = 15; k >= 0; k--)
    if (LEV((sbx[i] << 2) + px[k], (sby[i] << 2) + py[k])) { last_sb = i; last_pos = k; break; }
  int lx = (sbx[last_sb] << 2) + px[last_pos], ly = (sby[last_sb] << 2) + py[last_pos];
  if (scan == 2) { const int t = lx; lx = ly; ly = t; }
  const uint8_t* group = B200_T(kLastGroup);
  const uint8_t* min_in_group = B200_T(kLastGroupMin);
  const int cmax = (log2n << 1) - 1;
  int off, shift;
  if (c == 0) { off = 3 * (log2n - 2) + ((log2n - 1) >> 2); shift = (log2n + 1) >> 2; } else { off = 15; shift = log2n - 2; }
  const int gx = group[lx], gy = group[ly];
  for (int k = 0; k < gx; k++) cb.bin(CTX_LAST_X + off + (k >> shift), 1);
  if (gx < cmax) cb.bin(CTX_LAST_X + off + (gx >> shift), 0);
  for (int k = 0; k < gy; k++) cb.bin(CTX_LAST_Y + off + (k >> shift), 1);
  if (gy < cmax) cb.bin(CTX_LAST_Y + off + (gy >> shift), 0);
  if (gx > 3) cb.bypass_bits(lx - min_in_group[gx], (gx >> 1) - 1);
  if (gy > 3) cb.bypass_bits(ly - min_in_group[gy], (gy >> 1) - 1);
  uint64_t csbf = 0;                                        // coded_sub_block_flag, bit ys * 8 + xs
#define CSBF(xx, yy) ((int)((csbf >> ((yy) * 8 + (xx))) & 1))
  int carry = 1; bool first_done = false;
  for (int i = last_sb; i >= 0; i--) {
    const int xs = sbx[i], ys = sby[i];
    int v[16]; bool coded = false;
    for (int k = 0; k < 16; k++) { v[k] = LEV((xs << 2) + px[k], (ys << 2) + py[k]); coded |= v[k] != 0; }
    bool infer_dc = false;
    if (i < last_sb && i > 0) {
      int cs = 0;
      if (xs + 1 < (1 << l2sb)) cs |= CSBF(xs + 1, ys);
      if (ys + 1 < (1 << l2sb)) cs |= CSBF(xs, ys + 1);
      cb.bin(CTX_CSBF + (cs ? 1 : 0) + (c ? 2 : 0), coded);
      infer_dc = true;
    } else coded = true;
    if (coded) csbf |= 1ull << (ys * 8 + xs);
    if (!coded) continue;
    int prev = 0;
    if (xs + 1 < (1 << l2sb)) prev |= CSBF(xs + 1, ys);
    if (ys + 1 < (1 << l2sb)) prev |= CSBF(xs, ys + 1) << 1;
    const int start = i == last_sb ? last_pos - 1 : 15;
    for (int k = start; k >= 0; k--) {
      const int xc = (xs << 2) + px[k], yc = (ys << 2) + py[k];
      if (k > 0 || !infer_dc) {
        int sc;
        if (log2n == 2) sc = B200_T(kSigMap4)[(yc << 2) + xc];
        else if (xc + yc == 0) sc = 0;
        else {
          const int xp = xc & 3, yp = yc & 3;
          if (prev == 0) sc = (xp + yp == 0) ? 2 : (xp + yp < 3) ? 1 : 0;
          else if (prev == 1) sc = yp == 0 ? 2 : (yp == 1 ? 1 : 0);
          else if (prev == 2) sc = xp == 0 ? 2 : (xp == 1 ? 1 : 0);
          else sc = 2;
          if (c == 0) { if (xs || ys) sc += 3; sc += log2n == 3 ? (scan == 0 ? 9 : 15) : 21; }
          else sc += log2n == 3 ? 9 : 12;
        }
        cb.bin(CTX_SIG + (c == 0 ? sc : 27 + sc), v[k] != 0);
        if (v[k]) infer_dc = false;
      }
    }
    int first_sig = 16, last_sig = -1, ng1 = 0, last_g1 = -1, g1ctx = 1;
    int ctx_set = (i == 0 || c > 0) ? 0 : 2;
    if (first_done && carry == 0) ctx_set++;
    first_done = true;
    bool any = false;
    for (int k = 15; k >= 0; k--) if (v[k]) {
      any = true;
      if (ng1 < 8) {
        const int g = abs(v[k]) > 1;
        cb.bin(CTX_GT1 + ctx_set * 4 + imin(3, g1ctx) + (c ? 16 : 0), g);
        ng1++;
        if (g) { g1ctx = 0; if (last_g1 < 0) last_g1 = k; } else if (g1ctx > 0) g1ctx++;
      }
      if (last_sig < 0) last_sig = k;
      first_sig = k;
    }
    if (any) carry = g1ctx;
    const bool hidden = sign_hiding && last_sig - first_sig > 3;      // the first coefficient's sign is the parity of the sum
    if (last_g1 >= 0) cb.bin(CTX_GT2 + ctx_set + (c ? 4 : 0), abs(v[last_g1]) > 2);
    for (int k = 15; k >= 0; k--) if (v[k] && (!hidden || k != first_sig)) cb.bypass(v[k] < 0);
    int nsig = 0, rice = 0, cnt1 = 0;
    for (int k = 15; k >= 0; k--) if (v[k]) {
      const int av = abs(v[k]);
      const int g1 = cnt1 < 8 ? (av > 1) : 0; if (cnt1 < 8) cnt1++;
      const int g2 = (k == last_g1) ? (av > 2) : 0;
      const int base = 1 + g1 + g2;
      if (base == ((nsig < 8) ? ((k == last_g1) ? 3 : 2) : 1)) {      // coeff_abs_level_remaining (9.3.3.11)
        const int rem = av - base;
        if ((rem >> rice) <= 3) { const int pre = rem >> rice; for (int t = 0; t < pre; t++) cb.bypass(1); cb.bypass(0); cb.bypass_bits(rem & ((1 << rice) - 1), rice); }
        else {
          const int q = (rem >> rice) - 2; int kk = 0; while ((q >> (kk + 1)) > 0) kk++;
          for (int t = 0; t < kk + 3; t++) cb.bypass(1);
          cb.bypass(0);
          cb.bypass_bits(rem - (((1 << kk) + 2) << rice), kk + rice);
        }
        if (av > 3 * (1 << rice)) rice = imin(rice + 1, 4);
      }
      nsig++;
    }
  }
#undef LEV
#undef CSBF
}

}  // namespace enc
}  // namespace b200
