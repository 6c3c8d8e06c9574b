// b200_color.cu -- K6: fused colour post-stage for sm_90a.
//
// One pass over HBM does what the reference does in 2-4 passes with calloc'ed intermediates
// (libheif/color-conversion/colorconversion.cc:450-487 runs each op into a fresh image):
//   geometric transform (rotate_ccw / mirror / crop, libheif/image/pixelimage.cc:1175-1546) by addressing,
//   nearest-neighbour chroma upsampling (cx = x >> shiftH, cy = y >> shiftV, yuv2rgb.cc:226-229),
//   YCbCr -> RGB in the reference's integer arithmetic (yuv2rgb.cc:386-424) or float arithmetic
//   (yuv2rgb.cc:270-282, :696-709), optional ">> (bpp-8)" (hdr_sdr.cc:147-200), and the interleave /
//   endianness step (rgb2rgb.cc:71-150, yuv2rgb.cc:715-729).
//
// Layout: every CTA owns a 64x64 output tile.  The corresponding source window (also 64x64 because all
// transforms are axis permutations) is staged in shared memory with 16-byte loads, then each thread turns a
// 16-pixel strip into RGB and writes it with 128-bit stores (48 B of RGB24 = 3 x uint4).
// HBM-bound byte work: algorithmic traffic 4.5 B/px (8-bit -> RGB24), 9 B/px (16-bit -> RRGGBB).
//
// Bit-exactness: float expressions use __fmul_rn/__fadd_rn explicitly (no FMA contraction; the x86-64
// reference build has no FMA), evaluation order is the reference's, rounding is (int32)(fx + 0.5f).
#include "b200_internal.h"
#include <algorithm>

namespace b200 {

constexpr int TILE = 64;
constexpr int SROWS = TILE + 2;     // an odd source origin needs one extra chroma row/column
constexpr int SPAD = 4;             // padding elements per shared row

struct K6Args {
  const void *y, *cb, *cr, *a;
  long long ys, cs, as;             // strides in bytes
  void* out[3];
  long long os;                     // output stride in bytes
  int src_w, src_h;
  int out_w, out_h;                 // size of the colour-converted picture (geometry output)
  int dst_w, dst_h;                 // k6_scaled_kernel: size of the scaled result
  int m[6];
  int sh, sv;                       // chroma subsampling shifts; -1 = monochrome
  int bpp;
  int full_range;
  int int_mode;                     // 1: Op_YCbCr420_to_RGB24/32 integer arithmetic
  float cf[4];                      // r_cr, g_cb, g_cr, b_cb
  int ci[4];                        // lround(256*cf)
  int out_fmt;                      // b200_chroma value
  int sdr_shift;                    // Op_to_sdr_planes applied to the RGB result
  int pre_shift;                    // Op_to_sdr_planes applied to the YCbCr planes first (then integer op)
  int alpha_fill;                   // alpha value when the target wants alpha and the input has none
  int out_bytes;                    // bytes per output sample (1 or 2)
  int special;                      // matrix_coefficients branches of the generic op (yuv2rgb.cc:222-262): 1 = 0 (GBR), 2 = 8 (YCgCo), 3 = 16 (YCgCo-Re)
};

__device__ __forceinline__ int clip_f(float fx, int maxv) {      // common_utils.h:108-114 clip_f_u16
  int x = __float2int_rz(__fadd_rn(fx, 0.5f));
  return x < 0 ? 0 : (x > maxv ? maxv : x);
}
__device__ __forceinline__ int clip_u8(int x) { return x < 0 ? 0 : (x > 255 ? 255 : x); }

template <typename T>
__device__ __forceinline__ void convert_px(const K6Args& p, int Y, int Cb, int Cr, int& r, int& g, int& b) {
  if (p.sh < 0) { r = g = b = Y; return; }
  if (p.int_mode) {                                               // yuv2rgb.cc:401-417
    int cb = Cb - 128, cr = Cr - 128;
    r = clip_u8(Y + ((p.ci[0] * cr + 128) >> 8));
    g = clip_u8(Y + ((p.ci[1] * cb + p.ci[2] * cr + 128) >> 8));
    b = clip_u8(Y + ((p.ci[3] * cb + 128) >> 8));
    return;
  }
  const int half = 1 << (p.bpp - 1), maxv = (1 << p.bpp) - 1;     // yuv2rgb.cc:270-282
  if (p.special) {                                                // yuv2rgb.cc:222-262
    if (p.special == 1) {                                         // GBR: copy, or range-expand
      if (p.full_range) { r = Cr; g = Y; b = Cb; }
      else {
        const float lro = (float)(16 << (p.bpp - 8));
        r = clip_f(__fmul_rn(__fsub_rn((float)Cr, lro), 1.1429f), maxv);
        g = clip_f(__fmul_rn(__fsub_rn((float)Y, lro), 1.1689f), maxv);
        b = clip_f(__fmul_rn(__fsub_rn((float)Cb, lro), 1.1429f), maxv);
      }
    } else if (p.special == 2) {                                  // YCgCo; clip_int_u8 also for > 8 bit (reference quirk, :240-242)
      const int cb = Cb - half, cr = Cr - half;
      r = clip_u8(Y - cb + cr); g = clip_u8(Y + cb); b = clip_u8(Y - cb - cr);
    } else {                                                      // YCgCo-Re: int16 arithmetic, x4
      const short yy = (short)Y, cb = (short)((short)Cb - (short)half), cr = (short)((short)Cr - (short)half);
      const short t = (short)(yy - (cb >> 1)), gg = (short)(t + cb), bb = (short)(t - (cr >> 1)), rr = (short)(bb + cr);
      const int rv = rr * 4, gv = gg * 4, bv = bb * 4;
      r = rv < 0 ? 0 : (rv > maxv ? maxv : rv); g = gv < 0 ? 0 : (gv > maxv ? maxv : gv); b = bv < 0 ? 0 : (bv > maxv ? maxv : bv);
    }
    if (p.sdr_shift) { r >>= p.sdr_shift; g >>= p.sdr_shift; b >>= p.sdr_shift; }
    return;
  }
  float yv = (float)Y, cb = (float)(Cb - half), cr = (float)(Cr - half);
  if (!p.full_range) {
    yv = __fmul_rn(__fsub_rn(yv, (float)(16 << (p.bpp - 8))), 1.1689f);
    cb = __fmul_rn(cb, 1.1429f);
    cr = __fmul_rn(cr, 1.1429f);
  }
  r = clip_f(__fadd_rn(yv, __fmul_rn(p.cf[0], cr)), maxv);
  g = clip_f(__fadd_rn(__fadd_rn(yv, __fmul_rn(p.cf[1], cb)), __fmul_rn(p.cf[2], cr)), maxv);
  b = clip_f(__fadd_rn(yv, __fmul_rn(p.cf[3], cb)), maxv);
  if (p.sdr_shift) { r >>= p.sdr_shift; g >>= p.sdr_shift; b >>= p.sdr_shift; }
}

// stage a w x h window (origin x0,y0, clipped to pw x ph) of a plane into shared memory
template <typename T>
__device__ __forceinline__ void stage_plane(T (*dst)[TILE + SPAD], const void* base, long long stride, int x0, int y0,
                                            int w, int h, int pw, int ph) {
  const int tid = threadIdx.x;
  constexpr int VEC = 16 / sizeof(T);
  const bool vec_ok = (x0 % VEC == 0) && (w % VEC == 0) && (x0 + w <= pw) && (stride % 16 == 0) &&
                      ((reinterpret_cast<uintptr_t>(base) & 15) == 0);
  if (vec_ok) {
    const int per_row = w / VEC;
    for (int i = tid; i < per_row * h; i += blockDim.x) {
      int r = i / per_row, c = i - r * per_row;
      int sy = y0 + r;
      if (sy >= ph) continue;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(static_cast<const char*>(base) + (long long)sy * stride) + (x0 / VEC + c));
      T tmp[VEC];
      *reinterpret_cast<uint4*>(tmp) = v;
#pragma unroll
      for (int k = 0; k < VEC; k++) dst[r][c * VEC + k] = tmp[k];
    }
  } else {
    for (int i = tid; i < w * h; i += blockDim.x) {
      int r = i / w, c = i - r * w;
      int sy = y0 + r, sx = x0 + c;
      if (sy < ph && sx < pw) dst[r][c] = reinterpret_cast<const T*>(static_cast<const char*>(base) + (long long)sy * stride)[sx];
    }
  }
}

// One output pixel from the source position (sx, sy) of the decoded picture: luma and alpha there, chroma at
// (sx >> sh, sy >> sv) (nearest-neighbour upsampling), then convert_px.  at(c, x, y) reads sample (x, y) of plane c
// (0 Y, 1 Cb, 2 Cr, 3 alpha) wherever the kernel keeps it.
template <typename T, bool HAS_ALPHA, typename At>
__device__ __forceinline__ void k6_pixel(const K6Args& p, const At& at, int sx, int sy, int& r, int& g, int& b, int& a) {
  const int Y = at(0, sx, sy) >> p.pre_shift;
  int Cb = 0, Cr = 0;
  if (p.sh >= 0) { Cb = at(1, sx >> p.sh, sy >> p.sv) >> p.pre_shift; Cr = at(2, sx >> p.sh, sy >> p.sv) >> p.pre_shift; }
  convert_px<T>(p, Y, Cb, Cr, r, g, b);
  a = HAS_ALPHA ? at(3, sx, sy) >> (p.sdr_shift + p.pre_shift) : p.alpha_fill;
}

// Writes the npx (<= 16) converted pixels starting at output pixel (x_begin, y) in the target layout p.out_fmt.
__device__ __forceinline__ void k6_store_strip(const K6Args& p, int y, int x_begin, int npx, const int (&R)[16], const int (&G)[16],
                                               const int (&B)[16], const int (&A)[16]) {
  char* orow = static_cast<char*>(p.out[0]) + (long long)y * p.os;
  const int fmt = p.out_fmt;
  if (fmt == B200_CHROMA_444) {                      // planar RGB (yuv2rgb.cc Op_YCbCr_to_RGB output)
    for (int c = 0; c < 3; c++) {
      const int* v = c == 0 ? R : (c == 1 ? G : B);
      char* prow = static_cast<char*>(p.out[c]) + (long long)y * p.os;
      if (p.out_bytes == 1) for (int i = 0; i < npx; i++) reinterpret_cast<uint8_t*>(prow)[x_begin + i] = (uint8_t)v[i];
      else for (int i = 0; i < npx; i++) reinterpret_cast<uint16_t*>(prow)[x_begin + i] = (uint16_t)v[i];
    }
    return;
  }
  // interleaved formats: build the 16-pixel strip in registers, then 128-bit stores
  const int nch = (fmt == B200_CHROMA_INTERLEAVED_RGB || fmt == B200_CHROMA_INTERLEAVED_RRGGBB_BE || fmt == B200_CHROMA_INTERLEAVED_RRGGBB_LE) ? 3 : 4;
  const int bps = (fmt == B200_CHROMA_INTERLEAVED_RGB || fmt == B200_CHROMA_INTERLEAVED_RGBA) ? 1 : 2;
  const int le = (fmt == B200_CHROMA_INTERLEAVED_RRGGBB_LE || fmt == B200_CHROMA_INTERLEAVED_RRGGBBAA_LE);
  __align__(16) uint8_t buf[16 * 8];
  if (bps == 1) {
#pragma unroll
    for (int i = 0; i < 16; i++) {
      if (nch == 3) { buf[3 * i] = (uint8_t)R[i]; buf[3 * i + 1] = (uint8_t)G[i]; buf[3 * i + 2] = (uint8_t)B[i]; }
      else { buf[4 * i] = (uint8_t)R[i]; buf[4 * i + 1] = (uint8_t)G[i]; buf[4 * i + 2] = (uint8_t)B[i]; buf[4 * i + 3] = (uint8_t)A[i]; }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int v[4] = {R[i], G[i], B[i], A[i]};
#pragma unroll
      for (int c = 0; c < 4; c++) {
        if (c < nch) {
          buf[(nch * i + c) * 2 + (le ? 1 : 0)] = (uint8_t)(v[c] >> 8);     // yuv2rgb.cc:715-729
          buf[(nch * i + c) * 2 + (le ? 0 : 1)] = (uint8_t)(v[c] & 0xff);
        }
      }
    }
  }
  const int bpp_out = nch * bps;
  char* dst = orow + (long long)x_begin * bpp_out;
  const int nbytes = npx * bpp_out;
  if (npx == 16 && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
    const uint4* src = reinterpret_cast<const uint4*>(buf);
    const int nvec = bpp_out;                      // 16 px * bpp_out bytes / 16
    for (int k = 0; k < nvec; k++) __stcs(reinterpret_cast<uint4*>(dst) + k, src[k]);
  } else {
    for (int k = 0; k < nbytes; k++) dst[k] = buf[k];
  }
}

template <typename T, bool HAS_ALPHA>
__global__ void __launch_bounds__(256) k6_color_kernel(const K6Args p) {
  __shared__ __align__(16) T sY[TILE][TILE + SPAD];
  __shared__ __align__(16) T sCb[SROWS][TILE + SPAD];
  __shared__ __align__(16) T sCr[SROWS][TILE + SPAD];
  __shared__ __align__(16) T sA[HAS_ALPHA ? TILE : 1][TILE + SPAD];

  const int ox = blockIdx.x * TILE, oy = blockIdx.y * TILE;
  const int tw = min(TILE, p.out_w - ox), th = min(TILE, p.out_h - oy);
  // source window = image of the output tile's corners
  const int ax = p.m[0] * ox + p.m[1] * oy + p.m[2], ay = p.m[3] * ox + p.m[4] * oy + p.m[5];
  const int bx = p.m[0] * (ox + tw - 1) + p.m[1] * (oy + th - 1) + p.m[2];
  const int by = p.m[3] * (ox + tw - 1) + p.m[4] * (oy + th - 1) + p.m[5];
  const int s0x = min(ax, bx), s0y = min(ay, by);
  const int sw = abs(ax - bx) + 1, sh_ = abs(ay - by) + 1;

  // round the window out to 16-sample columns where the picture allows so the vector path is taken
  int lx0 = s0x & ~15, lw = ((s0x + sw + 15) & ~15) - lx0;
  if (lw > TILE || lx0 + lw > p.src_w) { lx0 = s0x; lw = sw; }
  stage_plane<T>(sY, p.y, p.ys, lx0, s0y, lw, sh_, p.src_w, p.src_h);
  if (HAS_ALPHA) stage_plane<T>(sA, p.a, p.as, lx0, s0y, lw, sh_, p.src_w, p.src_h);
  int c0x = 0, c0y = 0;
  if (p.sh >= 0) {
    const int cw_pl = (p.src_w + (1 << p.sh) - 1) >> p.sh, ch_pl = (p.src_h + (1 << p.sv) - 1) >> p.sv;
    c0x = lx0 >> p.sh; c0y = s0y >> p.sv;
    int cw = ((lx0 + lw - 1) >> p.sh) - c0x + 1, chh = ((s0y + sh_ - 1) >> p.sv) - c0y + 1;
    int cl0 = c0x & ~15, clw = ((c0x + cw + 15) & ~15) - cl0;
    if (clw > TILE || cl0 + clw > cw_pl) { cl0 = c0x; clw = cw; }
    stage_plane<T>(sCb, p.cb, p.cs, cl0, c0y, clw, chh, cw_pl, ch_pl);
    stage_plane<T>(sCr, p.cr, p.cs, cl0, c0y, clw, chh, cw_pl, ch_pl);
    c0x = cl0;
  }
  __syncthreads();

  const int row = threadIdx.x >> 2, strip = threadIdx.x & 3;
  const int y = oy + row, x_begin = ox + strip * 16;
  if (row >= th || x_begin >= p.out_w) return;
  const int npx = min(16, p.out_w - x_begin);
  auto at = [&](int c, int sx, int sy) -> int {
    return c == 0 ? sY[sy - s0y][sx - lx0] : c == 1 ? sCb[sy - c0y][sx - c0x] : c == 2 ? sCr[sy - c0y][sx - c0x] : sA[sy - s0y][sx - lx0];
  };

  int R[16], G[16], B[16], A[16];
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int x = x_begin + (i < npx ? i : 0);
    k6_pixel<T, HAS_ALPHA>(p, at, p.m[0] * x + p.m[1] * y + p.m[2], p.m[3] * x + p.m[4] * y + p.m[5], R[i], G[i], B[i], A[i]);
  }
  k6_store_strip(p, y, x_begin, npx, R, G, B, A);
}

// Scaled K6: the unscaled K6 picture (out_w x out_h) sampled by HeifPixelImage::scale_nearest_neighbor to dst_w x dst_h
// (pixelimage.cc:1876-1911, :1936-1966), computing only the kept pixels.  Output pixel (x, y) is K6 pixel
// (ix, iy) = (x * out_w / dst_w, y * out_h / dst_h) in 64-bit arithmetic, all components of a pixel together.  A CTA owns
// a 64 x 64 tile of the scaled picture with k6_color_kernel's thread layout; the tile's 64 column indices are computed once
// into shared memory, and samples are read from the planes directly (a downscaled tile's source does not fit a window).
template <typename T, bool HAS_ALPHA>
__global__ void __launch_bounds__(256) k6_scaled_kernel(const K6Args p) {
  __shared__ int s_ix[TILE];
  const int ox = blockIdx.x * TILE, oy = blockIdx.y * TILE;
  if (threadIdx.x < TILE) s_ix[threadIdx.x] = (int)((unsigned long long)(ox + threadIdx.x) * (unsigned)p.out_w / (unsigned)p.dst_w);
  __syncthreads();
  const int row = threadIdx.x >> 2, strip = threadIdx.x & 3;
  const int y = oy + row, x_begin = ox + strip * 16;
  if (y >= p.dst_h || x_begin >= p.dst_w) return;
  const int npx = min(16, p.dst_w - x_begin);
  const int iy = (int)((unsigned long long)y * (unsigned)p.out_h / (unsigned)p.dst_h);
  auto at = [&](int c, int sx, int sy) -> int {
    const void* base = c == 0 ? p.y : c == 1 ? p.cb : c == 2 ? p.cr : p.a;
    const long long stride = c == 0 ? p.ys : c == 3 ? p.as : p.cs;
    return __ldg(reinterpret_cast<const T*>(static_cast<const char*>(base) + (long long)sy * stride) + sx);
  };

  int R[16], G[16], B[16], A[16];
#pragma unroll
  for (int i = 0; i < 16; i++) {
    const int ix = s_ix[strip * 16 + (i < npx ? i : 0)];
    k6_pixel<T, HAS_ALPHA>(p, at, p.m[0] * ix + p.m[1] * iy + p.m[2], p.m[3] * ix + p.m[4] * iy + p.m[5], R[i], G[i], B[i], A[i]);
  }
  k6_store_strip(p, y, x_begin, npx, R, G, B, A);
}


// ---------------------------------------------------------------------------------------------- bilinear chroma
// Op_YCbCr420_bilinear_to_YCbCr444<T> (chroma_sampling.cc:623-700): one thread per full-resolution chroma sample.
// Interior: weights 9/3/3/1 (+8)/16; borders: 3/1 (+2)/4 with the reference's source indexing (cx/2, cy/2); corners copied.
template <typename T>
__global__ void __launch_bounds__(256) bilinear_420_to_444_kernel(const T* __restrict__ in_cb, const T* __restrict__ in_cr, long long cs,
                                                                  T* __restrict__ out_cb, T* __restrict__ out_cr, long long os, int w, int h) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const bool weven = (w & 1) == 0, heven = (h & 1) == 0;
  for (int c = 0; c < 2; c++) {
    const T* in = c ? in_cr : in_cb;
    T* out = c ? out_cr : out_cb;
    int v;
    const bool top = y == 0, left = x == 0, right = weven && x == w - 1, bottom = heven && y == h - 1;
    if ((top || bottom) && (left || right)) v = in[(long long)(top ? 0 : h / 2 - 1) * cs + (left ? 0 : w / 2 - 1)];
    else if (top || bottom) {
      const int cx = (x - 1) >> 1, row = top ? 0 : h / 2 - 1;
      const int a = in[(long long)row * cs + cx / 2], b = in[(long long)row * cs + cx / 2 + 1];
      v = (x & 1) ? (3 * a + b + 2) / 4 : (a + 3 * b + 2) / 4;
    } else if (left || right) {
      const int cy = (y - 1) >> 1, col = left ? 0 : w / 2 - 1;
      const int a = in[(long long)(cy / 2) * cs + col], b = in[(long long)(cy / 2 + 1) * cs + col];
      v = (y & 1) ? (3 * a + b + 2) / 4 : (a + 3 * b + 2) / 4;
    } else {
      const int cx = (x - 1) >> 1, cy = (y - 1) >> 1;
      const int c00 = in[(long long)cy * cs + cx], c01 = in[(long long)cy * cs + cx + 1], c10 = in[(long long)(cy + 1) * cs + cx], c11 = in[(long long)(cy + 1) * cs + cx + 1];
      const int wx0 = (x & 1) ? 3 : 1, wx1 = 4 - wx0, wy0 = (y & 1) ? 3 : 1, wy1 = 4 - wy0;
      v = (c00 * wx0 * wy0 + c01 * wx1 * wy0 + c10 * wx0 * wy1 + c11 * wx1 * wy1 + 8) / 16;
    }
    out[(long long)y * os + x] = (T)v;
  }
}

// ---------------------------------------------------------------------------------------------- fast path
// Identity geometry, 4:2:0, no alpha, 16-byte aligned rows: no shared-memory staging.  One thread = 16 x 2 output
// pixels: 2 x 16 luma samples and 8 + 8 chroma samples come in with 128-bit / 64-bit loads, the chroma terms are
// computed once per 2x2 block (identical values to the per-pixel evaluation of the reference: same float products,
// same evaluation order), and each row leaves as NCH * BPS 128-bit streaming stores.
template <typename T, int INT_MODE, int NCH, int BPS, int LE>
__global__ void __launch_bounds__(256) k6_direct_kernel(const K6Args p) {
  const int x16 = blockIdx.x * blockDim.x + threadIdx.x;
  const int y2 = blockIdx.y * blockDim.y + threadIdx.y;
  if (x16 * 16 >= p.out_w || y2 * 2 >= p.out_h) return;
  const int x = x16 * 16, y = y2 * 2;
  T Y[2][16], Cb[8], Cr[8];
  if (sizeof(T) == 1) {
    *reinterpret_cast<uint4*>(Y[0]) = __ldcs(reinterpret_cast<const uint4*>(static_cast<const char*>(p.y) + (long long)y * p.ys + x));
    *reinterpret_cast<uint4*>(Y[1]) = __ldcs(reinterpret_cast<const uint4*>(static_cast<const char*>(p.y) + (long long)(y + 1) * p.ys + x));
    *reinterpret_cast<uint2*>(Cb) = __ldcs(reinterpret_cast<const uint2*>(static_cast<const char*>(p.cb) + (long long)y2 * p.cs + x / 2));
    *reinterpret_cast<uint2*>(Cr) = __ldcs(reinterpret_cast<const uint2*>(static_cast<const char*>(p.cr) + (long long)y2 * p.cs + x / 2));
  } else {
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const uint4* src = reinterpret_cast<const uint4*>(static_cast<const char*>(p.y) + (long long)(y + r) * p.ys + x * 2);
      reinterpret_cast<uint4*>(Y[r])[0] = __ldcs(src); reinterpret_cast<uint4*>(Y[r])[1] = __ldcs(src + 1);
    }
    *reinterpret_cast<uint4*>(Cb) = __ldcs(reinterpret_cast<const uint4*>(static_cast<const char*>(p.cb) + (long long)y2 * p.cs + x));
    *reinterpret_cast<uint4*>(Cr) = __ldcs(reinterpret_cast<const uint4*>(static_cast<const char*>(p.cr) + (long long)y2 * p.cs + x));
  }
  const int bpp = p.bpp, half = 1 << (bpp - 1), maxv = (1 << bpp) - 1, pre = p.pre_shift, post = p.sdr_shift;
  const float lro = (float)(16 << (bpp - 8));
  const bool full = p.full_range != 0;
  // per chroma sample terms
  int ri[8], gi[8], bi[8]; float rf[8], g1f[8], g2f[8], bf[8];
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const int cbv = (int)Cb[i] >> pre, crv = (int)Cr[i] >> pre;
    if (INT_MODE) {
      const int cb = cbv - 128, cr = crv - 128;
      ri[i] = (p.ci[0] * cr + 128) >> 8; gi[i] = (p.ci[1] * cb + p.ci[2] * cr + 128) >> 8; bi[i] = (p.ci[3] * cb + 128) >> 8;
    } else {
      float cb = (float)(cbv - half), cr = (float)(crv - half);
      if (!full) { cb = __fmul_rn(cb, 1.1429f); cr = __fmul_rn(cr, 1.1429f); }
      rf[i] = __fmul_rn(p.cf[0], cr); g1f[i] = __fmul_rn(p.cf[1], cb); g2f[i] = __fmul_rn(p.cf[2], cr); bf[i] = __fmul_rn(p.cf[3], cb);
    }
  }
#pragma unroll
  for (int r = 0; r < 2; r++) {
    __align__(16) uint8_t buf[16 * NCH * BPS];
#pragma unroll
    for (int i = 0; i < 16; i++) {
      const int yv0 = (int)Y[r][i] >> pre;
      int R, G, B;
      if (INT_MODE) { R = clip_u8(yv0 + ri[i >> 1]); G = clip_u8(yv0 + gi[i >> 1]); B = clip_u8(yv0 + bi[i >> 1]); }
      else {
        float yv = (float)yv0;
        if (!full) yv = __fmul_rn(__fsub_rn(yv, lro), 1.1689f);
        R = clip_f(__fadd_rn(yv, rf[i >> 1]), maxv) >> post;
        G = clip_f(__fadd_rn(__fadd_rn(yv, g1f[i >> 1]), g2f[i >> 1]), maxv) >> post;
        B = clip_f(__fadd_rn(yv, bf[i >> 1]), maxv) >> post;
      }
      if (BPS == 1) {
        buf[NCH * i] = (uint8_t)R; buf[NCH * i + 1] = (uint8_t)G; buf[NCH * i + 2] = (uint8_t)B;
        if (NCH == 4) buf[NCH * i + 3] = (uint8_t)p.alpha_fill;
      } else {
        const int v[4] = {R, G, B, p.alpha_fill};
#pragma unroll
        for (int c = 0; c < NCH; c++) { buf[(NCH * i + c) * 2 + (LE ? 1 : 0)] = (uint8_t)(v[c] >> 8); buf[(NCH * i + c) * 2 + (LE ? 0 : 1)] = (uint8_t)(v[c] & 0xff); }
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(static_cast<char*>(p.out[0]) + (long long)(y + r) * p.os + (long long)x * NCH * BPS);
#pragma unroll
    for (int k = 0; k < NCH * BPS; k++) __stcs(dst + k, reinterpret_cast<const uint4*>(buf)[k]);
  }
}

template <typename T, int INT_MODE>
static bool launch_direct(const K6Args& a, cudaStream_t s) {
  dim3 blk(32, 8), grid((a.out_w / 16 + 31) / 32, (a.out_h / 2 + 7) / 8);
  switch (a.out_fmt) {
    case B200_CHROMA_INTERLEAVED_RGB: k6_direct_kernel<T, INT_MODE, 3, 1, 0><<<grid, blk, 0, s>>>(a); return true;
    case B200_CHROMA_INTERLEAVED_RGBA: k6_direct_kernel<T, INT_MODE, 4, 1, 0><<<grid, blk, 0, s>>>(a); return true;
    case B200_CHROMA_INTERLEAVED_RRGGBB_LE: if (INT_MODE) return false; k6_direct_kernel<T, 0, 3, 2, 1><<<grid, blk, 0, s>>>(a); return true;
    case B200_CHROMA_INTERLEAVED_RRGGBB_BE: if (INT_MODE) return false; k6_direct_kernel<T, 0, 3, 2, 0><<<grid, blk, 0, s>>>(a); return true;
    case B200_CHROMA_INTERLEAVED_RRGGBBAA_LE: if (INT_MODE) return false; k6_direct_kernel<T, 0, 4, 2, 1><<<grid, blk, 0, s>>>(a); return true;
    case B200_CHROMA_INTERLEAVED_RRGGBBAA_BE: if (INT_MODE) return false; k6_direct_kernel<T, 0, 4, 2, 0><<<grid, blk, 0, s>>>(a); return true;
    default: return false;
  }
}

// ---------------------------------------------------------------------------------------------- host
// nclx.cc:84-173, evaluated in float exactly as the reference does
static void primaries_of(int idx, float p[8], bool& defined) {
  defined = true;   // order: gx, gy, bx, by, rx, ry, wx, wy (nclx.cc:31-42 constructor argument order)
  switch (idx) {
    case 1: { const float v[8] = {0.300f, 0.600f, 0.150f, 0.060f, 0.640f, 0.330f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    case 4: { const float v[8] = {0.21f, 0.71f, 0.14f, 0.08f, 0.67f, 0.33f, 0.310f, 0.316f}; memcpy(p, v, sizeof v); break; }
    case 5: { const float v[8] = {0.29f, 0.60f, 0.15f, 0.06f, 0.64f, 0.33f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    case 6: case 7: { const float v[8] = {0.310f, 0.595f, 0.155f, 0.070f, 0.630f, 0.340f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    case 8: { const float v[8] = {0.243f, 0.692f, 0.145f, 0.049f, 0.681f, 0.319f, 0.310f, 0.316f}; memcpy(p, v, sizeof v); break; }
    case 9: { const float v[8] = {0.170f, 0.797f, 0.131f, 0.046f, 0.708f, 0.292f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    case 10: { const float v[8] = {0.0f, 1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 0.333333f, 0.33333f}; memcpy(p, v, sizeof v); break; }
    case 11: { const float v[8] = {0.265f, 0.690f, 0.150f, 0.060f, 0.680f, 0.320f, 0.314f, 0.351f}; memcpy(p, v, sizeof v); break; }
    case 12: { const float v[8] = {0.265f, 0.690f, 0.150f, 0.060f, 0.680f, 0.320f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    case 22: { const float v[8] = {0.295f, 0.605f, 0.155f, 0.077f, 0.630f, 0.340f, 0.3127f, 0.3290f}; memcpy(p, v, sizeof v); break; }
    default: defined = false; for (int i = 0; i < 8; i++) p[i] = 0.0f;
  }
}

static void kr_kb(int matrix, int primaries, float* pKr, float* pKb);
void ycbcr_to_rgb_coefficients(int matrix, int primaries, float out[4]) {
  float kr, kb; kr_kb(matrix, primaries, &kr, &kb);
  if (kb != 0 || kr != 0) {
    out[0] = 2 * (-kr + 1);
    out[1] = 2 * kb * (-kb + 1) / (kb + kr - 1);
    out[2] = 2 * kr * (-kr + 1) / (kb + kr - 1);
    out[3] = 2 * (-kb + 1);
  } else { out[0] = 1.402f; out[1] = -0.344136f; out[2] = -0.714136f; out[3] = 1.772f; }
}
// RGB -> YCbCr coefficients of the same matrix (nclx.cc:177-200)
static void rgb_to_ycbcr_coefficients(int matrix, int primaries, float c[3][3]) {
  float Kr, Kb; kr_kb(matrix, primaries, &Kr, &Kb);
  if (Kb != 0 || Kr != 0) {
    c[0][0] = Kr; c[0][1] = 1 - Kr - Kb; c[0][2] = Kb;
    c[1][0] = -Kr / (1 - Kb) / 2; c[1][1] = -(1 - Kr - Kb) / (1 - Kb) / 2; c[1][2] = 0.5f;
    c[2][0] = 0.5f; c[2][1] = -(1 - Kr - Kb) / (1 - Kr) / 2; c[2][2] = -Kb / (1 - Kr) / 2;
  } else {
    c[0][0] = 0.299f; c[0][1] = 0.587f; c[0][2] = 0.114f; c[1][0] = -0.168735f; c[1][1] = -0.331264f; c[1][2] = 0.5f;
    c[2][0] = 0.5f; c[2][1] = -0.418688f; c[2][2] = -0.081312f;
  }
}
static void kr_kb(int matrix, int primaries, float* pKr, float* pKb) {
  volatile float Kr = 0.0f, Kb = 0.0f;              // volatile: keep every intermediate rounded to float
  if (matrix == 12 || matrix == 13) {
    float p[8]; bool def;
    primaries_of(primaries, p, def);
    const float gx = p[0], gy = p[1], bx = p[2], by = p[3], rx = p[4], ry = p[5], wx = p[6], wy = p[7];
    float zr = 1 - (rx + ry), zg = 1 - (gx + gy), zb = 1 - (bx + by), zw = 1 - (wx + wy);
    float denom = wy * (rx * (gy * zb - by * zg) + gx * (by * zr - ry * zb) + bx * (ry * zg - gy * zr));
    if (denom != 0.0f) {
      Kr = (ry * (wx * (gy * zb - by * zg) + wy * (bx * zg - gx * zb) + zw * (gx * by - bx * gy))) / denom;
      Kb = (by * (wx * (ry * zg - gy * zr) + wy * (gx * zr - rx * zg) + zw * (rx * gy - gx * ry))) / denom;
    }
  } else {
    switch (matrix) {
      case 1: Kr = 0.2126f; Kb = 0.0722f; break;
      case 4: Kr = 0.30f; Kb = 0.11f; break;
      case 5: case 6: Kr = 0.299f; Kb = 0.114f; break;
      case 7: Kr = 0.212f; Kb = 0.087f; break;
      case 9: case 10: Kr = 0.2627f; Kb = 0.0593f; break;
      default: break;
    }
  }
  *pKr = Kr; *pKb = Kb;
}

// Plane-wise geometry (rotate / mirror / crop on a 4:2:0 picture as the reference's ComponentStorage code does it) for
// the transforms that precede the 4:4:4 conversion point: luma-resolution planes follow the affine map, chroma planes
// follow it at half resolution (those transforms keep the 2x2 chroma grid aligned, otherwise the conversion point would
// have been earlier).
template <typename T>
__global__ void plane_geometry_kernel(const T* __restrict__ in, long long in_stride, T* __restrict__ out, long long out_stride, int out_w, int out_h,
                                      int m0, int m1, int m2, int m3, int m4, int m5, int shx, int shy) {
  const int u = blockIdx.x * blockDim.x + threadIdx.x, v = blockIdx.y;
  if (u >= out_w || v >= out_h) return;
  const int sx = (m0 * (u << shx) + m1 * (v << shy) + m2) >> shx, sy = (m3 * (u << shx) + m4 * (v << shy) + m5) >> shy;
  out[(long long)v * out_stride + u] = in[(long long)sy * in_stride + sx];
}

// Op_YCbCr422_bilinear_to_YCbCr444<T> (chroma_sampling.cc:784-905): chroma (w + 1) / 2 x h -> w x h, both planes
template <typename T>
__global__ void bilinear_422_to_444_kernel(const T* __restrict__ cb, const T* __restrict__ cr, long long in_stride, T* __restrict__ ocb, T* __restrict__ ocr,
                                           long long out_stride, int w, int h) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= w || y >= h) return;
  const T* rb = cb + (long long)y * in_stride; const T* rr = cr + (long long)y * in_stride;
  unsigned vb, vr;
  if (x == 0) { vb = rb[0]; vr = rr[0]; }
  else if ((w & 1) == 0 && x == w - 1) { vb = rb[w / 2 - 1]; vr = rr[w / 2 - 1]; }
  else if (x & 1) { const int c = x >> 1; vb = ((unsigned)rb[c] * 3 + rb[c + 1] + 2) / 4; vr = ((unsigned)rr[c] * 3 + rr[c + 1] + 2) / 4; }
  else { const int c = (x - 1) >> 1; vb = ((unsigned)rb[c] + (unsigned)rb[c + 1] * 3 + 2) / 4; vr = ((unsigned)rr[c] + (unsigned)rr[c + 1] * 3 + 2) / 4; }
  ocb[(long long)y * out_stride + x] = (T)vb; ocr[(long long)y * out_stride + x] = (T)vr;
}

// The 4:4:4 conversion point of a LIMITED-range picture: the reference's target profile there is full range, and the path
// its planner finds is Op_YCbCr_to_RGB<T> (yuv2rgb.cc:263-279) followed by Op_RGB_to_YCbCr<T> (rgb2yuv.cc:226-300) with
// the same matrix.  One pass over the three 4:4:4 planes, float arithmetic in the reference's order.
struct RangeArgs { float cf[4]; float c[3][3]; int bpp; };
template <typename T>
__global__ void range_limited_to_full_444_kernel(const T* __restrict__ y, long long ys, const T* __restrict__ cb, const T* __restrict__ cr, long long cs,
                                                 T* __restrict__ oy, long long oys, T* __restrict__ ocb, T* __restrict__ ocr, long long ocs, int w, int h, RangeArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, yy = blockIdx.y;
  if (x >= w || yy >= h) return;
  const int half = 1 << (a.bpp - 1), maxv = (1 << a.bpp) - 1; const float lro = (float)(16 << (a.bpp - 8));
  float yv = (float)y[(long long)yy * ys + x], cbv = (float)((int)cb[(long long)yy * cs + x] - half), crv = (float)((int)cr[(long long)yy * cs + x] - half);
  yv = __fmul_rn(__fsub_rn(yv, lro), 1.1689f); cbv = __fmul_rn(cbv, 1.1429f); crv = __fmul_rn(crv, 1.1429f);
  const float r = (float)clip_f(__fadd_rn(yv, __fmul_rn(a.cf[0], crv)), maxv);
  const float g = (float)clip_f(__fadd_rn(__fadd_rn(yv, __fmul_rn(a.cf[1], cbv)), __fmul_rn(a.cf[2], crv)), maxv);
  const float b = (float)clip_f(__fadd_rn(yv, __fmul_rn(a.cf[3], cbv)), maxv);
  auto dot = [&](int k) { return __fadd_rn(__fadd_rn(__fmul_rn(r, a.c[k][0]), __fmul_rn(g, a.c[k][1])), __fmul_rn(b, a.c[k][2])); };
  oy[(long long)yy * oys + x] = (T)clip_f(dot(0), maxv);
  ocb[(long long)yy * ocs + x] = (T)clip_f(__fadd_rn(dot(1), (float)half), maxv);
  ocr[(long long)yy * ocs + x] = (T)clip_f(__fadd_rn(dot(2), (float)half), maxv);
}

// 4:2:0 / 4:2:2 picture -> (plane-wise geometry `pre`) -> Op_YCbCr420_bilinear_to_YCbCr444 / Op_YCbCr422_bilinear_to_YCbCr444
// -> (limited range: range conversion through RGB) -> the rest of the chain and the colour conversion from 4:4:4.
// Serves the reference's 4:4:4 conversion point and bilinear upsampling after geometry.  The 4:4:4 intermediates are full
// size; only the last conversion is scaled (scale_w x scale_h, 0 x 0 = unscaled).
static int convert_via_444(const b200_planes* in, const b200_geometry* g, const b200_color_options* opt, void* out, void* out_g, void* out_b,
                           size_t out_stride, cudaStream_t stream, int* pipeline, bool range_convert, int scale_w, int scale_h) {
  const int bps = in->bit_depth > 8 ? 2 : 1;
  const bool c422 = in->chroma == B200_CHROMA_422;
  const int shy = c422 ? 0 : 1;
  const int pw = g->pre_w, ph = g->pre_h;
  int pcw, pch;
  chroma_size(in->chroma, pw, ph, pcw, pch);
  const bool pre_identity = is_identity(g->pre, pw, ph, in->width, in->height);
  const size_t pitch = (((size_t)pw * bps) + 255) & ~(size_t)255, cpitch = (((size_t)pcw * bps) + 255) & ~(size_t)255;
  // scratch planes, each only where the call writes it: Y' (geometry or range conversion), A' (geometry of alpha),
  // Cb444, Cr444, Cb' and Cr' (geometry)
  const size_t n_full = pitch * ph, n_y = !pre_identity || range_convert ? n_full : 0, n_a = !pre_identity && in->alpha ? n_full : 0;
  const size_t n_c = pre_identity ? 0 : cpitch * pch;
  char* tmp = nullptr;
  B200_CUDA_CHECK(cudaMallocAsync(&tmp, n_y + n_a + 2 * n_full + 2 * n_c, stream));
  char *ty = tmp, *ta = ty + n_y, *u_cb = ta + n_a, *u_cr = u_cb + n_full, *tcb = u_cr + n_full, *tcr = tcb + n_c;
  b200_planes p = *in;
  auto run = [&](auto sample) {
    using T = decltype(sample);
    auto el = [](size_t stride) { return (long long)(stride / sizeof(T)); };      // byte stride -> elements
    if (!pre_identity) {
      const int* q = g->pre;
      auto geom = [&](const void* src, size_t sstride, void* dst, size_t dstride, int w, int h, int sx, int sy) {
        plane_geometry_kernel<T><<<dim3((w + 255) / 256, h), 256, 0, stream>>>((const T*)src, el(sstride), (T*)dst, el(dstride), w, h,
                                                                               q[0], q[1], q[2], q[3], q[4], q[5], sx, sy);
      };
      geom(in->y, in->y_stride, ty, pitch, pw, ph, 0, 0);
      geom(in->cb, in->c_stride, tcb, cpitch, pcw, pch, 1, shy);
      geom(in->cr, in->c_stride, tcr, cpitch, pcw, pch, 1, shy);
      if (in->alpha) geom(in->alpha, in->alpha_stride, ta, pitch, pw, ph, 0, 0);
      p.y = ty; p.y_stride = pitch; p.cb = tcb; p.cr = tcr; p.c_stride = cpitch;
      if (in->alpha) { p.alpha = ta; p.alpha_stride = pitch; }
      p.width = pw; p.height = ph;
    }
    const dim3 grid((pw + 255) / 256, ph);
    if (c422) bilinear_422_to_444_kernel<T><<<grid, 256, 0, stream>>>((const T*)p.cb, (const T*)p.cr, el(p.c_stride), (T*)u_cb, (T*)u_cr, el(pitch), pw, ph);
    else bilinear_420_to_444_kernel<T><<<grid, 256, 0, stream>>>((const T*)p.cb, (const T*)p.cr, el(p.c_stride), (T*)u_cb, (T*)u_cr, el(pitch), pw, ph);
    p.cb = u_cb; p.cr = u_cr; p.c_stride = pitch; p.chroma = B200_CHROMA_444;
    if (range_convert) {
      // limited -> full range through RGB; Y goes to the scratch plane (the caller's luma plane is never written)
      RangeArgs ra; ra.bpp = in->bit_depth;
      ycbcr_to_rgb_coefficients(in->matrix_coefficients, in->colour_primaries, ra.cf);
      rgb_to_ycbcr_coefficients(in->matrix_coefficients, in->colour_primaries, ra.c);
      range_limited_to_full_444_kernel<T><<<grid, 256, 0, stream>>>((const T*)p.y, el(p.y_stride), (const T*)u_cb, (const T*)u_cr, el(pitch), (T*)ty,
                                                                     el(pitch), (T*)u_cb, (T*)u_cr, el(pitch), pw, ph, ra);
      p.y = ty; p.y_stride = pitch; p.width = pw; p.height = ph; p.full_range = 1;
    }
  };
  if (bps == 1) run(uint8_t()); else run(uint16_t());
  b200_geometry rest = *g; rest.detour = 0; rest.chroma = B200_CHROMA_444;
  b200_color_options o2 = *opt; o2.chroma_upsampling = 0;
  int rc = launch_color(&p, &rest, &o2, out, out_g, out_b, out_stride, stream, pipeline, scale_w, scale_h);
  if (pipeline) *pipeline |= B200_PIPE_BILINEAR;
  cudaFreeAsync(tmp, stream);
  return rc;
}

// Mirror of the reference planner's choice for the supported states (colorconversion.cc:279-435; the
// measured pipelines are tabulated in SURVEY.md Appendix A and re-checked by tests/test_color_parity.py).
int launch_color(const b200_planes* in, const b200_geometry* g, const b200_color_options* opt, void* out, void* out_g,
                 void* out_b, size_t out_stride, cudaStream_t stream, int* pipeline, int scale_w, int scale_h) {
  if (!in || !g || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  if (in->bit_depth < 8 || in->bit_depth > 16) return set_error(B200_E_UNSUPPORTED, "bit depth %d", in->bit_depth);
  const int fmt = opt->out_chroma;
  const bool interleaved8 = fmt == B200_CHROMA_INTERLEAVED_RGB || fmt == B200_CHROMA_INTERLEAVED_RGBA;
  const bool interleaved16 = fmt >= B200_CHROMA_INTERLEAVED_RRGGBB_BE && fmt <= B200_CHROMA_INTERLEAVED_RRGGBBAA_LE;
  if (!interleaved8 && !interleaved16 && fmt != B200_CHROMA_444) return set_error(B200_E_UNSUPPORTED, "output chroma %d", fmt);
  const int mc = in->matrix_coefficients;
  if (in->chroma != B200_CHROMA_MONO && (mc == 11 || mc == 14))
    return set_error(B200_E_UNSUPPORTED, "matrix_coefficients %d: the reference has no YCbCr->RGB operation for it either (yuv2rgb.cc:107-112)", mc);
  if (interleaved16 && in->bit_depth == 8) return set_error(B200_E_UNSUPPORTED, "8-bit input to RRGGBB output");
  const bool subsampled = in->chroma == B200_CHROMA_420 || in->chroma == B200_CHROMA_422;
  if (g->detour && !subsampled) {
    // the chain was composed with the rules of a subsampled format but the picture is not subsampled: one affine map
    b200_geometry t = *g; t.detour = 0;
    affine_compose(g->pre, g->m, t.m);
    return launch_color(in, &t, opt, out, out_g, out_b, out_stride, stream, pipeline, scale_w, scale_h);
  }
  const bool geom_identity = is_identity(g->m, g->out_w, g->out_h, in->width, in->height) && !g->detour;
  if (subsampled && !geom_identity && g->chroma != in->chroma)
    return set_error(B200_E_INVALID, "geometry was composed for chroma format %d, the picture has %d (b200_geometry_init)", g->chroma, in->chroma);
  if (g->detour) {
    // 4:4:4 conversion point of the reference (see b200_geometry)
    // (a limited-range picture is also range-converted there: the conversion's target profile is full range)
    if (!in->full_range && (mc == 0 || mc == 8 || mc == 16))
      return set_error(B200_E_UNSUPPORTED, "limited-range picture with matrix_coefficients %d at the 4:4:4 conversion point", mc);
    return convert_via_444(in, g, opt, out, out_g, out_b, out_stride, stream, pipeline, !in->full_range, scale_w, scale_h);
  }
  if (opt->chroma_upsampling == 1 && in->chroma == B200_CHROMA_420) {
    // heif_color_conversion_options.only_use_preferred_chroma_algorithm with bilinear upsampling: the reference runs
    // Op_YCbCr420_bilinear_to_YCbCr444 first and converts from 4:4:4 with the generic float op.  Geometry happens on the
    // planes BEFORE the colour conversion in the reference, so the bilinear op sees the transformed 4:2:0 picture: all of
    // the chain is `pre`, nothing is left after the upsampling
    b200_geometry t = *g; t.detour = 1;
    for (int i = 0; i < 6; i++) t.pre[i] = g->m[i];
    t.pre_w = g->out_w; t.pre_h = g->out_h;
    t.m[0] = 1; t.m[1] = 0; t.m[2] = 0; t.m[3] = 0; t.m[4] = 1; t.m[5] = 0;
    return convert_via_444(in, &t, opt, out, out_g, out_b, out_stride, stream, pipeline, false, scale_w, scale_h);
  }
  K6Args a{};
  a.y = in->y; a.cb = in->cb; a.cr = in->cr; a.a = in->alpha;
  a.ys = (long long)in->y_stride; a.cs = (long long)in->c_stride; a.as = (long long)in->alpha_stride;
  a.out[0] = out; a.out[1] = out_g; a.out[2] = out_b; a.os = (long long)out_stride;
  a.src_w = in->width; a.src_h = in->height; a.out_w = g->out_w; a.out_h = g->out_h;
  for (int i = 0; i < 6; i++) a.m[i] = g->m[i];
  switch (in->chroma) {
    case B200_CHROMA_MONO: a.sh = a.sv = -1; break;
    case B200_CHROMA_420: a.sh = 1; a.sv = 1; break;
    case B200_CHROMA_422: a.sh = 1; a.sv = 0; break;
    case B200_CHROMA_444: a.sh = 0; a.sv = 0; break;
    default: return set_error(B200_E_INVALID, "input chroma %d", in->chroma);
  }
  a.bpp = in->bit_depth; a.full_range = in->full_range ? 1 : 0;
  ycbcr_to_rgb_coefficients(mc, in->colour_primaries, a.cf);
  for (int i = 0; i < 4; i++) a.ci[i] = (int)lroundf(256 * a.cf[i]);      // yuv2rgb.cc:377-380
  a.out_fmt = fmt;
  const bool want_alpha = fmt == B200_CHROMA_INTERLEAVED_RGBA || fmt == B200_CHROMA_INTERLEAVED_RRGGBBAA_BE || fmt == B200_CHROMA_INTERLEAVED_RRGGBBAA_LE;
  const bool has_alpha = in->alpha != nullptr && want_alpha;
  int pipe = 0;
  // integer fast path: 4:2:0, 8 bit, full range, interleaved 8-bit target (yuv2rgb.cc:300-340, :440-478)
  // matrix_coefficients 0 / 8: the dedicated 4:2:0 ops are not selected (the generic op with its special branch runs);
  // 16: they are, and convert with the default coefficients (they have no YCgCo-Re branch) -- planner behaviour pinned in
  // tests/test_color_oracle.py: test_special_matrices_match_reference
  const bool dedicated_ok = !(mc == 0 || mc == 8);
  a.int_mode = (in->chroma == B200_CHROMA_420 && in->bit_depth == 8 && in->full_range && interleaved8 && dedicated_ok) ? 1 : 0;
  pipe |= a.int_mode ? B200_PIPE_INT420 : B200_PIPE_FLOAT;
  a.sdr_shift = 0; a.pre_shift = 0;
  a.out_bytes = in->bit_depth > 8 ? 2 : 1;
  if (in->bit_depth > 8 && interleaved8) {
    a.out_bytes = 1; pipe |= B200_PIPE_SDR_SHIFT;
    if (in->chroma == B200_CHROMA_420 && in->full_range && dedicated_ok) {
      // the reference planner shifts the YCbCr planes to 8 bit first and then takes the integer op
      a.pre_shift = in->bit_depth - 8; a.int_mode = 1; a.bpp = 8; pipe = B200_PIPE_SDR_SHIFT | B200_PIPE_INT420;
    } else a.sdr_shift = in->bit_depth - 8;
  }
  const bool rrggbb_direct = in->chroma == B200_CHROMA_420 && in->bit_depth > 8 && interleaved16 && dedicated_ok;     // Op_YCbCr420_to_RRGGBBaa
  a.special = 0;
  if (in->chroma != B200_CHROMA_MONO && (mc == 0 || mc == 8 || mc == 16) && !a.int_mode && !rrggbb_direct) a.special = mc == 0 ? 1 : (mc == 8 ? 2 : 3);
  a.alpha_fill = a.out_bytes == 1 ? 0xFF : (1 << in->bit_depth) - 1;
  if (fmt == B200_CHROMA_444 && (!out_g || !out_b)) return set_error(B200_E_INVALID, "planar output needs three planes");
  if (pipeline) *pipeline = pipe;
  if (g->out_w <= 0 || g->out_h <= 0) return B200_OK;
  // a scale to the geometry's own size is the unscaled conversion
  const bool scaled = scale_w > 0 && scale_h > 0 && (scale_w != g->out_w || scale_h != g->out_h);
  if (scaled) {
    a.dst_w = scale_w; a.dst_h = scale_h;
    const dim3 sgrid((scale_w + TILE - 1) / TILE, (scale_h + TILE - 1) / TILE);
    if (in->bit_depth == 8) {
      if (has_alpha) k6_scaled_kernel<uint8_t, true><<<sgrid, 256, 0, stream>>>(a);
      else k6_scaled_kernel<uint8_t, false><<<sgrid, 256, 0, stream>>>(a);
    } else {
      if (has_alpha) k6_scaled_kernel<uint16_t, true><<<sgrid, 256, 0, stream>>>(a);
      else k6_scaled_kernel<uint16_t, false><<<sgrid, 256, 0, stream>>>(a);
    }
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(B200_E_CUDA, "k6 scaled launch: %s", cudaGetErrorString(e));
    return B200_OK;
  }
  // fast path: identity geometry, 4:2:0, no alpha, everything 16-byte aligned (the grid / single-image decode case)
  const bool identity = is_identity(g->m, g->out_w, g->out_h, in->width, in->height);
  const uintptr_t al = (uintptr_t)in->y | (uintptr_t)in->cb | (uintptr_t)in->cr | (uintptr_t)out | (uintptr_t)in->y_stride | (uintptr_t)in->c_stride | (uintptr_t)out_stride;
  if (identity && in->chroma == B200_CHROMA_420 && !has_alpha && !a.special && (al & 15) == 0 && in->width % 16 == 0 && in->height % 2 == 0 && fmt != B200_CHROMA_444 && !(a.sdr_shift && a.out_bytes == 2)) {
    bool done;
    if (in->bit_depth == 8) done = a.int_mode ? launch_direct<uint8_t, 1>(a, stream) : launch_direct<uint8_t, 0>(a, stream);
    else done = a.int_mode ? launch_direct<uint16_t, 1>(a, stream) : launch_direct<uint16_t, 0>(a, stream);
    if (done) {
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return set_error(B200_E_CUDA, "k6 direct launch: %s", cudaGetErrorString(e));
      return B200_OK;
    }
  }
  dim3 grid((g->out_w + TILE - 1) / TILE, (g->out_h + TILE - 1) / TILE);
  if (in->bit_depth == 8) {
    if (has_alpha) k6_color_kernel<uint8_t, true><<<grid, 256, 0, stream>>>(a);
    else k6_color_kernel<uint8_t, false><<<grid, 256, 0, stream>>>(a);
  } else {
    if (has_alpha) k6_color_kernel<uint16_t, true><<<grid, 256, 0, stream>>>(a);
    else k6_color_kernel<uint16_t, false><<<grid, 256, 0, stream>>>(a);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "k6 launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Encoder-side colour op: interleaved RGB / RGBA 8 bit -> planar YCbCr 4:2:0 / 4:2:2 / 4:4:4 8 bit
// (Op_RGB24_32_to_YCbCr, rgb2yuv.cc:575-808: float arithmetic in the reference's order, chroma of 4:2:0 from the integer
// mean of the 2x2 RGB quad -- 2x1 / 1x2 / 1x1 on an odd right column / bottom row --, chroma of 4:2:2 from the left pixel).
// One thread converts a 4 x 2 pixel block: 12 / 16 bytes per row in (vector loads when the rows are aligned), 4 luma bytes
// per row and 2..4 chroma bytes per plane out.  HBM bound: 3 or 4 bytes read, 1.5 .. 4 bytes written per pixel.
// ---------------------------------------------------------------------------------------------------------------
struct RgbToYccArgs {
  const uint8_t* in; long long in_stride;
  uint8_t *y, *cb, *cr, *a; long long ys, cs, as;
  int w, h, chroma, full, vec_in, vec_out;
  float c[3][3];
};
__device__ __forceinline__ int clip_round(float v, int maxv) {
  const int x = __float2int_rz(__fadd_rn(v, 0.5f));
  return x < 0 ? 0 : (x > maxv ? maxv : x);
}
__device__ __forceinline__ float dot3(int r, int g, int b, const float* c) {
  return __fadd_rn(__fadd_rn(__fmul_rn((float)r, c[0]), __fmul_rn((float)g, c[1])), __fmul_rn((float)b, c[2]));
}
// the per-pixel / per-quad arithmetic of Op_RGB24_32_to_YCbCr, shared by rgb_to_ycbcr_kernel and rgb_to_ycbcr_grid_kernel
__device__ __forceinline__ uint8_t luma_24_32(const float (&c)[3][3], int full, int r, int g, int b) {
  const float f = dot3(r, g, b, c[0]);
  return full ? (uint8_t)clip_round(f, 255) : (uint8_t)(clip_round(__fmul_rn(f, 0.85547f), 219) + 16);
}
__device__ __forceinline__ void put_chroma(const float (&c)[3][3], int full, int r, int g, int b, uint8_t* ocb, uint8_t* ocr) {
  const float cb = dot3(r, g, b, c[1]), cr = dot3(r, g, b, c[2]);
  if (full) { *ocb = (uint8_t)clip_round(__fadd_rn(cb, 128.0f), 255); *ocr = (uint8_t)clip_round(__fadd_rn(cr, 128.0f), 255); }
  else {
    *ocb = (uint8_t)clip_round(__fadd_rn(__fmul_rn(cb, 0.875f), 128.0f), 255);
    *ocr = (uint8_t)clip_round(__fadd_rn(__fmul_rn(cr, 0.875f), 128.0f), 255);
  }
}
// 4:2:0 chroma from the integer mean of the n (4, or 2 / 1 on an odd right column / bottom row) samples summed in s
__device__ __forceinline__ void quad_chroma_24_32(const float (&c)[3][3], int full, const int s[3], int n, uint8_t* ocb, uint8_t* ocr) {
  put_chroma(c, full, s[0] / n, s[1] / n, s[2] / n, ocb, ocr);
}
__device__ __forceinline__ void store_bytes(uint8_t* dst, const uint8_t* v, int n, bool vec) {
  if (vec && n == 4) *(uint32_t*)dst = (uint32_t)v[0] | ((uint32_t)v[1] << 8) | ((uint32_t)v[2] << 16) | ((uint32_t)v[3] << 24);
  else if (vec && n == 2) *(uint16_t*)dst = (uint16_t)((unsigned)v[0] | ((unsigned)v[1] << 8));
  else for (int i = 0; i < n; i++) dst[i] = v[i];
}
template <int BPP>
__global__ void __launch_bounds__(256) rgb_to_ycbcr_kernel(const RgbToYccArgs p) {
  const int x0 = (blockIdx.x * 64 + threadIdx.x) * 4, y0 = (blockIdx.y * 4 + threadIdx.y) * 2;
  if (x0 >= p.w || y0 >= p.h) return;
  const int nx = min(4, p.w - x0), ny = min(2, p.h - y0);
  uint8_t px[2][4][4];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    if (j >= ny) break;
    const uint8_t* row = p.in + (long long)(y0 + j) * p.in_stride + (long long)x0 * BPP;
    if (p.vec_in && nx == 4) {
      if (BPP == 4) {
        const uint4 v = __ldg((const uint4*)row);
        const uint32_t q[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; i++) { px[j][i][0] = q[i] & 255; px[j][i][1] = (q[i] >> 8) & 255; px[j][i][2] = (q[i] >> 16) & 255; px[j][i][3] = q[i] >> 24; }
      } else {
        const uint32_t a = __ldg((const uint32_t*)row), b = __ldg((const uint32_t*)row + 1), c = __ldg((const uint32_t*)row + 2);
        px[j][0][0] = a & 255; px[j][0][1] = (a >> 8) & 255; px[j][0][2] = (a >> 16) & 255;
        px[j][1][0] = a >> 24; px[j][1][1] = b & 255; px[j][1][2] = (b >> 8) & 255;
        px[j][2][0] = (b >> 16) & 255; px[j][2][1] = b >> 24; px[j][2][2] = c & 255;
        px[j][3][0] = (c >> 8) & 255; px[j][3][1] = (c >> 16) & 255; px[j][3][2] = c >> 24;
      }
    } else {
#pragma unroll
      for (int i = 0; i < 4; i++) {
        if (i >= nx) break;
#pragma unroll
        for (int k = 0; k < BPP; k++) px[j][i][k] = __ldg(row + i * BPP + k);
      }
    }
  }
  const bool vo = p.vec_out != 0;
  // luma (rgb2yuv.cc:640-665) and alpha (:667-691: copied, or 0xff when the source has none)
#pragma unroll
  for (int j = 0; j < 2; j++) {
    if (j >= ny) break;
    uint8_t yv[4], av[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      if (i >= nx) break;
      yv[i] = luma_24_32(p.c, p.full, px[j][i][0], px[j][i][1], px[j][i][2]);
      av[i] = BPP == 4 ? px[j][i][3] : 0xff;
    }
    store_bytes(p.y + (long long)(y0 + j) * p.ys + x0, yv, nx, vo);
    if (p.a) store_bytes(p.a + (long long)(y0 + j) * p.as + x0, av, nx, vo);
  }
  if (p.chroma == B200_CHROMA_444) {
#pragma unroll
    for (int j = 0; j < 2; j++) {
      if (j >= ny) break;
      uint8_t vb[4], vr[4];
#pragma unroll
      for (int i = 0; i < 4; i++) { if (i >= nx) break; put_chroma(p.c, p.full, px[j][i][0], px[j][i][1], px[j][i][2], &vb[i], &vr[i]); }
      store_bytes(p.cb + (long long)(y0 + j) * p.cs + x0, vb, nx, vo);
      store_bytes(p.cr + (long long)(y0 + j) * p.cs + x0, vr, nx, vo);
    }
  } else if (p.chroma == B200_CHROMA_422) {
    const int nc = (nx + 1) >> 1;
#pragma unroll
    for (int j = 0; j < 2; j++) {
      if (j >= ny) break;
      uint8_t vb[2], vr[2];
#pragma unroll
      for (int i = 0; i < 2; i++) { if (i >= nc) break; put_chroma(p.c, p.full, px[j][2 * i][0], px[j][2 * i][1], px[j][2 * i][2], &vb[i], &vr[i]); }
      store_bytes(p.cb + (long long)(y0 + j) * p.cs + (x0 >> 1), vb, nc, vo);
      store_bytes(p.cr + (long long)(y0 + j) * p.cs + (x0 >> 1), vr, nc, vo);
    }
  } else {
    const int nc = (nx + 1) >> 1;
    uint8_t vb[2], vr[2];
#pragma unroll
    for (int i = 0; i < 2; i++) {
      if (i >= nc) break;
      const int qx = (2 * i + 1 < nx) ? 2 : 1, n = qx * ny;
      int s[3];
#pragma unroll
      for (int k = 0; k < 3; k++) {
        int t = px[0][2 * i][k];
        if (qx == 2) t += px[0][2 * i + 1][k];
        if (ny == 2) { t += px[1][2 * i][k]; if (qx == 2) t += px[1][2 * i + 1][k]; }
        s[k] = t;
      }
      quad_chroma_24_32(p.c, p.full, s, n, &vb[i], &vr[i]);
    }
    store_bytes(p.cb + (long long)(y0 >> 1) * p.cs + (x0 >> 1), vb, nc, vo);
    store_bytes(p.cr + (long long)(y0 >> 1) * p.cs + (x0 >> 1), vr, nc, vo);
  }
}

int launch_rgb_to_ycbcr(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out, cudaStream_t stream) {
  if (!rgb || !out || !out->y) return set_error(B200_E_INVALID, "null argument");
  if (out->bit_depth != 8) return set_error(B200_E_UNSUPPORTED, "RGB -> YCbCr: %d-bit target (the 8-bit interleaved op only)", out->bit_depth);
  if (out->chroma != B200_CHROMA_420 && out->chroma != B200_CHROMA_422 && out->chroma != B200_CHROMA_444)
    return set_error(B200_E_UNSUPPORTED, "RGB -> YCbCr: target chroma %d", out->chroma);
  if (!out->cb || !out->cr) return set_error(B200_E_INVALID, "RGB -> YCbCr: chroma planes missing");
  int mc = out->matrix_coefficients, cp = out->colour_primaries;
  if (mc == 0 || mc == 8 || mc == 11 || mc == 14)
    return set_error(B200_E_UNSUPPORTED, "matrix_coefficients %d: not converted by this operation in the reference either (rgb2yuv.cc:536-539)", mc);
  if (mc == 2) mc = 6;              // unspecified -> sRGB defaults, as convert_colorspace() does with the target profile
  if (cp == 2) cp = 1;              // (nclx.cc:360-373 through colorconversion.cc:513-515)
  if (out->width <= 0 || out->height <= 0) return B200_OK;
  const int bpp = has_alpha ? 4 : 3;
  if (rgb_stride < (size_t)out->width * bpp) return set_error(B200_E_INVALID, "RGB stride %zu < row of %d pixels", rgb_stride, out->width);
  RgbToYccArgs a;
  a.in = (const uint8_t*)rgb; a.in_stride = (long long)rgb_stride;
  a.y = (uint8_t*)out->y; a.cb = (uint8_t*)out->cb; a.cr = (uint8_t*)out->cr; a.a = (uint8_t*)out->alpha;
  a.ys = (long long)out->y_stride; a.cs = (long long)out->c_stride; a.as = (long long)out->alpha_stride;
  a.w = out->width; a.h = out->height; a.chroma = out->chroma; a.full = out->full_range ? 1 : 0;
  rgb_to_ycbcr_coefficients(mc, cp, a.c);
  const uintptr_t ai = (uintptr_t)rgb | (uintptr_t)rgb_stride;
  a.vec_in = (ai & (has_alpha ? 15 : 3)) == 0;
  uintptr_t ao = (uintptr_t)out->y | (uintptr_t)out->cb | (uintptr_t)out->cr | (uintptr_t)out->y_stride | (uintptr_t)out->c_stride;
  if (out->alpha) ao |= (uintptr_t)out->alpha | (uintptr_t)out->alpha_stride;
  a.vec_out = (ao & 3) == 0;
  const dim3 block(64, 4), grid((a.w + 255) / 256, (a.h + 7) / 8);
  if (has_alpha) rgb_to_ycbcr_kernel<4><<<grid, block, 0, stream>>>(a);
  else rgb_to_ycbcr_kernel<3><<<grid, block, 0, stream>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "RGB -> YCbCr launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

// ---------------------------------------------------------------------------------------------------------------
// Encoder-side colour ops for the other RGB layouts: one kernel, templated on the sample type T (uint8 / uint16, the same
// for input and output, as the reference ops keep the depth), the loader (interleaved RGB[A] 8 bit / RRGGBB[AA] BE or LE,
// or planar R, G, B[, A]) and the arithmetic of one reference op:
//   YCC_HDR420  Op_RRGGBBxx_HDR_to_YCbCr420   rgb2yuv.cc:366-503  (full range, 4:2:0 only)
//   YCC_PLANAR  Op_RGB_to_YCbCr<T>            rgb2yuv.cc:100-305  (behind the lossless Op_RRGGBBaa_swap_endianness /
//               Op_RRGGBBaa_BE_to_RGB_HDR / Op_RGB24_32_to_RGB steps of the chain, which the loader folds in)
//   YCC_GBR444  Op_RGB24_32_to_YCbCr444_GBR   rgb2yuv.cc:850-919
// Every chroma value of these ops is a float sum of whole samples (exact in float) times 0.25, or one sample, so one thread
// converts a 2 x 2 pixel block and computes its chroma from the block: pairs of samples come in as 16- / 32-bit loads
// (interleaved 16 bit: 12- or 16-byte loads) and luma / alpha leave as pairs when the rows are aligned.
// ---------------------------------------------------------------------------------------------------------------
enum { YCC_HDR420 = 0, YCC_PLANAR = 1, YCC_GBR444 = 2 };
struct RgbExArgs {
  const uint8_t* in[4]; long long is[4];       // interleaved: in[0]; planar: R, G, B, A
  uint8_t *y, *cb, *cr, *a; long long ys, cs, as;
  int w, h, sh, sv, nch, le, full, bpp, mc, vec_in, vec_out;
  float c[3][3];
};

template <typename T, bool PLANAR_IN>
__device__ __forceinline__ void load_pair(const RgbExArgs& p, int x0, int y, int n, int v[2][4]) {
  if (PLANAR_IN) {
#pragma unroll
    for (int c = 0; c < 4; c++) {
      if (c == 3 && !p.a) break;
      const T* row = reinterpret_cast<const T*>(p.in[c] + (long long)y * p.is[c]) + x0;
      if (p.vec_in && n == 2) {
        if (sizeof(T) == 1) { const unsigned q = __ldg(reinterpret_cast<const unsigned short*>(row)); v[0][c] = q & 0xff; v[1][c] = q >> 8; }
        else { const unsigned q = __ldg(reinterpret_cast<const unsigned*>(row)); v[0][c] = q & 0xffff; v[1][c] = q >> 16; }
      } else {
        v[0][c] = __ldg(row);
        if (n == 2) v[1][c] = __ldg(row + 1);
      }
    }
    return;
  }
  // the (up to) 16 bytes of the pair in four registers; bytes are picked with selects, not an indexed local array
  const int bpp = p.nch * (int)sizeof(T);
  const uint8_t* row = p.in[0] + (long long)y * p.is[0] + (long long)x0 * bpp;
  unsigned wd[4] = {0, 0, 0, 0};
  if (sizeof(T) == 2 && p.vec_in && n == 2) {
    if (p.nch == 4) { const uint4 q = __ldg(reinterpret_cast<const uint4*>(row)); wd[0] = q.x; wd[1] = q.y; wd[2] = q.z; wd[3] = q.w; }
    else {
#pragma unroll
      for (int k = 0; k < 3; k++) wd[k] = __ldg(reinterpret_cast<const unsigned*>(row) + k);
    }
  } else {
#pragma unroll
    for (int k = 0; k < 16; k++) if (k < n * bpp) wd[k >> 2] |= (unsigned)__ldg(row + k) << ((k & 3) * 8);
  }
  auto byte_at = [&](int k) -> int {
    const unsigned w = k < 4 ? wd[0] : (k < 8 ? wd[1] : (k < 12 ? wd[2] : wd[3]));
    return (w >> ((k & 3) * 8)) & 0xff;
  };
#pragma unroll
  for (int i = 0; i < 2; i++) {
    if (i >= n) break;
#pragma unroll
    for (int c = 0; c < 4; c++) {
      if (c >= p.nch) break;
      const int k = i * bpp + c * (int)sizeof(T);
      v[i][c] = sizeof(T) == 1 ? byte_at(k) : ((byte_at(k + p.le) << 8) | byte_at(k + 1 - p.le));   // rgb2yuv.cc:443-445, rgb2rgb.cc:464-
    }
  }
}

__device__ __forceinline__ float dot3f(float r, float g, float b, const float* c) {
  return __fadd_rn(__fadd_rn(__fmul_rn(r, c[0]), __fmul_rn(g, c[1])), __fmul_rn(b, c[2]));
}
__device__ __forceinline__ float scale_256(float v, float f) { return __fdiv_rn(__fmul_rn(v, f), 256.0f); }   // (v * f) / 256

template <int ARITH>
__device__ __forceinline__ int luma_ex(const RgbExArgs& p, int r, int g, int b) {
  const int maxv = (1 << p.bpp) - 1;
  if (ARITH == YCC_GBR444) return g;
  if (ARITH == YCC_PLANAR && p.mc == 0) {                                     // rgb2yuv.cc:198-206
    if (p.full) return g;
    return clip_round(__fadd_rn(scale_256((float)g, 219.0f), (float)(16 << (p.bpp - 8))), maxv);
  }
  if (ARITH == YCC_PLANAR && p.mc == 8) return g / 2 + (r + b) / 4;            // :207-211
  float v = dot3f((float)r, (float)g, (float)b, p.c[0]);                      // :213-222, :443-453
  if (ARITH == YCC_PLANAR && !p.full) v = __fadd_rn(scale_256(v, 219.0f), (float)(16 << (p.bpp - 8)));
  return clip_round(v, maxv);
}

// s: the sample (GBR / matrix 0 / 8: the block's top-left pixel) or, for the matrix ops, the sum of the four quad samples
template <int ARITH>
__device__ __forceinline__ void chroma_ex(const RgbExArgs& p, const int s[3], bool sum4, int& cb, int& cr) {
  const int maxv = (1 << p.bpp) - 1, half = 1 << (p.bpp - 1);
  const int r = s[0], g = s[1], b = s[2];
  if (ARITH == YCC_GBR444 || (ARITH == YCC_PLANAR && p.mc == 0 && p.full)) { cb = b; cr = r; return; }
  if (ARITH == YCC_PLANAR && p.mc == 0) {                                                   // rgb2yuv.cc:237-240
    const float off = (float)(16 << (p.bpp - 8));
    cb = clip_round(__fadd_rn(scale_256((float)b, 224.0f), off), maxv);
    cr = clip_round(__fadd_rn(scale_256((float)r, 224.0f), off), maxv);
    return;
  }
  if (ARITH == YCC_PLANAR && p.mc == 8) {                                                   // :246-250 (C division)
    const int u = g / 2 - (r + b) / 4 + half, w = (r - b) / 2 + half;
    cb = u < 0 ? 0 : (u > maxv ? maxv : u); cr = w < 0 ? 0 : (w > maxv ? maxv : w);
    return;
  }
  float rf = (float)r, gf = (float)g, bf = (float)b;
  if (sum4) { rf = __fmul_rn(rf, 0.25f); gf = __fmul_rn(gf, 0.25f); bf = __fmul_rn(bf, 0.25f); }     // :273-275, :485-487
  float u = dot3f(rf, gf, bf, p.c[1]), w = dot3f(rf, gf, bf, p.c[2]);
  if (ARITH == YCC_PLANAR && !p.full) { u = scale_256(u, 224.0f); w = scale_256(w, 224.0f); }      // :283-286
  cb = clip_round(__fadd_rn(u, (float)half), maxv);
  cr = clip_round(__fadd_rn(w, (float)half), maxv);
}

// 4:2:0 chroma of the quad v[row][column] (nx x ny samples of it present, the others repeat the edge), shared by
// rgb_to_ycbcr_ex_kernel and rgb_to_ycbcr_grid_kernel
template <int ARITH>
__device__ __forceinline__ void quad_chroma_ex(const RgbExArgs& p, const int (&v)[2][2][4], int nx, int ny, int& cb, int& cr) {
  const bool special = ARITH == YCC_PLANAR && (p.mc == 0 || p.mc == 8);
  int s[3];
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const int a00 = v[0][0][c], a01 = nx == 2 ? v[0][1][c] : a00, a10 = ny == 2 ? v[1][0][c] : a00, a11 = ny == 2 ? (nx == 2 ? v[1][1][c] : a10) : a01;
    s[c] = special ? a00 : a00 + a01 + a10 + a11;
  }
  chroma_ex<ARITH>(p, s, !special, cb, cr);
}

template <typename T>
__device__ __forceinline__ void store_pair(uint8_t* plane, long long stride, int x0, int y, int n, int v0, int v1, bool vec) {
  T* row = reinterpret_cast<T*>(plane + (long long)y * stride) + x0;
  if (vec && n == 2) {
    if (sizeof(T) == 1) *reinterpret_cast<unsigned short*>(row) = (unsigned short)(v0 | (v1 << 8));
    else *reinterpret_cast<unsigned*>(row) = (unsigned)v0 | ((unsigned)v1 << 16);
  } else {
    row[0] = (T)v0;
    if (n == 2) row[1] = (T)v1;
  }
}

template <typename T, bool PLANAR_IN, int ARITH>
__global__ void __launch_bounds__(256) rgb_to_ycbcr_ex_kernel(const RgbExArgs p) {
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 2, y0 = (blockIdx.y * blockDim.y + threadIdx.y) * 2;
  if (x0 >= p.w || y0 >= p.h) return;
  const int nx = min(2, p.w - x0), ny = min(2, p.h - y0);
  int v[2][2][4];
#pragma unroll
  for (int j = 0; j < 2; j++) {
    if (j < ny) load_pair<T, PLANAR_IN>(p, x0, y0 + j, nx, v[j]);
  }
  const bool vo = p.vec_out != 0;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    if (j >= ny) break;
    int l[2] = {0, 0};
#pragma unroll
    for (int i = 0; i < 2; i++) if (i < nx) l[i] = luma_ex<ARITH>(p, v[j][i][0], v[j][i][1], v[j][i][2]);
    store_pair<T>(p.y, p.ys, x0, y0 + j, nx, l[0], l[1], vo);
    if (p.a) store_pair<T>(p.a, p.as, x0, y0 + j, nx, v[j][0][3], nx == 2 ? v[j][1][3] : 0, vo);   // alpha copied (:295-302, :455-458)
  }
  int cb, cr;
  if (p.sh == 0) {                                                                // 4:4:4: every pixel
#pragma unroll
    for (int j = 0; j < 2; j++) {
      if (j >= ny) break;
      int b2[2] = {0, 0}, r2[2] = {0, 0};
#pragma unroll
      for (int i = 0; i < 2; i++) if (i < nx) { chroma_ex<ARITH>(p, v[j][i], false, b2[i], r2[i]); }
      store_pair<T>(p.cb, p.cs, x0, y0 + j, nx, b2[0], b2[1], vo);
      store_pair<T>(p.cr, p.cs, x0, y0 + j, nx, r2[0], r2[1], vo);
    }
  } else if (p.sv == 0) {
    // 4:2:2: x2 = x and y2 = y (rgb2yuv.cc:258-259), so the float "mean" is 4 x the left pixel x 0.25 = the left pixel, exactly
#pragma unroll
    for (int j = 0; j < 2; j++) {
      if (j >= ny) break;
      chroma_ex<ARITH>(p, v[j][0], false, cb, cr);
      reinterpret_cast<T*>(p.cb + (long long)(y0 + j) * p.cs)[x0 >> 1] = (T)cb;
      reinterpret_cast<T*>(p.cr + (long long)(y0 + j) * p.cs)[x0 >> 1] = (T)cr;
    }
  } else {
    quad_chroma_ex<ARITH>(p, v, nx, ny, cb, cr);
    reinterpret_cast<T*>(p.cb + (long long)(y0 >> 1) * p.cs)[x0 >> 1] = (T)cb;
    reinterpret_cast<T*>(p.cr + (long long)(y0 >> 1) * p.cs)[x0 >> 1] = (T)cr;
  }
}

static bool rgb_interleaved(int chroma) { return chroma >= B200_CHROMA_INTERLEAVED_RGB && chroma <= B200_CHROMA_INTERLEAVED_RRGGBBAA_LE; }
static bool rgb_has_alpha(const b200_rgb_image* in) {
  return in->chroma == B200_CHROMA_INTERLEAVED_RGBA || in->chroma == B200_CHROMA_INTERLEAVED_RRGGBBAA_BE ||
         in->chroma == B200_CHROMA_INTERLEAVED_RRGGBBAA_LE || (in->chroma == B200_CHROMA_444 && in->alpha != nullptr);
}

// The chain the reference planner (colorconversion.cc:279-435) finds from this RGB input to `out`'s YCbCr state at the input
// depth, with convert_colorspace's target (colorconversion.cc:530-611); tabulated from its operations' state_after_conversion
// (rgb2yuv.cc:30-98, :311-363, :506-553, :812-847, rgb2rgb.cc) and pinned by tests/test_rgb_to_ycbcr_ex_plan.py.
int plan_rgb_to_ycbcr(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline) {
  if (pipeline) *pipeline = 0;
  if (!in || !out) return set_error(B200_E_INVALID, "null argument");
  const int ic = in->chroma, bd = in->bit_depth;
  const bool inter = rgb_interleaved(ic), inter8 = ic == B200_CHROMA_INTERLEAVED_RGB || ic == B200_CHROMA_INTERLEAVED_RGBA;
  if (!inter && ic != B200_CHROMA_444) return set_error(B200_E_INVALID, "RGB input chroma %d", ic);
  if (inter8 ? bd != 8 : (bd < (inter ? 9 : 8) || bd > 16)) return set_error(B200_E_INVALID, "RGB input chroma %d with bit depth %d", ic, bd);
  if (out->chroma != B200_CHROMA_420 && out->chroma != B200_CHROMA_422 && out->chroma != B200_CHROMA_444)
    return set_error(B200_E_UNSUPPORTED, "RGB -> YCbCr: target chroma %d", out->chroma);
  if (out->bit_depth != bd) return set_error(B200_E_INVALID, "target bit depth %d: the conversion keeps the input's %d", out->bit_depth, bd);
  if (out->width != in->width || out->height != in->height) return set_error(B200_E_INVALID, "target size differs from the input's");
  const int mc = out->matrix_coefficients;
  if (mc == 11 || mc == 14) return set_error(B200_E_UNSUPPORTED, "matrix_coefficients %d: no RGB -> YCbCr operation of the reference takes it (rgb2yuv.cc:57-60)", mc);
  if (ic == B200_CHROMA_444 && in->alpha && in->alpha_bit_depth && in->alpha_bit_depth != bd)
    return set_error(B200_E_UNSUPPORTED, "alpha depth %d differs from the colour depth %d (the reference inserts Op_adjust_alpha_bit_depth)", in->alpha_bit_depth, bd);
  const int ds = opt ? opt->chroma_downsampling : 2;
  if (out->chroma != B200_CHROMA_444 && opt && opt->only_use_preferred && ds != 1)
    return set_error(B200_E_UNSUPPORTED, "only_use_preferred_chroma_algorithm with downsampling %d: the reference converts to 4:4:4 and "
                                         "downsamples with a separate operation (or has no chain)", ds);
  const bool full = out->full_range != 0, special = mc == 0 || mc == 8;
  int pipe;
  if (inter8) pipe = !special ? B200_YCC_PIPE_RGB24_32 : (mc == 0 && full && out->chroma == B200_CHROMA_444) ? B200_YCC_PIPE_GBR444 : B200_YCC_PIPE_UNPACK | B200_YCC_PIPE_PLANAR;
  else if (inter) {
    const bool le = ic == B200_CHROMA_INTERLEAVED_RRGGBB_LE || ic == B200_CHROMA_INTERLEAVED_RRGGBBAA_LE;
    pipe = (full && out->chroma == B200_CHROMA_420 && !special) ? B200_YCC_PIPE_HDR420 : (le ? B200_YCC_PIPE_SWAP : 0) | B200_YCC_PIPE_UNPACK | B200_YCC_PIPE_PLANAR;
  } else pipe = B200_YCC_PIPE_PLANAR;
  if (pipeline) *pipeline = pipe;
  return B200_OK;
}

// the kernel arguments of rgb_to_ycbcr_ex_kernel / rgb_to_ycbcr_grid_kernel: input planes (strides checked against the input's
// width), output planes and size, vector-access flags, matrix and coefficients
static int ex_args(const b200_rgb_image* in, const b200_planes* out, bool has_alpha, RgbExArgs& a) {
  const bool inter = rgb_interleaved(in->chroma);
  const int bps = in->bit_depth > 8 ? 2 : 1;
  a.nch = inter ? (has_alpha ? 4 : 3) : 1;
  uintptr_t ai = 0;
  if (inter) {
    if (in->rgb_stride < (size_t)in->width * a.nch * bps) return set_error(B200_E_INVALID, "RGB stride %zu < row of %d pixels", in->rgb_stride, in->width);
    a.in[0] = (const uint8_t*)in->rgb; a.is[0] = (long long)in->rgb_stride;
    ai = (uintptr_t)in->rgb | (uintptr_t)in->rgb_stride;
    a.vec_in = bps == 2 && (ai & (a.nch == 4 ? 15 : 3)) == 0;
  } else {
    const void* pl[4] = {in->r, in->g, in->b, in->alpha};
    const size_t st[4] = {in->r_stride, in->g_stride, in->b_stride, in->alpha_stride};
    for (int c = 0; c < (has_alpha ? 4 : 3); c++) {
      if (st[c] < (size_t)in->width * bps) return set_error(B200_E_INVALID, "plane %d stride %zu < row of %d samples", c, st[c], in->width);
      a.in[c] = (const uint8_t*)pl[c]; a.is[c] = (long long)st[c]; ai |= (uintptr_t)pl[c] | (uintptr_t)st[c];
    }
    a.vec_in = (ai & (2 * bps - 1)) == 0;
  }
  a.le = in->chroma == B200_CHROMA_INTERLEAVED_RRGGBB_LE || in->chroma == B200_CHROMA_INTERLEAVED_RRGGBBAA_LE;
  a.y = (uint8_t*)out->y; a.cb = (uint8_t*)out->cb; a.cr = (uint8_t*)out->cr; a.a = (uint8_t*)out->alpha;
  a.ys = (long long)out->y_stride; a.cs = (long long)out->c_stride; a.as = (long long)out->alpha_stride;
  uintptr_t ao = (uintptr_t)out->y | (uintptr_t)out->cb | (uintptr_t)out->cr | (uintptr_t)out->y_stride | (uintptr_t)out->c_stride;
  if (out->alpha) ao |= (uintptr_t)out->alpha | (uintptr_t)out->alpha_stride;
  a.vec_out = (ao & (2 * bps - 1)) == 0;
  a.w = out->width; a.h = out->height; a.full = out->full_range ? 1 : 0; a.bpp = in->bit_depth;
  a.sh = out->chroma == B200_CHROMA_444 ? 0 : 1; a.sv = out->chroma == B200_CHROMA_420 ? 1 : 0;
  int mc = out->matrix_coefficients, cp = out->colour_primaries;
  if (mc == 2) mc = 6;              // unspecified -> the input's sRGB defaults (colorconversion.cc:513-515, :567-573)
  if (cp == 2) cp = 1;
  a.mc = mc;
  rgb_to_ycbcr_coefficients(mc, cp, a.c);
  return B200_OK;
}

int launch_rgb_to_ycbcr_ex(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, cudaStream_t stream, int* pipeline) {
  int pipe = 0;
  int rc = plan_rgb_to_ycbcr(in, out, opt, &pipe);
  if (rc) return rc;
  if (pipeline) *pipeline = pipe;
  const bool has_alpha = rgb_has_alpha(in);
  if (!out->y || !out->cb || !out->cr) return set_error(B200_E_INVALID, "RGB -> YCbCr: output planes missing");
  if (has_alpha != (out->alpha != nullptr))
    return set_error(B200_E_INVALID, "the result has an alpha plane exactly when the input has one (colorconversion.cc:575-585)");
  const bool inter = rgb_interleaved(in->chroma);
  if (inter ? !in->rgb : (!in->r || !in->g || !in->b)) return set_error(B200_E_INVALID, "RGB input planes missing");
  if (pipe == B200_YCC_PIPE_RGB24_32) return launch_rgb_to_ycbcr(in->rgb, in->rgb_stride, has_alpha, out, stream);
  if (out->width <= 0 || out->height <= 0) return B200_OK;
  RgbExArgs a{};
  if ((rc = ex_args(in, out, has_alpha, a))) return rc;
  const int bps = in->bit_depth > 8 ? 2 : 1;
  const dim3 block(64, 4), grid((a.w + 127) / 128, (a.h + 7) / 8);
  if (pipe == B200_YCC_PIPE_HDR420) rgb_to_ycbcr_ex_kernel<uint16_t, false, YCC_HDR420><<<grid, block, 0, stream>>>(a);
  else if (pipe == B200_YCC_PIPE_GBR444) rgb_to_ycbcr_ex_kernel<uint8_t, false, YCC_GBR444><<<grid, block, 0, stream>>>(a);
  else if (inter) {
    if (bps == 1) rgb_to_ycbcr_ex_kernel<uint8_t, false, YCC_PLANAR><<<grid, block, 0, stream>>>(a);
    else rgb_to_ycbcr_ex_kernel<uint16_t, false, YCC_PLANAR><<<grid, block, 0, stream>>>(a);
  } else {
    if (bps == 1) rgb_to_ycbcr_ex_kernel<uint8_t, true, YCC_PLANAR><<<grid, block, 0, stream>>>(a);
    else rgb_to_ycbcr_ex_kernel<uint16_t, true, YCC_PLANAR><<<grid, block, 0, stream>>>(a);
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "RGB -> YCbCr launch: %s", cudaGetErrorString(e));
  return B200_OK;
}


// ---------------------------------------------------------------------------------------------------------------
// Colour stage of the one-call grid encoder (b200_gpu_encode_rgb_grid_*): 8-bit RGB -> ONE padded cols * tile_w x
// rows * tile_h 4:2:0 picture (+ alpha plane) whose tile windows the GPU encoder codes in place.  Source reads are clamped to
// the picture (edge replication where the last tiles overhang it).  Tile origins are even and every output quad is complete,
// and each quad's chroma is a function of its four RGB pixels only, so the result equals converting each edge-padded tile on
// its own.  One thread per 2 x 2 quad; the loader and the per-pixel / per-quad arithmetic are the ones of
// rgb_to_ycbcr_kernel (Op_RGB24_32_to_YCbCr: OP_24_32) and rgb_to_ycbcr_ex_kernel<uint8_t, *, YCC_PLANAR> (Op_RGB_to_YCbCr).
// Launched per band of output rows [y0, y1), so that the host form converts band k while band k + 1 is uploaded.
// ---------------------------------------------------------------------------------------------------------------
struct RgbGridArgs { RgbExArgs e; int src_w, src_h, y0, y1; };

template <bool PLANAR_IN, bool OP_24_32>
__global__ void __launch_bounds__(256) rgb_to_ycbcr_grid_kernel(const RgbGridArgs g) {
  const RgbExArgs& p = g.e;
  const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * 2, y0 = g.y0 + (blockIdx.y * blockDim.y + threadIdx.y) * 2;
  if (x0 >= p.w || y0 >= g.y1) return;
  const int sx = min(x0, g.src_w - 1), n = x0 + 1 < g.src_w ? 2 : 1;
  int v[2][2][4] = {};
#pragma unroll
  for (int j = 0; j < 2; j++) {
    load_pair<uint8_t, PLANAR_IN>(p, sx, min(y0 + j, g.src_h - 1), n, v[j]);
    if (n == 1) {
#pragma unroll
      for (int c = 0; c < 4; c++) v[j][1][c] = v[j][0][c];
    }
  }
  const bool vo = p.vec_out != 0;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    int l[2];
#pragma unroll
    for (int i = 0; i < 2; i++)
      l[i] = OP_24_32 ? (int)luma_24_32(p.c, p.full, v[j][i][0], v[j][i][1], v[j][i][2]) : luma_ex<YCC_PLANAR>(p, v[j][i][0], v[j][i][1], v[j][i][2]);
    store_pair<uint8_t>(p.y, p.ys, x0, y0 + j, 2, l[0], l[1], vo);
    if (p.a) store_pair<uint8_t>(p.a, p.as, x0, y0 + j, 2, v[j][0][3], v[j][1][3], vo);
  }
  int cb, cr;
  if (OP_24_32) {
    int s[3];
#pragma unroll
    for (int c = 0; c < 3; c++) s[c] = v[0][0][c] + v[0][1][c] + v[1][0][c] + v[1][1][c];
    uint8_t b8, r8;
    quad_chroma_24_32(p.c, p.full, s, 4, &b8, &r8);
    cb = b8; cr = r8;
  } else {
    quad_chroma_ex<YCC_PLANAR>(p, v, 2, 2, cb, cr);
  }
  p.cb[(long long)(y0 >> 1) * p.cs + (x0 >> 1)] = (uint8_t)cb;
  p.cr[(long long)(y0 >> 1) * p.cs + (x0 >> 1)] = (uint8_t)cr;
}

int launch_rgb_to_ycbcr_grid(const b200_rgb_image* in, const b200_planes* out, int pipeline, int y0, int y1, cudaStream_t stream) {
  const bool has_alpha = rgb_has_alpha(in), inter = rgb_interleaved(in->chroma);
  if (in->bit_depth != 8 || out->bit_depth != 8 || out->chroma != B200_CHROMA_420 || (out->width | out->height | y0 | y1) & 1 ||
      out->width < in->width || out->height < in->height || in->width <= 0 || in->height <= 0)
    return set_error(B200_E_INVALID, "grid colour stage: 8-bit RGB into an even-sized 4:2:0 picture at least as large");
  if (pipeline != B200_YCC_PIPE_RGB24_32 && pipeline != B200_YCC_PIPE_PLANAR && pipeline != (B200_YCC_PIPE_UNPACK | B200_YCC_PIPE_PLANAR))
    return set_error(B200_E_UNSUPPORTED, "grid colour stage: chain %d", pipeline);
  if (!out->y || !out->cb || !out->cr || has_alpha != (out->alpha != nullptr)) return set_error(B200_E_INVALID, "grid colour stage: output planes");
  if (inter ? !in->rgb : (!in->r || !in->g || !in->b)) return set_error(B200_E_INVALID, "RGB input planes missing");
  RgbGridArgs g{};
  if (int rc = ex_args(in, out, has_alpha, g.e)) return rc;
  g.src_w = in->width; g.src_h = in->height;
  const dim3 block(64, 4);
  for (int c0 = y0; c0 < y1; c0 += 65535 * 8) {                   // grid.y <= 65535
    g.y0 = c0; g.y1 = std::min(y1, c0 + 65535 * 8);
    const dim3 grid((out->width / 2 + 63) / 64, ((g.y1 - g.y0) / 2 + 3) / 4);
    if (pipeline == B200_YCC_PIPE_RGB24_32) rgb_to_ycbcr_grid_kernel<false, true><<<grid, block, 0, stream>>>(g);
    else if (inter) rgb_to_ycbcr_grid_kernel<false, false><<<grid, block, 0, stream>>>(g);
    else rgb_to_ycbcr_grid_kernel<true, false><<<grid, block, 0, stream>>>(g);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(B200_E_CUDA, "grid colour stage launch: %s", cudaGetErrorString(e));
  }
  return B200_OK;
}

}  // namespace b200
