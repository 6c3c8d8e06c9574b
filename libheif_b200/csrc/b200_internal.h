// b200_internal.h -- shared declarations of libb200heif.so (not part of the public C ABI)
#pragma once
#include <cuda_runtime.h>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>
#include "../../include/b200_heif.h"

namespace b200 {

int set_error(int code, const char* fmt, ...);     // records a thread-local message, returns code
#define B200_CUDA_CHECK(expr)                                                                       \
  do {                                                                                               \
    cudaError_t e__ = (expr);                                                                        \
    if (e__ != cudaSuccess) return ::b200::set_error(B200_E_CUDA, "%s: %s", #expr, cudaGetErrorString(e__)); \
  } while (0)

// size of the chroma planes of a w x h picture; 0 x 0 for monochrome
inline void chroma_size(int chroma, int w, int h, int& cw, int& ch) {
  const int sh = chroma == B200_CHROMA_420 || chroma == B200_CHROMA_422, sv = chroma == B200_CHROMA_420;
  cw = chroma == B200_CHROMA_MONO ? 0 : (w + sh) >> sh;
  ch = chroma == B200_CHROMA_MONO ? 0 : (h + sv) >> sv;
}

// Affine maps of b200_geometry, {m0, ..., m5}: output (u, v) -> source (m0 u + m1 v + m2, m3 u + m4 v + m5).
// out = a o b, i.e. b applied first; out may be a or b.
inline void affine_compose(const int a[6], const int b[6], int out[6]) {
  const int n[6] = {a[0] * b[0] + a[1] * b[3], a[0] * b[1] + a[1] * b[4], a[0] * b[2] + a[1] * b[5] + a[2],
                    a[3] * b[0] + a[4] * b[3], a[3] * b[1] + a[4] * b[4], a[3] * b[2] + a[4] * b[5] + a[5]};
  for (int i = 0; i < 6; i++) out[i] = n[i];
}
// whether m with a w x h output leaves a w_in x h_in picture as it is
inline bool is_identity(const int m[6], int w, int h, int w_in, int h_in) {
  return m[0] == 1 && m[1] == 0 && m[2] == 0 && m[3] == 0 && m[4] == 1 && m[5] == 0 && w == w_in && h == h_in;
}

void ycbcr_to_rgb_coefficients(int matrix, int primaries, float out[4]);
// scale_w x scale_h > 0: the result scaled with HeifPixelImage::scale_nearest_neighbor (0 x 0: the geometry's size)
int launch_color(const b200_planes* in, const b200_geometry* g, const b200_color_options* opt, void* out, void* out_g,
                 void* out_b, size_t out_stride, cudaStream_t stream, int* pipeline, int scale_w = 0, int scale_h = 0);
int launch_rgb_to_ycbcr(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out, cudaStream_t stream);
int plan_rgb_to_ycbcr(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline);
int launch_rgb_to_ycbcr_ex(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, cudaStream_t stream, int* pipeline);
// 8-bit RGB -> rows [y0, y1) of a padded 4:2:0 picture (out: its size, planes and nclx) with clamped source reads; `pipeline`
// from plan_rgb_to_ycbcr for the input's size (Op_RGB24_32_to_YCbCr or Op_RGB_to_YCbCr)
int launch_rgb_to_ycbcr_grid(const b200_rgb_image* in, const b200_planes* out, int pipeline, int y0, int y1, cudaStream_t stream);

}  // namespace b200
