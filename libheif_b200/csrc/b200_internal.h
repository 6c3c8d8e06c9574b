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

void ycbcr_to_rgb_coefficients(int matrix, int primaries, float out[4]);
int launch_color(const b200_planes* in, const b200_geometry* g, const b200_color_options* opt, void* out, void* out_g,
                 void* out_b, size_t out_stride, cudaStream_t stream, int* pipeline);
int launch_rgb_to_ycbcr(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out, cudaStream_t stream);
int plan_rgb_to_ycbcr(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline);
int launch_rgb_to_ycbcr_ex(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, cudaStream_t stream, int* pipeline);
// 8-bit RGB -> rows [y0, y1) of a padded 4:2:0 picture (out: its size, planes and nclx) with clamped source reads; `pipeline`
// from plan_rgb_to_ycbcr for the input's size (Op_RGB24_32_to_YCbCr or Op_RGB_to_YCbCr)
int launch_rgb_to_ycbcr_grid(const b200_rgb_image* in, const b200_planes* out, int pipeline, int y0, int y1, cudaStream_t stream);

}  // namespace b200
