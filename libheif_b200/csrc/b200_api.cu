// b200_api.cu -- extern "C" surface of libb200heif.so (see include/b200_heif.h for the reference citations)
#include "b200_internal.h"
#include <algorithm>
#include <mutex>
#include <thread>
#include <vector>

namespace b200 {
static thread_local char g_err[512] = "";
int set_error(int code, const char* fmt, ...) {
  va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
  return code;
}
}  // namespace b200

using namespace b200;

extern "C" {

const char* b200_last_error(void) { return g_err; }
int b200_version(void) { return 100; }

void b200_ycbcr_to_rgb_coefficients(int mc, int cp, float out[4]) { ycbcr_to_rgb_coefficients(mc, cp, out); }

void b200_geometry_init(int w, int h, int chroma, b200_geometry* g) {
  g->m[0] = 1; g->m[1] = 0; g->m[2] = 0; g->m[3] = 0; g->m[4] = 1; g->m[5] = 0; g->out_w = w; g->out_h = h;
  g->chroma = chroma; g->detour = 0;
  for (int i = 0; i < 6; i++) g->pre[i] = g->m[i];
  g->pre_w = w; g->pre_h = h;
}
void b200_geometry_identity(int w, int h, b200_geometry* g) { b200_geometry_init(w, h, B200_CHROMA_420, g); }

// new(u,v) -> old(u',v') = T(u,v), then old mapping applied: m' = m o T
static void compose(b200_geometry* g, const int t[6], int nw, int nh) {
  int n[6];
  n[0] = g->m[0] * t[0] + g->m[1] * t[3]; n[1] = g->m[0] * t[1] + g->m[1] * t[4]; n[2] = g->m[0] * t[2] + g->m[1] * t[5] + g->m[2];
  n[3] = g->m[3] * t[0] + g->m[4] * t[3]; n[4] = g->m[3] * t[1] + g->m[4] * t[4]; n[5] = g->m[3] * t[2] + g->m[4] * t[5] + g->m[5];
  for (int i = 0; i < 6; i++) g->m[i] = n[i];
  g->out_w = nw; g->out_h = nh;
}

// The reference's "need_conversion" tests (pixelimage.cc:1187-1215 rotate, 1370-1381 mirror, 1458-1467 crop), on the picture
// as it is at this point of the chain.  Once taken, the picture is 4:4:4 and no further test applies.
static void detour_if(b200_geometry* g, bool need) {
  if (!need || g->detour) return;
  for (int i = 0; i < 6; i++) g->pre[i] = g->m[i];
  g->pre_w = g->out_w; g->pre_h = g->out_h;
  g->m[0] = 1; g->m[1] = 0; g->m[2] = 0; g->m[3] = 0; g->m[4] = 1; g->m[5] = 0;
  g->detour = 1;
}

int b200_geometry_rotate_ccw(b200_geometry* g, int degrees) {
  const int w = g->out_w, h = g->out_h;
  if (degrees == 0) return B200_OK;
  if (degrees != 90 && degrees != 180 && degrees != 270) return set_error(B200_E_INVALID, "rotation %d", degrees);
  const bool ow = w & 1, oh = h & 1;
  if (g->chroma == B200_CHROMA_422) detour_if(g, degrees == 90 || degrees == 270 || (degrees == 180 && oh));
  else if (g->chroma == B200_CHROMA_420) detour_if(g, (degrees == 90 && ow) || (degrees == 180 && (ow || oh)) || (degrees == 270 && oh));
  if (degrees == 90) { const int t[6] = {0, -1, w - 1, 1, 0, 0}; compose(g, t, h, w); }        // out[y][x] = in[x][w-1-y]
  else if (degrees == 180) { const int t[6] = {-1, 0, w - 1, 0, -1, h - 1}; compose(g, t, w, h); }
  else { const int t[6] = {0, 1, 0, -1, 0, h - 1}; compose(g, t, h, w); }                       // out[y][x] = in[h-1-x][y]
  return B200_OK;
}

int b200_geometry_mirror(b200_geometry* g, int direction) {
  const int w = g->out_w, h = g->out_h;
  if (direction != 0 && direction != 1) return set_error(B200_E_INVALID, "mirror direction %d", direction);
  if (g->chroma == B200_CHROMA_422) detour_if(g, direction == 1 && (w & 1));
  else if (g->chroma == B200_CHROMA_420) detour_if(g, (w & 1) || (h & 1));
  if (direction == 1) { const int t[6] = {-1, 0, w - 1, 0, 1, 0}; compose(g, t, w, h); }
  else { const int t[6] = {1, 0, 0, 0, -1, h - 1}; compose(g, t, w, h); }
  return B200_OK;
}

int b200_geometry_crop(b200_geometry* g, int left, int right, int top, int bottom) {
  if (left < 0 || top < 0 || right >= g->out_w || bottom >= g->out_h || right < left || bottom < top)
    return set_error(B200_E_INVALID, "crop window outside image");
  if (g->chroma == B200_CHROMA_422) detour_if(g, left & 1);
  else if (g->chroma == B200_CHROMA_420) detour_if(g, (left & 1) || (top & 1));
  const int t[6] = {1, 0, left, 0, 1, top};
  compose(g, t, right - left + 1, bottom - top + 1);
  return B200_OK;
}

int b200_color_convert_device(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt, void* out,
                              void* out_g, void* out_b, size_t out_stride, void* stream, int* pipeline) {
  return launch_color(in, geom, opt, out, out_g, out_b, out_stride, (cudaStream_t)stream, pipeline);
}

static size_t out_row_bytes(int fmt, int w, int bit_depth_in) {
  switch (fmt) {
    case B200_CHROMA_INTERLEAVED_RGB: return (size_t)w * 3;
    case B200_CHROMA_INTERLEAVED_RGBA: return (size_t)w * 4;
    case B200_CHROMA_INTERLEAVED_RRGGBB_BE: case B200_CHROMA_INTERLEAVED_RRGGBB_LE: return (size_t)w * 6;
    case B200_CHROMA_INTERLEAVED_RRGGBBAA_BE: case B200_CHROMA_INTERLEAVED_RRGGBBAA_LE: return (size_t)w * 8;
    default: return (size_t)w * (bit_depth_in > 8 ? 2 : 1);
  }
}

static int color_convert_host_simple(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt, void* out,
                            void* out_g, void* out_b, size_t out_stride, int* pipeline) {
  if (!in || !geom || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  const int bps = in->bit_depth > 8 ? 2 : 1;
  const int sh = (in->chroma == B200_CHROMA_420 || in->chroma == B200_CHROMA_422) ? 1 : 0;
  const int sv = in->chroma == B200_CHROMA_420 ? 1 : 0;
  const int cw = in->chroma == B200_CHROMA_MONO ? 0 : (in->width + sh) >> sh, ch = in->chroma == B200_CHROMA_MONO ? 0 : (in->height + sv) >> sv;
  const size_t ypitch = (((size_t)in->width * bps) + 255) & ~(size_t)255, cpitch = (((size_t)cw * bps) + 255) & ~(size_t)255;
  const size_t rowb = out_row_bytes(opt->out_chroma, geom->out_w, in->bit_depth);
  const size_t opitch = (rowb + 255) & ~(size_t)255;
  const int nout = opt->out_chroma == B200_CHROMA_444 ? 3 : 1;
  char *dy = nullptr, *dcb = nullptr, *dcr = nullptr, *da = nullptr, *dout = nullptr;
  cudaStream_t s; B200_CUDA_CHECK(cudaStreamCreate(&s));
  int rc = B200_OK;
  auto fail = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && rc == B200_OK) rc = set_error(B200_E_CUDA, "%s: %s", what, cudaGetErrorString(e)); };
  fail(cudaMalloc(&dy, ypitch * in->height), "cudaMalloc");
  if (cw) { fail(cudaMalloc(&dcb, cpitch * ch), "cudaMalloc"); fail(cudaMalloc(&dcr, cpitch * ch), "cudaMalloc"); }
  if (in->alpha) fail(cudaMalloc(&da, ypitch * in->height), "cudaMalloc");
  fail(cudaMalloc(&dout, opitch * geom->out_h * nout), "cudaMalloc");
  if (rc == B200_OK) {
    fail(cudaMemcpy2DAsync(dy, ypitch, in->y, in->y_stride, (size_t)in->width * bps, in->height, cudaMemcpyHostToDevice, s), "H2D");
    if (cw) {
      fail(cudaMemcpy2DAsync(dcb, cpitch, in->cb, in->c_stride, (size_t)cw * bps, ch, cudaMemcpyHostToDevice, s), "H2D");
      fail(cudaMemcpy2DAsync(dcr, cpitch, in->cr, in->c_stride, (size_t)cw * bps, ch, cudaMemcpyHostToDevice, s), "H2D");
    }
    if (in->alpha) fail(cudaMemcpy2DAsync(da, ypitch, in->alpha, in->alpha_stride, (size_t)in->width * bps, in->height, cudaMemcpyHostToDevice, s), "H2D");
  }
  if (rc == B200_OK) {
    b200_planes d = *in;
    d.y = dy; d.cb = dcb; d.cr = dcr; d.alpha = da; d.y_stride = ypitch; d.c_stride = cpitch; d.alpha_stride = ypitch;
    rc = launch_color(&d, geom, opt, dout, dout + opitch * geom->out_h, dout + 2 * opitch * geom->out_h, opitch, s, pipeline);
  }
  if (rc == B200_OK) {
    void* outs[3] = {out, out_g, out_b};
    for (int c = 0; c < nout; c++)
      fail(cudaMemcpy2DAsync(outs[c], out_stride, dout + c * opitch * geom->out_h, opitch, rowb, geom->out_h, cudaMemcpyDeviceToHost, s), "D2H");
    fail(cudaStreamSynchronize(s), "sync");
  }
  cudaFree(dy); cudaFree(dcb); cudaFree(dcr); cudaFree(da); cudaFree(dout); cudaStreamDestroy(s);
  return rc;
}

// ---- host <-> device staging of b200_color_convert_host (the call the GPU colour operation of integration/ makes from inside
// heif_decode_image, with libheif's pageable planes on both sides).  Pageable memory is moved through a page-locked bounce
// buffer in bands: a few host threads copy band k (+ take its page faults) while the DMA engine moves band k - 1, and the
// device buffers / bounce buffer / stream live as long as the process (cudaMalloc + cudaFree per call cost milliseconds and
// cudaFree synchronises the whole device, i.e. every other decoder of the process).  Page-locked operands are copied directly.
extern "C++" {
namespace {
struct HostXfer {
  std::mutex mu;
  cudaStream_t s = nullptr;
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool ev_used[2] = {false, false};
  char* dev = nullptr; size_t dev_cap = 0;
  uint8_t* pin = nullptr;
  int device = -1;
  unsigned slot = 0;
};
HostXfer g_xfer;
constexpr size_t kBounceSlot = (size_t)32 << 20;
constexpr unsigned kMaxCopyThreads = 16;           // host threads that fill / drain the bounce buffer: the online cores, at most this

bool host_page_locked(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}
int xfer_threads() {
  static const int n = [] { unsigned h = std::thread::hardware_concurrency(); return (int)(h < 1 ? 1 : (h > kMaxCopyThreads ? kMaxCopyThreads : h)); }();
  return n;
}
template <class F>
void parallel_rows(size_t rows, size_t bytes, const F& fn) {       // fn(r0, r1)
  int t = xfer_threads();
  if (bytes < ((size_t)1 << 20) || rows < 2) t = 1;
  if ((size_t)t > rows) t = (int)rows;
  if (t <= 1) { fn((size_t)0, rows); return; }
  std::vector<std::thread> th;
  for (int i = 1; i < t; i++) th.emplace_back([&, i] { fn(rows * (size_t)i / (size_t)t, rows * (size_t)(i + 1) / (size_t)t); });
  fn((size_t)0, rows / (size_t)t);
  for (auto& x : th) x.join();
}
// host plane (pageable or page-locked) -> device plane
cudaError_t upload_plane(HostXfer& X, char* dst, size_t dpitch, const void* src, size_t sstride, size_t wb, size_t h) {
  if (!wb || !h) return cudaSuccess;
  if (host_page_locked(src)) return cudaMemcpy2DAsync(dst, dpitch, src, sstride, wb, h, cudaMemcpyHostToDevice, X.s);
  const size_t rows_per = std::max<size_t>(1, kBounceSlot / wb);
  for (size_t y0 = 0; y0 < h; y0 += rows_per) {
    const unsigned k = X.slot++ & 1u;
    const size_t n = std::min(rows_per, h - y0);
    cudaError_t e;
    if (X.ev_used[k] && (e = cudaEventSynchronize(X.ev[k])) != cudaSuccess) return e;     // the DMA that last used this slot is done
    uint8_t* slot = X.pin + (size_t)k * kBounceSlot;
    const uint8_t* s0 = static_cast<const uint8_t*>(src) + y0 * sstride;
    parallel_rows(n, n * wb, [&](size_t r0, size_t r1) { for (size_t r = r0; r < r1; r++) memcpy(slot + r * wb, s0 + r * sstride, wb); });
    if ((e = cudaMemcpy2DAsync(dst + y0 * dpitch, dpitch, slot, wb, wb, n, cudaMemcpyHostToDevice, X.s)) != cudaSuccess) return e;
    if ((e = cudaEventRecord(X.ev[k], X.s)) != cudaSuccess) return e;
    X.ev_used[k] = true;
  }
  return cudaSuccess;
}
// device plane -> host plane (pageable or page-locked); returns with the data in place unless the destination is page-locked
// (then the copy is queued on X.s and the caller synchronises)
cudaError_t download_plane(HostXfer& X, void* dst, size_t dstride, const char* src, size_t spitch, size_t wb, size_t h) {
  if (!wb || !h) return cudaSuccess;
  if (host_page_locked(dst)) return cudaMemcpy2DAsync(dst, dstride, src, spitch, wb, h, cudaMemcpyDeviceToHost, X.s);
  const size_t rows_per = std::max<size_t>(1, kBounceSlot / wb);
  const size_t nb = (h + rows_per - 1) / rows_per;
  cudaError_t e;
  for (size_t k = 0; k <= nb; k++) {
    if (k < nb) {                                         // queue band k into slot k & 1 (its previous content, band k - 2, was copied out in iteration k - 1)
      const size_t y0 = k * rows_per, n = std::min(rows_per, h - y0);
      if ((e = cudaMemcpy2DAsync(X.pin + (k & 1) * kBounceSlot, wb, src + y0 * spitch, spitch, wb, n, cudaMemcpyDeviceToHost, X.s)) != cudaSuccess) return e;
      if ((e = cudaEventRecord(X.ev[k & 1], X.s)) != cudaSuccess) return e;
      X.ev_used[k & 1] = true;
    }
    if (k > 0) {                                          // band k - 1 has arrived: host threads move it to its place while band k is in flight
      const size_t j = k - 1, y0 = j * rows_per, n = std::min(rows_per, h - y0);
      if ((e = cudaEventSynchronize(X.ev[j & 1])) != cudaSuccess) return e;
      const uint8_t* slot = X.pin + (j & 1) * kBounceSlot;
      uint8_t* d0 = static_cast<uint8_t*>(dst) + y0 * dstride;
      parallel_rows(n, n * wb, [&](size_t r0, size_t r1) { for (size_t r = r0; r < r1; r++) memcpy(d0 + r * dstride, slot + r * wb, wb); });
    }
  }
  X.slot = 0;                                             // both slots are idle again (every band was waited for)
  return cudaSuccess;
}
}  // namespace
}  // extern "C++"

int b200_color_convert_host(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt, void* out,
                            void* out_g, void* out_b, size_t out_stride, int* pipeline) {
  if (!in || !geom || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  const int bps = in->bit_depth > 8 ? 2 : 1;
  const int sh = (in->chroma == B200_CHROMA_420 || in->chroma == B200_CHROMA_422) ? 1 : 0;
  const int sv = in->chroma == B200_CHROMA_420 ? 1 : 0;
  const int cw = in->chroma == B200_CHROMA_MONO ? 0 : (in->width + sh) >> sh, ch = in->chroma == B200_CHROMA_MONO ? 0 : (in->height + sv) >> sv;
  const size_t ypitch = (((size_t)in->width * bps) + 255) & ~(size_t)255, cpitch = (((size_t)cw * bps) + 255) & ~(size_t)255;
  const size_t rowb = out_row_bytes(opt->out_chroma, geom->out_w, in->bit_depth);
  const size_t opitch = (rowb + 255) & ~(size_t)255;
  const int nout = opt->out_chroma == B200_CHROMA_444 ? 3 : 1;
  if (nout == 3 && (!out_g || !out_b)) return set_error(B200_E_INVALID, "planar output needs three planes");
  int device = 0; B200_CUDA_CHECK(cudaGetDevice(&device));
  HostXfer& X = g_xfer;
  std::lock_guard<std::mutex> lock(X.mu);
  if (X.device >= 0 && X.device != device) return color_convert_host_simple(in, geom, opt, out, out_g, out_b, out_stride, pipeline);   // (the cached buffers belong to another GPU)
  if (!X.s) {
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&X.s, cudaStreamNonBlocking));
    for (auto& e : X.ev) B200_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    B200_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&X.pin), 2 * kBounceSlot, cudaHostAllocDefault));
    X.device = device;
  }
  const size_t ybytes = ypitch * (size_t)in->height, cbytes = cpitch * (size_t)ch, abytes = in->alpha ? ybytes : 0, obytes = opitch * (size_t)geom->out_h;
  const size_t need = ybytes + 2 * cbytes + abytes + obytes * (size_t)nout;
  if (need > X.dev_cap) {
    if (X.dev) { B200_CUDA_CHECK(cudaStreamSynchronize(X.s)); cudaFree(X.dev); X.dev = nullptr; X.dev_cap = 0; }
    B200_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&X.dev), need + need / 8));
    X.dev_cap = need + need / 8;
  }
  char* dy = X.dev; char* dcb = dy + ybytes; char* dcr = dcb + cbytes; char* da = dcr + cbytes; char* dout = da + abytes;
  X.slot = 0; X.ev_used[0] = X.ev_used[1] = false;
  int rc = B200_OK;
  auto fail = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && rc == B200_OK) rc = set_error(B200_E_CUDA, "%s: %s", what, cudaGetErrorString(e)); };
  fail(upload_plane(X, dy, ypitch, in->y, in->y_stride, (size_t)in->width * bps, (size_t)in->height), "H2D");
  if (cw && rc == B200_OK) {
    fail(upload_plane(X, dcb, cpitch, in->cb, in->c_stride, (size_t)cw * bps, (size_t)ch), "H2D");
    fail(upload_plane(X, dcr, cpitch, in->cr, in->c_stride, (size_t)cw * bps, (size_t)ch), "H2D");
  }
  if (in->alpha && rc == B200_OK) fail(upload_plane(X, da, ypitch, in->alpha, in->alpha_stride, (size_t)in->width * bps, (size_t)in->height), "H2D");
  if (rc == B200_OK) {
    b200_planes d = *in;
    d.y = dy; d.cb = cw ? dcb : nullptr; d.cr = cw ? dcr : nullptr; d.alpha = in->alpha ? da : nullptr; d.y_stride = ypitch; d.c_stride = cpitch; d.alpha_stride = ypitch;
    rc = launch_color(&d, geom, opt, dout, dout + obytes, dout + 2 * obytes, opitch, X.s, pipeline);
  }
  if (rc == B200_OK) {
    void* outs[3] = {out, out_g, out_b};
    for (int c = 0; c < nout && rc == B200_OK; c++) fail(download_plane(X, outs[c], out_stride, dout + (size_t)c * obytes, opitch, rowb, (size_t)geom->out_h), "D2H");
  }
  fail(cudaStreamSynchronize(X.s), "sync");
  return rc;
}

int b200_rgb_to_ycbcr_device(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out, void* stream) {
  return launch_rgb_to_ycbcr(rgb, rgb_stride, has_alpha, out, (cudaStream_t)stream);
}

int b200_rgb_to_ycbcr_host(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out) {
  if (!rgb || !out || !out->y) return set_error(B200_E_INVALID, "null argument");
  if (out->width <= 0 || out->height <= 0) return B200_OK;
  if (out->chroma != B200_CHROMA_420 && out->chroma != B200_CHROMA_422 && out->chroma != B200_CHROMA_444)
    return set_error(B200_E_UNSUPPORTED, "RGB -> YCbCr: target chroma %d", out->chroma);
  if (!out->cb || !out->cr) return set_error(B200_E_INVALID, "RGB -> YCbCr: chroma planes missing");
  const int w = out->width, h = out->height, bpp = has_alpha ? 4 : 3;
  const int sh = out->chroma == B200_CHROMA_444 ? 0 : 1, sv = out->chroma == B200_CHROMA_420 ? 1 : 0;
  const int cw = (w + sh) >> sh, ch = (h + sv) >> sv;
  const size_t ipitch = (((size_t)w * bpp) + 255) & ~(size_t)255, ypitch = ((size_t)w + 255) & ~(size_t)255, cpitch = ((size_t)cw + 255) & ~(size_t)255;
  char *din = nullptr, *dy = nullptr, *dcb = nullptr, *dcr = nullptr, *da = nullptr;
  cudaStream_t s; B200_CUDA_CHECK(cudaStreamCreate(&s));
  int rc = B200_OK;
  auto fail = [&](cudaError_t e, const char* what) { if (e != cudaSuccess && rc == B200_OK) rc = set_error(B200_E_CUDA, "%s: %s", what, cudaGetErrorString(e)); };
  fail(cudaMalloc(&din, ipitch * h), "cudaMalloc");
  fail(cudaMalloc(&dy, ypitch * h), "cudaMalloc");
  fail(cudaMalloc(&dcb, cpitch * ch), "cudaMalloc");
  fail(cudaMalloc(&dcr, cpitch * ch), "cudaMalloc");
  if (out->alpha) fail(cudaMalloc(&da, ypitch * h), "cudaMalloc");
  if (rc == B200_OK) fail(cudaMemcpy2DAsync(din, ipitch, rgb, rgb_stride, (size_t)w * bpp, h, cudaMemcpyHostToDevice, s), "H2D");
  if (rc == B200_OK) {
    b200_planes d = *out;
    d.y = dy; d.cb = dcb; d.cr = dcr; d.alpha = da; d.y_stride = ypitch; d.c_stride = cpitch; d.alpha_stride = ypitch;
    rc = launch_rgb_to_ycbcr(din, ipitch, has_alpha, &d, s);
  }
  if (rc == B200_OK) {
    fail(cudaMemcpy2DAsync((void*)out->y, out->y_stride, dy, ypitch, w, h, cudaMemcpyDeviceToHost, s), "D2H");
    fail(cudaMemcpy2DAsync((void*)out->cb, out->c_stride, dcb, cpitch, cw, ch, cudaMemcpyDeviceToHost, s), "D2H");
    fail(cudaMemcpy2DAsync((void*)out->cr, out->c_stride, dcr, cpitch, cw, ch, cudaMemcpyDeviceToHost, s), "D2H");
    if (out->alpha) fail(cudaMemcpy2DAsync((void*)out->alpha, out->alpha_stride, da, ypitch, w, h, cudaMemcpyDeviceToHost, s), "D2H");
    fail(cudaStreamSynchronize(s), "sync");
  }
  cudaFree(din); cudaFree(dy); cudaFree(dcb); cudaFree(dcr); cudaFree(da); cudaStreamDestroy(s);
  return rc;
}

}  // extern "C"
