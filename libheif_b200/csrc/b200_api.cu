// b200_api.cu -- extern "C" surface of libb200heif.so (see include/b200_heif.h for the reference citations)
#include "b200_internal.h"
#include "b200_staging.h"
#include <algorithm>
#include <memory>
#include <mutex>
#include <unistd.h>
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

// ---- host <-> device staging of the host entry points.  b200_color_convert_host is what the GPU colour operation of
// integration/ calls from inside heif_decode_image, with libheif's pageable planes on both sides.  Each GPU keeps its stream,
// bounce buffer and device buffer for the life of the process: cudaMalloc + cudaFree per call cost milliseconds, and cudaFree
// synchronises the whole device, i.e. every other decoder of the process.  The instances are never destroyed because the
// CUDA runtime may already be unloading at static destruction.  One mutex serialises all callers.
extern "C++" {
namespace {
struct HostXfer {
  Stream s;
  Bounce bounce;
  DevBuf<char> dev;
};
std::mutex g_xfer_mu;
std::vector<HostXfer*> g_xfer;                      // by device ordinal
constexpr long kMaxCopyThreads = 16;                // host threads that fill / drain the bounce buffers: the online cores, at most this

// the staging of the calling thread's current GPU (g_xfer_mu held), created on first use
int host_xfer(HostXfer** out) {
  int device = 0; B200_CUDA_CHECK(cudaGetDevice(&device));
  if ((size_t)device >= g_xfer.size()) g_xfer.resize((size_t)device + 1, nullptr);
  if (!g_xfer[device]) {
    std::unique_ptr<HostXfer> x(new HostXfer);
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&x->s.h, cudaStreamNonBlocking));
    g_xfer[device] = x.release();
  }
  *out = g_xfer[device];
  return B200_OK;
}
Pool& copy_pool() {                                 // (g_xfer_mu held: parallel_for takes one caller at a time)
  static Pool* pool = new Pool((int)std::max(1L, std::min(kMaxCopyThreads, sysconf(_SC_NPROCESSORS_ONLN))));
  return *pool;
}
// waits for the staging stream; the first error of the call wins
int finish(HostXfer& X, int rc) {
  const cudaError_t e = cudaStreamSynchronize(X.s);
  if (rc == B200_OK && e != cudaSuccess) return set_error(B200_E_CUDA, "sync: %s", cudaGetErrorString(e));
  return rc;
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
  const size_t ybytes = ypitch * (size_t)in->height, cbytes = cpitch * (size_t)ch, abytes = in->alpha ? ybytes : 0, obytes = opitch * (size_t)geom->out_h;
  std::lock_guard<std::mutex> lock(g_xfer_mu);
  HostXfer* X = nullptr;
  int rc;
  if ((rc = host_xfer(&X)) || (rc = X->dev.reserve(ybytes + 2 * cbytes + abytes + obytes * (size_t)nout, false))) return rc;
  char* dy = X->dev.d; char* dcb = dy + ybytes; char* dcr = dcb + cbytes; char* da = dcr + cbytes; char* dout = da + abytes;
  Pool& pool = copy_pool();
  rc = X->bounce.upload(dy, ypitch, in->y, in->y_stride, (size_t)in->width * bps, (size_t)in->height, X->s, pool);
  if (cw && rc == B200_OK) rc = X->bounce.upload(dcb, cpitch, in->cb, in->c_stride, (size_t)cw * bps, (size_t)ch, X->s, pool);
  if (cw && rc == B200_OK) rc = X->bounce.upload(dcr, cpitch, in->cr, in->c_stride, (size_t)cw * bps, (size_t)ch, X->s, pool);
  if (in->alpha && rc == B200_OK) rc = X->bounce.upload(da, ypitch, in->alpha, in->alpha_stride, (size_t)in->width * bps, (size_t)in->height, X->s, pool);
  if (rc == B200_OK) {
    b200_planes d = *in;
    d.y = dy; d.cb = cw ? dcb : nullptr; d.cr = cw ? dcr : nullptr; d.alpha = in->alpha ? da : nullptr; d.y_stride = ypitch; d.c_stride = cpitch; d.alpha_stride = ypitch;
    rc = launch_color(&d, geom, opt, dout, dout + obytes, dout + 2 * obytes, opitch, X->s, pipeline);
  }
  void* outs[3] = {out, out_g, out_b};
  for (int c = 0; c < nout && rc == B200_OK; c++) rc = X->bounce.download(outs[c], out_stride, dout + (size_t)c * obytes, opitch, rowb, (size_t)geom->out_h, X->s, pool);
  return finish(*X, rc);
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
  const size_t ibytes = ipitch * (size_t)h, ybytes = ypitch * (size_t)h, cbytes = cpitch * (size_t)ch, abytes = out->alpha ? ybytes : 0;
  std::lock_guard<std::mutex> lock(g_xfer_mu);
  HostXfer* X = nullptr;
  int rc;
  if ((rc = host_xfer(&X)) || (rc = X->dev.reserve(ibytes + ybytes + 2 * cbytes + abytes, false))) return rc;
  char* din = X->dev.d; char* dy = din + ibytes; char* dcb = dy + ybytes; char* dcr = dcb + cbytes; char* da = out->alpha ? dcr + cbytes : nullptr;
  Pool& pool = copy_pool();
  rc = X->bounce.upload(din, ipitch, rgb, rgb_stride, (size_t)w * bpp, (size_t)h, X->s, pool);
  if (rc == B200_OK) {
    b200_planes d = *out;
    d.y = dy; d.cb = dcb; d.cr = dcr; d.alpha = da; d.y_stride = ypitch; d.c_stride = cpitch; d.alpha_stride = ypitch;
    rc = launch_rgb_to_ycbcr(din, ipitch, has_alpha, &d, X->s);
  }
  if (rc == B200_OK) rc = X->bounce.download((void*)out->y, out->y_stride, dy, ypitch, (size_t)w, (size_t)h, X->s, pool);
  if (rc == B200_OK) rc = X->bounce.download((void*)out->cb, out->c_stride, dcb, cpitch, (size_t)cw, (size_t)ch, X->s, pool);
  if (rc == B200_OK) rc = X->bounce.download((void*)out->cr, out->c_stride, dcr, cpitch, (size_t)cw, (size_t)ch, X->s, pool);
  if (out->alpha && rc == B200_OK) rc = X->bounce.download((void*)out->alpha, out->alpha_stride, da, ypitch, (size_t)w, (size_t)h, X->s, pool);
  return finish(*X, rc);
}

int b200_rgb_to_ycbcr_plan(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline) {
  return plan_rgb_to_ycbcr(in, out, opt, pipeline);
}

int b200_rgb_to_ycbcr_ex_device(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, void* stream, int* pipeline) {
  return launch_rgb_to_ycbcr_ex(in, out, opt, (cudaStream_t)stream, pipeline);
}

int b200_rgb_to_ycbcr_ex_host(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline) {
  int rc = plan_rgb_to_ycbcr(in, out, opt, pipeline);         // refusals before any staging
  if (rc) return rc;
  if (!out->y || !out->cb || !out->cr) return set_error(B200_E_INVALID, "RGB -> YCbCr: output planes missing");
  if (out->width <= 0 || out->height <= 0) return B200_OK;
  const bool planar = in->chroma == B200_CHROMA_444;
  const int w = out->width, h = out->height, bps = in->bit_depth > 8 ? 2 : 1;
  int nch;
  switch (in->chroma) {
    case B200_CHROMA_INTERLEAVED_RGB: nch = 3; break;
    case B200_CHROMA_INTERLEAVED_RGBA: nch = 4; break;
    case B200_CHROMA_INTERLEAVED_RRGGBB_BE: case B200_CHROMA_INTERLEAVED_RRGGBB_LE: nch = 3; break;
    default: nch = planar ? 1 : 4;
  }
  const int nin = planar ? (in->alpha ? 4 : 3) : 1;
  const void* src[4] = {planar ? in->r : in->rgb, in->g, in->b, in->alpha};
  const size_t sstride[4] = {planar ? in->r_stride : in->rgb_stride, in->g_stride, in->b_stride, in->alpha_stride};
  const int sh = out->chroma == B200_CHROMA_444 ? 0 : 1, sv = out->chroma == B200_CHROMA_420 ? 1 : 0;
  const int cw = (w + sh) >> sh, ch = (h + sv) >> sv;
  const size_t irow = (size_t)w * nch * bps, ipitch = (irow + 255) & ~(size_t)255;
  // the caller's rows are read on the host: every stride is checked before anything is staged
  for (int c = 0; c < nin; c++) {
    if (!src[c]) return set_error(B200_E_INVALID, "RGB input planes missing");
    if (sstride[c] < irow) return set_error(B200_E_INVALID, "RGB input plane %d: stride %zu < row of %zu bytes", c, sstride[c], irow);
  }
  if (out->y_stride < (size_t)w * bps || out->c_stride < (size_t)cw * bps || (out->alpha && out->alpha_stride < (size_t)w * bps))
    return set_error(B200_E_INVALID, "YCbCr output stride smaller than a row");
  const size_t ypitch = (((size_t)w * bps) + 255) & ~(size_t)255, cpitch = (((size_t)cw * bps) + 255) & ~(size_t)255;
  const size_t ibytes = ipitch * (size_t)h, ybytes = ypitch * (size_t)h, cbytes = cpitch * (size_t)ch, abytes = out->alpha ? ybytes : 0;
  std::lock_guard<std::mutex> lock(g_xfer_mu);
  HostXfer* X = nullptr;
  if ((rc = host_xfer(&X)) || (rc = X->dev.reserve(ibytes * nin + ybytes + 2 * cbytes + abytes, false))) return rc;
  char* din = X->dev.d; char* dy = din + ibytes * nin; char* dcb = dy + ybytes; char* dcr = dcb + cbytes; char* da = out->alpha ? dcr + cbytes : nullptr;
  Pool& pool = copy_pool();
  for (int c = 0; c < nin && rc == B200_OK; c++) rc = X->bounce.upload(din + (size_t)c * ibytes, ipitch, src[c], sstride[c], irow, (size_t)h, X->s, pool);
  if (rc == B200_OK) {
    b200_rgb_image d = *in;
    if (planar) {
      d.r = din; d.g = din + ibytes; d.b = din + 2 * ibytes; d.alpha = in->alpha ? din + 3 * ibytes : nullptr;
      d.r_stride = d.g_stride = d.b_stride = d.alpha_stride = ipitch;
    } else { d.rgb = din; d.rgb_stride = ipitch; }
    b200_planes o = *out;
    o.y = dy; o.cb = dcb; o.cr = dcr; o.alpha = da; o.y_stride = ypitch; o.c_stride = cpitch; o.alpha_stride = ypitch;
    rc = launch_rgb_to_ycbcr_ex(&d, &o, opt, X->s, pipeline);
  }
  if (rc == B200_OK) rc = X->bounce.download((void*)out->y, out->y_stride, dy, ypitch, (size_t)w * bps, (size_t)h, X->s, pool);
  if (rc == B200_OK) rc = X->bounce.download((void*)out->cb, out->c_stride, dcb, cpitch, (size_t)cw * bps, (size_t)ch, X->s, pool);
  if (rc == B200_OK) rc = X->bounce.download((void*)out->cr, out->c_stride, dcr, cpitch, (size_t)cw * bps, (size_t)ch, X->s, pool);
  if (out->alpha && rc == B200_OK) rc = X->bounce.download((void*)out->alpha, out->alpha_stride, da, ypitch, (size_t)w * bps, (size_t)h, X->s, pool);
  return finish(*X, rc);
}

}  // extern "C"
