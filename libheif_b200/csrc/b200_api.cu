// b200_api.cu -- extern "C" surface of libb200heif.so (see include/b200_heif.h for the reference citations)
#include "b200_internal.h"
#include "b200_staging.h"
#include <algorithm>
#include <functional>
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
  affine_compose(g->m, t, g->m);
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

int b200_color_convert_scaled_device(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt, int scale_w, int scale_h,
                                     void* out, void* out_g, void* out_b, size_t out_stride, void* stream, int* pipeline) {
  if (scale_w < 1) return set_error(B200_E_INVALID, "scale_w %d: the scaled picture needs at least one column", scale_w);
  if (scale_h < 1) return set_error(B200_E_INVALID, "scale_h %d: the scaled picture needs at least one row", scale_h);
  const void* const args[] = {in, geom, opt, out};
  const char* const names[] = {"in", "geom", "opt", "out"};
  for (int i = 0; i < 4; i++) if (!args[i]) return set_error(B200_E_INVALID, "%s is NULL", names[i]);
  return launch_color(in, geom, opt, out, out_g, out_b, out_stride, (cudaStream_t)stream, pipeline, scale_w, scale_h);
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

// A host plane of `rows` rows of `row_bytes` bytes, `stride` bytes apart.  A plane with a null pointer is absent.
struct HostPlane { const void* p; size_t stride, row_bytes, rows; };
// A plane's device copy: a null pointer for an absent plane.
struct DevPlane { char* p; size_t pitch; };

// The staging of a host entry point: copies of the planes `in` and `out` (in that order) at 256-byte pitches in one block
// of the calling thread's GPU's device buffer.  Uploads `in` in order, calls `run` with the copies (dev[i]: the i-th plane
// of `in`, then of `out`) and the staging stream, downloads `out` in order and waits for the stream.
int stage(const std::vector<HostPlane>& in, const std::vector<HostPlane>& out, const std::function<int(const DevPlane*, cudaStream_t)>& run) {
  std::vector<HostPlane> all(in);
  all.insert(all.end(), out.begin(), out.end());
  std::vector<DevPlane> dev(all.size());
  size_t bytes = 0;
  for (size_t i = 0; i < all.size(); i++) {
    dev[i].pitch = (all[i].row_bytes + 255) & ~(size_t)255;
    if (all[i].p) bytes += dev[i].pitch * all[i].rows;
  }
  std::lock_guard<std::mutex> lock(g_xfer_mu);
  HostXfer* X = nullptr;
  int rc;
  if ((rc = host_xfer(&X)) || (rc = X->dev.reserve(bytes, false))) return rc;
  char* next = X->dev.d;
  for (size_t i = 0; i < all.size(); i++)
    if (all[i].p) { dev[i].p = next; next += dev[i].pitch * all[i].rows; }
  Pool& pool = copy_pool();
  for (size_t i = 0; i < in.size() && rc == B200_OK; i++)
    if (in[i].p) rc = X->bounce.upload(dev[i].p, dev[i].pitch, in[i].p, in[i].stride, in[i].row_bytes, in[i].rows, X->s, pool);
  if (rc == B200_OK) rc = run(dev.data(), X->s);
  for (size_t i = in.size(); i < all.size() && rc == B200_OK; i++)
    if (all[i].p) rc = X->bounce.download((void*)all[i].p, all[i].stride, dev[i].p, dev[i].pitch, all[i].row_bytes, all[i].rows, X->s, pool);
  return finish(*X, rc);
}

// Y, Cb, Cr and alpha of `p` at `bps` bytes per sample (no chroma planes for monochrome)
std::vector<HostPlane> ycc_planes(const b200_planes& p, size_t bps) {
  int cw, ch;
  chroma_size(p.chroma, p.width, p.height, cw, ch);
  const size_t w = (size_t)p.width, h = (size_t)p.height;
  return {{p.y, p.y_stride, w * bps, h}, {cw ? p.cb : nullptr, p.c_stride, cw * bps, (size_t)ch},
          {cw ? p.cr : nullptr, p.c_stride, cw * bps, (size_t)ch}, {p.alpha, p.alpha_stride, w * bps, h}};
}
// `p` on the device copies dev[0..3] of its ycc_planes()
b200_planes on_device(b200_planes p, const DevPlane* dev) {
  p.y = dev[0].p; p.cb = dev[1].p; p.cr = dev[2].p; p.alpha = dev[3].p;
  p.y_stride = dev[0].pitch; p.c_stride = dev[1].pitch; p.alpha_stride = dev[3].pitch;
  return p;
}
}  // namespace
}  // extern "C++"

int b200_color_convert_host(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt, void* out,
                            void* out_g, void* out_b, size_t out_stride, int* pipeline) {
  if (!in || !geom || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  const size_t rowb = out_row_bytes(opt->out_chroma, geom->out_w, in->bit_depth), oh = (size_t)geom->out_h;
  const bool planar = opt->out_chroma == B200_CHROMA_444;
  if (planar && (!out_g || !out_b)) return set_error(B200_E_INVALID, "planar output needs three planes");
  return stage(ycc_planes(*in, in->bit_depth > 8 ? 2 : 1),
               {{out, out_stride, rowb, oh}, {planar ? out_g : nullptr, out_stride, rowb, oh}, {planar ? out_b : nullptr, out_stride, rowb, oh}},
               [&](const DevPlane* dev, cudaStream_t s) {
                 const b200_planes d = on_device(*in, dev);
                 return launch_color(&d, geom, opt, dev[4].p, dev[5].p, dev[6].p, dev[4].pitch, s, pipeline);
               });
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
  return stage({{rgb, rgb_stride, (size_t)out->width * (has_alpha ? 4 : 3), (size_t)out->height}}, ycc_planes(*out, 1),
               [&](const DevPlane* dev, cudaStream_t s) {
                 const b200_planes d = on_device(*out, dev + 1);
                 return launch_rgb_to_ycbcr(dev[0].p, dev[0].pitch, has_alpha, &d, s);
               });
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
  int cw, ch;
  chroma_size(out->chroma, w, h, cw, ch);
  const size_t irow = (size_t)w * nch * bps;
  // the caller's rows are read on the host: every stride is checked before anything is staged
  std::vector<HostPlane> rgb(4);
  for (int c = 0; c < nin; c++) {
    if (!src[c]) return set_error(B200_E_INVALID, "RGB input planes missing");
    if (sstride[c] < irow) return set_error(B200_E_INVALID, "RGB input plane %d: stride %zu < row of %zu bytes", c, sstride[c], irow);
    rgb[c] = {src[c], sstride[c], irow, (size_t)h};
  }
  if (out->y_stride < (size_t)w * bps || out->c_stride < (size_t)cw * bps || (out->alpha && out->alpha_stride < (size_t)w * bps))
    return set_error(B200_E_INVALID, "YCbCr output stride smaller than a row");
  return stage(rgb, ycc_planes(*out, bps), [&](const DevPlane* dev, cudaStream_t s) {
    b200_rgb_image d = *in;
    if (planar) {
      d.r = dev[0].p; d.g = dev[1].p; d.b = dev[2].p; d.alpha = dev[3].p;
      d.r_stride = d.g_stride = d.b_stride = d.alpha_stride = dev[0].pitch;
    } else { d.rgb = dev[0].p; d.rgb_stride = dev[0].pitch; }
    const b200_planes o = on_device(*out, dev + 4);
    return launch_rgb_to_ycbcr_ex(&d, &o, opt, s, pipeline);
  });
}

}  // extern "C"
