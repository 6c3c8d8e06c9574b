// b200_plugin.cc -- the drop-in boundary: a heif_decoder_plugin and a heif_encoder_plugin backed by libb200heif.
//
// Decoder: replaces libheif/plugins/decoder_libde265.cc member for member (table :497-517): NAL push :322-368,
// decode :386-457, plane hand-over into a heif_image allocated with heif_image_add_plane_safe :97-171, nclx from the
// VUI :426-448, security limit :183-198.  libheif drives it as new_decoder2 -> push_data2 -> flush_data ->
// decode_next_image2 -> free_decoder (libheif/codecs/decoder.cc:388-405,441-446,458-460,487-493,317-324), from up to
// max_decoding_threads threads with one instance each (image-items/grid.cc:405-453).
// Encoder: the role of libheif/plugins/encoder_x265.cc (table :1247-1284): encode_image :1186-1203 then
// get_compressed_data :1206-1236 returning one NAL per call without start code (codecs/hevc_enc.cc:45-86).
//
// The plugin calls back into libheif's public C API only; those entry points are resolved at run time with dlsym so
// that libb200heif.so has no link-time dependency on libheif (see include/b200_heif_plugin_abi.h).
#include "b200_internal.h"
#include "../../include/b200_heif_plugin_abi.h"
#include <dlfcn.h>
#include <chrono>
#include <condition_variable>
#include <deque>
#include <map>
#include <mutex>
#include <thread>
#include <tuple>
#include <string>
#include <vector>

namespace {

// ---- libheif C API used by the plugins (signatures from libheif/api/libheif/heif_image.h, heif_color.h)
struct HeifApi {
  b200h_error (*image_create)(int w, int h, int colorspace, int chroma, b200h_image** out);
  b200h_error (*image_add_plane_safe)(b200h_image*, int channel, int w, int h, int bit_depth, const b200h_security_limits*);
  uint8_t* (*image_get_plane2)(b200h_image*, int channel, size_t* stride);
  const uint8_t* (*image_get_plane_readonly2)(const b200h_image*, int channel, size_t* stride);
  void (*image_release)(const b200h_image*);
  void* (*nclx_alloc)(void);
  void (*nclx_free)(void*);
  b200h_error (*nclx_set_primaries)(void*, uint16_t);
  b200h_error (*nclx_set_transfer)(void*, uint16_t);
  b200h_error (*nclx_set_matrix)(void*, uint16_t);
  b200h_error (*image_set_nclx)(b200h_image*, const void*);
  b200h_error (*image_get_nclx)(const b200h_image*, void** out);
  int (*image_get_width)(const b200h_image*, int channel);
  int (*image_get_height)(const b200h_image*, int channel);
  int (*image_get_bpp_range)(const b200h_image*, int channel);
  int (*image_get_colorspace)(const b200h_image*);
  int (*image_get_chroma)(const b200h_image*);
  const b200h_security_limits* (*global_limits)(void);
  bool ok = false;
};
HeifApi g_api;
void* g_heif_handle = nullptr;
std::once_flag g_api_once;

void resolve_api() {
  void* h = g_heif_handle ? g_heif_handle : RTLD_DEFAULT;
  bool ok = true;
  auto get = [&](const char* n) { void* p = dlsym(h, n); if (!p) ok = false; return p; };
  *(void**)&g_api.image_create = get("heif_image_create");
  *(void**)&g_api.image_add_plane_safe = get("heif_image_add_plane_safe");
  *(void**)&g_api.image_get_plane2 = get("heif_image_get_plane2");
  *(void**)&g_api.image_get_plane_readonly2 = get("heif_image_get_plane_readonly2");
  *(void**)&g_api.image_release = get("heif_image_release");
  *(void**)&g_api.nclx_alloc = get("heif_nclx_color_profile_alloc");
  *(void**)&g_api.nclx_free = get("heif_nclx_color_profile_free");
  *(void**)&g_api.nclx_set_primaries = get("heif_nclx_color_profile_set_color_primaries");
  *(void**)&g_api.nclx_set_transfer = get("heif_nclx_color_profile_set_transfer_characteristics");
  *(void**)&g_api.nclx_set_matrix = get("heif_nclx_color_profile_set_matrix_coefficients");
  *(void**)&g_api.image_set_nclx = get("heif_image_set_nclx_color_profile");
  *(void**)&g_api.image_get_nclx = get("heif_image_get_nclx_color_profile");
  *(void**)&g_api.image_get_width = get("heif_image_get_width");
  *(void**)&g_api.image_get_height = get("heif_image_get_height");
  *(void**)&g_api.image_get_bpp_range = get("heif_image_get_bits_per_pixel_range");
  *(void**)&g_api.image_get_colorspace = get("heif_image_get_colorspace");
  *(void**)&g_api.image_get_chroma = get("heif_image_get_chroma_format");
  *(void**)&g_api.global_limits = get("heif_get_global_security_limits");
  g_api.ok = ok;
}
bool api_ready() { std::call_once(g_api_once, resolve_api); return g_api.ok; }

// layout of the public heif_color_profile_nclx (libheif/api/libheif/heif_color.h): only full_range_flag is written
// directly, exactly like decoder_libde265.cc:446 does.
struct NclxPublic { uint8_t version; int color_primaries; int transfer_characteristics; int matrix_coefficients; uint8_t full_range_flag; };

const char kOk[] = "Success";
b200h_error ok_err() { return b200h_error{B200H_ERR_OK, B200H_SUBERR_UNSPECIFIED, kOk}; }

// error messages must outlive the call (decoder_libde265.cc:150-157): thread-local storage
thread_local std::string t_msg;
b200h_error make_err(int code, int sub, const std::string& m) { t_msg = m; return b200h_error{code, sub, t_msg.c_str()}; }
b200h_error from_b200(int rc, bool encoder) {
  std::string m = b200_last_error();
  switch (rc) {
    case B200_E_UNSUPPORTED: return make_err(B200H_ERR_UNSUPPORTED_FEATURE, B200H_SUBERR_UNSUPPORTED_CODEC, m);
    case B200_E_LIMIT: return make_err(B200H_ERR_MEMORY, B200H_SUBERR_SECURITY_LIMIT, m);
    default: return make_err(encoder ? B200H_ERR_ENCODER_PLUGIN : B200H_ERR_DECODER_PLUGIN, B200H_SUBERR_UNSPECIFIED, m);
  }
}

// One entry per push_data2 call: libheif pushes one access unit per call -- the header NALs + the slice NALs of a still image
// (codecs/decoder.cc:441-446), one sample of a sequence track with its user_data (sequences/track_visual.cc:212-275) -- and
// expects the pictures back in order, each with the user_data it came with.  (Intra-only streams: every access unit is an
// independent picture; P/B slices are refused by the header parser.)  Parameter sets seen in earlier pushes stay valid for
// later ones (a track pushes them once): they are kept and prepended.
struct Pending { std::vector<uint8_t> au; uintptr_t user; };
struct DecInstance { std::deque<Pending> q; std::vector<uint8_t> param_sets; std::vector<uint8_t> data; int strict = 0; const b200h_security_limits* limits = nullptr; };

const char* dec_name() { return "b200 HEVC intra decoder (sm_90a CUDA kernels)"; }
void dec_init() {}
void dec_deinit();
int dec_supports(int format) { return format == B200H_COMPRESSION_HEVC ? 200 : 0; }          // libde265 reports 100, ffmpeg 90
int dec_supports2(const b200h_format_description* f) { return f ? dec_supports(f->format) : 0; }
b200h_error dec_new2(void** out, const b200h_decoder_options* o) {
  if (!api_ready()) return make_err(B200H_ERR_DECODER_PLUGIN, B200H_SUBERR_UNSPECIFIED, "libheif C API not found in the process (b200_plugin_bind_libheif)");
  DecInstance* d = new DecInstance;
  if (o) { d->strict = o->strict_decoding; d->limits = o->limits; }
  *out = d;
  return ok_err();
}
b200h_error dec_new(void** out) { return dec_new2(out, nullptr); }
void dec_free(void* p) { delete (DecInstance*)p; }
b200h_error dec_push2(void* p, const void* data, size_t n, uintptr_t user) {
  DecInstance* d = (DecInstance*)p;
  const uint8_t* b = (const uint8_t*)data;
  // same framing check as decoder_libde265.cc:322-368: 4-byte big-endian NAL sizes
  size_t pos = 0; bool has_slice = false, has_ps = false;
  std::vector<uint8_t> ps;
  while (pos < n) {
    if (n - pos < 4) return make_err(B200H_ERR_DECODER_PLUGIN, B200H_SUBERR_END_OF_DATA, "truncated NAL size");
    uint32_t len = ((uint32_t)b[pos] << 24) | (b[pos + 1] << 16) | (b[pos + 2] << 8) | b[pos + 3];
    pos += 4;
    if (len > n - pos) return make_err(B200H_ERR_DECODER_PLUGIN, B200H_SUBERR_END_OF_DATA, "NAL size exceeds the pushed data");
    if (len >= 2) {
      const int type = (b[pos] >> 1) & 0x3f;
      if (type < 32) has_slice = true;
      else if (type <= 34) { has_ps = true; ps.insert(ps.end(), b + pos - 4, b + pos + len); }
    }
    pos += len;
  }
  if (has_ps) d->param_sets = ps;                               // the most recent VPS / SPS / PPS
  if (!has_slice) return ok_err();                               // parameter sets only: nothing to decode yet
  Pending e; e.user = user;
  if (!has_ps) e.au = d->param_sets;                             // a later sample of a track: re-use the parameter sets
  e.au.insert(e.au.end(), b, b + n);
  d->q.push_back(std::move(e));
  return ok_err();
}
b200h_error dec_push(void* p, const void* data, size_t n) { return dec_push2(p, data, n, 0); }
b200h_error dec_flush(void*) { return ok_err(); }
void dec_set_strict(void* p, int f) { ((DecInstance*)p)->strict = f; }

// ---- process-wide submission queue.  libheif decodes the tiles of a grid from up to max_decoding_threads threads, one
// plugin instance and one decode_next_image2 call per tile (image-items/grid.cc:405-453, codecs/decoder.cc:538-562).  A
// 1024x1024 tile cannot fill the GPU (its CABAC wavefront exposes ~16 runnable rows) and costs a full kernel sequence, so the
// calls that are in flight at the same time are decoded as ONE batch: every caller parses its headers, allocates its
// heif_image and enqueues {access unit, destination planes}; a worker thread takes whatever has arrived within a short
// window, groups pictures of equal format, runs one batched decode per group, copies the canvas into a page-locked staging
// buffer (one DMA) and wakes the callers, which copy their own tile into their planes in parallel and return.  libheif
// creates and destroys a plugin instance per image / tile (decoder.cc:388-405), so the decoder and the staging buffer live
// here, created on the first decode, released in deinit_plugin.
struct Request {
  const uint8_t* au = nullptr; size_t size = 0; uint64_t max_pixels = 0;
  b200_image_info info{};
  uint8_t* pl[3] = {nullptr, nullptr, nullptr}; size_t st[3] = {0, 0, 0};
  int rc = 0; std::string msg;
  // filled by the worker: where this picture sits in the staging buffer
  const uint8_t* src[3] = {nullptr, nullptr, nullptr}; size_t src_st[3] = {0, 0, 0};
  int state = 0;          // 0 queued, 1 staged (caller copies), 2 failed
  int* pending_copies = nullptr;   // staged pictures of the current run whose callers have not copied yet (worker's counter, guarded by the queue mutex)
};
struct SubmitQueue {
  std::mutex mu; std::condition_variable cv_worker, cv_done;
  std::deque<Request*> q; std::thread worker; bool started = false, stop = false;
  b200_decoder* dec = nullptr; uint8_t* staging = nullptr; size_t staging_cap = 0;
  uint64_t batches = 0, pictures = 0, max_batch = 0;
  // process exit without deinit_plugin (libheif only calls it from heif_deinit): stop the idle worker, leave the CUDA
  // objects alone (the runtime may already be shutting down)
  ~SubmitQueue() {
    { std::lock_guard<std::mutex> l(mu); stop = true; }
    cv_worker.notify_all();
    if (started && worker.joinable()) worker.join();
  }
};
SubmitQueue g_sq;

// Outcome of one request as the worker computed it; published to the caller (Request::state etc.) under the queue mutex only.
struct Outcome { int state = 0; int rc = 0; std::string msg; const uint8_t* src[3] = {nullptr, nullptr, nullptr}; size_t src_st[3] = {0, 0, 0}; };
void fail(Outcome& o, int rc) { o.state = 2; o.rc = rc; o.msg = b200_last_error(); }

// decode the requests of one format group; returns false if the batch as a whole failed (the caller retries one by one)
bool decode_group(SubmitQueue& Q, std::vector<Request*>& g, std::vector<Outcome>& out) {
  const int n = (int)g.size();
  out.assign((size_t)n, Outcome());
  std::vector<const uint8_t*> au((size_t)n); std::vector<size_t> sz((size_t)n);
  uint64_t maxpx = 0;
  for (int i = 0; i < n; i++) { au[(size_t)i] = g[(size_t)i]->au; sz[(size_t)i] = g[(size_t)i]->size; maxpx = std::max(maxpx, g[(size_t)i]->max_pixels); }
  b200_image_info info;
  int rc = b200_decoder_decode_grid(Q.dec, n, 1, au.data(), sz.data(), maxpx, 0, 0, &info, nullptr);
  if (rc) { if (n == 1) fail(out[0], rc); return n == 1; }
  const int bps = info.bit_depth > 8 ? 2 : 1, mono = info.chroma == B200_CHROMA_MONO;
  const int csx = (info.chroma == B200_CHROMA_420 || info.chroma == B200_CHROMA_422) ? 1 : 0, csy = info.chroma == B200_CHROMA_420 ? 1 : 0;
  const size_t yrow = (size_t)info.width * bps, crow = mono ? 0 : (size_t)((info.width + csx) >> csx) * bps;
  const size_t ch = mono ? 0 : (size_t)((info.height + csy) >> csy);
  const size_t need = yrow * info.height + 2 * crow * ch;
  if (need > Q.staging_cap) {
    if (Q.staging) b200_host_free(Q.staging);
    Q.staging = nullptr; Q.staging_cap = 0;
    void* p = nullptr;
    if (b200_host_alloc(need + need / 4, &p)) { for (auto& o : out) fail(o, B200_E_CUDA); return true; }
    Q.staging = (uint8_t*)p; Q.staging_cap = need + need / 4;
  }
  uint8_t* sy = Q.staging; uint8_t* scb = sy + yrow * info.height; uint8_t* scr = scb + crow * ch;
  rc = b200_decoder_read_planes(Q.dec, sy, yrow, mono ? nullptr : scb, mono ? nullptr : scr, crow, nullptr);
  if (rc) { if (n == 1) fail(out[0], rc); return n == 1; }
  const int tw = info.tile_width;
  for (int i = 0; i < n; i++) {
    Outcome& o = out[(size_t)i];
    o.src[0] = sy + (size_t)i * tw * bps; o.src_st[0] = yrow;
    if (!mono) { o.src[1] = scb + (size_t)i * (tw >> csx) * bps; o.src[2] = scr + (size_t)i * (tw >> csx) * bps; o.src_st[1] = o.src_st[2] = crow; }
    o.state = 1;
  }
  return true;
}

void worker_main() {
  SubmitQueue& Q = g_sq;
  std::unique_lock<std::mutex> lk(Q.mu);
  for (;;) {
    Q.cv_worker.wait(lk, [&] { return Q.stop || !Q.q.empty(); });
    if (Q.stop) return;
    // batching window: keep collecting while callers keep arriving (150 us of silence ends it, 3 ms at most)
    const auto t0 = std::chrono::steady_clock::now();
    size_t last = Q.q.size();
    for (;;) {
      Q.cv_worker.wait_for(lk, std::chrono::microseconds(150));
      if (Q.q.size() == last || std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(3)) break;
      last = Q.q.size();
    }
    std::vector<Request*> batch(Q.q.begin(), Q.q.end());
    Q.q.clear();
    lk.unlock();
    int create_rc = 0;
    if (!Q.dec) { create_rc = b200_decoder_create(&Q.dec, 0); if (create_rc) Q.dec = nullptr; }
    // groups of equal format (decode_grid needs equal tiles; 4:2:0 tiles of a multi-picture batch must have even sizes).
    // The requests' read-only fields (au, info) may be read here; their result fields are written under the mutex only.
    std::map<std::tuple<int, int, int, int>, std::vector<Request*>> groups;
    int odd_id = 0;
    for (auto* r : batch) {
      const bool odd = r->info.chroma != B200_CHROMA_MONO && ((r->info.width | r->info.height) & 1);
      groups[std::make_tuple(r->info.width, r->info.height, r->info.bit_depth * 4 + r->info.chroma, odd ? ++odd_id : 0)].push_back(r);
    }
    for (auto& kv : groups) {
      std::vector<std::vector<Request*>> runs;
      runs.push_back(kv.second);
      for (size_t ri = 0; ri < runs.size(); ri++) {
        std::vector<Request*> run = runs[ri];
        std::vector<Outcome> out;
        if (!Q.dec) { out.assign(run.size(), Outcome()); for (auto& o : out) { o.state = 2; o.rc = create_rc; o.msg = b200_last_error(); } }
        else if (!decode_group(Q, run, out)) { for (auto* r : run) runs.push_back(std::vector<Request*>{r}); continue; }   // a bad tile must not fail its batch mates
        // publish, wake the callers, and wait until the staged ones have copied their planes out of the staging buffer.  A
        // caller's Request lives on its stack and is gone once it has returned: after the publication the worker only looks at
        // its own counter, which the callers decrement under the queue mutex.
        int pending = 0;
        lk.lock();
        for (size_t i = 0; i < run.size(); i++) {
          Request* r = run[i]; const Outcome& o = out[i];
          r->rc = o.rc; r->msg = o.msg;
          for (int c = 0; c < 3; c++) { r->src[c] = o.src[c]; r->src_st[c] = o.src_st[c]; }
          if (o.state == 1) { r->pending_copies = &pending; pending++; }
          r->state = o.state;
        }
        Q.batches++; Q.pictures += run.size(); Q.max_batch = std::max<uint64_t>(Q.max_batch, run.size());
        Q.cv_done.notify_all();
        Q.cv_done.wait(lk, [&] { return pending == 0; });
        lk.unlock();
      }
    }
    lk.lock();
  }
}

void ensure_worker() {
  SubmitQueue& Q = g_sq;
  if (!Q.started) { Q.started = true; Q.stop = false; Q.worker = std::thread(worker_main); }
}

b200h_error dec_decode2(void* p, b200h_image** out_img, uintptr_t* out_user, const b200h_security_limits* limits) {
  DecInstance* d = (DecInstance*)p;
  *out_img = nullptr;
  if (d->q.empty()) return ok_err();
  d->data.swap(d->q.front().au);
  if (out_user) *out_user = d->q.front().user;
  d->q.pop_front();
  if (!limits) limits = d->limits ? d->limits : (g_api.global_limits ? g_api.global_limits() : nullptr);
  const uint64_t maxpx = limits ? limits->max_image_size_pixels : 0;
  // 1. headers: size and format of the picture (host, microseconds); the heif_image is allocated by this thread
  Request rq;
  rq.au = d->data.data(); rq.size = d->data.size(); rq.max_pixels = maxpx;
  int rc = b200_probe_access_unit(rq.au, rq.size, maxpx, &rq.info);
  if (rc) { d->data.clear(); return from_b200(rc, false); }
  const b200_image_info info = rq.info;
  const bool mono = info.chroma == B200_CHROMA_MONO;
  b200h_image* img = nullptr;
  b200h_error err = g_api.image_create(info.width, info.height, mono ? B200H_COLORSPACE_MONOCHROME : B200H_COLORSPACE_YCBCR, info.chroma /* heif_chroma_monochrome / 420 / 422 / 444 = 0..3 (heif_image.h:77-82) */, &img);
  if (err.code) { d->data.clear(); return err; }
  const int psx = (info.chroma == B200_CHROMA_420 || info.chroma == B200_CHROMA_422) ? 1 : 0, psy = info.chroma == B200_CHROMA_420 ? 1 : 0;
  for (int c = 0; c < (mono ? 1 : 3) && !err.code; c++) {
    const int w = c ? (info.width + psx) >> psx : info.width, h = c ? (info.height + psy) >> psy : info.height;
    err = g_api.image_add_plane_safe(img, c, w, h, info.bit_depth, limits);
    if (!err.code) rq.pl[c] = g_api.image_get_plane2(img, c, &rq.st[c]);
  }
  if (err.code) { g_api.image_release(img); d->data.clear(); return err; }
  if (!mono && rq.st[1] != rq.st[2]) { g_api.image_release(img); d->data.clear(); return make_err(B200H_ERR_DECODER_PLUGIN, 0, "chroma strides differ"); }
  // 2. decode through the submission queue, batched with the other callers in flight
  {
    SubmitQueue& Q = g_sq;
    std::unique_lock<std::mutex> lk(Q.mu);
    ensure_worker();
    Q.q.push_back(&rq);
    Q.cv_worker.notify_one();
    Q.cv_done.wait(lk, [&] { return rq.state != 0; });       // block inside the call: libheif re-polls without sleeping (decoder.cc:538-562)
    lk.unlock();
    if (rq.state == 1) {
      const int bps = info.bit_depth > 8 ? 2 : 1;
      for (int c = 0; c < (mono ? 1 : 3); c++) {
        const int w = c ? (info.width + psx) >> psx : info.width, h = c ? (info.height + psy) >> psy : info.height;
        for (int y = 0; y < h; y++) memcpy(rq.pl[c] + (size_t)y * rq.st[c], rq.src[c] + (size_t)y * rq.src_st[c], (size_t)w * bps);
      }
    }
    lk.lock(); if (rq.pending_copies) --*rq.pending_copies; Q.cv_done.notify_all(); lk.unlock();
    rc = rq.state == 1 ? 0 : rq.rc;
    if (rc) b200::set_error(rc, "%s", rq.msg.c_str());
  }
  d->data.clear();
  if (rc) { g_api.image_release(img); return from_b200(rc, false); }
  void* nclx = g_api.nclx_alloc();
  if (nclx) {
    g_api.nclx_set_primaries(nclx, (uint16_t)info.colour_primaries);
    g_api.nclx_set_transfer(nclx, (uint16_t)info.transfer_characteristics);
    g_api.nclx_set_matrix(nclx, (uint16_t)info.matrix_coefficients);
    ((NclxPublic*)nclx)->full_range_flag = (uint8_t)(info.full_range ? 1 : 0);
    g_api.image_set_nclx(img, nclx);
    g_api.nclx_free(nclx);
  }
  *out_img = img;
  return ok_err();
}
void dec_deinit() {
  SubmitQueue& Q = g_sq;
  { std::lock_guard<std::mutex> l(Q.mu); Q.stop = true; }
  Q.cv_worker.notify_all();
  if (Q.started && Q.worker.joinable()) Q.worker.join();
  Q.started = false;
  if (Q.dec) { b200_decoder_destroy(Q.dec); Q.dec = nullptr; }
  if (Q.staging) { b200_host_free(Q.staging); Q.staging = nullptr; Q.staging_cap = 0; }
}
b200h_error dec_decode_next(void* p, b200h_image** out, const b200h_security_limits* l) { return dec_decode2(p, out, nullptr, l); }
b200h_error dec_decode(void* p, b200h_image** out) { return dec_decode2(p, out, nullptr, nullptr); }

const b200h_decoder_plugin g_decoder_plugin = {
    6, dec_name, dec_init, dec_deinit, dec_supports, dec_new, dec_free, dec_push, dec_decode, dec_set_strict, "b200",
    dec_decode_next, (1u << 24) | (21u << 16), dec_supports2, dec_new2, dec_push2, dec_flush, dec_decode2};

// ------------------------------------------------------------------------------------------------ encoder plugin
struct EncInstance {
  int quality = 50, lossless = 0, logging = 0, log2_ctb = 5, wpp = 1;
  std::deque<std::vector<uint8_t>> nals; std::vector<uint8_t> active;
};
const char* enc_name() { return "b200 HEVC intra encoder (host, closed loop)"; }
void enc_init() {} void enc_cleanup() {}
b200h_error enc_new(void** out) { if (!api_ready()) return make_err(B200H_ERR_ENCODER_PLUGIN, 0, "libheif C API not found in the process"); *out = new EncInstance; return ok_err(); }
void enc_free(void* p) { delete (EncInstance*)p; }
b200h_error enc_set_quality(void* p, int q) { if (q < 0 || q > 100) return make_err(B200H_ERR_USAGE, 0, "quality out of range"); ((EncInstance*)p)->quality = q; return ok_err(); }
b200h_error enc_get_quality(void* p, int* q) { *q = ((EncInstance*)p)->quality; return ok_err(); }
b200h_error enc_set_lossless(void* p, int v) { if (v) return make_err(B200H_ERR_UNSUPPORTED_FEATURE, 0, "lossless coding is not supported"); ((EncInstance*)p)->lossless = 0; return ok_err(); }
b200h_error enc_get_lossless(void* p, int* v) { *v = ((EncInstance*)p)->lossless; return ok_err(); }
b200h_error enc_set_logging(void* p, int v) { ((EncInstance*)p)->logging = v; return ok_err(); }
b200h_error enc_get_logging(void* p, int* v) { *v = ((EncInstance*)p)->logging; return ok_err(); }

b200h_encoder_parameter g_params[5];
const b200h_encoder_parameter* g_param_ptrs[6];
std::once_flag g_params_once;
void init_params() {
  memset(g_params, 0, sizeof g_params);
  auto ip = [](b200h_encoder_parameter& p, const char* n, int def, int mn, int mx) { p.version = 2; p.name = n; p.type = 1; p.integer.default_value = def; p.integer.have_minimum_maximum = 1; p.integer.minimum = mn; p.integer.maximum = mx; p.has_default = 1; };
  ip(g_params[0], "quality", 50, 0, 100);
  g_params[1].version = 2; g_params[1].name = "lossless"; g_params[1].type = 2; g_params[1].boolean.default_value = 0; g_params[1].has_default = 1;
  ip(g_params[2], "log2-ctb-size", 5, 4, 6);
  g_params[3].version = 2; g_params[3].name = "wpp"; g_params[3].type = 2; g_params[3].boolean.default_value = 1; g_params[3].has_default = 1;
  for (int i = 0; i < 4; i++) g_param_ptrs[i] = &g_params[i];
  g_param_ptrs[4] = nullptr;
}
const b200h_encoder_parameter** enc_list(void*) { std::call_once(g_params_once, init_params); return g_param_ptrs; }
b200h_error enc_set_int(void* p, const char* n, int v) {
  EncInstance* e = (EncInstance*)p;
  if (!strcmp(n, "quality")) return enc_set_quality(p, v);
  if (!strcmp(n, "lossless")) return enc_set_lossless(p, v);
  if (!strcmp(n, "log2-ctb-size")) { if (v < 4 || v > 6) return make_err(B200H_ERR_USAGE, 0, "log2-ctb-size out of range"); e->log2_ctb = v; return ok_err(); }
  if (!strcmp(n, "wpp")) { e->wpp = v ? 1 : 0; return ok_err(); }
  return make_err(B200H_ERR_USAGE, 0, "unsupported encoder parameter");
}
b200h_error enc_get_int(void* p, const char* n, int* v) {
  EncInstance* e = (EncInstance*)p;
  if (!strcmp(n, "quality")) { *v = e->quality; return ok_err(); }
  if (!strcmp(n, "lossless")) { *v = e->lossless; return ok_err(); }
  if (!strcmp(n, "log2-ctb-size")) { *v = e->log2_ctb; return ok_err(); }
  if (!strcmp(n, "wpp")) { *v = e->wpp; return ok_err(); }
  return make_err(B200H_ERR_USAGE, 0, "unsupported encoder parameter");
}
b200h_error enc_set_str(void*, const char*, const char*) { return make_err(B200H_ERR_USAGE, 0, "unsupported encoder parameter"); }
b200h_error enc_get_str(void*, const char*, char*, int) { return make_err(B200H_ERR_USAGE, 0, "unsupported encoder parameter"); }
void enc_query_cs(int* cs, int* chroma) {
  if (*cs == B200H_COLORSPACE_MONOCHROME) { *chroma = 0; return; }
  *cs = B200H_COLORSPACE_YCBCR; *chroma = 1;                       // 4:2:0 only
}
void enc_query_cs2(void*, int* cs, int* chroma) { enc_query_cs(cs, chroma); }

// what both encoder tables read from the image: size and depth, nclx, planes (the quality -> QP mapping and CTB / WPP settings
// of the instance go into the parameters)
struct EncInput { b200_hevc_enc_params prm; const uint8_t *y = nullptr, *cb = nullptr, *cr = nullptr; size_t ys = 0, cs = 0; bool mono = false; };
b200h_error read_input(const EncInstance* e, const b200h_image* image, EncInput& in) {
  const int cs = g_api.image_get_colorspace(image);
  in.mono = cs == B200H_COLORSPACE_MONOCHROME;
  if (!in.mono && (cs != B200H_COLORSPACE_YCBCR || g_api.image_get_chroma(image) != 1))
    return make_err(B200H_ERR_ENCODER_PLUGIN, B200H_SUBERR_UNSUPPORTED_IMAGE_TYPE, "input must be YCbCr 4:2:0 or monochrome");
  b200_hevc_enc_params& prm = in.prm;
  b200_hevc_enc_params_default(&prm);
  prm.width = g_api.image_get_width(image, B200H_CHANNEL_Y); prm.height = g_api.image_get_height(image, B200H_CHANNEL_Y);
  prm.bit_depth = g_api.image_get_bpp_range(image, B200H_CHANNEL_Y);
  prm.chroma_format_idc = in.mono ? 0 : 1;
  prm.log2_ctb_size = e->log2_ctb; prm.wpp = e->wpp;
  prm.qp = 51 - (e->quality * 45 + 50) / 100;                     // quality 0..100 -> QP 51..6
  prm.seed = 0xB200u;
  void* nclx = nullptr;
  if (g_api.image_get_nclx(image, &nclx).code == 0 && nclx) {
    const NclxPublic* n = (const NclxPublic*)nclx;
    prm.vui_present = 1; prm.colour_description_present = 1; prm.colour_primaries = n->color_primaries;
    prm.transfer_characteristics = n->transfer_characteristics; prm.matrix_coefficients = n->matrix_coefficients; prm.full_range = n->full_range_flag;
    g_api.nclx_free(nclx);
  }
  size_t crs = 0;
  in.y = g_api.image_get_plane_readonly2(image, B200H_CHANNEL_Y, &in.ys);
  if (!in.mono) { in.cb = g_api.image_get_plane_readonly2(image, B200H_CHANNEL_CB, &in.cs); in.cr = g_api.image_get_plane_readonly2(image, B200H_CHANNEL_CR, &crs); }
  if (!in.y || (!in.mono && (!in.cb || !in.cr || in.cs != crs))) return make_err(B200H_ERR_ENCODER_PLUGIN, 0, "missing planes");
  return ok_err();
}
void push_nals(EncInstance* e, const uint8_t* out, size_t n) {   // split the length-prefixed stream into one NAL per packet
  for (size_t pos = 0; pos + 4 <= n;) {
    uint32_t len = ((uint32_t)out[pos] << 24) | (out[pos + 1] << 16) | (out[pos + 2] << 8) | out[pos + 3];
    pos += 4;
    e->nals.emplace_back(out + pos, out + pos + len);
    pos += len;
  }
}

b200h_error enc_encode(void* p, const b200h_image* image, int /*image_class*/) {
  EncInstance* e = (EncInstance*)p;
  e->nals.clear();                                              // same instance encodes every grid tile (grid.cc:886-906)
  EncInput in;
  b200h_error err = read_input(e, image, in);
  if (err.code) return err;
  const int bd = in.prm.bit_depth;
  if (bd != 8 && bd != 10 && bd != 12) return make_err(B200H_ERR_ENCODER_PLUGIN, B200H_SUBERR_UNSUPPORTED_BIT_DEPTH, "bit depth must be 8, 10 or 12");
  uint8_t* out = nullptr; size_t n = 0;
  int rc = b200_hevc_encode_intra(&in.prm, in.y, in.cb, in.cr, in.ys, in.cs, &out, &n);
  if (rc) return from_b200(rc, true);
  push_nals(e, out, n);
  b200_free(out);
  return ok_err();
}
b200h_error enc_get_data(void* p, uint8_t** data, int* size, int*) {
  EncInstance* e = (EncInstance*)p;
  if (e->nals.empty()) { *data = nullptr; *size = 0; return ok_err(); }
  e->active = std::move(e->nals.front()); e->nals.pop_front();
  *data = e->active.data(); *size = (int)e->active.size();
  return ok_err();
}
b200h_error enc_start_seq(void*, const b200h_image*, int, uint32_t, uint32_t, const void*) { return make_err(B200H_ERR_UNSUPPORTED_FEATURE, 0, "sequence encoding is not supported (intra still pictures only)"); }
b200h_error enc_seq_frame(void*, const b200h_image*, uintptr_t) { return make_err(B200H_ERR_UNSUPPORTED_FEATURE, 0, "sequence encoding is not supported"); }
b200h_error enc_end_seq(void*) { return ok_err(); }
b200h_error enc_get_data2(void* p, uint8_t** data, int* size, uintptr_t* frame, int* key, int* more) {
  if (frame) *frame = 0; if (key) *key = 1; if (more) *more = 0;
  return enc_get_data(p, data, size, nullptr);
}

const b200h_encoder_plugin g_encoder_plugin = {
    4, B200H_COMPRESSION_HEVC, "b200", 50, 1, 0, enc_name, enc_init, enc_cleanup, enc_new, enc_free, enc_set_quality, enc_get_quality,
    enc_set_lossless, enc_get_lossless, enc_set_logging, enc_get_logging, enc_list, enc_set_int, enc_get_int, enc_set_int, enc_get_int,
    enc_set_str, enc_get_str, enc_query_cs, enc_encode, enc_get_data, enc_query_cs2, nullptr, (1u << 24) | (21u << 16),
    enc_start_seq, enc_seq_frame, enc_end_seq, enc_get_data2, 0};


// ------------------------------------------------------------------------------------------------ GPU encoder plugin
// Second table ("b200-gpu"): the same parameters and quality -> QP mapping, encoded by b200_gpu_encode_intra_host (8-bit
// 4:2:0 / 4:0:0, CTB 32 or 64, WPP always on, no SAO / sign hiding / cu_qp_delta).  The GPU encoder is created on the first
// encode of an instance, so that registering and configuring the plugin touches no device.
struct GpuEncInstance : EncInstance {
  b200_gpu_encoder* gpu = nullptr;
  ~GpuEncInstance() { if (gpu) b200_gpu_encoder_destroy(gpu); }
};
const char* genc_name() { return "b200 HEVC intra encoder (GPU)"; }
b200h_error genc_new(void** out) {
  if (!api_ready()) return make_err(B200H_ERR_ENCODER_PLUGIN, 0, "libheif C API not found in the process");
  *out = static_cast<EncInstance*>(new GpuEncInstance);
  return ok_err();
}
void genc_free(void* p) { delete static_cast<GpuEncInstance*>((EncInstance*)p); }

b200h_encoder_parameter g_gpu_params[5];
const b200h_encoder_parameter* g_gpu_param_ptrs[6];
std::once_flag g_gpu_params_once;
void init_gpu_params() {
  std::call_once(g_params_once, init_params);
  memcpy(g_gpu_params, g_params, sizeof g_params);
  g_gpu_params[2].integer.minimum = 5;                           // log2-ctb-size 5..6
  for (int i = 0; i < 4; i++) g_gpu_param_ptrs[i] = &g_gpu_params[i];
  g_gpu_param_ptrs[4] = nullptr;
}
const b200h_encoder_parameter** genc_list(void*) { std::call_once(g_gpu_params_once, init_gpu_params); return g_gpu_param_ptrs; }
b200h_error genc_set_int(void* p, const char* n, int v) {
  if (!strcmp(n, "log2-ctb-size") && (v < 5 || v > 6)) return make_err(B200H_ERR_USAGE, 0, "log2-ctb-size out of range (5..6)");
  if (!strcmp(n, "wpp") && !v) return make_err(B200H_ERR_USAGE, 0, "wpp is always on in the GPU encoder");
  return enc_set_int(p, n, v);
}

b200h_error genc_encode(void* p, const b200h_image* image, int /*image_class*/) {
  GpuEncInstance* e = static_cast<GpuEncInstance*>((EncInstance*)p);
  e->nals.clear();
  EncInput in;
  b200h_error err = read_input(e, image, in);
  if (err.code) return err;
  if (in.prm.bit_depth != 8) return make_err(B200H_ERR_ENCODER_PLUGIN, B200H_SUBERR_UNSUPPORTED_BIT_DEPTH, "the GPU encoder codes 8-bit pictures");
  in.prm.sao = 0; in.prm.sign_data_hiding = 0; in.prm.cu_qp_delta = 0; in.prm.wpp = 1;
  b200_planes pl{};
  pl.y = in.y; pl.cb = in.cb; pl.cr = in.cr; pl.y_stride = in.ys; pl.c_stride = in.cs;
  pl.width = in.prm.width; pl.height = in.prm.height; pl.chroma = in.mono ? B200_CHROMA_MONO : B200_CHROMA_420; pl.bit_depth = 8;
  if (!e->gpu) { int rc = b200_gpu_encoder_create(&e->gpu); if (rc) return from_b200(rc, true); }
  int rc = b200_gpu_encode_intra_host(e->gpu, &in.prm, 1, &pl);
  if (rc) return from_b200(rc, true);
  const uint8_t* out = nullptr; size_t n = 0;
  rc = b200_gpu_encoder_output(e->gpu, 0, &out, &n);
  if (rc) return from_b200(rc, true);
  push_nals(e, out, n);
  return ok_err();
}

const b200h_encoder_plugin g_gpu_encoder_plugin = {
    4, B200H_COMPRESSION_HEVC, "b200-gpu", 60, 1, 0, genc_name, enc_init, enc_cleanup, genc_new, genc_free, enc_set_quality, enc_get_quality,
    enc_set_lossless, enc_get_lossless, enc_set_logging, enc_get_logging, genc_list, genc_set_int, enc_get_int, genc_set_int, enc_get_int,
    enc_set_str, enc_get_str, enc_query_cs, genc_encode, enc_get_data, enc_query_cs2, nullptr, (1u << 24) | (21u << 16),
    enc_start_seq, enc_seq_frame, enc_end_seq, enc_get_data2, 0};

}  // namespace

extern "C" {
b200h_plugin_info plugin_info = {1, 1 /* heif_plugin_type_decoder */, &g_decoder_plugin, nullptr};
b200h_plugin_info b200_encoder_plugin_info = {1, 0 /* heif_plugin_type_encoder */, &g_encoder_plugin, nullptr};
const b200h_decoder_plugin* b200_get_decoder_plugin(void) { return &g_decoder_plugin; }
const b200h_encoder_plugin* b200_get_encoder_plugin(void) { return &g_encoder_plugin; }
const b200h_encoder_plugin* b200_get_gpu_encoder_plugin(void) { return &g_gpu_encoder_plugin; }
// batches / pictures / largest batch the submission queue has decoded so far (tests, bench)
void b200_plugin_queue_stats(uint64_t out3[3]) { std::lock_guard<std::mutex> l(g_sq.mu); out3[0] = g_sq.batches; out3[1] = g_sq.pictures; out3[2] = g_sq.max_batch; }
int b200_plugin_bind_libheif(void* h) { g_heif_handle = h; resolve_api(); return g_api.ok ? B200_OK : b200::set_error(B200_E_INVALID, "libheif entry points not found in the given handle"); }
}
