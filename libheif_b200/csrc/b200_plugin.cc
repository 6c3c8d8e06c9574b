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
// Read-ahead (sequence tracks): libheif keeps pushing samples while decode_next_image2 returns no picture, and calls
// flush_data at the end of a track segment (sequences/track_visual.cc:200-282).  So decode_next_image2 returns no picture
// until the group is full or flush_data was called since the last push, then decodes every queued sample as one group through
// the submission queue and hands the pictures back one per call, in push order, each with its user_data or its own error.  A
// still image is pushed, flushed and decoded in one call (codecs/decoder.cc:527-550), as before.
// A group is full at `readahead` samples (B200_SEQ_READAHEAD, 1 = decode each sample when it is asked for), at kReadaheadBytes
// of access units, or when one more picture of the size of the last one would take the group's DECODED size past
// readahead_budget(): every picture of a group is a heif_image that libheif charges to the context's max_total_memory until the
// caller has taken it, so the group stays within 1/8 of that limit (and within kReadaheadDecoded), and a picture that is
// already larger than half of it is decoded alone, as without read-ahead.  The decoded size comes from the headers of each
// pushed sample (b200_probe_access_unit, host, microseconds).
struct Pending { std::vector<uint8_t> au; uintptr_t user; size_t decoded; };
struct Decoded { b200h_image* img = nullptr; uintptr_t user = 0; int code = 0, sub = 0; std::string msg; };
constexpr int kReadaheadSamples = 32;
constexpr size_t kReadaheadBytes = size_t(64) << 20;
constexpr size_t kReadaheadDecoded = size_t(256) << 20;
int readahead_samples() {
  const char* e = getenv("B200_SEQ_READAHEAD");
  return e && atoi(e) > 0 ? atoi(e) : kReadaheadSamples;
}
// heif_security_limits up to max_total_memory (heif_security.h:37-64, version >= 2); b200h_security_limits mirrors only the
// leading members
struct SecurityLimitsV2 {
  uint8_t version; uint64_t max_image_size_pixels, max_number_of_tiles; uint32_t max_bayer_pattern_pixels, max_items, max_color_profile_size;
  uint64_t max_memory_block_size; uint32_t max_components, max_iloc_extents_per_item, max_size_entity_group, max_children_per_box;
  uint64_t max_total_memory;
};
size_t readahead_budget(const b200h_security_limits* l) {
  size_t budget = kReadaheadDecoded;
  if (l && l->version >= 2) {
    const uint64_t total = reinterpret_cast<const SecurityLimitsV2*>(l)->max_total_memory;     // 0 = no limit
    if (total) budget = std::min<size_t>(budget, (size_t)(total / 8));
  }
  return budget;
}
// bytes of the heif_image planes of a picture (0 if the headers do not parse: the sample then fails when it is decoded)
size_t decoded_bytes(const uint8_t* au, size_t n) {
  b200_image_info info;
  if (b200_probe_access_unit(au, n, 0, &info)) return 0;
  const size_t bps = info.bit_depth > 8 ? 2 : 1, y = (size_t)info.width * info.height;
  const int csx = (info.chroma == B200_CHROMA_420 || info.chroma == B200_CHROMA_422) ? 1 : 0, csy = info.chroma == B200_CHROMA_420 ? 1 : 0;
  const size_t c = info.chroma == B200_CHROMA_MONO ? 0 : 2 * (size_t)((info.width + csx) >> csx) * ((info.height + csy) >> csy);
  return (y + c) * bps;
}
struct DecInstance {
  std::deque<Pending> q; size_t q_bytes = 0, q_decoded = 0; std::vector<uint8_t> param_sets; int strict = 0; const b200h_security_limits* limits = nullptr;
  int readahead = kReadaheadSamples; bool flushed = false;
  std::deque<Decoded> ready;                                      // decoded, not yet handed out
  ~DecInstance() { for (auto& r : ready) if (r.img) g_api.image_release(r.img); }
};

const char* dec_name() { return "b200 HEVC intra decoder (sm_90a CUDA kernels)"; }
void dec_init() {}
void dec_deinit();
int dec_supports(int format) { return format == B200H_COMPRESSION_HEVC ? 200 : 0; }          // libde265 reports 100, ffmpeg 90
int dec_supports2(const b200h_format_description* f) { return f ? dec_supports(f->format) : 0; }
b200h_error dec_new2(void** out, const b200h_decoder_options* o) {
  if (!api_ready()) return make_err(B200H_ERR_DECODER_PLUGIN, B200H_SUBERR_UNSPECIFIED, "libheif C API not found in the process (b200_plugin_bind_libheif)");
  DecInstance* d = new DecInstance;
  if (o) { d->strict = o->strict_decoding; d->limits = o->limits; }
  d->readahead = readahead_samples();
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
  e.decoded = decoded_bytes(e.au.data(), e.au.size());
  d->q_bytes += e.au.size(); d->q_decoded += e.decoded;
  d->q.push_back(std::move(e));
  d->flushed = false;                                            // pushes after a flush (a repeated track) start a new window
  return ok_err();
}
b200h_error dec_push(void* p, const void* data, size_t n) { return dec_push2(p, data, n, 0); }
b200h_error dec_flush(void* p) { ((DecInstance*)p)->flushed = true; return ok_err(); }
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
    if (b200_host_alloc(need + need / 4, &p)) { if (n == 1) fail(out[0], B200_E_CUDA); return n == 1; }
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

// One queued sample on its way through the submission queue: its access unit, heif_image and request.
struct Job { std::vector<uint8_t> au; Request rq; b200h_image* img = nullptr; bool queued = false, done = false; Decoded out; };
void job_fail(Job& j, const b200h_error& e) { j.out.code = e.code; j.out.sub = e.subcode; j.out.msg = e.message ? e.message : ""; }

// 1. headers: size and format of the picture (host, microseconds); the heif_image is allocated by the calling thread
void job_prepare(Job& j, const b200h_security_limits* limits) {
  const uint64_t maxpx = limits ? limits->max_image_size_pixels : 0;
  Request& rq = j.rq;
  rq.au = j.au.data(); rq.size = j.au.size(); rq.max_pixels = maxpx;
  int rc = b200_probe_access_unit(rq.au, rq.size, maxpx, &rq.info);
  if (rc) { job_fail(j, from_b200(rc, false)); return; }
  const b200_image_info info = rq.info;
  const bool mono = info.chroma == B200_CHROMA_MONO;
  b200h_error err = g_api.image_create(info.width, info.height, mono ? B200H_COLORSPACE_MONOCHROME : B200H_COLORSPACE_YCBCR, info.chroma /* heif_chroma_monochrome / 420 / 422 / 444 = 0..3 (heif_image.h:77-82) */, &j.img);
  if (err.code) { j.img = nullptr; job_fail(j, err); return; }
  const int psx = (info.chroma == B200_CHROMA_420 || info.chroma == B200_CHROMA_422) ? 1 : 0, psy = info.chroma == B200_CHROMA_420 ? 1 : 0;
  for (int c = 0; c < (mono ? 1 : 3) && !err.code; c++) {
    const int w = c ? (info.width + psx) >> psx : info.width, h = c ? (info.height + psy) >> psy : info.height;
    err = g_api.image_add_plane_safe(j.img, c, w, h, info.bit_depth, limits);
    if (!err.code) rq.pl[c] = g_api.image_get_plane2(j.img, c, &rq.st[c]);
  }
  if (!err.code && !mono && rq.st[1] != rq.st[2]) err = make_err(B200H_ERR_DECODER_PLUGIN, 0, "chroma strides differ");
  if (err.code) { g_api.image_release(j.img); j.img = nullptr; job_fail(j, err); return; }
  j.queued = true;
}

// 3. the planes from the staging buffer into the heif_image (caller thread, without the queue mutex)
void job_copy(Job& j) {
  const Request& rq = j.rq;
  const b200_image_info& info = rq.info;
  const bool mono = info.chroma == B200_CHROMA_MONO;
  const int psx = (info.chroma == B200_CHROMA_420 || info.chroma == B200_CHROMA_422) ? 1 : 0, psy = info.chroma == B200_CHROMA_420 ? 1 : 0;
  const int bps = info.bit_depth > 8 ? 2 : 1;
  for (int c = 0; c < (mono ? 1 : 3); c++) {
    const int w = c ? (info.width + psx) >> psx : info.width, h = c ? (info.height + psy) >> psy : info.height;
    for (int y = 0; y < h; y++) memcpy(rq.pl[c] + (size_t)y * rq.st[c], rq.src[c] + (size_t)y * rq.src_st[c], (size_t)w * bps);
  }
}

// 4. the outcome: the picture with its nclx, or the error of this sample alone
void job_finish(Job& j) {
  const Request& rq = j.rq;
  if (rq.state != 1) {
    b200::set_error(rq.rc, "%s", rq.msg.c_str());
    g_api.image_release(j.img); j.img = nullptr;
    job_fail(j, from_b200(rq.rc, false));
    return;
  }
  const b200_image_info& info = rq.info;
  void* nclx = g_api.nclx_alloc();
  if (nclx) {
    g_api.nclx_set_primaries(nclx, (uint16_t)info.colour_primaries);
    g_api.nclx_set_transfer(nclx, (uint16_t)info.transfer_characteristics);
    g_api.nclx_set_matrix(nclx, (uint16_t)info.matrix_coefficients);
    ((NclxPublic*)nclx)->full_range_flag = (uint8_t)(info.full_range ? 1 : 0);
    g_api.image_set_nclx(j.img, nclx);
    g_api.nclx_free(nclx);
  }
  j.out.img = j.img;
}

// decode every queued sample of the instance as one group; the outcomes go to d->ready in push order
void decode_queued(DecInstance* d, const b200h_security_limits* limits) {
  std::vector<Job> jobs(d->q.size());
  for (size_t i = 0; i < jobs.size(); i++) { jobs[i].au.swap(d->q[i].au); jobs[i].out.user = d->q[i].user; }
  d->q.clear(); d->q_bytes = 0; d->q_decoded = 0;
  size_t waiting = 0;
  for (auto& j : jobs) { job_prepare(j, limits); waiting += j.queued; }
  // 2. decode through the submission queue, batched with each other and with the other callers in flight.  The worker
  // publishes a run's outcomes and waits until the staged ones are copied out (pending_copies), so the copies happen as runs
  // complete.
  if (waiting) {
    SubmitQueue& Q = g_sq;
    std::unique_lock<std::mutex> lk(Q.mu);
    ensure_worker();
    for (auto& j : jobs) if (j.queued) Q.q.push_back(&j.rq);
    Q.cv_worker.notify_one();
    while (waiting) {
      // block inside the call: libheif re-polls without sleeping (decoder.cc:538-562)
      Q.cv_done.wait(lk, [&] { for (auto& j : jobs) if (j.queued && !j.done && j.rq.state != 0) return true; return false; });
      std::vector<Job*> now;
      for (auto& j : jobs) if (j.queued && !j.done && j.rq.state != 0) now.push_back(&j);
      lk.unlock();
      for (Job* j : now) if (j->rq.state == 1) job_copy(*j);
      lk.lock();
      for (Job* j : now) { if (j->rq.pending_copies) --*j->rq.pending_copies; j->done = true; waiting--; }
      Q.cv_done.notify_all();
    }
  }
  for (auto& j : jobs) {
    if (j.queued) job_finish(j);
    d->ready.push_back(std::move(j.out));
  }
}

b200h_error decode_next(DecInstance* d, b200h_image** out_img, uintptr_t* out_user, const b200h_security_limits* limits, bool now) {
  *out_img = nullptr;
  if (d->ready.empty()) {
    if (d->q.empty()) return ok_err();
    if (!limits) limits = d->limits ? d->limits : (g_api.global_limits ? g_api.global_limits() : nullptr);
    const bool full = (int)d->q.size() >= d->readahead || d->q_bytes >= kReadaheadBytes ||
                      d->q_decoded + d->q.back().decoded > readahead_budget(limits);
    if (!now && !d->flushed && !full) return ok_err();           // read ahead: libheif pushes the next sample
    decode_queued(d, limits);
  }
  Decoded r = std::move(d->ready.front());
  d->ready.pop_front();
  if (out_user) *out_user = r.user;
  if (r.code) return make_err(r.code, r.sub, r.msg);
  *out_img = r.img;
  return ok_err();
}
b200h_error dec_decode2(void* p, b200h_image** out_img, uintptr_t* out_user, const b200h_security_limits* limits) {
  return decode_next((DecInstance*)p, out_img, out_user, limits, false);
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
// the pre-v5 entry points have no flush_data: they decode what was pushed at once
b200h_error dec_decode_next(void* p, b200h_image** out, const b200h_security_limits* l) { return decode_next((DecInstance*)p, out, nullptr, l, true); }
b200h_error dec_decode(void* p, b200h_image** out) { return decode_next((DecInstance*)p, out, nullptr, nullptr, true); }

const b200h_decoder_plugin g_decoder_plugin = {
    6, dec_name, dec_init, dec_deinit, dec_supports, dec_new, dec_free, dec_push, dec_decode, dec_set_strict, "b200",
    dec_decode_next, (1u << 24) | (21u << 16), dec_supports2, dec_new2, dec_push2, dec_flush, dec_decode2};

// ------------------------------------------------------------------------------------------------ encoder plugin
// Sequences (v4 members, libheif/codecs/hevc_enc.cc:118-170, sequences/track_visual.cc:362-380,564-598): all-intra.  Every
// frame is an independent IDR picture coded exactly as encode_image codes it (same read_input, parameters and quality -> QP
// mapping), so any gop_structure is met, keyframe_distance_max trivially, and keyframe_distance_min is moot (every frame is a
// keyframe).  Each access unit keeps its VPS / SPS / PPS in front of the slice; libheif puts the first ones into the hvcC and
// drops the repeats (hevc_enc.cc:213-227), so the samples hold the slice NAL alone.
// Release pacing: libheif pulls get_compressed_data2 once before and once after each encode_sequence_frame, taking at most
// one frame per pull, and stores everything pulled by one encode_sequence_frame as ONE sample (track_visual.cc:598).  So
// `coded` frames are released one per encode_sequence_frame / end_sequence_encoding call; end_sequence_encoding is called in a
// loop until a call releases nothing (track_visual.cc:366-380), so it is idempotent and releases the next frame each time.
struct SeqFrame { uintptr_t nr = 0; std::vector<uint8_t> au; };
struct EncInstance {
  int quality = 50, lossless = 0, logging = 0, log2_ctb = 5, wpp = 1;
  std::deque<std::vector<uint8_t>> nals; std::vector<uint8_t> active;
  // sequence state
  int seq_w = 0, seq_h = 0, seq_mono = 0, seq_bd = 0;             // format of the sequence's first frame (seq_w = 0: none yet)
  std::deque<SeqFrame> coded;                                      // coded, not yet released
  std::deque<std::pair<uintptr_t, size_t>> released;               // frame number and NAL count of each released frame in `nals`
  std::string seq_err; int seq_err_code = 0, seq_err_sub = 0;      // a failure inside end_sequence_encoding (libheif ignores its
                                                                   // return value): reported by the next get_compressed_data2
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

// what the host table reads and refuses for one image (the still path and the sequence frames)
b200h_error host_input(EncInstance* e, const b200h_image* image, EncInput& in) {
  b200h_error err = read_input(e, image, in);
  if (err.code) return err;
  const int bd = in.prm.bit_depth;
  if (bd != 8 && bd != 10 && bd != 12) return make_err(B200H_ERR_ENCODER_PLUGIN, B200H_SUBERR_UNSUPPORTED_BIT_DEPTH, "bit depth must be 8, 10 or 12");
  return ok_err();
}
b200h_error host_code(const EncInput& in, std::vector<uint8_t>& au) {
  uint8_t* out = nullptr; size_t n = 0;
  int rc = b200_hevc_encode_intra(&in.prm, in.y, in.cb, in.cr, in.ys, in.cs, &out, &n);
  if (rc) return from_b200(rc, true);
  au.assign(out, out + n);
  b200_free(out);
  return ok_err();
}
b200h_error enc_encode(void* p, const b200h_image* image, int /*image_class*/) {
  EncInstance* e = (EncInstance*)p;
  e->nals.clear();                                              // same instance encodes every grid tile (grid.cc:886-906)
  EncInput in; std::vector<uint8_t> au;
  b200h_error err = host_input(e, image, in);
  if (!err.code) err = host_code(in, au);
  if (err.code) return err;
  push_nals(e, au.data(), au.size());
  return ok_err();
}
b200h_error enc_get_data(void* p, uint8_t** data, int* size, int*) {
  EncInstance* e = (EncInstance*)p;
  if (e->nals.empty()) { *data = nullptr; *size = 0; return ok_err(); }
  e->active = std::move(e->nals.front()); e->nals.pop_front();
  *data = e->active.data(); *size = (int)e->active.size();
  return ok_err();
}

// ---- sequence members shared by both tables
b200h_error seq_start(EncInstance* e) {
  e->seq_w = e->seq_h = e->seq_mono = e->seq_bd = 0;           // a new sequence may start with any format
  e->seq_err.clear(); e->seq_err_code = e->seq_err_sub = 0;
  // nothing of an earlier sequence that ended without end_sequence_encoding (a refused frame, an abandoned track) may leak
  // into this one
  e->coded.clear(); e->released.clear(); e->nals.clear();
  return ok_err();
}
b200h_error enc_start_seq(void* p, const b200h_image*, int, uint32_t, uint32_t, const void*) { return seq_start((EncInstance*)p); }
// every frame of a sequence has the first frame's size, chroma and bit depth
b200h_error seq_check_format(EncInstance* e, const b200_hevc_enc_params& prm, uintptr_t nr) {
  const int mono = prm.chroma_format_idc == 0;
  if (!e->seq_w) { e->seq_w = prm.width; e->seq_h = prm.height; e->seq_mono = mono; e->seq_bd = prm.bit_depth; return ok_err(); }
  if (prm.width == e->seq_w && prm.height == e->seq_h && mono == e->seq_mono && prm.bit_depth == e->seq_bd) return ok_err();
  char m[256];
  snprintf(m, sizeof m, "sequence frame %llu is %dx%d %s %d-bit, the sequence started with %dx%d %s %d-bit frames; all frames of a sequence must have the same format",
           (unsigned long long)nr, prm.width, prm.height, mono ? "4:0:0" : "4:2:0", prm.bit_depth, e->seq_w, e->seq_h, e->seq_mono ? "4:0:0" : "4:2:0", e->seq_bd);
  return make_err(B200H_ERR_USAGE, B200H_SUBERR_UNSPECIFIED, m);
}
// make the next coded frame available to get_compressed_data2 (at most one per encode_sequence_frame / end_sequence_encoding)
void seq_release(EncInstance* e) {
  if (e->coded.empty()) return;
  SeqFrame f = std::move(e->coded.front()); e->coded.pop_front();
  const size_t before = e->nals.size();
  push_nals(e, f.au.data(), f.au.size());
  e->released.emplace_back(f.nr, e->nals.size() - before);
}
b200h_error enc_seq_frame(void* p, const b200h_image* image, uintptr_t nr) {
  EncInstance* e = (EncInstance*)p;
  EncInput in; SeqFrame f; f.nr = nr;
  b200h_error err = host_input(e, image, in);
  if (err.code) return err;
  if ((err = seq_check_format(e, in.prm, nr)).code) return err;
  if ((err = host_code(in, f.au)).code) return err;
  e->coded.push_back(std::move(f));
  seq_release(e);
  return ok_err();
}
b200h_error enc_end_seq(void* p) { seq_release((EncInstance*)p); return ok_err(); }
// one NAL per call; frame_nr = the number the frame was passed with, every frame a keyframe, more_frame_packets = 0 on the
// last NAL of a frame
b200h_error enc_get_data2(void* p, uint8_t** data, int* size, uintptr_t* frame, int* key, int* more) {
  EncInstance* e = (EncInstance*)p;
  if (key) *key = 1;
  if (frame) *frame = 0;
  if (more) *more = 0;
  if (e->seq_err_code) {
    const int code = e->seq_err_code; e->seq_err_code = 0;
    *data = nullptr; *size = 0;
    return make_err(code, e->seq_err_sub, e->seq_err);
  }
  if (e->released.empty()) return enc_get_data(p, data, size, nullptr);
  auto& r = e->released.front();
  if (frame) *frame = r.first;
  b200h_error err = enc_get_data(p, data, size, nullptr);
  if (--r.second == 0) e->released.pop_front();
  else if (more) *more = 1;
  return err;
}

const b200h_encoder_plugin g_encoder_plugin = {
    4, B200H_COMPRESSION_HEVC, "b200", 50, 1, 0, enc_name, enc_init, enc_cleanup, enc_new, enc_free, enc_set_quality, enc_get_quality,
    enc_set_lossless, enc_get_lossless, enc_set_logging, enc_get_logging, enc_list, enc_set_int, enc_get_int, enc_set_int, enc_get_int,
    enc_set_str, enc_get_str, enc_query_cs, enc_encode, enc_get_data, enc_query_cs2, nullptr, (1u << 24) | (21u << 16),
    enc_start_seq, enc_seq_frame, enc_end_seq, enc_get_data2, 1};


// ------------------------------------------------------------------------------------------------ GPU encoder plugin
// Second table ("b200-gpu"): the same parameters and quality -> QP mapping, encoded by b200_gpu_encode_intra_host (8-bit
// 4:2:0 / 4:0:0, CTB 32 or 64, WPP always on, no SAO / sign hiding / cu_qp_delta).  The GPU encoder is created on the first
// encode of an instance, so that registering and configuring the plugin touches no device.
// Sequences: frames are copied into page-locked staging owned by the instance; once `sequence-batch` frames are queued (or at
// the first end_sequence_encoding) one b200_gpu_encode_intra_host call codes them all, and the access units join `coded`.
// The GPU encoder's bytes do not depend on the batch, so every frame is coded exactly as encode_image codes it.
struct GpuEncInstance : EncInstance {
  b200_gpu_encoder* gpu = nullptr;
  int seq_batch = 0;                                              // "sequence-batch": 0 = automatic
  int batch_cap = 0;                                              // frames per GPU call for the running sequence
  b200_hevc_enc_params batch_prm{};                               // parameters of the queued frames
  std::vector<uintptr_t> pend;                                    // frame numbers of the queued frames, in staging order
  uint8_t* stage = nullptr; size_t stage_cap = 0;
  ~GpuEncInstance() { if (gpu) b200_gpu_encoder_destroy(gpu); if (stage) b200_host_free(stage); }
};
// GPU encode calls / pictures / largest call of every GpuEncInstance of the process (tests, scripts/sequence_bench.py)
std::mutex g_genc_mu;
uint64_t g_genc_calls = 0, g_genc_pictures = 0, g_genc_max = 0;
void count_gpu_call(int n) {
  std::lock_guard<std::mutex> l(g_genc_mu);
  g_genc_calls++; g_genc_pictures += (uint64_t)n; g_genc_max = std::max<uint64_t>(g_genc_max, (uint64_t)n);
}
const char* genc_name() { return "b200 HEVC intra encoder (GPU)"; }
b200h_error genc_new(void** out) {
  if (!api_ready()) return make_err(B200H_ERR_ENCODER_PLUGIN, 0, "libheif C API not found in the process");
  *out = static_cast<EncInstance*>(new GpuEncInstance);
  return ok_err();
}
void genc_free(void* p) { delete static_cast<GpuEncInstance*>((EncInstance*)p); }

b200h_encoder_parameter g_gpu_params[6];
const b200h_encoder_parameter* g_gpu_param_ptrs[7];
std::once_flag g_gpu_params_once;
constexpr int kMaxSeqBatch = 4096;
void init_gpu_params() {
  std::call_once(g_params_once, init_params);
  memset(g_gpu_params, 0, sizeof g_gpu_params);
  memcpy(g_gpu_params, g_params, sizeof g_params);
  g_gpu_params[2].integer.minimum = 5;                           // log2-ctb-size 5..6
  // frames per GPU encode call of a sequence: 0 = automatic (seq_batch_frames), 1 = frame by frame
  auto& b = g_gpu_params[4];
  b.version = 2; b.name = "sequence-batch"; b.type = 1; b.integer.default_value = 0; b.integer.have_minimum_maximum = 1;
  b.integer.minimum = 0; b.integer.maximum = kMaxSeqBatch; b.has_default = 1;
  for (int i = 0; i < 5; i++) g_gpu_param_ptrs[i] = &g_gpu_params[i];
  g_gpu_param_ptrs[5] = nullptr;
}
const b200h_encoder_parameter** genc_list(void*) { std::call_once(g_gpu_params_once, init_gpu_params); return g_gpu_param_ptrs; }
b200h_error genc_set_int(void* p, const char* n, int v) {
  if (!strcmp(n, "log2-ctb-size") && (v < 5 || v > 6)) return make_err(B200H_ERR_USAGE, 0, "log2-ctb-size out of range (5..6)");
  if (!strcmp(n, "wpp") && !v) return make_err(B200H_ERR_USAGE, 0, "wpp is always on in the GPU encoder");
  if (!strcmp(n, "sequence-batch")) {
    if (v < 0 || v > kMaxSeqBatch) return make_err(B200H_ERR_USAGE, 0, "sequence-batch out of range (0..4096)");
    static_cast<GpuEncInstance*>((EncInstance*)p)->seq_batch = v;
    return ok_err();
  }
  return enc_set_int(p, n, v);
}
b200h_error genc_get_int(void* p, const char* n, int* v) {
  if (!strcmp(n, "sequence-batch")) { *v = static_cast<GpuEncInstance*>((EncInstance*)p)->seq_batch; return ok_err(); }
  return enc_get_int(p, n, v);
}

// what the GPU table reads and refuses for one image (the still path and the sequence frames)
b200h_error gpu_input(GpuEncInstance* e, const b200h_image* image, EncInput& in) {
  b200h_error err = read_input(e, image, in);
  if (err.code) return err;
  if (in.prm.bit_depth != 8) return make_err(B200H_ERR_ENCODER_PLUGIN, B200H_SUBERR_UNSUPPORTED_BIT_DEPTH, "the GPU encoder codes 8-bit pictures");
  in.prm.sao = 0; in.prm.sign_data_hiding = 0; in.prm.cu_qp_delta = 0; in.prm.wpp = 1;
  return ok_err();
}
b200h_error gpu_code(GpuEncInstance* e, const b200_hevc_enc_params& prm, int n, const b200_planes* pl) {
  if (!e->gpu) { int rc = b200_gpu_encoder_create(&e->gpu); if (rc) return from_b200(rc, true); }
  int rc = b200_gpu_encode_intra_host(e->gpu, &prm, n, pl);
  if (rc) return from_b200(rc, true);
  count_gpu_call(n);
  return ok_err();
}

b200h_error genc_encode(void* p, const b200h_image* image, int /*image_class*/) {
  GpuEncInstance* e = static_cast<GpuEncInstance*>((EncInstance*)p);
  e->nals.clear();
  EncInput in;
  b200h_error err = gpu_input(e, image, in);
  if (err.code) return err;
  b200_planes pl{};
  pl.y = in.y; pl.cb = in.cb; pl.cr = in.cr; pl.y_stride = in.ys; pl.c_stride = in.cs;
  pl.width = in.prm.width; pl.height = in.prm.height; pl.chroma = in.mono ? B200_CHROMA_MONO : B200_CHROMA_420; pl.bit_depth = 8;
  if ((err = gpu_code(e, in.prm, 1, &pl)).code) return err;
  const uint8_t* out = nullptr; size_t n = 0;
  int rc = b200_gpu_encoder_output(e->gpu, 0, &out, &n);
  if (rc) return from_b200(rc, true);
  push_nals(e, out, n);
  return ok_err();
}

// ---- GPU sequences
// Staging bytes of one queued frame: Y, then Cb and Cr, each packed at its width.
size_t frame_bytes(int w, int h, bool mono) { return (size_t)w * h + (mono ? 0 : 2 * (size_t)((w + 1) >> 1) * ((h + 1) >> 1)); }
// Automatic batch: enough frames for about one full wave of E1 (one warp per picture CTB row; 6 resident E1 warps per SM, set by
// its 33460 bytes of static shared memory per warp), capped so that the staging stays within kSeqStagingBudget.
constexpr int kE1WarpsPerSm = 6;
constexpr size_t kSeqStagingBudget = size_t(256) << 20;
int seq_batch_frames(const GpuEncInstance* e, const b200_hevc_enc_params& prm) {
  const size_t fb = frame_bytes(prm.width, prm.height, prm.chroma_format_idc == 0);
  const int budget = (int)std::max<size_t>(1, std::min<size_t>(kMaxSeqBatch, kSeqStagingBudget / fb));
  if (e->seq_batch > 0) return std::min(e->seq_batch, budget);
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) {
    cudaGetLastError();
    sms = 132;                                                    // H100 SXM; the encode call reports a missing device
  }
  const int ctb = 1 << prm.log2_ctb_size, rows = (((prm.height + 7) & ~7) + ctb - 1) / ctb;
  return std::max(1, std::min(budget, sms * kE1WarpsPerSm / rows));
}
// code the queued frames in one GPU call; their access units join `coded` in frame order
b200h_error gpu_flush(GpuEncInstance* e) {
  const int n = (int)e->pend.size();
  if (!n) return ok_err();
  const b200_hevc_enc_params& prm = e->batch_prm;
  const int w = prm.width, h = prm.height, cw = (w + 1) >> 1, ch = (h + 1) >> 1;
  const bool mono = prm.chroma_format_idc == 0;
  const size_t fb = frame_bytes(w, h, mono);
  std::vector<b200_planes> pl((size_t)n);
  for (int i = 0; i < n; i++) {
    b200_planes& q = pl[(size_t)i];
    const uint8_t* base = e->stage + (size_t)i * fb;
    q.y = base; q.y_stride = (size_t)w;
    if (!mono) { q.cb = base + (size_t)w * h; q.cr = base + (size_t)w * h + (size_t)cw * ch; q.c_stride = (size_t)cw; }
    q.width = w; q.height = h; q.chroma = mono ? B200_CHROMA_MONO : B200_CHROMA_420; q.bit_depth = 8;
  }
  std::vector<uintptr_t> nrs; nrs.swap(e->pend);
  b200h_error err = gpu_code(e, prm, n, pl.data());
  if (err.code) return err;
  for (int i = 0; i < n; i++) {
    const uint8_t* out = nullptr; size_t sz = 0;
    int rc = b200_gpu_encoder_output(e->gpu, i, &out, &sz);
    if (rc) return from_b200(rc, true);
    SeqFrame f; f.nr = nrs[(size_t)i]; f.au.assign(out, out + sz);
    e->coded.push_back(std::move(f));
  }
  return ok_err();
}
b200h_error genc_start_seq(void* p, const b200h_image*, int, uint32_t, uint32_t, const void*) {
  GpuEncInstance* e = static_cast<GpuEncInstance*>((EncInstance*)p);
  e->batch_cap = 0;
  e->pend.clear();                                               // frames staged by an earlier, unfinished sequence
  return seq_start(e);
}
b200h_error genc_seq_frame(void* p, const b200h_image* image, uintptr_t nr) {
  GpuEncInstance* e = static_cast<GpuEncInstance*>((EncInstance*)p);
  EncInput in;
  b200h_error err = gpu_input(e, image, in);
  if (err.code) return err;
  if ((err = seq_check_format(e, in.prm, nr)).code) return err;
  // the encode call's argument check, so that a frame it would refuse fails here and not inside a later batch
  b200_planes chk{};
  chk.y = in.y; chk.cb = in.cb; chk.cr = in.cr; chk.y_stride = in.ys; chk.c_stride = in.cs;
  chk.width = in.prm.width; chk.height = in.prm.height; chk.chroma = in.mono ? B200_CHROMA_MONO : B200_CHROMA_420; chk.bit_depth = 8;
  if (int rc = b200_gpu_encode_check(&in.prm, 1, &chk)) return from_b200(rc, true);
  // frames whose parameters differ (quality changed, another nclx) go into a call of their own
  if (!e->pend.empty() && memcmp(&in.prm, &e->batch_prm, sizeof in.prm)) { if ((err = gpu_flush(e)).code) return err; }
  if (!e->batch_cap) {
    e->batch_cap = seq_batch_frames(e, in.prm);
    const size_t need = (size_t)e->batch_cap * frame_bytes(in.prm.width, in.prm.height, in.mono);
    if (need > e->stage_cap) {
      if (e->stage) b200_host_free(e->stage);
      e->stage = nullptr; e->stage_cap = 0;
      void* s = nullptr;
      if (int rc = b200_host_alloc(need, &s)) return from_b200(rc, true);
      e->stage = (uint8_t*)s; e->stage_cap = need;
    }
  }
  e->batch_prm = in.prm;
  const int w = in.prm.width, h = in.prm.height, cw = (w + 1) >> 1, ch = (h + 1) >> 1;
  uint8_t* d = e->stage + e->pend.size() * frame_bytes(w, h, in.mono);
  for (int y = 0; y < h; y++) memcpy(d + (size_t)y * w, in.y + (size_t)y * in.ys, (size_t)w);
  if (!in.mono) {
    uint8_t* dcb = d + (size_t)w * h; uint8_t* dcr = dcb + (size_t)cw * ch;
    for (int y = 0; y < ch; y++) { memcpy(dcb + (size_t)y * cw, in.cb + (size_t)y * in.cs, (size_t)cw); memcpy(dcr + (size_t)y * cw, in.cr + (size_t)y * in.cs, (size_t)cw); }
  }
  e->pend.push_back(nr);
  if ((int)e->pend.size() >= e->batch_cap && (err = gpu_flush(e)).code) return err;
  seq_release(e);
  return ok_err();
}
b200h_error genc_end_seq(void* p) {
  GpuEncInstance* e = static_cast<GpuEncInstance*>((EncInstance*)p);
  b200h_error err = gpu_flush(e);
  if (err.code) { e->seq_err = err.message ? err.message : ""; e->seq_err_code = err.code; e->seq_err_sub = err.subcode; return err; }
  seq_release(e);
  return ok_err();
}

const b200h_encoder_plugin g_gpu_encoder_plugin = {
    4, B200H_COMPRESSION_HEVC, "b200-gpu", 60, 1, 0, genc_name, enc_init, enc_cleanup, genc_new, genc_free, enc_set_quality, enc_get_quality,
    enc_set_lossless, enc_get_lossless, enc_set_logging, enc_get_logging, genc_list, genc_set_int, genc_get_int, genc_set_int, genc_get_int,
    enc_set_str, enc_get_str, enc_query_cs, genc_encode, enc_get_data, enc_query_cs2, nullptr, (1u << 24) | (21u << 16),
    genc_start_seq, genc_seq_frame, genc_end_seq, enc_get_data2, 1};

}  // namespace

extern "C" {
b200h_plugin_info plugin_info = {1, 1 /* heif_plugin_type_decoder */, &g_decoder_plugin, nullptr};
b200h_plugin_info b200_encoder_plugin_info = {1, 0 /* heif_plugin_type_encoder */, &g_encoder_plugin, nullptr};
const b200h_decoder_plugin* b200_get_decoder_plugin(void) { return &g_decoder_plugin; }
const b200h_encoder_plugin* b200_get_encoder_plugin(void) { return &g_encoder_plugin; }
const b200h_encoder_plugin* b200_get_gpu_encoder_plugin(void) { return &g_gpu_encoder_plugin; }
// batches / pictures / largest batch the submission queue has decoded so far (tests, bench)
void b200_plugin_queue_stats(uint64_t out3[3]) { std::lock_guard<std::mutex> l(g_sq.mu); out3[0] = g_sq.batches; out3[1] = g_sq.pictures; out3[2] = g_sq.max_batch; }
// GPU encode calls / pictures / largest call of the "b200-gpu" encoder instances so far (tests, bench)
void b200_plugin_encoder_stats(uint64_t out3[3]) { std::lock_guard<std::mutex> l(g_genc_mu); out3[0] = g_genc_calls; out3[1] = g_genc_pictures; out3[2] = g_genc_max; }
int b200_plugin_bind_libheif(void* h) { g_heif_handle = h; resolve_api(); return g_api.ok ? B200_OK : b200::set_error(B200_E_INVALID, "libheif entry points not found in the given handle"); }
}
