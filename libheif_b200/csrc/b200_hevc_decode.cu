// b200_hevc_decode.cu -- decoder object behind the C ABI: header parsing on host threads (one tile per task), staging
// into pinned memory, one H2D per array, then the entropy (K0) / reconstruction (K1) / deblocking / SAO kernels for the
// whole batch of tiles.  With the host front-end the same threads also run the CABAC syntax decoder.
//
// Mirrors the call order libheif uses on a decoder plugin instance (new_decoder2 -> push_data2 -> flush_data ->
// decode_next_image2 -> free_decoder, libheif/codecs/decoder.cc:388-405,441-446,458-460,487-493), but for N
// independent tiles at once, which is how ImageItem_Grid::decode_full_grid_image (libheif/image-items/grid.cc:250-468)
// consumes it.  All expensive state (device arenas, pinned staging, streams, events) lives here and is reused.
#include "b200_hevc.h"
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <unistd.h>

using namespace b200;

namespace {

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// minimal persistent thread pool: parallel_for over [0, n)
class Pool {
 public:
  explicit Pool(int n) : stop_(false), gen_(0), next_(0), total_(0), pending_(0) { for (int i = 0; i < n; i++) th_.emplace_back([this] { run(); }); }
  ~Pool() { { std::lock_guard<std::mutex> l(mu_); stop_ = true; } cv_.notify_all(); for (auto& t : th_) t.join(); }
  void parallel_for(int n, const std::function<void(int)>& fn) {
    if (n <= 0) return;
    if (th_.empty() || n == 1) { for (int i = 0; i < n; i++) fn(i); return; }
    { std::lock_guard<std::mutex> l(mu_); fn_ = &fn; total_ = n; next_.store(0); pending_ = (int)th_.size(); gen_++; }
    cv_.notify_all();
    std::unique_lock<std::mutex> l(mu_);
    done_.wait(l, [this] { return pending_ == 0; });
  }
 private:
  void run() {
    unsigned seen = 0;
    for (;;) {
      const std::function<void(int)>* fn; int total;
      { std::unique_lock<std::mutex> l(mu_); cv_.wait(l, [&] { return stop_ || gen_ != seen; }); if (stop_) return; seen = gen_; fn = fn_; total = total_; }
      for (;;) { int i = next_.fetch_add(1); if (i >= total) break; (*fn)(i); }
      { std::lock_guard<std::mutex> l(mu_); if (--pending_ == 0) done_.notify_all(); }
    }
  }
  std::vector<std::thread> th_; std::mutex mu_; std::condition_variable cv_, done_;
  bool stop_; unsigned gen_; std::atomic<int> next_; int total_, pending_; const std::function<void(int)>* fn_ = nullptr;
};

template <typename T>
struct DevBuf {   // grow-only device buffer with optional pinned host staging of the same capacity
  T* d = nullptr; T* h = nullptr; size_t cap = 0, hcap = 0;
  int reserve(size_t n, bool host = true) {
    if (n > cap) {
      const size_t nc = n + n / 4 + 1024;
      if (d) cudaFree(d);
      d = nullptr; cap = 0;
      B200_CUDA_CHECK(cudaMalloc(&d, nc * sizeof(T)));
      cap = nc;
    }
    if (host && n > hcap) {
      if (h) cudaFreeHost(h);
      h = nullptr; hcap = 0;
      B200_CUDA_CHECK(cudaMallocHost(&h, cap * sizeof(T)));
      hcap = cap;
    }
    return B200_OK;
  }
  void release() { if (d) cudaFree(d); if (h) cudaFreeHost(h); d = nullptr; h = nullptr; cap = hcap = 0; }
};

}  // namespace

struct b200_decoder {
  Pool* pool = nullptr;
  std::vector<ParsedPicture> parsed;
  std::vector<int> parse_rc; std::vector<std::string> parse_msg;
  DevBuf<PicDesc> pics; DevBuf<CtuInfo> ctus; DevBuf<TuCmd> tus; DevBuf<CoefEntry> coefs; DevBuf<SliceInfo> slices;
  DevBuf<int8_t> qp8; DevBuf<uint8_t> edge8; DevBuf<uint8_t> scaling; DevBuf<uint2> rows; DevBuf<unsigned> sync;   // sync: [0] ticket, [1] error flag, [2..] progress
  DevBuf<uint8_t> rec; DevBuf<uint8_t> canvas; DevBuf<uint8_t> rgb2[2]; DevBuf<uint8_t> bounce;   // fused host entry points: two RGB buffers (D2H of one overlaps the kernels writing the other)
  cudaStream_t own = nullptr, copy = nullptr; cudaEvent_t ev_band[2] = {nullptr, nullptr}, ev_k6[2] = {nullptr, nullptr}, ev_d2h[2] = {nullptr, nullptr};
  unsigned* err_host = nullptr; int async_slot = 0; bool async_error = false;
  // device front-end (entropy decoding on the GPU)
  DevBuf<uint8_t> rbsp; DevBuf<syn::Substream> subs; DevBuf<unsigned> equeue; DevBuf<uint16_t> ctu_slice; DevBuf<EntropyPic> epics;
  DevBuf<uint8_t> ipm4, cd8, wpp_ctx, end_state; DevBuf<unsigned> esync; DevBuf<unsigned long long> ecount;
  int front_end = 1;               // 1 = CABAC on the GPU (default), 0 = CABAC on the host cores
  bool used_device_front_end = false; size_t n_subs = 0;
  size_t canvas_off[3] = {0, 0, 0}; size_t canvas_pitch[3] = {0, 0, 0};
  b200_image_info info{};
  b200_decode_stats stats{};
  std::vector<size_t> rec_off; int npics = 0;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // 0 start, 1 after H2D, 5 after entropy, 2 after recon, 3 after deblock, 4 after SAO
  cudaStream_t last_stream = nullptr;
  cudaStream_t side = nullptr;     // K0 runs here, concurrently with K1 on the caller's stream
  bool last_overlapped = false;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool have_result = false;
  int debug_stage = 0;
  size_t n_rows = 0, n_items = 0, cbytes = 0; bool canvas_fully_covered = true; int max_log2_ctb = 6, info_bps = 1;
  // Band pipeline of the fused host entry points (large grids): after K0, the tile rows go through K1 -> K3 -> K4 -> K6 in
  // bands (chunks), and the D2H of band c (copy stream, chunk_hook) overlaps the kernels of band c + 1.
  int nchunks = 1, grid_cols = 1; bool last_chunked = false;
  int chunk_pic[MAX_CHUNKS + 1] = {0}; size_t chunk_item[MAX_CHUNKS + 1] = {0};
  std::function<int(int, cudaStream_t)> chunk_hook;   // queued after K4 of band c on the decode stream
  cudaEvent_t ev_chunk[MAX_CHUNKS] = {nullptr};
  ~b200_decoder() {
    delete pool;
    pics.release(); ctus.release(); tus.release(); coefs.release(); slices.release(); qp8.release(); edge8.release(); scaling.release(); rows.release();
    sync.release(); rec.release(); canvas.release(); rgb2[0].release(); rgb2[1].release(); bounce.release();
    if (own) cudaStreamDestroy(own);
    if (copy) cudaStreamDestroy(copy);
    for (auto& e : ev_band) if (e) cudaEventDestroy(e);
    for (auto& e : ev_k6) if (e) cudaEventDestroy(e);
    for (auto& e : ev_d2h) if (e) cudaEventDestroy(e);
    if (err_host) cudaFreeHost(err_host);
    rbsp.release(); subs.release(); equeue.release(); ctu_slice.release(); epics.release(); ipm4.release(); cd8.release(); wpp_ctx.release();
    end_state.release(); esync.release(); ecount.release();
    for (auto& e : ev) if (e) cudaEventDestroy(e);
    if (ev_fork) cudaEventDestroy(ev_fork);
    if (ev_join) cudaEventDestroy(ev_join);
    if (side) cudaStreamDestroy(side);
    for (auto& e : ev_chunk) if (e) cudaEventDestroy(e);
  }
};

static int check_device_error(b200_decoder* d) {
  unsigned flag = 0;
  B200_CUDA_CHECK(cudaMemcpy(&flag, d->sync.d + 1, sizeof flag, cudaMemcpyDeviceToHost));
  if (flag) return set_error(B200_E_CUDA, "reconstruction kernel gave up waiting for a CTB row dependency");
  return B200_OK;
}

// K0 (entropy) and K1 (reconstruction) can run CONCURRENTLY: K1 consumes the command stream CTB by CTB as K0 publishes
// it.  Both kernels are persistent and ticket-driven, so they need not be fully co-resident (whatever part of either
// grid is resident finishes the work); the caps below only share the SM's registers between them.
// The overlap hides K1 completely while the batch is critical-path bound -- up to about one wave of sub-streams -- and
// LOSES once the GPU is throughput bound (the two instruction streams evict each other), so it is chosen
// per batch.  B200_OVERLAP=0/1 forces it.
static int overlap_blocks(const char* env, int dflt) { if (const char* e = getenv(env)) { const int v = atoi(e); if (v >= 1 && v <= 4) return v; } return dflt; }
// At most ONE overlapped K0/K1 pair is in flight per process: libheif drives many decoder instances from its own threads,
// and the spinning K1 grids of many instances must never be able to keep all their K0 grids off the GPU.  A batch that
// finds the slot taken simply runs its kernels back to back.
// (Successive batches of the SAME decoder are ordered by its stream and may all overlap.)
static std::mutex g_overlap_mutex;
static const void* g_overlap_owner = nullptr;
static int g_overlap_count = 0;
static bool overlap_acquire(const void* who) {
  std::lock_guard<std::mutex> lk(g_overlap_mutex);
  if (g_overlap_owner && g_overlap_owner != who) return false;
  g_overlap_owner = who; g_overlap_count++;
  return true;
}
static void overlap_release() {
  std::lock_guard<std::mutex> lk(g_overlap_mutex);
  if (g_overlap_count > 0 && --g_overlap_count == 0) g_overlap_owner = nullptr;
}
static void CUDART_CB overlap_done(void*) { overlap_release(); }

static bool use_overlap(size_t n_subs) {
  if (const char* e = getenv("B200_OVERLAP")) return atoi(e) != 0;
  int dev = 0, sms = 148; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return n_subs <= (size_t)sms * 16;      // one wave of K0: 4 CTAs x 4 warps per SM
}
// TAIL overlap, for batches of more than one wave: K0 keeps the whole GPU (4 CTAs per SM, launched first) and the LIVE K1
// is queued behind it on the other stream, so K1's CTAs become resident only where K0's persistent CTAs have left -- which
// they do over the last ~30 % of K0's run time, once every sub-stream has been handed out and the wavefronts of the tiles
// drain.  K1 (and, with bands, K3 / K4 / K6 / D2H of the first band) then runs in SM slots that would otherwise idle.
// B200_TAIL_OVERLAP=0 switches it off; 1 (default): with row bands, one live K1 per band (the first band's K1 ends with K0, its
// filters / K6 / D2H overlap the second band's K1); 2: ONE live K1 over the whole grid, bands only for K3 / K4 / K6 / D2H
// (slower end to end: nothing is left to overlap the first band's D2H).
static int use_tail_overlap() {
  if (const char* e = getenv("B200_TAIL_OVERLAP")) return atoi(e);
  return 1;
}

// Device half: K0 entropy decoding (device front-end only) on the side stream, concurrently K1 reconstruction on `s`
// consuming the command stream CTB by CTB as K0 publishes it, then deblocking and SAO / paste on `s`.
static int run_device_pipeline(b200_decoder* d, int n, cudaStream_t s, int* launches_out) {
  int rc;
  int launches = 0;
  const bool devfe = d->used_device_front_end;
  // bands only pay for the caller that takes them one by one (the synchronous fused entry point); everything else -- the
  // composition API, b200_decoder_rerun_device, the asynchronous entry point whose D2H already overlaps the next picture --
  // runs one launch per kernel (the band-major row list is a valid ticket order for that, too)
  const char* force = getenv("B200_CHUNKS");
  const bool chunked = d->nchunks > 1 && (d->chunk_hook || (force && atoi(force) != 0));
  bool overlap = devfe && !chunked && use_overlap(d->n_subs);
  const int tail_mode = use_tail_overlap();
  const bool tail = devfe && !getenv("B200_OVERLAP") && tail_mode != 0 && (!overlap || getenv("B200_TAIL_FORCE"));   // B200_TAIL_FORCE: small batches too (tests)
  if (tail) overlap = true;
  // K1 follows K0 through per-row progress counters in raster order; sub-streams of HEVC tiles produce CTBs tile by tile
  for (int i = 0; i < d->npics && overlap; i++) if (d->epics.h[i].sp.tiles) overlap = false;
  if (overlap) overlap = overlap_acquire(d);
  struct Release { bool armed; ~Release() { if (armed) overlap_release(); } } release{overlap};   // error paths
  d->last_overlapped = overlap; d->last_chunked = chunked;
  cudaEventRecord(d->ev[1], s);
  DeviceBatch b{};
  b.pics = d->pics.d; b.npics = n; b.ctus = d->ctus.d; b.tus = d->tus.d; b.coefs = d->coefs.d; b.slices = d->slices.d;
  b.qp8 = d->qp8.d; b.edge8 = d->edge8.d; b.scaling = d->scaling.d; b.ticket = d->sync.d + 2 + 3 * d->n_rows; b.error_flag = d->sync.d + 1; b.progress = d->sync.d + 2; b.row_list = d->rows.d; b.nrows = (int)d->n_items; b.max_log2_ctb = d->max_log2_ctb; b.wide_samples = d->info_bps == 2;
  if (devfe) {
    EntropyBatch e{};
    e.pics = d->epics.d; e.npics = d->npics; e.subs = d->subs.d; e.nsubs = (int)d->n_subs;
    e.qhead = d->equeue.d; e.qtail = d->equeue.d + 1; e.queue = d->equeue.d + 2; e.deps = d->equeue.d + 2 + d->n_subs;
    e.progress = d->esync.d + 1; e.sub_done = d->esync.d + 1 + d->n_rows; e.error_flag = d->sync.d + 1;
    e.common = 1;
    if (getenv("B200_ENTROPY_GENERIC")) e.common = 0;
    for (int i = 0; i < d->npics && e.common; i++) if (!syn::matches_common(d->epics.h[i].sp)) e.common = 0;
    if (overlap) {
      if (!d->side) { B200_CUDA_CHECK(cudaStreamCreateWithFlags(&d->side, cudaStreamNonBlocking)); B200_CUDA_CHECK(cudaEventCreate(&d->ev_fork)); B200_CUDA_CHECK(cudaEventCreate(&d->ev_join)); }
      e.blocks_per_sm = tail ? 0 : overlap_blocks("B200_OVERLAP_K0_BLOCKS", 3);
      b.blocks_per_sm = tail ? 0 : overlap_blocks("B200_OVERLAP_K1_BLOCKS", 2);
      b.entropy_progress = e.progress;
      cudaEventRecord(d->ev_fork, s);
      B200_CUDA_CHECK(cudaStreamWaitEvent(d->side, d->ev_fork, 0));
      int k0_warps = 0;
      if ((rc = launch_entropy(e, d->side, &k0_warps))) return rc;
      cudaEventRecord(d->ev[5], d->side);
      if ((rc = launch_entropy_stats(e, d->ecount.d, d->side))) return rc;
      cudaEventRecord(d->ev_join, d->side);
      if (tail) { if ((rc = launch_entropy_gate(e, k0_warps, s))) return rc; launches += 1; }   // K1 (next on s) must not take the SMs before K0 has them
    } else {
      if ((rc = launch_entropy(e, s))) return rc;
      cudaEventRecord(d->ev[5], s);
      if ((rc = launch_entropy_stats(e, d->ecount.d, s))) return rc;
    }
    launches += 1;
  } else cudaEventRecord(d->ev[5], s);
  if (chunked) {
    // Row bands of a large grid leave the pipeline one after the other: K1 -> K3 -> K4 of band c, then the caller's hook
    // (K6 of the band + its D2H on the copy stream, which overlaps the kernels of band c + 1).  K0 is NOT part of this:
    // letting the bands leave K0 in order (priority queues) and running these kernels beside it was measured slower --
    // K0 loses more from the co-residency (3 instead of 4 CTAs per SM) and the priorities than the overlap gains.
    const bool one_k1 = overlap && tail_mode == 2;
    if (one_k1) { if ((rc = launch_recon(b, s))) return rc; launches += 1; }   // the band-major row list is a valid ticket order for one launch
    for (int c = 0; c < d->nchunks; c++) {
      DeviceBatch bc = b;
      bc.row_list = d->rows.d + d->chunk_item[c]; bc.nrows = (int)(d->chunk_item[c + 1] - d->chunk_item[c]); bc.ticket = b.ticket + c;
      if (!one_k1 && (rc = launch_recon(bc, s))) return rc;
      if (overlap && (one_k1 ? c == 0 : c + 1 == d->nchunks)) {   // (tail overlap) K0 has finished before anything that follows the last K1
        B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_join, 0));
        B200_CUDA_CHECK(cudaLaunchHostFunc(s, overlap_done, nullptr));
        release.armed = false;
      }
      DeviceBatch bf = b;
      const int p0 = d->chunk_pic[c];
      bf.pics = d->pics.d + p0; bf.npics = d->chunk_pic[c + 1] - p0;
      if (d->debug_stage != 1 && (rc = launch_deblock(bf, d->pics.h + p0, s))) return rc;
      int nsao = 0;
      if (d->debug_stage == 0 && (rc = launch_sao(bf, d->pics.h + p0, s, &nsao))) return rc;
      launches += 3 + nsao;
      if (d->chunk_hook && (rc = d->chunk_hook(c, s))) return rc;
    }
    cudaEventRecord(d->ev[2], s); cudaEventRecord(d->ev[3], s); cudaEventRecord(d->ev[4], s);   // recon_ms = the whole band pipeline (incl. the hooks' K6)
    if (launches_out) *launches_out = launches;
    return B200_OK;
  }
  if ((rc = launch_recon(b, s))) return rc;
  if (devfe && overlap) {
    B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_join, 0));
    B200_CUDA_CHECK(cudaLaunchHostFunc(s, overlap_done, nullptr));   // the slot is free once K0 and K1 have both finished
    release.armed = false;
  }
  cudaEventRecord(d->ev[2], s);
  launches += 1;
  if (d->debug_stage != 1) { if ((rc = launch_deblock(b, d->pics.h, s))) return rc; launches += 2; }
  cudaEventRecord(d->ev[3], s);
  if (d->debug_stage == 0) { int nsao = 0; if ((rc = launch_sao(b, d->pics.h, s, &nsao))) return rc; launches += nsao; }
  cudaEventRecord(d->ev[4], s);
  if (launches_out) *launches_out = launches;
  return B200_OK;
}

extern "C" {

int b200_decoder_create(b200_decoder** out, int host_threads) {
  if (!out) return set_error(B200_E_INVALID, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_error(B200_E_CUDA, "no CUDA device: libb200heif has no CPU fallback");
  if (host_threads <= 0) { long n = sysconf(_SC_NPROCESSORS_ONLN); host_threads = n > 0 ? (int)n : 1; }
  b200_decoder* d = new b200_decoder;
  d->pool = new Pool(host_threads);
  for (auto& e : d->ev) if (cudaEventCreate(&e) != cudaSuccess) { delete d; return set_error(B200_E_CUDA, "cudaEventCreate failed"); }
  *out = d;
  return B200_OK;
}

void b200_decoder_destroy(b200_decoder* d) { delete d; }

int b200_decoder_set_debug_stage(b200_decoder* d, int stage) { if (!d) return B200_E_INVALID; d->debug_stage = stage; return B200_OK; }

int b200_decoder_set_front_end(b200_decoder* d, int device) { if (!d) return B200_E_INVALID; d->front_end = device ? 1 : 0; return B200_OK; }

int b200_decoder_decode_grid(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                             uint64_t max_pixels, int canvas_w, int canvas_h, b200_image_info* info, void* stream_) {
  if (!d || !au || !au_size || cols <= 0 || rows <= 0) return set_error(B200_E_INVALID, "bad argument");
  cudaStream_t s = (cudaStream_t)stream_;
  const int n = cols * rows;
  const double t0 = now_ms();
  const bool devfe = d->front_end != 0;
  d->have_result = false;
  d->parsed.resize((size_t)n); d->parse_rc.assign((size_t)n, 0); d->parse_msg.assign((size_t)n, std::string());
  ParseLimits lim; lim.max_image_size_pixels = max_pixels;
  // ---- 1. host stage, one tile per task.  Host front-end: headers + CABAC + syntax (serial per sub-stream).
  //         Device front-end: headers only (NAL split, emulation prevention removal, parameter sets, entry points).
  d->pool->parallel_for(n, [&](int i) {
    ParsedPicture& pp = d->parsed[(size_t)i];
    int rc = devfe ? parse_headers(au[i], au_size[i], lim, pp.hdr) : parse_access_unit(au[i], au_size[i], lim, pp);
    if (!rc && devfe) pp.desc = pp.hdr.desc;
    d->parse_rc[(size_t)i] = rc;
    if (rc) d->parse_msg[(size_t)i] = b200_last_error();
  });
  for (int i = 0; i < n; i++) if (d->parse_rc[(size_t)i]) return set_error(d->parse_rc[(size_t)i], "tile %d: %s", i, d->parse_msg[(size_t)i].c_str());
  const double t1 = now_ms();
  // ---- 2. layout
  const PicDesc& p0 = d->parsed[0].desc;
  const int tw = p0.out_w, th = p0.out_h, bd = p0.bit_depth, chroma = p0.chroma, bps = bd > 8 ? 2 : 1;
  for (int i = 1; i < n; i++) {
    const PicDesc& p = d->parsed[(size_t)i].desc;
    if (p.out_w != tw || p.out_h != th || p.bit_depth != bd || p.chroma != chroma)
      return set_error(B200_E_UNSUPPORTED, "grid tiles differ in size or format (tile %d)", i);   // grid.cc:261-375 requires equal tiles
  }
  const int csx = (chroma == 1 || chroma == 2) ? 1 : 0, csy = chroma == 1 ? 1 : 0;          // chroma sub-sampling shifts (Table 6-1)
  if (n > 1 && (((tw & 1) && csx) || ((th & 1) && csy))) return set_error(B200_E_UNSUPPORTED, "grid tiles of odd size with sub-sampled chroma");
  const int cw = canvas_w > 0 ? canvas_w : tw * cols, chh = canvas_h > 0 ? canvas_h : th * rows;
  size_t n_ctu = 0, n_tu = 0, n_coef = 0, n_slice = 0, n_map = 0, n_rows = 0, rec_bytes = 0, bits = 0, n_rbsp = 0, n_subs = 0, n_map4 = 0;
  d->rec_off.resize((size_t)n * 3);
  std::vector<size_t> rbsp_off((size_t)n), sub_off((size_t)n), map4_off((size_t)n);
  for (int i = 0; i < n; i++) {
    ParsedPicture& pp = d->parsed[(size_t)i]; PicDesc& p = pp.desc;
    const size_t nctb = (size_t)p.wctb * p.hctb;
    p.ctu_base = (uint32_t)n_ctu; p.tu_base = (uint32_t)n_tu; p.coef_base = n_coef; p.slice_base = (uint32_t)n_slice; p.map8_base = (uint32_t)n_map;
    p.progress_base = (uint32_t)n_rows;
    rbsp_off[(size_t)i] = n_rbsp; sub_off[(size_t)i] = n_subs; map4_off[(size_t)i] = n_map4;
    n_ctu += nctb; n_slice += (devfe ? pp.hdr.slices.size() : pp.slices.size()); n_map += (size_t)p.w8 * p.h8; n_map4 += (size_t)p.w8 * p.h8 * 4; n_rows += (size_t)p.hctb;
    if (devfe) { n_tu += nctb * (size_t)pp.hdr.sp.tu_slots; n_coef += nctb * (size_t)pp.hdr.sp.coef_slots; n_rbsp += (pp.hdr.rbsp.size() + 15) & ~(size_t)15; n_subs += pp.hdr.subs.size(); }
    else { n_tu += pp.n_tus; n_coef += pp.n_coefs; }
    bits += au_size[i];
    for (int c = 0; c < (chroma ? 3 : 1); c++) {
      const int w = c ? p.width >> csx : p.width, h = c ? p.height >> csy : p.height;
      const int st = (w + 63) & ~63;
      p.rec_stride[c] = st;
      d->rec_off[(size_t)i * 3 + c] = rec_bytes;
      rec_bytes += (size_t)st * h * bps; rec_bytes = (rec_bytes + 255) & ~(size_t)255;
    }
  }
  // scaling lists: one 780-byte factor table per picture that enables them (784-byte slots)
  int n_scaling = 0;
  for (int i = 0; i < n; i++) { ParsedPicture& pp = d->parsed[(size_t)i]; pp.desc.scaling_idx = pp.hdr.scaling_enabled ? n_scaling++ : -1; }
  if (n_tu > 0xffffffffull) return set_error(B200_E_UNSUPPORTED, "batch too large");
  int rc;
  if ((rc = d->scaling.reserve((size_t)n_scaling * 784 + 16))) return rc;
  for (int i = 0; i < n; i++) { const ParsedPicture& pp = d->parsed[(size_t)i]; if (pp.desc.scaling_idx >= 0) memcpy(d->scaling.h + (size_t)pp.desc.scaling_idx * 784, &pp.hdr.scaling, sizeof(sl::Factors)); }
  if ((rc = d->pics.reserve((size_t)n)) || (rc = d->ctus.reserve(n_ctu, !devfe)) || (rc = d->tus.reserve(n_tu, !devfe)) || (rc = d->coefs.reserve(n_coef + 1, !devfe)) ||
      (rc = d->slices.reserve(n_slice)) || (rc = d->qp8.reserve(n_map, !devfe)) || (rc = d->edge8.reserve(n_map, !devfe)) || (rc = d->rows.reserve(3 * n_rows)) ||
      (rc = d->sync.reserve(3 * n_rows + 2 + MAX_CHUNKS, false)) || (rc = d->rec.reserve(rec_bytes, false)))
    return rc;
  if (devfe && ((rc = d->rbsp.reserve(n_rbsp + 16)) || (rc = d->subs.reserve(n_subs)) || (rc = d->equeue.reserve(2 + 2 * n_subs)) || (rc = d->ctu_slice.reserve(n_ctu)) ||
                (rc = d->epics.reserve((size_t)n)) || (rc = d->ipm4.reserve(n_map4, false)) || (rc = d->cd8.reserve(n_map, false)) ||
                (rc = d->wpp_ctx.reserve(n_rows * syn::CTX_STRIDE, false)) || (rc = d->end_state.reserve(n_subs * syn::CTX_STRIDE + 16, false)) ||
                (rc = d->esync.reserve(1 + n_rows + n_subs, false)) || (rc = d->ecount.reserve(2, true))))
    return rc;
  // canvas planes
  size_t cbytes = 0;
  for (int c = 0; c < (chroma ? 3 : 1); c++) {
    const int w = c ? (cw + csx) >> csx : cw, h = c ? (chh + csy) >> csy : chh;
    d->canvas_pitch[c] = (((size_t)w * bps) + 255) & ~(size_t)255;
    d->canvas_off[c] = cbytes; cbytes += d->canvas_pitch[c] * h;
  }
  const bool canvas_fully_covered = tw * cols >= cw && th * rows >= chh;
  if ((rc = d->canvas.reserve(cbytes, false))) return rc;
  // ---- 3. pack into pinned staging (parallel) and fix up device pointers
  for (int i = 0; i < n; i++) {
    ParsedPicture& pp = d->parsed[(size_t)i]; PicDesc& p = pp.desc;
    const int col = i % cols, row = i / cols;
    const int px = col * tw, py = row * th;
    p.out_w = std::max(0, std::min(tw, cw - px)); p.out_h = std::max(0, std::min(th, chh - py));     // clip like copy_image_to
    for (int c = 0; c < 3; c++) {
      if (c && !chroma) { p.rec[c] = nullptr; p.dst[c] = nullptr; continue; }
      p.rec[c] = d->rec.d + d->rec_off[(size_t)i * 3 + c];
      const int sx = c ? px >> csx : px, sy = c ? py >> csy : py;
      p.dst[c] = d->canvas.d + d->canvas_off[c] + (size_t)sy * d->canvas_pitch[c] + (size_t)sx * bps;
      p.dst_stride[c] = (int)(d->canvas_pitch[c] / bps);
    }
    d->pics.h[i] = p;
  }
  // Launch order of the CTB rows: row-major ACROSS pictures (all first rows, then all second rows, ...).  A row's
  // predecessor always holds a smaller ticket (deadlock freedom), and the resident warps spread over every tile's
  // wavefront instead of idling behind one tile's 2-CTB stagger.
  // Chunks: bands of whole tile rows for callers that take the result band by band (the fused host
  // entry points: D2H of band c overlaps the kernels of band c + 1), when the batch is larger than what K0 and K1 overlap
  // CTB by CTB (use_overlap).  One chunk = the classic back-to-back pipeline.
  { int nch = 1, rpc = rows;
    const char* ce = getenv("B200_CHUNKS");
    if (rows >= 2 && (ce ? atoi(ce) != 0 : (d->chunk_hook && (!devfe || !use_overlap(n_subs))))) {      // B200_CHUNKS=0 / 1: never / always (tests, diagnostics)
      // two bands by default: every K1 launch costs one tile's wavefront latency (~5 ms for 1024x1024), so more bands lose
      // more than their finer D2H overlap gains
      int target = (n + 1) / 2; if (const char* e = getenv("B200_CHUNK_TILES")) { const int v = atoi(e); if (v > 0) target = v; }
      rpc = std::max(1, (target + cols / 2) / cols);
      nch = (rows + rpc - 1) / rpc;
      if (nch > MAX_CHUNKS) { rpc = (rows + MAX_CHUNKS - 1) / MAX_CHUNKS; nch = (rows + rpc - 1) / rpc; }
    }
    d->nchunks = nch; d->grid_cols = cols;
    for (int c = 0; c <= nch; c++) d->chunk_pic[c] = std::min(n, c * rpc * cols);
    d->chunk_pic[nch] = n; }
  { size_t row_cursor = 0; d->max_log2_ctb = 4;
    for (int i = 0; i < n; i++) d->max_log2_ctb = std::max(d->max_log2_ctb, d->parsed[(size_t)i].desc.log2_ctb);
    for (int c = 0; c < d->nchunks; c++) {
      d->chunk_item[c] = row_cursor;
      int max_h = 0;
      for (int i = d->chunk_pic[c]; i < d->chunk_pic[c + 1]; i++) max_h = std::max(max_h, d->parsed[(size_t)i].desc.hctb);
      for (int r = 0; r < max_h; r++) for (int i = d->chunk_pic[c]; i < d->chunk_pic[c + 1]; i++) if (r < d->parsed[(size_t)i].desc.hctb) {
        d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r);                                        // luma
        if (chroma == 1) d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (1u << 30));           // Cb + Cr of a 4:2:0 picture on the two half-warps
        else if (chroma >= 2) { d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (2u << 30)); d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (3u << 30)); }   // Cb, Cr planes (4:2:2 / 4:4:4)
      }
    }
    d->chunk_item[d->nchunks] = row_cursor;
    d->n_items = row_cursor; d->info_bps = bps; }
  d->pool->parallel_for(n, [&](int i) {
    const ParsedPicture& pp = d->parsed[(size_t)i]; const PicDesc& p = pp.desc;
    if (!devfe) {
      memcpy(d->ctus.h + p.ctu_base, pp.ctus.data(), (size_t)p.wctb * p.hctb * sizeof(CtuInfo));
      memcpy(d->tus.h + p.tu_base, pp.tus.data(), pp.n_tus * sizeof(TuCmd));
      memcpy(d->coefs.h + p.coef_base, pp.coefs.data(), pp.n_coefs * sizeof(CoefEntry));
      memcpy(d->slices.h + p.slice_base, pp.slices.data(), pp.slices.size() * sizeof(SliceInfo));
      memcpy(d->qp8.h + p.map8_base, pp.qp8.data(), (size_t)p.w8 * p.h8);
      memcpy(d->edge8.h + p.map8_base, pp.edge8.data(), (size_t)p.w8 * p.h8);
    } else {
      const PictureHeaders& H = pp.hdr;
      memcpy(d->slices.h + p.slice_base, H.slices.data(), H.slices.size() * sizeof(SliceInfo));
      memcpy(d->rbsp.h + rbsp_off[(size_t)i], H.rbsp.data(), H.rbsp.size());
      memcpy(d->ctu_slice.h + p.ctu_base, H.ctu_slice.data(), H.ctu_slice.size() * sizeof(uint16_t));
      // Ready-queue links (batch-wide indices): which sub-stream each one releases, and how many events each waits for before
      // its first bin -- the conditions of run_substream (b200_hevc_syntax.h): the contexts stored after the 2nd CTB of the
      // row above (WPP, 9.3.2.2) and the end state of the slice segment it continues.
      const size_t so = sub_off[(size_t)i];
      for (size_t k = 0; k < H.subs.size(); k++) { syn::Substream ss = H.subs[k]; ss.pic = (uint32_t)i; ss.wake_ctb2 = ss.wake_end = -1; ss.deps = 0; d->subs.h[so + k] = ss; }
      for (size_t k = 0; k < H.subs.size(); k++) {
        syn::Substream& ss = d->subs.h[so + k];
        if (ss.prev >= 0) { ss.deps++; d->subs.h[so + (size_t)ss.prev].wake_end = (int32_t)(so + k); }
        const int wctb = H.desc.wctb, rx0 = (int)(ss.ctb_begin % (uint32_t)wctb), ry0 = (int)(ss.ctb_begin / (uint32_t)wctb);
        if (H.sp.wpp && rx0 == 0 && (!ss.init_contexts || ss.prev >= 0) && ss.ctb_begin != ss.slice_addr_rs && ry0 > 0 && (1 << H.desc.log2_ctb) < H.desc.width &&
            H.ctu_slice[(size_t)(ry0 - 1) * wctb + 1] == (uint16_t)ss.slice_idx) {
          const uint32_t a = (uint32_t)(ry0 - 1) * (uint32_t)wctb + 1;
          for (size_t j = 0; j < H.subs.size(); j++) if (H.subs[j].ctb_begin <= a && a < H.subs[j].ctb_end) { ss.deps++; d->subs.h[so + j].wake_ctb2 = (int32_t)(so + k); break; }
        }
      }
      EntropyPic ep{};
      ep.sp = H.sp; ep.sp.dense = 0;
      ep.pb.rbsp = d->rbsp.d + rbsp_off[(size_t)i]; ep.pb.rbsp_size = (uint32_t)H.rbsp.size();
      ep.pb.tus = d->tus.d + p.tu_base; ep.pb.coefs = d->coefs.d + p.coef_base; ep.pb.ctus = d->ctus.d + p.ctu_base; ep.pb.slices = d->slices.d + p.slice_base;
      ep.pb.ctu_slice = d->ctu_slice.d + p.ctu_base; ep.pb.qp8 = d->qp8.d + p.map8_base; ep.pb.edge8 = d->edge8.d + p.map8_base;
      ep.pb.ipm4 = d->ipm4.d + map4_off[(size_t)i]; ep.pb.cd8 = d->cd8.d + p.map8_base;
      ep.pb.wpp_ctx = d->wpp_ctx.d + (size_t)p.progress_base * syn::CTX_STRIDE; ep.pb.end_state = d->end_state.d + sub_off[(size_t)i] * syn::CTX_STRIDE;
      ep.progress_base = p.progress_base; ep.sub_base = (uint32_t)sub_off[(size_t)i];
      d->epics.h[i] = ep;
    }
  });
  if (devfe) {
    // ready queue image: cursors, the sub-streams without prerequisites in "k-th sub-stream of every picture" order (so
    // that whatever a popped sub-stream polls for was popped before it), empty slots, the dependency counters
    unsigned* q = d->equeue.h; size_t cur = 0, maxs = 0;
    for (int i = 0; i < n; i++) maxs = std::max(maxs, d->parsed[(size_t)i].hdr.subs.size());
    for (size_t k = 0; k < maxs; k++) for (int i = 0; i < n; i++) if (k < d->parsed[(size_t)i].hdr.subs.size() && d->subs.h[sub_off[(size_t)i] + k].deps == 0) q[2 + cur++] = (unsigned)(sub_off[(size_t)i] + k) + 1u;
    q[0] = 0; q[1] = (unsigned)cur;
    for (size_t k = cur; k < n_subs; k++) q[2 + k] = 0;
    for (size_t k = 0; k < n_subs; k++) q[2 + n_subs + k] = d->subs.h[k].deps;
  }
  const double t2 = now_ms();
  // ---- 4. H2D + kernels
  cudaEventRecord(d->ev[0], s);
  B200_CUDA_CHECK(cudaMemcpyAsync(d->pics.d, d->pics.h, (size_t)n * sizeof(PicDesc), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d->slices.d, d->slices.h, n_slice * sizeof(SliceInfo), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d->rows.d, d->rows.h, d->n_items * sizeof(uint2), cudaMemcpyHostToDevice, s));
  if (n_scaling) B200_CUDA_CHECK(cudaMemcpyAsync(d->scaling.d, d->scaling.h, (size_t)n_scaling * 784, cudaMemcpyHostToDevice, s));
  size_t h2d = (size_t)n_scaling * 784 + (size_t)n * sizeof(PicDesc) + n_slice * sizeof(SliceInfo) + d->n_items * sizeof(uint2);
  if (!devfe) {
    B200_CUDA_CHECK(cudaMemcpyAsync(d->ctus.d, d->ctus.h, n_ctu * sizeof(CtuInfo), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->tus.d, d->tus.h, n_tu * sizeof(TuCmd), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->coefs.d, d->coefs.h, n_coef * sizeof(CoefEntry), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->qp8.d, d->qp8.h, n_map, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->edge8.d, d->edge8.h, n_map, cudaMemcpyHostToDevice, s));
    h2d += n_ctu * sizeof(CtuInfo) + n_tu * sizeof(TuCmd) + n_coef * sizeof(CoefEntry) + 2 * n_map;
  } else {
    B200_CUDA_CHECK(cudaMemcpyAsync(d->rbsp.d, d->rbsp.h, n_rbsp, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->subs.d, d->subs.h, n_subs * sizeof(syn::Substream), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->equeue.d, d->equeue.h, (2 + 2 * n_subs) * sizeof(unsigned), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->ctu_slice.d, d->ctu_slice.h, n_ctu * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->epics.d, d->epics.h, (size_t)n * sizeof(EntropyPic), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemsetAsync(d->esync.d, 0, (1 + n_rows + n_subs) * sizeof(unsigned), s));
    B200_CUDA_CHECK(cudaMemsetAsync(d->ecount.d, 0, 2 * sizeof(unsigned long long), s));
    h2d += n_rbsp + n_subs * (sizeof(syn::Substream) + 2 * sizeof(unsigned)) + n_ctu * sizeof(uint16_t) + (size_t)n * sizeof(EntropyPic);
  }
  B200_CUDA_CHECK(cudaMemsetAsync(d->sync.d, 0, (3 * n_rows + 2 + MAX_CHUNKS) * sizeof(unsigned), s));
  if (!canvas_fully_covered) B200_CUDA_CHECK(cudaMemsetAsync(d->canvas.d, 0, cbytes, s));     // uncovered canvas stays zero (calloc in the reference)
  d->n_rows = n_rows; d->cbytes = cbytes; d->canvas_fully_covered = canvas_fully_covered; d->npics = n; d->n_subs = n_subs; d->used_device_front_end = devfe;
  b200_image_info& inf = d->info;
  inf.width = cw; inf.height = chh; inf.tile_width = tw; inf.tile_height = th; inf.chroma = chroma;        /* B200_CHROMA_MONO / 420 / 422 / 444 = chroma_format_idc */ inf.bit_depth = bd;
  inf.colour_primaries = d->parsed[0].hdr.colour_primaries; inf.transfer_characteristics = d->parsed[0].hdr.transfer_characteristics;
  inf.matrix_coefficients = d->parsed[0].hdr.matrix_coefficients; inf.full_range = d->parsed[0].hdr.full_range;
  if (info) *info = inf;
  int launches = 0;
  if ((rc = run_device_pipeline(d, n, s, &launches))) return rc;
  d->last_stream = s; d->have_result = true;
  b200_decode_stats& st = d->stats;
  memset(&st, 0, sizeof st);
  st.parse_ms = t1 - t0; st.pack_ms = t2 - t1; st.total_ms = now_ms() - t0;
  st.bitstream_bytes = bits; st.ctus = n_ctu;
  if (!devfe) {
    st.coefficient_entries = n_coef; st.transform_units = n_tu;
    st.command_bytes = n_ctu * sizeof(CtuInfo) + n_tu * sizeof(TuCmd) + n_coef * sizeof(CoefEntry) + n_slice * sizeof(SliceInfo) + 2 * n_map + (size_t)n * sizeof(PicDesc);
  }
  st.h2d_bytes = h2d;
  st.pixels = (uint64_t)cw * chh; st.kernel_launches = launches;
  return B200_OK;
}

// Re-run only the device kernels on the already uploaded command stream ("inputs resident in HBM" timing leg).
int b200_decoder_rerun_device(b200_decoder* d, void* stream_) {
  if (!d || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  cudaStream_t s = (cudaStream_t)stream_;
  B200_CUDA_CHECK(cudaMemsetAsync(d->sync.d, 0, (3 * d->n_rows + 2 + MAX_CHUNKS) * sizeof(unsigned), s));
  if (d->used_device_front_end) {
    B200_CUDA_CHECK(cudaMemsetAsync(d->esync.d, 0, (1 + d->n_rows + d->n_subs) * sizeof(unsigned), s));
    B200_CUDA_CHECK(cudaMemsetAsync(d->ecount.d, 0, 2 * sizeof(unsigned long long), s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->equeue.d, d->equeue.h, (2 + 2 * d->n_subs) * sizeof(unsigned), cudaMemcpyHostToDevice, s));
  }
  int launches = 0;
  int rc = run_device_pipeline(d, d->npics, s, &launches);
  d->last_stream = s;
  return rc;
}

int b200_decoder_get_stats(b200_decoder* d, b200_decode_stats* out) {
  if (!d || !out || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  B200_CUDA_CHECK(cudaEventSynchronize(d->ev[4]));
  float a = 0, en = 0, b = 0, c = 0, e = 0;
  cudaEventElapsedTime(&a, d->ev[0], d->ev[1]); cudaEventElapsedTime(&en, d->ev[1], d->ev[5]); cudaEventElapsedTime(&b, d->ev[5], d->ev[2]);
  cudaEventElapsedTime(&c, d->ev[2], d->ev[3]); cudaEventElapsedTime(&e, d->ev[3], d->ev[4]);
  if (b < 0) { en += b; b = 0; }   // K0 and K1 overlap: recon_ms is the part of K1 that runs after K0 has finished
  d->stats.h2d_ms = a; d->stats.entropy_ms = en; d->stats.recon_ms = b; d->stats.deblock_ms = c; d->stats.sao_ms = e; d->stats.gpu_ms = en + b + c + e;
  d->stats.front_end = d->used_device_front_end ? (d->last_chunked ? 3 : (d->last_overlapped ? 2 : 1)) : 0;
  d->stats.bands = d->last_chunked ? d->nchunks : 1;
  if (d->used_device_front_end) {
    B200_CUDA_CHECK(cudaMemcpy(d->ecount.h, d->ecount.d, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    d->stats.transform_units = d->ecount.h[0]; d->stats.coefficient_entries = d->ecount.h[1];
    d->stats.command_bytes = d->stats.ctus * sizeof(CtuInfo) + d->ecount.h[0] * sizeof(TuCmd) + d->ecount.h[1] * sizeof(CoefEntry) + 2 * (d->stats.pixels / 64);
  }
  *out = d->stats;
  return B200_OK;
}

int b200_decoder_get_planes(b200_decoder* d, b200_planes* out) {
  if (!d || !out || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  memset(out, 0, sizeof *out);
  out->y = d->canvas.d + d->canvas_off[0]; out->y_stride = d->canvas_pitch[0];
  if (d->info.chroma != B200_CHROMA_MONO) { out->cb = d->canvas.d + d->canvas_off[1]; out->cr = d->canvas.d + d->canvas_off[2]; out->c_stride = d->canvas_pitch[1]; }
  out->width = d->info.width; out->height = d->info.height; out->chroma = d->info.chroma; out->bit_depth = d->info.bit_depth;
  out->colour_primaries = d->info.colour_primaries; out->transfer_characteristics = d->info.transfer_characteristics;
  out->matrix_coefficients = d->info.matrix_coefficients; out->full_range = d->info.full_range;
  return B200_OK;
}

int b200_decoder_read_planes(b200_decoder* d, void* y, size_t ys, void* cb, void* cr, size_t cs, void* stream_) {
  if (!d || !y || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  cudaStream_t s = (cudaStream_t)stream_;
  const int bps = d->info.bit_depth > 8 ? 2 : 1, w = d->info.width, h = d->info.height;
  B200_CUDA_CHECK(cudaMemcpy2DAsync(y, ys, d->canvas.d + d->canvas_off[0], d->canvas_pitch[0], (size_t)w * bps, h, cudaMemcpyDeviceToHost, s));
  if (d->info.chroma != B200_CHROMA_MONO && cb && cr) {
    const int fsx = (d->info.chroma == B200_CHROMA_420 || d->info.chroma == B200_CHROMA_422) ? 1 : 0, fsy = d->info.chroma == B200_CHROMA_420 ? 1 : 0;
    const int cw = (w + fsx) >> fsx, ch = (h + fsy) >> fsy;
    B200_CUDA_CHECK(cudaMemcpy2DAsync(cb, cs, d->canvas.d + d->canvas_off[1], d->canvas_pitch[1], (size_t)cw * bps, ch, cudaMemcpyDeviceToHost, s));
    B200_CUDA_CHECK(cudaMemcpy2DAsync(cr, cs, d->canvas.d + d->canvas_off[2], d->canvas_pitch[2], (size_t)cw * bps, ch, cudaMemcpyDeviceToHost, s));
  }
  B200_CUDA_CHECK(cudaStreamSynchronize(s));
  return check_device_error(d);
}

int b200_decoder_debug_read_tile(b200_decoder* d, int index, int stage, void* y, void* cb, void* cr) {
  if (!d || !d->have_result || index < 0 || index >= d->npics) return set_error(B200_E_INVALID, "bad tile index");
  (void)stage;
  const PicDesc& p = d->pics.h[index];
  const int bps = p.bit_depth > 8 ? 2 : 1;
  void* outs[3] = {y, cb, cr};
  B200_CUDA_CHECK(cudaStreamSynchronize(d->last_stream));
  for (int c = 0; c < (p.chroma ? 3 : 1); c++) {
    if (!outs[c]) continue;
    const int fsx = (p.chroma == 1 || p.chroma == 2) ? 1 : 0, fsy = p.chroma == 1 ? 1 : 0;
    const int w = c ? p.width >> fsx : p.width, h = c ? p.height >> fsy : p.height;
    B200_CUDA_CHECK(cudaMemcpy2D(outs[c], (size_t)w * bps, p.rec[c], (size_t)p.rec_stride[c] * bps, (size_t)w * bps, h, cudaMemcpyDeviceToHost));
  }
  return B200_OK;
}

// Common part of the fused entry points: decode -> colour conversion into one of the two device RGB buffers.
static int decode_to_rgb_device(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size, uint64_t max_pixels, int canvas_w,
                                int canvas_h, const b200_geometry* geom, const b200_color_options* opt, b200_image_info* info, int slot, size_t* rowb_out,
                                size_t* pitch_out, int* out_h, void* direct_out, size_t direct_stride, bool* bands_copied, bool allow_bands) {
  if (!d->own) {
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&d->own, cudaStreamNonBlocking));
    B200_CUDA_CHECK(cudaStreamCreateWithFlags(&d->copy, cudaStreamNonBlocking));
    for (int i = 0; i < 2; i++) { B200_CUDA_CHECK(cudaEventCreateWithFlags(&d->ev_k6[i], cudaEventDisableTiming)); B200_CUDA_CHECK(cudaEventCreateWithFlags(&d->ev_d2h[i], cudaEventDisableTiming)); }
    B200_CUDA_CHECK(cudaHostAlloc((void**)&d->err_host, 2 * sizeof(unsigned), cudaHostAllocDefault));
    d->err_host[0] = d->err_host[1] = 0;
  }
  cudaStream_t s = d->own;
  // the page-locked staging of the previous call must have left for the device before the host overwrites it
  B200_CUDA_CHECK(cudaEventSynchronize(d->ev[1]));
  b200_image_info inf;
  size_t bpp;
  switch (opt->out_chroma) {
    case B200_CHROMA_INTERLEAVED_RGB: bpp = 3; break; case B200_CHROMA_INTERLEAVED_RGBA: bpp = 4; break;
    case B200_CHROMA_INTERLEAVED_RRGGBB_BE: case B200_CHROMA_INTERLEAVED_RRGGBB_LE: bpp = 6; break;
    case B200_CHROMA_INTERLEAVED_RRGGBBAA_BE: case B200_CHROMA_INTERLEAVED_RRGGBBAA_LE: bpp = 8; break;
    default: return set_error(B200_E_UNSUPPORTED, "the fused entry points need an interleaved target");
  }
  // Large grids into page-locked memory: after the entropy kernel the tile rows are reconstructed, filtered and converted in
  // bands, and the copy of band c to the host overlaps the kernels of band c + 1.  Band-wise conversion equals the
  // whole-picture one for the reference's default planner choice (nearest-neighbour chroma, per-sample arithmetic) without
  // rotate / mirror / crop; every other request converts the finished canvas in one go, below.
  bool banded = false; int hook_rc = B200_OK;
  *bands_copied = false;
  if (!geom && opt->chroma_upsampling == 0 && direct_out && allow_bands) {
    d->chunk_hook = [&, slot, bpp](int c, cudaStream_t side) -> int {
      const b200_image_info& I = d->info;
      const int th = I.tile_height, y0 = std::min(I.height, (d->chunk_pic[c] / d->grid_cols) * th);
      const int y1 = c + 1 == d->nchunks ? I.height : std::min(I.height, (d->chunk_pic[c + 1] / d->grid_cols) * th);
      const size_t rowb = (size_t)I.width * bpp, pitch = (rowb + 255) & ~(size_t)255;
      int rc2;
      if (c == 0) {
        if ((rc2 = d->rgb2[slot].reserve(pitch * (size_t)I.height, false))) return hook_rc = rc2;
        B200_CUDA_CHECK(cudaStreamWaitEvent(side, d->ev_d2h[slot], 0));       // the copy that last read this buffer has finished
        banded = true;
      }
      if (y1 <= y0) return B200_OK;
      const int bps = I.bit_depth > 8 ? 2 : 1; (void)bps;
      b200_planes pl; memset(&pl, 0, sizeof pl);
      pl.y = d->canvas.d + d->canvas_off[0] + (size_t)y0 * d->canvas_pitch[0]; pl.y_stride = d->canvas_pitch[0];
      if (I.chroma != B200_CHROMA_MONO) {
        const int bsy = I.chroma == B200_CHROMA_420 ? 1 : 0;
        pl.cb = d->canvas.d + d->canvas_off[1] + (size_t)(y0 >> bsy) * d->canvas_pitch[1]; pl.cr = d->canvas.d + d->canvas_off[2] + (size_t)(y0 >> bsy) * d->canvas_pitch[2];
        pl.c_stride = d->canvas_pitch[1];
      }
      pl.width = I.width; pl.height = y1 - y0; pl.chroma = I.chroma; pl.bit_depth = I.bit_depth;
      pl.colour_primaries = I.colour_primaries; pl.transfer_characteristics = I.transfer_characteristics; pl.matrix_coefficients = I.matrix_coefficients; pl.full_range = I.full_range;
      b200_geometry g; b200_geometry_identity(pl.width, pl.height, &g);
      uint8_t* dst = d->rgb2[slot].d + (size_t)y0 * pitch;
      if ((rc2 = b200_color_convert_device(&pl, &g, opt, dst, nullptr, nullptr, pitch, side, nullptr))) return hook_rc = rc2;
      if (direct_out) {
        if (!d->ev_chunk[c]) B200_CUDA_CHECK(cudaEventCreateWithFlags(&d->ev_chunk[c], cudaEventDisableTiming));
        B200_CUDA_CHECK(cudaEventRecord(d->ev_chunk[c], side));
        B200_CUDA_CHECK(cudaStreamWaitEvent(d->copy, d->ev_chunk[c], 0));
        B200_CUDA_CHECK(cudaMemcpy2DAsync(static_cast<uint8_t*>(direct_out) + (size_t)y0 * direct_stride, direct_stride, dst, pitch, rowb, (size_t)(y1 - y0), cudaMemcpyDeviceToHost, d->copy));
      }
      return B200_OK;
    };
  }
  int rc = b200_decoder_decode_grid(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, &inf, s);
  d->chunk_hook = nullptr;
  if (rc) return rc;
  if (hook_rc) return hook_rc;
  if (info) *info = inf;
  B200_CUDA_CHECK(cudaMemcpyAsync(&d->err_host[slot], d->sync.d + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, s));   // this step's error flag (the next step clears the device copy)
  b200_planes pl; if ((rc = b200_decoder_get_planes(d, &pl))) return rc;
  b200_geometry g; if (geom) g = *geom; else b200_geometry_identity(inf.width, inf.height, &g);
  const size_t rowb = (size_t)g.out_w * bpp, pitch = (rowb + 255) & ~(size_t)255;
  if (!banded) {
    if ((rc = d->rgb2[slot].reserve(pitch * g.out_h, false))) return rc;
    B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_d2h[slot], 0));           // the copy that last read this buffer has finished
    if ((rc = b200_color_convert_device(&pl, &g, opt, d->rgb2[slot].d, nullptr, nullptr, pitch, s, nullptr))) return rc;
  }
  B200_CUDA_CHECK(cudaEventRecord(d->ev_k6[slot], s));
  *bands_copied = banded && direct_out != nullptr;
  *rowb_out = rowb; *pitch_out = pitch; *out_h = g.out_h;
  return B200_OK;
}

static bool is_page_locked(const void* p) {
  cudaPointerAttributes pa{};
  const bool pinned = cudaPointerGetAttributes(&pa, p) == cudaSuccess && (pa.type == cudaMemoryTypeHost || pa.type == cudaMemoryTypeManaged);
  cudaGetLastError();
  return pinned;
}

int b200_decode_grid_to_rgb_host(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                 uint64_t max_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                 const b200_color_options* opt, void* out, size_t out_stride, b200_image_info* info) {
  if (!d || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  size_t rowb = 0, pitch = 0; int oh = 0; bool copied = false;
  const bool pinned = is_page_locked(out);
  int rc = decode_to_rgb_device(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, info, 0, &rowb, &pitch, &oh, pinned ? out : nullptr, out_stride, &copied, true);
  if (rc) return rc;
  cudaStream_t s = d->own;
  uint8_t* rgb = d->rgb2[0].d;
  // D2H: straight into the caller's buffer when it is page-locked (b200_host_alloc, cudaHostAlloc, cudaHostRegister);
  // pageable memory goes through a page-locked bounce buffer in row bands, the copy of band i overlapping the memcpy of
  // band i - 1 on the decoder's host threads
  if (copied) {                                         // the bands left through the copy stream as they were finished
    B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[0], d->copy));
    B200_CUDA_CHECK(cudaStreamSynchronize(s));
    B200_CUDA_CHECK(cudaStreamSynchronize(d->copy));
  } else if (pinned) {
    B200_CUDA_CHECK(cudaMemcpy2DAsync(out, out_stride, rgb, pitch, rowb, (size_t)oh, cudaMemcpyDeviceToHost, s));
    B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[0], s));
    B200_CUDA_CHECK(cudaStreamSynchronize(s));
  } else {
    const size_t band_rows = std::max<size_t>(1, (size_t)(32u << 20) / rowb);
    const int nb = (int)(((size_t)oh + band_rows - 1) / band_rows);
    if ((rc = d->bounce.reserve(2 * band_rows * rowb, true))) return rc;
    for (auto& e : d->ev_band) if (!e) B200_CUDA_CHECK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    for (int k = 0; k <= nb; k++) {
      if (k < nb) {
        const size_t y0 = (size_t)k * band_rows, h = std::min(band_rows, (size_t)oh - y0);
        B200_CUDA_CHECK(cudaMemcpy2DAsync(d->bounce.h + (size_t)(k & 1) * band_rows * rowb, rowb, rgb + y0 * pitch, pitch, rowb, h, cudaMemcpyDeviceToHost, s));
        B200_CUDA_CHECK(cudaEventRecord(d->ev_band[k & 1], s));
      }
      if (k > 0) {
        const int j = k - 1;
        const size_t y0 = (size_t)j * band_rows, h = std::min(band_rows, (size_t)oh - y0);
        B200_CUDA_CHECK(cudaEventSynchronize(d->ev_band[j & 1]));
        const uint8_t* src = d->bounce.h + (size_t)(j & 1) * band_rows * rowb;
        const int parts = 8;
        d->pool->parallel_for(parts, [&](int t) {
          const size_t r0 = h * (size_t)t / parts, r1 = h * (size_t)(t + 1) / parts;
          for (size_t y = r0; y < r1; y++) memcpy(static_cast<uint8_t*>(out) + (y0 + y) * out_stride, src + y * rowb, rowb);
        });
      }
    }
    B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[0], s));
    B200_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  if (d->err_host[0]) return set_error(B200_E_CUDA, "a decoding kernel gave up waiting for a dependency or met corrupt slice data");
  return B200_OK;
}

// Throughput form of the fused entry point: returns once the work is queued (the host part -- header parsing, packing -- is
// done); the RGB reaches `out` (page-locked memory, see b200_host_alloc) through a second stream, so the D2H of picture i
// overlaps the kernels of picture i + 1 (two device RGB buffers).  b200_decoder_wait() blocks until everything submitted
// has arrived and reports the first error.  `out` of consecutive calls may be the same buffer (copies are ordered).
int b200_decode_grid_to_rgb_host_async(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                       uint64_t max_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                       const b200_color_options* opt, void* out, size_t out_stride, b200_image_info* info) {
  if (!d || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  if (!is_page_locked(out)) return set_error(B200_E_INVALID, "the asynchronous entry point needs a page-locked output buffer (b200_host_alloc / b200_host_register)");
  const int slot = d->async_slot; d->async_slot ^= 1;
  if (d->err_host && d->err_host[slot]) d->async_error = true;                 // the step that used this slot two calls ago failed
  size_t rowb = 0, pitch = 0; int oh = 0; bool copied = false;
  int rc = decode_to_rgb_device(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, info, slot, &rowb, &pitch, &oh, out, out_stride, &copied, getenv("B200_CHUNKS") && atoi(getenv("B200_CHUNKS")) != 0);
  if (rc) return rc;
  if (!copied) {
    B200_CUDA_CHECK(cudaStreamWaitEvent(d->copy, d->ev_k6[slot], 0));
    B200_CUDA_CHECK(cudaMemcpy2DAsync(out, out_stride, d->rgb2[slot].d, pitch, rowb, (size_t)oh, cudaMemcpyDeviceToHost, d->copy));
  }
  B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[slot], d->copy));
  return B200_OK;
}

int b200_decoder_wait(b200_decoder* d) {
  if (!d) return set_error(B200_E_INVALID, "null argument");
  if (!d->own) return B200_OK;
  B200_CUDA_CHECK(cudaStreamSynchronize(d->own));
  B200_CUDA_CHECK(cudaStreamSynchronize(d->copy));
  const bool bad = d->async_error || d->err_host[0] || d->err_host[1];
  d->async_error = false;
  if (bad) return set_error(B200_E_CUDA, "a decoding kernel gave up waiting for a dependency or met corrupt slice data");
  return B200_OK;
}

// Host-only: size, format and colour description of the picture an access unit holds (headers only, microseconds).
int b200_probe_access_unit(const uint8_t* au, size_t size, uint64_t max_pixels, b200_image_info* info) {
  if (!au || !info) return set_error(B200_E_INVALID, "null argument");
  PictureHeaders H; ParseLimits lim; lim.max_image_size_pixels = max_pixels;
  int rc = parse_headers(au, size, lim, H);
  if (rc) return rc;
  memset(info, 0, sizeof *info);
  info->width = info->tile_width = H.desc.out_w; info->height = info->tile_height = H.desc.out_h;
  info->chroma = H.desc.chroma; info->bit_depth = H.desc.bit_depth;       /* B200_CHROMA_* = chroma_format_idc */
  info->colour_primaries = H.colour_primaries; info->transfer_characteristics = H.transfer_characteristics;
  info->matrix_coefficients = H.matrix_coefficients; info->full_range = H.full_range;
  return B200_OK;
}

// Page-locked host memory for the outputs of b200_decode_grid_to_rgb_host / b200_decoder_read_planes (DMA target).
int b200_host_alloc(size_t bytes, void** out) {
  if (!out) return set_error(B200_E_INVALID, "null argument");
  B200_CUDA_CHECK(cudaHostAlloc(out, bytes, cudaHostAllocDefault));
  return B200_OK;
}
void b200_host_free(void* p) { if (p) cudaFreeHost(p); }
// Page-lock memory the caller already owns (e.g. a shared-memory mapping several processes write their bands into).
int b200_host_register(void* p, size_t bytes) {
  if (!p) return set_error(B200_E_INVALID, "null argument");
  B200_CUDA_CHECK(cudaHostRegister(p, bytes, cudaHostRegisterPortable));
  return B200_OK;
}
int b200_host_unregister(void* p) { if (p) B200_CUDA_CHECK(cudaHostUnregister(p)); return B200_OK; }

}  // extern "C"

// Host-only introspection of the front-end (no CUDA involved): lets tests pin the CABAC/syntax layer on machines
// without a GPU.  Outputs: per 8x8 block QpY / filterEdgeFlags, per 4x4 block luma and chroma intra mode, and
// {order-independent coefficient hash, coefficient count, TU count, W, H}.
extern "C" int b200_debug_parse(const uint8_t* au, size_t size, int8_t* qp8, uint8_t* edge8, uint8_t* lmode4, uint8_t* cmode4,
                                unsigned long long* out5) {
  ParsedPicture pp; ParseLimits lim;
  int rc = parse_access_unit(au, size, lim, pp);
  if (rc) return rc;
  const PicDesc& p = pp.desc;
  const int w4 = p.width >> 2;
  memcpy(qp8, pp.qp8.data(), (size_t)p.w8 * p.h8); memcpy(edge8, pp.edge8.data(), (size_t)p.w8 * p.h8);
  unsigned long long hash = 0;
  for (size_t ti = 0; ti < pp.n_tus; ti++) {
    const TuCmd& t = pp.tus[ti];
    const int x4 = t.w0 & 0xfff, y4 = (t.w0 >> 12) & 0xfff, log2n = 2 + ((t.w0 >> 24) & 3), n4 = 1 << (log2n - 2);
    const int lm = t.w1 & 63, cm = (t.w1 >> 6) & 63;
    const int comp = (int)((t.w1 >> 23) & 3);            // 4:2:2 / 4:4:4: one command per block; 0 = luma block (or a 4:2:0 / 4:0:0 unit)
    if (p.chroma >= 2) {
      const int sx = p.chroma == 2 ? 1 : 0;
      if (comp == 0) { for (int y = 0; y < n4; y++) for (int x = 0; x < n4; x++) lmode4[(size_t)(y4 + y) * w4 + x4 + x] = (uint8_t)lm; }
      else for (int y = 0; y < n4; y++) for (int x = 0; x < (n4 << sx); x++) cmode4[(size_t)(y4 + y) * w4 + x4 + x] = (uint8_t)lm;
    } else
    for (int y = 0; y < n4; y++) for (int x = 0; x < n4; x++) { lmode4[(size_t)(y4 + y) * w4 + x4 + x] = (uint8_t)lm; cmode4[(size_t)(y4 + y) * w4 + x4 + x] = (uint8_t)cm; }
    const int nl = ((t.w0 >> 26) & 1) ? (int)(t.w3 & 0x7ff) : 0, ncb = ((t.w0 >> 27) & 1) ? (int)((t.w3 >> 11) & 0x3ff) : 0, ncr = ((t.w0 >> 28) & 1) ? (int)((t.w3 >> 21) & 0x3ff) : 0;
    const CoefEntry* ce = pp.coefs.data() + t.w2;
    int cx = x4 << 2, cy = y4 << 2;
    if (log2n == 2 && p.chroma < 2) { cx -= 4; cy -= 4; }     // chroma of the parent 8x8 node
    for (int k = 0; k < nl + ncb + ncr; k++) {
      const int c = comp ? comp : (k < nl ? 0 : (k < nl + ncb ? 1 : 2));
      const unsigned long long bx = c ? (unsigned long long)cx : (unsigned long long)(x4 << 2), by = c ? (unsigned long long)cy : (unsigned long long)(y4 << 2);
      unsigned long long hh = (bx * 1000003ULL + by) * 1000003ULL + (unsigned long long)c;
      hh = hh * 1000003ULL + ce[k].pos; hh = hh * 1000003ULL + (unsigned long long)(unsigned short)ce[k].level;
      hh ^= hh >> 29; hh *= 0x9E3779B97F4A7C15ULL; hash += hh;
    }
  }
  size_t units = 0;                                  // transform units = luma blocks (4:2:2 / 4:4:4 commands are per block)
  for (size_t ti = 0; ti < pp.n_tus; ti++) if (((pp.tus[ti].w1 >> 23) & 3) == 0) units++;
  out5[0] = hash; out5[1] = pp.n_coefs; out5[2] = units; out5[3] = (unsigned long long)p.width; out5[4] = (unsigned long long)p.height;
  return B200_OK;
}

// Host-only: parse n access units with `threads` parser threads (the decoder's front-end stage in isolation).
// Returns the wall-clock milliseconds of the parallel parse in *ms_out.  Used by tests and for tuning on CPU-only hosts.
extern "C" int b200_debug_parse_many(const uint8_t* const* au, const size_t* au_size, int n, int threads, int repeat, double* ms_out) {
  if (!au || !au_size || n <= 0) return set_error(B200_E_INVALID, "bad argument");
  const bool headers_only = threads < 0;
  if (headers_only) threads = -threads;
  Pool pool(threads > 0 ? threads : 1);
  std::vector<ParsedPicture> parsed((size_t)n);
  std::vector<int> rcs((size_t)n, 0);
  ParseLimits lim;
  double best = 1e30;
  for (int r = 0; r < (repeat > 0 ? repeat : 1); r++) {
    const double t0 = now_ms();
    // repeat < 0 is not used; threads < 0 selects the headers-only stage of the device front-end (NAL split, emulation prevention, headers)
    if (headers_only) pool.parallel_for(n, [&](int i) { rcs[(size_t)i] = parse_headers(au[i], au_size[i], lim, parsed[(size_t)i].hdr); });
    else pool.parallel_for(n, [&](int i) { rcs[(size_t)i] = parse_access_unit(au[i], au_size[i], lim, parsed[(size_t)i]); });
    best = std::min(best, now_ms() - t0);
  }
  for (int i = 0; i < n; i++) if (rcs[(size_t)i]) return rcs[(size_t)i];
  if (ms_out) *ms_out = best;
  return B200_OK;
}
