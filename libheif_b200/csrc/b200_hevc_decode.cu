// b200_hevc_decode.cu -- decoder object behind the C ABI: header parsing on host threads (one tile per task), staging
// into pinned memory, one H2D per array, then the entropy (K0) / reconstruction (K1) / deblocking / SAO kernels for the
// whole batch of tiles.  With the host front-end the same threads also run the CABAC syntax decoder.
//
// Mirrors the call order libheif uses on a decoder plugin instance (new_decoder2 -> push_data2 -> flush_data ->
// decode_next_image2 -> free_decoder, libheif/codecs/decoder.cc:388-405,441-446,458-460,487-493), but for N
// independent tiles at once, which is how ImageItem_Grid::decode_full_grid_image (libheif/image-items/grid.cc:250-468)
// consumes it.  All expensive state (device arenas, pinned staging, streams, events) lives here and is reused.
#include "b200_hevc.h"
#include "b200_staging.h"
#include <chrono>
#include <functional>
#include <memory>
#include <mutex>
#include <string>
#include <unistd.h>

using namespace b200;

namespace {

double now_ms() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// The counters and queues the kernels share, one batch-wide array each.  Their offsets follow from the batch's CTB rows and
// sub-streams alone; sizing, clearing and the kernels' batch descriptors all go through this one layout.
struct ScratchLayout {
  size_t n_rows = 0, n_subs = 0;
  // sync (K1 .. K4): [0] unused, [1] error flag, three progress counters per CTB row, then one work ticket per band
  static constexpr size_t error_flag = 1, progress = 2;
  size_t tickets() const { return progress + 3 * n_rows; }
  size_t sync_size() const { return tickets() + MAX_CHUNKS; }
  // esync (K0): [0] unused, one progress counter per CTB row, then one entry per sub-stream (EntropyBatch::sub_done)
  static constexpr size_t entropy_progress = 1;
  size_t sub_done() const { return entropy_progress + n_rows; }
  size_t esync_size() const { return sub_done() + n_subs; }
  // equeue (K0's ready queue): [0] pop cursor, [1] push cursor, one queue slot per sub-stream, then its dependency count
  static constexpr size_t qhead = 0, qtail = 1, queue = 2;
  size_t deps() const { return queue + n_subs; }
  size_t equeue_size() const { return deps() + n_subs; }
};

// Overrides of the launch schedule from the environment (tests, bench.py, diagnostics).  Read at the start of every
// decode_grid and rerun_device call, since callers change them between calls.
struct Overrides {
  enum Force { AUTO, OFF, ON };
  Force bands = AUTO;          // B200_CHUNKS=0 / 1: never / always run the tile rows in bands
  int band_tiles = 0;          // B200_CHUNK_TILES=n: tiles per band (default: half the grid)
  Force overlap = AUTO;        // B200_OVERLAP=0 / 1: K0 and K1 back to back / concurrently
  bool tail = true;            // B200_TAIL_OVERLAP=0: no tail overlap
  bool tail_force = false;     // B200_TAIL_FORCE: tail overlap for batches of at most one K0 wave too
  static Overrides read() {
    auto force = [](const char* name) { const char* e = getenv(name); return !e ? AUTO : (atoi(e) != 0 ? ON : OFF); };
    Overrides o;
    o.bands = force("B200_CHUNKS"); o.overlap = force("B200_OVERLAP");
    if (const char* e = getenv("B200_CHUNK_TILES")) o.band_tiles = std::max(0, atoi(e));
    if (const char* e = getenv("B200_TAIL_OVERLAP")) o.tail = atoi(e) != 0;
    o.tail_force = getenv("B200_TAIL_FORCE") != nullptr;
    return o;
  }
};

struct BatchShape {            // what the launch schedule depends on in a batch
  int cols = 1, rows = 1;      // grid of pictures
  bool device_front_end = false;
  size_t n_subs = 0;           // CABAC sub-streams (device front-end)
  bool any_tiles = false;      // a picture uses HEVC tiles
  bool all_common = false;     // every picture has the syn::CfgCommon parameter combination
  int bands = 0;               // row bands the row list is laid out in (0: not laid out yet)
};

// Resident CTAs per SM while K0 and K1 share the SMs.  Both kernels run 128 threads per CTA at 96 registers (K0: CfgCommon),
// so 3 + 2 CTAs fill 60 K of the SM's 64 K registers.  (K0 with CfgRuntime needs 124 registers: there the 2nd K1 CTA does
// not fit and waits for a free slot.)
enum { OVERLAP_K0_BLOCKS_PER_SM = 3, OVERLAP_K1_BLOCKS_PER_SM = 2 };

struct LaunchPlan {
  int bands = 1, rows_per_band = 1;   // row bands of whole tile rows (rows_per_band: when the plan lays them out)
  bool banded = false;                // K1 -> K3 -> K4 (-> the caller's band hook) run band by band
  bool overlap = false;               // K0 on the side stream, K1 following it CTB by CTB (if the process-wide slot is free)
  bool tail = false;                  // ... with K0 at full occupancy and K1 queued behind it
  int k0_blocks_per_sm = 0, k1_blocks_per_sm = 0;   // CTA caps of an overlapped run (0: none)
  bool common_k0 = false;             // the entropy kernel specialised for syn::CfgCommon
};

int sm_count() { int dev = 0, sms = 148; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); return sms; }

// The launch schedule of one run, from the batch, whether the caller takes the result band by band (`hook`), and the
// overrides.
// Bands: only a caller that takes the bands one by one (the synchronous fused entry point: the D2H of band c overlaps the
// kernels of band c + 1) gets them, and only when the batch is larger than what K0 and K1 overlap CTB by CTB.  Two bands by
// default: every K1 launch costs one tile's wavefront latency (~5 ms for 1024x1024), so more bands lose more than their
// finer D2H overlap gains.  Everything else -- the composition API, rerun_device, the asynchronous entry point whose D2H
// already overlaps the next picture -- runs one launch per kernel (the band-major row list is a valid ticket order for that).
// Overlap: K0 and K1 are persistent and ticket-driven, so they need not be fully co-resident (whatever part of either grid
// is resident finishes the work); the CTA caps only share the SM's registers between them.  Running them concurrently hides
// K1 completely while the batch is critical-path bound -- up to about one wave of sub-streams -- and LOSES once the GPU is
// throughput bound (the two instruction streams evict each other).
// Tail overlap, for batches of more than one wave: K0 keeps the whole GPU (5 CTAs per SM for CfgCommon, else 4; launched first) and the live K1 is
// queued behind it on the other stream, so K1's CTAs become resident only where K0's persistent CTAs have left -- which they
// do over the last ~30 % of K0's run time, once every sub-stream has been handed out and the wavefronts of the tiles drain.
// K1 (and, with bands, K3 / K4 / K6 / D2H of the first band; one K1 per band) then runs in SM slots that would otherwise idle.
// K1 follows K0 through per-row progress counters in raster order; sub-streams of HEVC tiles produce CTBs tile by tile, so
// a batch with tiles never overlaps.
LaunchPlan plan_launches(const BatchShape& b, bool hook, const Overrides& env) {
  LaunchPlan p;
  const bool devfe = b.device_front_end;
  const bool one_wave = devfe && (env.overlap == Overrides::AUTO ? b.n_subs <= (size_t)sm_count() * entropy_warps_per_sm(b.all_common)   // K0 decoders per SM: 20 (CfgCommon) or 16
                                                                  : env.overlap == Overrides::ON);
  p.bands = b.bands;
  if (!p.bands) {
    p.bands = 1; p.rows_per_band = b.rows;
    if (b.rows >= 2 && (env.bands != Overrides::AUTO ? env.bands == Overrides::ON : hook && !one_wave)) {
      const int target = env.band_tiles > 0 ? env.band_tiles : (b.cols * b.rows + 1) / 2;
      int rpb = std::max(1, (target + b.cols / 2) / b.cols);
      if ((b.rows + rpb - 1) / rpb > MAX_CHUNKS) rpb = (b.rows + MAX_CHUNKS - 1) / MAX_CHUNKS;
      p.rows_per_band = rpb; p.bands = (b.rows + rpb - 1) / rpb;
    }
  }
  p.banded = p.bands > 1 && (hook || env.bands == Overrides::ON);
  p.overlap = !p.banded && one_wave;
  p.tail = devfe && env.overlap == Overrides::AUTO && env.tail && (!p.overlap || env.tail_force);
  if (p.tail) p.overlap = true;
  if (b.any_tiles) p.overlap = p.tail = false;
  if (p.overlap && !p.tail) { p.k0_blocks_per_sm = OVERLAP_K0_BLOCKS_PER_SM; p.k1_blocks_per_sm = OVERLAP_K1_BLOCKS_PER_SM; }
  p.common_k0 = b.all_common;
  return p;
}

}  // namespace

struct b200_decoder {
  std::unique_ptr<Pool> pool;
  std::vector<ParsedPicture> parsed;
  std::vector<int> parse_rc; std::vector<std::string> parse_msg;
  DevBuf<PicDesc> pics; DevBuf<CtuInfo> ctus; DevBuf<TuCmd> tus; DevBuf<CoefEntry> coefs; DevBuf<SliceInfo> slices;
  DevBuf<int8_t> qp8; DevBuf<uint8_t> edge8; DevBuf<uint8_t> scaling; DevBuf<uint2> rows; DevBuf<unsigned> sync;   // sync: ScratchLayout
  DevBuf<uint8_t> rec; DevBuf<uint8_t> canvas; DevBuf<uint8_t> rgb2[2];   // fused host entry points: two RGB buffers (D2H of one overlaps the kernels writing the other)
  // device front-end (entropy decoding on the GPU)
  DevBuf<uint8_t> rbsp; DevBuf<syn::Substream> subs; DevBuf<unsigned> equeue; DevBuf<uint16_t> ctu_slice; DevBuf<EntropyPic> epics;
  DevBuf<uint8_t> ipm4, cd8, wpp_ctx, end_state; DevBuf<unsigned> esync; DevBuf<unsigned long long> ecount;
  // streams and events, all created by b200_decoder_create
  Stream own, copy;                // fused host entry points: the decode stream and the D2H stream
  Stream side;                     // K0 runs here, concurrently with K1 on the decode stream
  Event ev_fork, ev_join;          // decode stream -> side before K0, side -> decode stream after it
  Event t_start, t_h2d, t_entropy, t_recon, t_deblock, t_sao;   // stage ends on the decode stream (b200_decoder_get_stats)
  Event ev_k6[2], ev_d2h[2];       // per RGB buffer: colour conversion done, D2H done
  Event ev_band[MAX_CHUNKS];       // band pipeline: RGB of the band done
  Pinned<unsigned> err_host;       // per RGB buffer: the error flag of the step that used it last
  Bounce bounce;                   // synchronous fused entry point: the D2H into pageable memory
  int async_slot = 0; bool async_error = false;
  int front_end = 1;               // 1 = CABAC on the GPU (default), 0 = CABAC on the host cores
  int debug_stage = 0;
  // the batch decode_grid laid out last
  BatchShape shape;
  ScratchLayout scratch;
  int npics = 0; size_t n_items = 0; int max_log2_ctb = 6, info_bps = 1;
  int band_pic[MAX_CHUNKS + 1] = {0}; size_t band_item[MAX_CHUNKS + 1] = {0};   // first picture / row-list item of each band
  size_t canvas_off[3] = {0, 0, 0}; size_t canvas_pitch[3] = {0, 0, 0};
  b200_image_info info{};
  b200_decode_stats stats{};
  bool have_result = false, last_overlapped = false, last_banded = false;
  cudaStream_t last_stream = nullptr;
  // Band pipeline of the synchronous fused entry point (large grids): after K0, the tile rows go through K1 -> K3 -> K4 -> K6
  // in bands, and the D2H of band c (copy stream, band_hook) overlaps the kernels of band c + 1.
  std::function<int(int, cudaStream_t)> band_hook;    // queued after K4 of band c on the decode stream
};

static int check_device_error(b200_decoder* d) {
  unsigned flag = 0;
  B200_CUDA_CHECK(cudaMemcpy(&flag, d->sync.d + ScratchLayout::error_flag, sizeof flag, cudaMemcpyDeviceToHost));
  if (flag) return set_error(B200_E_CUDA, "reconstruction kernel gave up waiting for a CTB row dependency");
  return B200_OK;
}

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

// Device half, as the plan says: K0 entropy decoding (device front-end only), on the side stream when it overlaps K1
// reconstruction on `s`, then deblocking and SAO / paste on `s` -- for the whole batch or band by band.
static int run_device_pipeline(b200_decoder* d, const LaunchPlan& plan, cudaStream_t s, int* launches_out) {
  int rc;
  int launches = 0;
  const bool devfe = d->shape.device_front_end;
  const bool overlap = plan.overlap && overlap_acquire(d);
  struct Release { bool armed; ~Release() { if (armed) overlap_release(); } } release{overlap};   // error paths
  d->last_overlapped = overlap; d->last_banded = plan.banded;
  cudaEventRecord(d->t_h2d, s);
  const ScratchLayout& L = d->scratch;
  DeviceBatch b{};
  b.pics = d->pics.d; b.npics = d->npics; b.ctus = d->ctus.d; b.tus = d->tus.d; b.coefs = d->coefs.d; b.slices = d->slices.d;
  b.qp8 = d->qp8.d; b.edge8 = d->edge8.d; b.scaling = d->scaling.d; b.ticket = d->sync.d + L.tickets(); b.error_flag = d->sync.d + L.error_flag; b.progress = d->sync.d + L.progress;
  b.row_list = d->rows.d; b.nrows = (int)d->n_items; b.max_log2_ctb = d->max_log2_ctb; b.wide_samples = d->info_bps == 2;
  if (devfe) {
    EntropyBatch e{};
    e.pics = d->epics.d; e.npics = d->npics; e.subs = d->subs.d; e.nsubs = (int)L.n_subs;
    e.qhead = d->equeue.d + L.qhead; e.qtail = d->equeue.d + L.qtail; e.queue = d->equeue.d + L.queue; e.deps = d->equeue.d + L.deps();
    e.progress = d->esync.d + L.entropy_progress; e.sub_done = d->esync.d + L.sub_done(); e.error_flag = d->sync.d + L.error_flag;
    e.common = plan.common_k0;
    if (overlap) {
      e.blocks_per_sm = plan.k0_blocks_per_sm;
      b.blocks_per_sm = plan.k1_blocks_per_sm;
      b.entropy_progress = e.progress;
      cudaEventRecord(d->ev_fork, s);
      B200_CUDA_CHECK(cudaStreamWaitEvent(d->side, d->ev_fork, 0));
      int k0_warps = 0;
      if ((rc = launch_entropy(e, d->side, &k0_warps))) return rc;
      cudaEventRecord(d->t_entropy, d->side);
      if ((rc = launch_entropy_stats(e, d->ecount.d, d->side))) return rc;
      cudaEventRecord(d->ev_join, d->side);
      if (plan.tail) { if ((rc = launch_entropy_gate(e, k0_warps, s))) return rc; launches += 1; }   // K1 (next on s) must not take the SMs before K0 has them
    } else {
      if ((rc = launch_entropy(e, s))) return rc;
      cudaEventRecord(d->t_entropy, s);
      if ((rc = launch_entropy_stats(e, d->ecount.d, s))) return rc;
    }
    launches += 1;
  } else cudaEventRecord(d->t_entropy, s);
  if (plan.banded) {
    // Row bands of a large grid leave the pipeline one after the other: K1 -> K3 -> K4 of band c, then the caller's hook
    // (K6 of the band + its D2H on the copy stream, which overlaps the kernels of band c + 1).  K0 is NOT part of this:
    // letting the bands leave K0 in order (priority queues) and running these kernels beside it was measured slower --
    // K0 loses more from the co-residency (3 instead of 4 CTAs per SM) and the priorities than the overlap gains.
    for (int c = 0; c < d->shape.bands; c++) {
      DeviceBatch bc = b;
      bc.row_list = d->rows.d + d->band_item[c]; bc.nrows = (int)(d->band_item[c + 1] - d->band_item[c]); bc.ticket = b.ticket + c;
      if ((rc = launch_recon(bc, s))) return rc;
      if (overlap && c + 1 == d->shape.bands) {   // (tail overlap) K0 has finished before anything that follows the last K1
        B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_join, 0));
        B200_CUDA_CHECK(cudaLaunchHostFunc(s, overlap_done, nullptr));
        release.armed = false;
      }
      DeviceBatch bf = b;
      const int p0 = d->band_pic[c];
      bf.pics = d->pics.d + p0; bf.npics = d->band_pic[c + 1] - p0;
      if (d->debug_stage != 1 && (rc = launch_deblock(bf, d->pics.h + p0, s))) return rc;
      int nsao = 0;
      if (d->debug_stage == 0 && (rc = launch_sao(bf, d->pics.h + p0, s, &nsao))) return rc;
      launches += 3 + nsao;
      if (d->band_hook && (rc = d->band_hook(c, s))) return rc;
    }
    cudaEventRecord(d->t_recon, s); cudaEventRecord(d->t_deblock, s); cudaEventRecord(d->t_sao, s);   // recon_ms = the whole band pipeline (incl. the hooks' K6)
    if (launches_out) *launches_out = launches;
    return B200_OK;
  }
  if ((rc = launch_recon(b, s))) return rc;
  if (overlap) {
    B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_join, 0));
    B200_CUDA_CHECK(cudaLaunchHostFunc(s, overlap_done, nullptr));   // the slot is free once K0 and K1 have both finished
    release.armed = false;
  }
  cudaEventRecord(d->t_recon, s);
  launches += 1;
  if (d->debug_stage != 1) { if ((rc = launch_deblock(b, d->pics.h, s))) return rc; launches += 2; }
  cudaEventRecord(d->t_deblock, s);
  if (d->debug_stage == 0) { int nsao = 0; if ((rc = launch_sao(b, d->pics.h, s, &nsao))) return rc; launches += nsao; }
  cudaEventRecord(d->t_sao, s);
  if (launches_out) *launches_out = launches;
  return B200_OK;
}

// ---- the stages of b200_decoder_decode_grid

// Host stage, one tile per task.  Host front-end: headers + CABAC + syntax (serial per sub-stream).  Device front-end:
// headers only (NAL split, emulation prevention removal, parameter sets, entry points).
static int parse_stage(b200_decoder* d, int n, const uint8_t* const* au, const size_t* au_size, uint64_t max_pixels, bool devfe) {
  d->parsed.resize((size_t)n); d->parse_rc.assign((size_t)n, 0); d->parse_msg.assign((size_t)n, std::string());
  ParseLimits lim; lim.max_image_size_pixels = max_pixels;
  d->pool->parallel_for(n, [&](int i) {
    ParsedPicture& pp = d->parsed[(size_t)i];
    int rc = devfe ? parse_headers(au[i], au_size[i], lim, pp.hdr) : parse_access_unit(au[i], au_size[i], lim, pp);
    if (!rc && devfe) pp.desc = pp.hdr.desc;
    d->parse_rc[(size_t)i] = rc;
    if (rc) d->parse_msg[(size_t)i] = b200_last_error();
  });
  for (int i = 0; i < n; i++) if (d->parse_rc[(size_t)i]) return set_error(d->parse_rc[(size_t)i], "tile %d: %s", i, d->parse_msg[(size_t)i].c_str());
  return B200_OK;
}

struct Layout {                 // the sizes of one batch and where each picture sits in the batch-wide arrays
  int n = 0, cols = 1, rows = 1, tw = 0, th = 0, bd = 8, chroma = 0, bps = 1, csx = 0, csy = 0, cw = 0, ch = 0;
  size_t n_ctu = 0, n_tu = 0, n_coef = 0, n_slice = 0, n_map = 0, n_map4 = 0, n_rows = 0, n_rbsp = 0, n_subs = 0;
  size_t rec_bytes = 0, canvas_bytes = 0, bits = 0;
  int n_scaling = 0;            // pictures with scaling lists: one 780-byte factor table each (784-byte slots)
  std::vector<size_t> rec_off, rbsp_off, sub_off, map4_off;   // per picture (rec_off: per plane)
  bool canvas_covered = true;   // the tiles cover the whole canvas
};

// Checks that the tiles agree, gives every picture its offsets in the batch-wide arrays (written into its PicDesc) and
// lays out the canvas planes.
static int layout_stage(b200_decoder* d, int cols, int rows, const size_t* au_size, int canvas_w, int canvas_h, bool devfe, Layout& L) {
  const int n = cols * rows;
  L.n = n; L.cols = cols; L.rows = rows;
  const PicDesc& p0 = d->parsed[0].desc;
  L.tw = p0.out_w; L.th = p0.out_h; L.bd = p0.bit_depth; L.chroma = p0.chroma; L.bps = L.bd > 8 ? 2 : 1;
  for (int i = 1; i < n; i++) {
    const PicDesc& p = d->parsed[(size_t)i].desc;
    if (p.out_w != L.tw || p.out_h != L.th || p.bit_depth != L.bd || p.chroma != L.chroma)
      return set_error(B200_E_UNSUPPORTED, "grid tiles differ in size or format (tile %d)", i);   // grid.cc:261-375 requires equal tiles
  }
  L.csx = (L.chroma == 1 || L.chroma == 2) ? 1 : 0; L.csy = L.chroma == 1 ? 1 : 0;          // chroma sub-sampling shifts (Table 6-1)
  if (n > 1 && (((L.tw & 1) && L.csx) || ((L.th & 1) && L.csy))) return set_error(B200_E_UNSUPPORTED, "grid tiles of odd size with sub-sampled chroma");
  L.cw = canvas_w > 0 ? canvas_w : L.tw * cols; L.ch = canvas_h > 0 ? canvas_h : L.th * rows;
  L.rec_off.resize((size_t)n * 3); L.rbsp_off.resize((size_t)n); L.sub_off.resize((size_t)n); L.map4_off.resize((size_t)n);
  for (int i = 0; i < n; i++) {
    ParsedPicture& pp = d->parsed[(size_t)i]; PicDesc& p = pp.desc;
    const size_t nctb = (size_t)p.wctb * p.hctb;
    p.ctu_base = (uint32_t)L.n_ctu; p.tu_base = (uint32_t)L.n_tu; p.coef_base = L.n_coef; p.slice_base = (uint32_t)L.n_slice; p.map8_base = (uint32_t)L.n_map;
    p.progress_base = (uint32_t)L.n_rows;
    L.rbsp_off[(size_t)i] = L.n_rbsp; L.sub_off[(size_t)i] = L.n_subs; L.map4_off[(size_t)i] = L.n_map4;
    L.n_ctu += nctb; L.n_slice += (devfe ? pp.hdr.slices.size() : pp.slices.size()); L.n_map += (size_t)p.w8 * p.h8; L.n_map4 += (size_t)p.w8 * p.h8 * 4; L.n_rows += (size_t)p.hctb;
    if (devfe) { L.n_tu += nctb * (size_t)pp.hdr.sp.tu_slots; L.n_coef += nctb * (size_t)pp.hdr.sp.coef_slots; L.n_rbsp += (pp.hdr.rbsp.size() + 15) & ~(size_t)15; L.n_subs += pp.hdr.subs.size(); }
    else { L.n_tu += pp.n_tus; L.n_coef += pp.n_coefs; }
    L.bits += au_size[i];
    for (int c = 0; c < (L.chroma ? 3 : 1); c++) {
      const int w = c ? p.width >> L.csx : p.width, h = c ? p.height >> L.csy : p.height;
      const int st = (w + 63) & ~63;
      p.rec_stride[c] = st;
      L.rec_off[(size_t)i * 3 + c] = L.rec_bytes;
      L.rec_bytes += (size_t)st * h * L.bps; L.rec_bytes = (L.rec_bytes + 255) & ~(size_t)255;
    }
  }
  for (int i = 0; i < n; i++) { ParsedPicture& pp = d->parsed[(size_t)i]; pp.desc.scaling_idx = pp.hdr.scaling_enabled ? L.n_scaling++ : -1; }
  if (L.n_tu > 0xffffffffull) return set_error(B200_E_UNSUPPORTED, "batch too large");
  for (int c = 0; c < (L.chroma ? 3 : 1); c++) {
    const int w = c ? (L.cw + L.csx) >> L.csx : L.cw, h = c ? (L.ch + L.csy) >> L.csy : L.ch;
    d->canvas_pitch[c] = (((size_t)w * L.bps) + 255) & ~(size_t)255;
    d->canvas_off[c] = L.canvas_bytes; L.canvas_bytes += d->canvas_pitch[c] * h;
  }
  L.canvas_covered = L.tw * cols >= L.cw && L.th * rows >= L.ch;
  return B200_OK;
}

static int reserve_stage(b200_decoder* d, const Layout& L, const ScratchLayout& S, bool devfe) {
  int rc;
  if ((rc = d->scaling.reserve((size_t)L.n_scaling * 784 + 16))) return rc;
  if ((rc = d->pics.reserve((size_t)L.n)) || (rc = d->ctus.reserve(L.n_ctu, !devfe)) || (rc = d->tus.reserve(L.n_tu, !devfe)) || (rc = d->coefs.reserve(L.n_coef + 1, !devfe)) ||
      (rc = d->slices.reserve(L.n_slice)) || (rc = d->qp8.reserve(L.n_map, !devfe)) || (rc = d->edge8.reserve(L.n_map, !devfe)) || (rc = d->rows.reserve(3 * L.n_rows)) ||
      (rc = d->sync.reserve(S.sync_size(), false)) || (rc = d->rec.reserve(L.rec_bytes, false)))
    return rc;
  if (devfe && ((rc = d->rbsp.reserve(L.n_rbsp + 16)) || (rc = d->subs.reserve(L.n_subs)) || (rc = d->equeue.reserve(S.equeue_size())) || (rc = d->ctu_slice.reserve(L.n_ctu)) ||
                (rc = d->epics.reserve((size_t)L.n)) || (rc = d->ipm4.reserve(L.n_map4, false)) || (rc = d->cd8.reserve(L.n_map, false)) ||
                (rc = d->wpp_ctx.reserve(L.n_rows * syn::CTX_STRIDE, false)) || (rc = d->end_state.reserve(L.n_subs * syn::CTX_STRIDE + 16, false)) ||
                (rc = d->esync.reserve(S.esync_size(), false)) || (rc = d->ecount.reserve(2, true))))
    return rc;
  return d->canvas.reserve(L.canvas_bytes, false);
}

// Picture descriptors with their device pointers and paste positions, the scaling factors, and the row list: the CTB rows in
// launch order, row-major ACROSS pictures (all first rows, then all second rows, ...) within each band.  A row's predecessor
// always holds a smaller ticket (deadlock freedom), and the resident warps spread over every tile's wavefront instead of
// idling behind one tile's 2-CTB stagger.
static void pack_pictures(b200_decoder* d, const Layout& L, const LaunchPlan& plan) {
  const int n = L.n;
  for (int i = 0; i < n; i++) {
    ParsedPicture& pp = d->parsed[(size_t)i]; PicDesc& p = pp.desc;
    if (p.scaling_idx >= 0) memcpy(d->scaling.h + (size_t)p.scaling_idx * 784, &pp.hdr.scaling, sizeof(sl::Factors));
    const int col = i % L.cols, row = i / L.cols;
    const int px = col * L.tw, py = row * L.th;
    p.out_w = std::max(0, std::min(L.tw, L.cw - px)); p.out_h = std::max(0, std::min(L.th, L.ch - py));     // clip like copy_image_to
    for (int c = 0; c < 3; c++) {
      if (c && !L.chroma) { p.rec[c] = nullptr; p.dst[c] = nullptr; continue; }
      p.rec[c] = d->rec.d + L.rec_off[(size_t)i * 3 + c];
      const int sx = c ? px >> L.csx : px, sy = c ? py >> L.csy : py;
      p.dst[c] = d->canvas.d + d->canvas_off[c] + (size_t)sy * d->canvas_pitch[c] + (size_t)sx * L.bps;
      p.dst_stride[c] = (int)(d->canvas_pitch[c] / L.bps);
    }
    d->pics.h[i] = p;
  }
  for (int c = 0; c <= plan.bands; c++) d->band_pic[c] = std::min(n, c * plan.rows_per_band * L.cols);
  d->band_pic[plan.bands] = n;
  size_t row_cursor = 0; d->max_log2_ctb = 4;
  for (int i = 0; i < n; i++) d->max_log2_ctb = std::max(d->max_log2_ctb, d->parsed[(size_t)i].desc.log2_ctb);
  for (int c = 0; c < plan.bands; c++) {
    d->band_item[c] = row_cursor;
    int max_h = 0;
    for (int i = d->band_pic[c]; i < d->band_pic[c + 1]; i++) max_h = std::max(max_h, d->parsed[(size_t)i].desc.hctb);
    for (int r = 0; r < max_h; r++) for (int i = d->band_pic[c]; i < d->band_pic[c + 1]; i++) if (r < d->parsed[(size_t)i].desc.hctb) {
      d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r);                                        // luma
      if (L.chroma == 1) d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (1u << 30));         // Cb + Cr of a 4:2:0 picture on the two half-warps
      else if (L.chroma >= 2) { d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (2u << 30)); d->rows.h[row_cursor++] = make_uint2((unsigned)i, (unsigned)r | (3u << 30)); }   // Cb, Cr planes (4:2:2 / 4:4:4)
    }
  }
  d->band_item[plan.bands] = row_cursor;
  d->n_items = row_cursor; d->info_bps = L.bps;
}

// Host front-end: each picture's command stream into the page-locked staging (parallel)
static void pack_host_front_end(b200_decoder* d, const Layout& L) {
  d->pool->parallel_for(L.n, [&](int i) {
    const ParsedPicture& pp = d->parsed[(size_t)i]; const PicDesc& p = pp.desc;
    memcpy(d->ctus.h + p.ctu_base, pp.ctus.data(), (size_t)p.wctb * p.hctb * sizeof(CtuInfo));
    memcpy(d->tus.h + p.tu_base, pp.tus.data(), pp.n_tus * sizeof(TuCmd));
    memcpy(d->coefs.h + p.coef_base, pp.coefs.data(), pp.n_coefs * sizeof(CoefEntry));
    memcpy(d->slices.h + p.slice_base, pp.slices.data(), pp.slices.size() * sizeof(SliceInfo));
    memcpy(d->qp8.h + p.map8_base, pp.qp8.data(), (size_t)p.w8 * p.h8);
    memcpy(d->edge8.h + p.map8_base, pp.edge8.data(), (size_t)p.w8 * p.h8);
  });
}

// Device front-end: each picture's slice data, sub-streams and entropy descriptor into the page-locked staging (parallel)
static void pack_device_front_end(b200_decoder* d, const Layout& L) {
  d->pool->parallel_for(L.n, [&](int i) {
    const ParsedPicture& pp = d->parsed[(size_t)i]; const PicDesc& p = pp.desc;
    const PictureHeaders& H = pp.hdr;
    memcpy(d->slices.h + p.slice_base, H.slices.data(), H.slices.size() * sizeof(SliceInfo));
    memcpy(d->rbsp.h + L.rbsp_off[(size_t)i], H.rbsp.data(), H.rbsp.size());
    memcpy(d->ctu_slice.h + p.ctu_base, H.ctu_slice.data(), H.ctu_slice.size() * sizeof(uint16_t));
    // Ready-queue links (batch-wide indices): which sub-stream each one releases, and how many events each waits for before
    // its first bin -- the conditions of run_substream (b200_hevc_syntax.h): the contexts stored after the 2nd CTB of the
    // row above (WPP, 9.3.2.2) and the end state of the slice segment it continues.
    const size_t so = L.sub_off[(size_t)i];
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
    ep.pb.rbsp = d->rbsp.d + L.rbsp_off[(size_t)i]; ep.pb.rbsp_size = (uint32_t)H.rbsp.size();
    ep.pb.tus = d->tus.d + p.tu_base; ep.pb.coefs = d->coefs.d + p.coef_base; ep.pb.ctus = d->ctus.d + p.ctu_base; ep.pb.slices = d->slices.d + p.slice_base;
    ep.pb.ctu_slice = d->ctu_slice.d + p.ctu_base; ep.pb.qp8 = d->qp8.d + p.map8_base; ep.pb.edge8 = d->edge8.d + p.map8_base;
    ep.pb.ipm4 = d->ipm4.d + L.map4_off[(size_t)i]; ep.pb.cd8 = d->cd8.d + p.map8_base;
    ep.pb.wpp_ctx = d->wpp_ctx.d + (size_t)p.progress_base * syn::CTX_STRIDE; ep.pb.end_state = d->end_state.d + L.sub_off[(size_t)i] * syn::CTX_STRIDE;
    ep.progress_base = p.progress_base; ep.sub_base = (uint32_t)L.sub_off[(size_t)i];
    d->epics.h[i] = ep;
  });
}

// Ready queue image (device front-end): cursors, the sub-streams without prerequisites in "k-th sub-stream of every
// picture" order (so that whatever a popped sub-stream polls for was popped before it), empty slots, the dependency counters
static void build_ready_queue(b200_decoder* d, const Layout& L, const ScratchLayout& S) {
  unsigned* q = d->equeue.h; size_t cur = 0, maxs = 0;
  for (int i = 0; i < L.n; i++) maxs = std::max(maxs, d->parsed[(size_t)i].hdr.subs.size());
  for (size_t k = 0; k < maxs; k++) for (int i = 0; i < L.n; i++)
    if (k < d->parsed[(size_t)i].hdr.subs.size() && d->subs.h[L.sub_off[(size_t)i] + k].deps == 0) q[S.queue + cur++] = (unsigned)(L.sub_off[(size_t)i] + k) + 1u;
  q[S.qhead] = 0; q[S.qtail] = (unsigned)cur;
  for (size_t k = cur; k < L.n_subs; k++) q[S.queue + k] = 0;
  for (size_t k = 0; k < L.n_subs; k++) q[S.deps() + k] = d->subs.h[k].deps;
}

// Clears the counters of a run (and restores K0's ready queue), on `s`
static int reset_scratch(b200_decoder* d, const ScratchLayout& S, bool devfe, cudaStream_t s) {
  if (devfe) {
    B200_CUDA_CHECK(cudaMemsetAsync(d->esync.d, 0, S.esync_size() * sizeof(unsigned), s));
    B200_CUDA_CHECK(cudaMemsetAsync(d->ecount.d, 0, 2 * sizeof(unsigned long long), s));
  }
  B200_CUDA_CHECK(cudaMemsetAsync(d->sync.d, 0, S.sync_size() * sizeof(unsigned), s));
  return B200_OK;
}

// H2D of the staged batch on `s`; *h2d = the bytes copied
static int upload_stage(b200_decoder* d, const Layout& L, const ScratchLayout& S, bool devfe, cudaStream_t s, size_t* h2d) {
  const int n = L.n;
  B200_CUDA_CHECK(cudaMemcpyAsync(d->pics.d, d->pics.h, (size_t)n * sizeof(PicDesc), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d->slices.d, d->slices.h, L.n_slice * sizeof(SliceInfo), cudaMemcpyHostToDevice, s));
  B200_CUDA_CHECK(cudaMemcpyAsync(d->rows.d, d->rows.h, d->n_items * sizeof(uint2), cudaMemcpyHostToDevice, s));
  if (L.n_scaling) B200_CUDA_CHECK(cudaMemcpyAsync(d->scaling.d, d->scaling.h, (size_t)L.n_scaling * 784, cudaMemcpyHostToDevice, s));
  *h2d = (size_t)L.n_scaling * 784 + (size_t)n * sizeof(PicDesc) + L.n_slice * sizeof(SliceInfo) + d->n_items * sizeof(uint2);
  if (!devfe) {
    B200_CUDA_CHECK(cudaMemcpyAsync(d->ctus.d, d->ctus.h, L.n_ctu * sizeof(CtuInfo), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->tus.d, d->tus.h, L.n_tu * sizeof(TuCmd), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->coefs.d, d->coefs.h, L.n_coef * sizeof(CoefEntry), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->qp8.d, d->qp8.h, L.n_map, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->edge8.d, d->edge8.h, L.n_map, cudaMemcpyHostToDevice, s));
    *h2d += L.n_ctu * sizeof(CtuInfo) + L.n_tu * sizeof(TuCmd) + L.n_coef * sizeof(CoefEntry) + 2 * L.n_map;
  } else {
    B200_CUDA_CHECK(cudaMemcpyAsync(d->rbsp.d, d->rbsp.h, L.n_rbsp, cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->subs.d, d->subs.h, L.n_subs * sizeof(syn::Substream), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->equeue.d, d->equeue.h, S.equeue_size() * sizeof(unsigned), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->ctu_slice.d, d->ctu_slice.h, L.n_ctu * sizeof(uint16_t), cudaMemcpyHostToDevice, s));
    B200_CUDA_CHECK(cudaMemcpyAsync(d->epics.d, d->epics.h, (size_t)n * sizeof(EntropyPic), cudaMemcpyHostToDevice, s));
    *h2d += L.n_rbsp + L.n_subs * (sizeof(syn::Substream) + 2 * sizeof(unsigned)) + L.n_ctu * sizeof(uint16_t) + (size_t)n * sizeof(EntropyPic);
  }
  int rc;
  if ((rc = reset_scratch(d, S, devfe, s))) return rc;
  if (!L.canvas_covered) B200_CUDA_CHECK(cudaMemsetAsync(d->canvas.d, 0, L.canvas_bytes, s));     // uncovered canvas stays zero (calloc in the reference)
  return B200_OK;
}

static int decode_grid(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size, uint64_t max_pixels,
                       int canvas_w, int canvas_h, b200_image_info* info, cudaStream_t s, const Overrides& env) {
  if (!d || !au || !au_size || cols <= 0 || rows <= 0) return set_error(B200_E_INVALID, "bad argument");
  const double t0 = now_ms();
  const bool devfe = d->front_end != 0;
  d->have_result = false;
  int rc;
  if ((rc = parse_stage(d, cols * rows, au, au_size, max_pixels, devfe))) return rc;
  const double t1 = now_ms();
  Layout L;
  if ((rc = layout_stage(d, cols, rows, au_size, canvas_w, canvas_h, devfe, L))) return rc;
  BatchShape shape;
  shape.cols = cols; shape.rows = rows; shape.device_front_end = devfe; shape.n_subs = L.n_subs; shape.all_common = devfe;
  if (devfe) for (int i = 0; i < L.n; i++) {
    syn::SeqParams sp = d->parsed[(size_t)i].hdr.sp; sp.dense = 0;       // as K0 sees it (EntropyPic::sp)
    shape.any_tiles |= sp.tiles != 0; shape.all_common &= syn::matches_common(sp);
  }
  const LaunchPlan plan = plan_launches(shape, bool(d->band_hook), env);
  shape.bands = plan.bands;
  const ScratchLayout S{L.n_rows, L.n_subs};
  if ((rc = reserve_stage(d, L, S, devfe))) return rc;
  pack_pictures(d, L, plan);
  if (devfe) { pack_device_front_end(d, L); build_ready_queue(d, L, S); }
  else pack_host_front_end(d, L);
  const double t2 = now_ms();
  cudaEventRecord(d->t_start, s);
  size_t h2d = 0;
  if ((rc = upload_stage(d, L, S, devfe, s, &h2d))) return rc;
  d->shape = shape; d->scratch = S; d->npics = L.n;
  b200_image_info& inf = d->info;
  inf.width = L.cw; inf.height = L.ch; inf.tile_width = L.tw; inf.tile_height = L.th; inf.chroma = L.chroma;        /* B200_CHROMA_MONO / 420 / 422 / 444 = chroma_format_idc */ inf.bit_depth = L.bd;
  inf.colour_primaries = d->parsed[0].hdr.colour_primaries; inf.transfer_characteristics = d->parsed[0].hdr.transfer_characteristics;
  inf.matrix_coefficients = d->parsed[0].hdr.matrix_coefficients; inf.full_range = d->parsed[0].hdr.full_range;
  if (info) *info = inf;
  int launches = 0;
  if ((rc = run_device_pipeline(d, plan, s, &launches))) return rc;
  d->last_stream = s; d->have_result = true;
  b200_decode_stats& st = d->stats;
  memset(&st, 0, sizeof st);
  st.parse_ms = t1 - t0; st.pack_ms = t2 - t1; st.total_ms = now_ms() - t0;
  st.bitstream_bytes = L.bits; st.ctus = L.n_ctu;
  if (!devfe) {
    st.coefficient_entries = L.n_coef; st.transform_units = L.n_tu;
    st.command_bytes = L.n_ctu * sizeof(CtuInfo) + L.n_tu * sizeof(TuCmd) + L.n_coef * sizeof(CoefEntry) + L.n_slice * sizeof(SliceInfo) + 2 * L.n_map + (size_t)L.n * sizeof(PicDesc);
  }
  st.h2d_bytes = h2d;
  st.pixels = (uint64_t)L.cw * L.ch; st.kernel_launches = launches;
  return B200_OK;
}

extern "C" {

int b200_decoder_create(b200_decoder** out, int host_threads) {
  if (!out) return set_error(B200_E_INVALID, "null argument");
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return set_error(B200_E_CUDA, "no CUDA device: libb200heif has no CPU fallback");
  if (host_threads <= 0) { long n = sysconf(_SC_NPROCESSORS_ONLN); host_threads = n > 0 ? (int)n : 1; }
  std::unique_ptr<b200_decoder> d(new b200_decoder);
  d->pool.reset(new Pool(host_threads));
  for (Stream* st : {&d->own, &d->copy, &d->side}) B200_CUDA_CHECK(cudaStreamCreateWithFlags(&st->h, cudaStreamNonBlocking));
  for (Event* e : {&d->t_start, &d->t_h2d, &d->t_entropy, &d->t_recon, &d->t_deblock, &d->t_sao, &d->ev_fork, &d->ev_join}) B200_CUDA_CHECK(cudaEventCreate(&e->h));
  for (int i = 0; i < 2; i++)
    for (Event* e : {&d->ev_k6[i], &d->ev_d2h[i]}) B200_CUDA_CHECK(cudaEventCreateWithFlags(&e->h, cudaEventDisableTiming));
  for (Event& e : d->ev_band) B200_CUDA_CHECK(cudaEventCreateWithFlags(&e.h, cudaEventDisableTiming));
  B200_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&d->err_host.h), 2 * sizeof(unsigned), cudaHostAllocDefault));
  d->err_host.h[0] = d->err_host.h[1] = 0;
  *out = d.release();
  return B200_OK;
}

void b200_decoder_destroy(b200_decoder* d) { delete d; }

int b200_decoder_set_debug_stage(b200_decoder* d, int stage) { if (!d) return B200_E_INVALID; d->debug_stage = stage; return B200_OK; }

int b200_decoder_set_front_end(b200_decoder* d, int device) { if (!d) return B200_E_INVALID; d->front_end = device ? 1 : 0; return B200_OK; }

int b200_decoder_decode_grid(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                             uint64_t max_pixels, int canvas_w, int canvas_h, b200_image_info* info, void* stream_) {
  return decode_grid(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, info, (cudaStream_t)stream_, Overrides::read());
}

// Re-run only the device kernels on the already uploaded command stream ("inputs resident in HBM" timing leg).
int b200_decoder_rerun_device(b200_decoder* d, void* stream_) {
  if (!d || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  cudaStream_t s = (cudaStream_t)stream_;
  const LaunchPlan plan = plan_launches(d->shape, false, Overrides::read());
  int rc;
  if ((rc = reset_scratch(d, d->scratch, d->shape.device_front_end, s))) return rc;
  if (d->shape.device_front_end)
    B200_CUDA_CHECK(cudaMemcpyAsync(d->equeue.d, d->equeue.h, d->scratch.equeue_size() * sizeof(unsigned), cudaMemcpyHostToDevice, s));
  int launches = 0;
  rc = run_device_pipeline(d, plan, s, &launches);
  d->last_stream = s;
  return rc;
}

int b200_decoder_get_stats(b200_decoder* d, b200_decode_stats* out) {
  if (!d || !out || !d->have_result) return set_error(B200_E_INVALID, "no decode result");
  B200_CUDA_CHECK(cudaEventSynchronize(d->t_sao));
  float a = 0, en = 0, b = 0, c = 0, e = 0;
  cudaEventElapsedTime(&a, d->t_start, d->t_h2d); cudaEventElapsedTime(&en, d->t_h2d, d->t_entropy); cudaEventElapsedTime(&b, d->t_entropy, d->t_recon);
  cudaEventElapsedTime(&c, d->t_recon, d->t_deblock); cudaEventElapsedTime(&e, d->t_deblock, d->t_sao);
  if (b < 0) { en += b; b = 0; }   // K0 and K1 overlap: recon_ms is the part of K1 that runs after K0 has finished
  d->stats.h2d_ms = a; d->stats.entropy_ms = en; d->stats.recon_ms = b; d->stats.deblock_ms = c; d->stats.sao_ms = e; d->stats.gpu_ms = en + b + c + e;
  const bool devfe = d->shape.device_front_end;
  d->stats.front_end = devfe ? (d->last_banded ? 3 : (d->last_overlapped ? 2 : 1)) : 0;
  d->stats.bands = d->last_banded ? d->shape.bands : 1;
  if (devfe) {
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

}  // extern "C"

struct DeviceRgb {                  // where decode_to_rgb_device left the RGB of a call
  size_t rowb = 0, pitch = 0;       // bytes per output row, pitch of the device RGB buffer
  int height = 0;                   // output rows
  bool bands_copied = false;        // the bands already left for the destination through the copy stream
};

// Common part of the fused entry points: decode -> colour conversion into one of the two device RGB buffers.  `direct_out`:
// the page-locked destination the bands may be copied into as they are finished (nullptr: none).  The synchronous entry point
// takes bands whenever the plan gives them; the asynchronous one, whose D2H already overlaps the next call's kernels, only
// when B200_CHUNKS asks for them.  scale_w x scale_h > 0: the RGB scaled with HeifPixelImage::scale_nearest_neighbor, converted
// from the finished canvas in one launch (no bands: the copy of a scaled result is small).
static int decode_to_rgb_device(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size, uint64_t max_pixels, int canvas_w,
                                int canvas_h, const b200_geometry* geom, const b200_color_options* opt, int scale_w, int scale_h, b200_image_info* info,
                                int slot, void* direct_out, size_t direct_stride, bool async, DeviceRgb* res) {
  const Overrides env = Overrides::read();
  cudaStream_t s = d->own;
  // the page-locked staging of the previous call must have left for the device before the host overwrites it
  B200_CUDA_CHECK(cudaEventSynchronize(d->t_h2d));
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
  const bool scaled = scale_w > 0 && scale_h > 0;
  if (!scaled && !geom && opt->chroma_upsampling == 0 && direct_out && (!async || env.bands == Overrides::ON)) {
    d->band_hook = [&, slot, bpp](int c, cudaStream_t side) -> int {
      const b200_image_info& I = d->info;
      const int th = I.tile_height, y0 = std::min(I.height, (d->band_pic[c] / d->shape.cols) * th);
      const int y1 = c + 1 == d->shape.bands ? I.height : std::min(I.height, (d->band_pic[c + 1] / d->shape.cols) * th);
      const size_t rowb = (size_t)I.width * bpp, pitch = (rowb + 255) & ~(size_t)255;
      int rc2;
      if (c == 0) {
        if ((rc2 = d->rgb2[slot].reserve(pitch * (size_t)I.height, false))) return hook_rc = rc2;
        B200_CUDA_CHECK(cudaStreamWaitEvent(side, d->ev_d2h[slot], 0));       // the copy that last read this buffer has finished
        banded = true;
      }
      if (y1 <= y0) return B200_OK;
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
      B200_CUDA_CHECK(cudaEventRecord(d->ev_band[c], side));
      B200_CUDA_CHECK(cudaStreamWaitEvent(d->copy, d->ev_band[c], 0));
      B200_CUDA_CHECK(cudaMemcpy2DAsync(static_cast<uint8_t*>(direct_out) + (size_t)y0 * direct_stride, direct_stride, dst, pitch, rowb, (size_t)(y1 - y0), cudaMemcpyDeviceToHost, d->copy));
      return B200_OK;
    };
  }
  int rc = decode_grid(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, &inf, s, env);
  d->band_hook = nullptr;
  if (rc) return rc;
  if (hook_rc) return hook_rc;
  if (info) *info = inf;
  B200_CUDA_CHECK(cudaMemcpyAsync(&d->err_host.h[slot], d->sync.d + ScratchLayout::error_flag, sizeof(unsigned), cudaMemcpyDeviceToHost, s));   // this step's error flag (the next step clears the device copy)
  b200_planes pl; if ((rc = b200_decoder_get_planes(d, &pl))) return rc;
  b200_geometry g; if (geom) g = *geom; else b200_geometry_identity(inf.width, inf.height, &g);
  const int ow = scaled ? scale_w : g.out_w, oh = scaled ? scale_h : g.out_h;
  const size_t rowb = (size_t)ow * bpp, pitch = (rowb + 255) & ~(size_t)255;
  if (!banded) {
    if ((rc = d->rgb2[slot].reserve(pitch * oh, false))) return rc;
    B200_CUDA_CHECK(cudaStreamWaitEvent(s, d->ev_d2h[slot], 0));           // the copy that last read this buffer has finished
    if ((rc = b200_color_convert_scaled_device(&pl, &g, opt, ow, oh, d->rgb2[slot].d, nullptr, nullptr, pitch, s, nullptr))) return rc;
  }
  B200_CUDA_CHECK(cudaEventRecord(d->ev_k6[slot], s));
  res->rowb = rowb; res->pitch = pitch; res->height = oh; res->bands_copied = banded;
  return B200_OK;
}

// The synchronous fused entry points (scale_w x scale_h: 0 x 0 = unscaled)
static int decode_to_rgb_host(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size, uint64_t max_pixels, int canvas_w,
                              int canvas_h, const b200_geometry* geom, const b200_color_options* opt, int scale_w, int scale_h, void* out,
                              size_t out_stride, b200_image_info* info) {
  const bool pinned = is_page_locked(out);
  DeviceRgb r;
  int rc = decode_to_rgb_device(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, scale_w, scale_h, info, 0, pinned ? out : nullptr,
                                out_stride, false, &r);
  if (rc) return rc;
  cudaStream_t s = d->own;
  if (r.bands_copied) {                                 // the bands left through the copy stream as they were finished
    B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[0], d->copy));
    B200_CUDA_CHECK(cudaStreamSynchronize(s));
    B200_CUDA_CHECK(cudaStreamSynchronize(d->copy));
  } else {                                              // pageable memory is drained from the bounce buffer by the decoder's host threads
    if ((rc = d->bounce.download(out, out_stride, d->rgb2[0].d, r.pitch, r.rowb, (size_t)r.height, s, *d->pool))) return rc;
    B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[0], s));
    B200_CUDA_CHECK(cudaStreamSynchronize(s));
  }
  if (d->err_host.h[0]) return set_error(B200_E_CUDA, "a decoding kernel gave up waiting for a dependency or met corrupt slice data");
  return B200_OK;
}

extern "C" {

int b200_decode_grid_to_rgb_host(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                 uint64_t max_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                 const b200_color_options* opt, void* out, size_t out_stride, b200_image_info* info) {
  if (!d || !opt || !out) return set_error(B200_E_INVALID, "null argument");
  return decode_to_rgb_host(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, 0, 0, out, out_stride, info);
}

// heif_decode_image + heif_image_scale_image (heif-thumbnailer) in one call: the scaled result is all that is converted and copied
int b200_decode_grid_to_rgb_scaled_host(b200_decoder* d, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                        uint64_t max_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                        const b200_color_options* opt, int scale_w, int scale_h, void* out, size_t out_stride,
                                        b200_image_info* info) {
  if (scale_w < 1) return set_error(B200_E_INVALID, "scale_w %d: the scaled picture needs at least one column", scale_w);
  if (scale_h < 1) return set_error(B200_E_INVALID, "scale_h %d: the scaled picture needs at least one row", scale_h);
  const void* const args[] = {d, au, au_size, opt, out};
  const char* const names[] = {"dec", "au", "au_size", "opt", "out"};
  for (int i = 0; i < 5; i++) if (!args[i]) return set_error(B200_E_INVALID, "%s is NULL", names[i]);
  return decode_to_rgb_host(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, scale_w, scale_h, out, out_stride, info);
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
  if (d->err_host.h[slot]) d->async_error = true;                 // the step that used this slot two calls ago failed
  DeviceRgb r;
  int rc = decode_to_rgb_device(d, cols, rows, au, au_size, max_pixels, canvas_w, canvas_h, geom, opt, 0, 0, info, slot, out, out_stride, true, &r);
  if (rc) return rc;
  if (!r.bands_copied) {
    B200_CUDA_CHECK(cudaStreamWaitEvent(d->copy, d->ev_k6[slot], 0));
    B200_CUDA_CHECK(cudaMemcpy2DAsync(out, out_stride, d->rgb2[slot].d, r.pitch, r.rowb, (size_t)r.height, cudaMemcpyDeviceToHost, d->copy));
  }
  B200_CUDA_CHECK(cudaEventRecord(d->ev_d2h[slot], d->copy));
  return B200_OK;
}

int b200_decoder_wait(b200_decoder* d) {
  if (!d) return set_error(B200_E_INVALID, "null argument");
  B200_CUDA_CHECK(cudaStreamSynchronize(d->own));
  B200_CUDA_CHECK(cudaStreamSynchronize(d->copy));
  const bool bad = d->async_error || d->err_host.h[0] || d->err_host.h[1];
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

// Host-only: what the in-loop filters read of an access unit beyond b200_debug_parse's qp8 / edge8, in the record layouts of
// b200_debug_loop_filters.  hdr[13]: coded width, height, log2 CTB size, bit depth, chroma_format_idc, pps Cb / Cr QP offsets,
// sample_adaptive_offset_enabled_flag, number of regions, conformance window (crop_x, crop_y, out_w, out_h in luma samples).
// ctbs[k * 19 ..] (raster order, room for `max_ctbs`): region index and the three SaoComp (type, band position / EO class,
// four offsets).  regions[k * 6 ..] (room for `max_regions`): beta offset, tc offset, slice_loop_filter_across_slices_enabled_flag,
// slice index, TileId, loop_filter_across_tiles_enabled_flag.  With ctbs / regions NULL only hdr is filled.
extern "C" int b200_debug_parse_filters(const uint8_t* au, size_t size, int32_t* hdr, int32_t* ctbs, int max_ctbs, int32_t* regions, int max_regions) {
  if (!au || !hdr) return set_error(B200_E_INVALID, "parse_filters: null argument");
  ParsedPicture pp; ParseLimits lim;
  int rc = parse_access_unit(au, size, lim, pp);
  if (rc) return rc;
  const PicDesc& p = pp.desc;
  const int32_t h[13] = {p.width, p.height, p.log2_ctb, p.bit_depth, p.chroma, p.pps_cb_qp_offset, p.pps_cr_qp_offset, p.sao_enabled, (int32_t)pp.slices.size(),
                         p.crop_x, p.crop_y, p.out_w, p.out_h};
  memcpy(hdr, h, sizeof h);
  const size_t nctb = (size_t)p.wctb * p.hctb;
  if (ctbs) {
    if (max_ctbs < 0 || (size_t)max_ctbs < nctb) return set_error(B200_E_INVALID, "parse_filters: room for %d CTBs, %zu needed", max_ctbs, nctb);
    for (size_t k = 0; k < nctb; k++) {
      const CtuInfo& ci = pp.ctus[k];
      int32_t* o = ctbs + k * 19;
      o[0] = ci.slice_idx;
      for (int c = 0; c < 3; c++) {
        o[1 + 6 * c] = ci.sao[c].type; o[2 + 6 * c] = ci.sao[c].band_or_class;
        for (int j = 0; j < 4; j++) o[3 + 6 * c + j] = ci.sao[c].offset[j];
      }
    }
  }
  if (regions) {
    if (max_regions < 0 || (size_t)max_regions < pp.slices.size()) return set_error(B200_E_INVALID, "parse_filters: room for %d regions, %zu needed", max_regions, pp.slices.size());
    for (size_t k = 0; k < pp.slices.size(); k++) {
      const SliceInfo& s = pp.slices[k];
      int32_t* o = regions + k * 6;
      o[0] = s.beta_offset; o[1] = s.tc_offset; o[2] = s.lf_across_slices; o[3] = s.slice_id; o[4] = s.tile_id; o[5] = s.lf_across_tiles;
    }
  }
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
