// b200_hevc_entropy.cu -- K0: CABAC entropy decoding + slice-data syntax on the GPU.
//
// The serial half of libde265's decode (H.265 9.3 CABAC, 7.3.8 coding-quadtree syntax, 8.4.2 / 8.6.1 derivations) for
// a whole batch of tiles at once: ONE WARP PER CABAC SUB-STREAM (all 32 lanes run the shared syntax decoder of
// b200_hevc_syntax.h, the same source the host front-end uses, on identical data, and split the map fills, context copies
// and coefficient emission between them).  With entropy_coding_sync every CTB row is its own
// sub-stream, located by the slice header's entry points, so a 16384x16384 grid of 1024x1024 tiles exposes 8192
// independent-ish streams: rows of one picture advance as a wavefront (context hand-over after the 2nd CTB of the row
// above, 9.3.2.2), pictures are independent.  Sub-streams are handed out through a READY QUEUE: a sub-stream enters it when
// the events it has to wait for before its first bin have happened (context hand-over stored by the row above; end of the
// slice segment it continues) -- the warp that causes the last such event pushes it.  A resident warp therefore never sits
// on a sub-stream that cannot start (18 % of all warp time with static tickets), and whatever is popped only ever waits for
// sub-streams popped before it (no deadlock, no co-residency requirement).
// Output: the command stream of b200_hevc_types.h, written into fixed per-CTB slots in HBM (worst-case sized; only the
// used entries are ever touched).  Why on the GPU: the host has 16 usable cores on the target box and CABAC is the
// end-to-end bottleneck there; the arithmetic decoder is serial per sub-stream but there are thousands of sub-streams.
#include <cstdint>
#include <cstdlib>
// The syntax decoder's lookup tables live in SHARED memory on the device (the dependent table look-ups of every CABAC
// bin would otherwise go through L1/L2): file-scope __shared__ copies, filled at kernel start, reached through B200_T.
namespace b200 { namespace syn {
__shared__ uint32_t s_kLps4[64];
__shared__ uint8_t s_kTransLps[64];
__shared__ uint8_t s_kNextState[256];
__shared__ unsigned long long s_kState[128];
__shared__ uint8_t s_kInitI[135];                     // CTX_COUNT (declared before the syntax header is included; checked below)
__shared__ uint8_t s_kSigMap4[16];
__shared__ uint8_t s_kScanPos[3][16];
__shared__ uint8_t s_kScanInv[3][16];
__shared__ uint8_t s_kSbInv[4][3][64];
__shared__ uint8_t s_kSigCtx4[3][16];
__shared__ uint8_t s_kSigCtxN[3][4][16];
__shared__ uint8_t s_kChromaTab[4];
__shared__ uint8_t s_kScanX[4][3][64];
__shared__ uint8_t s_kScanY[4][3][64];
} }
#ifdef __CUDA_ARCH__
#define B200_T(name) s_##name
#endif
#include "b200_hevc.h"
static_assert(b200::syn::CTX_COUNT == 135, "s_kInitI above is sized for 135 context variables");

namespace b200 {

#ifndef B200_ENTROPY_WARPS
#define B200_ENTROPY_WARPS 4
#endif
constexpr int EWARPS = B200_ENTROPY_WARPS;

// Polling load: relaxed + gpu scope (served by L2).  ld.acquire would make ptxas emit CCTL.IVALL -- an SM-wide L1 invalidation --
// on EVERY poll (measured: 43 % of all stall samples of the first version); ordering is obtained instead by reading every
// piece of cross-thread data with L1-bypassing loads (B200_LD_SHARED / __ldcg) after the control-dependent loop exit.
__device__ __forceinline__ unsigned e_ld_acquire(const unsigned* p) {
  unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void e_st_release(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// A decoder warp's poll: lane 0's value for every lane, so that the loop it controls stays warp-uniform.
__device__ __forceinline__ unsigned e_poll(const unsigned* p) { return __shfl_sync(0xffffffffu, e_ld_acquire(p), 0); }
__device__ __forceinline__ bool lane0() { return syn::lane_id() == 0; }

#ifdef B200_ENTROPY_TRACE
// Per sub-stream (batch-wide index): globaltimer at the queue pop and at the end, and the SM it ran on.  For
// scripts/k0_trace_probe.py only; b200_debug_entropy_trace() copies it out.
constexpr int TRACE_CAP = 1 << 16;
__device__ unsigned long long g_trace[TRACE_CAP][2];
__device__ unsigned g_trace_sm[TRACE_CAP];
__device__ __forceinline__ unsigned long long e_globaltimer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
__device__ __forceinline__ unsigned e_smid() { unsigned s; asm volatile("mov.u32 %0, %%smid;" : "=r"(s)); return s; }
#endif

// Every lane of a decoder warp calls these (the decoder runs warp-wide, b200_hevc_syntax.h); the atomics and the releases
// happen once, on lane 0, after a warp barrier that orders the other lanes' stores (map cells, contexts) before them.
struct DevSync {
  unsigned* progress;      // per CTB row of this picture
  unsigned* sub_done;      // per sub-stream of this picture
  unsigned* error_flag;
  unsigned* queue; unsigned* qtail; unsigned* deps;               // batch-wide ready queue (see the kernel)
  uint32_t dense_tu, dense_coef, dense_tu_cap, dense_coef_cap;   // unused on the device (fixed slots)
  uint64_t end_bit_position;
  // Waits inside a sub-stream are short (the row above runs two CTBs ahead): poll with a sub-microsecond back-off.  Gives
  // up (error 3) after ~60 s -- only a lost producer can cause that.  The caps (8 us here, 16 us for a queue slot) are the
  // measured optimum: 1.6 / 2 us made K0 ~1 % slower and 0.8 / 1 us ~2 % (polls take issue slots from the busy decoders),
  // 16 / 32 us gained nothing (H100 80GB HBM3 SXM at 400 W, bench.py).
  __device__ static void spin_until(const unsigned* p, unsigned need, unsigned* error_flag) {
    if (e_poll(p) >= need) return;
    unsigned ns = 200, spins = 0;
    for (;;) {
      __nanosleep(ns); if (ns < 8000) ns <<= 1;
      if (e_poll(p) >= need) return;
      if ((++spins & 63u) != 0) continue;
      if (e_poll(error_flag)) return;                    // a producer failed: do not wait for progress that will never come
      if (spins > (1u << 23)) { if (lane0()) atomicExch(error_flag, 3u); return; }
    }
  }
  __device__ void wait_row(int row, int need) { spin_until(progress + row, (unsigned)need, error_flag); }
  __device__ void publish_row(int row, int done) { syn::warp_sync(); if (lane0()) e_st_release(progress + row, (unsigned)done); }
  __device__ void wait_substream(int idx) { spin_until(sub_done + idx, 1u, error_flag); }
  __device__ void finish_substream(int idx, int err) {
    syn::warp_sync();
    if (lane0()) {
      e_st_release(sub_done + idx, 1u);
      if (err) atomicExch(error_flag, (unsigned)err);
    }
  }
  // One of the events sub-stream `target` (batch-wide index) waits for has happened; the last one makes it ready.
  __device__ void notify(int target) {
    if (target < 0) return;
    syn::warp_sync();
    if (lane0()) {
      __threadfence();                                   // what the target will read (contexts, end state) is published first
      if (atomicSub(deps + target, 1u) == 1u) { const unsigned s = atomicAdd(qtail, 1u); e_st_release(queue + s, (unsigned)target + 1u); }
    }
  }
};

#ifndef B200_ENTROPY_MIN_BLOCKS
#define B200_ENTROPY_MIN_BLOCKS 1
#endif
// Compile-time cap of resident K0 CTAs per SM (0: none, occupancy decides) -- for measuring how K0 scales with the number of
// decoders per SM.
#ifndef B200_ENTROPY_MAX_BLOCKS_PER_SM
#define B200_ENTROPY_MAX_BLOCKS_PER_SM 0
#endif
// CfgCommon's call chain (kernel -> decode_ctb -> residual -> refill) fits in 96 registers without spilling, which makes 5 CTAs
// (20 decoders) per SM: registers are allocated for all 32 lanes of a warp, so they, not the work, cap the number of decoders.
// The bound holds that figure: should a change need more, ptxas reports spills (-Xptxas -v) instead of silently dropping
// to 4 CTAs.  CfgRuntime needs 124 registers: 4 CTAs.
template <class Cfg> constexpr int entropy_min_blocks() { return B200_ENTROPY_MIN_BLOCKS; }
template <> constexpr int entropy_min_blocks<syn::CfgCommon>() { return B200_ENTROPY_MIN_BLOCKS > 5 ? B200_ENTROPY_MIN_BLOCKS : 5; }
template <class Cfg>
__global__ void __launch_bounds__(EWARPS * 32, entropy_min_blocks<Cfg>()) hevc_entropy_kernel(const EntropyBatch b) {
  __shared__ __align__(8) syn::U2 s_ctx[EWARPS][syn::CTX_COUNT + syn::CTX_SCRATCH];   // context variables: one state-table entry each (+ scratch)
  __shared__ syn::DecoderT<Cfg> s_dec[EWARPS];                    // per-warp decoder state (see run_substream)
  __shared__ DevSync s_sync[EWARPS];                              // per-warp hand-shake pointers (shared: no register holds them across the CTB loop)
  for (int i = threadIdx.x; i < 64; i += blockDim.x) { syn::s_kLps4[i] = syn::d_kLps4[i]; syn::s_kTransLps[i] = syn::d_kTransLps[i]; }
  for (int i = threadIdx.x; i < syn::CTX_COUNT; i += blockDim.x) syn::s_kInitI[i] = syn::d_kInitI[i];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) syn::s_kNextState[i] = syn::d_kNextState[i];
  for (int i = threadIdx.x; i < 128; i += blockDim.x) syn::s_kState[i] = syn::d_kState[i];
  for (int i = threadIdx.x; i < 16; i += blockDim.x) syn::s_kSigMap4[i] = syn::d_kSigMap4[i];
  for (int i = threadIdx.x; i < 48; i += blockDim.x) { (&syn::s_kScanPos[0][0])[i] = (&syn::d_kScanPos[0][0])[i]; (&syn::s_kScanInv[0][0])[i] = (&syn::d_kScanInv[0][0])[i]; (&syn::s_kSigCtx4[0][0])[i] = (&syn::d_kSigCtx4[0][0])[i]; }
  for (int i = threadIdx.x; i < 192; i += blockDim.x) (&syn::s_kSigCtxN[0][0][0])[i] = (&syn::d_kSigCtxN[0][0][0])[i];
  for (int i = threadIdx.x; i < 768; i += blockDim.x) (&syn::s_kSbInv[0][0][0])[i] = (&syn::d_kSbInv[0][0][0])[i];
  for (int i = threadIdx.x; i < 4; i += blockDim.x) syn::s_kChromaTab[i] = syn::d_kChromaTab[i];
  for (int i = threadIdx.x; i < 4 * 3 * 64; i += blockDim.x) { (&syn::s_kScanX[0][0][0])[i] = (&syn::d_kScanX[0][0][0])[i]; (&syn::s_kScanY[0][0][0])[i] = (&syn::d_kScanY[0][0][0])[i]; }
  __syncthreads();
  // Every warp decodes one sub-stream at a time, all 32 lanes on identical data: CABAC is serial per sub-stream, and the
  // lanes share the per-cell / per-context / per-coefficient work around the bins (b200_hevc_syntax.h).  (Several decoders
  // per warp on diverged lanes were measured 25-70 % slower: the diverged paths of one warp serialise.)
  const int slot_w = threadIdx.x >> 5;
  const syn::CtxPtr ctx = (syn::CtxPtr)__cvta_generic_to_shared(s_ctx[slot_w]);
  for (;;) {
    unsigned slot = 0;
    if (lane0()) slot = atomicAdd(b.qhead, 1u);
    slot = __shfl_sync(0xffffffffu, slot, 0);
    if (slot >= (unsigned)b.nsubs) break;
    // the slot is filled when the sub-stream becomes ready (already, for those without prerequisites)
    unsigned item = e_poll(b.queue + slot);
    if (!item) {
      unsigned ns = 500, spins = 0;
      for (;;) {
        __nanosleep(ns); if (ns < 16000) ns <<= 1;
        if ((item = e_poll(b.queue + slot)) != 0u) break;
        if ((++spins & 31u) != 0) continue;
        if (e_poll(b.error_flag)) return;                // a producer failed: its dependants never become ready
        if (spins > (1u << 22)) { if (lane0()) atomicExch(b.error_flag, 3u); return; }
      }
    }
#ifdef B200_ENTROPY_TRACE
    if (lane0() && item - 1u < (unsigned)TRACE_CAP) { g_trace[item - 1u][0] = e_globaltimer(); g_trace_sm[item - 1u] = e_smid(); }
#endif
    const syn::Substream& gs = b.subs[item - 1u];
    const EntropyPic& ep = b.pics[gs.pic];
    DevSync& sync = s_sync[slot_w];
    sync.progress = b.progress + ep.progress_base; sync.sub_done = b.sub_done + ep.sub_base; sync.error_flag = b.error_flag;
    sync.queue = b.queue; sync.qtail = b.qtail; sync.deps = b.deps;
    sync.dense_tu = sync.dense_coef = sync.dense_tu_cap = sync.dense_coef_cap = 0; sync.end_bit_position = 0;
    syn::run_substream<Cfg>(s_dec[slot_w], ep.sp, ep.pb, b.subs + ep.sub_base, (int)(item - 1u - ep.sub_base), ctx, sync);
#ifdef B200_ENTROPY_TRACE
    if (lane0() && item - 1u < (unsigned)TRACE_CAP) g_trace[item - 1u][1] = e_globaltimer();
#endif
  }
}

#ifdef B200_ENTROPY_TRACE
// n records of {pop ns, end ns, SM} (3 x u64 each) of the last entropy launch; sub-streams past TRACE_CAP are not recorded
extern "C" int b200_debug_entropy_trace(unsigned long long* out, int n) {
  if (!out || n < 0 || n > TRACE_CAP) return set_error(B200_E_INVALID, "bad trace request");
  static unsigned long long t[TRACE_CAP][2]; static unsigned sm[TRACE_CAP];
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(t, g_trace, sizeof t);
  if (e == cudaSuccess) e = cudaMemcpyFromSymbol(sm, g_trace_sm, sizeof sm);
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "entropy trace: %s", cudaGetErrorString(e));
  for (int i = 0; i < n; i++) { out[3 * i] = t[i][0]; out[3 * i + 1] = t[i][1]; out[3 * i + 2] = sm[i]; }
  return B200_OK;
}
#endif

// sums the per-CTB TU / coefficient counts (statistics only: command-stream bytes actually produced)
__global__ void entropy_stats_kernel(const EntropyBatch b, unsigned long long* out2) {
  const int pi = blockIdx.y;
  const EntropyPic& ep = b.pics[pi];
  const int nctb = ep.sp.wctb * ep.sp.hctb;
  unsigned long long tus = 0, coefs = 0;
  for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < nctb; a += gridDim.x * blockDim.x) {
    const CtuInfo ci = ep.pb.ctus[a];
    tus += ci.tu_count;
    for (unsigned k = 0; k < ci.tu_count; k++) { const TuCmd t = ep.pb.tus[ci.tu_start + k]; coefs += (t.w3 & 0x7ff) + ((t.w3 >> 11) & 0x3ff) + ((t.w3 >> 21) & 0x3ff); }
  }
  atomicAdd(out2, tus); atomicAdd(out2 + 1, coefs);
}

// Tail overlap (b200_hevc_decode.cu): the stream that carries K1 passes this one-thread kernel first, so that K1's CTAs are
// handed to the SMs only after K0's whole grid is resident (every decoder warp has popped its first queue slot).  Purely
// a scheduling aid: it gives up after ~2 s (K0 kept off the SMs that long by other work of the process) and correctness never
// depends on it -- should K1 then take every SM slot first, its own dependency time-out turns the stall into an error.
__global__ void entropy_gate_kernel(const unsigned* qhead, unsigned need, const unsigned* error_flag) {
  for (unsigned spins = 0; spins < 2000000u; spins++) {
    if (e_ld_acquire(qhead) >= need || e_ld_acquire(error_flag)) return;
    __nanosleep(1000);
  }
}

int launch_entropy_gate(const EntropyBatch& b, int resident_warps, cudaStream_t s) {
  if (b.nsubs <= 0 || resident_warps <= 0) return B200_OK;
  entropy_gate_kernel<<<1, 1, 0, s>>>(b.qhead, (unsigned)(resident_warps < b.nsubs ? resident_warps : b.nsubs), b.error_flag);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "entropy gate launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

// resident CTAs per SM of the entropy kernel, before a caller's cap (EntropyBatch::blocks_per_sm).  common: every picture of
// the batch has the CfgCommon parameter combination -> the specialised (smaller) kernel
static int entropy_blocks_per_sm(bool common) {
  auto kern = common ? hevc_entropy_kernel<syn::CfgCommon> : hevc_entropy_kernel<syn::CfgRuntime>;
  int occ = 1; cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, EWARPS * 32, 0);
  if (occ < 1) occ = 1;
  if (B200_ENTROPY_MAX_BLOCKS_PER_SM > 0 && occ > B200_ENTROPY_MAX_BLOCKS_PER_SM) occ = B200_ENTROPY_MAX_BLOCKS_PER_SM;
  return occ;
}

int entropy_warps_per_sm(bool common) { return entropy_blocks_per_sm(common) * EWARPS; }

int launch_entropy(const EntropyBatch& b, cudaStream_t s, int* resident_warps) {
  if (resident_warps) *resident_warps = 0;
  if (b.nsubs <= 0) return B200_OK;
  int dev = 0, sms = 148; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  auto kern = b.common ? hevc_entropy_kernel<syn::CfgCommon> : hevc_entropy_kernel<syn::CfgRuntime>;
  int occ = entropy_blocks_per_sm(b.common != 0);
  if (b.blocks_per_sm > 0 && b.blocks_per_sm < occ) occ = b.blocks_per_sm;
  const int want = (b.nsubs + EWARPS - 1) / EWARPS;
  const int grid = want < sms * occ ? want : sms * occ;
  if (resident_warps) *resident_warps = grid * EWARPS;
  kern<<<grid, EWARPS * 32, 0, s>>>(b);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "entropy launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

int launch_entropy_stats(const EntropyBatch& b, unsigned long long* out2, cudaStream_t s) {
  if (b.npics <= 0) return B200_OK;
  entropy_stats_kernel<<<dim3(8, b.npics), 128, 0, s>>>(b, out2);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(B200_E_CUDA, "entropy stats launch: %s", cudaGetErrorString(e));
  return B200_OK;
}

}  // namespace b200
