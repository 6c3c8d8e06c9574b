// b200_hevc.h -- internal interfaces of the HEVC intra decoder (host front-end + device back-end)
#pragma once
#include "b200_internal.h"
#include "b200_hevc_types.h"
#include "b200_hevc_syntax.h"
#include "b200_hevc_scaling.h"
#include <vector>

namespace b200 {

struct ParseLimits { uint64_t max_image_size_pixels = 0; };   // heif_security_limits.max_image_size_pixels (0 = unlimited)

// Everything the slice data depends on, produced by the host from the headers alone (cheap, serial).
struct PictureHeaders {
  PicDesc desc;                          // dimensions, conformance window, tool flags (device pointers filled later)
  syn::SeqParams sp;
  std::vector<SliceInfo> slices;
  std::vector<syn::Substream> subs;      // CABAC sub-streams in decoding order
  std::vector<uint8_t> rbsp;             // slice-segment data of the picture, emulation prevention removed, zero padded
  std::vector<uint16_t> ctu_slice;       // slice index per CTB
  // VUI colour description as the libde265 plugin reports it (decoder_libde265.cc:426-448)
  int colour_primaries = 2, transfer_characteristics = 2, matrix_coefficients = 2, full_range = 0;
  bool scaling_enabled = false;          // scaling_list_enabled_flag: `scaling` holds the factors in effect (PPS > SPS > default lists, 7.4.5)
  sl::Factors scaling;
};

struct ParsedPicture {                   // host front-end result: headers + dense command stream
  PictureHeaders hdr;
  PicDesc desc;
  std::vector<CtuInfo> ctus;
  std::vector<TuCmd> tus; size_t n_tus = 0;          // vectors are capacity buffers; n_* entries are valid
  std::vector<CoefEntry> coefs; size_t n_coefs = 0;
  std::vector<SliceInfo> slices;
  std::vector<int8_t> qp8;
  std::vector<uint8_t> edge8, ipm4, cd8, wpp_ctx, end_state;
};

// Host front-end.  Thread-safe (no shared state).
int parse_headers(const uint8_t* data, size_t size, const ParseLimits& limits, PictureHeaders& out);
int parse_access_unit(const uint8_t* data, size_t size, const ParseLimits& limits, ParsedPicture& out);

// Device back-end (b200_hevc_recon.cu / b200_hevc_filters.cu).  All arrays are batch-wide device buffers.
struct DeviceBatch {
  const PicDesc* pics; int npics;
  const CtuInfo* ctus; const TuCmd* tus; const CoefEntry* coefs; const SliceInfo* slices;
  const int8_t* qp8; const uint8_t* edge8;
  const uint8_t* scaling;        // sl::Factors of the pictures that use scaling lists (PicDesc::scaling_idx)
  unsigned int* progress;        // two counters (luma, chroma) per CTB row of every picture, zeroed before launch
  const unsigned int* entropy_progress;   // K0's counters of the same rows when K0 runs CONCURRENTLY (nullptr: command stream complete)
  int blocks_per_sm;             // > 0: cap of resident CTAs per SM (co-residency with K0)
  unsigned int* ticket;          // work-distribution counter, zeroed before launch
  unsigned int* error_flag;      // set by a kernel that gave up waiting (zeroed before launch)
  const uint2* row_list;         // (picture, ctb row | component group << 31) in launch order
  int nrows;                     // work items: CTB rows x component groups (luma; Cb + Cr)
  int wide_samples;              // 1: planes hold uint16 samples (bit depth > 8)
  int max_log2_ctb;              // largest CTB size of the batch (sizes the per-warp shared memory)
};
// Device front-end (b200_hevc_entropy.cu)
enum { MAX_CHUNKS = 16 };   // row bands of a large grid that leave the pipeline one after the other (b200_hevc_decode.cu)
struct EntropyPic { syn::SeqParams sp; syn::PicBuffers pb; uint32_t progress_base, sub_base; };
struct EntropyBatch {
  const EntropyPic* pics; int npics;
  const syn::Substream* subs;    // batch-wide, grouped per picture (EntropyPic::sub_base)
  int nsubs;
  // ready queue: queue[0 .. nsubs) holds (batch-wide sub-stream index + 1), 0 = not yet pushed; qhead / qtail are the pop and
  // push cursors; deps[i] counts the events sub-stream i still waits for (wake_* links in syn::Substream are batch-wide)
  unsigned int* queue; unsigned int* qhead; unsigned int* qtail; unsigned int* deps;
  unsigned int* progress; unsigned int* sub_done; unsigned int* error_flag;
  int blocks_per_sm;             // > 0: cap of resident CTAs per SM (co-residency with K1)
  int common;                    // 1: every picture matches syn::CfgCommon (specialised kernel)
};
int entropy_warps_per_sm(bool common);    // resident K0 decoders (warps) per SM at full occupancy (common: the CfgCommon instantiation)
int launch_entropy(const EntropyBatch& b, cudaStream_t s, int* resident_warps = nullptr);   // resident_warps: decoders of the launched grid (all co-resident)
int launch_entropy_gate(const EntropyBatch& b, int resident_warps, cudaStream_t s);            // returns (in stream order) once every K0 warp has taken its first sub-stream
int launch_entropy_stats(const EntropyBatch& b, unsigned long long* out2, cudaStream_t s);
int launch_recon(const DeviceBatch& b, cudaStream_t s);
int launch_deblock(const DeviceBatch& b, const PicDesc* host_pics, cudaStream_t s);
int launch_sao(const DeviceBatch& b, const PicDesc* host_pics, cudaStream_t s, int* launches = nullptr);

}  // namespace b200
