// b200_hevc_types.h -- command stream between the entropy stage (K0 on the GPU, b200_hevc_entropy.cu; or the same
// syntax decoder on the host, b200_hevc_parse.cc) and the sm_90a reconstruction kernels (b200_hevc_recon.cu,
// b200_hevc_filters.cu).  Plain PODs, identical on host and device.
//
// Division of labour: NAL / parameter-set / slice-header parsing runs on the host (microseconds per tile); everything
// that is serial per CABAC sub-stream -- the arithmetic decoder, the coding quadtree syntax, intra-mode (MPM) and QP
// derivation -- produces this stream (BASELINE.json's north_star put it on the host; the GPU box has 16 usable cores, so
// it is on the GPU, one warp per sub-stream: SURVEY 8(f) N1); everything per-sample -- scaling, inverse DCT/DST, intra
// prediction, reconstruction, deblocking, SAO, conformance crop + paste -- consumes it.
#pragma once
#include <cstdint>

namespace b200 {

// One transform unit in decoding order (z-order inside a CTU).  16 bytes.  In 4:2:2 / 4:4:4 pictures every BLOCK is a command of its
// own: the luma block (chroma_here = 0) and then each chroma block, laid out like a luma one (cbf in bit 26, transform skip in bit 30,
// its intra mode in luma_mode, nnz in w3[0:11)) with the component in w1[23:25) and its LUMA location as position.
//  w0: x4[0:12) y4[12:24) log2m2[24:26) cbf_luma[26] cbf_cb[27] cbf_cr[28] chroma_here[29] ts_luma[30] ts_cb[31]
//  w1: luma_mode[0:6) chroma_mode[6:12) qpy+64 [12:20) ts_cr[20] pcm[21] cu_transquant_bypass[22] component[23:25)
//  w2: index of this TU's first coefficient entry (relative to the picture's coefficient base)
//  w3: nnz_luma[0:11) nnz_cb[11:21) nnz_cr[21:31)
// x4,y4: luma position of the luma transform block in 4-sample units.  When log2 size is 2 and chroma_here is set,
// the chroma blocks are the 4x4 blocks of the parent 8x8 node (blkIdx 3 rule, H.265 7.3.8.10).
struct TuCmd { uint32_t w0, w1, w2, w3; };

// One coefficient: position inside the transform block (y * nTbS + x) and the parsed level (TransCoeffLevel).
struct CoefEntry { uint16_t pos; int16_t level; };

// SAO parameters of one CTB component (H.265 7.4.9.3): 8 bytes.
struct SaoComp { uint8_t type; uint8_t band_or_class; int8_t offset[4]; uint8_t pad[2]; };

// One CTU: 40 bytes.
struct alignas(8) CtuInfo {
  uint32_t tu_start;     // first TuCmd of this CTU, relative to the picture's TU base
  uint16_t tu_count;
  uint16_t slice_idx;    // index into the picture's region table (SliceInfo)
  SaoComp sao[3];
  uint32_t pad[2];
};

// One REGION of a picture = the CTBs of one slice inside one tile (without HEVC tiles: one slice).  Availability (6.4.1) is
// "same region"; a slice that spans several tiles appears once per tile with the same parameters.  16 bytes.
struct SliceInfo {
  int8_t cb_qp_offset, cr_qp_offset;     // pps + slice offsets used for dequantisation (8.6.1)
  int8_t beta_offset, tc_offset;         // slice_beta_offset_div2 * 2, slice_tc_offset_div2 * 2
  uint8_t deblocking_disabled, lf_across_slices;
  uint16_t slice_id;                     // index of the slice in decoding order (in-loop filter rules compare slices, not regions)
  uint32_t first_ctb_rs;
  uint16_t tile_id;                      // TileId of the region's CTBs (0 without tiles)
  uint8_t lf_across_tiles;               // loop_filter_across_tiles_enabled_flag
  uint8_t pad;
};

// Per 8x8 luma block (one byte each in two maps):
//   qp8  : QpY of the coding unit covering the block (int8)
//   edge8: bit0 = left edge is a filtered transform edge, bit1 = top edge is one (slice / picture rules applied, bS = 2)
// Because transform blocks are aligned to their size, an edge on the 8x8 grid is uniform along the 8 samples.

struct PicDesc {         // one per picture (tile) of a batch
  int32_t width, height;             // coded luma size (multiple of MinCbSizeY)
  int32_t log2_ctb, wctb, hctb;
  int32_t bit_depth, chroma;         // chroma = chroma_format_idc: 0 = 4:0:0, 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4
  int32_t crop_x, crop_y, out_w, out_h;   // conformance window in luma samples
  int32_t strong_intra, pps_cb_qp_offset, pps_cr_qp_offset, sao_enabled;
  int32_t log2_sao_scale_luma, log2_sao_scale_chroma;
  int32_t nslices;
  // bases into the batch-wide arrays
  uint32_t ctu_base, tu_base, slice_base, map8_base;
  uint64_t coef_base;
  int32_t w8, h8;                    // map8 dimensions
  // device planes: reconstruction (pre/post deblocking, in place) and destination (after SAO + crop)
  void* rec[3]; int32_t rec_stride[3];           // strides in samples
  void* dst[3]; int32_t dst_stride[3];           // dst already offset to the paste position
  uint32_t progress_base;            // first per-CTB-row progress counter of this picture
  int32_t scaling_idx;               // index of the picture's scaling factors (sl::Factors, 780 bytes each) in the batch-wide array; -1: flat (m = 16)
};

}  // namespace b200
