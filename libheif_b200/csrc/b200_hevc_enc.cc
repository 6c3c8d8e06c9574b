// b200_hevc_enc.cc -- host-side HEVC intra-only encoder (fixture generator / heif_encoder_plugin back end).
//
// Role in the reference: the x265 plugin (libheif/plugins/encoder_x265.cc:752-1051 encode_image,
// :1186-1244 get_compressed_data) as driven by Encoder_HEVC::encode (libheif/codecs/hevc_enc.cc:33-115):
// one call per image/tile, output = VPS, SPS, PPS and slice NAL units without start codes.
// x265 is absent from this image, so synthetic inputs for the decoder (BASELINE configs 2-5, SURVEY 8d) are
// produced by this closed-loop encoder.  It is deliberately simple (no RDO) but emits every syntax element
// the decoder supports: CTB 16/32/64, CU quadtree, 2Nx2N / NxN, all 35 intra modes, TU trees with TB 4..32,
// DST 4x4, transform skip, sign-data hiding, cu_qp_delta, chroma QP offsets, SAO band/edge with merges,
// deblocking overrides, WPP entry points, multiple slices and dependent slice segments, 8..12 bit,
// 4:2:0 and 4:0:0.  Syntax follows ITU-T H.265 7.3 / 9.3; the reconstruction loop follows 8.4 / 8.6.
// The arithmetic coder, residual_coding() and intra mode signalling (b200_hevc_enc_cabac.h) and the prediction, transform
// and (de)quantisation arithmetic (b200_hevc_enc_recon.h) are the ones the GPU encoder uses too; transform skip,
// cu_transquant_bypass, sign-data hiding, scaling lists and PCM are this encoder's alone.  The parameter sets and slice
// header come from b200_hevc_enc_headers.h.
#define B200_SYNTAX_HOST_ONLY 1   // this translation unit uses the shared encoder / syntax code on the host only
#include "b200_hevc_enc_cabac.h"
#include "b200_hevc_enc_headers.h"
#include "b200_hevc_enc_recon.h"
#include <algorithm>
#include <vector>

namespace b200 {
namespace enc {

using namespace syn;

// ------------------------------------------------------------------------------------------ NAL framing
void append_nal(std::vector<uint8_t>& out, int type, const std::vector<uint8_t>& rbsp) {
  std::vector<uint8_t> nal;
  nal.reserve(rbsp.size() + rbsp.size() / 64 + 2);
  nal.push_back((uint8_t)(type << 1)); nal.push_back(1);
  int zeros = 0;
  for (uint8_t b : rbsp) {
    if (zeros >= 2 && b <= 3) { nal.push_back(3); zeros = 0; }
    nal.push_back(b);
    zeros = b == 0 ? zeros + 1 : 0;
  }
  uint32_t n = (uint32_t)nal.size();
  out.push_back((uint8_t)(n >> 24)); out.push_back((uint8_t)(n >> 16)); out.push_back((uint8_t)(n >> 8)); out.push_back((uint8_t)n);
  out.insert(out.end(), nal.begin(), nal.end());
}
size_t escaped_size(const uint8_t* d, size_t len) {
  size_t n = 0; int zeros = 0;
  for (size_t i = 0; i < len; i++) { const uint8_t b = d[i]; if (zeros >= 2 && b <= 3) { n++; zeros = 0; } n++; zeros = b == 0 ? zeros + 1 : 0; }
  return n;
}

// ------------------------------------------------------------------------------------------ parameter sets, slice header
static void write_scaling_list_data(BitWriter& b, const SeqHeader& s) {          // 7.3.4
  for (int sz = 0; sz < 4; sz++) for (int m = 0; m < 6; m += (sz == 3 ? 3 : 1)) {
    if (s.sl_kind[sz][m] < 2) { b.put(0, 1); b.ue(s.sl_kind[sz][m]); continue; }   // pred_mode_flag = 0: delta 0 = default, 1 = previous matrix
    b.put(1, 1);
    int next = 8; const int num = sz == 0 ? 16 : 64;
    if (sz > 1) { b.se((int)s.sl_lists->dc[sz][m] - 8); next = s.sl_lists->dc[sz][m]; }
    for (int i = 0; i < num; i++) { int d = (int)s.sl_lists->list[sz][m][i] - next; if (d > 127) d -= 256; if (d < -128) d += 256; b.se(d); next = s.sl_lists->list[sz][m][i]; }
  }
}

static void profile_tier_level(BitWriter& b, const SeqHeader& s) {
  const b200_hevc_enc_params& P = *s.P;
  const int cfmt = s.cfmt, bd = s.bd, chroma = s.chroma;
  int profile = cfmt >= 2 ? 4 : (bd == 8 ? (P.still_picture ? 3 : 1) : (bd == 10 && chroma ? 2 : 4));
  b.put(0, 2); b.put(0, 1); b.put(profile, 5);
  uint32_t compat = 0;
  if (profile == 1) compat = (1u << 30) | (1u << 29);       // Main => also Main 10 compatible
  else if (profile == 2) compat = 1u << 29;
  else if (profile == 3) compat = (1u << 28) | (1u << 30) | (1u << 29);
  else compat = 1u << 27;
  b.put(compat, 32);
  b.put(1, 1); b.put(0, 1); b.put(0, 1); b.put(1, 1);        // progressive, !interlaced, !non_packed, frame_only
  if (profile == 4) {                                         // RExt constraint flags: Main 12 / Monochrome 12 family
    b.put(1, 1);                                              // max_12bit_constraint
    b.put(bd <= 10, 1); b.put(bd <= 8, 1);                    // max_10bit, max_8bit
    b.put(cfmt <= 2, 1); b.put(cfmt <= 1, 1); b.put(chroma == 0, 1);   // max_422chroma, max_420chroma, max_monochrome
    b.put(1, 1); b.put(1, 1); b.put(1, 1);                    // intra, one_picture_only, lower_bit_rate
    b.put(0, 32); b.put(0, 2);                                // reserved 34 bits
  } else { b.put(0, 32); b.put(0, 11); }
  b.put(0, 1);                                                // general_inbld / reserved
  long px = (long)s.W * s.H;
  int level = px <= 36864 ? 30 : px <= 122880 ? 60 : px <= 245760 ? 63 : px <= 552960 ? 90 : px <= 983040 ? 93 :
              px <= 2228224 ? 120 : px <= 8912896 ? 150 : 180;
  b.put(level, 8);
}

void write_vps(std::vector<uint8_t>& out, const SeqHeader& s) {
  BitWriter b;
  b.put(0, 4); b.put(1, 1); b.put(1, 1); b.put(0, 6); b.put(0, 3); b.put(1, 1); b.put(0xffff, 16);
  profile_tier_level(b, s);
  b.put(1, 1);                      // sub_layer_ordering_info_present
  b.ue(0); b.ue(0); b.ue(0);        // max_dec_pic_buffering_minus1, num_reorder, max_latency
  b.put(0, 6); b.ue(0);             // max_layer_id, num_layer_sets_minus1
  b.put(0, 1);                      // timing_info_present
  b.put(0, 1);                      // extension
  b.trailing();
  append_nal(out, 32, b.buf);
}

void write_sps(std::vector<uint8_t>& out, const SeqHeader& s) {
  const b200_hevc_enc_params& P = *s.P;
  BitWriter b;
  b.put(0, 4); b.put(0, 3); b.put(1, 1);
  profile_tier_level(b, s);
  b.ue(0);
  b.ue(s.cfmt);
  if (s.cfmt == 3) b.put(0, 1);                                 // separate_colour_plane_flag
  b.ue(s.W); b.ue(s.H);
  int cr = (s.W - P.width) >> (s.chroma ? s.sx : 0), cbm = (s.H - P.height) >> (s.chroma ? s.sy : 0);     // conformance window in chroma units
  if (cr || cbm) { b.put(1, 1); b.ue(0); b.ue(cr); b.ue(0); b.ue(cbm); } else b.put(0, 1);
  b.ue(s.bd - 8); b.ue(s.bd - 8);
  b.ue(4);                          // log2_max_pic_order_cnt_lsb_minus4
  b.put(1, 1); b.ue(0); b.ue(0); b.ue(0);
  b.ue(0);                          // log2_min_luma_coding_block_size_minus3 (8)
  b.ue(s.log2ctb - 3);
  b.ue(s.log2_min_tb - 2); b.ue(s.log2_max_tb - s.log2_min_tb);
  b.ue(0); b.ue(s.max_th_depth);
  b.put(s.sl_on ? 1 : 0, 1);        // scaling_list_enabled
  if (s.sl_on) { b.put(P.scaling_lists == 2 ? 1 : 0, 1); if (P.scaling_lists == 2) write_scaling_list_data(b, s); }
  b.put(0, 1);                      // amp
  b.put(P.sao ? 1 : 0, 1);
  b.put(P.pcm ? 1 : 0, 1);          // pcm_enabled
  if (P.pcm) {
    b.put(s.pcm_bd_y - 1, 4); b.put(s.pcm_bd_c - 1, 4);
    b.ue(0); b.ue(std::min(5, s.log2ctb) - 3);                    // Log2MinIpcmCbSizeY = 3, Log2MaxIpcmCbSizeY = min(CtbLog2SizeY, 5)
    b.put(P.pcm == 2 ? 1 : 0, 1);                                 // pcm_loop_filter_disabled_flag
  }
  b.ue(0);                          // num_short_term_ref_pic_sets
  b.put(0, 1);                      // long_term_ref_pics_present
  b.put(0, 1);                      // temporal_mvp
  b.put(P.strong_intra_smoothing ? 1 : 0, 1);
  if (P.vui_present) {
    b.put(1, 1);
    b.put(0, 1); b.put(0, 1);       // aspect_ratio_info, overscan_info
    b.put(1, 1);                    // video_signal_type_present
    b.put(5, 3); b.put(P.full_range ? 1 : 0, 1);
    if (P.colour_description_present) { b.put(1, 1); b.put(P.colour_primaries, 8); b.put(P.transfer_characteristics, 8); b.put(P.matrix_coefficients, 8); }
    else b.put(0, 1);
    b.put(0, 1); b.put(0, 1); b.put(0, 1); b.put(0, 1);   // chroma_loc, neutral_chroma, field_seq, frame_field_info
    b.put(0, 1); b.put(0, 1); b.put(0, 1);                // default_display_window, timing_info, bitstream_restriction
  } else b.put(0, 1);
  b.put(0, 1);                      // sps_extension_present
  b.trailing();
  append_nal(out, 33, b.buf);
}

void write_pps(std::vector<uint8_t>& out, const SeqHeader& s) {
  const b200_hevc_enc_params& P = *s.P;
  BitWriter b;
  b.ue(0); b.ue(0);
  b.put(P.dependent_slice_segments ? 1 : 0, 1);
  b.put(0, 1); b.put(0, 3);
  b.put(P.sign_data_hiding ? 1 : 0, 1);
  b.put(0, 1);
  b.ue(0); b.ue(0);
  b.se(P.init_qp - 26);
  b.put(0, 1);                      // constrained_intra_pred
  b.put(P.transform_skip ? 1 : 0, 1);
  b.put(P.cu_qp_delta ? 1 : 0, 1);
  if (P.cu_qp_delta) b.ue(s.log2ctb - s.qg_log2);
  b.se(P.cb_qp_offset); b.se(P.cr_qp_offset);
  b.put(P.slice_chroma_qp_offsets ? 1 : 0, 1);
  b.put(0, 1); b.put(0, 1);
  b.put(P.transquant_bypass ? 1 : 0, 1);   // transquant_bypass_enabled
  b.put(s.tiles ? 1 : 0, 1);        // tiles_enabled_flag
  b.put(P.wpp ? 1 : 0, 1);
  if (s.tiles) {
    const std::vector<int>& col_bd = *s.col_bd; const std::vector<int>& row_bd = *s.row_bd;
    b.ue((unsigned)col_bd.size() - 2); b.ue((unsigned)row_bd.size() - 2);
    b.put(P.tiles_uniform ? 1 : 0, 1);
    if (!P.tiles_uniform) {
      for (size_t i = 0; i + 2 < col_bd.size(); i++) b.ue((unsigned)(col_bd[i + 1] - col_bd[i] - 1));
      for (size_t i = 0; i + 2 < row_bd.size(); i++) b.ue((unsigned)(row_bd[i + 1] - row_bd[i] - 1));
    }
    b.put(P.loop_filter_across_tiles ? 1 : 0, 1);
  }
  b.put(P.loop_filter_across_slices ? 1 : 0, 1);
  b.put(1, 1);                      // deblocking_filter_control_present
  b.put(1, 1);                      // deblocking_filter_override_enabled
  b.put(P.deblocking_disabled ? 1 : 0, 1);
  if (!P.deblocking_disabled) { b.se(P.beta_offset_div2); b.se(P.tc_offset_div2); }
  b.put(P.scaling_lists == 3 ? 1 : 0, 1);   // pps_scaling_list_data_present
  if (P.scaling_lists == 3) write_scaling_list_data(b, s);
  b.put(0, 1);                      // lists_modification_present
  b.ue(0);                          // log2_parallel_merge_level_minus2
  b.put(0, 1);                      // slice_segment_header_extension_present
  b.put(0, 1);                      // pps_extension_present
  b.trailing();
  append_nal(out, 34, b.buf);
}

void write_slice_header(BitWriter& b, const SeqHeader& s, int addr0, bool dependent, int slice_qp, const std::vector<size_t>& escaped) {
  const b200_hevc_enc_params& P = *s.P;
  const int total = ((s.W + (1 << s.log2ctb) - 1) >> s.log2ctb) * ((s.H + (1 << s.log2ctb) - 1) >> s.log2ctb);
  bool first = addr0 == 0;
  b.put(first ? 1 : 0, 1);
  b.put(0, 1);                                           // no_output_of_prior_pics (IRAP)
  b.ue(0);
  if (!first) {
    if (P.dependent_slice_segments) b.put(dependent ? 1 : 0, 1);
    int bits = 0; while ((1 << bits) < total) bits++;
    b.put(addr0, bits);
  }
  if (!dependent) {
    b.ue(2);                                             // slice_type I
    if (P.sao) { b.put(1, 1); if (s.chroma) b.put(1, 1); }
    b.se(slice_qp - P.init_qp);
    if (P.slice_chroma_qp_offsets) { b.se(P.slice_cb_qp_offset); b.se(P.slice_cr_qp_offset); }
    bool override = P.slice_deblocking_override != 0;
    b.put(override ? 1 : 0, 1);
    bool dis = P.deblocking_disabled;
    if (override) {
      dis = P.slice_deblocking_disabled != 0;
      b.put(dis ? 1 : 0, 1);
      if (!dis) { b.se(P.slice_beta_offset_div2); b.se(P.slice_tc_offset_div2); }
    }
    if (P.loop_filter_across_slices && (P.sao || !dis)) b.put(P.slice_loop_filter_across_slices ? 1 : 0, 1);
  }
  if (P.wpp || s.tiles) {
    int ne = (int)escaped.size() - 1;
    b.ue(ne);
    if (ne > 0) { b.ue(31); for (int i = 0; i < ne; i++) b.put((unsigned)(escaped[i] - 1), 32); }
  }
  b.trailing();                                          // byte_alignment()
}

struct Lcg { uint32_t s; uint32_t next() { s = s * 1664525u + 1013904223u; return s >> 8; } int range(int n) { return (int)(next() % (uint32_t)n); } };

struct SaoParams { int type[3], band_pos[3], eo_class[3], abs[3][4], sign[3][4]; int merge_left, merge_up; };

// ------------------------------------------------------------------------------------------ encoder
class Encoder {
 public:
  Encoder(const b200_hevc_enc_params& p, const uint16_t* const src[3], const int stride[3]) : P(p) {
    W = (p.width + 7) & ~7; H = (p.height + 7) & ~7;       // multiples of MinCbSizeY (8); conformance window crops
    cfmt = p.chroma_format_idc; chroma = cfmt ? 1 : 0;
    sx = (cfmt == 1 || cfmt == 2) ? 1 : 0; sy = cfmt == 1 ? 1 : 0;       // SubWidthC = 1 << sx, SubHeightC = 1 << sy (Table 6-1)
    Wc = chroma ? W >> sx : 0; Hc = chroma ? H >> sy : 0;
    log2ctb = p.log2_ctb_size; ctb = 1 << log2ctb;
    wctb = (W + ctb - 1) >> log2ctb; hctb = (H + ctb - 1) >> log2ctb;
    w4 = W / 4; h4 = H / 4;
    bd = p.bit_depth;
    for (int c = 0; c < (chroma ? 3 : 1); c++) {
      int pw = c ? Wc : W, ph = c ? Hc : H, sw = c ? (p.width + (1 << sx) - 1) >> sx : p.width, sh = c ? (p.height + (1 << sy) - 1) >> sy : p.height;
      org[c].assign((size_t)pw * ph, 0); rec[c].assign((size_t)pw * ph, 0);
      for (int y = 0; y < ph; y++) for (int x = 0; x < pw; x++)
        org[c][(size_t)y * pw + x] = src[c][(size_t)std::min(y, sh - 1) * stride[c] + std::min(x, sw - 1)];   // edge padding
    }
    slice_of4.assign((size_t)w4 * h4, 0); ipm4.assign((size_t)w4 * h4, 1); qp4.assign((size_t)w4 * h4, 0); cd4.assign((size_t)w4 * h4, 0);
    rng.s = p.seed ? p.seed : 0xB200u;
    log2_min_tb = 2; log2_max_tb = std::min(5, log2ctb);
    max_th_depth = clip3(0, 4, p.max_transform_hierarchy_depth_intra);
    qg_log2 = log2ctb - clip3(0, log2ctb - 3, p.diff_cu_qp_delta_depth);
    // scaling lists (7.3.4): what gets coded (or defaulted) and the factors the closed-loop reconstruction uses
    sl::set_all_default(sl_lists);
    if (p.scaling_lists >= 2) {
      for (int s = 0; s < 4; s++) for (int m = 0; m < 6; m += (s == 3 ? 3 : 1)) {
        const int kind = (int)rng.range(4);                       // 0 default, 1 copy of the previous matrix, 2/3 explicit
        sl_kind[s][m] = (uint8_t)((kind == 1 && m == 0) ? 0 : (kind >= 2 ? 2 : kind));
        if (sl_kind[s][m] == 0) sl::set_default(sl_lists, s, m);
        else if (sl_kind[s][m] == 1) { const int ref = m - (s == 3 ? 3 : 1); memcpy(sl_lists.list[s][m], sl_lists.list[s][ref], 64); sl_lists.dc[s][m] = sl_lists.dc[s][ref]; }
        else {
          const int num = s == 0 ? 16 : 64; int v = 8 + (int)rng.range(16);
          if (s > 1) sl_lists.dc[s][m] = (uint8_t)(8 + rng.range(40));
          for (int i = 0; i < num; i++) { v = clip3(1, 255, v + (int)rng.range(7) - 2); sl_lists.list[s][m][i] = (uint8_t)v; }
        }
      }
    }
    {
      const int tc = std::max(1, std::min(p.tile_cols, wctb)), tr = std::max(1, std::min(p.tile_rows, hctb));
      tiles = (tc > 1 || tr > 1) && !p.wpp;
      if (tiles) {
        auto bounds = [&](int n, int size) {
          std::vector<int> b(1, 0);
          if (p.tiles_uniform) for (int i = 1; i <= n; i++) b.push_back((i * size) / n);               // 6.5.1 (6-3)
          else { std::vector<int> cuts; while ((int)cuts.size() < n - 1) { int c = 1 + (int)rng.range(size - 1); if (std::find(cuts.begin(), cuts.end(), c) == cuts.end()) cuts.push_back(c); }
                 std::sort(cuts.begin(), cuts.end()); for (int c : cuts) b.push_back(c); b.push_back(size); }
          return b;
        };
        col_bd = bounds(tc, wctb); row_bd = bounds(tr, hctb);
      }
    }
    pcm_bd_y = p.pcm == 2 ? bd - 1 : bd; pcm_bd_c = p.pcm == 2 ? bd - 2 : bd;
    sl_on = p.scaling_lists != 0;
    if (sl_on) sl::derive(sl_lists, sl_f);
  }

  void encode(std::vector<uint8_t>& out) {
    write_vps(out); write_sps(out); write_pps(out);
    int rows_per_slice = P.slice_ctb_rows > 0 ? P.slice_ctb_rows : hctb;
    slice_idx = 0; region_idx = 0;
    ctb_region.assign((size_t)wctb * hctb, -1);
    if (tiles) {
      // CTBs in tile scan (6.5.1): tile after tile in raster order of the tiles, raster inside each tile
      std::vector<int> order, tile_start;
      for (size_t tr = 0; tr + 1 < row_bd.size(); tr++) for (size_t tc = 0; tc + 1 < col_bd.size(); tc++) {
        tile_start.push_back((int)order.size());
        for (int y = row_bd[tr]; y < row_bd[tr + 1]; y++) for (int x = col_bd[tc]; x < col_bd[tc + 1]; x++) order.push_back(y * wctb + x);
      }
      tile_start.push_back((int)order.size());
      if (P.slice_per_tile) {
        for (size_t t = 0; t + 1 < tile_start.size(); t++) {
          std::vector<int> o(order.begin() + tile_start[t], order.begin() + tile_start[t + 1]);
          encode_slice_segment_list(out, o, {0, (int)o.size()}, false, o[0]);
          slice_idx++;
        }
      } else encode_slice_segment_list(out, order, tile_start, false, 0);
      return;
    }
    for (int r0 = 0; r0 < hctb; r0 += rows_per_slice) {
      int r1 = std::min(hctb, r0 + rows_per_slice);
      if (P.dependent_slice_segments && P.wpp == 0 && r1 - r0 > 1) {
        // split the slice into an independent segment and dependent segments, one CTB row each
        for (int r = r0; r < r1; r++) encode_slice_segment(out, r * wctb, (r + 1) * wctb, r != r0, r0 * wctb);
      } else encode_slice_segment(out, r0 * wctb, r1 * wctb, false, r0 * wctb);
      slice_idx++;
    }
  }

  const std::vector<uint16_t>& recon(int c) const { return rec[c]; }
  int coded_w() const { return W; } int coded_h() const { return H; }
  // test-only: the levels of the first `count` transform-coded blocks of 8x8 and larger of every component become the
  // top-left n x n of `pattern` (32 x 32, raster), whatever quantisation gave; the reconstruction follows those levels
  void force_levels(const int16_t* pattern, int count) { forced = pattern; forced_left[0] = forced_left[1] = forced_left[2] = count; }

 private:
  b200_hevc_enc_params P;
  int cfmt = 1, sx = 1, sy = 1;
  int W, H, Wc, Hc, chroma, log2ctb, ctb, wctb, hctb, w4, h4, bd, log2_min_tb, log2_max_tb, max_th_depth, qg_log2;
  std::vector<uint16_t> org[3], rec[3];
  std::vector<uint16_t> slice_of4; std::vector<uint8_t> ipm4, cd4; std::vector<int8_t> qp4;
  Lcg rng;
  uint8_t ctx[CTX_COUNT], ctx_wpp[CTX_COUNT];          // context states, pStateIdx << 1 | valMps
  CabacWriter<BitWriter> cabac{BitWriter(), ctx};
  std::vector<SaoParams> sao;
  int slice_idx = 0, slice_addr_rs = 0, slice_qp = 26;
  int region_idx = 0;                                  // counts (slice, tile) regions: availability = same region
  bool tiles = false; std::vector<int> col_bd, row_bd;   // tile column / row boundaries in CTBs (6.5.1)
  std::vector<int> ctb_region;                         // region of every coded CTB (SAO merge candidates)
  int is_qp_delta_coded = 0, cu_qp_delta_val = 0, qpy_prev_qg = 0, last_cu_qpy = 0, first_qg = 1, cur_qpy = 0, qg_target_qp = 0;
  int cu_x0 = 0, cu_y0 = 0;
  sl::Lists sl_lists; sl::Factors sl_f; uint8_t sl_kind[4][6] = {}; bool sl_on = false;
  int pcm_bd_y = 8, pcm_bd_c = 8; bool cu_bypass = false;
  const int16_t* forced = nullptr; int forced_left[3] = {0, 0, 0};

  int scaling_factor(int c, int log2n, int pos) const {          // m[x][y] of 8.6.4.2 for raster position pos of an n x n block
    if (!sl_on) return 16;
    const int n = 1 << log2n, x = pos & (n - 1), y = pos >> log2n, sid = log2n - 2;
    if (sid == 0) return sl_f.m[c][0][y * 4 + x];
    if (pos == 0 && sid >= 2) return sl_f.dc[c][sid];
    return sl_f.m[c][sid][((y >> (log2n - 3)) << 3) + (x >> (log2n - 3))];
  }

  int stride_of(int c) const { return c ? Wc : W; }
  bool avail(int x, int y) const {
    if (x < 0 || y < 0 || x >= W || y >= H) return false;
    unsigned s = slice_of4[(size_t)(y >> 2) * w4 + (x >> 2)];      // 1 + region (slice x tile) of a decoded block: 6.4.1 wants same slice AND same tile
    return s != 0 && s == (unsigned)(region_idx + 1);
  }

  // ---------------------------------------------------------------------------- parameter sets
  SeqHeader seq_header() const {
    return SeqHeader{&P, W, H, cfmt, chroma, sx, sy, bd, log2ctb, log2_min_tb, log2_max_tb, max_th_depth, qg_log2, pcm_bd_y, pcm_bd_c,
                     sl_on, sl_kind, &sl_lists, tiles, &col_bd, &row_bd};
  }
  void write_vps(std::vector<uint8_t>& out) { enc::write_vps(out, seq_header()); }
  void write_sps(std::vector<uint8_t>& out) { enc::write_sps(out, seq_header()); }
  void write_pps(std::vector<uint8_t>& out) { enc::write_pps(out, seq_header()); }

  // ---------------------------------------------------------------------------- slice segment
  void encode_slice_segment(std::vector<uint8_t>& out, int addr0, int addr1, bool dependent, int slice_addr) {
    std::vector<int> order; for (int a = addr0; a < addr1; a++) order.push_back(a);
    encode_slice_segment_list(out, order, {0, (int)order.size()}, dependent, slice_addr);
  }
  // order: raster addresses of the segment's CTBs in coding order; starts: indices into `order` where a tile begins (+ the end)
  void encode_slice_segment_list(std::vector<uint8_t>& out, const std::vector<int>& order, const std::vector<int>& starts, bool dependent, int slice_addr) {
    slice_addr_rs = slice_addr;
    const int addr0 = order.front();
    int total = wctb * hctb;
    if (!dependent) {
      slice_qp = clip3(0, 51, P.qp + (slice_idx ? (int)(rng.range(5)) - 2 : 0));
      init_contexts(ctx, slice_qp);
      last_cu_qpy = slice_qp; first_qg = 1;
      region_idx++;
    }
    if (sao.empty()) sao.resize((size_t)total);
    // slice data: one CABAC sub-stream per CTB row when WPP is on, one per tile when tiles are on
    std::vector<std::vector<uint8_t>> substreams;
    cabac = {BitWriter(), ctx};
    size_t next_start = 1;
    for (size_t k = 0; k < order.size(); k++) {
      const int a = order[k];
      int rx = a % wctb, ry = a / wctb;
      if (tiles && next_start + 1 < starts.size() && (int)k == starts[next_start]) {      // first CTB of the next tile: 9.3.1 initialisation
        next_start++;
        init_contexts(ctx, slice_qp); first_qg = 1; region_idx++;
      }
      if (P.wpp && rx == 0 && a != addr0) {
        if (avail((rx + 1) << log2ctb, (ry - 1) << log2ctb)) memcpy(ctx, ctx_wpp, sizeof ctx); else init_contexts(ctx, slice_qp);
        first_qg = 1;
      }
      ctb_region[(size_t)a] = region_idx;
      if (P.sao) { choose_sao(rx, ry); write_sao(rx, ry); }
      coding_quadtree(rx << log2ctb, ry << log2ctb, log2ctb, 0);
      if (P.wpp && rx == 1) memcpy(ctx_wpp, ctx, sizeof ctx);
      bool end = k + 1 == order.size();
      cabac.terminate(end ? 1 : 0);                        // end_of_slice_segment_flag
      const bool tile_end = tiles && next_start < starts.size() && (int)k + 1 == starts[next_start];
      if (!end && ((P.wpp && (a + 1) % wctb == 0) || tile_end)) {
        cabac.terminate(1);                                // end_of_subset_one_bit (+ byte_alignment)
        substreams.push_back(cabac.bits.buf); cabac = {BitWriter(), ctx};
      }
    }
    substreams.push_back(cabac.bits.buf);
    // header
    BitWriter b;
    std::vector<size_t> escaped;
    for (auto& ss : substreams) escaped.push_back(escaped_size(ss.data(), ss.size()));
    write_slice_header(b, seq_header(), addr0, dependent, slice_qp, escaped);
    std::vector<uint8_t> rbsp = b.buf;
    for (auto& s : substreams) rbsp.insert(rbsp.end(), s.begin(), s.end());
    append_nal(out, 19 /* IDR_W_RADL */, rbsp);
  }

  // ---------------------------------------------------------------------------- SAO (7.3.8.3)
  void choose_sao(int rx, int ry) {
    int addr = ry * wctb + rx;
    SaoParams& s = sao[addr];
    memset(&s, 0, sizeof s);
    bool left_ok = rx > 0 && ctb_region[(size_t)addr - 1] == region_idx, up_ok = ry > 0 && ctb_region[(size_t)(addr - wctb)] == region_idx;
    int r = rng.range(16);
    if (left_ok && r < 3) { s = sao[addr - 1]; s.merge_left = 1; s.merge_up = 0; return; }
    if (up_ok && r < 6) { s = sao[addr - wctb]; s.merge_up = 1; s.merge_left = 0; return; }
    int cmax = (1 << (std::min(bd, 10) - 5)) - 1;
    for (int c = 0; c < (chroma ? 2 : 1); c++) {
      int t = rng.range(8);
      s.type[c] = t < 3 ? 0 : (t < 5 ? 1 : 2);
      for (int i = 0; i < 4; i++) { s.abs[c][i] = rng.range(4) == 0 ? rng.range(cmax + 1) : rng.range(std::min(cmax, 2) + 1); s.sign[c][i] = rng.range(2); }
      s.band_pos[c] = rng.range(32); s.eo_class[c] = rng.range(4);
    }
    if (chroma) {
      s.type[2] = s.type[1]; s.eo_class[2] = s.eo_class[1];
      for (int i = 0; i < 4; i++) { s.abs[2][i] = rng.range(std::min(cmax, 2) + 1); s.sign[2][i] = rng.range(2); }
      s.band_pos[2] = rng.range(32);
    }
  }
  void write_sao(int rx, int ry) {
    int addr = ry * wctb + rx;
    const SaoParams& s = sao[addr];
    if (rx > 0 && ctb_region[(size_t)addr - 1] == region_idx) cabac.bin(CTX_SAO_MERGE, s.merge_left);
    if (s.merge_left) return;
    if (ry > 0 && ctb_region[(size_t)(addr - wctb)] == region_idx) cabac.bin(CTX_SAO_MERGE, s.merge_up);
    if (s.merge_up) return;
    int cmax = (1 << (std::min(bd, 10) - 5)) - 1;
    for (int c = 0; c < (chroma ? 3 : 1); c++) {
      if (c < 2) {
        cabac.bin(CTX_SAO_TYPE, s.type[c] != 0);
        if (s.type[c]) cabac.bypass(s.type[c] == 2);
      }
      if (!s.type[c]) continue;
      for (int i = 0; i < 4; i++) { int v = s.abs[c][i]; for (int k = 0; k < v; k++) cabac.bypass(1); if (v < cmax) cabac.bypass(0); }
      if (s.type[c] == 1) {
        for (int i = 0; i < 4; i++) if (s.abs[c][i]) cabac.bypass(s.sign[c][i]);
        cabac.bypass_bits(s.band_pos[c], 5);
      } else if (c < 2) cabac.bypass_bits(s.eo_class[c], 2);
    }
  }

  // ---------------------------------------------------------------------------- intra prediction (8.4.4.2)
  void predict(int c, int x0, int y0, int log2n, int mode, uint16_t* dst /* n*n */) const {
    const int n = 1 << log2n, shx = c ? sx : 0, shy = c ? sy : 0, st = stride_of(c);
    const uint16_t* pl = rec[c].data();
    int16_t r[129], f[129];
    for (int i = 0; i <= 4 * n; i++) {
      int px, py;
      if (i < 2 * n) { px = x0 - 1; py = y0 + 2 * n - 1 - i; } else if (i == 2 * n) { px = x0 - 1; py = y0 - 1; } else { px = x0 + (i - 2 * n - 1); py = y0 - 1; }
      r[i] = avail(px << shx, py << shy) ? (int16_t)pl[(size_t)py * st + px] : (int16_t)-1;
    }
    substitute_refs(r, n, bd);
    const bool filt = refs_filtered(c == 0 || cfmt == 3, mode, log2n);
    if (filt) filter_refs(r, f, log2n, P.strong_intra_smoothing && c == 0, bd);
    const int dc = dc_value(r, log2n), maxv = (1 << bd) - 1;
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) dst[y * n + x] = (uint16_t)pred_sample(filt ? f : r, dc, log2n, mode, x, y, c == 0, maxv);
  }

  // ---------------------------------------------------------------------------- transforms
  void forward(const int* res, int* coef, int log2n, bool dst4, bool tskip) const {
    const int n = 1 << log2n;
    if (tskip) { int s = 15 - bd - log2n; for (int i = 0; i < n * n; i++) coef[i] = res[i] << s; return; }
    int tmp[1024];
    for (int k = 0; k < n; k++) for (int x = 0; x < n; x++) tmp[k * n + x] = fwd_col(res, dst4, log2n, k, x, bd);
    for (int y = 0; y < n; y++) for (int k = 0; k < n; k++) coef[y * n + k] = fwd_row(tmp, dst4, log2n, y, k);
  }
  void inverse(const int* d, int* res, int log2n, bool dst4, bool tskip) const {     // 8.6.4.2
    const int n = 1 << log2n;
    if (tskip) { const int bs = 20 - bd; for (int i = 0; i < n * n; i++) res[i] = ((d[i] << 7) + (1 << (bs - 1))) >> bs; return; }
    int tmp[1024];
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) tmp[y * n + x] = inv_col(d, dst4, log2n, y, x);
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) res[y * n + x] = inv_row(tmp, dst4, log2n, y, x, bd);
  }

  // ---------------------------------------------------------------------------- QP (8.6.1)
  int predict_qpy(int xcb, int ycb) const {
    int mask = (1 << qg_log2) - 1, xqg = xcb & ~mask, yqg = ycb & ~mask, cm = ~(ctb - 1);
    int qa = qpy_prev_qg, qb = qpy_prev_qg;
    if (avail(xqg - 1, yqg) && ((xqg - 1) & cm) == (xqg & cm)) qa = qp4[(size_t)(yqg >> 2) * w4 + ((xqg - 1) >> 2)];
    if (avail(xqg, yqg - 1) && ((yqg - 1) & cm) == (yqg & cm)) qb = qp4[(size_t)((yqg - 1) >> 2) * w4 + (xqg >> 2)];
    return (qa + qb + 1) >> 1;
  }

  // ---------------------------------------------------------------------------- residual (7.3.8.11)
  // quantise + (optionally) sign-hide; returns cbf. levels are in raster order [y][x].
  bool quantise(const int* coef, int16_t* lev, int log2n, int qp, int scan) const {
    const int n = 1 << log2n;
    bool any = false;
    for (int i = 0; i < n * n; i++) { lev[i] = (int16_t)quant_level(coef[i], qp, log2n, bd); any |= lev[i] != 0; }
    if (any && P.sign_data_hiding && !cu_bypass) {
      const int l2sb = log2n - 2;
      const uint8_t *sbx = B200_T(kScanX)[l2sb][scan], *sby = B200_T(kScanY)[l2sb][scan], *px = B200_T(kScanX)[2][scan], *py = B200_T(kScanY)[2][scan];
      for (int i = 0; i < (1 << (2 * l2sb)); i++) {
        int xs = sbx[i], ys = sby[i];
        int first = 16, last = -1, sum = 0;
        for (int k = 0; k < 16; k++) {
          int v = lev[((ys << 2) + py[k]) * n + (xs << 2) + px[k]];
          if (v) { if (first == 16) first = k; last = k; sum += std::abs(v); }
        }
        if (last - first > 3) {
          int16_t& f = lev[((ys << 2) + py[first]) * n + (xs << 2) + px[first]];
          if ((sum & 1) != (f < 0 ? 1 : 0)) {               // parity must equal the sign of the first coefficient
            int16_t& t = lev[((ys << 2) + py[last]) * n + (xs << 2) + px[last]];
            t = (int16_t)(t < 0 ? t - 1 : t + 1);
          }
        }
      }
    }
    return any;
  }

  // one transform block: predict, transform, quantise, (write), reconstruct. Returns cbf.
  struct TbResult { bool cbf; int16_t lev[1024]; int scan; bool tskip; };
  void write_residual(const TbResult& t, int log2n, int c) {
    residual_coding(cabac, t.lev, 1 << log2n, log2n, c, t.scan, P.transform_skip && !cu_bypass, t.tskip, P.sign_data_hiding && !cu_bypass);
  }
  void code_tb(int c, int x0, int y0, int log2n, int mode, TbResult& r) {
    const int n = 1 << log2n, st = stride_of(c);
    uint16_t pred[1024]; int res[1024], coef[1024];
    predict(c, x0, y0, log2n, mode, pred);
    for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) res[y * n + x] = (int)org[c][(size_t)(y0 + y) * st + x0 + x] - pred[y * n + x];
    bool dst4 = c == 0 && log2n == 2;
    r.scan = log2n == 2 || (log2n == 3 && (c == 0 || cfmt == 3)) ? scan_idx(mode) : 0;
    if (cu_bypass) {                                  // cu_transquant_bypass_flag: the residual is coded as is (8.6.2), lossless
      r.tskip = false;
      r.cbf = false;
      for (int i = 0; i < n * n; i++) { r.lev[i] = (int16_t)res[i]; r.cbf |= res[i] != 0; }
      uint16_t* rq = rec[c].data();
      for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) rq[(size_t)(y0 + y) * st + x0 + x] = org[c][(size_t)(y0 + y) * st + x0 + x];
      return;
    }
    r.tskip = P.transform_skip && log2n == 2 && rng.range(4) == 0;
    forward(res, coef, log2n, dst4, r.tskip);
    int qp = c == 0 ? qg_target_qp + 6 * (bd - 8) : chroma_qp(qg_target_qp + (c == 1 ? P.cb_qp_offset : P.cr_qp_offset) + (P.slice_chroma_qp_offsets ? (c == 1 ? P.slice_cb_qp_offset : P.slice_cr_qp_offset) : 0), cfmt, bd);
    r.cbf = quantise(coef, r.lev, log2n, qp, r.scan);
    if (forced && log2n >= 3 && forced_left[c] > 0) {        // test-only: the caller's levels instead of the quantised ones
      forced_left[c]--;
      r.cbf = false;
      for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) { r.lev[y * n + x] = forced[y * 32 + x]; r.cbf |= forced[y * 32 + x] != 0; }
    }
    // NOTE: the QP used here (qg_target_qp) is only valid if a cu_qp_delta can still be sent (or already
    // was); the caller re-runs with the predicted QP when neither holds.
    uint16_t* rp = rec[c].data();
    if (r.cbf) {
      int d[1024];
      for (int i = 0; i < n * n; i++) d[i] = dequant(r.lev[i], scaling_factor(c, log2n, i), qp, log2n, bd);
      inverse(d, res, log2n, dst4, r.tskip);
      int maxv = (1 << bd) - 1;
      for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) rp[(size_t)(y0 + y) * st + x0 + x] = (uint16_t)clip3(0, maxv, pred[y * n + x] + res[y * n + x]);
    } else for (int y = 0; y < n; y++) for (int x = 0; x < n; x++) rp[(size_t)(y0 + y) * st + x0 + x] = pred[y * n + x];
  }

  void mark_tu(int x0, int y0, int log2n) {
    int n4 = 1 << (log2n - 2);
    for (int y = 0; y < n4; y++) for (int x = 0; x < n4; x++) { size_t i = (size_t)((y0 >> 2) + y) * w4 + (x0 >> 2) + x; slice_of4[i] = (uint16_t)(region_idx + 1); qp4[i] = (int8_t)cur_qpy; }
  }

  // ---------------------------------------------------------------------------- transform tree (7.3.8.8)
  struct Cu { int x0, y0, log2cb, nxn, lmode[4], cmode[4]; };      // cmode: IntraPredModeC per prediction unit (one per PU only in 4:4:4)

  // Decide the TU split structure first (so that cbf_cb/cbf_cr of inner nodes are known before they are
  // written) by coding leaves depth-first into a node list, then emit the syntax in a second walk.
  // chroma: [t] = the upper / lower square block of a 4:2:2 transform unit (t = 0 only otherwise)
  struct Node { int x0, y0, log2n, depth, blk, split, child[4]; bool cbf_l, cbf_cb[2], cbf_cr[2]; TbResult *l, *cb[2], *cr[2]; };
  std::vector<Node> nodes; std::vector<TbResult*> pool;
  TbResult* new_tb() { TbResult* t = new TbResult; pool.push_back(t); return t; }

  int build_tree(const Cu& cu, int x0, int y0, int log2n, int depth, int blk, int max_depth, int parent) {
    Node nd{}; nd.x0 = x0; nd.y0 = y0; nd.log2n = log2n; nd.depth = depth; nd.blk = blk;
    bool can_split = log2n <= log2_max_tb && log2n > log2_min_tb && depth < max_depth && !(cu.nxn && depth == 0);
    if (can_split) nd.split = rng.range(log2n >= 5 ? 2 : 3) == 0;
    else nd.split = (log2n > log2_max_tb || (cu.nxn && depth == 0)) ? 1 : 0;
    int me = (int)nodes.size(); nodes.push_back(nd);
    if (nd.split) {
      int h = 1 << (log2n - 1);
      bool cb = false, cr = false;
      for (int k = 0; k < 4; k++) {
        int ch = build_tree(cu, x0 + (k & 1) * h, y0 + (k >> 1) * h, log2n - 1, depth + 1, k, max_depth, me);
        nodes[me].child[k] = ch; cb |= nodes[ch].cbf_cb[0] || nodes[ch].cbf_cb[1]; cr |= nodes[ch].cbf_cr[0] || nodes[ch].cbf_cr[1];
      }
      nodes[me].cbf_cb[0] = cb; nodes[me].cbf_cr[0] = cr; nodes[me].cbf_cb[1] = nodes[me].cbf_cr[1] = false;
      if (log2n == 3 && chroma && cfmt != 3) {   // 4x4 luma children: the chroma 4x4 blocks are coded with child 3 at this node's origin
        for (int t = 0; t < 2; t++) {
          nodes[me].cbf_cb[t] = nodes[nodes[me].child[3]].cb[t] ? nodes[nodes[me].child[3]].cb[t]->cbf : false;
          nodes[me].cbf_cr[t] = nodes[nodes[me].child[3]].cr[t] ? nodes[nodes[me].child[3]].cr[t]->cbf : false;
        }
      }
    } else {
      int pu = cu.nxn ? ((y0 >= cu.y0 + (1 << (cu.log2cb - 1))) ? 2 : 0) + ((x0 >= cu.x0 + (1 << (cu.log2cb - 1))) ? 1 : 0) : 0;
      Node& m = nodes[me];
      m.l = new_tb(); code_tb(0, x0, y0, log2n, cu.lmode[pu], *m.l); m.cbf_l = m.l->cbf;
      mark_tu(x0, y0, log2n);
      if (chroma) {
        const int nb = cfmt == 2 ? 2 : 1;                       // 4:2:2: two square blocks, one above the other (7.3.8.10)
        if (log2n > 2 || cfmt == 3) {
          const int lc = cfmt == 3 ? log2n : log2n - 1, cm = cu.cmode[cfmt == 3 ? pu : 0];
          for (int t = 0; t < nb; t++) { m.cb[t] = new_tb(); code_tb(1, x0 >> sx, (y0 >> sy) + (t << lc), lc, cm, *m.cb[t]); m.cbf_cb[t] = m.cb[t]->cbf; }
          for (int t = 0; t < nb; t++) { m.cr[t] = new_tb(); code_tb(2, x0 >> sx, (y0 >> sy) + (t << lc), lc, cm, *m.cr[t]); m.cbf_cr[t] = m.cr[t]->cbf; }
        } else if (blk == 3) {
          const Node& par = nodes[parent];
          for (int t = 0; t < nb; t++) { m.cb[t] = new_tb(); code_tb(1, par.x0 >> sx, (par.y0 >> sy) + (t << 2), 2, cu.cmode[0], *m.cb[t]); }
          for (int t = 0; t < nb; t++) { m.cr[t] = new_tb(); code_tb(2, par.x0 >> sx, (par.y0 >> sy) + (t << 2), 2, cu.cmode[0], *m.cr[t]); }
        }
      }
    }
    return me;
  }

  // parent_cb / parent_cr: the cbf_cb / cbf_cr flags of the parent node ([1]: lower 4:2:2 block)
  void write_tree(const Cu& cu, int me, const bool parent_cb[2], const bool parent_cr[2], int max_depth) {
    const Node& nd = nodes[me];
    bool can_split = nd.log2n <= log2_max_tb && nd.log2n > log2_min_tb && nd.depth < max_depth && !(cu.nxn && nd.depth == 0);
    if (can_split) cabac.bin(CTX_SPLIT_TR + 5 - nd.log2n, nd.split);
    bool cb[2] = {false, false}, cr[2] = {false, false};
    if (chroma) {
      if (nd.log2n > 2 || cfmt == 3) {
        const bool two = cfmt == 2 && (!nd.split || nd.log2n == 3);
        if (nd.depth == 0 || parent_cb[0]) { cb[0] = nd.cbf_cb[0]; cabac.bin(CTX_CBF_CHROMA + nd.depth, cb[0]); if (two) { cb[1] = nd.cbf_cb[1]; cabac.bin(CTX_CBF_CHROMA + nd.depth, cb[1]); } }
        if (nd.depth == 0 || parent_cr[0]) { cr[0] = nd.cbf_cr[0]; cabac.bin(CTX_CBF_CHROMA + nd.depth, cr[0]); if (two) { cr[1] = nd.cbf_cr[1]; cabac.bin(CTX_CBF_CHROMA + nd.depth, cr[1]); } }
      } else { cb[0] = parent_cb[0]; cb[1] = parent_cb[1]; cr[0] = parent_cr[0]; cr[1] = parent_cr[1]; }
    }
    if (nd.split) { for (int k = 0; k < 4; k++) write_tree(cu, nd.child[k], cb, cr, max_depth); return; }
    cabac.bin(CTX_CBF_LUMA + (nd.depth == 0 ? 1 : 0), nd.cbf_l);
    bool cbf_chroma = chroma && (cb[0] || cb[1] || cr[0] || cr[1]);
    if ((nd.cbf_l || cbf_chroma) && P.cu_qp_delta && !is_qp_delta_coded) {
      int v = cu_qp_delta_val, a = std::abs(v);
      for (int k = 0; k < std::min(a, 5); k++) cabac.bin(CTX_QP_DELTA + (k ? 1 : 0), 1);
      if (a < 5) cabac.bin(CTX_QP_DELTA + (a ? 1 : 0), 0);
      else { int rem = a - 5, k = 0; while (rem >= (1 << k)) { cabac.bypass(1); rem -= 1 << k; k++; } cabac.bypass(0); cabac.bypass_bits(rem, k); }
      if (a) cabac.bypass(v < 0);
      is_qp_delta_coded = 1;
    }
    if (nd.cbf_l) write_residual(*nd.l, nd.log2n, 0);
    if (chroma) {
      const int nb = cfmt == 2 ? 2 : 1;
      if (nd.log2n > 2 || cfmt == 3) {
        const int lc = cfmt == 3 ? nd.log2n : nd.log2n - 1;
        for (int t = 0; t < nb; t++) if (cb[t]) write_residual(*nd.cb[t], lc, 1);
        for (int t = 0; t < nb; t++) if (cr[t]) write_residual(*nd.cr[t], lc, 2);
      } else if (nd.blk == 3) {
        for (int t = 0; t < nb; t++) if (parent_cb[t]) write_residual(*nd.cb[t], 2, 1);
        for (int t = 0; t < nb; t++) if (parent_cr[t]) write_residual(*nd.cr[t], 2, 2);
      }
    }
  }

  // ---------------------------------------------------------------------------- coding unit (7.3.8.5)
  void mpm(int x, int y, int cand[3]) const {
    int ca = 1, cb = 1;
    if (avail(x - 1, y)) ca = ipm4[(size_t)(y >> 2) * w4 + ((x - 1) >> 2)];
    if (avail(x, y - 1) && (y - 1) >= ((y >> log2ctb) << log2ctb)) cb = ipm4[(size_t)((y - 1) >> 2) * w4 + (x >> 2)];
    mpm_candidates(ca, cb, cand);
  }

  int choose_mode(int x0, int y0, int log2n, const int cand[3]) {
    if (P.mode_decision == 0) return rng.range(35);
    const int n = 1 << log2n;
    int tries[8] = {0, 1, 10, 26, cand[0], 2 + rng.range(33), 2 + rng.range(33), 2 + rng.range(33)};
    int best = 0; long best_cost = -1;
    uint16_t pred[1024];
    int lg = std::min(log2n, 5);                       // evaluate on (at most) 32x32 at the CU origin
    int m = 1 << lg;
    for (int t = 0; t < 8; t++) {
      predict(0, x0, y0, lg, tries[t], pred);
      long sad = 0;
      for (int y = 0; y < m; y++) for (int x = 0; x < m; x++) sad += std::abs((int)org[0][(size_t)(y0 + y) * W + x0 + x] - pred[y * m + x]);
      if (best_cost < 0 || sad < best_cost) { best_cost = sad; best = tries[t]; }
    }
    (void)n;
    return best;
  }

  void coding_unit(int x0, int y0, int log2cb, int depth) {
    Cu cu{}; cu.x0 = x0; cu.y0 = y0; cu.log2cb = log2cb;
    const int n = 1 << log2cb;
    cu_bypass = false;
    if (P.transquant_bypass) { cu_bypass = P.transquant_bypass == 2 || rng.range(4) == 0; cabac.bin(CTX_TQ_BYPASS, cu_bypass); }
    if (log2cb == 3) { cu.nxn = rng.range(3) == 0; cabac.bin(CTX_PART_MODE, !cu.nxn); }
    if (P.pcm && !cu.nxn && log2cb <= std::min(5, log2ctb)) {
      const bool pcm = rng.range(6) == 0;
      cabac.terminate(pcm ? 1 : 0);                   // pcm_flag (terminate bin); value 1: flush, stop bit, pcm_alignment_zero_bits
      if (pcm) {
        for (int c = 0; c < (chroma ? 3 : 1); c++) {
          const int shx = c ? sx : 0, shy = c ? sy : 0, pbd = c ? pcm_bd_c : pcm_bd_y, st = stride_of(c);
          uint16_t* rq = rec[c].data();
          for (int y = 0; y < (n >> shy); y++) for (int x = 0; x < (n >> shx); x++) {
            const size_t idx = (size_t)((y0 >> shy) + y) * st + (x0 >> shx) + x;
            const unsigned v = org[c][idx] >> (bd - pbd);
            cabac.bits.put(v, pbd);                     // pcm_sample_luma / pcm_sample_chroma
            rq[idx] = (uint16_t)(v << (bd - pbd));
          }
        }
        cabac.restart();
        for (int yy = 0; yy < n; yy += 4) for (int xx = 0; xx < n; xx += 4) {
          const size_t idx = (size_t)((y0 + yy) >> 2) * w4 + ((x0 + xx) >> 2);
          ipm4[idx] = 1; slice_of4[idx] = (uint16_t)(region_idx + 1); cd4[idx] = (uint8_t)depth;       // a PCM unit counts as INTRA_DC for its neighbours (8.4.2)
        }
        // no transform tree, no cu_qp_delta: QpY = predicted QP (+ the delta already coded in this quantization group, 8.6.1)
        const int pred_qp = P.cu_qp_delta ? predict_qpy(x0, y0) : slice_qp;
        cur_qpy = P.cu_qp_delta ? pred_qp + (is_qp_delta_coded ? cu_qp_delta_val : 0) : slice_qp;
        for (int yy = 0; yy < n; yy += 4) for (int xx = 0; xx < n; xx += 4) qp4[(size_t)((y0 + yy) >> 2) * w4 + ((x0 + xx) >> 2)] = (int8_t)cur_qpy;
        last_cu_qpy = cur_qpy;
        return;
      }
    }
    int np = cu.nxn ? 4 : 1, pb = cu.nxn ? n / 2 : n;
    int code[4];
    for (int i = 0; i < np; i++) {
      int px = x0 + (i & 1) * pb, py = y0 + (i >> 1) * pb, cand[3];
      mpm(px, py, cand);
      int mode = choose_mode(px, py, cu.nxn ? 2 : log2cb, cand);
      cu.lmode[i] = mode;
      code[i] = mpm_code(mode, cand);
      for (int yy = 0; yy < pb; yy += 4) for (int xx = 0; xx < pb; xx += 4) {
        size_t idx = (size_t)((py + yy) >> 2) * w4 + ((px + xx) >> 2);
        ipm4[idx] = (uint8_t)mode; slice_of4[idx] = (uint16_t)(region_idx + 1);
      }
    }
    write_luma_modes(cabac, np, code);
    if (chroma) {
      // intra_chroma_pred_mode: one per prediction unit in 4:4:4, else one per coding unit (7.3.8.5); 8.4.3 + Table 8-3 for 4:2:2
      static const uint8_t k422[35] = {0, 1, 2, 2, 2, 2, 3, 5, 7, 8, 10, 12, 13, 15, 17, 18, 19, 20, 21, 22, 23, 23, 24, 24, 25, 25, 26, 27, 27, 28, 28, 29, 29, 30, 31};
      for (int i = 0; i < (cfmt == 3 ? np : 1); i++) {
        int v = rng.range(8); if (v > 4) v = 4;
        int m = (v < 4 && B200_T(kChromaTab)[v] == cu.lmode[i]) ? 34 : (v == 4 ? cu.lmode[i] : B200_T(kChromaTab)[v]);
        if (cfmt == 2) m = k422[m];
        cu.cmode[i] = m;
        cabac.bin(CTX_CHROMA_PRED, v != 4);
        if (v != 4) cabac.bypass_bits(v, 2);
      }
    }
    for (int yy = 0; yy < n; yy += 4) for (int xx = 0; xx < n; xx += 4) {
      size_t idx = (size_t)((y0 + yy) >> 2) * w4 + ((x0 + xx) >> 2);
      slice_of4[idx] = 0; cd4[idx] = (uint8_t)depth;
    }
    // QP of this CU: target QP if the delta of this quantization group was (or can still be) sent, else predicted
    int pred_qp = P.cu_qp_delta ? predict_qpy(x0, y0) : slice_qp;
    int qbd = 6 * (bd - 8);
    if (P.cu_qp_delta && !is_qp_delta_coded) {
      cu_qp_delta_val = clip3(-(26 + qbd / 2), 25 + qbd / 2, qg_target_qp - pred_qp);
      qg_target_qp = pred_qp + cu_qp_delta_val;
    } else if (!P.cu_qp_delta) qg_target_qp = slice_qp;
    cur_qpy = qg_target_qp;
    nodes.clear();
    int max_depth = max_th_depth + cu.nxn;
    int root = build_tree(cu, x0, y0, log2cb, 0, 0, max_depth, -1);
    bool any_cbf = false;
    for (const Node& nd : nodes) if (!nd.split) for (int t = 0; t < 2; t++) any_cbf |= nd.cbf_l || (nd.cb[t] && nd.cb[t]->cbf) || (nd.cr[t] && nd.cr[t]->cbf);
    if (P.cu_qp_delta && !is_qp_delta_coded && !any_cbf) {
      // nothing coded: the decoder will use the predicted QP (CuQpDeltaVal stays 0); pixels are pure prediction so
      // the reconstruction above is already what the decoder produces.
      cur_qpy = pred_qp;
    }
    { const bool none[2] = {false, false}; write_tree(cu, root, none, none, max_depth); }
    for (TbResult* t : pool) delete t;
    pool.clear();
    for (int yy = 0; yy < n; yy += 4) for (int xx = 0; xx < n; xx += 4) qp4[(size_t)((y0 + yy) >> 2) * w4 + ((x0 + xx) >> 2)] = (int8_t)cur_qpy;
    last_cu_qpy = cur_qpy;
  }

  long block_activity(int x0, int y0, int n) const {
    long s = 0, s2 = 0;
    for (int y = 0; y < n; y += 2) for (int x = 0; x < n; x += 2) { int v = org[0][(size_t)(y0 + y) * W + x0 + x]; s += v; s2 += (long)v * v; }
    long cnt = (long)(n / 2) * (n / 2);
    return (s2 - s * s / cnt) / cnt >> (2 * (bd - 8));
  }

  void coding_quadtree(int x0, int y0, int log2cb, int depth) {
    int n = 1 << log2cb;
    bool split;
    if (x0 + n <= W && y0 + n <= H && log2cb > 3) {
      long act = block_activity(x0, y0, n);
      int r = rng.range(8);
      split = P.mode_decision == 0 ? r < 4 : (act > (long)P.split_threshold * (log2cb - 2) ? r != 0 : r == 0);
      int inc = 0;
      if (avail(x0 - 1, y0) && cd4[(size_t)(y0 >> 2) * w4 + ((x0 - 1) >> 2)] > depth) inc++;
      if (avail(x0, y0 - 1) && cd4[(size_t)((y0 - 1) >> 2) * w4 + (x0 >> 2)] > depth) inc++;
      cabac.bin(CTX_SPLIT_CU + inc, split);
    } else split = log2cb > 3;
    if (P.cu_qp_delta && log2cb >= qg_log2) {
      is_qp_delta_coded = 0; cu_qp_delta_val = 0;
      if (!split || log2cb == qg_log2) {
        if (first_qg) { qpy_prev_qg = slice_qp; first_qg = 0; } else qpy_prev_qg = last_cu_qpy;
        qg_target_qp = clip3(0, 51, slice_qp + (P.dqp_range ? rng.range(2 * P.dqp_range + 1) - P.dqp_range : 0));
      }
    }
    if (split) {
      int h = n >> 1;
      for (int k = 0; k < 4; k++) { int x1 = x0 + (k & 1) * h, y1 = y0 + (k >> 1) * h; if (x1 < W && y1 < H) coding_quadtree(x1, y1, log2cb - 1, depth + 1); }
    } else coding_unit(x0, y0, log2cb, depth);
  }
};

}  // namespace enc
}  // namespace b200

extern "C" {

void b200_hevc_enc_params_default(b200_hevc_enc_params* p) {
  memset(p, 0, sizeof *p);
  p->tile_cols = p->tile_rows = 1; p->tiles_uniform = 1; p->loop_filter_across_tiles = 1; p->slice_per_tile = 0;
  p->bit_depth = 8; p->chroma_format_idc = 1; p->log2_ctb_size = 5; p->qp = 27; p->init_qp = 26;
  p->max_transform_hierarchy_depth_intra = 1; p->sao = 1; p->sign_data_hiding = 1; p->cu_qp_delta = 1;
  p->diff_cu_qp_delta_depth = 1; p->dqp_range = 3; p->strong_intra_smoothing = 1; p->loop_filter_across_slices = 1;
  p->slice_loop_filter_across_slices = 1; p->mode_decision = 1; p->split_threshold = 40; p->seed = 0xB200;
  p->still_picture = 1; p->vui_present = 0; p->colour_primaries = 2; p->transfer_characteristics = 2; p->matrix_coefficients = 2;
}

}  // extern "C"

namespace b200 {
namespace enc {
// b200_hevc_encode_intra; forced / nforced: Encoder::force_levels (test-only), rec[3]: the encoder's reconstruction of the
// coded size (rounded up to 8), or nullptr
static int encode_intra(const b200_hevc_enc_params* p, const void* y, const void* cb, const void* cr, size_t y_stride, size_t c_stride,
                        uint8_t** out_data, size_t* out_size, const int16_t* forced, int nforced, uint16_t* const rec[3]) {
  if (!p || !y || !out_data || !out_size) return set_error(B200_E_INVALID, "null argument");
  if (p->width < 8 || p->height < 8 || p->width > 16384 || p->height > 16384) return set_error(B200_E_INVALID, "size %dx%d", p->width, p->height);
  if (p->bit_depth < 8 || p->bit_depth > 12) return set_error(B200_E_UNSUPPORTED, "bit depth %d", p->bit_depth);
  if (p->log2_ctb_size < 4 || p->log2_ctb_size > 6) return set_error(B200_E_INVALID, "log2_ctb_size %d", p->log2_ctb_size);
  if (p->chroma_format_idc && (!cb || !cr)) return set_error(B200_E_INVALID, "missing chroma planes");
  const int bps = p->bit_depth > 8 ? 2 : 1;
  std::vector<uint16_t> tmp[3];
  const uint16_t* src[3] = {nullptr, nullptr, nullptr}; int stride[3] = {0, 0, 0};
  const void* in[3] = {y, cb, cr};
  for (int c = 0; c < (p->chroma_format_idc ? 3 : 1); c++) {
    const int csx = (p->chroma_format_idc == 1 || p->chroma_format_idc == 2) ? 1 : 0, csy = p->chroma_format_idc == 1 ? 1 : 0;
    int w = c ? (p->width + (1 << csx) - 1) >> csx : p->width, h = c ? (p->height + (1 << csy) - 1) >> csy : p->height;
    size_t st = c ? c_stride : y_stride;
    tmp[c].resize((size_t)w * h);
    for (int yy = 0; yy < h; yy++) for (int xx = 0; xx < w; xx++)
      tmp[c][(size_t)yy * w + xx] = bps == 1 ? ((const uint8_t*)in[c])[yy * st + xx] : ((const uint16_t*)((const uint8_t*)in[c] + yy * st))[xx];
    src[c] = tmp[c].data(); stride[c] = w;
  }
  Encoder e(*p, src, stride);
  if (forced) e.force_levels(forced, nforced);
  std::vector<uint8_t> out;
  e.encode(out);
  *out_data = (uint8_t*)malloc(out.size() ? out.size() : 1);
  if (!*out_data) return set_error(B200_E_INVALID, "out of memory");
  memcpy(*out_data, out.data(), out.size());
  *out_size = out.size();
  if (rec)
    for (int c = 0; c < (p->chroma_format_idc ? 3 : 1); c++) if (rec[c]) memcpy(rec[c], e.recon(c).data(), e.recon(c).size() * 2);
  return B200_OK;
}

}  // namespace enc
}  // namespace b200

extern "C" {

int b200_hevc_encode_intra(const b200_hevc_enc_params* p, const void* y, const void* cb, const void* cr, size_t y_stride,
                           size_t c_stride, uint8_t** out_data, size_t* out_size) {
  return b200::enc::encode_intra(p, y, cb, cr, y_stride, c_stride, out_data, out_size, nullptr, 0, nullptr);
}

void b200_free(void* p) { free(p); }

// Test-only entry points (declared by the tests, not in include/b200_heif.h).
//
// b200_hevc_encode_intra, except that the levels of the first `count` transform-coded blocks of 8x8 and larger of every
// component are the top-left n x n of `pattern` (32 x 32 raster int16) instead of the quantised ones.  Sign-data hiding must be
// off: it would drop signs of the pattern.  rec_*: the encoder's reconstruction before the in-loop filters, coded size
// (width and height rounded up to 8; chroma planes subsampled from that), uint16.
int b200_debug_hevc_encode_forced_levels(const b200_hevc_enc_params* p, const void* y, const void* cb, const void* cr, size_t y_stride,
                                         size_t c_stride, const int16_t* pattern, int count, uint8_t** out_data, size_t* out_size,
                                         uint16_t* rec_y, uint16_t* rec_cb, uint16_t* rec_cr) {
  using namespace b200;
  if (!p || !pattern || !rec_y || (p->chroma_format_idc && (!rec_cb || !rec_cr))) return set_error(B200_E_INVALID, "null argument");
  if (count < 0) return set_error(B200_E_INVALID, "count %d", count);
  if (p->sign_data_hiding) return set_error(B200_E_INVALID, "forced levels need sign_data_hiding = 0");
  uint16_t* const rec[3] = {rec_y, rec_cb, rec_cr};
  return enc::encode_intra(p, y, cb, cr, y_stride, c_stride, out_data, out_size, pattern, count, rec);
}

// The transform chain of the host encoder, element by element on n given blocks: prm[i * DT_FIELDS ..] = (log2 size 2..5,
// DST 0/1 (4x4 only), bit depth 8..12, qp 0 .. 51 + 6 * (bd - 8), scaling factor 1..255), in[i * 1024 ..] = the block's
// input (n x n raster, int16 range).  out[(i * 6 + st) * 1024 ..] = stage st applied to that input: fwd_col (row k, column
// x), fwd_row (row y, column k), quant_level, dequant (the inputs as levels), inv_col, inv_row.
int b200_debug_enc_transform_host(int n, const int32_t* prm, const int32_t* in, int32_t* out) {
  using namespace b200;
  if (n < 1 || n > 65536 || !prm || !in || !out) return set_error(B200_E_INVALID, "enc_transform: %d blocks, null argument", n);
  for (int i = 0; i < n; i++)
    if (const char* why = enc::debug_transform_args(prm + (size_t)i * enc::DT_FIELDS, in + (size_t)i * 1024)) return set_error(B200_E_INVALID, "enc_transform: block %d: %s", i, why);
  for (int i = 0; i < n; i++) {
    const int32_t* p = prm + (size_t)i * enc::DT_FIELDS;
    const int lg = p[enc::DT_LOG2N], nn = 1 << lg;
    for (int st = 0; st < enc::DT_STAGES; st++)
      for (int e = 0; e < nn * nn; e++) out[((size_t)i * enc::DT_STAGES + st) * 1024 + e] = enc::debug_transform_stage(st, p, in + (size_t)i * 1024, e >> lg, e & (nn - 1));
  }
  return B200_OK;
}

// Intra prediction of the host encoder on n given blocks: prm[i * DP_FIELDS ..] = (log2 size 2..5, bit depth 8..12, luma (DC
// and mode 10 / 26 edge filters), plane filtered (luma, or chroma in 4:4:4), strong intra smoothing), refs[i * 129 ..] = the
// neighbours r[0 .. 4n] of b200_hevc_enc_recon.h, -1 = unavailable.  Outputs: rf[i * 258 ..] = r after substitute_refs and
// filter_refs of it (129 each), pred[(i * 35 + mode) * 1024 ..] = the n x n prediction of every mode, raster.
int b200_debug_enc_predict_host(int n, const int32_t* prm, const int16_t* refs, int16_t* rf, int32_t* pred) {
  using namespace b200;
  if (n < 1 || n > 65536 || !prm || !refs || !rf || !pred) return set_error(B200_E_INVALID, "enc_predict: %d blocks, null argument", n);
  for (int i = 0; i < n; i++)
    if (const char* why = enc::debug_predict_args(prm + (size_t)i * enc::DP_FIELDS, refs + (size_t)i * 129)) return set_error(B200_E_INVALID, "enc_predict: block %d: %s", i, why);
  for (int i = 0; i < n; i++) {
    const int32_t* p = prm + (size_t)i * enc::DP_FIELDS;
    const int lg = p[enc::DP_LOG2N], bd = p[enc::DP_BD], nn = 1 << lg;
    int16_t* r = rf + (size_t)i * 258; int16_t* f = r + 129;
    memcpy(r, refs + (size_t)i * 129, 129 * 2);
    enc::substitute_refs(r, nn, bd);
    enc::filter_refs(r, f, lg, p[enc::DP_STRONG] != 0, bd);
    const int dc = enc::dc_value(r, lg);
    for (int mode = 0; mode < 35; mode++) {
      const bool filt = enc::refs_filtered(p[enc::DP_PLANE] != 0, mode, lg);
      for (int e = 0; e < nn * nn; e++)
        pred[((size_t)i * 35 + mode) * 1024 + e] = enc::pred_sample(filt ? f : r, dc, lg, mode, e & (nn - 1), e >> lg, p[enc::DP_LUMA] != 0, (1 << bd) - 1);
    }
  }
  return B200_OK;
}

}  // extern "C"
