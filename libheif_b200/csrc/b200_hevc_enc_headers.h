// b200_hevc_enc_headers.h -- the parts of an HEVC intra access unit that both encoders write on the host: bit writer,
// VPS / SPS / PPS, the slice segment header (with WPP / tile entry points over the escaped sub-stream sizes), emulation
// prevention and the uint32 BE length prefix of every NAL unit.  Used by the host encoder (b200_hevc_enc.cc) and by the
// framing stage of the GPU encoder (b200_hevc_gpu_enc.cu).
#pragma once
#include "b200_internal.h"
#include "b200_hevc_scaling.h"
#include <vector>

namespace b200 {
namespace enc {

struct BitWriter {
  std::vector<uint8_t> buf; int nbits = 0; uint8_t cur = 0;
  void put1(unsigned b) { put(b, 1); }
  void put(unsigned v, int n) { for (int i = n - 1; i >= 0; i--) { cur = (uint8_t)((cur << 1) | ((v >> i) & 1)); if (++nbits == 8) { buf.push_back(cur); cur = 0; nbits = 0; } } }
  void ue(unsigned v) { unsigned x = v + 1; int len = 0; while ((x >> len) > 1) len++; put(0, len); put(x, len + 1); }
  void se(int v) { ue(v > 0 ? 2 * v - 1 : -2 * v); }
  void trailing() { put(1, 1); while (nbits) put(0, 1); }
  void align_zero() { while (nbits) put(0, 1); }
};

// rbsp -> NAL unit (2-byte header, emulation prevention) appended to `out` behind its uint32 BE length
void append_nal(std::vector<uint8_t>& out, int type, const std::vector<uint8_t>& rbsp);
// size of `d` after emulation prevention (what an entry point offset counts)
size_t escaped_size(const uint8_t* d, size_t n);

// Everything the parameter sets and the slice segment header say about one coded picture.
struct SeqHeader {
  const b200_hevc_enc_params* P;
  int W, H;                          // coded size (multiples of 8)
  int cfmt, chroma, sx, sy, bd;
  int log2ctb, log2_min_tb, log2_max_tb, max_th_depth, qg_log2;
  int pcm_bd_y, pcm_bd_c;
  bool sl_on; const uint8_t (*sl_kind)[6]; const sl::Lists* sl_lists;   // scaling lists (sl_kind: 0 default, 1 previous, 2 explicit)
  bool tiles; const std::vector<int>* col_bd; const std::vector<int>* row_bd;
};

void write_vps(std::vector<uint8_t>& out, const SeqHeader& s);
void write_sps(std::vector<uint8_t>& out, const SeqHeader& s);
void write_pps(std::vector<uint8_t>& out, const SeqHeader& s);
// slice_segment_header() + byte_alignment() of the segment starting at CTB addr0; `escaped` = escaped sizes of its
// sub-streams (entry points are written when WPP or tiles are on)
void write_slice_header(BitWriter& b, const SeqHeader& s, int addr0, bool dependent, int slice_qp, const std::vector<size_t>& escaped);

}  // namespace enc
}  // namespace b200
