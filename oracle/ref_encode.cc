/*
 * oracle/ref_encode.cc -- TEST INFRASTRUCTURE ONLY. Never linked, imported or executed by the product.
 *
 * The encoder side of the UNMODIFIED reference colour stage (libheif_ref.so, oracle/Makefile) on caller-provided RGB input:
 * what heif_context_encode_image() runs before an encoder plugin sees the picture
 * (Encoder::convert_colorspace_for_encoding, libheif/codecs/encoder.cc:116-175: convert_colorspace with output_bpp = 0).
 * Input layouts: interleaved RGB / RGBA 8 bit, interleaved RRGGBB(AA)_BE / _LE 9..16 bit, planar R, G, B (+ A) 8..16 bit.
 * Besides the planes, the chain the reference's planner picked (ColorConversionPipeline::construct_pipeline,
 * colorconversion.cc:279-435) is reported as the demangled operation names, separated by ';'.
 */
#include <cxxabi.h>
#include <cstdlib>
#include <cstring>
#include <typeinfo>
#include <string>
#include <vector>
#include <libheif/heif.h>
#include "image/pixelimage.h"
#define private public            // the planner's steps (ColorConversionPipeline::m_conversion_steps) are private
#include "color-conversion/colorconversion.h"
#undef private
#include "security_limits.h"

namespace {
std::string demangled_pipeline(const ColorConversionPipeline& p) {
  std::string out;
  for (const auto& step : p.m_conversion_steps) {
    const ColorConversionOperation& op = *step.operation;
    int st = 0;
    char* d = abi::__cxa_demangle(typeid(op).name(), nullptr, nullptr, &st);
    std::string name = (st == 0 && d) ? d : typeid(op).name();
    free(d);
    if (!out.empty()) out += ";";
    out += name;
  }
  return out;
}
}  // namespace

// in_chroma: heif_chroma of the input (10..15 interleaved, 3 = planar 4:4:4 RGB).  planes: interleaved -> planes[0];
// planar -> R, G, B, A (A only when has_alpha).  Rows packed (w * components * bytes per sample).  Samples > 8 bit:
// interleaved as the layout names them (BE / LE bytes), planar as native uint16.
// Output planes packed (Y w x h, Cb / Cr cw x ch, alpha w x h when the result has one).  Returns 0, or < 0 when the
// reference's convert_colorspace fails (-4) or the input cannot be built (-1).
extern "C" int ref_rgb_to_ycbcr_ex(int in_chroma, int bpp, int alpha_bpp, int has_alpha, int w, int h, const void* const* planes,
                                   int out_chroma, int cp, int tc, int mc, int full_range, int downsampling, int only_preferred,
                                   void* oy, void* ocb, void* ocr, void* oa, int* out_has_alpha, char* pipeline, int pipeline_len) {
  const heif_security_limits* limits = heif_get_global_security_limits();
  auto img = std::make_shared<HeifPixelImage>();
  const int bps = bpp > 8 ? 2 : 1;
  if (in_chroma == heif_chroma_444) {
    img->create(w, h, heif_colorspace_RGB, heif_chroma_444);
    const heif_channel chans[4] = {heif_channel_R, heif_channel_G, heif_channel_B, heif_channel_Alpha};
    for (int c = 0; c < (has_alpha ? 4 : 3); c++) {
      const int d = c == 3 ? alpha_bpp : bpp, b = d > 8 ? 2 : 1;
      if (img->add_channel(chans[c], w, h, d, limits)) return -1;
      size_t stride; uint8_t* dst = img->get_channel_memory(chans[c], &stride);
      for (int r = 0; r < h; r++) memcpy(dst + r * stride, (const uint8_t*)planes[c] + (size_t)r * w * b, (size_t)w * b);
    }
  } else {
    img->create(w, h, heif_colorspace_RGB, (heif_chroma)in_chroma);
    if (img->add_channel(heif_channel_interleaved, w, h, bpp, limits)) return -1;
    const size_t rowb = (size_t)w * num_interleaved_components_per_plane((heif_chroma)in_chroma) * bps;
    size_t stride; uint8_t* dst = img->get_channel_memory(heif_channel_interleaved, &stride);
    for (int r = 0; r < h; r++) memcpy(dst + r * stride, (const uint8_t*)planes[0] + (size_t)r * rowb, rowb);
  }
  nclx_profile target;
  target.set_colour_primaries((uint16_t)cp); target.set_transfer_characteristics((uint16_t)tc);
  target.set_matrix_coefficients((uint16_t)mc); target.set_full_range_flag(full_range != 0);
  heif_color_conversion_options copt{};
  copt.version = 1;
  copt.preferred_chroma_downsampling_algorithm = (heif_chroma_downsampling_algorithm)downsampling;
  copt.preferred_chroma_upsampling_algorithm = heif_chroma_upsampling_bilinear;
  copt.only_use_preferred_chroma_algorithm = (uint8_t)only_preferred;

  if (pipeline && pipeline_len > 0) {
    // convert_colorspace keeps its pipeline to itself, so the chain is planned a second time here from the states it derives
    // (colorconversion.cc:530-611), restated for this input and a YCbCr target at the input depth.  The planes below come from
    // the real convert_colorspace; a drift of this restatement (alpha_bits_per_pixel, nclx defaults) would show as a chain
    // whose operations do not produce those planes on the GPU (tests/test_rgb_to_ycbcr_ex_gpu.py checks both).
    ColorState in;
    in.colorspace = heif_colorspace_RGB; in.chroma = (heif_chroma)in_chroma;
    in.has_alpha = has_alpha || in_chroma == heif_chroma_interleaved_RGBA || in_chroma == heif_chroma_interleaved_RRGGBBAA_BE ||
                   in_chroma == heif_chroma_interleaved_RRGGBBAA_LE;
    in.nclx.replace_undefined_values_with_sRGB_defaults();
    in.bits_per_pixel = bpp;
    if (in_chroma == heif_chroma_444 && has_alpha) in.alpha_bits_per_pixel = alpha_bpp;
    ColorState out = in;
    out.colorspace = heif_colorspace_YCbCr; out.chroma = (heif_chroma)out_chroma; out.nclx = target;
    if (out.nclx.get_matrix_coefficients() == heif_matrix_coefficients_unspecified) out.nclx.set_matrix_coefficients(in.nclx.get_matrix_coefficients());
    if (out.nclx.get_colour_primaries() == heif_color_primaries_unspecified) out.nclx.set_colour_primaries(in.nclx.get_colour_primaries());
    if (out.nclx.get_transfer_characteristics() == heif_transfer_characteristic_unspecified) out.nclx.set_transfer_characteristics(in.nclx.get_transfer_characteristics());
    out.alpha_bits_per_pixel = out.bits_per_pixel;
    heif_color_conversion_options_ext* ext = heif_color_conversion_options_ext_alloc();
    ColorConversionPipeline p;
    const bool ok = p.construct_pipeline(in, out, copt, *ext);
    heif_color_conversion_options_ext_free(ext);
    const std::string s = ok ? demangled_pipeline(p) : std::string("none");
    snprintf(pipeline, (size_t)pipeline_len, "%s", s.c_str());
  }

  auto res = convert_colorspace(img, heif_colorspace_YCbCr, (heif_chroma)out_chroma, target, 0, copt, nullptr, limits);
  if (!res) return -4;
  auto o = *res;
  *out_has_alpha = o->has_channel(heif_channel_Alpha) ? 1 : 0;
  struct { heif_channel c; void* p; } pl[4] = {{heif_channel_Y, oy}, {heif_channel_Cb, ocb}, {heif_channel_Cr, ocr}, {heif_channel_Alpha, oa}};
  for (auto& q : pl) {
    if (!o->has_channel(q.c)) { if (q.c == heif_channel_Alpha) continue; return -5; }
    if (!q.p) continue;
    size_t stride; const uint8_t* src = o->get_channel_memory(q.c, &stride);
    const int pw = o->get_width(q.c), ph = o->get_height(q.c), b = o->get_bits_per_pixel(q.c) > 8 ? 2 : 1;
    for (int r = 0; r < ph; r++) memcpy((uint8_t*)q.p + (size_t)r * pw * b, src + r * stride, (size_t)pw * b);
  }
  return 0;
}
