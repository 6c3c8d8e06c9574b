// Layout of include/b200_heif_plugin_abi.h next to the reference's own headers (libheif/api/libheif/heif_plugin.h,
// heif_error.h, heif_library.h).  Prints one line per size, offset and constant the mirror depends on, always under the
// reference's name:
//   g++ -std=c++17 tests/abi/abi_check.cc                      -> what the mirror has (tests/test_plugin.py)
//   g++ -std=c++17 -DREFERENCE -I<libheif>/libheif/api -I<dir of heif_version.h> tests/abi/abi_check.cc
//                                                               -> what libheif has (tests/golden/abi/reference_layout.txt)
#include <cstddef>
#include <cstdint>
#include <cstdio>
#ifdef REFERENCE
#include <libheif/heif.h>
#include <libheif/heif_plugin.h>
#define T(mirror, ref) ref
#else
#include "../../include/b200_heif_plugin_abi.h"
#define T(mirror, ref) mirror
#endif

struct NclxPublic { uint8_t version; int color_primaries; int transfer_characteristics; int matrix_coefficients; uint8_t full_range_flag; };

#define SIZE(m, r) printf("sizeof %s %zu\n", #r, sizeof(T(m, r)));
#define OFF(m, r, f) printf("offsetof %s.%s %zu\n", #r, #f, offsetof(T(m, r), f));
#define VAL(m, r) printf("value %s %lld\n", #r, (long long)(T(m, r)));

#define D(f) OFF(b200h_decoder_plugin, heif_decoder_plugin, f)
#define E(f) OFF(b200h_encoder_plugin, heif_encoder_plugin, f)

int main() {
  SIZE(b200h_error, heif_error) OFF(b200h_error, heif_error, message)
  SIZE(b200h_decoder_plugin, heif_decoder_plugin)
  D(plugin_api_version) D(get_plugin_name) D(does_support_format) D(new_decoder) D(push_data) D(decode_image)
  D(set_strict_decoding) D(id_name) D(decode_next_image) D(minimum_required_libheif_version) D(does_support_format2)
  D(new_decoder2) D(push_data2) D(flush_data) D(decode_next_image2)
  SIZE(b200h_encoder_plugin, heif_encoder_plugin)
  E(compression_format) E(id_name) E(priority) E(supports_lossless_compression) E(new_encoder) E(list_parameters)
  E(get_parameter_string) E(query_input_colorspace) E(encode_image) E(get_compressed_data) E(query_input_colorspace2)
  E(query_encoded_size) E(minimum_required_libheif_version) E(start_sequence_encoding) E(get_compressed_data2)
  E(does_indicate_keyframes)
  SIZE(b200h_encoder_parameter, heif_encoder_parameter) OFF(b200h_encoder_parameter, heif_encoder_parameter, has_default)
  SIZE(b200h_decoder_options, heif_decoder_plugin_options) OFF(b200h_decoder_options, heif_decoder_plugin_options, limits)
  OFF(b200h_security_limits, heif_security_limits, max_image_size_pixels)
  SIZE(b200h_plugin_info, heif_plugin_info)
  VAL(B200H_ERR_DECODER_PLUGIN, heif_error_Decoder_plugin_error) VAL(B200H_ERR_ENCODER_PLUGIN, heif_error_Encoder_plugin_error)
  VAL(B200H_ERR_UNSUPPORTED_FEATURE, heif_error_Unsupported_feature) VAL(B200H_ERR_MEMORY, heif_error_Memory_allocation_error)
  VAL(B200H_ERR_USAGE, heif_error_Usage_error)
  VAL(B200H_SUBERR_SECURITY_LIMIT, heif_suberror_Security_limit_exceeded) VAL(B200H_SUBERR_UNSUPPORTED_CODEC, heif_suberror_Unsupported_codec)
  VAL(B200H_SUBERR_END_OF_DATA, heif_suberror_End_of_data) VAL(B200H_SUBERR_UNSUPPORTED_BIT_DEPTH, heif_suberror_Unsupported_bit_depth)
  VAL(B200H_COMPRESSION_HEVC, heif_compression_HEVC) VAL(B200H_COLORSPACE_YCBCR, heif_colorspace_YCbCr)
  VAL(B200H_COLORSPACE_MONOCHROME, heif_colorspace_monochrome)
  VAL(B200H_CHANNEL_Y, heif_channel_Y) VAL(B200H_CHANNEL_CB, heif_channel_Cb) VAL(B200H_CHANNEL_CR, heif_channel_Cr)
  VAL(1, heif_chroma_420) VAL(1, heif_plugin_type_decoder) VAL(0, heif_plugin_type_encoder)   // what b200_plugin.cc passes
  VAL(((1u << 24) | (21u << 16)), LIBHEIF_MAKE_VERSION(1, 21, 0))
  OFF(NclxPublic, heif_color_profile_nclx, full_range_flag) OFF(NclxPublic, heif_color_profile_nclx, matrix_coefficients)
  return 0;
}
