/*
 * b200_heif_plugin_abi.h -- the slice of libheif's plugin ABI that libb200heif.so implements, declared locally so the
 * product builds without libheif's headers.  Layout and values mirror (and are cross-checked by
 * tests/test_plugin_abi.py against) the reference:
 *   heif_error, error / suberror codes                  libheif/api/libheif/heif_error.h:35-301
 *   heif_compression_format                             libheif/api/libheif/heif_context.h:44-52
 *   heif_colorspace / heif_chroma / heif_channel        libheif/api/libheif/heif_image.h:53-150
 *   heif_decoder_plugin (api version 5/6, 18 members)   libheif/api/libheif/heif_plugin.h:85-169
 *   heif_encoder_plugin (api version 4, 35 members)     libheif/api/libheif/heif_plugin.h:192-313
 *   heif_plugin_info                                    libheif/api/libheif/heif_library.h:155-167
 * A maintainer integrating into libheif proper would include <libheif/heif_plugin.h> instead (see INTEGRATION.md).
 */
#ifndef B200_HEIF_PLUGIN_ABI_H
#define B200_HEIF_PLUGIN_ABI_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200h_error { int code; int subcode; const char* message; } b200h_error;   /* == heif_error */
enum { B200H_ERR_OK = 0, B200H_ERR_INVALID_INPUT = 2, B200H_ERR_UNSUPPORTED_FEATURE = 4, B200H_ERR_USAGE = 5,
       B200H_ERR_MEMORY = 6, B200H_ERR_DECODER_PLUGIN = 7, B200H_ERR_ENCODER_PLUGIN = 8 };
enum { B200H_SUBERR_UNSPECIFIED = 0, B200H_SUBERR_END_OF_DATA = 100, B200H_SUBERR_SECURITY_LIMIT = 1000,
       B200H_SUBERR_UNSUPPORTED_CODEC = 3000, B200H_SUBERR_UNSUPPORTED_IMAGE_TYPE = 3001, B200H_SUBERR_UNSUPPORTED_BIT_DEPTH = 4000 };
enum { B200H_COMPRESSION_HEVC = 1 };
enum { B200H_COLORSPACE_YCBCR = 0, B200H_COLORSPACE_RGB = 1, B200H_COLORSPACE_MONOCHROME = 2 };
enum { B200H_CHANNEL_Y = 0, B200H_CHANNEL_CB = 1, B200H_CHANNEL_CR = 2 };

typedef struct b200h_image b200h_image;                       /* heif_image (opaque) */
typedef struct b200h_security_limits {                        /* leading members of heif_security_limits (heif_security.h:37-62) */
  uint8_t version; uint64_t max_image_size_pixels;
} b200h_security_limits;
typedef struct b200h_format_description { int format; } b200h_format_description;
typedef struct b200h_decoder_options { int format; int strict_decoding; int num_threads; const b200h_security_limits* limits; } b200h_decoder_options;

typedef struct b200h_decoder_plugin {                         /* == heif_decoder_plugin, member for member */
  int plugin_api_version;
  const char* (*get_plugin_name)(void);
  void (*init_plugin)(void);
  void (*deinit_plugin)(void);
  int (*does_support_format)(int format);
  b200h_error (*new_decoder)(void** decoder);
  void (*free_decoder)(void* decoder);
  b200h_error (*push_data)(void* decoder, const void* data, size_t size);
  b200h_error (*decode_image)(void* decoder, b200h_image** out_img);
  void (*set_strict_decoding)(void* decoder, int flag);
  const char* id_name;
  b200h_error (*decode_next_image)(void* decoder, b200h_image** out_img, const b200h_security_limits* limits);
  uint32_t minimum_required_libheif_version;
  int (*does_support_format2)(const b200h_format_description* format);
  b200h_error (*new_decoder2)(void** decoder, const b200h_decoder_options* options);
  b200h_error (*push_data2)(void* decoder, const void* data, size_t size, uintptr_t user_data);
  b200h_error (*flush_data)(void* decoder);
  b200h_error (*decode_next_image2)(void* decoder, b200h_image** out_img, uintptr_t* out_user_data, const b200h_security_limits* limits);
} b200h_decoder_plugin;

typedef struct b200h_encoder_parameter {                      /* == heif_encoder_parameter (heif_plugin.h:323-360) */
  int version; const char* name; int type;
  union {
    struct { int default_value; uint8_t have_minimum_maximum; int minimum; int maximum; int* valid_values; int num_valid_values; } integer;
    struct { const char* default_value; const char* const* valid_values; } string;
    struct { int default_value; } boolean;
  };
  int has_default;
} b200h_encoder_parameter;

typedef struct b200h_encoder_plugin {                         /* == heif_encoder_plugin, member for member */
  int plugin_api_version;
  int compression_format;
  const char* id_name;
  int priority;
  int supports_lossy_compression;
  int supports_lossless_compression;
  const char* (*get_plugin_name)(void);
  void (*init_plugin)(void);
  void (*cleanup_plugin)(void);
  b200h_error (*new_encoder)(void** encoder);
  void (*free_encoder)(void* encoder);
  b200h_error (*set_parameter_quality)(void* encoder, int quality);
  b200h_error (*get_parameter_quality)(void* encoder, int* quality);
  b200h_error (*set_parameter_lossless)(void* encoder, int lossless);
  b200h_error (*get_parameter_lossless)(void* encoder, int* lossless);
  b200h_error (*set_parameter_logging_level)(void* encoder, int logging);
  b200h_error (*get_parameter_logging_level)(void* encoder, int* logging);
  const b200h_encoder_parameter** (*list_parameters)(void* encoder);
  b200h_error (*set_parameter_integer)(void* encoder, const char* name, int value);
  b200h_error (*get_parameter_integer)(void* encoder, const char* name, int* value);
  b200h_error (*set_parameter_boolean)(void* encoder, const char* name, int value);
  b200h_error (*get_parameter_boolean)(void* encoder, const char* name, int* value);
  b200h_error (*set_parameter_string)(void* encoder, const char* name, const char* value);
  b200h_error (*get_parameter_string)(void* encoder, const char* name, char* value, int value_size);
  void (*query_input_colorspace)(int* inout_colorspace, int* inout_chroma);
  b200h_error (*encode_image)(void* encoder, const b200h_image* image, int image_class);
  b200h_error (*get_compressed_data)(void* encoder, uint8_t** data, int* size, int* type);
  void (*query_input_colorspace2)(void* encoder, int* inout_colorspace, int* inout_chroma);
  void (*query_encoded_size)(void* encoder, uint32_t input_width, uint32_t input_height, uint32_t* encoded_width, uint32_t* encoded_height);
  uint32_t minimum_required_libheif_version;
  b200h_error (*start_sequence_encoding)(void* encoder, const b200h_image* image, int image_class, uint32_t framerate_num,
                                         uint32_t framerate_denom, const void* options);
  b200h_error (*encode_sequence_frame)(void* encoder, const b200h_image* image, uintptr_t frame_nr);
  b200h_error (*end_sequence_encoding)(void* encoder);
  b200h_error (*get_compressed_data2)(void* encoder, uint8_t** data, int* size, uintptr_t* frame_nr, int* is_keyframe, int* more_frame_packets);
  int does_indicate_keyframes;
} b200h_encoder_plugin;

typedef struct b200h_plugin_info { int version; int type; const void* plugin; void* internal_handle; } b200h_plugin_info;   /* == heif_plugin_info (heif_library.h:161-167); type 0 = encoder, 1 = decoder; internal_handle is written by libheif's loader */

/* Exported by libb200heif.so:
 *   plugin_info          -- the symbol libheif's loader looks up (libheif/plugins_unix.cc:103-119): the DECODER plugin
 *   b200_encoder_plugin_info -- the same structure for the encoder plugin (register with heif_register_encoder_plugin)
 *   b200_get_decoder_plugin / b200_get_encoder_plugin -- plugin tables for heif_register_*_plugin()
 *   b200_plugin_bind_libheif(handle) -- hosts that dlopen()ed libheif privately pass its handle here; otherwise the
 *                          heif_image_* entry points are looked up with dlsym(RTLD_DEFAULT, ...) on first use. */
extern b200h_plugin_info plugin_info;
extern b200h_plugin_info b200_encoder_plugin_info;
const b200h_decoder_plugin* b200_get_decoder_plugin(void);
const b200h_encoder_plugin* b200_get_encoder_plugin(void);
/* the GPU encoder's table (id "b200-gpu", priority 60): 8-bit 4:2:0 / monochrome input, log2-ctb-size 5..6, WPP always on */
const b200h_encoder_plugin* b200_get_gpu_encoder_plugin(void);
int b200_plugin_bind_libheif(void* dl_handle);
/* Submission queue of the decoder plugin (concurrent decode_next_image2 calls are decoded as one batch, see b200_plugin.cc):
   out3 = {batches decoded, pictures decoded, largest batch}. */
void b200_plugin_queue_stats(uint64_t out3[3]);

#ifdef __cplusplus
}
#endif
#endif
