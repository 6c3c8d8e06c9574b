/*
 * b200_heif.h -- C ABI of libb200heif.so: the H100-native replacement for libheif's per-tile decode
 * pixel pipeline (HEVC-intra decoder in the libde265 role + colour-conversion / rotate / mirror / crop /
 * overlay post-stage).  Plain pointers and sizes only; no C++ or torch types.
 *
 * Every entry point cites the reference interface it replaces (paths relative to the libheif tree).
 * Device pointers are ordinary CUDA device pointers of the current device; `stream` is a cudaStream_t
 * passed as void* (NULL = default stream).  All functions return 0 on success or a negative B200_E_* code;
 * b200_last_error() gives a thread-local message.  Nothing here falls back to a CPU path: without a
 * CUDA device the device functions fail with B200_E_CUDA.
 */
#ifndef B200_HEIF_H
#define B200_HEIF_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_OK 0
#define B200_E_INVALID (-1)      /* bad argument */
#define B200_E_UNSUPPORTED (-2)  /* valid input outside the supported tool set (maps to heif_error_Unsupported_feature) */
#define B200_E_BITSTREAM (-3)    /* corrupt HEVC stream (maps to heif_error_Decoder_plugin_error) */
#define B200_E_CUDA (-4)         /* CUDA runtime error / no device */
#define B200_E_LIMIT (-5)        /* security limit exceeded (heif_security_limits.max_image_size_pixels) */

const char* b200_last_error(void);
int b200_version(void);

/* ------------------------------------------------------------------------------------------------
 * Colour post-stage (K6): chroma upsample + YCbCr->RGB + bit depth / interleave / endianness, fused with
 * the geometric transforms, one pass over HBM.
 * Replaces: convert_colorspace()                     libheif/color-conversion/colorconversion.cc:490-623
 *           Op_YCbCr_to_RGB<T>                       libheif/color-conversion/yuv2rgb.cc:92-292
 *           Op_YCbCr420_to_RGB24 / _RGB32            yuv2rgb.cc:345-426 / :481-562
 *           Op_YCbCr420_to_RRGGBBaa                  yuv2rgb.cc:622-734
 *           Op_RGB_to_RGB24_32, Op_to_sdr_planes     rgb2rgb.cc:71-150, hdr_sdr.cc:147-200
 *           HeifPixelImage::rotate_ccw / mirror_inplace / crop   libheif/image/pixelimage.cc:1175-1546
 * ------------------------------------------------------------------------------------------------ */

/* heif_chroma values of the reference (api/libheif/heif_image.h) used for input and output layouts */
enum b200_chroma {
  B200_CHROMA_MONO = 0, B200_CHROMA_420 = 1, B200_CHROMA_422 = 2, B200_CHROMA_444 = 3,
  B200_CHROMA_INTERLEAVED_RGB = 10, B200_CHROMA_INTERLEAVED_RGBA = 11,
  B200_CHROMA_INTERLEAVED_RRGGBB_BE = 12, B200_CHROMA_INTERLEAVED_RRGGBBAA_BE = 13,
  B200_CHROMA_INTERLEAVED_RRGGBB_LE = 14, B200_CHROMA_INTERLEAVED_RRGGBBAA_LE = 15
};

/* One YCbCr (or monochrome) picture in device or host memory.  Samples are uint8 when bit_depth == 8,
   otherwise native-endian uint16 (reference plane layout, pixelimage.cc:389-501).  Strides in bytes. */
typedef struct b200_planes {
  const void* y; const void* cb; const void* cr; const void* alpha;   /* alpha may be NULL */
  size_t y_stride, c_stride, alpha_stride;
  int width, height;       /* luma size */
  int chroma;              /* B200_CHROMA_MONO/420/422/444 */
  int bit_depth;           /* 8..16 (alpha must have the same depth) */
  /* CICP as carried by the image's nclx (nclx.h:121-173); 2 = unspecified */
  int colour_primaries, transfer_characteristics, matrix_coefficients, full_range;
} b200_planes;

/* Geometry applied BEFORE colour conversion (image-items/image_item.cc:947-1020 applies irot / imir / clap
   in ipma property order).  Any chain of those transforms is an affine map with coefficients in {-1,0,1}
   from an output pixel (u,v) back to the decoded picture; the host composes the chain by calling the
   b200_geometry_* functions in the same order libheif applies the properties. */
typedef struct b200_geometry {
  int m[6];          /* src_x = m[0]*u + m[1]*v + m[2] ;  src_y = m[3]*u + m[4]*v + m[5] */
  int out_w, out_h;  /* size of the transformed picture */
  /* The reference converts a subsampled picture to 4:4:4 before a transform its plane-wise code cannot express -- 4:2:0:
     rotate 90 with odd width, 180 with an odd side, 270 with odd height; any mirror with an odd side; crop with odd left
     or top (pixelimage.cc:1187-1215, 1370-1396, 1458-1481).  The composition functions record that point: transforms
     before it are kept in `pre` (applied to the subsampled planes), then chroma is upsampled bilinearly
     (Op_YCbCr420_bilinear_to_YCbCr444, what convert_colorspace picks there), then `m` applies to the 4:4:4 picture. */
  int chroma;        /* chroma format the chain started from (B200_CHROMA_*); decides the rules above */
  int detour;        /* 1: the 4:4:4 conversion point was reached */
  int pre[6]; int pre_w, pre_h;
} b200_geometry;

void b200_geometry_identity(int width, int height, b200_geometry* g);               /* = b200_geometry_init(width, height, B200_CHROMA_420, g) */
void b200_geometry_init(int width, int height, int chroma, b200_geometry* g);
int b200_geometry_rotate_ccw(b200_geometry* g, int degrees /*0,90,180,270*/);   /* HeifPixelImage::rotate_ccw, pixelimage.cc:1175-1333 */
int b200_geometry_mirror(b200_geometry* g, int direction /*heif_transform_mirror_direction: 0 = vertical (top<->bottom), 1 = horizontal (left<->right)*/); /* pixelimage.cc:1336-1424 */
int b200_geometry_crop(b200_geometry* g, int left, int right, int top, int bottom); /* HeifPixelImage::crop, inclusive right/bottom, pixelimage.cc:1433-1546 */

typedef struct b200_color_options {
  int out_chroma;                 /* B200_CHROMA_INTERLEAVED_* or B200_CHROMA_444 (planar RGB) */
  int out_bit_depth;              /* 0 = reference default (8 for RGB/RGBA, input depth for RRGGBB*, colorconversion.cc:591-605) */
  int chroma_upsampling;          /* 0 = reference default planner choice (nearest neighbour), 1 = bilinear forced
                                     (heif_color_conversion_options.only_use_preferred_chroma_algorithm) */
} b200_color_options;

/* Device -> device.  `out` points to out_h rows of out_stride bytes (planar RGB: out, out_g, out_b).
   Reports which reference op chain was mirrored in *pipeline (bit mask B200_PIPE_*), may be NULL. */
#define B200_PIPE_INT420 1       /* Op_YCbCr420_to_RGB24 / RGB32 integer arithmetic */
#define B200_PIPE_FLOAT 2        /* Op_YCbCr_to_RGB<T> / Op_YCbCr420_to_RRGGBBaa float arithmetic */
#define B200_PIPE_BILINEAR 4     /* Op_YCbCr420_bilinear_to_YCbCr444 first */
#define B200_PIPE_SDR_SHIFT 8    /* Op_to_sdr_planes (>> (bpp-8)) */
int b200_color_convert_device(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt,
                              void* out, void* out_g, void* out_b, size_t out_stride, void* stream, int* pipeline);

/* Device -> device: b200_color_convert_device followed by HeifPixelImage::scale_nearest_neighbor
   (libheif/image/pixelimage.cc:1783-1972, what heif_image_scale_image runs) to scale_w x scale_h, without the full-size
   RGB picture: only the pixels the scaler keeps are converted.  Result pixel (x, y) = pixel (x * out_w / scale_w,
   y * out_h / scale_h) (64-bit integer arithmetic) of the b200_color_convert_device picture, all components together (the
   planes of planar RGB with the same indices); up- and down-scaling, any scale_w, scale_h >= 1.  out / out_g / out_b /
   out_stride describe the scale_w x scale_h result.  The 4:4:4 conversion point and bilinear upsampling keep their full-size
   4:4:4 intermediates; only the last conversion is scaled.  *pipeline as for the unscaled call.  B200_E_INVALID (before any
   CUDA call, message naming the argument) for scale_w or scale_h < 1 or a NULL in / geom / opt / out; everything else as
   b200_color_convert_device. */
int b200_color_convert_scaled_device(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt,
                                     int scale_w, int scale_h, void* out, void* out_g, void* out_b, size_t out_stride,
                                     void* stream, int* pipeline);

/* Host -> host form with H2D / D2H inside (what a libheif ColorConversionOperation calls: integration/b200_color_op.cc).
   Pageable operands move through a page-locked bounce buffer in bands (host threads fill / drain band k while the DMA
   engine moves band k - 1); the device buffers, the bounce buffer and the stream are kept per GPU for the life of the
   process and concurrent callers are serialised.  Page-locked operands (b200_host_alloc / b200_host_register) are copied
   directly. */
int b200_color_convert_host(const b200_planes* in, const b200_geometry* geom, const b200_color_options* opt,
                            void* out, void* out_g, void* out_b, size_t out_stride, int* pipeline);

/* Encoder-side direction (what heif_context_encode_image runs before the encoder plugin sees the picture,
   HeifContext::encode_image -> Encoder::convert_colorspace_for_encoding, libheif/context.cc:1642, libheif/codecs/encoder.cc:116-175):
   interleaved RGB (has_alpha = 0, 3 bytes / pixel) or RGBA (has_alpha = 1, 4 bytes / pixel), 8 bit
     -> planar YCbCr 8 bit in the chroma format, matrix and range that `out` names.
   Replaces: Op_RGB24_32_to_YCbCr::convert_colorspace   libheif/color-conversion/rgb2yuv.cc:575-808
             (float arithmetic in the reference's order; 4:2:0 chroma from the integer mean of the 2x2 RGB quad with the
              reference's odd-width / odd-height border rules; 4:2:2 chroma from the left pixel; limited range
              Y*0.85547+16, C*0.875+128; nclx "unspecified" (2) -> matrix 6 / primaries 1 as colorconversion.cc:513-515 does)
   `out`: caller-owned planes, written through the (const-declared) pointers of b200_planes (y, cb, cr required; alpha optional: receives the source alpha, or 0xff when has_alpha = 0),
   width / height / chroma (B200_CHROMA_420 / 422 / 444) / bit_depth (8) / colour_primaries / matrix_coefficients /
   full_range are inputs.  matrix_coefficients 0, 8, 11, 14 -> B200_E_UNSUPPORTED (the reference's op refuses them as
   well, rgb2yuv.cc:536-539). */
int b200_rgb_to_ycbcr_device(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out, void* stream);
/* Host -> host form: stages its operands as b200_color_convert_host does, with the same buffers, kept per GPU for the life
   of the process. */
int b200_rgb_to_ycbcr_host(const void* rgb, size_t rgb_stride, int has_alpha, const b200_planes* out);

/* Encoder-side direction for every RGB layout heif_context_encode_image accepts: the chain convert_colorspace
   (colorconversion.cc:490-623) picks from the input to YCbCr at the input's depth (output_bpp = 0, encoder.cc:168-174).
   Replaces: Op_RGB24_32_to_YCbCr              rgb2yuv.cc:506-808 (interleaved RGB / RGBA 8 bit; b200_rgb_to_ycbcr_device's kernel)
             Op_RRGGBBxx_HDR_to_YCbCr420       rgb2yuv.cc:311-503 (RRGGBB[AA] BE / LE, full range, 4:2:0)
             Op_RGB_to_YCbCr<uint8_t / uint16_t> rgb2yuv.cc:30-305 (planar RGB; matrix 0 and 8 branches, limited range x219/256,
                                               x224/256; 4:2:0 chroma from the float mean of the quad, 4:2:2 from the left pixel)
             Op_RGB24_32_to_YCbCr444_GBR       rgb2yuv.cc:812-919 (interleaved 8 bit, matrix 0, full range, 4:4:4)
   with the lossless steps the reference runs before Op_RGB_to_YCbCr -- Op_RRGGBBaa_swap_endianness, Op_RRGGBBaa_BE_to_RGB_HDR,
   Op_RGB24_32_to_RGB (rgb2rgb.cc) -- folded into the kernel's loader. */
typedef struct b200_rgb_image {
  const void* rgb; size_t rgb_stride;            /* interleaved layouts: the one plane (> 8 bit: bytes in the layout's order) */
  const void* r; const void* g; const void* b; const void* alpha;   /* planar (chroma B200_CHROMA_444): > 8 bit as native uint16;
                                                                       alpha may be NULL */
  size_t r_stride, g_stride, b_stride, alpha_stride;
  int width, height;
  int chroma;                 /* B200_CHROMA_INTERLEAVED_* (heif_chroma_interleaved_*), or B200_CHROMA_444 = planar R, G, B */
  int bit_depth;              /* 8 for RGB / RGBA, 9..16 for RRGGBB[AA], 8..16 planar */
  int alpha_bit_depth;        /* planar alpha plane: 0 = bit_depth */
} b200_rgb_image;

typedef struct b200_rgb_to_ycbcr_options {   /* the two members of heif_color_conversion_options the planner reads here */
  int chroma_downsampling;    /* heif_chroma_downsampling_algorithm: 1 nearest neighbour, 2 average (libheif's default), 3 sharp YUV */
  int only_use_preferred;     /* only_use_preferred_chroma_algorithm */
} b200_rgb_to_ycbcr_options;

/* *pipeline of the calls below: the reference operations of the chain (bit mask) */
#define B200_YCC_PIPE_RGB24_32 1     /* Op_RGB24_32_to_YCbCr */
#define B200_YCC_PIPE_GBR444 2       /* Op_RGB24_32_to_YCbCr444_GBR */
#define B200_YCC_PIPE_HDR420 4       /* Op_RRGGBBxx_HDR_to_YCbCr420 */
#define B200_YCC_PIPE_PLANAR 8       /* Op_RGB_to_YCbCr<T> */
#define B200_YCC_PIPE_UNPACK 16      /* Op_RGB24_32_to_RGB / Op_RRGGBBaa_BE_to_RGB_HDR before it */
#define B200_YCC_PIPE_SWAP 32        /* Op_RRGGBBaa_swap_endianness before that */

/* Host only, no CUDA: the chain the reference would run, or the refusal the conversion would return.
   `out`: width / height (= the input's) / chroma (B200_CHROMA_420 / 422 / 444) / bit_depth (= the input's) / colour_primaries /
   matrix_coefficients / full_range are read (nclx "unspecified" (2) -> matrix 6 / primaries 1, colorconversion.cc:567-573).
   opt NULL = libheif's defaults (average, not only preferred).
   B200_E_UNSUPPORTED: matrix_coefficients 11 or 14 (the reference has no chain either); a planar alpha plane whose depth
   differs from the colour depth (the reference adds Op_adjust_alpha_bit_depth: not mirrored); only_use_preferred with
   average or sharp-YUV downsampling to 4:2:0 / 4:2:2 (the reference then converts to 4:4:4 and downsamples with
   Op_YCbCr444_to_YCbCr420/422_average, or has no chain: not mirrored). */
int b200_rgb_to_ycbcr_plan(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline);
/* Device -> device.  `out` as above, plus the caller-owned planes (uint8 at 8 bit, native uint16 above), written through the
   const-declared pointers; out->alpha is required exactly when the input has alpha (the result has an alpha plane then,
   colorconversion.cc:575-585) and receives it unchanged.  pipeline may be NULL. */
int b200_rgb_to_ycbcr_ex_device(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, void* stream, int* pipeline);
/* Host -> host form: stages its operands with the buffers of b200_rgb_to_ycbcr_host. */
int b200_rgb_to_ycbcr_ex_host(const b200_rgb_image* in, const b200_planes* out, const b200_rgb_to_ycbcr_options* opt, int* pipeline);

/* nclx helper: the 4 float coefficients exactly as nclx.cc:84-173 derives them */
void b200_ycbcr_to_rgb_coefficients(int matrix_coefficients, int colour_primaries, float out_coeffs[4] /* r_cr,g_cb,g_cr,b_cb */);

/* ------------------------------------------------------------------------------------------------
 * Overlay compositing (SURVEY 8 a11) and nearest-neighbour plane scaling (a12).  Device -> device.
 * Replaces: HeifPixelImage::fill_RGB_16bit           libheif/image/pixelimage.cc:1549-1621
 *           HeifPixelImage::overlay                  libheif/image/pixelimage.cc:1637-1780
 *           (driven by ImageItem_Overlay::decode_overlay_image, libheif/image-items/overlay.cc:290-393: an 8-bit planar
 *            RGB 4:4:4 canvas filled with background >> 8, children converted to planar RGB 4:4:4 -- use
 *            b200_color_convert_device with out_chroma = B200_CHROMA_444 -- and composited in 'iovl' order)
 *           HeifPixelImage::scale_nearest_neighbor   libheif/image/pixelimage.cc:1783-1972
 * The overlay reproduces the reference's arithmetic (in*a + out*(255-a)) / 255 and its clipping, including the loop
 * bounds it uses for negative offsets (fewer rows / columns are drawn than overlap; see oracle/color_oracle.c).
 * ------------------------------------------------------------------------------------------------ */
/* planes R,G,B of width x height bytes: every sample = background_rgba[c] >> 8 */
int b200_overlay_fill_device(void* const planes[3], const size_t strides[3], int width, int height, const uint16_t background_rgba[4], void* stream);
/* overlay[3] = alpha plane of the child or NULL (opaque copy).  An overlay entirely outside the canvas draws nothing and
   is not an error (overlay.cc:372-379). */
int b200_overlay_device(void* const canvas[3], const size_t canvas_strides[3], int canvas_w, int canvas_h, const void* const overlay[4],
                        const size_t overlay_strides[4], int overlay_w, int overlay_h, int32_t dx, int32_t dy, void* stream);
/* One plane: out[y][x] = in[y * image_h_in / image_h_out][x * image_w_in / image_w_out] for x < out_w, y < out_h, with the
   IMAGE sizes in the index arithmetic also for subsampled planes (as the reference does); bytes_per_pixel = interleaved
   components x bytes per sample (1, 2, 3, 4, 6 or 8).  The caller loops over the planes like pixelimage.cc:1917. */
int b200_scale_nearest_device(const void* in, size_t in_stride, void* out, size_t out_stride, uint32_t out_w, uint32_t out_h,
                              uint32_t image_w_in, uint32_t image_h_in, uint32_t image_w_out, uint32_t image_h_out, int bytes_per_pixel, void* stream);

/* ------------------------------------------------------------------------------------------------
 * HEVC intra encoder (host): produces the synthetic inputs of BASELINE configs 2-5 and backs the
 * heif_encoder_plugin (libheif/api/libheif/heif_plugin.h:192-313) exported by this library.
 * Role of: x265 behind libheif/plugins/encoder_x265.cc:752-1051 (encode_image) and :1186-1244
 * (get_compressed_data: one NAL per call, no start code), driven by libheif/codecs/hevc_enc.cc:33-115.
 * Output here: every NAL of the access unit (VPS, SPS, PPS, slice segments), each prefixed by its
 * uint32 big-endian length -- the framing libheif pushes into a decoder plugin.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b200_hevc_enc_params {
  int width, height;                 /* luma size; coded size is rounded up to 8 and cropped by the conformance window */
  int bit_depth;                     /* 8, 10, 12 */
  int chroma_format_idc;             /* 1 = 4:2:0, 0 = 4:0:0 */
  int log2_ctb_size;                 /* 4, 5, 6 */
  int qp, init_qp;                   /* slice QP target and pps init_qp_minus26 + 26 */
  int max_transform_hierarchy_depth_intra;
  int sao, sign_data_hiding, transform_skip, strong_intra_smoothing;
  int cu_qp_delta, diff_cu_qp_delta_depth, dqp_range;
  int cb_qp_offset, cr_qp_offset, slice_chroma_qp_offsets, slice_cb_qp_offset, slice_cr_qp_offset;
  int wpp;                           /* entropy_coding_sync_enabled_flag + entry points */
  int slice_ctb_rows;                /* > 0: start a new slice every N CTB rows */
  int dependent_slice_segments;      /* with slice_ctb_rows > 1 and !wpp: one dependent segment per CTB row */
  int loop_filter_across_slices, slice_loop_filter_across_slices;
  int deblocking_disabled, beta_offset_div2, tc_offset_div2;
  int slice_deblocking_override, slice_deblocking_disabled, slice_beta_offset_div2, slice_tc_offset_div2;
  int mode_decision;                 /* 0 = pseudo-random modes/partitions (syntax coverage), 1 = SAD-based choice */
  int split_threshold;               /* activity threshold of the CU split heuristic */
  int still_picture;                 /* Main Still Picture profile signalling for 8-bit 4:2:0 */
  int vui_present, colour_description_present, colour_primaries, transfer_characteristics, matrix_coefficients, full_range;
  uint32_t seed;                     /* LCG seed (SURVEY 8d: 0xB200 + tile index) */
  int scaling_lists;                 /* 0 = off, 1 = scaling_list_enabled_flag with the default lists (Tables 7-5 / 7-6), 2 = lists coded in the SPS,
                                        3 = lists coded in the PPS (both with predicted / default / explicit matrices chosen by the LCG) */
  int pcm;                           /* 0 = off; 1 = pcm_enabled_flag, some 2Nx2N coding units coded as PCM at the full bit depth; 2 = PCM bit depths
                                        reduced by 1 (luma) / 2 (chroma) and pcm_loop_filter_disabled_flag = 1 */
  int transquant_bypass;             /* 0 = off; 1 = transquant_bypass_enabled_flag, some coding units lossless; 2 = every coding unit lossless */
  int tile_cols, tile_rows;          /* > 1 in either: tiles_enabled_flag (6.5.1); not together with wpp */
  int tiles_uniform;                 /* 1 = uniform_spacing_flag, 0 = column widths / row heights drawn by the LCG and coded explicitly */
  int loop_filter_across_tiles;      /* loop_filter_across_tiles_enabled_flag */
  int slice_per_tile;                /* 1 = every tile is a slice of its own, 0 = one slice holds all tiles (one entry point per tile) */
  int speed;                         /* GPU encoder only (the host encoder ignores it): mode-decision speed 0..2, see below */
} b200_hevc_enc_params;

void b200_hevc_enc_params_default(b200_hevc_enc_params* p);
/* planes: uint8 (bit_depth 8) or native-endian uint16; *out_data is malloc'ed, release with b200_free */
int b200_hevc_encode_intra(const b200_hevc_enc_params* p, const void* y, const void* cb, const void* cr, size_t y_stride,
                           size_t c_stride, uint8_t** out_data, size_t* out_size);
void b200_free(void* p);

/* ------------------------------------------------------------------------------------------------
 * HEVC intra encoder (GPU): n same-sized 8-bit pictures (a grid's tiles, or one image) per call, analysis / reconstruction
 * and CABAC as sm_90a kernels, parameter sets / slice header / emulation prevention on the host.  Output framing as
 * b200_hevc_encode_intra: VPS, SPS, PPS and one IDR slice segment, each behind its uint32 BE length.
 * Coding decisions are deterministic (no LCG): the same input gives the same bytes, alone or in any batch.
 * Accepted b200_hevc_enc_params: width / height 8..16384 (coded size rounded up to 8, conformance window), log2_ctb_size 5
 * or 6, qp / init_qp 0..51, wpp = 1 (required), max_transform_hierarchy_depth_intra, strong_intra_smoothing, PPS and slice
 * Cb / Cr QP offsets, every deblocking field, still_picture, VUI / colour fields, speed.  mode_decision, split_threshold and
 * seed are ignored.  B200_E_UNSUPPORTED (message names the field): sao, sign_data_hiding, transform_skip, cu_qp_delta,
 * scaling_lists, pcm, transquant_bypass, tile_cols / tile_rows > 1, slice_ctb_rows, dependent_slice_segments, bit_depth != 8,
 * chroma_format_idc 2 / 3, wpp = 0.  B200_E_INVALID (message names `speed`): speed outside 0..2.  All validation happens
 * before any CUDA call.
 * speed trades compression for encoding time in the mode decision; the quadtree walk (CTB down to 8x8, NxN at 8x8) and the
 * final pass, which codes the chosen CUs closed loop in decoding order, are the same at every speed:
 *   0 (default): all 35 luma modes of every PU, decisions in closed loop (neighbours from the reconstruction);
 *   1: coarse-to-fine search of at most 18 modes per PU (planar, DC, angular 2, 6, .., 34 and the three MPMs, then the
 *      angular modes within 2 of the best angular one), closed loop;
 *   2: as 1, with open-loop decisions: neighbours from the source, no transform round trip before the final pass.
 * Pictures: b200_planes with width / height = the params', chroma B200_CHROMA_420 (chroma_format_idc 1) or B200_CHROMA_MONO
 * (0, cb / cr ignored), bit_depth 8.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b200_gpu_encoder b200_gpu_encoder;
typedef struct b200_gpu_encode_stats {
  double analyse_ms, entropy_ms;     /* CUDA events: E1 (analysis + reconstruction), E2 (CABAC) of the last call */
  double framing_ms, total_ms;       /* host clock: sub-stream D2H + framing; the whole call */
  uint64_t bytes, ctus, pictures;    /* access-unit bytes, CTBs and pictures of the last call */
  uint64_t mode_evaluations;         /* decision pass: candidate luma modes whose SATD was computed, over all PU searches */
  uint64_t cu_evaluations;           /* decision pass: coding units evaluated (the no-split CU and, at 8x8, the NxN one) */
} b200_gpu_encode_stats;

/* Host only, no CUDA: B200_OK if b200_gpu_encode_intra_* would accept these arguments, else the code and message it would
   return (the encode calls run the same check first). */
int b200_gpu_encode_check(const b200_hevc_enc_params* p, int n, const b200_planes* pics);
int b200_gpu_encoder_create(b200_gpu_encoder** enc);      /* on the current CUDA device */
void b200_gpu_encoder_destroy(b200_gpu_encoder* enc);
/* device planes; `stream` = cudaStream_t (NULL = default stream); returns when the access units are in host memory */
int b200_gpu_encode_intra_device(b200_gpu_encoder* enc, const b200_hevc_enc_params* p, int n, const b200_planes* pics, void* stream);
/* host planes (staged through a page-locked bounce buffer) */
int b200_gpu_encode_intra_host(b200_gpu_encoder* enc, const b200_hevc_enc_params* p, int n, const b200_planes* pics);
/* access unit of picture i of the last call (valid until the next call on this encoder) */
int b200_gpu_encoder_output(b200_gpu_encoder* enc, int i, const uint8_t** data, size_t* size);
/* picture i of the last call as reconstructed before in-loop filtering, cropped to width x height (host copy): what a decoder
   holds before deblocking.  cb / cr may be NULL. */
int b200_gpu_encoder_read_recon(b200_gpu_encoder* enc, int i, void* y, void* cb, void* cr, size_t y_stride, size_t c_stride);
int b200_gpu_encoder_get_stats(b200_gpu_encoder* enc, b200_gpu_encode_stats* out);
/* Host only: bytes reserved per CABAC sub-stream (one CTB row) -- the worst case of the syntax; a sub-stream that would need
   more fails the call instead of writing past it. */
size_t b200_gpu_encoder_substream_capacity(int width, int log2_ctb_size, int chroma_format_idc);
/* Resident E1 (analysis) warps per SM of the current device for the given speed (cudaOccupancyMaxActiveBlocksPerMultiprocessor):
   what sizes a batch that fills the device in one wave. */
int b200_gpu_encoder_e1_warps_per_sm(int speed, int* warps);

/* One call from an 8-bit RGB picture to the access units of a HEIC grid: colour conversion, tiling and HEVC coding on the
 * device -- what heif_context_encode_grid with the "b200-gpu" plugin does one tile per encode_image call
 * (libheif/image-items/grid.cc:886-906), as two batches on the GPU.
 * Tiles: cols = ceil(width / tile_w) x rows = ceil(height / tile_h), raster order; tile (c, r) is the tile_w x tile_h window at
 * (c * tile_w, r * tile_h), edge-replicated (clamped coordinates) where it overhangs the picture.  Its access unit is byte for
 * byte what b200_gpu_encode_intra_* writes for the 4:2:0 picture b200_rgb_to_ycbcr_ex_* makes from that padded window.
 * Input: RGB24 / RGBA32 (B200_CHROMA_INTERLEAVED_RGB / _RGBA) or planar 8-bit R, G, B (B200_CHROMA_444) with an optional alpha
 * plane.  Conversion target and SPS signalling: p's colour_primaries / matrix_coefficients / full_range; chroma_downsampling /
 * only_use_preferred from opt (NULL = libheif's defaults).  p: as for b200_gpu_encode_intra_* with chroma_format_idc 1;
 * width / height are set by the call (tile_w x tile_h).  An input with alpha gives a second batch of tiles, the padded alpha
 * windows coded as 4:0:0 pictures with the same parameters (libheif codes alpha through the same plugin the same way).
 * Output: b200_gpu_encoder_output(enc, i) -- i in [0, n) the colour tiles, [n, 2n) the alpha tiles (n = cols * rows);
 * b200_gpu_encoder_get_stats sums both batches; b200_gpu_encoder_read_recon holds the last batch coded (alpha when present).
 * Refusals, all before any CUDA call (b200_gpu_encode_rgb_grid_check): B200_E_UNSUPPORTED for a depth above 8 bits, for
 * what b200_rgb_to_ycbcr_plan refuses for this target, and for what b200_gpu_encode_check refuses for a tile_w x tile_h
 * picture; B200_E_INVALID for odd tile sizes or tiles outside 8..16384, NULL pointers, strides shorter than a row. */
typedef struct b200_grid_encode_info {
  int cols, rows, tile_w, tile_h;      /* tiles = ceil(W / tile_w) x ceil(H / tile_h), raster order */
  int width, height;                   /* grid output size = the input picture's size */
  int has_alpha;                       /* alpha tiles coded as 4:0:0 pictures in the same call */
  int pipeline;                        /* B200_YCC_PIPE_* of the colour chain, as b200_rgb_to_ycbcr_plan reports */
  double colour_ms, upload_ms;         /* CUDA events: colour kernels (summed over the bands of the host form), H2D of the host
                                          form (0 for the device form); E1 / E2 / framing stay in b200_gpu_encoder_get_stats */
} b200_grid_encode_info;

int b200_gpu_encode_rgb_grid_check(const b200_rgb_image* in, int tile_w, int tile_h, const b200_hevc_enc_params* p,
                                   const b200_rgb_to_ycbcr_options* opt);              /* host only, no CUDA */
/* device RGB; `stream` = cudaStream_t (NULL = default stream); returns when the access units are in host memory.
   info may be NULL. */
int b200_gpu_encode_rgb_grid_device(b200_gpu_encoder* enc, const b200_rgb_image* in, int tile_w, int tile_h,
                                    const b200_hevc_enc_params* p, const b200_rgb_to_ycbcr_options* opt,
                                    void* stream, b200_grid_encode_info* info);
/* host RGB: uploaded in row bands through the encoder's page-locked bounce buffer; band k is converted on the device while
   band k + 1 is in flight.  The device buffers stay with the encoder for its next call. */
int b200_gpu_encode_rgb_grid_host(b200_gpu_encoder* enc, const b200_rgb_image* in, int tile_w, int tile_h,
                                  const b200_hevc_enc_params* p, const b200_rgb_to_ycbcr_options* opt,
                                  b200_grid_encode_info* info);

/* ------------------------------------------------------------------------------------------------
 * HEVC intra decoder: header parsing on the host; CABAC + slice-data syntax, reconstruction, deblocking and SAO as
 * sm_90a kernels (CABAC can be moved to host threads with b200_decoder_set_front_end).
 * Replaces: the libde265 calls of libheif/plugins/decoder_libde265.cc -- de265_new_decoder :181,
 *   de265_push_NAL :360, de265_decode :402, de265_get_next_picture :410, de265_get_image_plane :137,
 *   de265_get_image_{colour_primaries,transfer_characteristics,matrix_coefficients,full_range_flag} :428-446,
 *   de265_free_decoder :233 -- and, for grids, the per-tile paste HeifPixelImage::copy_image_to
 *   (libheif/image/pixelimage.cc:1115-1172) driven by ImageItem_Grid::decode_and_paste_tile_image
 *   (libheif/image-items/grid.cc:482-577).
 * Input framing: every access unit is [uint32 BE length][NAL]... exactly as Decoder::get_compressed_data
 * (libheif/codecs/decoder.cc:275-308) hands it to push_data2.
 * ------------------------------------------------------------------------------------------------ */
typedef struct b200_decoder b200_decoder;

typedef struct b200_image_info {
  int width, height;          /* canvas size (single image: conformance-cropped picture size) */
  int tile_width, tile_height;
  int chroma;                 /* B200_CHROMA_MONO / 420 / 422 / 444 (= chroma_format_idc of the coded pictures) */
  int bit_depth;
  int colour_primaries, transfer_characteristics, matrix_coefficients, full_range;   /* from the SPS VUI, defaults 2/2/2/0 */
} b200_image_info;

typedef struct b200_decode_stats {
  double parse_ms, pack_ms, h2d_ms, gpu_ms, total_ms;   /* host wall-clock of the last decode call (gpu_ms: CUDA events) */
  double entropy_ms, recon_ms, deblock_ms, sao_ms;      /* per-kernel device times of the last call (entropy_ms: device front-end only) */
  uint64_t bitstream_bytes, command_bytes, coefficient_entries, transform_units, ctus, h2d_bytes, pixels;
  int kernel_launches;
  int front_end;                                        /* 0 = CABAC decoded on the host cores, 1 = on the GPU, 2 = on the GPU with the
                                                           reconstruction kernel running concurrently (entropy_ms then covers both),
                                                           3 = on the GPU, and after it the tile rows went through reconstruction .. colour
                                                           conversion in `bands` row bands, the D2H of a band overlapping the kernels of the
                                                           next (fused host entry points, large grids); recon_ms is then the whole band
                                                           pipeline, deblock_ms = sao_ms = 0 (B200_CHUNKS=0: separate kernels and times) */
  int bands;
} b200_decode_stats;

/* host_threads: CABAC parser threads (0 = number of online cores).  The CUDA device is the current one. */
int b200_decoder_create(b200_decoder** dec, int host_threads);
void b200_decoder_destroy(b200_decoder* dec);

/* Decode cols*rows independent access units (row-major grid tiles; 1x1 = a single image) into the decoder's
   device canvas (planar Y/Cb/Cr, 4:2:0 or 4:0:0).  canvas_w/h = 0 -> cols*tile_w x rows*tile_h.  Tiles overhanging
   the canvas are clipped like HeifPixelImage::copy_image_to does.  max_image_size_pixels = 0 -> unlimited
   (heif_security_limits, enforced per coded picture like decoder_libde265.cc:189-198).
   Asynchronous with respect to `stream` unless stats are requested (b200_decoder_get_stats synchronises). */
int b200_decoder_decode_grid(b200_decoder* dec, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                             uint64_t max_image_size_pixels, int canvas_w, int canvas_h, b200_image_info* info, void* stream);

/* Device planes of the canvas (valid until the next decode call on this decoder). */
int b200_decoder_get_planes(b200_decoder* dec, b200_planes* out);
/* Copy the canvas planes to host memory (D2H + synchronise).  cb/cr may be NULL for 4:0:0. */
int b200_decoder_read_planes(b200_decoder* dec, void* y, size_t y_stride, void* cb, void* cr, size_t c_stride, void* stream);
/* Reconstruction planes of tile `index` before/after deblocking (debug / parity of intermediate stages):
   stage 1 = before deblocking, 2 = after deblocking (coded size, no conformance crop).  Host copies. */
int b200_decoder_debug_read_tile(b200_decoder* dec, int index, int stage, void* y, void* cb, void* cr);
/* Where CABAC + slice-data syntax run: 1 (default) = on the GPU, one warp per WPP sub-stream / slice segment;
   0 = on the host cores (BASELINE north_star wording), host_threads parser threads.  Same command stream either way. */
int b200_decoder_set_front_end(b200_decoder* dec, int device);
int b200_decoder_set_debug_stage(b200_decoder* dec, int stage /* 0 = full pipeline, 1 = stop after reconstruction, 2 = stop after deblocking */);
int b200_decoder_get_stats(b200_decoder* dec, b200_decode_stats* out);
/* Re-launch the device kernels on the command stream already resident in HBM (no host parse, no H2D). */
int b200_decoder_rerun_device(b200_decoder* dec, void* stream);

/* Host only, no CUDA: what de265_get_image_width / _height / de265_get_bits_per_pixel / de265_get_chroma_format and the colour
   getters (decoder_libde265.cc:102-137, 428-446) would report for this access unit, from its parameter sets alone. */
int b200_probe_access_unit(const uint8_t* au, size_t au_size, uint64_t max_image_size_pixels, b200_image_info* info);

/* Fused convenience: decode grid -> geometry -> colour conversion -> interleaved RGB in HOST memory. */
int b200_decode_grid_to_rgb_host(b200_decoder* dec, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                 uint64_t max_image_size_pixels, int canvas_w, int canvas_h, const b200_geometry* geom /* NULL = identity */,
                                 const b200_color_options* opt, void* out, size_t out_stride, b200_image_info* info);

/* Fused: b200_decode_grid_to_rgb_host whose result is scaled to scale_w x scale_h -- heif_decode_image followed by
   heif_image_scale_image (HeifPixelImage::scale_nearest_neighbor, libheif/image/pixelimage.cc:1783-1972), as
   heif-thumbnailer does (examples/heif_thumbnailer.cc:148-207).  One scaled colour conversion of the finished canvas
   (b200_color_convert_scaled_device), so the full-size RGB picture is never written and only the scale_w x scale_h result is
   copied to `out` (pageable: through the decoder's bounce buffer; page-locked: directly).  Interleaved targets, as there.
   B200_E_INVALID (before any CUDA call, message naming the argument) for scale_w or scale_h < 1 or a NULL dec / au / au_size /
   opt / out; everything else as b200_decode_grid_to_rgb_host. */
int b200_decode_grid_to_rgb_scaled_host(b200_decoder* dec, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                        uint64_t max_image_size_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                        const b200_color_options* opt, int scale_w, int scale_h, void* out, size_t out_stride,
                                        b200_image_info* info);

/* Throughput form: returns when the work is queued; the D2H of this picture overlaps the kernels of the next call (two device
   RGB buffers, a second stream).  `out` must be page-locked.  b200_decoder_wait() blocks until everything submitted has
   arrived in host memory and returns the first error.  (The reference has no asynchronous decode; a caller that decodes many
   pictures -- heif-thumbnailer style batch jobs -- is who this is for.) */
int b200_decode_grid_to_rgb_host_async(b200_decoder* dec, int cols, int rows, const uint8_t* const* au, const size_t* au_size,
                                       uint64_t max_image_size_pixels, int canvas_w, int canvas_h, const b200_geometry* geom,
                                       const b200_color_options* opt, void* out, size_t out_stride, b200_image_info* info);
int b200_decoder_wait(b200_decoder* dec);

/* Page-locked host memory: outputs of b200_decode_grid_to_rgb_host / b200_decoder_read_planes placed here are written by
   DMA directly (no bounce copy).  b200_host_register page-locks memory the caller owns (e.g. the planes of a heif_image,
   or a shared-memory mapping several ranks write their row bands into).  Counterpart in the reference: none (its planes
   are plain calloc memory, libheif/image/pixelimage.cc:409-442). */
int b200_host_alloc(size_t bytes, void** out);
void b200_host_free(void* p);
int b200_host_register(void* p, size_t bytes);
int b200_host_unregister(void* p);

#ifdef __cplusplus
}
#endif
#endif
