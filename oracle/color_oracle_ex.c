/*
 * oracle/color_oracle_ex.c -- TEST INFRASTRUCTURE ONLY. C restatement of the encoder-side colour stage for every RGB layout
 * heif_context_encode_image accepts: the chain convert_colorspace picks from an RGB input to YCbCr at the input depth, and the
 * reference ops of that chain restated loop for loop, in their float order (built with -ffp-contract=off, like the reference's
 * x86-64 build without FMA):
 *   Op_RGB24_32_to_YCbCr          rgb2yuv.cc:506-808   (co_rgb_to_ycbcr of color_oracle.c)
 *   Op_RRGGBBxx_HDR_to_YCbCr420   rgb2yuv.cc:311-503
 *   Op_RGB_to_YCbCr<T>            rgb2yuv.cc:30-305    (after Op_RRGGBBaa_swap_endianness / Op_RRGGBBaa_BE_to_RGB_HDR /
 *                                                        Op_RGB24_32_to_RGB, rgb2rgb.cc: lossless, restated as sample reads)
 *   Op_RGB24_32_to_YCbCr444_GBR   rgb2yuv.cc:812-919
 * It needs no reference source; tests pin it against the reference's own convert_colorspace (oracle/ref_encode.cc).
 */
#include "color_oracle.c"     /* one copy of the restated nclx coefficients (co_kr_kb), clip_f_u16 and co_rgb_to_ycbcr */

typedef struct { int planar, bps, nch, le; const uint8_t* p[4]; size_t stride[4]; } co_rgb_in;

static int co_px(const co_rgb_in* in, int c, int x, int y) {
  if (in->planar) {
    const uint8_t* row = in->p[c] + (size_t)y * in->stride[c];
    return in->bps == 2 ? ((const uint16_t*)row)[x] : row[x];
  }
  const uint8_t* q = in->p[0] + (size_t)y * in->stride[0] + (size_t)x * in->nch * in->bps + (size_t)c * in->bps;
  return in->bps == 1 ? q[0] : ((q[in->le] << 8) | q[1 - in->le]);      /* rgb2yuv.cc:443-445 */
}

static void co_rgb_coeffs(int mc, int cp, float c[3][3]) {                 /* nclx.cc:176-200 */
  float Kr, Kb; co_kr_kb(mc, cp, &Kr, &Kb);
  if (Kb != 0 || Kr != 0) {
    c[0][0] = Kr; c[0][1] = 1 - Kr - Kb; c[0][2] = Kb;
    c[1][0] = -Kr / (1 - Kb) / 2; c[1][1] = -(1 - Kr - Kb) / (1 - Kb) / 2; c[1][2] = 0.5f;
    c[2][0] = 0.5f; c[2][1] = -(1 - Kr - Kb) / (1 - Kr) / 2; c[2][2] = -Kb / (1 - Kr) / 2;
  } else {
    c[0][0] = 0.299f; c[0][1] = 0.587f; c[0][2] = 0.114f; c[1][0] = -0.168735f; c[1][1] = -0.331264f; c[1][2] = 0.5f;
    c[2][0] = 0.5f; c[2][1] = -0.418688f; c[2][2] = -0.081312f;
  }
}

static void co_put(void* plane, int bps, size_t idx, int v) { if (bps == 2) ((uint16_t*)plane)[idx] = (uint16_t)v; else ((uint8_t*)plane)[idx] = (uint8_t)v; }

/* in_chroma: 10..15 interleaved (planes[0], rows packed, > 8 bit in the layout's byte order) or 3 = planar R, G, B[, A]
   (native uint16 above 8 bit).  Output planes packed.  *pipeline: the B200_YCC_PIPE_* bits of the chain.
   Returns 0; -2 where convert_colorspace has no chain, or one with an operation restated nowhere here (matrix 11 / 14,
   only_use_preferred with average / sharp-YUV downsampling to 4:2:0 / 4:2:2). */
int co_rgb_to_ycbcr_ex(int in_chroma, int bpp, int has_alpha, int w, int h, const void* const* planes, int out_chroma, int cp, int mc, int full,
                       int downsampling, int only_preferred, void* oy, void* ocb, void* ocr, void* oa, int* pipeline) {
  co_rgb_in in = {0};
  in.planar = in_chroma == 3; in.bps = bpp > 8 ? 2 : 1;
  in.nch = in.planar ? 1 : ((in_chroma == 11 || in_chroma == 13 || in_chroma == 15) ? 4 : 3);
  in.le = in_chroma == 14 || in_chroma == 15;
  for (int c = 0; c < (in.planar ? 3 + has_alpha : 1); c++) { in.p[c] = (const uint8_t*)planes[c]; in.stride[c] = (size_t)w * (in.planar ? 1 : in.nch) * in.bps; }
  if (!in.planar) has_alpha = in.nch == 4;
  if (mc == 2) mc = 6;                                   /* target nclx "unspecified" -> the input's sRGB defaults (colorconversion.cc:567-573) */
  if (cp == 2) cp = 1;
  /* the planner's choice, from the ops' state_after_conversion (rgb2yuv.cc:30-98, :311-363, :506-553, :812-847) */
  const int sub = out_chroma != 3, special = mc == 0 || mc == 8, inter8 = in_chroma == 10 || in_chroma == 11;
  if (mc == 11 || mc == 14) return -2;
  if (sub && only_preferred && downsampling != 1) return -2;
  int pipe;
  if (inter8) pipe = !special ? 1 : (mc == 0 && full && out_chroma == 3) ? 2 : 16 | 8;
  else if (!in.planar) pipe = (full && out_chroma == 1 && !special) ? 4 : (in.le ? 32 : 0) | 16 | 8;
  else pipe = 8;
  *pipeline = pipe;
  if (pipe == 1) return co_rgb_to_ycbcr((const uint8_t*)planes[0], in.stride[0], w, h, has_alpha, out_chroma, mc, cp, full, oy, ocb, ocr, oa);

  const int subH = out_chroma == 3 ? 1 : 2, subV = out_chroma == 1 ? 2 : 1, cw = (w + subH - 1) / subH;
  const int halfRange = 1 << (bpp - 1), fullRange = (1 << bpp) - 1, bps = in.bps;
  const float limited_range_offset = (float)(16 << (bpp - 8));
  float c[3][3]; co_rgb_coeffs(mc, cp, c);
  if (pipe == 2) {                                                                    /* rgb2yuv.cc:900-916 */
    for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
      const size_t i = (size_t)y * w + x;
      co_put(oy, 1, i, co_px(&in, 1, x, y)); co_put(ocb, 1, i, co_px(&in, 2, x, y)); co_put(ocr, 1, i, co_px(&in, 0, x, y));
      if (oa) co_put(oa, 1, i, has_alpha ? co_px(&in, 3, x, y) : 0xff);
    }
    return 0;
  }
  if (pipe == 4) {                                                                    /* rgb2yuv.cc:438-500, full range */
    for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
      const float r = (float)co_px(&in, 0, x, y), g = (float)co_px(&in, 1, x, y), b = (float)co_px(&in, 2, x, y);
      const float v = r * c[0][0] + g * c[0][1] + b * c[0][2];
      co_put(oy, 2, (size_t)y * w + x, clip_f_u16(v, fullRange));
      if (oa) co_put(oa, 2, (size_t)y * w + x, co_px(&in, 3, x, y));
    }
    for (int y = 0; y < h; y += 2) for (int x = 0; x < w; x += 2) {
      const int x2 = x + 1 < w ? x + 1 : x, y2 = y + 1 < h ? y + 1 : y;             /* dx / dy = 0 on the last column / row */
      float r = (float)co_px(&in, 0, x, y), g = (float)co_px(&in, 1, x, y), b = (float)co_px(&in, 2, x, y);
      r += (float)co_px(&in, 0, x2, y); g += (float)co_px(&in, 1, x2, y); b += (float)co_px(&in, 2, x2, y);
      r += (float)co_px(&in, 0, x, y2); g += (float)co_px(&in, 1, x, y2); b += (float)co_px(&in, 2, x, y2);
      r += (float)co_px(&in, 0, x2, y2); g += (float)co_px(&in, 1, x2, y2); b += (float)co_px(&in, 2, x2, y2);
      r *= 0.25f; g *= 0.25f; b *= 0.25f;
      const float cb = r * c[1][0] + g * c[1][1] + b * c[1][2], cr = r * c[2][0] + g * c[2][1] + b * c[2][2];
      co_put(ocb, 2, (size_t)(y / 2) * cw + x / 2, clip_f_u16(halfRange + cb, fullRange));
      co_put(ocr, 2, (size_t)(y / 2) * cw + x / 2, clip_f_u16(halfRange + cr, fullRange));
    }
    return 0;
  }
  /* Op_RGB_to_YCbCr<T>, rgb2yuv.cc:196-302 */
  for (int y = 0; y < h; y++) for (int x = 0; x < w; x++) {
    const int R = co_px(&in, 0, x, y), G = co_px(&in, 1, x, y), B = co_px(&in, 2, x, y);
    int out;
    if (mc == 0) out = full ? G : clip_f_u16(((G * 219.0f) / 256) + limited_range_offset, fullRange);
    else if (mc == 8) out = G / 2 + (R + B) / 4;
    else {
      float v = (float)R * c[0][0] + (float)G * c[0][1] + (float)B * c[0][2];
      if (!full) v = (((v * 219) / 256) + limited_range_offset);
      out = clip_f_u16(v, fullRange);
    }
    co_put(oy, bps, (size_t)y * w + x, out);
    if (oa) co_put(oa, bps, (size_t)y * w + x, co_px(&in, 3, x, y));
  }
  for (int y = 0; y < h; y += subV) for (int x = 0; x < w; x += subH) {
    const size_t ci = (size_t)(y / subV) * cw + x / subH;
    const int R = co_px(&in, 0, x, y), G = co_px(&in, 1, x, y), B = co_px(&in, 2, x, y);
    int ocbv, ocrv;
    if (mc == 0) {
      if (full) { ocbv = B; ocrv = R; }
      else { ocbv = clip_f_u16(((B * 224.0f) / 256) + limited_range_offset, fullRange); ocrv = clip_f_u16(((R * 224.0f) / 256) + limited_range_offset, fullRange); }
    } else if (mc == 8) {
      const int u = G / 2 - (R + B) / 4 + halfRange, v = (R - B) / 2 + halfRange;
      ocbv = u < 0 ? 0 : (u > fullRange ? fullRange : u); ocrv = v < 0 ? 0 : (v > fullRange ? fullRange : v);
    } else {
      float r = (float)R, g = (float)G, b = (float)B;
      if (subH > 1 || subV > 1) {
        const int x2 = (x + 1 < w && subH == 2 && subV == 2) ? x + 1 : x, y2 = (y + 1 < h && subV == 2) ? y + 1 : y;
        r += (float)co_px(&in, 0, x2, y); g += (float)co_px(&in, 1, x2, y); b += (float)co_px(&in, 2, x2, y);
        r += (float)co_px(&in, 0, x, y2); g += (float)co_px(&in, 1, x, y2); b += (float)co_px(&in, 2, x, y2);
        r += (float)co_px(&in, 0, x2, y2); g += (float)co_px(&in, 1, x2, y2); b += (float)co_px(&in, 2, x2, y2);
        r *= 0.25f; g *= 0.25f; b *= 0.25f;
      }
      float cb = r * c[1][0] + g * c[1][1] + b * c[1][2], cr = r * c[2][0] + g * c[2][1] + b * c[2][2];
      if (!full) { cb = (cb * 224) / 256; cr = (cr * 224) / 256; }
      ocbv = clip_f_u16(cb + halfRange, fullRange); ocrv = clip_f_u16(cr + halfRange, fullRange);
    }
    co_put(ocb, bps, ci, ocbv); co_put(ocr, bps, ci, ocrv);
  }
  return 0;
}
