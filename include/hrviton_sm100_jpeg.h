/* hrviton_sm100_jpeg.h — baseline JPEG decoding entry points of libhrviton_sm100.so (H100 / sm_90a only), bit-identical to PIL's
 * libjpeg-turbo decode (islow IDCT, fancy upsampling, YCbCr -> RGB by the separate upsample-then-convert path).  The host side is
 * hrviton_b200.jpeg: it parses the files, decides which ones the device decodes and fills one hrv_jpeg_image per file.
 *
 * Same conventions as hrviton_sm100.h (device pointers owned by the caller, enqueued on `stream`, 0 or a negative hrv_status, text via
 * hrv_last_error()).  uint8 in and out, integer arithmetic only: ONE flavour of each (no _f16 twin).
 *
 * A batch decodes in three launches, whatever its images' sizes, samplings and component counts:
 *   hrv_jpeg_huffman  entropy-coded bytes -> raw int16 coefficients (natural order), one thread per entropy-coded segment;
 *   hrv_jpeg_idct     coefficients -> uint8 sample planes (libjpeg's jpeg_idct_islow);
 *   hrv_jpeg_color    sample planes -> each image's destination (upsampling, YCbCr -> RGB, cropping).
 */
#ifndef HRVITON_SM100_JPEG_H_
#define HRVITON_SM100_JPEG_H_

#include "hrviton_sm100.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Per-image error codes hrv_jpeg_huffman writes (0: decoded). */
enum hrv_jpeg_error { HRV_JPEG_OK = 0, HRV_JPEG_BAD_CODE = 1, HRV_JPEG_TRUNCATED = 2 };

/* One image of a batch.  Components are in frame order; component 0 is sampled hmax x vmax (1x1, 2x1 or 2x2; 1x1 for a grayscale
 * file), components 1 and 2 are 1x1.  Its coefficient grid is bw[c] x bh[c] blocks (mcus_x * samp by mcus_y * samp, padding blocks
 * included); its sample plane c is (8 bh[c]) x (8 bw[c]) bytes.  Huffman tables: DC of component c at slot 2c, AC at 2c + 1. */
typedef struct hrv_jpeg_image {
  int64_t data;          /* byte offset of its entropy-coded data in the batch's `data` */
  int64_t coef;          /* element offset of its coefficients (component after component) in `coefs` */
  int64_t plane;         /* byte offset of its sample planes in `planes` (each plane starts 16-byte aligned) */
  uint64_t dst;          /* device pointer of the output: (height, width, out_channels) uint8, contiguous */
  int32_t seg0, nseg;    /* its entropy-coded segments: segs[2 (seg0 + s)] = offset from `data`, segs[2 (seg0 + s) + 1] = length */
  int32_t height, width;
  int32_t ncomp;         /* 1 (grayscale) or 3 (YCbCr) */
  int32_t hmax, vmax;
  int32_t mcus_x, mcus_y;
  int32_t restart;       /* MCUs per segment (0: one segment) */
  int32_t out_channels;  /* 3 for YCbCr; 1, or 3 to replicate a grayscale image as convert('RGB') does */
  int32_t bw[3], bh[3];
  uint16_t quant[3][64]; /* quantisation table of each component, natural order */
  uint8_t bits[6][16];   /* BITS: codes of each length 1..16 */
  uint8_t vals[6][256];  /* HUFFVAL */
} hrv_jpeg_image;

/* Entropy decoding: one CTA per image builds its Huffman lookup tables in shared memory; each thread decodes whole segments (the scan,
 * or one restart interval), handling 0xFF00 stuffing and resetting the DC predictors per segment, and writes every coefficient of its
 * blocks (raw, natural order) into `coefs`.  Reads stay inside each segment's byte range.  errors[i] (int32, zeroed by the caller)
 * receives HRV_JPEG_TRUNCATED when a segment ends before its last block and HRV_JPEG_BAD_CODE for a code with no table entry. */
int hrv_jpeg_huffman(const hrv_jpeg_image* images, int32_t n, const uint8_t* data, const int32_t* segs, int16_t* coefs, int32_t* errors,
                     hrv_stream stream);

/* libjpeg's jpeg_idct_islow (jidctint.c) of every block: dequantise in 32 bits, column pass, row pass (CONST_BITS 13, PASS1_BITS 2),
 * descale with rounding, +128, clamp.  max_blocks: the largest bw * bh of any component of the batch. */
int hrv_jpeg_idct(const hrv_jpeg_image* images, int32_t n, const int16_t* coefs, uint8_t* planes, int32_t max_blocks, hrv_stream stream);

/* Upsampling (libjpeg-turbo's fancy h2v1 / h2v2 when the downsampled component is wider than 2 samples, replication otherwise; edges
 * repeat the last real sample), YCbCr -> RGB with libjpeg's 16-bit fixed point, or the Y plane of a grayscale image, cropped to the
 * image and written to each image's dst.  max_pixels: the largest height * width of the batch. */
int hrv_jpeg_color(const hrv_jpeg_image* images, int32_t n, const uint8_t* planes, int32_t max_pixels, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_JPEG_H_ */
