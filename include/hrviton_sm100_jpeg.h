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

/* ---------------------------------------------------------------------------------------------------------------- encoding
 * What PIL writes for Image.fromarray(rgb).save(f, format='JPEG'): quality 75, 4:2:0 (Y 2x2, Cb / Cr 1x1), libjpeg-turbo's colour
 * conversion, h2v2 downsampling, islow FDCT and quantisation, the standard Huffman tables, no restart interval.  The images of a batch
 * have one size, with height and width multiples of 16 (whole MCUs: no edge padding).  The device writes the entropy-coded data of
 * each image, 0x00-stuffed and followed by EOI; the host prepends the header (SOI .. SOS), which is fixed for a size
 * (hrviton_b200.jpeg.encode_header). */

/* Source layouts of hrv_jpeg_encode. */
enum hrv_jpeg_src { HRV_JPEG_SRC_U8_NHWC = 0, HRV_JPEG_SRC_F32_NCHW = 1 };

/* The tables the device encodes with, built on the host from the ones the header carries. */
typedef struct hrv_jpeg_enc_tables {
  uint16_t quant[2][64];  /* quantisation tables, natural order: luminance, chrominance */
  uint16_t code[4][256];  /* Huffman code of each symbol: DC luminance, AC luminance, DC chrominance, AC chrominance */
  uint8_t size[4][256];   /* its length in bits (0: no code) */
} hrv_jpeg_enc_tables;

/* Device memory hrv_jpeg_encode needs for n images of height x width: the workspace, and `out`.  Both are worst cases computed from
 * the shape.  A block codes to at most 1665 bits: a DC code of up to 16 bits with up to 11 magnitude bits, and for each of the 63 AC
 * coefficients at most one code of up to 16 bits with up to 10 magnitude bits.  A ZRL or an EOB stands in for at least one zero
 * coefficient, which codes nothing itself, so it fits inside that bound.  Per image, out_bytes holds 2 * ceil(blocks * 1665 / 8)
 * + 2 bytes: every byte stuffed, plus EOI.  Blocks = height * width / 256 * 6. */
int hrv_jpeg_encode_bounds(int32_t n, int32_t height, int32_t width, size_t* workspace_bytes, size_t* out_bytes);

/* Encodes n images.  src: uint8 (n, height, width, 3) RGB (HRV_JPEG_SRC_U8_NHWC), or fp32 (n, 3, height, width) in [-1, 1]
 * (HRV_JPEG_SRC_F32_NCHW) converted as the reference's utils.save_images does: (x + 1) * 0.5 * 255 with each operation rounded
 * (no FMA), clamped to [0, 255] by fmaxf / fminf (NaN becomes 0), truncated.  Launches, in order:
 *   colour + FDCT + quantisation   64 threads per MCU: int16 coefficients, zig-zag order, blocks in scan order (Y00 Y01 Y10 Y11 Cb Cr)
 *   length pass                    one thread per block: its bit count, DC predicted from the previous block of its component
 *   scan                           one CTA per image: bit offset of every block
 *   write pass                     one thread per block: its codes at its offset (integer atomicOr on the words it shares)
 *   0xFF count, scan               4096-byte chunks: stuffed length of each image
 *   sizes                          sizes[2 i] = byte length of image i's data after the header (EOI included), sizes[2 i + 1] =
 *                                  its offset in `out`; images are back to back from offset 0
 *   stuffing                       every byte at its stuffed position, 0x00 after each 0xFF, EOI
 * The caller copies `sizes` (int64 [2 n], device) to the host, then the sum of the lengths from `out`. */
int hrv_jpeg_encode(const void* src, int32_t src_kind, int32_t n, int32_t height, int32_t width, const hrv_jpeg_enc_tables* tables,
                    void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, int64_t* sizes, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_JPEG_H_ */
