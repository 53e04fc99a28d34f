/* hrviton_sm100_png.h — PNG encoding and the stage-1 multi-task grid of libhrviton_sm100.so (H100 / sm_90a only).  The host side is
 * hrviton_b200.png: it writes the signature, IHDR and IEND around the IDAT chunks the device makes, and hrviton_b200.png.encode_np
 * states the same encoder in numpy.
 *
 * Same conventions as hrviton_sm100.h (device pointers owned by the caller, enqueued on `stream`, 0 or a negative hrv_status, text via
 * hrv_last_error()).  uint8 / fp32 in, uint8 out: ONE flavour of each (no _f16 twin).
 */
#ifndef HRVITON_SM100_PNG_H_
#define HRVITON_SM100_PNG_H_

#include "hrviton_sm100.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------------------------------------------------------- encoding
 * 8-bit RGB (colour type 2), no interlace.  Every scanline is Paeth-filtered (filter type 4); the filtered stream of each image is
 * cut into HRV_PNG_CHUNK_BYTES-byte chunks (the last one shorter) and each chunk is compressed by one CTA, into one IDAT chunk:
 *   RLE matching: each maximal run of equal bytes of the chunk is one literal, then matches of distance 1 and length min(258, rest)
 *     while at least 3 bytes are left, then the 1 or 2 bytes left as literals;
 *   one dynamic Huffman block (code lengths limited to 15 bits, 7 for the code-length code, by halving the frequencies until the
 *     code fits; one distance code of length 1), or one stored block when that is not larger;
 *   a chunk that is not the last ends its Huffman block with an empty stored block (byte alignment); only the last sets BFINAL;
 *   the zlib header (78 01) opens the first IDAT, the Adler-32 of the filtered stream closes the last.
 * Every IDAT carries its own CRC-32.  No atomic operation decides where a byte goes: a chunk's bytes are placed by its size, in a
 * bounded slot first and then, after a scan of the sizes, at their place in `out`. */
#define HRV_PNG_CHUNK_BYTES 65535

/* Device memory hrv_png_encode needs for n images of height x width: the workspace, and `out`.  Both are worst cases computed from
 * the shape: per chunk, a stored block and its framing. */
int hrv_png_encode_bounds(int32_t n, int32_t height, int32_t width, size_t* workspace_bytes, size_t* out_bytes);

/* Encodes n uint8 (n, height, width, 3) RGB images (contiguous).  Launches, in order:
 *   compress   one CTA per chunk: filter, RLE tokens, Huffman code, the IDAT chunk (length, type, data, CRC) into its slot
 *   layout     one CTA per image: the offset of each of its IDAT chunks, the Adler-32 (combined from per-chunk partial sums) and the
 *              last chunk's CRC
 *   sizes      sizes[2 i] = byte length of image i's IDAT chunks, sizes[2 i + 1] = their offset in `out`; images back to back
 *   copy       one CTA per chunk: its slot to its place in `out`
 * The caller copies `sizes` (int64 [2 n], device) to the host, then the sum of the lengths from `out`, and writes the signature and
 * IHDR before and IEND after each image's IDAT chunks. */
int hrv_png_encode(const uint8_t* src, int32_t n, int32_t height, int32_t width, void* workspace, size_t workspace_bytes, uint8_t* out,
                   size_t out_bytes, int64_t* sizes, hrv_stream stream);

/* ---------------------------------------------------------------------------------------------------------------- the grid
 * The reference's test_condition.py:135-143 for a batch: make_grid of 12 panels (nrow 4, padding 2, pad value 0) and save_image's
 * uint8 conversion (x * 255 + 0.5, clamped to [0, 255], truncated), as out: uint8 (n, 3 (height + 2) + 2, 4 (width + 2) + 2, 3).
 * Panels, in order: cloth / 2 + 0.5, cloth_mask > 0.5, segmap(parse_agnostic), (densepose + 1) / 2, parse_cloth / 2 + 0.5, pcm,
 * warped_cloth / 2 + 0.5, warped_cm > 0.5, segmap(parse), segmap(seg'), image / 2 + 0.5, max(0, (argmax seg' == 3) - (warped_cm >
 * 0.5)).  seg' is seg with channel 3 multiplied by warped_cm (HRV_GRID_WARP_GRAD) or by warped_cm > 0.5 (HRV_GRID_DETACH), or seg
 * (HRV_GRID_NO_COMPOSITION).  segmap(x): the first-index arg-max over the channels, utils.visualize_segmap's 20-entry palette
 * (black past it), / 255.  fp32 operations in the reference's order, each rounded (no FMA contraction).
 * Every tensor is fp32 NCHW contiguous with n x height x width pixels: cloth, densepose, parse_cloth, warped_cloth, image 3 channels;
 * cloth_mask, pcm, warped_cm 1; parse_agnostic, parse, seg `classes`. */
enum hrv_grid_composition { HRV_GRID_NO_COMPOSITION = 0, HRV_GRID_DETACH = 1, HRV_GRID_WARP_GRAD = 2 };

typedef struct hrv_condition_panels {
  const float* cloth;
  const float* cloth_mask;
  const float* parse_agnostic;
  const float* densepose;
  const float* parse_cloth;
  const float* pcm;
  const float* warped_cloth;
  const float* warped_cm;
  const float* parse;
  const float* seg;
  const float* image;
} hrv_condition_panels;

int hrv_condition_grid(const hrv_condition_panels* panels, int32_t n, int32_t height, int32_t width, int32_t classes, int32_t composition,
                       uint8_t* out, hrv_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* HRVITON_SM100_PNG_H_ */
