// jpeg_kernels.cu — baseline JPEG decoding on the device (include/hrviton_sm100_jpeg.h, hrviton_b200/jpeg.py), bit-identical to
// libjpeg-turbo's default decode as PIL runs it: Huffman decoding, the islow IDCT of jidctint.c, fancy upsampling (jdsample.c) and
// YCbCr -> RGB (jdcolor.c).  Every stage is integer arithmetic; hrviton_b200.jpeg.decode_np states the same decoder in numpy and the
// tests hold both against PIL.  uint8 in and out, so this translation unit is compiled once.
#include "hrv_host.h"
#include "../../include/hrviton_sm100_jpeg.h"

namespace hrv_jpeg {
using hrv_host::set_error;
static_assert(sizeof(hrv_jpeg_image) == 2120, "hrviton_b200.jpeg.Image mirrors this layout");

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

// natural index of each zig-zag position; 16 entries of 63 past the end, as libjpeg's jpeg_natural_order, so that a corrupt run
// past the last coefficient stays inside the block
__constant__ unsigned char kNatural[80] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63,
    63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63, 63};

// ------------------------------------------------------------------------------------------------ stage 1: entropy decoding
constexpr int kLookBits = 9;  // codes up to 9 bits resolve in one shared-memory lookup; longer ones walk maxcode as libjpeg does
constexpr int kHuffThreads = 64;

struct HuffTable {
  unsigned short look[1 << kLookBits];  // (length << 8) | symbol of the code a 9-bit prefix starts; 0: a longer code or none
  int maxcode[17];                      // largest code of each length, -1 when there is none
  int valoff[17];                       // HUFFVAL index of a code of each length = valoff + code
  unsigned char vals[256];
};

// jpeg_make_d_derived_tbl: canonical codes from BITS (the host has checked that no code overflows its length)
__device__ void build_table(const uint8_t* __restrict__ bits, const uint8_t* __restrict__ vals, HuffTable& t) {
  for (int i = 0; i < (1 << kLookBits); ++i) t.look[i] = 0;
  for (int i = 0; i < 256; ++i) t.vals[i] = vals[i];
  int code = 0, p = 0;
  for (int l = 1; l <= 16; ++l) {
    const int cnt = bits[l - 1];
    t.maxcode[l] = cnt ? code + cnt - 1 : -1;
    t.valoff[l] = p - code;
    for (int k = 0; k < cnt; ++k, ++code, ++p) {
      if (l <= kLookBits) {
        const int first = code << (kLookBits - l), span = 1 << (kLookBits - l);
        for (int j = 0; j < span; ++j) t.look[first + j] = (unsigned short)((l << 8) | vals[p & 255]);
      }
    }
    code <<= 1;
  }
}

// MSB-first bit buffer over one segment.  Reads never pass `end`: past it the buffer is fed zero bytes (as libjpeg does at a marker)
// and `pad` counts those bits, so a decode that consumes any of them (n < pad) has run off the end of its segment.
struct BitReader {
  const uint8_t* p;
  const uint8_t* end;
  unsigned long long buf;
  int n, pad;
  __device__ __forceinline__ void fill() {
    while (n <= 56) {
      unsigned b = 0;
      if (p < end) {
        b = *p++;
        if (b == 0xFF && p < end && *p == 0) ++p;  // a stuffed zero byte
      } else {
        pad += 8;
      }
      buf |= (unsigned long long)b << (56 - n);
      n += 8;
    }
  }
  __device__ __forceinline__ void skip(int k) {
    buf <<= k;
    n -= k;
  }
  // the next k bits (1 <= k <= 16) as the JPEG magnitude category k encodes them (HUFF_EXTEND)
  __device__ __forceinline__ int extend(int k) {
    const int v = (int)(buf >> (64 - k));
    skip(k);
    return v < (1 << (k - 1)) ? v - (1 << k) + 1 : v;
  }
};

// one Huffman symbol, or -1 for a code with no table entry; at least 16 bits must be buffered
__device__ __forceinline__ int decode_symbol(BitReader& br, const HuffTable& t) {
  const unsigned look = (unsigned)(br.buf >> 48);
  const unsigned e = t.look[look >> (16 - kLookBits)];
  if (e) {
    br.skip((int)(e >> 8));
    return (int)(e & 0xFF);
  }
  for (int l = kLookBits + 1; l <= 16; ++l) {
    const int code = (int)(look >> (16 - l));
    if (code <= t.maxcode[l]) {
      br.skip(l);
      return t.vals[(t.valoff[l] + code) & 255];
    }
  }
  return -1;
}

// CTA = one image: its six tables in shared memory, then each thread decodes whole segments
__global__ void __launch_bounds__(kHuffThreads, 1) jpeg_huffman_kernel(const hrv_jpeg_image* __restrict__ images, const uint8_t* __restrict__ data,
                                                                     const int32_t* __restrict__ segs, int16_t* __restrict__ coefs,
                                                                     int32_t* __restrict__ errors) {
  __shared__ HuffTable tables[6];
  const hrv_jpeg_image& im = images[blockIdx.x];
  const int ncomp = im.ncomp;
  if (threadIdx.x < 2 * ncomp) build_table(im.bits[threadIdx.x], im.vals[threadIdx.x], tables[threadIdx.x]);
  __syncthreads();
  const int mcus_x = im.mcus_x, total = im.mcus_x * im.mcus_y;
  const int per = im.restart > 0 ? im.restart : total;
  const long long size0 = (long long)im.bw[0] * im.bh[0] * 64, size1 = (long long)im.bw[1] * im.bh[1] * 64;
  for (int s = threadIdx.x; s < im.nseg; s += blockDim.x) {
    const uint8_t* start = data + im.data + segs[2 * (im.seg0 + s)];
    BitReader br{start, start + segs[2 * (im.seg0 + s) + 1], 0ull, 0, 0};
    int pred0 = 0, pred1 = 0, pred2 = 0;  // DC predictors, in registers (no per-component array in local memory)
    const int m1 = min((s + 1) * per, total);
    int err = HRV_JPEG_OK;
    for (int m = s * per; m < m1 && err == HRV_JPEG_OK; ++m) {
      const int mx = m % mcus_x, my = m / mcus_x;
      for (int c = 0; c < ncomp && err == HRV_JPEG_OK; ++c) {
        const int hs = c == 0 ? im.hmax : 1, vs = c == 0 ? im.vmax : 1;
        const HuffTable& dc = tables[2 * c];
        const HuffTable& ac = tables[2 * c + 1];
        const long long comp_off = im.coef + (c >= 1 ? size0 : 0) + (c >= 2 ? size1 : 0);
        const int bw = c == 0 ? im.bw[0] : c == 1 ? im.bw[1] : im.bw[2];
        int pred = c == 0 ? pred0 : c == 1 ? pred1 : pred2;
        for (int b = 0; b < hs * vs && err == HRV_JPEG_OK; ++b) {
          const int by = my * vs + b / hs, bx = mx * hs + b % hs;
          int16_t* blk = coefs + comp_off + ((long long)by * bw + bx) * 64;
          int4* b4 = reinterpret_cast<int4*>(blk);
#pragma unroll
          for (int i = 0; i < 8; ++i) b4[i] = make_int4(0, 0, 0, 0);
          br.fill();
          int sym = decode_symbol(br, dc);
          if (sym > 16) sym = -1;  // a DC category above 16 has no meaning in an 8-bit file
          if (sym >= 0) {
            pred += sym ? br.extend(sym) : 0;  // symbol + category <= 32 bits; the buffer holds >= 57 after fill()
            blk[0] = (int16_t)pred;
            for (int k = 1; k < 64; ++k) {
              br.fill();
              sym = decode_symbol(br, ac);
              if (sym < 0) break;
              const int r = sym >> 4, sz = sym & 15;
              if (sz) {
                k += r;
                blk[kNatural[k]] = (int16_t)br.extend(sz);
              } else if (r != 15) {
                break;
              } else {
                k += 15;
              }
            }
          }
          if (br.n < br.pad) err = HRV_JPEG_TRUNCATED;  // consumed bits past the segment's end
          else if (sym < 0) err = br.pad > 0 && br.n - br.pad < 16 ? HRV_JPEG_TRUNCATED : HRV_JPEG_BAD_CODE;
        }
        if (c == 0) pred0 = pred;
        else if (c == 1) pred1 = pred;
        else pred2 = pred;
      }
    }
    if (err != HRV_JPEG_OK) atomicMax(errors + blockIdx.x, err);
  }
}

// ------------------------------------------------------------------------------------------------ stage 2: islow IDCT
// jidctint.c: CONST_BITS 13, PASS1_BITS 2, FIX(x) = round(x * 2^13).
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633;
constexpr int F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172;
constexpr int kIdctBlocks = 32;  // DCT blocks per CTA, 8 threads each

// one 1-D pass over x[0..7], descaled by SHIFT with rounding, in jidctint.c's order of operations (32-bit: a valid file's
// dequantised coefficients stay within +-2^14, far from overflow)
template <int SHIFT>
__device__ __forceinline__ void idct_1d(const int (&x)[8], int (&o)[8]) {
  int z2 = x[2], z3 = x[6];
  int z1 = (z2 + z3) * F_0_541;
  const int tmp2 = z1 - z3 * F_1_847;
  const int tmp3 = z1 + z2 * F_0_765;
  const int tmp0 = (x[0] + x[4]) * (1 << kConstBits);
  const int tmp1 = (x[0] - x[4]) * (1 << kConstBits);
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  int o0 = x[7], o1 = x[5], o2 = x[3], o3 = x[1];
  z1 = o0 + o3;
  z2 = o1 + o2;
  z3 = o0 + o2;
  int z4 = o1 + o3;
  const int z5 = (z3 + z4) * F_1_175;
  o0 *= F_0_298;
  o1 *= F_2_053;
  o2 *= F_3_072;
  o3 *= F_1_501;
  z1 *= -F_0_899;
  z2 *= -F_2_562;
  z3 = z3 * -F_1_961 + z5;
  z4 = z4 * -F_0_390 + z5;
  o0 += z1 + z3;
  o1 += z2 + z4;
  o2 += z2 + z3;
  o3 += z1 + z4;
  constexpr int r = 1 << (SHIFT - 1);
  o[0] = (t10 + o3 + r) >> SHIFT;
  o[7] = (t10 - o3 + r) >> SHIFT;
  o[1] = (t11 + o2 + r) >> SHIFT;
  o[6] = (t11 - o2 + r) >> SHIFT;
  o[2] = (t12 + o1 + r) >> SHIFT;
  o[5] = (t12 - o1 + r) >> SHIFT;
  o[3] = (t13 + o0 + r) >> SHIFT;
  o[4] = (t13 - o0 + r) >> SHIFT;
}

// grid (blocks / 32, images * 3): thread = one column, then one row, of one DCT block of component blockIdx.y % 3
__global__ void __launch_bounds__(kIdctBlocks * 8) jpeg_idct_kernel(const hrv_jpeg_image* __restrict__ images, const int16_t* __restrict__ coefs,
                                                                     uint8_t* __restrict__ planes) {
  __shared__ int ws[kIdctBlocks][64];
  const hrv_jpeg_image& im = images[blockIdx.y / 3];
  const int c = blockIdx.y % 3;
  if (c >= im.ncomp) return;  // uniform over the CTA
  const int lb = threadIdx.x >> 3, lane = threadIdx.x & 7;
  const int bw = im.bw[c], nblk = bw * im.bh[c];
  const int b = blockIdx.x * kIdctBlocks + lb;
  const bool live = b < nblk;
  long long coef_off = im.coef, plane_off = im.plane;
  for (int k = 0; k < c; ++k) {
    coef_off += (long long)im.bw[k] * im.bh[k] * 64;
    plane_off += ((long long)im.bw[k] * im.bh[k] * 64 + 15) / 16 * 16;
  }
  if (live) {  // column `lane`: dequantise in 32 bits (coef x q can overflow int16), then pass 1
    const int16_t* blk = coefs + coef_off + (long long)b * 64;
    int x[8], o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = (int)__ldg(blk + k * 8 + lane) * (int)im.quant[c][k * 8 + lane];
    idct_1d<kConstBits - kPass1Bits>(x, o);
#pragma unroll
    for (int k = 0; k < 8; ++k) ws[lb][k * 8 + lane] = o[k];
  }
  __syncthreads();
  if (!live) return;
  int x[8], o[8];  // row `lane`
#pragma unroll
  for (int k = 0; k < 8; ++k) x[k] = ws[lb][lane * 8 + k];
  idct_1d<kConstBits + kPass1Bits + 3>(x, o);
  // range limit: clamp.  libjpeg-turbo's SIMD IDCTs saturate; its C IDCT masks an index into a table, which differs only for values a
  // valid file does not produce.
  unsigned lo = 0, hi = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    lo |= (unsigned)min(max(o[k] + 128, 0), 255) << (8 * k);
    hi |= (unsigned)min(max(o[k + 4] + 128, 0), 255) << (8 * k);
  }
  const int by = b / bw, bx = b - by * bw;
  uint8_t* row = planes + plane_off + ((long long)by * 8 + lane) * (bw * 8) + bx * 8;
  *reinterpret_cast<uint2*>(row) = make_uint2(lo, hi);
}

// ------------------------------------------------------------------------------------------------ stage 3: upsample and colour
// Sample (x, y) of a chroma plane upsampled by (fx, fy) to full size: libjpeg-turbo's h2v1 / h2v2 fancy upsampling when the
// downsampled component is wider than 2 samples (jdsample.c's jinit_upsampler), plain replication otherwise.  The neighbour of an
// edge sample is the sample itself: the last real sample, never the encoder's padding.
__device__ __forceinline__ int upsample(const uint8_t* __restrict__ p, int pitch, int cw, int ch, int fx, int fy, int x, int y) {
  if (fx == 1) return __ldg(p + (long long)y * pitch + x);
  const int cx = x >> 1, cy = fy == 2 ? y >> 1 : y;
  if (cw <= 2) return __ldg(p + (long long)cy * pitch + cx);
  const int odd = x & 1;
  const int fxn = odd ? min(cx + 1, cw - 1) : max(cx - 1, 0);
  if (fy == 1) {  // h2v1: (3 near + far + 1) >> 2 for an even output, + 2 for an odd one
    const uint8_t* r = p + (long long)cy * pitch;
    return (3 * __ldg(r + cx) + __ldg(r + fxn) + 1 + odd) >> 2;
  }
  // h2v2: column sums 3 near + far over the rows, then (3 a + b + 8) >> 4 for an even output, + 7 for an odd one
  const int fyn = (y & 1) ? min(cy + 1, ch - 1) : max(cy - 1, 0);
  const uint8_t* r0 = p + (long long)cy * pitch;
  const uint8_t* r1 = p + (long long)fyn * pitch;
  const int a = 3 * __ldg(r0 + cx) + __ldg(r1 + cx);
  const int bb = 3 * __ldg(r0 + fxn) + __ldg(r1 + fxn);
  return (3 * a + bb + 8 - odd) >> 4;
}

__device__ __forceinline__ uint8_t clamp8(int v) { return (uint8_t)min(max(v, 0), 255); }

// jdcolor.c's ycc_rgb_convert: SCALEBITS 16, FIX(x) = round(x * 2^16)
constexpr int kCrR = 91881, kCbG = 22554, kCrG = 46802, kCbB = 116130, kHalf = 1 << 15;

// grid (pixels / 256, images): thread = one output pixel
__global__ void __launch_bounds__(256) jpeg_color_kernel(const hrv_jpeg_image* __restrict__ images, const uint8_t* __restrict__ planes) {
  const hrv_jpeg_image& im = images[blockIdx.y];
  const int w = im.width, h = im.height;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)w * h) return;
  const int y = (int)(i / w), x = (int)(i - (long long)y * w);
  uint8_t* dst = reinterpret_cast<uint8_t*>(im.dst);
  const uint8_t* py = planes + im.plane;
  const int yv = __ldg(py + (long long)y * (im.bw[0] * 8) + x);
  if (im.ncomp == 1) {
    if (im.out_channels == 3) {
      dst[i * 3] = dst[i * 3 + 1] = dst[i * 3 + 2] = (uint8_t)yv;
    } else {
      dst[i] = (uint8_t)yv;
    }
    return;
  }
  const long long size0 = ((long long)im.bw[0] * im.bh[0] * 64 + 15) / 16 * 16;
  const long long size1 = ((long long)im.bw[1] * im.bh[1] * 64 + 15) / 16 * 16;
  const int cw = (w + im.hmax - 1) / im.hmax, ch = (h + im.vmax - 1) / im.vmax;
  const int cb = upsample(py + size0, im.bw[1] * 8, cw, ch, im.hmax, im.vmax, x, y) - 128;
  const int cr = upsample(py + size0 + size1, im.bw[2] * 8, cw, ch, im.hmax, im.vmax, x, y) - 128;
  dst[i * 3] = clamp8(yv + ((kCrR * cr + kHalf) >> 16));
  dst[i * 3 + 1] = clamp8(yv + ((-kCbG * cb + kHalf - kCrG * cr) >> 16));
  dst[i * 3 + 2] = clamp8(yv + ((kCbB * cb + kHalf) >> 16));
}

}  // namespace hrv_jpeg

using namespace hrv_jpeg;

extern "C" int hrv_jpeg_huffman(const hrv_jpeg_image* images, int32_t n, const uint8_t* data, const int32_t* segs, int16_t* coefs,
                                int32_t* errors, hrv_stream stream) {
  if (!images || !data || !segs || !coefs || !errors || n < 1) return set_error(HRV_EINVAL, "jpeg_huffman: bad arguments");
  jpeg_huffman_kernel<<<n, kHuffThreads, 0, (cudaStream_t)stream>>>(images, data, segs, coefs, errors);
  return launched("jpeg_huffman");
}

extern "C" int hrv_jpeg_idct(const hrv_jpeg_image* images, int32_t n, const int16_t* coefs, uint8_t* planes, int32_t max_blocks,
                             hrv_stream stream) {
  if (!images || !coefs || !planes || n < 1 || n > 65535 / 3 || max_blocks < 1) return set_error(HRV_EINVAL, "jpeg_idct: bad arguments");
  const dim3 grid((unsigned)((max_blocks + kIdctBlocks - 1) / kIdctBlocks), (unsigned)(3 * n));
  jpeg_idct_kernel<<<grid, kIdctBlocks * 8, 0, (cudaStream_t)stream>>>(images, coefs, planes);
  return launched("jpeg_idct");
}

extern "C" int hrv_jpeg_color(const hrv_jpeg_image* images, int32_t n, const uint8_t* planes, int32_t max_pixels, hrv_stream stream) {
  if (!images || !planes || n < 1 || n > 65535 || max_pixels < 1) return set_error(HRV_EINVAL, "jpeg_color: bad arguments");
  const dim3 grid((unsigned)((max_pixels + 255) / 256), (unsigned)n);
  jpeg_color_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(images, planes);
  return launched("jpeg_color");
}
