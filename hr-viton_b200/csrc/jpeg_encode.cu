// jpeg_encode.cu — baseline JPEG encoding on the device (include/hrviton_sm100_jpeg.h, hrviton_b200/jpeg.py), byte-identical to
// what PIL writes for Image.fromarray(rgb).save(f, format='JPEG'): libjpeg-turbo's rgb_ycc_convert (jccolor.c), h2v2_downsample
// (jcsample.c), jpeg_fdct_islow (jfdctint.c), quantize() with compute_reciprocal's divisors (jcdctmgr.c, 16-bit DCTELEM) and
// encode_one_block (jchuff.c) with the standard tables.  Integer arithmetic only; hrviton_b200.jpeg.encode_np states the same encoder
// in numpy and the tests hold both against PIL.  uint8 / fp32 in, bytes out: compiled once.
#include "hrv_host.h"
#include "../../include/hrviton_sm100_jpeg.h"

namespace hrv_jpeg_enc {
using hrv_host::set_error;
static_assert(sizeof(hrv_jpeg_enc_tables) == 3328, "hrviton_b200.jpeg.EncTables mirrors this layout");

constexpr int kMaxBlockBits = 1665;  // (16 + 11) DC + 63 x (16 + 10) AC: see hrv_jpeg_encode_bounds
constexpr int kChunkBytes = 4096;    // stuffing: 256 threads x 16 bytes
constexpr int kMcuPerCta = 4;        // colour / FDCT: 64 threads per MCU

__constant__ unsigned char kNaturalOf[64] = {
    0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,  7,  14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

struct Geometry {
  long long blocks;      // 8x8 blocks per image (6 per MCU)
  long long word_cap;    // 32-bit words of entropy-coded bits per image, a whole number of stuffing chunks
  long long chunk_cap;   // stuffing chunks per image
  long long out_cap;     // worst-case file bytes after the header per image: every byte stuffed, plus EOI
};

Geometry geometry(int height, int width) {
  Geometry g;
  g.blocks = (long long)(height / 16) * (width / 16) * 6;
  const long long bytes = (g.blocks * kMaxBlockBits + 7) / 8;
  g.chunk_cap = (bytes + kChunkBytes - 1) / kChunkBytes;
  g.word_cap = g.chunk_cap * (kChunkBytes / 4);
  g.out_cap = 2 * bytes + 2;
  return g;
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

// ------------------------------------------------------------------------------------------------ stage 1: colour, FDCT, quantise
// jccolor.c: SCALEBITS 16, FIX(x) = round(x * 2^16); Cb / Cr round with ONE_HALF - 1 so that 255 stays in range
constexpr int kYR = 19595, kYG = 38470, kYB = 7471, kCbR = 11059, kCbG = 21709, kHalfFix = 32768, kCrG = 27439, kCrB = 5329;
constexpr int kOneHalf = 1 << 15, kCbCrOffset = 128 << 16;
// jfdctint.c: CONST_BITS 13, PASS1_BITS 2
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int F_0_298 = 2446, F_0_390 = 3196, F_0_541 = 4433, F_0_765 = 6270, F_0_899 = 7373, F_1_175 = 9633;
constexpr int F_1_501 = 12299, F_1_847 = 15137, F_1_961 = 16069, F_2_053 = 16819, F_2_562 = 20995, F_3_072 = 25172;

template <int N>
__device__ __forceinline__ int descale(int v) { return (v + (1 << (N - 1))) >> N; }

// one pass of jpeg_fdct_islow over x[0..7]: the rows pass (LAST false) or the columns pass, in jfdctint.c's order of operations
template <bool LAST>
__device__ __forceinline__ void fdct_1d(int (&x)[8]) {
  constexpr int S = LAST ? kConstBits + kPass1Bits : kConstBits - kPass1Bits;
  const int t0 = x[0] + x[7], t7 = x[0] - x[7], t1 = x[1] + x[6], t6 = x[1] - x[6];
  const int t2 = x[2] + x[5], t5 = x[2] - x[5], t3 = x[3] + x[4], t4 = x[3] - x[4];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  x[0] = LAST ? descale<kPass1Bits>(t10 + t11) : (t10 + t11) * (1 << kPass1Bits);
  x[4] = LAST ? descale<kPass1Bits>(t10 - t11) : (t10 - t11) * (1 << kPass1Bits);
  int z1 = (t12 + t13) * F_0_541;
  x[2] = descale<S>(z1 + t13 * F_0_765);
  x[6] = descale<S>(z1 - t12 * F_1_847);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7;
  const int z5 = (z3 + z4) * F_1_175;
  z1 *= -F_0_899;
  z2 *= -F_2_562;
  z3 = z3 * -F_1_961 + z5;
  z4 = z4 * -F_0_390 + z5;
  x[7] = descale<S>(t4 * F_0_298 + z1 + z3);
  x[5] = descale<S>(t5 * F_2_053 + z2 + z4);
  x[3] = descale<S>(t6 * F_3_072 + z2 + z3);
  x[1] = descale<S>(t7 * F_1_501 + z1 + z4);
}

// utils.save_images: (x + 1) * 0.5 * 255 rounded at each step (no FMA contraction), clamp to [0, 255] (NaN -> 0), truncate
__device__ __forceinline__ int save_images_u8(float x) {
  const float v = __fmul_rn(__fmul_rn(__fadd_rn(x, 1.0f), 0.5f), 255.0f);
  return (int)fminf(fmaxf(v, 0.0f), 255.0f);
}

// grid (ceil(MCUs / 4), images), 256 threads: 64 threads per MCU convert its 16x16 pixels, downsample the chroma, transform and
// quantise its six blocks, and write them in scan order (Y00 Y01 Y10 Y11 Cb Cr), coefficients in zig-zag order
template <bool F32>
__global__ void __launch_bounds__(64 * kMcuPerCta) jpeg_enc_coefs_kernel(const void* __restrict__ src, int height, int width,
                                                                          const hrv_jpeg_enc_tables* __restrict__ tables,
                                                                          int16_t* __restrict__ coefs) {
  __shared__ int ws[kMcuPerCta][6][64];
  __shared__ int cbf[kMcuPerCta][256], crf[kMcuPerCta][256];  // full-resolution chroma of each MCU
  __shared__ unsigned recip[2][64], corr[2][64], shift[2][64];
  const int g = threadIdx.x >> 6, t = threadIdx.x & 63;
  if (threadIdx.x < 128) {  // jcdctmgr.c compute_reciprocal over qtbl << 3, DCTELEM 16 bits (libjpeg-turbo with SIMD)
    const int tb = threadIdx.x >> 6, i = threadIdx.x & 63;
    const unsigned div = (unsigned)tables->quant[tb][i] << 3;
    const int b = 31 - __clz(div);
    int r = 16 + b;
    unsigned fq = (1u << r) / div, c = div / 2;
    const unsigned fr = (1u << r) % div;
    if (fr == 0) {  // a power of two
      fq >>= 1;
      --r;
    } else if (fr <= div / 2) {
      ++c;
    } else {
      ++fq;
    }
    recip[tb][i] = fq;
    corr[tb][i] = c;
    shift[tb][i] = (unsigned)r;
  }
  const int mcus_x = width >> 4, mcus = mcus_x * (height >> 4);
  const int m = blockIdx.x * kMcuPerCta + g, img = blockIdx.y;
  const bool live = m < mcus;
  const int my = live ? m / mcus_x : 0, mx = live ? m - my * mcus_x : 0;
  if (live) {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int p = t + 64 * k, py = p >> 4, px = p & 15;
      const long long y = my * 16 + py, x = mx * 16 + px;
      int r, gg, b;
      if (F32) {
        const long long plane = (long long)height * width;
        const float* s = static_cast<const float*>(src) + (long long)img * 3 * plane + y * width + x;
        r = save_images_u8(__ldg(s));
        gg = save_images_u8(__ldg(s + plane));
        b = save_images_u8(__ldg(s + 2 * plane));
      } else {
        const uint8_t* s = static_cast<const uint8_t*>(src) + (((long long)img * height + y) * width + x) * 3;
        r = __ldg(s);
        gg = __ldg(s + 1);
        b = __ldg(s + 2);
      }
      ws[g][(py >> 3) * 2 + (px >> 3)][(py & 7) * 8 + (px & 7)] = (kYR * r + kYG * gg + kYB * b + kOneHalf) >> 16;
      cbf[g][p] = (-kCbR * r - kCbG * gg + kHalfFix * b + kCbCrOffset + kOneHalf - 1) >> 16;
      crf[g][p] = (kHalfFix * r - kCrG * gg - kCrB * b + kCbCrOffset + kOneHalf - 1) >> 16;
    }
  }
  __syncthreads();
  if (live) {  // h2v2_downsample: bias 1, 2, 1, 2 ... along each output row (the MCU's first output column is even)
    const int oy = t >> 3, ox = t & 7, i0 = (2 * oy) * 16 + 2 * ox, bias = 1 + (ox & 1);
    ws[g][4][t] = (cbf[g][i0] + cbf[g][i0 + 1] + cbf[g][i0 + 16] + cbf[g][i0 + 17] + bias) >> 2;
    ws[g][5][t] = (crf[g][i0] + crf[g][i0 + 1] + crf[g][i0 + 16] + crf[g][i0 + 17] + bias) >> 2;
  }
  __syncthreads();
  const int blk = t >> 3, lane = t & 7;
  if (live && t < 48) {  // rows: block t / 8, row t % 8, samples centred on 0
    int x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = ws[g][blk][lane * 8 + k] - 128;
    fdct_1d<false>(x);
#pragma unroll
    for (int k = 0; k < 8; ++k) ws[g][blk][lane * 8 + k] = x[k];
  }
  __syncthreads();
  if (live && t < 48) {  // columns
    int x[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) x[k] = ws[g][blk][k * 8 + lane];
    fdct_1d<true>(x);
#pragma unroll
    for (int k = 0; k < 8; ++k) ws[g][blk][k * 8 + lane] = x[k];
  }
  __syncthreads();
  if (!live) return;
  int16_t* out = coefs + ((long long)img * mcus + m) * 6 * 64;
#pragma unroll
  for (int k = 0; k < 6; ++k) {  // quantize(): ((|x| + corr) * recip) >> shift, sign restored
    const int idx = t + 64 * k, b = idx >> 6, zz = idx & 63, tb = b < 4 ? 0 : 1, nat = kNaturalOf[zz];
    const int v = ws[g][b][nat];
    const unsigned a = (unsigned)(v < 0 ? -v : v);
    const int q = (int)(((a + corr[tb][nat]) * recip[tb][nat]) >> shift[tb][nat]);
    out[idx] = (int16_t)(v < 0 ? -q : q);
  }
}

// ------------------------------------------------------------------------------------------------ stage 2: Huffman coding
struct CodeTables {
  unsigned short code[4][256];  // DC0, AC0, DC1, AC1
  unsigned char size[4][256];
};

__device__ void load_codes(const hrv_jpeg_enc_tables* __restrict__ tables, CodeTables& s) {
  for (int i = threadIdx.x; i < 4 * 256; i += blockDim.x) {
    s.code[i >> 8][i & 255] = tables->code[i >> 8][i & 255];
    s.size[i >> 8][i & 255] = tables->size[i >> 8][i & 255];
  }
}

__device__ __forceinline__ int category(int a) { return a ? 32 - __clz(a) : 0; }

struct BitCounter {
  int n = 0;
  __device__ __forceinline__ void put(unsigned, int len) { n += len; }
};

// MSB-first bits into zeroed 32-bit words from bit `pos` on.  A completed word is stored, except the first when it began in the
// previous block's bits; that one and the last, partial word are OR-ed in, as the neighbouring blocks share them.
struct BitWriter {
  uint32_t* w;
  long long word, first;
  bool first_shared;
  unsigned long long acc;
  int n;
  __device__ BitWriter(uint32_t* words, long long pos) : w(words), word(pos >> 5), first(pos >> 5), first_shared((pos & 31) != 0), acc(0), n((int)(pos & 31)) {}
  __device__ __forceinline__ void put(unsigned code, int len) {  // 1 <= len <= 16
    acc |= (unsigned long long)code << (64 - n - len);
    n += len;
    if (n >= 32) {
      const unsigned v = (unsigned)(acc >> 32);
      if (word == first && first_shared) atomicOr(w + word, v);
      else w[word] = v;
      ++word;
      acc <<= 32;
      n -= 32;
    }
  }
  __device__ __forceinline__ void flush() {
    if (n > 0) atomicOr(w + word, (unsigned)(acc >> 32));
  }
};

// scan-order block j of an image: its component (0 Y, 1 Cb, 2 Cr) and the block whose DC predicts it (-1: the predictor is 0)
__device__ __forceinline__ void block_links(long long j, int& comp, long long& prev) {
  const long long mcu = j / 6;
  const int sub = (int)(j - mcu * 6);
  comp = sub < 4 ? 0 : sub - 3;
  if (sub >= 1 && sub <= 3) prev = j - 1;
  else if (mcu == 0) prev = -1;
  else prev = sub == 0 ? j - 3 : j - 6;
}

// jchuff.c encode_one_block: DC difference category and bits, AC runs (ZRL for runs past 15), EOB when zeros trail
template <class Sink>
__device__ __forceinline__ void encode_block(const int16_t* __restrict__ blk, int pred, int comp, const CodeTables& t, Sink& s) {
  const int dct = comp ? 2 : 0, act = dct + 1;
  const int4* b4 = reinterpret_cast<const int4*>(blk);
  int r = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const int4 q4 = __ldg(b4 + w);
    const int words[4] = {q4.x, q4.y, q4.z, q4.w};
#pragma unroll
    for (int h = 0; h < 8; ++h) {
      const int v = (int)(short)((h & 1) ? (words[h >> 1] >> 16) : (words[h >> 1] & 0xFFFF));
      if (w == 0 && h == 0) {
        const int diff = v - pred, nb = category(diff < 0 ? -diff : diff);
        s.put(t.code[dct][nb], t.size[dct][nb]);
        if (nb) s.put((unsigned)(diff < 0 ? diff - 1 : diff) & ((1u << nb) - 1), nb);
        continue;
      }
      if (v == 0) {
        ++r;
        continue;
      }
      while (r > 15) {
        s.put(t.code[act][0xF0], t.size[act][0xF0]);
        r -= 16;
      }
      const int nb = category(v < 0 ? -v : v), sym = (r << 4) + nb;
      s.put(t.code[act][sym], t.size[act][sym]);
      s.put((unsigned)(v < 0 ? v - 1 : v) & ((1u << nb) - 1), nb);
      r = 0;
    }
  }
  if (r > 0) s.put(t.code[act][0], t.size[act][0]);
}

// length pass: thread = one block of the batch
__global__ void __launch_bounds__(256) jpeg_enc_bits_kernel(const int16_t* __restrict__ coefs, long long blocks, int n,
                                                            const hrv_jpeg_enc_tables* __restrict__ tables, int32_t* __restrict__ bits) {
  __shared__ CodeTables t;
  load_codes(tables, t);
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= blocks * n) return;
  const long long img = i / blocks, j = i - img * blocks;
  int comp;
  long long prev;
  block_links(j, comp, prev);
  const int16_t* base = coefs + img * blocks * 64;
  const int pred = prev < 0 ? 0 : base[prev * 64];
  BitCounter c;
  encode_block(base + j * 64, pred, comp, t, c);
  bits[i] = c.n;
}

// block-wide exclusive scan (blockDim.x a multiple of 32): this thread's prefix, and the block's total in *total
__device__ long long block_exclusive_scan(long long v, long long* total) {
  __shared__ long long warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    long long s = lane < nw ? warp_sums[lane] : 0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  const long long before = warp ? warp_sums[warp - 1] : 0;
  *total = warp_sums[nw - 1];
  __syncthreads();
  return before + x - v;
}

// CTA = one image: exclusive scan of its blocks' bit counts into bit offsets; totals[img] = the image's bits
__global__ void __launch_bounds__(1024) jpeg_enc_scan_kernel(const int32_t* __restrict__ bits, long long blocks, long long* __restrict__ offsets,
                                                             long long* __restrict__ totals) {
  const long long base = (long long)blockIdx.x * blocks;
  long long carry = 0;
  for (long long j0 = 0; j0 < blocks; j0 += blockDim.x) {
    const long long j = j0 + threadIdx.x;
    const long long v = j < blocks ? bits[base + j] : 0;
    long long sum;
    const long long p = block_exclusive_scan(v, &sum);
    if (j < blocks) offsets[base + j] = carry + p;
    carry += sum;
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// write pass: thread = one block, its codes at its offset; the image's last block pads the last byte with 1-bits
__global__ void __launch_bounds__(256) jpeg_enc_write_kernel(const int16_t* __restrict__ coefs, long long blocks, int n, long long word_cap,
                                                             const hrv_jpeg_enc_tables* __restrict__ tables, const long long* __restrict__ offsets,
                                                             const long long* __restrict__ totals, uint32_t* __restrict__ words) {
  __shared__ CodeTables t;
  load_codes(tables, t);
  __syncthreads();
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= blocks * n) return;
  const long long img = i / blocks, j = i - img * blocks;
  int comp;
  long long prev;
  block_links(j, comp, prev);
  const int16_t* base = coefs + img * blocks * 64;
  const int pred = prev < 0 ? 0 : base[prev * 64];
  BitWriter bw(words + img * word_cap, offsets[i]);
  encode_block(base + j * 64, pred, comp, t, bw);
  if (j == blocks - 1) {
    const int pad = (int)((8 - (totals[img] & 7)) & 7);
    if (pad) bw.put((1u << pad) - 1, pad);
  }
  bw.flush();
}

// ------------------------------------------------------------------------------------------------ stage 3: byte stuffing
// byte k (0..15) of four words of MSB-first bits: k is a compile-time constant wherever this is unrolled
__device__ __forceinline__ unsigned byte_of(const uint4& q, int k) {
  const unsigned word = (k >> 2) == 0 ? q.x : (k >> 2) == 1 ? q.y : (k >> 2) == 2 ? q.z : q.w;
  return (word >> (24 - 8 * (k & 3))) & 0xFF;
}

// grid (chunks, images): the 0xFF bytes of each 4096-byte chunk of the image's ceil(bits / 8) bytes
__global__ void __launch_bounds__(256) jpeg_enc_ffcount_kernel(const uint32_t* __restrict__ words, long long word_cap,
                                                               const long long* __restrict__ totals, long long chunk_cap, int32_t* __restrict__ chunk_ff) {
  const long long img = blockIdx.y, nbytes = (totals[img] + 7) >> 3;
  for (long long c = blockIdx.x; c * kChunkBytes < nbytes; c += gridDim.x) {
    const long long b0 = c * kChunkBytes + threadIdx.x * 16;
    int cnt = 0;
    if (b0 < nbytes) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(words + img * word_cap) + (b0 >> 4));
#pragma unroll
      for (int k = 0; k < 16; ++k) cnt += (b0 + k < nbytes && byte_of(q, k) == 0xFF) ? 1 : 0;
    }
    long long total;
    block_exclusive_scan(cnt, &total);
    if (threadIdx.x == 0) chunk_ff[img * chunk_cap + c] = (int32_t)total;
  }
}

// CTA = one image: chunk_ff becomes the 0xFF count before each chunk; lengths[img] = bytes + stuffed zeros + EOI
__global__ void __launch_bounds__(1024) jpeg_enc_ffscan_kernel(int32_t* __restrict__ chunk_ff, long long chunk_cap, const long long* __restrict__ totals,
                                                              long long* __restrict__ lengths) {
  const long long img = blockIdx.x, nbytes = (totals[img] + 7) >> 3, chunks = (nbytes + kChunkBytes - 1) / kChunkBytes;
  long long carry = 0;
  for (long long c0 = 0; c0 < chunks; c0 += blockDim.x) {
    const long long c = c0 + threadIdx.x;
    const long long v = c < chunks ? chunk_ff[img * chunk_cap + c] : 0;
    long long sum;
    const long long p = block_exclusive_scan(v, &sum);
    if (c < chunks) chunk_ff[img * chunk_cap + c] = (int32_t)(carry + p);
    carry += sum;
  }
  if (threadIdx.x == 0) lengths[img] = nbytes + carry + 2;
}

// one thread: sizes[2 i] = length of image i's data after the header, sizes[2 i + 1] = its offset in `out` (images back to back)
__global__ void jpeg_enc_sizes_kernel(const long long* __restrict__ lengths, int n, int64_t* __restrict__ sizes) {
  long long off = 0;
  for (int i = 0; i < n; ++i) {
    sizes[2 * i] = lengths[i];
    sizes[2 * i + 1] = off;
    off += lengths[i];
  }
}

// grid (chunks, images): every byte at its stuffed position, 0x00 after each 0xFF, and EOI at the end
__global__ void __launch_bounds__(256) jpeg_enc_stuff_kernel(const uint32_t* __restrict__ words, long long word_cap, const long long* __restrict__ totals,
                                                             const int32_t* __restrict__ chunk_ff, long long chunk_cap, const int64_t* __restrict__ sizes,
                                                             uint8_t* __restrict__ out) {
  const long long img = blockIdx.y, nbytes = (totals[img] + 7) >> 3;
  uint8_t* dst = out + sizes[2 * img + 1];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const long long len = sizes[2 * img];
    dst[len - 2] = 0xFF;
    dst[len - 1] = 0xD9;
  }
  for (long long c = blockIdx.x; c * kChunkBytes < nbytes; c += gridDim.x) {
    const long long b0 = c * kChunkBytes + threadIdx.x * 16;
    uint4 q = make_uint4(0, 0, 0, 0);
    int cnt = 0;
    if (b0 < nbytes) {
      q = __ldg(reinterpret_cast<const uint4*>(words + img * word_cap) + (b0 >> 4));
#pragma unroll
      for (int k = 0; k < 16; ++k) cnt += (b0 + k < nbytes && byte_of(q, k) == 0xFF) ? 1 : 0;
    }
    long long total;
    long long pos = b0 + chunk_ff[img * chunk_cap + c] + block_exclusive_scan(cnt, &total);
    if (b0 < nbytes) {
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        if (b0 + k < nbytes) {
          const unsigned v = byte_of(q, k);
          dst[pos++] = (uint8_t)v;
          if (v == 0xFF) dst[pos++] = 0;
        }
      }
    }
  }
}

constexpr int kChunkGrid = 64;  // CTAs per image of the chunk kernels (grid-stride over the chunks)

}  // namespace hrv_jpeg_enc

using namespace hrv_jpeg_enc;

namespace {
struct Workspace {
  int16_t* coefs;
  int32_t* bits;
  long long* offsets;
  long long* totals;
  long long* lengths;
  uint32_t* words;
  int32_t* chunk_ff;
  size_t bytes;
};

Workspace carve(void* base, int n, const Geometry& g) {
  Workspace w;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    char* p = static_cast<char*>(base) + o;
    o += align256(bytes);
    return p;
  };
  w.coefs = reinterpret_cast<int16_t*>(take((size_t)n * g.blocks * 64 * sizeof(int16_t)));
  w.bits = reinterpret_cast<int32_t*>(take((size_t)n * g.blocks * sizeof(int32_t)));
  w.offsets = reinterpret_cast<long long*>(take((size_t)n * g.blocks * sizeof(long long)));
  w.totals = reinterpret_cast<long long*>(take((size_t)n * sizeof(long long)));
  w.lengths = reinterpret_cast<long long*>(take((size_t)n * sizeof(long long)));
  w.words = reinterpret_cast<uint32_t*>(take((size_t)n * g.word_cap * sizeof(uint32_t)));
  w.chunk_ff = reinterpret_cast<int32_t*>(take((size_t)n * g.chunk_cap * sizeof(int32_t)));
  w.bytes = o;
  return w;
}

bool bad_shape(int32_t n, int32_t height, int32_t width) {
  return n < 1 || n > 65535 || height < 16 || width < 16 || height % 16 || width % 16 || height > 65535 || width > 65535;
}
}  // namespace

extern "C" int hrv_jpeg_encode_bounds(int32_t n, int32_t height, int32_t width, size_t* workspace_bytes, size_t* out_bytes) {
  if (bad_shape(n, height, width) || !workspace_bytes || !out_bytes)
    return set_error(HRV_EINVAL, "jpeg_encode_bounds: need 1 <= n <= 65535 and a height and width that are multiples of 16");
  const Geometry g = geometry(height, width);
  *workspace_bytes = carve(nullptr, n, g).bytes;
  *out_bytes = (size_t)n * g.out_cap;
  return HRV_OK;
}

extern "C" int hrv_jpeg_encode(const void* src, int32_t src_kind, int32_t n, int32_t height, int32_t width, const hrv_jpeg_enc_tables* tables,
                               void* workspace, size_t workspace_bytes, uint8_t* out, size_t out_bytes, int64_t* sizes, hrv_stream stream) {
  if (!src || !tables || !workspace || !out || !sizes || bad_shape(n, height, width) ||
      (src_kind != HRV_JPEG_SRC_U8_NHWC && src_kind != HRV_JPEG_SRC_F32_NCHW))
    return set_error(HRV_EINVAL, "jpeg_encode: bad arguments");
  const Geometry g = geometry(height, width);
  const Workspace w = carve(workspace, n, g);
  if (workspace_bytes < w.bytes || out_bytes < (size_t)n * g.out_cap)
    return set_error(HRV_EINVAL, "jpeg_encode: workspace %zu / out %zu bytes, need %zu / %zu (hrv_jpeg_encode_bounds)", workspace_bytes, out_bytes,
                     w.bytes, (size_t)n * g.out_cap);
  cudaStream_t st = (cudaStream_t)stream;
  const long long mcus = g.blocks / 6, nblocks = g.blocks * n;
  const dim3 cgrid((unsigned)((mcus + kMcuPerCta - 1) / kMcuPerCta), (unsigned)n);
  if (src_kind == HRV_JPEG_SRC_F32_NCHW)
    jpeg_enc_coefs_kernel<true><<<cgrid, 64 * kMcuPerCta, 0, st>>>(src, height, width, tables, w.coefs);
  else
    jpeg_enc_coefs_kernel<false><<<cgrid, 64 * kMcuPerCta, 0, st>>>(src, height, width, tables, w.coefs);
  const unsigned bgrid = (unsigned)((nblocks + 255) / 256);
  jpeg_enc_bits_kernel<<<bgrid, 256, 0, st>>>(w.coefs, g.blocks, n, tables, w.bits);
  jpeg_enc_scan_kernel<<<n, 1024, 0, st>>>(w.bits, g.blocks, w.offsets, w.totals);
  if (cudaMemsetAsync(w.words, 0, (size_t)n * g.word_cap * sizeof(uint32_t), st) != cudaSuccess) return launched("jpeg_encode (memset)");
  jpeg_enc_write_kernel<<<bgrid, 256, 0, st>>>(w.coefs, g.blocks, n, g.word_cap, tables, w.offsets, w.totals, w.words);
  const dim3 sgrid((unsigned)(g.chunk_cap < kChunkGrid ? g.chunk_cap : kChunkGrid), (unsigned)n);
  jpeg_enc_ffcount_kernel<<<sgrid, 256, 0, st>>>(w.words, g.word_cap, w.totals, g.chunk_cap, w.chunk_ff);
  jpeg_enc_ffscan_kernel<<<n, 1024, 0, st>>>(w.chunk_ff, g.chunk_cap, w.totals, w.lengths);
  jpeg_enc_sizes_kernel<<<1, 1, 0, st>>>(w.lengths, n, sizes);
  jpeg_enc_stuff_kernel<<<sgrid, 256, 0, st>>>(w.words, g.word_cap, w.totals, w.chunk_ff, g.chunk_cap, sizes, out);
  return launched("jpeg_encode");
}
