// png_encode.cu — PNG encoding on the device (include/hrviton_sm100_png.h, hrviton_b200/png.py) and the stage-1 multi-task grid
// kernel.  Integer arithmetic in the encoder; hrviton_b200.png.encode_np states the same encoder in numpy and the tests hold the
// device's bytes to it.  uint8 / fp32 in, uint8 out: compiled once.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "hrv_host.h"
#include "../../include/hrviton_sm100_png.h"

namespace hrv_png {
using hrv_host::set_error;

constexpr int kChunk = HRV_PNG_CHUNK_BYTES;
constexpr int kThreads = 1024;
constexpr int kLayoutThreads = 256;
constexpr int kSeg = (kChunk + kThreads - 1) / kThreads;  // filtered bytes per thread in the token passes
// one IDAT chunk: length, type, zlib header (first chunk), at most a stored block (5 + kChunk bytes), Adler-32 (last chunk), CRC
constexpr int kSlotCap = (8 + 2 + 5 + kChunk + 4 + 4 + 7) / 8 * 8;
constexpr int kStageWords = kSlotCap / 4;
constexpr int kBufBytes = (kChunk + 15) / 16 * 16;
constexpr size_t kSmem = kBufBytes + (size_t)kStageWords * 4;
constexpr unsigned kAdlerMod = 65521;
constexpr int kLitSyms = 286, kClSyms = 19;

__constant__ unsigned short kLenBase[29] = {3,  4,  5,  6,  7,  8,  9,  10, 11,  13,  15,  17,  19,  23, 27,
                                            31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned char kClOrder[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
// x^(2^k) modulo the CRC-32 polynomial (reflected): the shift of a CRC over 2^k zero bits (zlib's x2n_table)
__constant__ unsigned kX2n[32] = {0x40000000, 0x20000000, 0x08000000, 0x00800000, 0x00008000, 0xedb88320, 0xb1e6b092, 0xa06a2517,
                                  0xed627dae, 0x88d14467, 0xd7bbfe6a, 0xec447f11, 0x8e7ea170, 0x6427800e, 0x4d47bae0, 0x09fe548f,
                                  0x83852d0f, 0x30362f1a, 0x7b5a9cc3, 0x31fec169, 0x9fec022a, 0x6c8dedc4, 0x15d6874d, 0x5fde7a4e,
                                  0xbad90e37, 0x2e4e5eef, 0x4eaba214, 0xa8a472c0, 0x429a969e, 0x148d302a, 0xc40ba6d0, 0xc4e22c3c};

int launched(const char* what) {
  cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? HRV_OK : set_error(HRV_ECUDA, "%s: %s", what, cudaGetErrorString(e));
}

// ------------------------------------------------------------------------------------------------ CRC-32
__device__ unsigned multmodp(unsigned a, unsigned b) {  // a * b modulo the polynomial (zlib's multmodp)
  unsigned m = 1u << 31, p = 0;
  for (;;) {
    if (a & m) {
      p ^= b;
      if ((a & (m - 1)) == 0) break;
    }
    m >>= 1;
    b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
  }
  return p;
}

// the CRC of a message followed by n zero bytes, given the CRC of the message: crc(A B) = shift(crc(A), |B|) ^ crc(B)
__device__ unsigned crc_shift(unsigned crc, long long n) {
  unsigned p = 1u << 31;
  for (int k = 3; n; n >>= 1, ++k)
    if (n & 1) p = multmodp(kX2n[k & 31], p);
  return multmodp(p, crc);
}

__device__ unsigned crc_bytes(const unsigned* table, const uint8_t* d, int len) {
  unsigned c = 0xffffffffu;
  for (int i = 0; i < len; ++i) c = table[(c ^ d[i]) & 0xff] ^ (c >> 8);
  return c ^ 0xffffffffu;
}

// ------------------------------------------------------------------------------------------------ Huffman code lengths
struct HuffScratch {
  unsigned f[kLitSyms];         // working frequencies
  unsigned nf[2 * kLitSyms];    // node frequencies: leaves in (freq, symbol) order, then internal nodes in creation order
  short order[kLitSyms];        // leaf q -> symbol
  short parent[2 * kLitSyms];
  unsigned char depth[2 * kLitSyms];
  int m, done;
};

// png.huffman_lengths: a Huffman code for freq[0..nsym) (0: no code) of at most `limit` bits; every nonzero frequency f becomes
// (f + 1) >> 1 until it fits.  The whole CTA calls it; one thread merges.
__device__ void huffman_lengths(const unsigned* freq, int nsym, int limit, unsigned char* len, HuffScratch& w) {
  const int tid = threadIdx.x;
  if (tid < nsym) {
    w.f[tid] = freq[tid];
    len[tid] = 0;
  }
  if (tid == 0) w.done = 0;
  __syncthreads();
  while (!w.done) {
    const bool used = tid < nsym && w.f[tid] > 0;
    const int m = __syncthreads_count(used);
    if (used) {  // rank in (freq, symbol) order
      const unsigned fv = w.f[tid];
      int rank = 0;
      for (int s = 0; s < nsym; ++s) {
        const unsigned g = w.f[s];
        rank += g > 0 && (g < fv || (g == fv && s < tid));
      }
      w.order[rank] = (short)tid;
      w.nf[rank] = fv;
    }
    __syncthreads();
    if (tid == 0) {
      if (m == 1) {
        const int s = w.order[0];
        len[s] = 1;
        len[s == 0 ? 1 : 0] = 1;
        w.done = 1;
      } else {
        int i = 0, j = m;
        for (int t = m; t < 2 * m - 1; ++t) {
          int pick[2];
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            if (i < m && (j >= t || w.nf[i] <= w.nf[j])) pick[k] = i++;
            else pick[k] = j++;
          }
          w.nf[t] = w.nf[pick[0]] + w.nf[pick[1]];
          w.parent[pick[0]] = w.parent[pick[1]] = (short)t;
        }
        w.depth[2 * m - 2] = 0;
        int mx = 0;
        for (int t = 2 * m - 3; t >= 0; --t) {
          w.depth[t] = w.depth[w.parent[t]] + 1;
          if (t < m && w.depth[t] > mx) mx = w.depth[t];
        }
        w.done = mx <= limit;
        w.m = m;
      }
    }
    __syncthreads();
    if (w.done) {
      if (tid < w.m && m > 1) len[w.order[tid]] = w.depth[tid];
    } else if (tid < nsym && w.f[tid] > 0) {
      w.f[tid] = (w.f[tid] + 1) >> 1;
    }
    __syncthreads();
  }
}

// canonical codes of len[0..nsym), bit-reversed for LSB-first output (one thread; count and next: 16 ints of shared scratch each)
__device__ void canonical_codes(const unsigned char* len, int nsym, unsigned short* code, int* count, int* next) {
  for (int b = 0; b < 16; ++b) count[b] = 0;
  for (int s = 0; s < nsym; ++s) count[len[s]]++;
  count[0] = 0;
  int c = 0;
  for (int b = 1; b < 16; ++b) {
    c = (c + count[b - 1]) << 1;
    next[b] = c;
  }
  for (int s = 0; s < nsym; ++s) {
    const int n = len[s];
    code[s] = n ? (unsigned short)(__brev((unsigned)next[n]++) >> (32 - n)) : 0;
  }
}

// ------------------------------------------------------------------------------------------------ the compress kernel
struct Smem {
  unsigned hist[kLitSyms];
  unsigned cl_hist[kClSyms];
  unsigned char lit_len[kLitSyms], cl_len[kClSyms];
  unsigned short lit_code[kLitSyms], cl_code[kClSyms];
  unsigned short len_sym[259];
  unsigned crc_table[256];
  unsigned char item_sym[kLitSyms + 1], item_extra[kLitSyms + 1];
  int seg_first[kThreads], seg_next[kThreads];
  HuffScratch huff;
  int cc_count[16], cc_next[16];
  int nlit, ncl, hdr_bits, use_dyn, deflate_bytes, slot_len;
  union {
    cub::BlockScan<int, kThreads>::TempStorage scan;
    cub::BlockReduce<unsigned long long, kThreads>::TempStorage reduce;
    cub::BlockReduce<unsigned, kThreads>::TempStorage reduce32;
  } cub;
};

// value (up to 25 bits) at bit `pos` of the zeroed LSB-first stage
__device__ __forceinline__ void put_bits(unsigned* stage, long long pos, unsigned v, int len) {
  const int w = (int)(pos >> 5), sh = (int)(pos & 31);
  atomicOr(stage + w, v << sh);
  if (sh + len > 32) atomicOr(stage + w + 1, v >> (32 - sh));
}

// walks the RLE tokens of filtered positions [a, b) of the chunk buf[0..n): run_start is the start of the run holding a, next_start
// the first run start at or after b (n when none).  emit(position, match length or 0 for a literal).
template <class F>
__device__ __forceinline__ void walk_tokens(const uint8_t* buf, int a, int b, int run_start, int next_start, F&& emit) {
  int i = a, s = (a == 0 || buf[a] != buf[a - 1]) ? a : run_start;
  while (i < b) {
    const uint8_t v = buf[i];
    int j = i + 1;
    while (j < b && buf[j] == v) ++j;
    const int r = (j < b ? j : next_start) - s;
    for (int p = i; p < j; ++p) {
      const int k = p - s;
      if (k == 0) {
        emit(p, 0);
        continue;
      }
      const int base = k - (k - 1) % 258, mlen = min(258, r - base);
      if (mlen < 3) emit(p, 0);
      else if (k == base) emit(p, mlen);
    }
    i = j;
    s = j;
  }
}

__device__ __forceinline__ uint8_t paeth_byte(const uint8_t* __restrict__ img, long long p, long long rowbytes, int width) {
  const long long row = p / rowbytes;
  const int col = (int)(p - row * rowbytes);
  if (col == 0) return 4;
  const int x = col - 1;
  const uint8_t* r = img + row * (long long)width * 3;
  const int a = x >= 3 ? r[x - 3] : 0;
  const int b = row ? r[x - (long long)width * 3] : 0;
  const int c = (row && x >= 3) ? r[x - 3 - (long long)width * 3] : 0;
  const int q = a + b - c, pa = abs(q - a), pb = abs(q - b), pc = abs(q - c);
  const int pred = (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
  return (uint8_t)(r[x] - pred);
}

// grid (chunks of all images), kThreads threads, kSmem bytes of dynamic shared memory (the filtered chunk, then the stage the IDAT
// chunk is assembled in)
__global__ void __launch_bounds__(kThreads, 1) png_compress_kernel(const uint8_t* __restrict__ src, int height, int width, long long total,
                                                                   int cpi, uint8_t* __restrict__ slots, int32_t* __restrict__ slot_len,
                                                                   unsigned* __restrict__ crc_part, unsigned* __restrict__ adler) {
  extern __shared__ __align__(16) uint8_t dyn[];
  __shared__ Smem sm;
  uint8_t* buf = dyn;
  unsigned* stage = reinterpret_cast<unsigned*>(dyn + kBufBytes);
  uint8_t* stage8 = reinterpret_cast<uint8_t*>(stage);
  const int tid = threadIdx.x;
  const long long g = blockIdx.x;
  const int img = (int)(g / cpi), c = (int)(g - (long long)img * cpi);
  const long long o = (long long)c * kChunk, rowbytes = 3LL * width + 1;
  const int n = (int)min((long long)kChunk, total - o);
  const bool first = c == 0, last = c == cpi - 1;
  const int base = first ? 10 : 8;  // the deflate bytes' offset in the IDAT chunk

  for (int i = tid; i < kLitSyms; i += kThreads) sm.hist[i] = 0;
  if (tid < kClSyms) sm.cl_hist[tid] = 0;
  for (int l = tid; l < 259; l += kThreads) {
    int k = 0;
    while (k < 28 && kLenBase[k + 1] <= l) ++k;
    sm.len_sym[l] = (unsigned short)k;
  }
  if (tid < 256) {
    unsigned v = tid;
    for (int k = 0; k < 8; ++k) v = v & 1 ? 0xedb88320u ^ (v >> 1) : v >> 1;
    sm.crc_table[tid] = v;
  }
  for (int i = tid; i < kStageWords; i += kThreads) stage[i] = 0;

  // the filtered bytes, and the chunk's Adler-32 partial sums: sum f_i and sum (n - i) f_i
  const uint8_t* im = src + (long long)img * height * width * 3;
  unsigned long long s1 = 0, s2 = 0;
  for (int i = tid; i < n; i += kThreads) {
    const uint8_t f = paeth_byte(im, o + i, rowbytes, width);
    buf[i] = f;
    s1 += f;
    s2 += (unsigned long long)(n - i) * f;
  }
  s1 = cub::BlockReduce<unsigned long long, kThreads>(sm.cub.reduce).Sum(s1);
  __syncthreads();
  s2 = cub::BlockReduce<unsigned long long, kThreads>(sm.cub.reduce).Sum(s2);
  if (tid == 0) {
    adler[2 * g] = (unsigned)(s1 % kAdlerMod);
    adler[2 * g + 1] = (unsigned)(s2 % kAdlerMod);
  }
  __syncthreads();

  // each thread's segment: the run start holding its first byte (a max-scan of the last run start of the segments before) and the
  // first run start after it (a min over the segments after)
  const int a = min(tid * kSeg, n), b = min(a + kSeg, n);
  int last_start = -1, first_start = n;
  for (int i = a; i < b; ++i)
    if (i == 0 || buf[i] != buf[i - 1]) {
      if (first_start == n) first_start = i;
      last_start = i;
    }
  int run_start;
  cub::BlockScan<int, kThreads>(sm.cub.scan).ExclusiveScan(last_start, run_start, -1, cub::Max());
  sm.seg_first[kThreads - 1 - tid] = first_start;
  __syncthreads();
  int after;  // min of first_start over the segments after this one's mirror
  cub::BlockScan<int, kThreads>(sm.cub.scan).ExclusiveScan(sm.seg_first[tid], after, n, cub::Min());
  sm.seg_next[kThreads - 1 - tid] = after;
  __syncthreads();
  const int next_start = sm.seg_next[tid];

  walk_tokens(buf, a, b, run_start, next_start, [&](int p, int len) { atomicAdd(&sm.hist[len ? 257 + sm.len_sym[len] : buf[p]], 1u); });
  __syncthreads();
  if (tid == 0) sm.hist[256] = 1;
  __syncthreads();
  huffman_lengths(sm.hist, kLitSyms, 15, sm.lit_len, sm.huff);
  if (tid == 0) {  // the code-length items of the literal/length lengths and the one distance length (1)
    int nlit = kLitSyms;
    while (sm.lit_len[nlit - 1] == 0) --nlit;
    nlit = max(nlit, 257);
    int items = 0, i = 0;
    const int total_len = nlit + 1;
    auto L = [&](int k) { return k < nlit ? (int)sm.lit_len[k] : 1; };
    auto add = [&](int s, int x) {
      sm.item_sym[items] = (unsigned char)s;
      sm.item_extra[items++] = (unsigned char)x;
      sm.cl_hist[s]++;
    };
    while (i < total_len) {
      const int v = L(i);
      int r = 1;
      while (i + r < total_len && L(i + r) == v) ++r;
      i += r;
      if (v == 0) {
        while (r >= 11) {
          const int m = min(r, 138);
          add(18, m - 11);
          r -= m;
        }
        if (r >= 3) {
          add(17, r - 3);
          r = 0;
        }
      } else {
        add(v, 0);
        --r;
        while (r >= 3) {
          const int m = min(r, 6);
          add(16, m - 3);
          r -= m;
        }
      }
      for (; r > 0; --r) add(v, 0);
    }
    sm.nlit = nlit;
    sm.ncl = items;  // the item count, until the code-length code is known
  }
  __syncthreads();
  huffman_lengths(sm.cl_hist, kClSyms, 7, sm.cl_len, sm.huff);
  if (tid == 0) {
    const int items = sm.ncl;
    int ncl = kClSyms;
    while (ncl > 4 && sm.cl_len[kClOrder[ncl - 1]] == 0) --ncl;
    canonical_codes(sm.lit_len, kLitSyms, sm.lit_code, sm.cc_count, sm.cc_next);
    canonical_codes(sm.cl_len, kClSyms, sm.cl_code, sm.cc_count, sm.cc_next);
    long long hdr = 17 + 3 * ncl;
    for (int k = 0; k < items; ++k) {
      const int s = sm.item_sym[k];
      hdr += sm.cl_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0);
    }
    long long bits = hdr;
    for (int s = 0; s < kLitSyms; ++s) bits += (long long)sm.hist[s] * (sm.lit_len[s] + (s >= 257 ? kLenExtra[s - 257] + 1 : 0));
    const long long dyn_bytes = last ? (bits + 7) / 8 : (bits + 3 + 7) / 8 + 4;
    const int stored_bytes = n + 5;
    const int use_dyn = dyn_bytes < stored_bytes;
    sm.use_dyn = use_dyn;
    sm.deflate_bytes = use_dyn ? (int)dyn_bytes : stored_bytes;
    sm.hdr_bits = (int)hdr;
    if (use_dyn) {  // the block header
      long long pos = base * 8LL;
      auto put = [&](unsigned v, int len) {
        put_bits(stage, pos, v, len);
        pos += len;
      };
      put(last ? 1 : 0, 1);
      put(2, 2);
      put(sm.nlit - 257, 5);
      put(0, 5);
      put(ncl - 4, 4);
      for (int q = 0; q < ncl; ++q) put(sm.cl_len[kClOrder[q]], 3);
      for (int k = 0; k < items; ++k) {
        const int s = sm.item_sym[k];
        put(sm.cl_code[s] | ((unsigned)sm.item_extra[k] << sm.cl_len[s]), sm.cl_len[s] + (s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0));
      }
    }
    const int data_len = (first ? 2 : 0) + sm.deflate_bytes + (last ? 4 : 0);
    sm.slot_len = data_len + 12;
    stage8[0] = (uint8_t)(data_len >> 24);
    stage8[1] = (uint8_t)(data_len >> 16);
    stage8[2] = (uint8_t)(data_len >> 8);
    stage8[3] = (uint8_t)data_len;
    stage8[4] = 'I';
    stage8[5] = 'D';
    stage8[6] = 'A';
    stage8[7] = 'T';
    if (first) {
      stage8[8] = 0x78;
      stage8[9] = 0x01;
    }
  }
  __syncthreads();
  if (sm.use_dyn) {
    auto token_bits = [&](int p, int len) {
      if (!len) return (int)sm.lit_len[buf[p]];
      const int k = sm.len_sym[len];
      return (int)sm.lit_len[257 + k] + kLenExtra[k] + 1;
    };
    int mine = 0;
    walk_tokens(buf, a, b, run_start, next_start, [&](int p, int len) { mine += token_bits(p, len); });
    int before, sum;
    cub::BlockScan<int, kThreads>(sm.cub.scan).ExclusiveSum(mine, before, sum);
    long long pos = base * 8LL + sm.hdr_bits + before;
    walk_tokens(buf, a, b, run_start, next_start, [&](int p, int len) {
      if (!len) {
        const int s = buf[p];
        put_bits(stage, pos, sm.lit_code[s], sm.lit_len[s]);
        pos += sm.lit_len[s];
      } else {
        const int k = sm.len_sym[len], s = 257 + k;
        put_bits(stage, pos, sm.lit_code[s] | ((unsigned)(len - kLenBase[k]) << sm.lit_len[s]), sm.lit_len[s] + kLenExtra[k]);
        pos += sm.lit_len[s] + kLenExtra[k] + 1;  // the distance code: one 0 bit
      }
    });
    if (tid == kThreads - 1) {
      put_bits(stage, base * 8LL + sm.hdr_bits + sum, sm.lit_code[256], sm.lit_len[256]);  // end of block
      if (!last) {  // then an empty stored block: 3 zero bits, padding, LEN 0, NLEN 0xFFFF
        const int end = base + sm.deflate_bytes;
        stage8[end - 2] = 0xff;
        stage8[end - 1] = 0xff;
      }
    }
  } else {
    if (tid == 0) {
      stage8[base] = last ? 1 : 0;
      stage8[base + 1] = (uint8_t)n;
      stage8[base + 2] = (uint8_t)(n >> 8);
      stage8[base + 3] = (uint8_t)~n;
      stage8[base + 4] = (uint8_t)(~n >> 8);
    }
    for (int i = tid; i < n; i += kThreads) stage8[base + 5 + i] = buf[i];
  }
  __syncthreads();

  // CRC-32 of the type and data (without the Adler-32 of the last chunk, which the layout kernel appends): one segment per thread,
  // each shifted past the bytes after it, XOR-ed together
  const int slot = sm.slot_len, crc_len = slot - 8 - (last ? 4 : 0);
  const int per = (crc_len + kThreads - 1) / kThreads, ca = min(tid * per, crc_len), cb = min(ca + per, crc_len);
  unsigned crc = crc_shift(crc_bytes(sm.crc_table, stage8 + 4 + ca, cb - ca), crc_len - cb);
  crc = cub::BlockReduce<unsigned, kThreads>(sm.cub.reduce32).Reduce(crc, [](unsigned x, unsigned y) { return x ^ y; });
  if (tid == 0) {
    if (last) {
      crc_part[g] = crc;
    } else {
      stage8[slot - 4] = (uint8_t)(crc >> 24);
      stage8[slot - 3] = (uint8_t)(crc >> 16);
      stage8[slot - 2] = (uint8_t)(crc >> 8);
      stage8[slot - 1] = (uint8_t)crc;
    }
    slot_len[g] = slot;
  }
  __syncthreads();
  uint8_t* dst = slots + g * kSlotCap;
  const int words = (slot + 3) / 4;
  for (int i = tid; i < words; i += kThreads) reinterpret_cast<unsigned*>(dst)[i] = stage[i];
}

// CTA = one image: chunk offsets (exclusive scan of the slot lengths), the image's IDAT length, its Adler-32 combined from the chunks'
// partial sums, written with the last chunk's CRC into the last slot
__global__ void __launch_bounds__(kLayoutThreads) png_layout_kernel(long long total, int cpi, uint8_t* __restrict__ slots,
                                                              const int32_t* __restrict__ slot_len, const unsigned* __restrict__ crc_part,
                                                              const unsigned* __restrict__ adler, long long* __restrict__ chunk_off,
                                                              long long* __restrict__ lengths) {
  __shared__ union {
    cub::BlockScan<long long, kLayoutThreads>::TempStorage scan;
    cub::BlockReduce<unsigned long long, kLayoutThreads>::TempStorage reduce;
  } tmp;
  const long long img = blockIdx.x, g0 = img * cpi;
  long long carry = 0;
  unsigned long long s1 = 0, s2 = 0;
  for (int c0 = 0; c0 < cpi; c0 += kLayoutThreads) {
    const int c = c0 + threadIdx.x;
    const long long v = c < cpi ? slot_len[g0 + c] : 0;
    long long p, sum;
    cub::BlockScan<long long, kLayoutThreads>(tmp.scan).ExclusiveSum(v, p, sum);
    __syncthreads();
    if (c < cpi) {
      chunk_off[g0 + c] = carry + p;
      const long long o = (long long)c * kChunk, n = min((long long)kChunk, total - o);
      const unsigned long long a = adler[2 * (g0 + c)], b = adler[2 * (g0 + c) + 1];
      s1 += a;
      s2 += (b + (unsigned long long)((total - o - n) % kAdlerMod) * a) % kAdlerMod;
    }
    carry += sum;
  }
  s1 = cub::BlockReduce<unsigned long long, kLayoutThreads>(tmp.reduce).Sum(s1);
  __syncthreads();
  s2 = cub::BlockReduce<unsigned long long, kLayoutThreads>(tmp.reduce).Sum(s2);
  if (threadIdx.x == 0) {
    const unsigned A = (unsigned)((1 + s1) % kAdlerMod), B = (unsigned)(((unsigned long long)(total % kAdlerMod) + s2) % kAdlerMod);
    const unsigned adl = (B << 16) | A;
    const long long g = g0 + cpi - 1;
    const int len = slot_len[g];
    uint8_t* s = slots + g * kSlotCap + len - 8;
    unsigned c = 0xffffffffu;
    for (int k = 0; k < 4; ++k) {
      s[k] = (uint8_t)(adl >> (24 - 8 * k));
      c ^= s[k];
      for (int j = 0; j < 8; ++j) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1;
    }
    const unsigned crc = crc_shift(crc_part[g], 4) ^ (c ^ 0xffffffffu);
    for (int k = 0; k < 4; ++k) s[4 + k] = (uint8_t)(crc >> (24 - 8 * k));
    lengths[img] = carry;
  }
}

// one thread: sizes[2 i] = image i's IDAT bytes, sizes[2 i + 1] = its offset in `out`
__global__ void png_sizes_kernel(const long long* __restrict__ lengths, int n, int64_t* __restrict__ sizes) {
  long long off = 0;
  for (int i = 0; i < n; ++i) {
    sizes[2 * i] = lengths[i];
    sizes[2 * i + 1] = off;
    off += lengths[i];
  }
}

// CTA = one chunk: its slot to its place in `out`
__global__ void __launch_bounds__(kThreads) png_copy_kernel(const uint8_t* __restrict__ slots, const int32_t* __restrict__ slot_len, int cpi,
                                                            const long long* __restrict__ chunk_off, const int64_t* __restrict__ sizes,
                                                            uint8_t* __restrict__ out) {
  const long long g = blockIdx.x, img = g / cpi;
  const uint8_t* s = slots + g * kSlotCap;
  uint8_t* d = out + sizes[2 * img + 1] + chunk_off[g];
  const int len = slot_len[g];
  for (int i = threadIdx.x; i < len; i += kThreads) d[i] = s[i];
}

// ------------------------------------------------------------------------------------------------ the multi-task grid
__constant__ unsigned char kPalette[20][3] = {{0, 0, 0},      {128, 0, 0},   {254, 0, 0},    {0, 85, 0},     {169, 0, 51},
                                              {254, 85, 0},   {0, 0, 85},    {0, 119, 220},  {85, 85, 0},    {0, 85, 85},
                                              {85, 51, 0},    {52, 86, 128}, {0, 128, 0},    {0, 0, 254},    {51, 169, 220},
                                              {0, 254, 254},  {85, 254, 169}, {169, 254, 85}, {254, 254, 0}, {254, 169, 0}};

// numpy's argmax over the channels of pixel `px`: the first maximum, or the first NaN
__device__ __forceinline__ int argmax_c(const float* __restrict__ x, long long plane, int classes) {
  float best = x[0];
  if (best != best) return 0;
  int idx = 0;
  for (int k = 1; k < classes; ++k) {
    const float v = x[k * plane];
    if (v != v) return k;
    if (v > best) {
      best = v;
      idx = k;
    }
  }
  return idx;
}

// the composed segmentation's arg-max: channel 3 times warped_cm (or its threshold), one fp32 multiply
__device__ __forceinline__ int argmax_composed(const float* __restrict__ x, long long plane, int classes, float wcm, int composition) {
  float best = -INFINITY;
  int idx = 0;
  for (int k = 0; k < classes; ++k) {
    float v = x[k * plane];
    if (k == 3 && composition == HRV_GRID_WARP_GRAD) v = __fmul_rn(v, wcm);
    if (k == 3 && composition == HRV_GRID_DETACH) v = __fmul_rn(v, wcm > 0.5f ? 1.0f : 0.0f);
    if (v != v) return k;
    if (k == 0 || v > best) {
      best = v;
      idx = k;
    }
  }
  return idx;
}

__device__ __forceinline__ float half_shift(float v) { return __fadd_rn(__fdiv_rn(v, 2.0f), 0.5f); }

// thread = one output pixel (3 bytes)
__global__ void __launch_bounds__(256) condition_grid_kernel(hrv_condition_panels p, int n, int height, int width, int classes,
                                                             int composition, uint8_t* __restrict__ out) {
  const int gh = 3 * (height + 2) + 2, gw = 4 * (width + 2) + 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)n * gh * gw) return;
  const int x = (int)(i % gw);
  const long long t = i / gw;
  const int y = (int)(t % gh), img = (int)(t / gh);
  uint8_t* o = out + i * 3;
  const int yy = y - 2, xx = x - 2;
  const int ry = yy >= 0 ? yy / (height + 2) : -1, rx = xx >= 0 ? xx / (width + 2) : -1;
  const int iy = yy - ry * (height + 2), ix = xx - rx * (width + 2);
  if (ry < 0 || rx < 0 || iy >= height || ix >= width) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  const long long plane = (long long)height * width, pix = (long long)iy * width + ix;
  auto rgb = [&](const float* s) { return s + (long long)img * 3 * plane + pix; };
  auto one = [&](const float* s) { return s[(long long)img * plane + pix]; };
  auto seg = [&](const float* s) { return s + (long long)img * classes * plane + pix; };
  float v[3];
  auto set3 = [&](float a) { v[0] = v[1] = v[2] = a; };
  auto palette = [&](int k) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) v[ch] = __fdiv_rn(k < 20 ? (float)kPalette[k][ch] : 0.0f, 255.0f);
  };
  auto halves = [&](const float* s) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) v[ch] = half_shift(s[ch * plane]);
  };
  switch (ry * 4 + rx) {
    case 0: halves(rgb(p.cloth)); break;
    case 1: set3(one(p.cloth_mask) > 0.5f ? 1.0f : 0.0f); break;
    case 2: palette(argmax_c(seg(p.parse_agnostic), plane, classes)); break;
    case 3: {
      const float* s = rgb(p.densepose);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) v[ch] = __fdiv_rn(__fadd_rn(s[ch * plane], 1.0f), 2.0f);
      break;
    }
    case 4: halves(rgb(p.parse_cloth)); break;
    case 5: set3(one(p.pcm)); break;
    case 6: halves(rgb(p.warped_cloth)); break;
    case 7: set3(one(p.warped_cm) > 0.5f ? 1.0f : 0.0f); break;
    case 8: palette(argmax_c(seg(p.parse), plane, classes)); break;
    case 9: palette(argmax_composed(seg(p.seg), plane, classes, one(p.warped_cm), composition)); break;
    case 10: halves(rgb(p.image)); break;
    default: {
      const float wcm = one(p.warped_cm);
      set3(argmax_composed(seg(p.seg), plane, classes, wcm, composition) == 3 && !(wcm > 0.5f) ? 1.0f : 0.0f);
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) o[ch] = (uint8_t)fminf(fmaxf(__fadd_rn(__fmul_rn(v[ch], 255.0f), 0.5f), 0.0f), 255.0f);
}

}  // namespace hrv_png

using namespace hrv_png;

namespace {
struct Geometry {
  long long total;  // filtered bytes per image
  long long cpi;    // chunks per image
};

Geometry geometry(int height, int width) {
  Geometry g;
  g.total = (long long)height * (3LL * width + 1);
  g.cpi = (g.total + kChunk - 1) / kChunk;
  return g;
}

size_t align256(size_t v) { return (v + 255) / 256 * 256; }

struct Workspace {
  uint8_t* slots;
  int32_t* slot_len;
  unsigned* crc_part;
  unsigned* adler;
  long long* chunk_off;
  long long* lengths;
  size_t bytes;
};

Workspace carve(void* base, long long n, const Geometry& g) {
  Workspace w;
  size_t o = 0;
  auto take = [&](size_t bytes) {
    char* p = static_cast<char*>(base) + o;
    o += align256(bytes);
    return p;
  };
  const long long chunks = n * g.cpi;
  w.slots = reinterpret_cast<uint8_t*>(take((size_t)chunks * kSlotCap));
  w.slot_len = reinterpret_cast<int32_t*>(take((size_t)chunks * sizeof(int32_t)));
  w.crc_part = reinterpret_cast<unsigned*>(take((size_t)chunks * sizeof(unsigned)));
  w.adler = reinterpret_cast<unsigned*>(take((size_t)chunks * 2 * sizeof(unsigned)));
  w.chunk_off = reinterpret_cast<long long*>(take((size_t)chunks * sizeof(long long)));
  w.lengths = reinterpret_cast<long long*>(take((size_t)n * sizeof(long long)));
  w.bytes = o;
  return w;
}

bool bad_shape(int32_t n, int32_t height, int32_t width) {
  if (n < 1 || height < 1 || width < 1 || n > 65535 || width > 0x7FFFFFFE / 3) return true;
  return (long long)n * geometry(height, width).cpi > 0x7FFFFFFFLL;
}
}  // namespace

extern "C" int hrv_png_encode_bounds(int32_t n, int32_t height, int32_t width, size_t* workspace_bytes, size_t* out_bytes) {
  if (bad_shape(n, height, width) || !workspace_bytes || !out_bytes)
    return set_error(HRV_EINVAL, "png_encode_bounds: need 1 <= n <= 65535, height and width >= 1 and fewer than 2^31 chunks");
  const Geometry g = geometry(height, width);
  *workspace_bytes = carve(nullptr, n, g).bytes;
  *out_bytes = (size_t)n * g.cpi * kSlotCap;
  return HRV_OK;
}

extern "C" int hrv_png_encode(const uint8_t* src, int32_t n, int32_t height, int32_t width, void* workspace, size_t workspace_bytes, uint8_t* out,
                              size_t out_bytes, int64_t* sizes, hrv_stream stream) {
  if (!src || !workspace || !out || !sizes || bad_shape(n, height, width)) return set_error(HRV_EINVAL, "png_encode: bad arguments");
  const Geometry g = geometry(height, width);
  const Workspace w = carve(workspace, n, g);
  if (workspace_bytes < w.bytes || out_bytes < (size_t)n * g.cpi * kSlotCap)
    return set_error(HRV_EINVAL, "png_encode: workspace %zu / out %zu bytes, need %zu / %zu (hrv_png_encode_bounds)", workspace_bytes, out_bytes,
                     w.bytes, (size_t)n * g.cpi * kSlotCap);
  cudaStream_t st = (cudaStream_t)stream;
  static bool raised = false;
  if (!raised) {
    cudaError_t e = cudaFuncSetAttribute(png_compress_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem);
    if (e != cudaSuccess) return set_error(HRV_ECUDA, "cudaFuncSetAttribute(png_compress_kernel): %s", cudaGetErrorString(e));
    raised = true;
  }
  const unsigned chunks = (unsigned)(n * g.cpi);
  png_compress_kernel<<<chunks, kThreads, kSmem, st>>>(src, height, width, g.total, (int)g.cpi, w.slots, w.slot_len, w.crc_part, w.adler);
  png_layout_kernel<<<n, kLayoutThreads, 0, st>>>(g.total, (int)g.cpi, w.slots, w.slot_len, w.crc_part, w.adler, w.chunk_off, w.lengths);
  png_sizes_kernel<<<1, 1, 0, st>>>(w.lengths, n, sizes);
  png_copy_kernel<<<chunks, kThreads, 0, st>>>(w.slots, w.slot_len, (int)g.cpi, w.chunk_off, sizes, out);
  return launched("png_encode");
}

extern "C" int hrv_condition_grid(const hrv_condition_panels* panels, int32_t n, int32_t height, int32_t width, int32_t classes, int32_t composition,
                                  uint8_t* out, hrv_stream stream) {
  if (!panels || !out || n < 1 || height < 1 || width < 1 || classes < 4 || composition < HRV_GRID_NO_COMPOSITION ||
      composition > HRV_GRID_WARP_GRAD || (long long)n * (3LL * (height + 2) + 2) * (4LL * (width + 2) + 2) > (1LL << 40))
    return set_error(HRV_EINVAL, "condition_grid: bad arguments");
  const hrv_condition_panels& p = *panels;
  const float* ptrs[] = {p.cloth, p.cloth_mask, p.parse_agnostic, p.densepose, p.parse_cloth, p.pcm, p.warped_cloth, p.warped_cm, p.parse, p.seg, p.image};
  for (const float* q : ptrs)
    if (!q) return set_error(HRV_EINVAL, "condition_grid: a panel tensor is null");
  const long long px = (long long)n * (3 * (height + 2) + 2) * (4 * (width + 2) + 2);
  condition_grid_kernel<<<(unsigned)((px + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, n, height, width, classes, composition, out);
  return launched("condition_grid");
}
