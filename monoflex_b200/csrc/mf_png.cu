// PNG image data on the GPU (what Image.open(f).convert('RGB') does on the host for KITTI's 8-bit RGB non-interlaced PNGs,
// data/datasets/kitti.py:106-114), as two kernels over a whole decode window. The host (monoflex_b200/png.py) walks the
// chunks, checks every CRC, the IHDR and the zlib header, and joins the IDAT payloads; everything from the first deflate
// block on happens here, and every byte of it is treated as untrusted.
//
//   inflate_kernel  : one warp per image. RFC 1950 / 1951 (stored, fixed- and dynamic-Huffman blocks) straight into the
//                     image's filtered-scanline buffer of h * (1 + 3 w) bytes, which is the whole output and therefore also
//                     the LZ77 window. The 32 lanes step through the same bit stream in lockstep (identical, warp-uniform
//                     state, so there is nothing to broadcast): symbols come from LUT_BITS-bit lookup tables built in
//                     shared memory for each block, codes longer than that from a canonical decode over the code counts.
//                     Lane 0 stores the literals; the warp copies stored blocks and back-references together, a reference
//                     shorter than its length reading byte j from j mod distance of the period. Adler-32 of the output
//                     is summed by all lanes over coalesced words and reduced with shuffles.
//   unfilter_kernel : one CTA per image. The five PNG filters on 3-byte pixels, filtered buffer -> uint8 HWC. Pixel (r, x)
//                     reads only (r, x-1), (r-1, x) and (r-1, x-1), so each thread owns one row of a band of blockDim rows
//                     and runs one pixel behind the thread above it (a wavefront of w + rows - 1 steps per band).
//
// Every read of the compressed stream is bounds-checked against its length (bits past the end read as zero and mark the
// stream truncated), every write against the image's buffer. A malformed stream sets its image's status (MF_PNG_*) and
// stops that image; no other image of the launch is touched.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"

namespace mf {
namespace {

constexpr int kLitBits = 10;            // litlen lookup: 1024 entries
constexpr int kDistBits = 8;            // distance (and code-length code) lookup: 256 entries
constexpr int kUnfilterThreads = 256;

// base value and extra bits of length symbols 257..285 and distance symbols 0..29 (RFC 1951 3.2.5)
__constant__ unsigned short c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59,
                                              67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ unsigned char c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ unsigned short c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769,
                                               1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ unsigned char c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11,
                                               12, 12, 13, 13};
__constant__ unsigned char c_clen_order[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

// A canonical Huffman code: counts per length, symbols sorted by (length, value), and a lookup table indexed by the next
// `bits` stream bits whose entry is symbol | length << 9, or 0 where the code is longer than `bits` (or invalid).
struct Huff {
  unsigned short cnt[16];
  unsigned short sym[288];
  unsigned short lut[1 << kLitBits];
};
struct HuffSmall {
  unsigned short cnt[16];
  unsigned short sym[32];
  unsigned short lut[1 << kDistBits];
};
struct InflateSmem {
  Huff lit;
  HuffSmall dist;                        // also holds the code-length code while a dynamic header is read
  unsigned char lens[288 + 32];
};

// canonical decode of the (LSB-first) bits `b`: symbol | length << 9, or 0 if no code of <= 15 bits matches
template <class H>
MF_DEVINL unsigned slow_decode(const H& h, unsigned b) {
  int code = 0, first = 0, index = 0;
  for (int len = 1; len <= 15; ++len) {
    code |= (b >> (len - 1)) & 1u;
    const int count = h.cnt[len];
    if (code - count < first) return static_cast<unsigned>(h.sym[index + (code - first)]) | (static_cast<unsigned>(len) << 9);
    index += count;
    first += count;
    first <<= 1;
    code <<= 1;
  }
  return 0u;
}

// Build `h` from lens[0..n): zlib's rules (inftrees.c) - an over-subscribed set is invalid; an incomplete one is accepted
// only for a literal/length or distance code whose longest code has length 1 (is_clen = 0), and a set without codes is
// accepted (every decode then fails). Lane 0 counts and sorts, the warp fills the lookup table. Returns false if invalid.
template <class H>
MF_DEVINL bool build_huff(H& h, const unsigned char* lens, int n, int bits, bool is_clen, int lane) {
  int ok = 1;
  if (lane == 0) {
    for (int l = 0; l < 16; ++l) h.cnt[l] = 0;
    for (int s = 0; s < n; ++s) h.cnt[lens[s]]++;
    h.cnt[0] = 0;
    int max = 15;
    while (max >= 1 && h.cnt[max] == 0) --max;
    int left = 1;
    for (int l = 1; l <= 15; ++l) {
      left = (left << 1) - h.cnt[l];
      if (left < 0) ok = 0;
    }
    if (ok && max > 0 && left > 0 && (is_clen || max != 1)) ok = 0;
    unsigned short offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = offs[l] + h.cnt[l];
    if (ok)
      for (int s = 0; s < n; ++s)
        if (lens[s]) h.sym[offs[lens[s]]++] = static_cast<unsigned short>(s);
  }
  ok = __shfl_sync(0xffffffffu, ok, 0);
  __syncwarp();
  if (!ok) return false;
  for (int i = lane; i < (1 << bits); i += 32) {
    const unsigned e = slow_decode(h, static_cast<unsigned>(i));
    h.lut[i] = static_cast<unsigned short>((e >> 9) <= static_cast<unsigned>(bits) ? e : 0u);
  }
  __syncwarp();
  return true;
}

// The bit reader every lane of the warp runs identically. Bytes at or past `end` read as zero; consumed() > 8 * len marks
// the stream as truncated.
struct Bits {
  const unsigned char* src;
  long long p, len;                      // next byte to load, stream length
  unsigned long long buf;
  int cnt;
  MF_DEVINL void refill() {
    if (cnt <= 32) {
      unsigned v = 0;
      if (p + 4 <= len) {
        v = static_cast<unsigned>(__ldg(src + p)) | (static_cast<unsigned>(__ldg(src + p + 1)) << 8) |
            (static_cast<unsigned>(__ldg(src + p + 2)) << 16) | (static_cast<unsigned>(__ldg(src + p + 3)) << 24);
      } else {
        for (int k = 0; k < 4; ++k)
          if (p + k < len) v |= static_cast<unsigned>(__ldg(src + p + k)) << (8 * k);
      }
      buf |= static_cast<unsigned long long>(v) << cnt;
      cnt += 32;
      p += 4;
    }
  }
  MF_DEVINL unsigned peek(int n) const { return static_cast<unsigned>(buf & ((1ull << n) - 1)); }
  MF_DEVINL void drop(int n) { buf >>= n; cnt -= n; }
  MF_DEVINL unsigned get(int n) {        // n <= 32, after a refill when n > cnt could happen
    refill();
    const unsigned v = peek(n);
    drop(n);
    return v;
  }
  MF_DEVINL long long consumed() const { return 8 * p - cnt; }
  MF_DEVINL bool overrun() const { return consumed() > 8 * len; }
  // drop to a byte boundary and hand back the byte position; the reader restarts there
  MF_DEVINL long long align() {
    drop(cnt & 7);
    const long long q = p - cnt / 8;
    p = q;
    buf = 0;
    cnt = 0;
    return q;
  }
};

template <class H>
MF_DEVINL unsigned decode_sym(const H& h, Bits& br, int bits) {
  unsigned e = h.lut[br.peek(bits)];
  if (e == 0u) e = slow_decode(h, br.peek(15));
  if (e != 0u) br.drop(static_cast<int>(e >> 9));
  return e;                              // 0: no code matches
}

__global__ void __launch_bounds__(32) inflate_kernel(const unsigned char* __restrict__ src, const long long* __restrict__ desc,
                                                     int n, unsigned char* __restrict__ filtered, int* __restrict__ status) {
  __shared__ InflateSmem sm;
  const int img = blockIdx.x, lane = threadIdx.x;
  if (img >= n) return;
  const long long* d = desc + 6 * img;
  const long long w = d[2], h = d[3];
  const long long out_len = h * (1 + 3 * w);
  unsigned char* out = filtered + d[4];
  Bits br{src + d[0], 2, d[1], 0ull, 0};     // the host checked the 2-byte zlib header
  long long o = 0;
  int err = MF_PNG_OK;
  bool final_block = false;

  while (!final_block && err == MF_PNG_OK) {
    final_block = br.get(1) != 0;
    const unsigned type = br.get(2);
    if (type == 0) {                                                       // stored
      const long long q = br.align();
      if (q + 4 > br.len) { err = MF_PNG_TRUNCATED; break; }
      const unsigned ln = br.src[q] | (br.src[q + 1] << 8), nln = br.src[q + 2] | (br.src[q + 3] << 8);
      if ((ln ^ 0xffffu) != nln) { err = MF_PNG_BAD_BLOCK; break; }
      if (q + 4 + ln > br.len) { err = MF_PNG_TRUNCATED; break; }
      if (ln > out_len - o) { err = MF_PNG_TOO_LONG; break; }
      for (unsigned j = lane; j < ln; j += 32) out[o + j] = __ldg(br.src + q + 4 + j);
      o += ln;
      br.p = q + 4 + ln;
      continue;
    }
    if (type == 3) { err = MF_PNG_BAD_BLOCK; break; }
    if (type == 1) {                                                       // fixed Huffman codes
      if (lane == 0) {
        for (int s = 0; s < 288; ++s) sm.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        for (int s = 0; s < 32; ++s) sm.lens[288 + s] = 5;
      }
      __syncwarp();
      build_huff(sm.lit, sm.lens, 288, kLitBits, false, lane);
      build_huff(sm.dist, sm.lens + 288, 32, kDistBits, false, lane);
    } else {                                                               // dynamic Huffman codes
      const int nlen = static_cast<int>(br.get(5)) + 257, ndist = static_cast<int>(br.get(5)) + 1;
      const int ncode = static_cast<int>(br.get(4)) + 4;
      if (nlen > 286 || ndist > 30) { err = MF_PNG_BAD_CODE; break; }
      if (lane == 0)
        for (int k = 0; k < 19; ++k) sm.lens[k] = 0;
      __syncwarp();
      for (int k = 0; k < ncode; ++k) {
        const unsigned v = br.get(3);
        if (lane == 0) sm.lens[c_clen_order[k]] = static_cast<unsigned char>(v);
      }
      __syncwarp();
      if (!build_huff(sm.dist, sm.lens, 19, 7, true, lane)) { err = MF_PNG_BAD_CODE; break; }
      int k = 0, prev = -1;
      while (k < nlen + ndist) {
        br.refill();
        const unsigned e = decode_sym(sm.dist, br, 7);
        if (e == 0u) { err = MF_PNG_BAD_CODE; break; }
        const int sym = e & 511;
        int val, rep;
        if (sym < 16) { val = sym; rep = 1; prev = sym; }
        else if (sym == 16) {
          if (prev < 0) { err = MF_PNG_BAD_CODE; break; }
          val = prev; rep = 3 + static_cast<int>(br.get(2));
        } else if (sym == 17) { val = 0; rep = 3 + static_cast<int>(br.get(3)); prev = 0; }
        else { val = 0; rep = 11 + static_cast<int>(br.get(7)); prev = 0; }
        if (k + rep > nlen + ndist) { err = MF_PNG_BAD_CODE; break; }
        if (lane == 0)
          for (int r = 0; r < rep; ++r) sm.lens[k + r] = static_cast<unsigned char>(val);
        k += rep;
      }
      if (err != MF_PNG_OK) break;
      __syncwarp();
      if (sm.lens[256] == 0) { err = MF_PNG_BAD_CODE; break; }            // no end-of-block code
      // the distance lengths follow the literal/length lengths in sm.lens; move them past the 288 litlen slots first
      unsigned char dl[30];
#pragma unroll
      for (int s = 0; s < 30; ++s) dl[s] = s < ndist ? sm.lens[nlen + s] : 0;
      __syncwarp();
      if (lane == 0)
        for (int s = 0; s < 30; ++s) sm.lens[288 + s] = dl[s];
      __syncwarp();
      if (!build_huff(sm.lit, sm.lens, nlen, kLitBits, false, lane) ||
          !build_huff(sm.dist, sm.lens + 288, ndist, kDistBits, false, lane)) { err = MF_PNG_BAD_CODE; break; }
    }
    // the block's symbols
    for (;;) {
      br.refill();
      const unsigned e = decode_sym(sm.lit, br, kLitBits);
      if (e == 0u) { err = MF_PNG_BAD_CODE; break; }
      const unsigned sym = e & 511u;
      if (sym < 256) {
        if (o >= out_len) { err = MF_PNG_TOO_LONG; break; }
        if (lane == 0) out[o] = static_cast<unsigned char>(sym);
        ++o;
      } else if (sym == 256) {
        break;
      } else {
        if (sym > 285) { err = MF_PNG_BAD_CODE; break; }
        const int li = static_cast<int>(sym) - 257;
        const int len = c_len_base[li] + static_cast<int>(br.get(c_len_extra[li]));
        br.refill();
        const unsigned de = decode_sym(sm.dist, br, kDistBits);
        if (de == 0u || (de & 511u) > 29) { err = MF_PNG_BAD_CODE; break; }
        const int di = static_cast<int>(de & 511u);
        const long long dist = c_dist_base[di] + br.get(c_dist_extra[di]);
        if (br.overrun()) { err = MF_PNG_TRUNCATED; break; }
        if (dist > o) { err = MF_PNG_FAR_DISTANCE; break; }
        if (len > out_len - o) { err = MF_PNG_TOO_LONG; break; }
        __syncwarp();                                                      // earlier literals and copies are visible
        const unsigned char* from = out + (o - dist);
        if (dist >= len) {
          for (int j = lane; j < len; j += 32) out[o + j] = from[j];
        } else {
          for (int j = lane; j < len; j += 32) out[o + j] = from[j % static_cast<int>(dist)];
        }
        o += len;
      }
      if (br.overrun()) { err = MF_PNG_TRUNCATED; break; }
    }
  }
  if (err != MF_PNG_OK && br.overrun()) err = MF_PNG_TRUNCATED;          // a cut stream decodes zeros before it stops
  if (err == MF_PNG_OK && o != out_len) err = MF_PNG_TOO_SHORT;
  if (err == MF_PNG_OK) {
    const long long q = br.align();
    if (q + 4 > br.len) {
      err = MF_PNG_TRUNCATED;
    } else {
      const unsigned want = (static_cast<unsigned>(br.src[q]) << 24) | (static_cast<unsigned>(br.src[q + 1]) << 16) |
                            (static_cast<unsigned>(br.src[q + 2]) << 8) | static_cast<unsigned>(br.src[q + 3]);
      // A = 1 + sum x_k, B = N + sum (N - k) x_k (mod 65521); each lane sums 4-byte words lane, lane + 32, ... with the
      // weights N - k reduced mod 65521 first, so a lane's sums stay far below 2^64 for any N
      __syncwarp();
      unsigned long long a = 0, b = 0;
      const long long nw = out_len / 4;
      const unsigned* words = reinterpret_cast<const unsigned*>(out);       // the host aligns every buffer to 16 bytes
      for (long long i = lane; i < nw; i += 32) {
        const unsigned v = words[i];
        const unsigned w0 = static_cast<unsigned>((out_len - 4 * i) % 65521ll) + 65521u;   // + 65521: w0 - 3 >= 0
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const unsigned x = (v >> (8 * k)) & 255u;
          a += x;
          b += static_cast<unsigned long long>(w0 - k) * x;
        }
      }
      for (long long i = 4 * nw + lane; i < out_len; i += 32) {
        a += out[i];
        b += static_cast<unsigned long long>((out_len - i) % 65521ll) * out[i];
      }
      a %= 65521ull;
      b %= 65521ull;
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, s);
        b += __shfl_xor_sync(0xffffffffu, b, s);
      }
      const unsigned A = static_cast<unsigned>((1ull + a) % 65521ull);
      const unsigned B = static_cast<unsigned>((static_cast<unsigned long long>(out_len) % 65521ull + b) % 65521ull);
      if (((B << 16) | A) != want) err = MF_PNG_ADLER;
    }
  }
  if (lane == 0) status[img] = err;
}

MF_DEVINL int paeth(int a, int b, int c) {
  const int p = a + b - c;
  const int pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
  return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

__global__ void __launch_bounds__(kUnfilterThreads) unfilter_kernel(const unsigned char* __restrict__ filtered,
                                                                    const long long* __restrict__ desc, int n,
                                                                    unsigned char* __restrict__ images,
                                                                    int* __restrict__ status) {
  __shared__ unsigned char up[2][kUnfilterThreads][3];   // each row's newest pixel, read one step later by the row below
  __shared__ int bad;
  const int img = blockIdx.x, t = threadIdx.x;
  if (img >= n || status[img] != MF_PNG_OK) return;      // uniform over the CTA
  const long long* d = desc + 6 * img;
  const long long w = d[2], h = d[3];                   // all indexing in 64 bits: w and h are the file's values
  const long long stride = 1 + 3 * w;
  const unsigned char* f = filtered + d[4];
  unsigned char* out = images + d[5];
  if (t == 0) bad = 0;
  __syncthreads();
  for (long long r0 = 0; r0 < h; r0 += kUnfilterThreads) {
    const int rows = static_cast<int>(min(static_cast<long long>(kUnfilterThreads), h - r0));
    const long long r = r0 + t;
    const bool live = t < rows;
    int ft = 0;
    if (live) {
      ft = f[r * stride];
      if (ft > 4) { bad = 1; ft = 0; }
    }
    const unsigned char* frow = f + r * stride + 1;
    unsigned char* orow = out + r * w * 3;
    const unsigned char* prev_row = (r > 0 && t == 0) ? out + (r - 1) * w * 3 : nullptr;
    int a[3] = {0, 0, 0}, c[3] = {0, 0, 0};
    for (long long s = 0; s < w + rows - 1; ++s) {
      const long long x = s - t;
      if (live && x >= 0 && x < w) {
        int b[3] = {0, 0, 0};
        if (r > 0) {
          if (t == 0) {
            for (int k = 0; k < 3; ++k) b[k] = prev_row[3 * x + k];   // the band above is finished
          } else {
            for (int k = 0; k < 3; ++k) b[k] = up[(s - 1) & 1][t - 1][k];
          }
        }
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int raw = frow[3 * x + k];
          int v;
          switch (ft) {
            case 1: v = raw + a[k]; break;
            case 2: v = raw + b[k]; break;
            case 3: v = raw + ((a[k] + b[k]) >> 1); break;
            case 4: v = raw + paeth(a[k], b[k], c[k]); break;
            default: v = raw; break;
          }
          v &= 255;
          orow[3 * x + k] = static_cast<unsigned char>(v);
          up[s & 1][t][k] = static_cast<unsigned char>(v);
          a[k] = v;
          c[k] = b[k];
        }
      }
      __syncthreads();
    }
  }
  if (t == 0 && bad) status[img] = MF_PNG_BAD_FILTER;
}

int check_desc(const char* who, int n) {
  if (n < 0) {
    set_error("%s: n = %d", who, n);
    return -1;
  }
  return 0;
}

}  // namespace
}  // namespace mf

using namespace mf;

extern "C" {

int mf_png_inflate(const unsigned char* src, const long long* desc, int n, unsigned char* filtered, int* status,
                   void* stream) {
  if (check_desc("mf_png_inflate", n)) return -1;
  if (n == 0) return 0;
  (void)launch_k(inflate_kernel, dim3(static_cast<unsigned>(n)), dim3(32), 0, MF_STREAM(stream), src, desc, n, filtered,
                 status);
  return check_cuda(cudaGetLastError(), "png_inflate");
}

int mf_png_unfilter(const unsigned char* filtered, const long long* desc, int n, unsigned char* images, int* status,
                    void* stream) {
  if (check_desc("mf_png_unfilter", n)) return -1;
  if (n == 0) return 0;
  (void)launch_k(unfilter_kernel, dim3(static_cast<unsigned>(n)), dim3(kUnfilterThreads), 0, MF_STREAM(stream), filtered,
                 desc, n, images, status);
  return check_cuda(cudaGetLastError(), "png_unfilter");
}

}  // extern "C"
