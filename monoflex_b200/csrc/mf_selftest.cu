// Self-test of the wgmma MN-major ("transposed") operand path that the weight-gradient GEMM of the training rows needs
// (dW[co, (tap, ci)] = sum_pixels dY[pixel, co] * X[pixel + tap, ci]: both operands have the REDUCTION index (pixels) as their
// row index in memory, i.e. they are M-/N-major, not K-major).
//
// Layout used (MN-major, SWIZZLE_128B canonical layout of the wgmma shared-memory descriptors):
//   a tile is a stack of 64-element (128 B) MN blocks; inside a block, K row k lives at (k / 8) * SBO + (k % 8) * 128 B and the
//   16-byte chunk c of that row at ((c ^ (k % 8)) * 16 B; block j of the MN dimension starts at j * LBO.
// This is exactly what a SWIZZLE_128B TMA box [K rows x 64 channels] produces (SBO = 1024 B, LBO = rows * 128 B), so a
// [pixels x channels] NHWC activation tile can be consumed as an MN-major operand without any transposition.
// The wgmma transpose immediates are set for A and B; one K = 16 step advances the start address by two 8-row groups (2 * SBO).
// D[m, n] = sum_k A[k, m] * B[k, n], M = N = 128, K = 64, one CTA of two warpgroups (one per 64-row half of M).
// Diagnostics only (tests/test_gpu_ops.py).
//
// sw128_shift_selftest: the K-major SWIZZLE_128B A descriptor of the offset/mask convolution (csrc/mf_offset_conv.cu), whose
// start is moved by whole 128-byte rows (pixels) and so lies 1..7 rows past an 8-row (1024-byte) swizzle atom. The rows are
// written with the swizzle of their ABSOLUTE shared-memory address, as a SWIZZLE_128B TMA box at a 1024-aligned destination
// writes them; each (shift s, base-offset variant v) runs one m64n32 x K = 64 product D = A[s .. s + 63] B^T with the
// descriptor's matrix-base-offset field (bits 49-51) = 0 (v = 0) or (start >> 7) & 7 (v = 1). A wrong variant gives wrong
// numbers, never an out-of-range address: every row read lies in the 80-row buffer (tests/test_gpu_offset_conv.py).
#include "mf_common.cuh"
#include "../../include/monoflex_b200.h"

namespace mf {

__global__ void __launch_bounds__(256) mn_major_selftest_kernel(const __half* __restrict__ a_km, const __half* __restrict__ b_kn,
                                                                float* __restrict__ d_mn) {
  constexpr int M = 128, N = 128, K = 64;
  constexpr uint32_t BLK = K * 128;                       // bytes of one 64-wide MN block holding all K rows (= LBO)
  __shared__ __align__(1024) uint8_t a_s[2 * BLK];
  __shared__ __align__(1024) uint8_t b_s[2 * BLK];
  const int tid = threadIdx.x, wg = tid >> 7;
  // fill: 16-byte chunk q (8 elements along MN) of K row k
  for (int i = tid; i < K * (M / 8); i += blockDim.x) {
    const int k = i / (M / 8), q = i % (M / 8);
    const uint32_t off = (q >> 3) * BLK + (k >> 3) * 1024 + (k & 7) * 128 + (((q & 7) ^ (k & 7)) << 4);
    *reinterpret_cast<uint4*>(a_s + off) = *reinterpret_cast<const uint4*>(a_km + k * M + q * 8);
    *reinterpret_cast<uint4*>(b_s + off) = *reinterpret_cast<const uint4*>(b_kn + k * N + q * 8);
  }
  fence_proxy_async();
  __syncthreads();
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  const uint64_t ad = gmma_desc(smem_u32(a_s) + wg * BLK, BLK, 1024, 128), bd = gmma_desc(smem_u32(b_s), BLK, 1024, 128);
  gmma_fence();
#pragma unroll
  for (int k4 = 0; k4 < K / 16; ++k4)
    Gmma<N>::mma<1, 1>(d, ad + static_cast<uint64_t>(k4 * ((2 * 1024) >> 4)), bd + static_cast<uint64_t>(k4 * ((2 * 1024) >> 4)),
                       k4 != 0 ? 1u : 0u);
  gmma_commit();
  gmma_wait<0>();
  gmma_hold(d);
  const int t = tid & 127, w = t >> 5, l = t & 31;
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const int row = wg * 64 + 16 * w + (l >> 2) + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + 2 * (l & 3) + (i & 1);
    d_mn[row * N + col] = d[i];
  }
}

__global__ void __launch_bounds__(128) sw128_shift_selftest_kernel(const __half* __restrict__ a_rows,
                                                                   const __half* __restrict__ b_rows, float* __restrict__ d) {
  constexpr int AR = 80, N = 32;                          // A rows (shift 7 + 64 rows fit), B rows (outputs)
  __shared__ __align__(1024) uint8_t a_s[AR * 128];
  __shared__ __align__(1024) uint8_t b_s[N * 128];
  const int tid = threadIdx.x;
  for (int i = tid; i < AR * 8; i += 128) {
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(a_s + sw128_off(r, c)) = *reinterpret_cast<const uint4*>(a_rows + r * 64 + c * 8);
  }
  for (int i = tid; i < N * 8; i += 128) {
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(b_s + sw128_off(r, c)) = *reinterpret_cast<const uint4*>(b_rows + r * 64 + c * 8);
  }
  fence_proxy_async();
  __syncthreads();
  const int w = tid >> 5, l = tid & 31;
  for (int v = 0; v < 2; ++v)
    for (int s = 0; s < 8; ++s) {
      float acc[N / 2];
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
      const uint32_t a_addr = smem_u32(a_s) + s * 128;
      const uint64_t bo = v == 1 ? static_cast<uint64_t>((a_addr >> 7) & 7) << 49 : 0ull;
      gmma_fence();
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4)
        Gmma<N>::mma<0, 0>(acc, (gmma_desc_sw128(a_addr) | bo) + 2 * k4, gmma_desc_sw128(smem_u32(b_s)) + 2 * k4,
                           k4 != 0 ? 1u : 0u);
      gmma_commit();
      gmma_wait<0>();
      gmma_hold(acc);
      float* dv = d + (v * 8 + s) * 64 * N;
#pragma unroll
      for (int i = 0; i < N / 2; ++i)
        dv[(16 * w + (l >> 2) + 8 * ((i >> 1) & 1)) * N + 8 * (i >> 2) + 2 * (l & 3) + (i & 1)] = acc[i];
    }
}

}  // namespace mf

using namespace mf;

extern "C" {

int mf_selftest_mn_major(const void* a_km, const void* b_kn, float* d_mn, void* stream) {
  mn_major_selftest_kernel<<<1, 256, 0, MF_STREAM(stream)>>>(static_cast<const __half*>(a_km), static_cast<const __half*>(b_kn),
                                                                 d_mn);
  return check_cuda(cudaGetLastError(), "mn_major_selftest");
}

int mf_selftest_sw128_shift(const void* a_rows, const void* b_rows, float* d, void* stream) {
  sw128_shift_selftest_kernel<<<1, 128, 0, MF_STREAM(stream)>>>(static_cast<const __half*>(a_rows),
                                                                    static_cast<const __half*>(b_rows), d);
  return check_cuda(cudaGetLastError(), "sw128_shift_selftest");
}

}  // extern "C"
