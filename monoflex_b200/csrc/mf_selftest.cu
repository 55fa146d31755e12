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
#include "mf_common.cuh"
#include "mf_launch.h"

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

int launch_mn_major_selftest(const __half* a_km, const __half* b_kn, float* d_mn, cudaStream_t st) {
  mn_major_selftest_kernel<<<1, 256, 0, st>>>(a_km, b_kn, d_mn);
  return check_cuda(cudaGetLastError(), "mn_major_selftest");
}

}  // namespace mf
