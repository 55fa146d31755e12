// Weight gradient of the two full-resolution 16 -> 16 channel convolutions of the stem (level0 3x3 and the 7x7 base layer on the
// zero-padded 16-channel image rows; stride 1, "same" padding). These layers are all reduction and no tile: dW is 16 x 16 x k x k
// numbers summed over B*H*W = 3.9 M pixels. The general wgmma wgrad (mf_wgrad.cu) feeds them through 2 KB im2col TMA boxes
// (64 pixels x 16 channels, request-bound inside the TMA unit: 2.15 ms per layer at B = 8, 8 % of the train step); here a
// warp owns one kernel ROW (ky) of taps and walks 16-pixel blocks of an output row:
//     dW[co, ci, ky, kx] += sum_p X[p + (ky - pad, kx - pad), ci] * dY[p, co]
// with X^T (channels x pixels, i.e. the NHWC rows read column-major) as the A operand and dY (pixels x channels) as the B
// operand of a warp-level m16n16k16 MMA (nvcuda::wmma, fp32 accumulate), kw accumulator fragments per warp, the k input
// rows of a block staged once in shared memory with zero fill at the image borders and shared by the k tap warps.
// The per-CTA partial sums meet in global memory through fp32 atomics (the summation order over CTAs is not fixed, like the
// split-K of mf_wgrad.cu and cuDNN's non-deterministic wgrad algorithms).
#include <mma.h>
#include "mf_common.cuh"
#include "mf_kernels.h"

namespace mf {

using namespace nvcuda;

template <int K>
struct NarrowCfg {
  static constexpr int G = K == 3 ? 2 : 1;                 // pixel blocks in flight per CTA
  static constexpr int WARPS = K * G;
  static constexpr int TW = 16 + K - 1;                    // staged pixels per row
  static constexpr int X_TILE = K * TW * 16;               // halves per group
  static constexpr int Y_TILE = 16 * 16;
};

template <int K>
__global__ void __launch_bounds__(NarrowCfg<K>::WARPS * 32)
wgrad_narrow_kernel(const __half* __restrict__ x, int x_ld, const __half* __restrict__ dy, int dy_ld, int B, int H, int W,
                    float* __restrict__ dw) {
  using C = NarrowCfg<K>;
  constexpr int PAD = K / 2;
  __shared__ __align__(32) __half xs[2][C::G][C::X_TILE];
  __shared__ __align__(32) __half ys[2][C::G][C::Y_TILE];
  __shared__ __align__(32) float red[C::WARPS][16 * 16];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = warp / K, ky = warp - grp * K;
  const int bw = (W + 15) >> 4;                            // 16-pixel blocks per row
  const long long nblocks = static_cast<long long>(B) * H * bw;
  const long long nunits = (nblocks + C::G - 1) / C::G;    // one unit = G consecutive blocks
  wmma::fragment<wmma::accumulator, 16, 16, 16, float> acc[K];
#pragma unroll
  for (int kx = 0; kx < K; ++kx) wmma::fill_fragment(acc[kx], 0.f);

  auto stage = [&](const long long unit, const int buf) {
    // every thread copies 16-byte chunks: X tiles (K rows x TW pixels x 2 chunks) and dY blocks (16 pixels x 2 chunks) of G blocks.
    // The block -> (image row, x0) decode is done once per block in 32-bit arithmetic, not per chunk (the 64-bit divisions of
    // the first version were the kernel: ~7 k warp instructions per 16-pixel block)
    constexpr int XCH = K * C::TW * 2, YCH = 16 * 2;
#pragma unroll
    for (int g = 0; g < C::G; ++g) {
      const long long blk = unit * C::G + g;
      const bool live = blk < nblocks;
      const int blk32 = live ? static_cast<int>(blk) : 0;  // launcher guarantees B*H*ceil(W/16) < 2^31
      const int row = blk32 / bw;                          // (b, y)
      const int x0 = (blk32 - row * bw) * 16;
      const int y = row % H;
      const long long rowbase = static_cast<long long>(row - y) * W;     // first pixel of the image
      for (int r = threadIdx.x; r < XCH + YCH; r += blockDim.x) {
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (r < XCH) {
          const int half_id = r & 1, pr = r >> 1, ry = pr / C::TW, px = pr - ry * C::TW;
          const int yy = y + ry - PAD, xx = x0 + px - PAD;
          if (live && yy >= 0 && yy < H && xx >= 0 && xx < W)
            v = __ldg(reinterpret_cast<const uint4*>(x + (rowbase + static_cast<long long>(yy) * W + xx) * x_ld + half_id * 8));
          *reinterpret_cast<uint4*>(&xs[buf][g][(ry * C::TW + px) * 16 + half_id * 8]) = v;
        } else {
          const int q = r - XCH, half_id = q & 1, px = q >> 1;
          if (live && x0 + px < W)
            v = __ldg(reinterpret_cast<const uint4*>(dy + (static_cast<long long>(row) * W + x0 + px) * dy_ld + half_id * 8));
          *reinterpret_cast<uint4*>(&ys[buf][g][px * 16 + half_id * 8]) = v;
        }
      }
    }
  };

  int buf = 0;
  long long unit = blockIdx.x;
  if (unit < nunits) stage(unit, 0);
  __syncthreads();
  for (; unit < nunits; unit += gridDim.x) {
    const long long next = unit + gridDim.x;
    if (next < nunits) stage(next, buf ^ 1);               // global loads of the next unit overlap this unit's MMAs
    wmma::fragment<wmma::matrix_b, 16, 16, 16, __half, wmma::row_major> bf;
    wmma::load_matrix_sync(bf, &ys[buf][grp][0], 16);      // B[k = pixel][n = co]
#pragma unroll
    for (int kx = 0; kx < K; ++kx) {
      wmma::fragment<wmma::matrix_a, 16, 16, 16, __half, wmma::col_major> af;
      wmma::load_matrix_sync(af, &xs[buf][grp][(ky * C::TW + kx) * 16], 16);   // A[m = ci][k = pixel] = X[pixel + kx][ci]
      wmma::mma_sync(acc[kx], af, bf, acc[kx]);
    }
    __syncthreads();
    buf ^= 1;
  }
  // acc[kx](m = ci, n = co) -> dW[co][ci][ky][kx]; the G groups of a CTA are summed through the atomics as well
#pragma unroll
  for (int kx = 0; kx < K; ++kx) {
    wmma::store_matrix_sync(&red[warp][0], acc[kx], 16, wmma::mem_row_major);
    __syncwarp();
    for (int i = lane; i < 256; i += 32) {
      const int ci = i >> 4, co = i & 15;
      const float v = red[warp][i];
      if (v != 0.f) atomicAdd(dw + ((co * 16 + ci) * K + ky) * K + kx, v);
    }
    __syncwarp();
  }
}

// x: [B*H*W, x_ld >= 16] fp16 rows, dy: [B*H*W, dy_ld >= 16] fp16 rows; dw: [16, 16, k, k] fp32, zeroed here
int launch_conv_wgrad_narrow(const __half* x, int x_ld, int B, int H, int W, const __half* dy, int dy_ld, int k, float* dw,
                             cudaStream_t st) {
  if ((k != 3 && k != 7) || x_ld % 8 != 0 || dy_ld % 8 != 0 || (reinterpret_cast<uintptr_t>(x) & 15) ||
      (reinterpret_cast<uintptr_t>(dy) & 15)) {
    set_error("conv wgrad (narrow): k in {3, 7}, 16-byte aligned rows");
    return -1;
  }
  if (static_cast<long long>(B) * H * ((W + 15) / 16) >= (1ll << 31)) { set_error("conv wgrad (narrow): too many pixel blocks"); return -1; }
  if (check_cuda(cudaMemsetAsync(dw, 0, sizeof(float) * 16 * 16 * k * k, st), "conv wgrad narrow memset")) return -1;
  int dev = 0, nsm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  const int grid = nsm * 4;
  if (k == 3) wgrad_narrow_kernel<3><<<grid, NarrowCfg<3>::WARPS * 32, 0, st>>>(x, x_ld, dy, dy_ld, B, H, W, dw);
  else wgrad_narrow_kernel<7><<<grid, NarrowCfg<7>::WARPS * 32, 0, st>>>(x, x_ld, dy, dy_ld, B, H, W, dw);
  return check_cuda(cudaGetLastError(), "conv wgrad narrow launch");
}

}  // namespace mf
