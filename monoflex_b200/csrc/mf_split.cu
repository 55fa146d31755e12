// Conversions that exist only for strict precision's pair rows: the split weight packer, the two image packers and the
// pair-rows -> fp32 NCHW export.
//
// Number format: an fp32-grade value v travels as TWO fp16 numbers, hi = fp16(v) and lo = fp16(v - hi) (22 significant
// bits, absolute floor 2^-25), stored in the same NHWC pixel row: the lo block starts `*_lo` elements after the hi block
// (engine.py gives every strict activation buffer the row layout [hi channels | lo channels]). The tensor-core kernels
// consume such operands as the K-concatenation A_hi W_hi + A_lo W_hi + A_hi W_lo (mf_igemm2.cu, `split_in`), which is what
// brings the end-to-end forward within 1e-3 of the fp32 reference (DESIGN.md §4 "Precision modes"); the layout kernels
// between those GEMMs (max-pool, up-sample + add, edge-fusion gather / final add) read and write either format
// (mf_elementwise.cu, PairRows in mf_common.cuh).
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"

namespace mf {

// ---------------------------------------------------------------- split weight packer
// OIHW fp32 -> [n_pad, k_pad] fp16 in the virtual K order of `split_in` GEMMs:
//   k' = (((tap * nchunk + chunk) * 3 + which) * cw + c),  cw = min(Cin, 64), channel = chunk * cw + c,
//   which 0, 1 -> W_hi (multiplies A_hi, A_lo), which 2 -> W_lo = fp16(W - W_hi) (multiplies A_hi).
__global__ void pack_conv_weight_split_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, int cw, int n_pad,
                                              int k_pad, __half* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n_pad) * k_pad) return;
  const int k = static_cast<int>(i % k_pad), n = static_cast<int>(i / k_pad);
  const int unit = k / cw, c = k - unit * cw;
  const int tc = unit / 3, which = unit - tc * 3;
  const int nch = Cin / cw;
  const int tap = tc / nch, ci = (tc - tap * nch) * cw + c;
  __half r = __float2half_rn(0.f);
  if (n < Cout && tap < taps) {
    const float v = w[(static_cast<long long>(n) * Cin + ci) * taps + tap];
    const __half hi = __float2half_rn(v);
    r = which == 2 ? __float2half_rn(v - __half2float(hi)) : hi;
  }
  out[i] = r;
}

// ---------------------------------------------------------------- image: NCHW fp32 [B,3,H,W] -> [B*H*W, 16] fp16 rows
// channels [hi(3) | lo(3) | hi(3) | 0 x 7]: the 7x7 stem then is an ORDINARY 16-channel convolution whose per-tap weights are
// [W_hi | W_hi | W_lo | 0] (engine.py), i.e. the three split products in one pass over 16 instead of 3 x 8 channels.
__global__ void pack_image_split_kernel(const float* __restrict__ x, __half* __restrict__ y, int B, int C, long long HW) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const long long b = i / HW, pix = i - b * HW;
  __half o[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) o[c] = __float2half_rn(0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c < C) {
      const float v = __ldg(x + (b * C + c) * HW + pix);
      const __half hi = __float2half_rn(v);
      o[c] = hi;
      o[3 + c] = __float2half_rn(v - __half2float(hi));
      o[6 + c] = hi;
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(y + i * 16);
  dst[0] = *reinterpret_cast<uint4*>(&o[0]);
  dst[1] = *reinterpret_cast<uint4*>(&o[8]);
}

// image -> ONE 16-byte-pixel plane [hi3 | lo3 | 0 0] for the row-segment stem kernel (mf_rows.cu, in_mode 1)
__global__ void pack_image_pair8_kernel(const float* __restrict__ x, __half* __restrict__ y, int B, int C, long long HW) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= B * HW) return;
  const long long b = i / HW, pix = i - b * HW;
  __half o[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) o[c] = __float2half_rn(0.f);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    if (c < C) {
      const float v = __ldg(x + (b * C + c) * HW + pix);
      const __half hi = __float2half_rn(v);
      o[c] = hi;
      o[3 + c] = __float2half_rn(v - __half2float(hi));
    }
  }
  *reinterpret_cast<uint4*>(y + i * 8) = *reinterpret_cast<uint4*>(&o[0]);
}

// hi/lo rows -> fp32 NCHW (tests / feature-map export): y = float(hi) + float(lo)
__global__ void split_to_nchw_kernel(const __half* __restrict__ x, int x_ld, int x_lo, float* __restrict__ y, int C, int HW) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int pp = p0 + i, c = c0 + threadIdx.x;
    float v = 0.f;
    if (pp < HW && c < C) {
      const __half* r = x + (static_cast<long long>(b) * HW + pp) * x_ld + c;
      v = __half2float(r[0]) + __half2float(r[x_lo]);
    }
    tile[i][threadIdx.x] = v;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, pp = p0 + threadIdx.x;
    if (c < C && pp < HW) y[(static_cast<long long>(b) * C + c) * HW + pp] = tile[threadIdx.x][i];
  }
}

}  // namespace mf

using namespace mf;

extern "C" {

int mf_pack_conv_weight_split(const float* w, int Cout, int Cin, int kh, int kw, int n_pad, int k_pad, void* out, void* stream) {
  const int cw = Cin < 64 ? Cin : 64;
  if (Cin % cw != 0 || 64 % cw != 0 || k_pad < 3 * kh * kw * Cin || n_pad < Cout) {
    set_error("pack_conv_weight_split: Cin=%d must be a multiple of 64 or one of 8/16/32; k_pad >= 3*taps*Cin", Cin);
    return -1;
  }
  const long long n = static_cast<long long>(n_pad) * k_pad;
  pack_conv_weight_split_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, MF_STREAM(stream)>>>(w, Cout, Cin, kh * kw, cw, n_pad,
                                                                                                k_pad, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "pack_conv_weight_split");
}

int mf_pack_image_split(const float* x, void* y, int B, int C, int H, int W, void* stream) {
  const cudaStream_t st = MF_STREAM(stream);
  if (C > 3) { set_error("pack_image_split: C=%d > 3", C); return -1; }
  const long long n = static_cast<long long>(B) * H * W;
  (void)launch_k(pack_image_split_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, x, y, B, C,
                 static_cast<long long>(H) * W);
  return check_cuda(cudaGetLastError(), "pack_image_split");
}

int mf_pack_image_pair8(const float* x, void* y, int B, int C, int H, int W, void* stream) {
  const cudaStream_t st = MF_STREAM(stream);
  if (C > 3) { set_error("pack_image_pair8: C=%d > 3", C); return -1; }
  const long long n = static_cast<long long>(B) * H * W;
  (void)launch_k(pack_image_pair8_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, x, y, B, C,
                 static_cast<long long>(H) * W);
  return check_cuda(cudaGetLastError(), "pack_image_pair8");
}

int mf_split_to_nchw_f32(const void* x, int x_ld, int x_lo, float* y, int B, int C, int HW, void* stream) {
  const cudaStream_t st = MF_STREAM(stream);
  dim3 grid((HW + 31) / 32, (C + 31) / 32, B), block(32, 8);
  (void)launch_k(split_to_nchw_kernel, dim3(grid), dim3(block), 0, st, x, x_ld, x_lo, y, C, HW);
  return check_cuda(cudaGetLastError(), "split_to_nchw");
}

}  // extern "C"
