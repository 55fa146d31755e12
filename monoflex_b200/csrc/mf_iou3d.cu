// get_iou_3d(pred_corners, target_corners) (model/layers/iou_loss.py:99-136) as a standalone op: one thread per box pair,
// grid-stride, over [N, 8, 3] float32 corner tables. The IoU itself is mf_iou3d.cuh, shared with the fused loss.
#include "mf_common.cuh"
#include "mf_iou3d.cuh"
#include "../../include/monoflex_b200.h"

namespace mf {
namespace {

__global__ void __launch_bounds__(256) iou3d_corners_kernel(const float* __restrict__ pred, const float* __restrict__ target,
                                                            long long n, float* __restrict__ out) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float a[24], b[24];
#pragma unroll
    for (int k = 0; k < 24; ++k) {
      a[k] = __ldg(pred + i * 24 + k);
      b[k] = __ldg(target + i * 24 + k);
    }
    out[i] = iou3d_corners(a, b);
  }
}

}  // namespace
}  // namespace mf

extern "C" {

int mf_iou3d_corners(const float* pred, const float* target, long long n, float* out, void* stream) {
  if (n < 0) {
    mf::set_error("mf_iou3d_corners: N = %lld < 0", n);
    return -1;
  }
  if (n == 0) return 0;
  if (!pred || !target || !out) {
    mf::set_error("mf_iou3d_corners: NULL pointer (pred %p, target %p, out %p)", static_cast<const void*>(pred),
                  static_cast<const void*>(target), static_cast<void*>(out));
    return -1;
  }
  const long long blocks = (n + 255) / 256;
  (void)mf::launch_k(mf::iou3d_corners_kernel, dim3(static_cast<unsigned>(blocks < 4096 ? blocks : 4096)), dim3(256), 0,
                     MF_STREAM(stream), pred, target, n, out);
  return mf::check_cuda(cudaGetLastError(), "iou3d_corners");
}

}  // extern "C"
