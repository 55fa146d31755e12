// Library state of libmonoflex_b200.so (the thread-local last-error string, the debug conv-implementation switch), the
// weight packers and the conv / DCN GEMM entry points, which check their arguments and pick the kernel (mf_igemm2.cu,
// mf_offset_conv.cu, mf_simt.cu). Every other entry point of include/monoflex_b200.h is defined beside its kernels.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"
#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace mf {

static thread_local char g_err[512] = "";
static int g_conv_impl = 0;  // 0 = wgmma implicit GEMM, 1 = CUDA-core cross-check

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
int check_cuda(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return 0;
  set_error("%s: %s", what, cudaGetErrorString(e));
  return -1;
}

// ---------------------------------------------------------------- weight repack: OIHW fp32 -> [n_pad, k_pad] fp16, k = tap*cin_pad + c
__global__ void pack_conv_weight_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, int cin_pad, int n_pad,
                                        int k_pad, __half* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n_pad) * k_pad) return;
  const int k = static_cast<int>(i % k_pad), n = static_cast<int>(i / k_pad);
  const int tap = k / cin_pad, c = k - tap * cin_pad;
  float v = 0.f;
  if (n < Cout && tap < taps && c < Cin) v = w[(static_cast<long long>(n) * Cin + c) * taps + tap];
  out[i] = __float2half_rn(v);
}

// data-gradient weights straight from the live OIHW parameter: the stride-1 dX conv is the forward kernel on dY with the taps
// rotated by 180 degrees and in / out channels transposed - out[n = ci][k = tap' * cout_pad + co] = w[co][ci][taps - 1 - tap']
// (one launch instead of flip + transpose + contiguous + zero-pad cat + pack)
__global__ void pack_conv_weight_dgrad_kernel(const float* __restrict__ w, int Cout, int Cin, int taps, int cout_pad, int n_pad,
                                              int k_pad, __half* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n_pad) * k_pad) return;
  const int k = static_cast<int>(i % k_pad), n = static_cast<int>(i / k_pad);
  const int tap = k / cout_pad, co = k - tap * cout_pad;
  float v = 0.f;
  if (n < Cin && tap < taps && co < Cout) v = w[(static_cast<long long>(co) * Cin + n) * taps + (taps - 1 - tap)];
  out[i] = __float2half_rn(v);
}

// batched form for training plans: all weights of a plan are re-packed from their live fp32 parameters at the start of every
// run - one launch over a device table of descriptors instead of ~190 small ones. desc (5 x int64): w ptr, out ptr,
// Cout | Cin << 32, taps | cin_pad << 32, n_pad | k_pad << 32.
__global__ void pack_conv_weight_batched_kernel(const long long* __restrict__ descs, int n) {
  const int d = blockIdx.y;
  if (d >= n) return;
  const long long* q = descs + 5 * d;
  const float* w = reinterpret_cast<const float*>(q[0]);
  __half* out = reinterpret_cast<__half*>(q[1]);
  const int Cout = static_cast<int>(q[2] & 0xffffffffll), Cin = static_cast<int>(q[2] >> 32);
  const int taps = static_cast<int>(q[3] & 0xffffffffll), cin_pad = static_cast<int>(q[3] >> 32);
  const int n_pad = static_cast<int>(q[4] & 0xffffffffll), k_pad = static_cast<int>(q[4] >> 32);
  const long long total = static_cast<long long>(n_pad) * k_pad;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int k = static_cast<int>(i % k_pad), nn = static_cast<int>(i / k_pad);
    const int tap = k / cin_pad, c = k - tap * cin_pad;
    float v = 0.f;
    if (nn < Cout && tap < taps && c < Cin) v = w[(static_cast<long long>(nn) * Cin + c) * taps + tap];
    out[i] = __float2half_rn(v);
  }
}

// the implicit-GEMM parameters every conv entry point fills alike; each adds its own residual / split / DCN / head fields.
// The K axis of a split-input GEMM is 3 x taps x Cin.
static IgemmParams conv_params(const void* x, int x_ld, int B, int H, int W, int Cin, int kh, int kw, int stride, int pad,
                               bool split_in, int Cout, const float* scale, const float* shift, int act, int out_mode, void* y,
                               int y_ld) {
  IgemmParams p;
  memset(&p, 0, sizeof(p));
  p.x = static_cast<const __half*>(x); p.x_ld = x_ld; p.B = B; p.H = H; p.W = W; p.Cin = Cin;
  p.kh = kh; p.kw = kw; p.stride = stride; p.pad = pad;
  p.Ho = (H + 2 * pad - kh) / stride + 1;
  p.Wo = (W + 2 * pad - kw) / stride + 1;
  p.M = B * p.Ho * p.Wo;
  p.split_in = split_in ? 1 : 0;
  p.K_real = (split_in ? 3 : 1) * kh * kw * Cin;
  p.nkb = (p.K_real + 63) / 64;
  p.Cout = Cout; p.scale = scale; p.shift = shift; p.act = act; p.out_mode = out_mode; p.y = y; p.y_ld = y_ld;
  return p;
}

// ACT_OFFMASK = the DCN offset/mask convolution, which has one kernel (mf_offset_conv.cu): 3x3, stride 1, pad 1,
// Cin % 64 == 0, no residual, fp32 NHWC rows
static bool offset_conv_shape(const IgemmParams& p) {
  if (p.out_mode == OUT_F32_NHWC && p.kh == 3 && p.kw == 3 && p.stride == 1 && p.pad == 1 && p.Cin % 64 == 0 &&
      p.res == nullptr)
    return true;
  set_error("offset/mask conv (ACT_OFFMASK): only 3x3 stride 1 pad 1, Cin %% 64 == 0, fp32 NHWC rows, no residual "
            "(got %dx%d stride %d pad %d Cin %d out_mode %d)", p.kh, p.kw, p.stride, p.pad, p.Cin, p.out_mode);
  return false;
}

static int run_gemm(const IgemmParams& p, const void* wp, int n_pad, int k_pad, int mode, cudaStream_t st) {
  if (g_conv_impl == 1) return launch_simt_gemm(p, static_cast<const __half*>(wp), n_pad, k_pad, mode, st);
  return launch_igemm2(p, static_cast<const __half*>(wp), n_pad, k_pad, mode, st);
}

}  // namespace mf

using namespace mf;

extern "C" {

const char* mf_last_error(void) { return g_err; }
int mf_version(void) { return 100; }
int mf_set_conv_impl(int impl) {
  if (impl != 0 && impl != 1) { set_error("mf_set_conv_impl: impl must be 0 or 1"); return -1; }
  g_conv_impl = impl;
  return 0;
}
int mf_conv_block_n(int cout) {
  if (cout <= 16) return 16;
  if (cout <= 32) return 32;
  if (cout <= 64) return 64;
  return 128;
}

int mf_pack_conv_weight(const float* w, int Cout, int Cin, int kh, int kw, int cin_pad, int n_pad, int k_pad, void* out,
                        void* stream) {
  if (cin_pad < Cin || k_pad < kh * kw * cin_pad || n_pad < Cout) { set_error("pack_conv_weight: bad padding"); return -1; }
  const long long n = static_cast<long long>(n_pad) * k_pad;
  pack_conv_weight_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, MF_STREAM(stream)>>>(
      w, Cout, Cin, kh * kw, cin_pad, n_pad, k_pad, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "pack_conv_weight");
}

int mf_pack_conv_weight_dgrad(const float* w, int Cout, int Cin, int kh, int kw, int cout_pad, int n_pad, int k_pad, void* out,
                              void* stream) {
  if (cout_pad < Cout || k_pad < kh * kw * cout_pad || n_pad < Cin) { set_error("pack_conv_weight_dgrad: bad padding"); return -1; }
  const long long n = static_cast<long long>(n_pad) * k_pad;
  pack_conv_weight_dgrad_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, MF_STREAM(stream)>>>(
      w, Cout, Cin, kh * kw, cout_pad, n_pad, k_pad, static_cast<__half*>(out));
  return check_cuda(cudaGetLastError(), "pack_conv_weight_dgrad");
}

int mf_pack_conv_weights_batched(const void* descs, int n, void* stream) {
  if (n <= 0) return 0;
  pack_conv_weight_batched_kernel<<<dim3(64, n), 256, 0, MF_STREAM(stream)>>>(static_cast<const long long*>(descs), n);
  return check_cuda(cudaGetLastError(), "pack_conv_weight_batched");
}

int mf_conv2d_nhwc_f16(const void* x, int x_ld, int B, int H, int W, int Cin, const void* w_packed, int n_pad, int k_pad,
                       int kh, int kw, int stride, int pad, int Cout, const float* scale, const float* shift,
                       const void* res, int res_ld, int act, int out_mode, void* y, int y_ld, void* stream) {
  IgemmParams p = conv_params(x, x_ld, B, H, W, Cin, kh, kw, stride, pad, false, Cout, scale, shift, act, out_mode, y, y_ld);
  p.res = static_cast<const __half*>(res); p.res_ld = res_ld;
  if (p.Ho <= 0 || p.Wo <= 0 || Cout <= 0) { set_error("mf_conv2d_nhwc_f16: empty output"); return -1; }
  if (act == ACT_OFFMASK && g_conv_impl == 0) {
    if (!offset_conv_shape(p)) return -1;
    return launch_offset_conv(p.x, x_ld, 0, B, H, W, Cin, static_cast<const __half*>(w_packed), n_pad, k_pad, scale, shift,
                              static_cast<float*>(y), y_ld, false, MF_STREAM(stream));
  }
  return run_gemm(p, w_packed, n_pad, k_pad, MODE_CONV, MF_STREAM(stream));
}

// strict-precision variants: operands / outputs are hi/lo fp16 pairs (mf_split.cu); K axis of a split-input GEMM = 3 x taps x Cin
int mf_conv2d_nhwc_f16x2(const void* x, int x_ld, int x_lo, int B, int H, int W, int Cin, const void* w_packed, int n_pad,
                         int k_pad, int kh, int kw, int stride, int pad, int Cout, const float* scale, const float* shift,
                         const void* res, int res_ld, int res_lo, int act, int out_mode, void* y, int y_ld, int y_lo,
                         int split_in, int split_out, void* stream) {
  IgemmParams p =
      conv_params(x, x_ld, B, H, W, Cin, kh, kw, stride, pad, split_in != 0, Cout, scale, shift, act, out_mode, y, y_ld);
  p.split_out = split_out ? 1 : 0;
  p.x_lo = x_lo; p.res_lo = res_lo; p.y_lo = y_lo;
  p.cw = Cin < 64 ? Cin : 64;
  p.res = static_cast<const __half*>(res); p.res_ld = res_ld;
  if (p.Ho <= 0 || p.Wo <= 0 || Cout <= 0) { set_error("mf_conv2d_nhwc_f16x2: empty output"); return -1; }
  if (g_conv_impl == 1) { set_error("mf_conv2d_nhwc_f16x2: no CUDA-core cross-check of the split path"); return -1; }
  if (act == ACT_OFFMASK) {
    if (!offset_conv_shape(p)) return -1;
    if (p.split_out) { set_error("mf_conv2d_nhwc_f16x2: the offset/mask rows are fp32, not a split output"); return -1; }
    return launch_offset_conv(p.x, x_ld, x_lo, B, H, W, Cin, static_cast<const __half*>(w_packed), n_pad, k_pad, scale, shift,
                              static_cast<float*>(y), y_ld, p.split_in != 0, MF_STREAM(stream));
  }
  return launch_igemm2(p, static_cast<const __half*>(w_packed), n_pad, k_pad, MODE_CONV, MF_STREAM(stream));
}

int mf_head_conv_f16x2(const void* x, int x_ld, int x_lo, int B, int H, int W, int Cin, const void* w_packed, int n_pad, int k_pad,
                       int nbranch, const float* scale, const float* shift, int act, const void* w2, float* part, int ntot,
                       const int* out_nch, const int* out_ch0, const int* hid_col, void* hid, int hid_ld, int hid_lo,
                       const unsigned char* hid_mask, void* stream) {
  if (nbranch <= 0 || nbranch > 12) { set_error("mf_head_conv_f16x2: 1..12 branches"); return -1; }
  // no output tensor map (OUT_F32_NCHW): the consumers write partial planes + masked hidden rows
  IgemmParams p = conv_params(x, x_ld, B, H, W, Cin, 3, 3, 1, 1, true, nbranch * 256, scale, shift, act, OUT_F32_NCHW, hid,
                              hid_ld);
  p.x_lo = x_lo; p.y_lo = hid_lo; p.cw = 64;
  p.h2_w = static_cast<const __half*>(w2); p.h2_part = part; p.h2_ntot = ntot; p.h2_mask = hid_mask;
  bool need_hid = false;
  for (int i = 0; i < nbranch; ++i) {
    if (out_nch[i] < 0 || out_nch[i] > 32 || out_ch0[i] < 0 || out_ch0[i] + out_nch[i] > ntot) {
      set_error("mf_head_conv_f16x2: branch %d has %d outputs at %d of %d", i, out_nch[i], out_ch0[i], ntot);
      return -1;
    }
    p.h2_nch[i] = out_nch[i]; p.h2_ch0[i] = out_ch0[i]; p.h2_hid_col[i] = hid_col[i];
    need_hid = need_hid || hid_col[i] >= 0;
  }
  if (need_hid && (hid == nullptr || hid_mask == nullptr || hid_ld % 8 != 0 || hid_lo % 8 != 0)) {
    set_error("mf_head_conv_f16x2: hidden rows requested without a buffer / mask (or unaligned strides)");
    return -1;
  }
  if (Cin % 64 != 0 || w2 == nullptr || part == nullptr) { set_error("mf_head_conv_f16x2: Cin %% 64, w2 and part are required"); return -1; }
  return launch_igemm2(p, static_cast<const __half*>(w_packed), n_pad, k_pad, MODE_CONV, MF_STREAM(stream));
}

int mf_dcn_nhwc_f16x2(const void* x, int x_ld, int x_lo, int B, int H, int W, int Cin, const float* offmask, int om_ld,
                      const void* w_packed, int n_pad, int k_pad, int Cout, const float* scale, const float* shift, int act,
                      void* y, int y_ld, int y_lo, void* stream) {
  IgemmParams p = conv_params(x, x_ld, B, H, W, Cin, 3, 3, 1, 1, true, Cout, scale, shift, act, OUT_F16_NHWC, y, y_ld);
  p.split_out = 1; p.x_lo = x_lo; p.y_lo = y_lo; p.cw = 64;
  p.offmask = offmask; p.om_ld = om_ld;
  if (om_ld < 27) { set_error("mf_dcn_nhwc_f16x2: om_ld < 27"); return -1; }
  return launch_igemm2(p, static_cast<const __half*>(w_packed), n_pad, k_pad, MODE_DCN, MF_STREAM(stream));
}

int mf_dcn_nhwc_f16(const void* x, int x_ld, int B, int H, int W, int Cin, const float* offmask, int om_ld,
                    const void* w_packed, int n_pad, int k_pad, int Cout, const float* scale, const float* shift, int act,
                    int out_mode, void* y, int y_ld, void* stream) {
  IgemmParams p = conv_params(x, x_ld, B, H, W, Cin, 3, 3, 1, 1, false, Cout, scale, shift, act, out_mode, y, y_ld);
  p.offmask = offmask; p.om_ld = om_ld;
  if (om_ld < 27) { set_error("mf_dcn_nhwc_f16: om_ld < 27"); return -1; }
  return run_gemm(p, w_packed, n_pad, k_pad, MODE_DCN, MF_STREAM(stream));
}

}  // extern "C"
