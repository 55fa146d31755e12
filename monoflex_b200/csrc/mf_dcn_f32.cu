// Boundary B (SURVEY §8b, rows R4/R5): the reference's native operator pair `_ext.dcn_v2_forward / dcn_v2_backward`
// (src/dcn_v2.h:9-23, 48-59) in EXACT fp32 on reference-layout tensors (NCHW, contiguous), general geometry (kernel,
// stride, pad, dilation, deformable groups). The detector's hot path uses the fused fp16 tensor-core kernel of
// mf_igemm2.cu; this file is what `dcn_v2.py`'s autograd Function, testcuda.py's KATs and gradcheck run on.
//
// The reference (dcn_v2_cuda.cu:42-172, 206-335) loops over the batch on the host and per sample launches im2col + SGEMM
// (+ col2im, col2im_coord, SGEMM, SGEMV), with a [C*k*k, H*W] columns buffer. Here, with smem-tiled fp32 CUDA-core GEMMs
// (64 x 64 tiles, 16-deep k steps, 4 x 4 outputs per thread) whose operand tiles are produced on the fly:
//   forward   one launch: the column tile (mask * bilinear sample) is built straight in shared memory from a per-(pixel, tap)
//             sampling record - no columns buffer, offsets/masks read once per (pixel, tap) instead of once per channel;
//   backward  k1: grad-columns GEMM  gcol[b, c*T+tap, p] = sum_o W[o, c*T+tap] dY[b, o, p]                 (workspace)
//             k2: one thread per (b, group, tap, pixel): scatter of gcol * mask * bilinear weights into dX (atomicAdd, the
//                 reference's col2im) and d offset / d mask accumulated over the group's channels in registers and
//                 written once (the reference's col2im_coord runs a thread per (offset channel, pixel) over all columns);
//             k3: weight gradient as a split-K GEMM over (b, pixel) whose column operand is re-sampled on the fly;
//                 partial sums per split go to the workspace and are reduced in a fixed order (deterministic);
//             k4: bias gradient, one block per output channel.
#include "mf_common.cuh"
#include "mf_launch.h"

namespace mf {

struct DcnGeom {
  int B, C, H, W, Co, kh, kw, sh, sw, ph, pw, dh, dw, dg, Ho, Wo;
};

// bilinear sampling record of one (pixel, tap): corner weights (0 where the corner is outside the image), the derivative
// coefficients of the sample w.r.t. the fractional position, clamped corner indices (dcn_v2_im2col_cuda.cu:27-123)
struct DcnSample {
  float w1, w2, w3, w4;
  float dh1, dh2, dh3, dh4;
  float dw1, dw2, dw3, dw4;
  int i1, i2, i3, i4;
  bool inside;
};
__device__ __forceinline__ DcnSample dcn_sample(int H, int W, float h_im, float w_im) {
  DcnSample s;
  s.inside = h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(H) && w_im < static_cast<float>(W);
  s.w1 = s.w2 = s.w3 = s.w4 = s.dh1 = s.dh2 = s.dh3 = s.dh4 = s.dw1 = s.dw2 = s.dw3 = s.dw4 = 0.f;
  s.i1 = s.i2 = s.i3 = s.i4 = 0;
  if (!s.inside) return s;
  const float hlf = floorf(h_im), wlf = floorf(w_im);
  const float lh = h_im - hlf, lw = w_im - wlf, hh = 1.f - lh, hw = 1.f - lw;
  const int hl = static_cast<int>(hlf), wl = static_cast<int>(wlf), hi = hl + 1, wi = wl + 1;
  const bool tp = hl >= 0, bt = hi <= H - 1, lf = wl >= 0, rt = wi <= W - 1;
  const int hlc = max(hl, 0), hic = min(hi, H - 1), wlc = max(wl, 0), wic = min(wi, W - 1);
  s.i1 = hlc * W + wlc; s.i2 = hlc * W + wic; s.i3 = hic * W + wlc; s.i4 = hic * W + wic;
  if (tp && lf) { s.w1 = hh * hw; s.dh1 = -hw; s.dw1 = -hh; }
  if (tp && rt) { s.w2 = hh * lw; s.dh2 = -lw; s.dw2 = hh; }
  if (bt && lf) { s.w3 = lh * hw; s.dh3 = hw; s.dw3 = -lh; }
  if (bt && rt) { s.w4 = lh * lw; s.dh4 = lw; s.dw4 = lh; }
  return s;
}
// sampling position of output pixel `pix` under tap `tap` for deformable group `grp` of image b
__device__ __forceinline__ void dcn_pos(const DcnGeom& g, const float* __restrict__ off, int b, int grp, int tap,
                                        long long pix, float& h_im, float& w_im) {
  const int taps = g.kh * g.kw;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo;
  const int oy = static_cast<int>(pix / g.Wo), ox = static_cast<int>(pix - static_cast<long long>(oy) * g.Wo);
  const int ki = tap / g.kw, kj = tap - ki * g.kw;
  const float* offp = off + (static_cast<long long>(b) * g.dg + grp) * 2 * taps * HoWo;
  h_im = static_cast<float>(oy * g.sh - g.ph + ki * g.dh) + __ldg(offp + (2 * tap) * HoWo + pix);
  w_im = static_cast<float>(ox * g.sw - g.pw + kj * g.dw) + __ldg(offp + (2 * tap + 1) * HoWo + pix);
}

constexpr int TM = 64, TN = 64, TK = 16;     // CTA tile; 256 threads, 4 x 4 outputs each
#define MF_FMA_TILE(As, Bs, acc)                                             \
  _Pragma("unroll") for (int kk = 0; kk < TK; ++kk) {                        \
    float a[4], bq[4];                                                       \
    _Pragma("unroll") for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i]; \
    _Pragma("unroll") for (int j = 0; j < 4; ++j) bq[j] = Bs[kk][tx * 4 + j];\
    _Pragma("unroll") for (int i = 0; i < 4; ++i)                            \
      _Pragma("unroll") for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * bq[j]; \
  }

// ------------------------------------------------------------------------------------------------ forward
// y[b, o, p] = bias[o] + sum_{c, tap} W[o, c, tap] * mask[b, tap, p] * bilinear(x[b, c], p, tap)
// grid (ceil(HoWo / 64), ceil(Co / 64), B); rows of the tile = output channels, columns = pixels
__global__ void __launch_bounds__(256) dcn_f32_forward_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                                              const float* __restrict__ bias, const float* __restrict__ off,
                                                              const float* __restrict__ mask, float* __restrict__ y,
                                                              const DcnGeom g) {
  __shared__ float As[TK][TM + 4];           // W tile   [k = channel][o]
  __shared__ float Bs[TK][TN + 4];           // columns  [k = channel][pixel]
  __shared__ float4 rw[TN];                  // record of (pixel, current tap): corner weights x mask
  __shared__ int4 ri[TN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, o0 = blockIdx.y * TM;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo, p0 = static_cast<long long>(blockIdx.x) * TN;
  const int taps = g.kh * g.kw, cpg = g.C / g.dg;
  const long long HW = static_cast<long long>(g.H) * g.W;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int grp = 0; grp < g.dg; ++grp) {
    for (int tap = 0; tap < taps; ++tap) {
      __syncthreads();                       // previous tap's records are no longer read
      if (tid < TN) {
        float4 rwv = make_float4(0.f, 0.f, 0.f, 0.f);
        int4 riv = make_int4(0, 0, 0, 0);
        const long long pix = p0 + tid;
        if (pix < HoWo) {
          float h_im, w_im;
          dcn_pos(g, off, b, grp, tap, pix, h_im, w_im);
          const DcnSample s = dcn_sample(g.H, g.W, h_im, w_im);
          if (s.inside) {
            const float mk = __ldg(mask + ((static_cast<long long>(b) * g.dg + grp) * taps + tap) * HoWo + pix);
            rwv = make_float4(s.w1 * mk, s.w2 * mk, s.w3 * mk, s.w4 * mk);
            riv = make_int4(s.i1, s.i2, s.i3, s.i4);
          }
        }
        rw[tid] = rwv; ri[tid] = riv;
      }
      __syncthreads();
      for (int c0 = grp * cpg; c0 < (grp + 1) * cpg; c0 += TK) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {        // 16 x 64 entries of each operand tile, 4 per thread
          const int idx = tid + e * 256, kk = idx >> 6, col = idx & 63;
          const int c = c0 + kk;
          const bool cok = c < (grp + 1) * cpg;
          const int o = o0 + col;
          As[kk][col] = (cok && o < g.Co) ? __ldg(w + (static_cast<long long>(o) * g.C + c) * taps + tap) : 0.f;
          float v = 0.f;
          if (cok) {
            const float4 q = rw[col];
            const int4 ix = ri[col];
            const float* xp = x + (static_cast<long long>(b) * g.C + c) * HW;
            v = q.x * __ldg(xp + ix.x) + q.y * __ldg(xp + ix.y) + q.z * __ldg(xp + ix.z) + q.w * __ldg(xp + ix.w);
          }
          Bs[kk][col] = v;
        }
        __syncthreads();
        MF_FMA_TILE(As, Bs, acc)
        __syncthreads();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int o = o0 + ty * 4 + i;
    if (o >= g.Co) continue;
    const float bo = bias[o];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long pix = p0 + tx * 4 + j;
      if (pix < HoWo) y[(static_cast<long long>(b) * g.Co + o) * HoWo + pix] = acc[i][j] + bo;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward k1: grad columns
// gcol[b, m, p] = sum_o W[o, m] dY[b, o, p],  m = c*taps + tap (W viewed as [Co, C*taps]).  grid (ceil(HoWo/64), ceil(CT/64), B)
__global__ void __launch_bounds__(256) dcn_f32_gcol_kernel(const float* __restrict__ w, const float* __restrict__ dy,
                                                           float* __restrict__ gcol, const DcnGeom g) {
  __shared__ float As[TK][TM + 4];           // [k = o][m]
  __shared__ float Bs[TK][TN + 4];           // [k = o][pixel]
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int b = blockIdx.z, m0 = blockIdx.y * TM;
  const int CT = g.C * g.kh * g.kw;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo, p0 = static_cast<long long>(blockIdx.x) * TN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int k0 = 0; k0 < g.Co; k0 += TK) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int idx = tid + e * 256, kk = idx >> 6, col = idx & 63;
      const int o = k0 + kk;
      const int m = m0 + col;
      const long long pix = p0 + col;
      As[kk][col] = (o < g.Co && m < CT) ? __ldg(w + static_cast<long long>(o) * CT + m) : 0.f;
      Bs[kk][col] = (o < g.Co && pix < HoWo) ? __ldg(dy + (static_cast<long long>(b) * g.Co + o) * HoWo + pix) : 0.f;
    }
    __syncthreads();
    MF_FMA_TILE(As, Bs, acc)
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= CT) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const long long pix = p0 + tx * 4 + j;
      if (pix < HoWo) gcol[(static_cast<long long>(b) * CT + m) * HoWo + pix] = acc[i][j];
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward k2: col2im + coord
// one thread per (b, group, tap, pixel): loops over the group's channels
__global__ void __launch_bounds__(256) dcn_f32_col2im_kernel(const float* __restrict__ x, const float* __restrict__ off,
                                                             const float* __restrict__ mask, const float* __restrict__ gcol,
                                                             float* __restrict__ gx, float* __restrict__ goff,
                                                             float* __restrict__ gmask, const DcnGeom g) {
  const int taps = g.kh * g.kw, cpg = g.C / g.dg;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo;
  const long long total = static_cast<long long>(g.B) * g.dg * taps * HoWo;
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long pix = i % HoWo;
  long long t = i / HoWo;
  const int tap = static_cast<int>(t % taps);
  t /= taps;
  const int grp = static_cast<int>(t % g.dg);
  const int b = static_cast<int>(t / g.dg);
  float h_im, w_im;
  dcn_pos(g, off, b, grp, tap, pix, h_im, w_im);
  const DcnSample s = dcn_sample(g.H, g.W, h_im, w_im);
  const long long om = (static_cast<long long>(b) * g.dg + grp) * taps;
  float s_h = 0.f, s_w = 0.f, s_m = 0.f;
  if (s.inside) {
    const float mk = __ldg(mask + (om + tap) * HoWo + pix);
    const long long HW = static_cast<long long>(g.H) * g.W;
    const int CT = g.C * taps;
    for (int c = grp * cpg; c < (grp + 1) * cpg; ++c) {
      const float gc = __ldg(gcol + (static_cast<long long>(b) * CT + c * taps + tap) * HoWo + pix);
      const float* xp = x + (static_cast<long long>(b) * g.C + c) * HW;
      float* gxp = gx + (static_cast<long long>(b) * g.C + c) * HW;
      const float v1 = __ldg(xp + s.i1), v2 = __ldg(xp + s.i2), v3 = __ldg(xp + s.i3), v4 = __ldg(xp + s.i4);
      const float gm = gc * mk;
      if (s.w1 != 0.f) atomicAdd(gxp + s.i1, gm * s.w1);
      if (s.w2 != 0.f) atomicAdd(gxp + s.i2, gm * s.w2);
      if (s.w3 != 0.f) atomicAdd(gxp + s.i3, gm * s.w3);
      if (s.w4 != 0.f) atomicAdd(gxp + s.i4, gm * s.w4);
      s_h += gm * (s.dh1 * v1 + s.dh2 * v2 + s.dh3 * v3 + s.dh4 * v4);
      s_w += gm * (s.dw1 * v1 + s.dw2 * v2 + s.dw3 * v3 + s.dw4 * v4);
      s_m += gc * (s.w1 * v1 + s.w2 * v2 + s.w3 * v3 + s.w4 * v4);
    }
  }
  goff[(om * 2 + 2 * tap) * HoWo + pix] = s_h;
  goff[(om * 2 + 2 * tap + 1) * HoWo + pix] = s_w;
  gmask[(om + tap) * HoWo + pix] = s_m;
}

// ------------------------------------------------------------------------------------------------ backward k3: weight gradient
// part[s, o, c*taps + tap] = sum over split s of (b, p):  dY[b, o, p] * mask * bilinear(x[b, c], p, tap)
// grid (n_tiles = dg * taps * ceil(cpg / 64), ceil(Co / 64), S). Tile rows = o, columns = 64 channels of ONE (group, tap),
// k = pixels (16 per step); the pixel chunks of all images are dealt round-robin to the S splits.
__global__ void __launch_bounds__(256) dcn_f32_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ off,
                                                            const float* __restrict__ mask, const float* __restrict__ dy,
                                                            float* __restrict__ part, const DcnGeom g, int S) {
  __shared__ float As[TK][TM + 4];           // [k = pixel][o]
  __shared__ float Bs[TK][TN + 4];           // [k = pixel][channel]
  __shared__ float4 rw[TK];
  __shared__ int4 ri[TK];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int taps = g.kh * g.kw, cpg = g.C / g.dg, ctiles = (cpg + TN - 1) / TN;
  int nt = blockIdx.x;
  const int ct = nt % ctiles; nt /= ctiles;
  const int tap = nt % taps;
  const int grp = nt / taps;
  const int c0 = grp * cpg + ct * TN, c_end = (grp + 1) * cpg;
  const int o0 = blockIdx.y * TM;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo, HW = static_cast<long long>(g.H) * g.W;
  const long long chunks_per_img = (HoWo + TK - 1) / TK, nchunks = chunks_per_img * g.B;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long ch = blockIdx.z; ch < nchunks; ch += S) {
    const int b = static_cast<int>(ch / chunks_per_img);
    const long long p0 = (ch - static_cast<long long>(b) * chunks_per_img) * TK;
    __syncthreads();
    if (tid < TK) {
      float4 rwv = make_float4(0.f, 0.f, 0.f, 0.f);
      int4 riv = make_int4(0, 0, 0, 0);
      const long long pix = p0 + tid;
      if (pix < HoWo) {
        float h_im, w_im;
        dcn_pos(g, off, b, grp, tap, pix, h_im, w_im);
        const DcnSample s = dcn_sample(g.H, g.W, h_im, w_im);
        if (s.inside) {
          const float mk = __ldg(mask + ((static_cast<long long>(b) * g.dg + grp) * taps + tap) * HoWo + pix);
          rwv = make_float4(s.w1 * mk, s.w2 * mk, s.w3 * mk, s.w4 * mk);
          riv = make_int4(s.i1, s.i2, s.i3, s.i4);
        }
      }
      rw[tid] = rwv; ri[tid] = riv;
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // A: pixel fastest (dY rows are contiguous along pixels); B: pixel fastest too (neighbouring samples, same plane)
      const int idx = tid + e * 256, kk = idx & 15, col = idx >> 4;
      const long long pix = p0 + kk;
      const int o = o0 + col, c = c0 + col;
      As[kk][col] = (pix < HoWo && o < g.Co) ? __ldg(dy + (static_cast<long long>(b) * g.Co + o) * HoWo + pix) : 0.f;
      float v = 0.f;
      if (c < c_end) {
        const float4 q = rw[kk];
        const int4 ix = ri[kk];
        const float* xp = x + (static_cast<long long>(b) * g.C + c) * HW;
        v = q.x * __ldg(xp + ix.x) + q.y * __ldg(xp + ix.y) + q.z * __ldg(xp + ix.z) + q.w * __ldg(xp + ix.w);
      }
      Bs[kk][col] = v;
    }
    __syncthreads();
    MF_FMA_TILE(As, Bs, acc)
  }
  const int CT = g.C * taps;
  float* dst = part + static_cast<long long>(blockIdx.z) * g.Co * CT;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int o = o0 + ty * 4 + i;
    if (o >= g.Co) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tx * 4 + j;
      if (c < c_end) dst[static_cast<long long>(o) * CT + c * taps + tap] = acc[i][j];
    }
  }
}
__global__ void dcn_f32_wgrad_reduce_kernel(const float* __restrict__ part, float* __restrict__ gw, long long n, int S) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float s = 0.f;
  for (int k = 0; k < S; ++k) s += part[static_cast<long long>(k) * n + i];       // fixed order: deterministic
  gw[i] = s;
}

// ------------------------------------------------------------------------------------------------ backward k4: bias gradient
__global__ void __launch_bounds__(256) dcn_f32_bias_grad_kernel(const float* __restrict__ dy, float* __restrict__ gb, int B,
                                                                int Co, long long HoWo) {
  const int o = blockIdx.x;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const float* p = dy + (static_cast<long long>(b) * Co + o) * HoWo;
    for (long long i = threadIdx.x; i < HoWo; i += blockDim.x) acc += __ldg(p + i);
  }
  __shared__ float sm[8];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < 8; ++k) s += sm[k];
    gb[o] = s;
  }
}

// ------------------------------------------------------------------------------------------------ launchers
static int make_geom(DcnGeom& g, int B, int C, int H, int W, int Co, int kh, int kw, int sh, int sw, int ph, int pw, int dh,
                     int dw, int dg, const char* who) {
  if (dg < 1 || C % dg != 0) { set_error("%s: channels %d not divisible by deformable_group %d", who, C, dg); return -1; }
  if (B < 1 || C < 1 || Co < 1 || kh < 1 || kw < 1 || sh < 1 || sw < 1 || dh < 1 || dw < 1) {
    set_error("%s: bad geometry", who);
    return -1;
  }
  g.B = B; g.C = C; g.H = H; g.W = W; g.Co = Co; g.kh = kh; g.kw = kw; g.sh = sh; g.sw = sw; g.ph = ph; g.pw = pw;
  g.dh = dh; g.dw = dw; g.dg = dg;
  g.Ho = (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1;
  g.Wo = (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1;
  if (g.Ho < 1 || g.Wo < 1) { set_error("%s: empty output", who); return -1; }
  return 0;
}
static int wgrad_splits(const DcnGeom& g) {
  const int taps = g.kh * g.kw, cpg = g.C / g.dg;
  const long long tiles = static_cast<long long>(g.dg) * taps * ((cpg + TN - 1) / TN) * ((g.Co + TM - 1) / TM);
  long long S = (132LL * 4 + tiles - 1) / tiles;
  const long long nchunks = ((static_cast<long long>(g.Ho) * g.Wo + TK - 1) / TK) * g.B;
  if (S > nchunks) S = nchunks;
  if (S > 64) S = 64;
  if (S < 1) S = 1;
  return static_cast<int>(S);
}

int launch_dcn_v2_forward_f32(const float* x, const float* w, const float* bias, const float* off, const float* mask,
                              float* y, int B, int Cin, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph,
                              int pw, int dh, int dw, int dg, cudaStream_t st) {
  DcnGeom g;
  if (make_geom(g, B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, "mf_dcn_v2_forward")) return -1;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo;
  dim3 grid(static_cast<unsigned>((HoWo + TN - 1) / TN), static_cast<unsigned>((Cout + TM - 1) / TM), static_cast<unsigned>(B));
  dcn_f32_forward_kernel<<<grid, 256, 0, st>>>(x, w, bias, off, mask, y, g);
  return check_cuda(cudaGetLastError(), "dcn_v2_forward_f32");
}

size_t dcn_v2_backward_f32_workspace(int B, int Cin, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                                     int dh, int dw, int dg) {
  DcnGeom g;
  if (make_geom(g, B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, "mf_dcn_v2_backward_workspace")) return 0;
  const size_t CT = static_cast<size_t>(Cin) * kh * kw, HoWo = static_cast<size_t>(g.Ho) * g.Wo;
  return sizeof(float) * (static_cast<size_t>(B) * CT * HoWo + static_cast<size_t>(wgrad_splits(g)) * Cout * CT);
}

int launch_dcn_v2_backward_f32(const float* x, const float* w, const float* off, const float* mask, const float* dy,
                               float* gx, float* goff, float* gmask, float* gw, float* gb, int B, int Cin, int H, int W,
                               int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int dg,
                               void* workspace, size_t ws_bytes, cudaStream_t st) {
  DcnGeom g;
  if (make_geom(g, B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg, "mf_dcn_v2_backward")) return -1;
  const size_t need = dcn_v2_backward_f32_workspace(B, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, dg);
  if (workspace == nullptr || ws_bytes < need) {
    set_error("mf_dcn_v2_backward: workspace of %zu bytes required (got %zu); query mf_dcn_v2_backward_workspace()", need,
              ws_bytes);
    return -1;
  }
  const int taps = kh * kw, CT = Cin * taps, cpg = Cin / dg;
  const long long HoWo = static_cast<long long>(g.Ho) * g.Wo;
  float* gcol = static_cast<float*>(workspace);
  float* part = gcol + static_cast<long long>(B) * CT * HoWo;
  if (check_cuda(cudaMemsetAsync(gx, 0, sizeof(float) * B * Cin * H * W, st), "memset gx")) return -1;
  dim3 g1(static_cast<unsigned>((HoWo + TN - 1) / TN), static_cast<unsigned>((CT + TM - 1) / TM), static_cast<unsigned>(B));
  dcn_f32_gcol_kernel<<<g1, 256, 0, st>>>(w, dy, gcol, g);
  const long long n2 = static_cast<long long>(B) * dg * taps * HoWo;
  dcn_f32_col2im_kernel<<<static_cast<unsigned>((n2 + 255) / 256), 256, 0, st>>>(x, off, mask, gcol, gx, goff, gmask, g);
  const int S = wgrad_splits(g);
  dim3 g3(static_cast<unsigned>(dg * taps * ((cpg + TN - 1) / TN)), static_cast<unsigned>((Cout + TM - 1) / TM),
          static_cast<unsigned>(S));
  dcn_f32_wgrad_kernel<<<g3, 256, 0, st>>>(x, off, mask, dy, part, g, S);
  const long long nw = static_cast<long long>(Cout) * CT;
  dcn_f32_wgrad_reduce_kernel<<<static_cast<unsigned>((nw + 255) / 256), 256, 0, st>>>(part, gw, nw, S);
  dcn_f32_bias_grad_kernel<<<Cout, 256, 0, st>>>(dy, gb, B, Cout, HoWo);
  return check_cuda(cudaGetLastError(), "dcn_v2_backward_f32");
}

}  // namespace mf
