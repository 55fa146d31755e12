// Training-side HBM kernels (SURVEY §8 rows R11 backward, R13).
//
//  * adamw_arena_dyn_kernel: torch.optim.AdamW over ONE flat parameter / gradient / moment arena. The reference builds one
//    param group per tensor (solver/__init__.py:10-24, lr = BASE_LR or BASE_LR * BIAS_LR_FACTOR when "bias" is in the
//    name) => ~280 groups and ~1000 tiny kernels per step in eager torch; here each tensor is padded to a multiple of
//    ADAMW_CHUNK elements inside the arena and a per-chunk lr table selects the group's lr, so the update is one
//    launch that streams 28 B/parameter (read p, g, m, v; write p, m, v).
//    The same update also runs torch.optim.Adam (coupled L2 weight decay, the reference's SOLVER.OPTIMIZER 'adam') and the
//    fastai one-cycle Adam ('adam_onecycle') through its rule template; the hyper-parameters a schedule moves (lr
//    multiplier, beta1, weight decay) come from a device block the host rewrites in place between captured replays.
//  * focal_loss_backward_kernel: d/dpred of FocalLoss.forward (model/layers/focal_loss.py:35-55) scaled by a device
//    scalar (loss weight / clamp(num_pos, 1), detector_loss.py:276).
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"

#define MF_MAX_PEERS 16
#define MF_ADAMW_CHUNK 512   /* arena granularity (elements) of the per-chunk lr table */
#define MF_UNSCALE_MAX_TENSORS 1024   /* (dst, src, n) triples of one mf_unscale_accumulate launch (by-value kernel params) */

namespace mf {

// ---------------------------------------------------------------- AdamW (torch/optim/adamw.py single-tensor semantics)
//   p   <- p * (1 - lr * wd)
//   m   <- m + (g - m) * (1 - beta1)                (torch: exp_avg.lerp_(grad, 1 - beta1))
//   v   <- v * beta2 + (1 - beta2) * g * g          (torch: exp_avg_sq.mul_(beta2).addcmul_(g, g, value = 1 - beta2))
//   p   <- p - (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// g is first multiplied by grad_scale (1 / world_size when the arena holds an NCCL SUM; 1 otherwise).
// torch.optim.Adam (torch/optim/adam.py single-tensor semantics, RULE = MF_OPTIM_ADAM) differs only in the weight decay:
//   g   <- g + wd * p                                (coupled L2: torch's grad.add(param, alpha=weight_decay)), no p decay
struct AdamwConsts {
  float beta1, beta2, eps, wd, bc1, rsqrt_bc2, grad_scale, lr_scale;
};
template <int RULE = MF_OPTIM_ADAMW>
__device__ __forceinline__ void adamw_update4(float4& pp, const float4& gg, float4& mm, float4& vv, float lr,
                                              const AdamwConsts& k) {
  const float omb1 = 1.f - k.beta1, omb2 = 1.f - k.beta2;
  const float decay = 1.f - lr * k.wd, step = lr / k.bc1;
  float* pe = reinterpret_cast<float*>(&pp);
  float* me = reinterpret_cast<float*>(&mm);
  float* ve = reinterpret_cast<float*>(&vv);
  const float* ge = reinterpret_cast<const float*>(&gg);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float gk, pk;
    if (RULE == MF_OPTIM_ADAMW) {
      gk = ge[e] * k.grad_scale;
      pk = pe[e] * decay;
    } else {
      pk = pe[e];
      gk = ge[e] * k.grad_scale + k.wd * pk;
    }
    const float mk = me[e] + (gk - me[e]) * omb1;
    const float vk = ve[e] * k.beta2 + omb2 * gk * gk;
    const float denom = sqrtf(vk) * k.rsqrt_bc2 + k.eps;
    pk -= step * (mk / denom);
    pe[e] = pk; me[e] = mk; ve[e] = vk;
  }
}

// ---------------------------------------------------------------- gradient exchange fused with the update (row R13, N > 1)
// DDP's allreduce + optimizer.step (tools/plain_train_net.py:100-104, engine/trainer.py:116-121) as ONE kernel over peer
// memory: every rank owns a contiguous 1/world shard of the arena's chunks. For its shard it
//   1. reduces the gradient of all ranks - either `multimem.ld_reduce` on the NVLS multicast address (the NVSwitch adds
//      the world copies in the fabric, one 16-byte request per float4) or a fixed-order sum of peer loads over NVLink;
//   2. applies AdamW with ITS shard of the moments (the optimizer state is only ever touched by the owner: ZeRO-1);
//   3. writes the new parameters into EVERY rank's parameter arena (`multimem.st` broadcast or peer stores).
// Per rank and step that is 1/world of (world x 4 + 12) bytes per parameter read and world x 4 + 8 written, against NCCL
// allreduce (2 x 4 x (world-1)/world over NVLink + 8 B HBM) followed by the 28 B/parameter update; the two system-scope
// barriers around the kernel are the only other synchronisation. Each element is produced by exactly one rank with a
// rank-independent summation order, so all replicas stay bit-identical.
struct PeerPtrs {
  float* p[MF_MAX_PEERS];
  const float* g[MF_MAX_PEERS];
};
__device__ __forceinline__ float4 multimem_ld_reduce_add(const float* addr) {
  float4 r;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(addr) : "memory");
  return r;
}
__device__ __forceinline__ void multimem_st(float* addr, const float4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1, %2, %3, %4};"
               :: "l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__global__ void __launch_bounds__(256) adamw_p2p_kernel(PeerPtrs peers, int world, int rank, float* mc_p, const float* mc_g,
                                                        float* __restrict__ m, float* __restrict__ v,
                                                        const float* __restrict__ chunk_lr, long long chunk_lo,
                                                        long long chunk_hi, AdamwConsts k) {
  constexpr int VEC_PER_CHUNK = MF_ADAMW_CHUNK / 4;
  const long long v_lo = chunk_lo * VEC_PER_CHUNK, v_hi = chunk_hi * VEC_PER_CHUNK;
  for (long long i = v_lo + static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < v_hi;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float lr = __ldg(chunk_lr + i / VEC_PER_CHUNK) * k.lr_scale;
    if (lr == 0.f) continue;
    float4 gg;
    if (mc_g != nullptr) {
      gg = multimem_ld_reduce_add(mc_g + 4 * i);
    } else {
      gg = __ldcg(reinterpret_cast<const float4*>(peers.g[0]) + i);
      for (int r = 1; r < world; ++r) {
        const float4 t = __ldcg(reinterpret_cast<const float4*>(peers.g[r]) + i);
        gg.x += t.x; gg.y += t.y; gg.z += t.z; gg.w += t.w;
      }
    }
    float4 pp = reinterpret_cast<const float4*>(peers.p[rank])[i];
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    adamw_update4(pp, gg, mm, vv, lr, k);
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
    if (mc_p != nullptr) {
      multimem_st(mc_p + 4 * i, pp);
    } else {
      for (int r = 0; r < world; ++r) reinterpret_cast<float4*>(peers.p[r])[i] = pp;
    }
  }
}

static AdamwConsts adamw_consts(double beta1, float beta2, float eps, float wd, long long step, float grad_scale,
                                float lr_scale) {
  // bias corrections in double like torch's Python scalars (beta1 is the Python double itself, as in the hyper block)
  const double bc1 = 1.0 - pow(beta1, static_cast<double>(step));
  const double bc2 = 1.0 - pow(static_cast<double>(beta2), static_cast<double>(step));
  AdamwConsts k;
  k.beta1 = static_cast<float>(beta1); k.beta2 = beta2; k.eps = eps; k.wd = wd;
  k.bc1 = static_cast<float>(bc1); k.rsqrt_bc2 = static_cast<float>(1.0 / sqrt(bc2));
  k.grad_scale = grad_scale; k.lr_scale = lr_scale;
  return k;
}

// ---------------------------------------------------------------- CUDA-graph-safe optimiser step with a finite guard
// The step count (for the bias corrections) lives on the device, so a captured graph does not freeze it, and the
// hyper-parameters a schedule moves are read from the device block hyper = double[4] {lr_mult, beta1, weight_decay,
// unused}, which the host rewrites in place between launches / replays. Three launches make one optimiser step:
//   1. grad_finite_kernel : state[1] |= any non-finite element in the gradient arena (fp16 gradient flow under a loss
//                           scale can overflow; one inf written by the update poisons params, exp_avg and exp_avg_sq for
//                           good);
//   2. adamw_prepare_kernel (1 thread): if the flag is clean, step += 1 and the bias corrections of the new step are
//                           computed in double from beta1 = hyper[1] (torch computes them in Python doubles); else the
//                           step is skipped (state[2] += 1). Either way it publishes (bc1, rsqrt_bc2, skip) and clears
//                           the flag;
//   3. adamw_arena_dyn_kernel: the arena update, reading those three values from device memory.
// state = long long[4]: [0] step count, [1] found-non-finite flag of the current step, [2] skipped steps, [3] unused.
//
// With gradient-norm clipping (max_norm > 0; torch.nn.utils.clip_grad_norm_ between backward and step, the reference's
// SOLVER.GRAD_NORM_CLIP, engine/trainer.py:119) the same three launches become:
//   1. grad_sumsq_kernel  : each CTA writes the float64 sum of squares of its fixed grid-stride share of the arena to
//                           partials[blockIdx.x] (the grid depends on n_chunks only, so the norm is run-to-run identical);
//   2. adamw_prepare_clip_kernel (1 CTA): reduces the partials in a fixed order, total_norm = float(sqrt(sum) * grad_scale)
//                           (the norm of the gradient the update uses: with an NCCL SUM in the arena, of the rank mean) and
//                           clip_coef = min(reciprocal(total_norm + 1e-6) * max_norm, 1) in torch's float32 steps
//                           (_clip_grads_with_norm_; `scalar / tensor` is `reciprocal() * scalar`). A norm that is not
//                           finite is the finite guard's skip; otherwise the step bookkeeping above;
//   3. adamw_arena_dyn_kernel<true>: g <- g * clip_coef, written back to the arena when clip_coef != 1 (p.grad then holds what
//                           clip_grad_norm_ leaves there; torch's multiply by exactly 1 is exact, so nothing is written),
//                           then the update as above.
struct AdamwDyn { float bc1, rsqrt_bc2; int skip; float clip_coef; };

__device__ __forceinline__ void adamw_prepare_step(long long* state, AdamwDyn* dyn, double beta1, float beta2, bool skip) {
  if (skip) state[2] += 1; else state[0] += 1;
  state[1] = 0;
  const double step = static_cast<double>(state[0] < 1 ? 1 : state[0]);
  const double bc1 = 1.0 - pow(beta1, step);
  const double bc2 = 1.0 - pow(static_cast<double>(beta2), step);
  dyn->bc1 = static_cast<float>(bc1);
  dyn->rsqrt_bc2 = static_cast<float>(1.0 / sqrt(bc2));
  dyn->skip = skip ? 1 : 0;
}

// sum over a 256-thread CTA in a fixed order (butterfly within each warp, then the 8 warp sums in order); valid in thread 0
__device__ __forceinline__ double block_sum_256(double s, double* red8) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
  if ((threadIdx.x & 31) == 0) red8[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    s = red8[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) s += red8[w];
  }
  return s;
}

__global__ void __launch_bounds__(256) grad_sumsq_kernel(const float* __restrict__ g, long long n_vec, double* __restrict__ partials) {
  __shared__ double red[8];
  double s = 0.0;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    const double x = v.x, y = v.y, z = v.z, w = v.w;
    s += x * x + y * y + z * z + w * w;
  }
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

__global__ void __launch_bounds__(256) adamw_prepare_clip_kernel(long long* state, AdamwDyn* dyn, float beta2,
                                                                 const double* __restrict__ partials, int n_partials,
                                                                 float grad_scale, float max_norm, float* total_norm_out,
                                                                 const double* __restrict__ hyper) {
  __shared__ double red[8];
  double s = 0.0;
  for (int i = threadIdx.x; i < n_partials; i += 256) s += partials[i];
  s = block_sum_256(s, red);
  if (threadIdx.x != 0) return;
  const float norm = static_cast<float>(sqrt(s) * static_cast<double>(grad_scale));
  *total_norm_out = norm;
  adamw_prepare_step(state, dyn, hyper[1], beta2, !isfinite(norm));
  const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
  dyn->clip_coef = c > 1.f ? 1.f : c;                          // torch.clamp(max=1.0) keeps a NaN
}

__global__ void __launch_bounds__(256) grad_finite_kernel(const float* __restrict__ g, long long n_vec, long long* state) {
  bool bad = false;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(g) + i);
    // x - x is 0 for finite x and NaN for inf / NaN
    const float t = (v.x - v.x) + (v.y - v.y) + (v.z - v.z) + (v.w - v.w);
    bad |= !(t == 0.f);
  }
  if (__syncthreads_or(bad ? 1 : 0) && threadIdx.x == 0) atomicExch(reinterpret_cast<unsigned long long*>(state + 1), 1ull);
}
__global__ void adamw_prepare_kernel(long long* state, AdamwDyn* dyn, float beta2, const double* __restrict__ hyper) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  adamw_prepare_step(state, dyn, hyper[1], beta2, state[1] != 0);
}
// CLIP = false never writes g; chunks with lr 0 (padding-only, mark_unused) are neither updated nor clipped.
// lr = chunk_lr * hyper[0]; beta1 and weight decay are hyper[1] and hyper[2]. A chunk whose lr is negative is decay-only:
// p <- p * (1 - |lr| * wd), no gradient, no moments (fastai's OptimWrapper decays every grouped tensor, torch's Adam then
// skips the ones with grad None).
template <bool CLIP, int RULE>
__global__ void __launch_bounds__(256) adamw_arena_dyn_kernel(float* __restrict__ p, float* __restrict__ g,
                                                              float* __restrict__ m, float* __restrict__ v,
                                                              const float* __restrict__ chunk_lr, long long n_chunks,
                                                              AdamwConsts k, const AdamwDyn* __restrict__ dyn,
                                                              const double* __restrict__ hyper) {
  if (dyn->skip) return;
  k.bc1 = dyn->bc1;
  k.rsqrt_bc2 = dyn->rsqrt_bc2;
  k.lr_scale = static_cast<float>(hyper[0]);
  k.beta1 = static_cast<float>(hyper[1]);
  k.wd = static_cast<float>(hyper[2]);
  const float coef = CLIP ? dyn->clip_coef : 1.f;
  constexpr int VEC_PER_CHUNK = MF_ADAMW_CHUNK / 4;
  const long long n_vec = n_chunks * VEC_PER_CHUNK;
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n_vec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float lr = __ldg(chunk_lr + i / VEC_PER_CHUNK) * k.lr_scale;
    if (lr == 0.f) continue;
    float4 pp = reinterpret_cast<float4*>(p)[i];
    if (lr < 0.f) {
      const float decay = 1.f - (-lr) * k.wd;
      pp.x *= decay; pp.y *= decay; pp.z *= decay; pp.w *= decay;
      reinterpret_cast<float4*>(p)[i] = pp;
      continue;
    }
    float4 gg = __ldcs(reinterpret_cast<const float4*>(g) + i);
    if (CLIP && coef != 1.f) {
      gg.x *= coef; gg.y *= coef; gg.z *= coef; gg.w *= coef;
      __stcs(reinterpret_cast<float4*>(g) + i, gg);
    }
    float4 mm = reinterpret_cast<float4*>(m)[i];
    float4 vv = reinterpret_cast<float4*>(v)[i];
    adamw_update4<RULE>(pp, gg, mm, vv, lr, k);
    reinterpret_cast<float4*>(p)[i] = pp;
    reinterpret_cast<float4*>(m)[i] = mm;
    reinterpret_cast<float4*>(v)[i] = vv;
  }
}
template <bool CLIP>
static void launch_dyn_update(int rule, dim3 grid, cudaStream_t st, float* p, float* g, float* m, float* v,
                              const float* chunk_lr, long long n_chunks, const AdamwConsts& k, const AdamwDyn* dyn,
                              const double* hyper) {
  if (rule == MF_OPTIM_ADAM)
    (void)launch_k(adamw_arena_dyn_kernel<CLIP, MF_OPTIM_ADAM>, grid, dim3(256), 0, st, p, g, m, v, chunk_lr, n_chunks, k,
                   dyn, hyper);
  else
    (void)launch_k(adamw_arena_dyn_kernel<CLIP, MF_OPTIM_ADAMW>, grid, dim3(256), 0, st, p, g, m, v, chunk_lr, n_chunks, k,
                   dyn, hyper);
}
// ---------------------------------------------------------------- dynamic loss scale (torch.amp.GradScaler's rule)
// The scale is device state (float scale, int growth_tracker), so a captured training step reads and updates it without
// the host. Two kernels:
//   * unscale_accumulate_kernel: dst_i += src_i * inv_scale over a list of (dst, src, n) triples in ONE launch (the
//     backward tape's ~280 parameter gradients into p.grad), inv_scale = float(1.0 / double(scale)) - GradScaler's
//     scale.double().reciprocal().float(). The product-add is one fma like torch._foreach_add_(dst, src, alpha) (exact
//     for a power-of-two scale either way). A triple flagged `assign` is dst_i = src_i * inv_scale (p.grad None).
//   * loss_scale_update_kernel (1 thread): torch._amp_update_scale_ on the skip flag the optimiser's prepare kernel
//     published in AdamwDyn (a non-finite gradient arena or clipping norm): backoff on a skip, growth after
//     growth_interval clean steps unless the grown scale is not finite.
struct UnscaleList {
  const float* src[MF_UNSCALE_MAX_TENSORS];
  float* dst[MF_UNSCALE_MAX_TENSORS];
  int n[MF_UNSCALE_MAX_TENSORS];
  int tile0[MF_UNSCALE_MAX_TENSORS + 1];       // first tile of tensor i; tile0[count] = the grid
  unsigned char assign[MF_UNSCALE_MAX_TENSORS];
  int count;
};
constexpr int UNSCALE_TILE = 4096;              // elements per CTA: 256 threads x 4 float4

__global__ void __launch_bounds__(256) unscale_accumulate_kernel(const __grid_constant__ UnscaleList L,
                                                                 const float* __restrict__ scale) {
  const float inv = static_cast<float>(1.0 / static_cast<double>(__ldg(scale)));
  const int tile = blockIdx.x;
  int lo = 0, hi = L.count - 1;                 // the tensor whose tiles cover this CTA: largest i with tile0[i] <= tile
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (L.tile0[mid] <= tile) lo = mid; else hi = mid - 1;
  }
  const int t = lo;
  const long long base = static_cast<long long>(tile - L.tile0[t]) * UNSCALE_TILE;
  const int n = L.n[t];
  const float* __restrict__ src = L.src[t];
  float* __restrict__ dst = L.dst[t];
  const bool assign = L.assign[t] != 0;
  const int end = static_cast<int>(min(static_cast<long long>(n), base + UNSCALE_TILE));
  const bool vec = ((reinterpret_cast<unsigned long long>(src) | reinterpret_cast<unsigned long long>(dst)) & 15) == 0;
  if (vec) {
    const int v_end = end & ~3;
    for (int i = static_cast<int>(base) + 4 * threadIdx.x; i < v_end; i += 4 * 256) {
      const float4 s = __ldcs(reinterpret_cast<const float4*>(src + i));
      float4 d;
      if (assign) {
        d.x = s.x * inv; d.y = s.y * inv; d.z = s.z * inv; d.w = s.w * inv;
      } else {
        d = *reinterpret_cast<const float4*>(dst + i);
        d.x = __fmaf_rn(s.x, inv, d.x); d.y = __fmaf_rn(s.y, inv, d.y);
        d.z = __fmaf_rn(s.z, inv, d.z); d.w = __fmaf_rn(s.w, inv, d.w);
      }
      *reinterpret_cast<float4*>(dst + i) = d;
    }
    for (int i = v_end + threadIdx.x; i < end; i += 256)
      dst[i] = assign ? src[i] * inv : __fmaf_rn(src[i], inv, dst[i]);
  } else {
    for (int i = static_cast<int>(base) + threadIdx.x; i < end; i += 256)
      dst[i] = assign ? src[i] * inv : __fmaf_rn(src[i], inv, dst[i]);
  }
}

__global__ void loss_scale_update_kernel(const AdamwDyn* __restrict__ dyn, float* scale, int* growth_tracker,
                                         double growth_factor, double backoff_factor, int growth_interval) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (dyn->skip) {
    *scale = static_cast<float>(static_cast<double>(*scale) * backoff_factor);
    *growth_tracker = 0;
  } else {
    const int successful = *growth_tracker + 1;
    if (successful == growth_interval) {
      const float grown = static_cast<float>(static_cast<double>(*scale) * growth_factor);
      if (isfinite(grown)) *scale = grown;            // never grow past float32's range to inf
      *growth_tracker = 0;
    } else {
      *growth_tracker = successful;
    }
  }
}

// ---------------------------------------------------------------- focal loss backward (layers/focal_loss.py:35-55)
// L = -sum_{t==1} log(p)(1-p)^2 - sum_{0<=t<1} log(1-p) p^2 (1-t)^4
// dL/dp = -( (1-p)^2 / p - 2 (1-p) log p )                          at t == 1
//       = -(1-t)^4 ( 2 p log(1-p) - p^2 / (1-p) )                   at 0 <= t < 1,   0 elsewhere (ignored pixels, t = -1)
__global__ void focal_loss_backward_kernel(const float* __restrict__ pred, const float* __restrict__ tgt, long long n,
                                           const float* __restrict__ scale, float* __restrict__ grad) {
  const float s = __ldg(scale);
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float p = __ldg(pred + i), t = __ldg(tgt + i);
    float d = 0.f;
    if (t == 1.f) {
      const float q = 1.f - p;
      d = -(q * q / p - 2.f * q * logf(p));
    } else if (t < 1.f && t >= 0.f) {
      const float omt = 1.f - t, omt2 = omt * omt;
      d = -omt2 * omt2 * (2.f * p * logf(1.f - p) - p * p / (1.f - p));
    }
    grad[i] = d * s;
  }
}

int launch_focal_loss_backward(const float* pred, const float* tgt, long long n, const float* scale, float* grad,
                               cudaStream_t st) {
  if (n <= 0) return 0;
  long long blocks = (n + 1023) / 1024;
  if (blocks > 132 * 8) blocks = 132 * 8;
  (void)launch_k(focal_loss_backward_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, st, pred, tgt, n, scale,
                 grad);
  return check_cuda(cudaGetLastError(), "focal_loss_backward");
}

}  // namespace mf

using namespace mf;

extern "C" {

int mf_adamw_chunk(void) { return MF_ADAMW_CHUNK; }
int mf_unscale_max_tensors(void) { return MF_UNSCALE_MAX_TENSORS; }

int mf_adamw_step_p2p(const unsigned long long* param_ptrs, const unsigned long long* grad_ptrs, int world, int rank,
                      unsigned long long mc_params, unsigned long long mc_grads, float* m, float* v, const float* chunk_lr,
                      long long n_chunks, double beta1, float beta2, float eps, float wd, long long step, float lr_scale,
                      void* stream) {
  if (world < 1 || world > MF_MAX_PEERS || rank < 0 || rank >= world) {
    set_error("adamw_p2p: world %d (max %d) / rank %d", world, MF_MAX_PEERS, rank);
    return -1;
  }
  if (step < 1) { set_error("adamw_p2p: step must be >= 1"); return -1; }
  if ((mc_params == 0) != (mc_grads == 0)) { set_error("adamw_p2p: give both multicast addresses or neither"); return -1; }
  PeerPtrs peers;
  for (int r = 0; r < MF_MAX_PEERS; ++r) {
    peers.p[r] = r < world ? reinterpret_cast<float*>(param_ptrs[r]) : nullptr;
    peers.g[r] = r < world ? reinterpret_cast<const float*>(grad_ptrs[r]) : nullptr;
  }
  const long long base = n_chunks / world, extra = n_chunks % world;      // parallel.shard_range semantics
  const long long lo = rank * base + (rank < extra ? rank : extra), hi = lo + base + (rank < extra ? 1 : 0);
  if (hi <= lo) return 0;
  const long long n_vec = (hi - lo) * (MF_ADAMW_CHUNK / 4);
  long long blocks = (n_vec + 255) / 256;
  const long long cap = 132LL * 8 * 4;
  if (blocks > cap) blocks = cap;
  const AdamwConsts k = adamw_consts(beta1, beta2, eps, wd, step, 1.f / static_cast<float>(world), lr_scale);
  adamw_p2p_kernel<<<dim3(static_cast<unsigned>(blocks)), dim3(256), 0, MF_STREAM(stream)>>>(
      peers, world, rank, reinterpret_cast<float*>(mc_params), reinterpret_cast<const float*>(mc_grads), m, v, chunk_lr, lo,
      hi, k);
  return check_cuda(cudaGetLastError(), "adamw_p2p");
}

// max_norm <= 0: no clipping (g is only read; partials and total_norm_out are not used and may be NULL).
// hyper: device double[4] {lr_mult, beta1, weight_decay, unused}, never NULL.
int mf_optim_step_dyn(int rule, float* p, float* g, float* m, float* v, const float* chunk_lr, long long n_chunks,
                      const double* hyper, float beta2, float eps, float grad_scale, long long* state4, void* dyn16,
                      float max_norm, double* partials, float* total_norm_out, void* stream) {
  if (hyper == nullptr) { set_error("mf_optim_step_dyn: hyper (device double[4]) is NULL"); return -1; }
  if (rule != MF_OPTIM_ADAMW && rule != MF_OPTIM_ADAM) {
    set_error("mf_optim_step_dyn: rule %d (0 = AdamW, 1 = Adam with L2 weight decay)", rule);
    return -1;
  }
  if (n_chunks <= 0) return 0;
  const bool clip = max_norm > 0.f;
  if (clip && (partials == nullptr || total_norm_out == nullptr)) {
    set_error("mf_optim_step_dyn: max_norm > 0 needs the partials buffer and total_norm_out");
    return -1;
  }
  const long long n_vec = n_chunks * (MF_ADAMW_CHUNK / 4);
  long long blocks = (n_vec + 255) / 256;                       // <= (n_chunks + 1) / 2: the partials the caller provides
  const long long cap = 132LL * 8 * 4;
  if (blocks > cap) blocks = cap;
  AdamwDyn* dyn = static_cast<AdamwDyn*>(dyn16);
  const cudaStream_t st = MF_STREAM(stream);
  if (clip) {
    (void)launch_k(grad_sumsq_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, st, g, n_vec, partials);
    (void)launch_k(adamw_prepare_clip_kernel, dim3(1), dim3(256), 0, st, state4, dyn, beta2, partials,
                   static_cast<int>(blocks), grad_scale, max_norm, total_norm_out, hyper);
  } else {
    (void)launch_k(grad_finite_kernel, dim3(static_cast<unsigned>(blocks)), dim3(256), 0, st, g, n_vec, state4);
    (void)launch_k(adamw_prepare_kernel, dim3(1), dim3(32), 0, st, state4, dyn, beta2, hyper);
  }
  AdamwConsts k{};                                              // beta1, wd, lr_scale and the bias corrections: on the device
  k.beta2 = beta2; k.eps = eps; k.grad_scale = grad_scale;
  const dim3 grid(static_cast<unsigned>(blocks));
  if (clip)
    launch_dyn_update<true>(rule, grid, st, p, g, m, v, chunk_lr, n_chunks, k, dyn, hyper);
  else
    launch_dyn_update<false>(rule, grid, st, p, g, m, v, chunk_lr, n_chunks, k, dyn, hyper);
  return check_cuda(cudaGetLastError(), "mf_optim_step_dyn");
}

int mf_unscale_accumulate(const unsigned long long* dst_ptrs, const unsigned long long* src_ptrs, const long long* numels,
                          const unsigned char* assign, int count, const float* scale, void* stream) {
  if (count < 0 || count > MF_UNSCALE_MAX_TENSORS) {
    set_error("mf_unscale_accumulate: %d tensors (0 .. %d in one launch)", count, MF_UNSCALE_MAX_TENSORS);
    return -1;
  }
  if (count > 0 && (dst_ptrs == nullptr || src_ptrs == nullptr || numels == nullptr)) {
    set_error("mf_unscale_accumulate: dst_ptrs, src_ptrs and numels are host arrays of count entries, not NULL");
    return -1;
  }
  if (scale == nullptr) { set_error("mf_unscale_accumulate: scale (device float) is NULL"); return -1; }
  UnscaleList L;
  long long tiles = 0;
  int k = 0;
  for (int i = 0; i < count; ++i) {
    if (numels[i] < 0 || numels[i] > 0x7fffffffLL) {
      set_error("mf_unscale_accumulate: tensor %d has %lld elements (0 .. 2^31 - 1)", i, numels[i]);
      return -1;
    }
    if (numels[i] == 0) continue;
    if (dst_ptrs[i] == 0 || src_ptrs[i] == 0) {
      set_error("mf_unscale_accumulate: tensor %d has a NULL dst or src", i);
      return -1;
    }
    L.dst[k] = reinterpret_cast<float*>(dst_ptrs[i]);
    L.src[k] = reinterpret_cast<const float*>(src_ptrs[i]);
    L.n[k] = static_cast<int>(numels[i]);
    L.assign[k] = (assign != nullptr && assign[i]) ? 1 : 0;
    L.tile0[k] = static_cast<int>(tiles);
    tiles += (numels[i] + UNSCALE_TILE - 1) / UNSCALE_TILE;
    ++k;
  }
  if (k == 0) return 0;
  if (tiles > 0x7fffffffLL) { set_error("mf_unscale_accumulate: %lld tiles exceed one grid", tiles); return -1; }
  L.tile0[k] = static_cast<int>(tiles);
  L.count = k;
  (void)launch_k(unscale_accumulate_kernel, dim3(static_cast<unsigned>(tiles)), dim3(256), 0, MF_STREAM(stream), L, scale);
  return check_cuda(cudaGetLastError(), "mf_unscale_accumulate");
}

int mf_loss_scale_update(const void* dyn16, float* scale, int* growth_tracker, double growth_factor, double backoff_factor,
                         int growth_interval, void* stream) {
  if (dyn16 == nullptr || scale == nullptr || growth_tracker == nullptr) {
    set_error("mf_loss_scale_update: dyn16, scale and growth_tracker are device pointers, not NULL");
    return -1;
  }
  if (!(growth_factor > 1.0) || !(backoff_factor > 0.0 && backoff_factor < 1.0) || growth_interval < 1) {
    set_error("mf_loss_scale_update: needs growth_factor > 1, 0 < backoff_factor < 1, growth_interval >= 1 "
              "(got %g, %g, %d)", growth_factor, backoff_factor, growth_interval);
    return -1;
  }
  (void)launch_k(loss_scale_update_kernel, dim3(1), dim3(32), 0, MF_STREAM(stream), static_cast<const AdamwDyn*>(dyn16), scale,
                 growth_tracker, growth_factor, backoff_factor, growth_interval);
  return check_cuda(cudaGetLastError(), "mf_loss_scale_update");
}

int mf_focal_loss_backward(const float* pred, const float* target, long long n, const float* scale, float* grad_pred,
                           void* stream) {
  return launch_focal_loss_backward(pred, target, n, scale, grad_pred, MF_STREAM(stream));
}

}  // extern "C"
