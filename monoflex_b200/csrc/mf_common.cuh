// Common device helpers for the sm_90a kernels of monoflex_b200: mbarrier / cp.async / TMA / wgmma PTX.
// Everything here is hand-written inline PTX (no CUTLASS); compile with -gencode arch=compute_90a,code=sm_90a.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cuda.h>
#include <stdint.h>

#define MF_DEVINL __device__ __forceinline__

namespace mf {

// ------------------------------------------------------------------------------------------------ error state
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

// the C ABI passes the caller's cudaStream_t as void*
#define MF_STREAM(s) reinterpret_cast<cudaStream_t>(s)

// kernel<<<grid, block, smem, st>>>(args...) through cudaLaunchKernelEx, converting each argument to the kernel's parameter type
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = nullptr;
  cfg.numAttrs = 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

MF_DEVINL uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ------------------------------------------------------------------------------------------------ mbarrier
MF_DEVINL void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
MF_DEVINL void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
MF_DEVINL void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
MF_DEVINL void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
MF_DEVINL uint32_t mbar_try_wait(uint32_t addr, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(addr), "r"(parity)
      : "memory");
  return ok;
}
MF_DEVINL void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  while (!mbar_try_wait(addr, parity)) {
  }
}

// generic-proxy smem writes -> visible to the async proxy (wgmma / TMA reads)
MF_DEVINL void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ explicit shared-space ld/st
// (pointers carved out of the dynamic smem block through integer alignment lose their address space: the compiler then
// emits generic LD.E / ST.E with 64-bit address arithmetic; these keep the hot loops on LDS / STS with 32-bit addresses)
MF_DEVINL uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
MF_DEVINL float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
MF_DEVINL float2 lds64f(uint32_t addr) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(addr));
  return v;
}
MF_DEVINL void sts128(uint32_t addr, const uint4& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
MF_DEVINL void sts128f(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
MF_DEVINL void sts32f(uint32_t addr, float v) { asm volatile("st.shared.f32 [%0], %1;" ::"r"(addr), "f"(v) : "memory"); }
MF_DEVINL void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory"); }

// ------------------------------------------------------------------------------------------------ two-lane fp32 math
// (a pair of channels per call; sm_90 has no packed fp32 FMA, so these are two scalar FFMAs with round-to-nearest)
MF_DEVINL float2 f2_mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
MF_DEVINL float2 f2_fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }

// ------------------------------------------------------------------------------------------------ 8 channels of an activation row
// The two storage formats of NHWC activation rows, 8 channels (16 bytes per block) at a time. load() only issues the loads
// and to_f32() converts, so a kernel can issue all its loads before any arithmetic; pack() rounds, store() writes.
// Fp16Rows: one fp16 block. PairRows (strict precision): v = float(hi) + float(lo) with hi = fp16(v), lo = fp16(v - hi),
// the lo block `lo` elements after hi in the same row (`lo` is ignored for fp16 rows).
struct Fp16Rows {
  static constexpr int kBlocks = 1;
  using Raw = uint4;
  MF_DEVINL static Raw load(const __half* p, int) { return __ldg(reinterpret_cast<const uint4*>(p)); }
  MF_DEVINL static Raw zero() { return make_uint4(0u, 0u, 0u, 0u); }
  MF_DEVINL static void to_f32(const Raw& v, float (&f)[8]) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 t = __half22float2(h[e]);
      f[2 * e] = t.x;
      f[2 * e + 1] = t.y;
    }
  }
  MF_DEVINL static Raw pack(const float (&f)[8]) {
    __half2 o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) o[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
    return *reinterpret_cast<uint4*>(o);
  }
  MF_DEVINL static void store(__half* p, int, const Raw& v) { *reinterpret_cast<uint4*>(p) = v; }
  // MaxPool2d on the fp16 values themselves (exact)
  MF_DEVINL static Raw max4(const Raw& a, const Raw& b, const Raw& c, const Raw& d) {
    uint4 o;
    const __half2 *ha = reinterpret_cast<const __half2*>(&a), *hb = reinterpret_cast<const __half2*>(&b);
    const __half2 *hc = reinterpret_cast<const __half2*>(&c), *hd = reinterpret_cast<const __half2*>(&d);
    __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) ho[e] = __hmax2(__hmax2(ha[e], hb[e]), __hmax2(hc[e], hd[e]));
    return o;
  }
};

struct PairRows {
  static constexpr int kBlocks = 2;
  struct Raw { uint4 hi, lo; };
  MF_DEVINL static Raw load(const __half* p, int lo) {
    return {__ldg(reinterpret_cast<const uint4*>(p)), __ldg(reinterpret_cast<const uint4*>(p + lo))};
  }
  MF_DEVINL static Raw zero() { return {make_uint4(0u, 0u, 0u, 0u), make_uint4(0u, 0u, 0u, 0u)}; }
  MF_DEVINL static void to_f32(const Raw& v, float (&f)[8]) {
    const __half2* hh = reinterpret_cast<const __half2*>(&v.hi);
    const __half2* ll = reinterpret_cast<const __half2*>(&v.lo);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 a = __half22float2(hh[e]), b = __half22float2(ll[e]);
      f[2 * e] = a.x + b.x;
      f[2 * e + 1] = a.y + b.y;
    }
  }
  MF_DEVINL static Raw pack(const float (&f)[8]) {
    __half2 h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      h[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
      const float2 hf = __half22float2(h[e]);
      l[e] = __floats2half2_rn(f[2 * e] - hf.x, f[2 * e + 1] - hf.y);
    }
    return {*reinterpret_cast<uint4*>(h), *reinterpret_cast<uint4*>(l)};
  }
  MF_DEVINL static void store(__half* p, int lo, const Raw& v) {
    *reinterpret_cast<uint4*>(p) = v.hi;
    *reinterpret_cast<uint4*>(p + lo) = v.lo;
  }
  // MaxPool2d on the fp32 values; hi + lo of one input is exactly representable again, so the pair max is lossless
  MF_DEVINL static Raw max4(const Raw& a, const Raw& b, const Raw& c, const Raw& d) {
    float fa[8], fb[8], fc[8], fd[8], o[8];
    to_f32(a, fa);
    to_f32(b, fb);
    to_f32(c, fc);
    to_f32(d, fd);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = fmaxf(fmaxf(fa[e], fb[e]), fmaxf(fc[e], fd[e]));
    return pack(o);
  }
};

// ------------------------------------------------------------------------------------------------ edge-fusion sampling point
// F.grid_sample(bilinear, align_corners=True) coordinate of border position e of image b (edge_idx [B, K, 2] = (x, y) on the
// out_w x out_h output map) on an H x W map: the top-left corner (x0, y0) and the bilinear weights, in the reference's fp32
// operation order. The edge gather, its backward and mf_edge_mask all take it from here, so the mask marks exactly the
// pixels the gather reads.
struct EdgeSample {
  int x0, y0;
  float wx0, wx1, wy0, wy1;
};
MF_DEVINL EdgeSample edge_sample(const long long* edge_idx, int b, int K, int e, int H, int W, int out_w, int out_h) {
  const float ex = static_cast<float>(edge_idx[(static_cast<long long>(b) * K + e) * 2 + 0]);
  const float ey = static_cast<float>(edge_idx[(static_cast<long long>(b) * K + e) * 2 + 1]);
  const float gx = ex / static_cast<float>(out_w - 1) * 2.f - 1.f;
  const float gy = ey / static_cast<float>(out_h - 1) * 2.f - 1.f;
  const float ix = ((gx + 1.f) / 2.f) * static_cast<float>(W - 1);
  const float iy = ((gy + 1.f) / 2.f) * static_cast<float>(H - 1);
  const float x0f = floorf(ix), y0f = floorf(iy);
  EdgeSample s;
  s.x0 = static_cast<int>(x0f);
  s.y0 = static_cast<int>(y0f);
  s.wx1 = ix - x0f;
  s.wy1 = iy - y0f;
  s.wx0 = 1.f - s.wx1;
  s.wy0 = 1.f - s.wy1;
  return s;
}

// ------------------------------------------------------------------------------------------------ cp.async
// 16-byte global->shared copy; src_bytes == 0 zero-fills the destination (used for conv padding / K tail).
MF_DEVINL void cp_async16(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
// same, allocating in L1 (.ca): the gather of small-Cin layers re-reads every input pixel kh*kw times from the same CTA
MF_DEVINL void cp_async16_ca(uint32_t dst_smem, const void* src, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(dst_smem), "l"(src), "r"(src_bytes) : "memory");
}
MF_DEVINL void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
MF_DEVINL void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ------------------------------------------------------------------------------------------------ TMA
MF_DEVINL void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
MF_DEVINL void tma_load_2d(uint32_t dst_smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// One lane of a fully converged warp. The TMA issuing warps walk their loops with ALL lanes (warp-uniform control flow
// keeps descriptors and addresses in uniform registers) and issue under `if (elect_one())`: under `if (lane == 0)` ptxas
// wraps every UTMALDG in an ELECT + R2UR + BRA.U.ANY "waterfall" loop.
MF_DEVINL bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P1;\n"
      "elect.sync _|P1, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P1;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------------ named barriers, TMA store, im2col-mode TMA load
MF_DEVINL void tma_load_im2col_4d(uint32_t dst_smem, const CUtensorMap* m, uint64_t* bar, int c, int w, int h, int n,
                                  uint16_t off_w, uint16_t off_h) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
      "[%2], {%7, %8};" ::"r"(dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c), "r"(w), "r"(h), "r"(n), "h"(off_w), "h"(off_h)
      : "memory");
}

MF_DEVINL void bar_sync_named(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// tiled 4D load (coordinates may lie outside the tensor: those elements are zero-filled and still counted in the tx bytes)
MF_DEVINL void tma_load_4d(uint32_t dst_smem, const CUtensorMap* m, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          dst_smem),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
MF_DEVINL void tma_store_2d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src_smem), "r"(c0), "r"(c1)
               : "memory");
}
MF_DEVINL void tma_store_4d(const CUtensorMap* m, uint32_t src_smem, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(src_smem), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
MF_DEVINL void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
MF_DEVINL void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
MF_DEVINL void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }


// ------------------------------------------------------------------------------------------------ wgmma (sm_90a)
// D[64 x N] (+)= A[64 x 16] * B[16 x N], fp16 operands from shared memory, fp32 accumulators in the registers of the
// issuing warpgroup (4 consecutive warps, the first one's index a multiple of 4). TA / TB = 1: the operand is MN-major.
// Accumulator fragment of thread t (warp w = t / 32 of the warpgroup, lane l): d[4 j + 2 h + e] is row 16 w + l / 4 + 8 h,
// column 8 j + 2 (l % 4) + e.
template <int N> struct Gmma;
template <> struct Gmma<16> {
  template <int TA, int TB>
  MF_DEVINL static void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %10, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <> struct Gmma<32> {
  template <int TA, int TB>
  MF_DEVINL static void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %18, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
  // A from registers: a[0..3] = fp16 pairs (row 16 w + l / 4 + 8 (i & 1), columns 8 (i >> 1) + 2 (l % 4) + {0, 1}). That is
  // the accumulator fragment layout above: columns [16 s, 16 s + 16) of an m64nN accumulator d are A = {d[8 s], d[8 s + 1]},
  // {d[8 s + 2], d[8 s + 3]}, {d[8 s + 4], d[8 s + 5]}, {d[8 s + 6], d[8 s + 7]}, with no data movement between threads.
  template <int TB>
  MF_DEVINL static void mma_rs(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, %22;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc), "n"(TB));
  }
};
template <> struct Gmma<64> {
  template <int TA, int TB>
  MF_DEVINL static void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};
template <> struct Gmma<128> {
  template <int TA, int TB>
  MF_DEVINL static void mma(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(acc), "n"(TA), "n"(TB));
  }
};

MF_DEVINL void gmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
MF_DEVINL void gmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
MF_DEVINL void gmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
template <int R>
MF_DEVINL void gmma_hold(float (&d)[R]) {      // keeps the accumulators in place across gmma_wait (no reordering)
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (sm_90 "GmmaDescriptor"): start>>4 [0,14) | LBO>>4 [16,30) | SBO>>4 [32,46)
// | layout_type [62,64) (1 = SWIZZLE_128B, 2 = 64B, 3 = 32B, 0 = none).
// K-major operand tile, 128-byte swizzle, rows of 64 fp16 (=128 B), 8-row atoms of 1024 B: LBO unused, SBO = 1024 B.
MF_DEVINL uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
// generic descriptor; `swz` = 0 (no swizzle: LBO = byte distance between the two 16-byte K chunks of a K-major MMA, SBO =
// distance between 8-row groups), 32 / 64 / 128 (K-major: LBO unused, SBO = 8 * row bytes; MN-major: LBO = distance
// between MN atoms, SBO = distance between 8-row K groups)
MF_DEVINL uint64_t gmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, int swz) {
  const uint64_t lt = swz == 128 ? 1ull : swz == 64 ? 2ull : swz == 32 ? 3ull : 0ull;
  return static_cast<uint64_t>((smem_addr >> 4) & 0x3FFFu) | (static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         (static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32) | (lt << 62);
}
// accumulator fragment of a m64nN tile -> rows [64][ld] fp32 at `base` (thread-per-row epilogues read it back); ld % 32 == 4
// makes both the float2 stores here and row-wise float4 loads conflict-free
template <int N>
MF_DEVINL void gmma_store_rows(const float (&d)[N / 2], uint32_t base, int ld) {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  const uint32_t r0 = base + ((16 * w + (l >> 2)) * ld + 2 * (l & 3)) * 4;
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + j * 32), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + (8 * ld + 8 * j) * 4), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}

// byte offset of 16-byte chunk `c` (0..7) of row `r` inside a [rows x 64 fp16] SWIZZLE_128B tile
MF_DEVINL uint32_t sw128_off(int r, int c) { return (r >> 3) * 1024 + (r & 7) * 128 + ((c ^ (r & 7)) << 4); }

}  // namespace mf
