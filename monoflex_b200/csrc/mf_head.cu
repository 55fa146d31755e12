// Fused predictor head (detector_predictor.py:121-135): the nine shared-input 3x3 convs (64 -> 9 x 256) + InPlaceABN +
// the 1x1 output convs (256 -> {3,4,2,20,3,3,16,1,1}) in ONE persistent kernel. The 2304-channel hidden map (1.13 GB at
// B = 8) is never written to HBM except for the two branches the edge-fusion gather needs.
//
// Per CTA (one per SM): for every 128-pixel m-tile, for every 128-channel n-tile nt (branch b = nt/2, half h = nt%2):
//   main GEMM   TMA warp: im2col-mode TMA A boxes + weight boxes -> 4-stage ring; two consumer warpgroups (rows 0-63 and
//               64-127 of the tile) issue wgmma m64n128k16 with fp32 accumulators in registers
//   epilogue    the same warpgroups: |gamma| BN affine -> leaky 0.01 -> fp16 -> 128B-swizzled smem staging. The staged
//               128 x 128 tile IS a canonical K-major wgmma A operand (two 64-channel sub-tiles), so ...
//   stage 2     ... each warpgroup contracts its 64 staged rows with the branch's 1x1 weights (32 x 256, TMA-loaded per
//               branch into a 2-deep ring) into a 64 x 32 register accumulator, accumulating over the branch's two n-tiles,
//               and after the second one adds the 1x1 bias and writes the fp32 NCHW `cls` / `reg` channels of that branch.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include <cstring>

namespace mf {

static constexpr int HBM = 128, HBN = 128, HBK = 64;
static constexpr int H_STAGES = 4;
static constexpr int H_ASTAGE = HBM * HBK * 2;          // 16 KB
static constexpr int H_BSTAGE = HBN * HBK * 2;          // 16 KB
static constexpr int H_OUT = 2 * H_ASTAGE;              // staged 128 x 128 fp16 tile
static constexpr int H_W2 = 4 * 32 * 128;               // 1x1 weights of one branch: 4 K blocks x [32 rows x 128 B]
static constexpr int H_MAXBR = 16;
static constexpr int H_SMEM = H_STAGES * (H_ASTAGE + H_BSTAGE) + H_OUT + 2 * H_W2 + 2048 + 1024;
static constexpr int H_THREADS = 288;                   // 8 consumer warps + the TMA warp

struct HeadParams {
  int B, H, W, Cin;              // feature map [B,H,W,Cin] fp16 rows, x_ld given to the tensor map
  int M, nkb, nbranch;           // M = B*H*W, nkb = 9*Cin/64
  const float* scale;            // [nbranch*256] folded |gamma| BN
  const float* shift;
  const float* bias2;            // [nbranch*32]
  float* out[H_MAXBR];           // per branch: fp32 NCHW base pointer already offset to its first channel
  int out_ctot[H_MAXBR];         // channels of the tensor it points into (batch stride = out_ctot*H*W)
  int out_nch[H_MAXBR];          // real output channels of the branch (<= 32)
  int hid_col[H_MAXBR];          // >= 0: hidden activations of this branch are stored at this column of `hid`
  __half* hid;                   // [M, hid_ld]
  int hid_ld;
  const unsigned char* hid_mask; // [M]: only flagged pixels are stored (the ~830 border pixels per image the edge fusion
};                               // gathers); null only when no branch has hid_col >= 0

__global__ void __launch_bounds__(H_THREADS, 1)
head_fused_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                  const __grid_constant__ CUtensorMap tmap_w2, const __grid_constant__ HeadParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_smem = smem;
  uint8_t* b_smem = a_smem + H_STAGES * H_ASTAGE;
  uint8_t* o_smem = b_smem + H_STAGES * H_BSTAGE;
  uint8_t* w2_smem = o_smem + H_OUT;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(w2_smem + 2 * H_W2);
  uint64_t* empty_bar = full_bar + H_STAGES;
  uint64_t* w2_full = empty_bar + H_STAGES;     // [2]
  uint64_t* w2_empty = w2_full + 2;             // [2]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  const int ntn = p.nbranch * 2;
  const int ntm = (p.M + HBM - 1) / HBM;
  const int HW = p.H * p.W;
  const int nkb = p.nkb;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&tmap_x); tma_prefetch_desc(&tmap_w); tma_prefetch_desc(&tmap_w2);
    for (int s = 0; s < H_STAGES; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    for (int a = 0; a < 2; ++a) { mbar_init(&w2_full[a], 1); mbar_init(&w2_empty[a], 8); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ================================================================ TMA producer (all lanes walk the loops, one issues)
    {
      int stage = 0, bc = 0;
      uint32_t phase = 0;
      for (int mt = blockIdx.x; mt < ntm; mt += gridDim.x) {
        const int m0 = mt * HBM;
        const int cn = m0 / HW, rem = m0 - cn * HW;
        const int cw = rem % p.W - 1, chh = rem / p.W - 1;          // 3x3, stride 1, pad 1
        for (int nt = 0; nt < ntn; ++nt) {
          if ((nt & 1) == 0) {                                       // 1x1 weights of branch nt/2 -> w2 ring
            const int buf = bc & 1;
            mbar_wait(&w2_empty[buf], ((bc >> 1) & 1) ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&w2_full[buf], H_W2);
              for (int kk = 0; kk < 4; ++kk)
                tma_load_2d(smem_u32(w2_smem + buf * H_W2 + kk * 32 * 128), &tmap_w2, &w2_full[buf], kk * 64, (nt >> 1) * 32);
            }
            __syncwarp();
            ++bc;
          }
          int tap = 0, c0 = 0, kx = 0, ky = 0;
          for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&full_bar[stage], H_ASTAGE + H_BSTAGE);
              tma_load_im2col_4d(smem_u32(a_smem + stage * H_ASTAGE), &tmap_x, &full_bar[stage], c0, cw, chh, cn,
                                 static_cast<uint16_t>(kx), static_cast<uint16_t>(ky));
              tma_load_2d(smem_u32(b_smem + stage * H_BSTAGE), &tmap_w, &full_bar[stage], kb * HBK, nt * HBN);
            }
            __syncwarp();
            c0 += HBK;
            if (c0 >= p.Cin) { c0 = 0; ++tap; if (++kx == 3) { kx = 0; ++ky; } }
            if (++stage == H_STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ================================================================ consumers: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    const int wg = warp >> 2, w = warp & 3;
    const uint32_t o_u = smem_u32(o_smem);
    const uint64_t a_d0 = gmma_desc_sw128(smem_u32(a_smem) + wg * 64 * 128), b_d0 = gmma_desc_sw128(smem_u32(b_smem));
    const uint64_t o_d0 = gmma_desc_sw128(o_u + wg * 64 * 128), w2_d0 = gmma_desc_sw128(smem_u32(w2_smem));
    float d[HBN / 2], d2[16];
    int stage = 0, ti = 0;
    uint32_t phase = 0;
    for (int mt = blockIdx.x; mt < ntm; mt += gridDim.x) {
      for (int nt = 0; nt < ntn; ++nt, ++ti) {
        const int br = nt >> 1, h = nt & 1, n0 = nt * HBN, bcj = ti >> 1, buf = bcj & 1;   // ntn is even: tile parity == half
        gmma_fence();
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint64_t a_off = static_cast<uint64_t>((stage * H_ASTAGE) >> 4);
          const uint64_t b_off = static_cast<uint64_t>((stage * H_BSTAGE) >> 4);
#pragma unroll
          for (int k4 = 0; k4 < HBK / 16; ++k4)
            Gmma<HBN>::mma<0, 0>(d, a_d0 + a_off + 2 * k4, b_d0 + b_off + 2 * k4, (kb | k4) != 0 ? 1u : 0u);
          gmma_commit();
          gmma_wait<0>();
          gmma_hold(d);
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
          if (++stage == H_STAGES) { stage = 0; phase ^= 1; }
        }
        // ---- epilogue: affine + leaky -> fp16 staging (and the hidden rows the edge fusion gathers)
        bar_sync_named(1, 256);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int row = wg * 64 + 16 * w + (lane >> 2) + 8 * hh;
          __half* hid_row = nullptr;                           // this thread's pixel is one the edge fusion will gather
          if (p.hid_col[br] >= 0) {
            const int m = mt * HBM + row;
            if (m < p.M && __ldg(p.hid_mask + m)) hid_row = p.hid + static_cast<long long>(m) * p.hid_ld + p.hid_col[br] + h * HBN;
          }
#pragma unroll
          for (int j = 0; j < HBN / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const float2 s2 = __ldg(reinterpret_cast<const float2*>(p.scale + n0 + c));
            const float2 h2 = __ldg(reinterpret_cast<const float2*>(p.shift + n0 + c));
            const float t0 = d[4 * j + 2 * hh] * s2.x + h2.x, t1 = d[4 * j + 2 * hh + 1] * s2.y + h2.y;
            const __half2 o = __floats2half2_rn(fmaxf(t0, 0.01f * t0), fmaxf(t1, 0.01f * t1));     // leaky_relu(0.01)
            const uint32_t addr = o_u + (j >> 3) * H_ASTAGE + sw128_off(row, j & 7) + 2 * (c & 7);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&o)) : "memory");
            if (hid_row != nullptr) *reinterpret_cast<__half2*>(hid_row + c) = o;
          }
        }
        fence_proxy_async();
        bar_sync_named(1, 256);
        // ---- stage 2: this warpgroup's 64 staged rows x the branch's 1x1 weights (K = 128 hidden channels of this half)
        if (h == 0) mbar_wait(&w2_full[buf], (bcj >> 1) & 1);
        gmma_fence();
#pragma unroll
        for (int s = 0; s < 2; ++s)
#pragma unroll
          for (int k4 = 0; k4 < 4; ++k4)
            Gmma<32>::mma<0, 0>(d2, o_d0 + ((s * H_ASTAGE) >> 4) + 2 * k4,
                                w2_d0 + ((buf * H_W2 + (2 * h + s) * 32 * 128) >> 4) + 2 * k4, (h | s | k4) != 0 ? 1u : 0u);
        gmma_commit();
        gmma_wait<0>();
        gmma_hold(d2);
        if (h == 1) {
          __syncwarp();
          if (lane == 0) mbar_arrive(&w2_empty[buf]);
          // ---- 1x1 outputs of the branch: bias, fp32 NCHW
          const int nch = p.out_nch[br];
#pragma unroll
          for (int hh = 0; hh < 2; ++hh) {
            const int m = mt * HBM + wg * 64 + 16 * w + (lane >> 2) + 8 * hh;
            if (m >= p.M) continue;
            const int img = m / HW, pix = m - img * HW;
            float* yp = p.out[br] + static_cast<long long>(img) * p.out_ctot[br] * HW + pix;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int n = 8 * j + 2 * (lane & 3) + e;
                if (n < nch) yp[static_cast<long long>(n) * HW] = d2[4 * j + 2 * hh + e] + __ldg(p.bias2 + br * 32 + n);
              }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encTiledH)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
typedef CUresult (*PFN_encIm2colH)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                   const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void* driver_fn(const char* name) {
  void* ptr = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint(name, &ptr, cudaEnableDefault, &qres) != cudaSuccess || qres != cudaDriverEntryPointSuccess)
    return nullptr;
  return ptr;
}

// x: features [B*H*W, x_ld] fp16 (Cin channels used); w3: packed 3x3 weights [nbranch*256, 9*Cin]; w2: packed 1x1 weights
// [nbranch*32, 256]; hid: [M, hid_ld] fp16 buffer receiving the hidden activations of the branches with hid_col >= 0 at the
// pixels hid_mask flags.
int launch_head_fused(const __half* x, int x_ld, int B, int H, int W, int Cin, const __half* w3, const __half* w2,
                      const float* scale, const float* shift, const float* bias2, int nbranch, float* const* out,
                      const int* out_ctot, const int* out_nch, const int* hid_col, __half* hid, int hid_ld,
                      const unsigned char* hid_mask, cudaStream_t st) {
  static PFN_encTiledH enc = reinterpret_cast<PFN_encTiledH>(driver_fn("cuTensorMapEncodeTiled"));
  static PFN_encIm2colH enc2 = reinterpret_cast<PFN_encIm2colH>(driver_fn("cuTensorMapEncodeIm2col"));
  if (!enc || !enc2) { set_error("head_fused: tensor-map driver entry points unavailable"); return -1; }
  if (Cin % 64 != 0 || nbranch < 1 || nbranch > H_MAXBR || x_ld % 8 != 0 || hid_ld % 8 != 0) {
    set_error("head_fused: unsupported shape Cin=%d nbranch=%d", Cin, nbranch);
    return -1;
  }
  for (int i = 0; i < nbranch; ++i) {
    if (hid_col[i] >= 0 && hid_mask == nullptr) { set_error("head_fused: branch %d stores hidden rows but hid_mask is null", i); return -1; }
  }
  HeadParams p;
  memset(&p, 0, sizeof(p));
  p.B = B; p.H = H; p.W = W; p.Cin = Cin; p.M = B * H * W; p.nkb = 9 * Cin / 64; p.nbranch = nbranch;
  p.scale = scale; p.shift = shift; p.bias2 = bias2;
  p.hid = hid; p.hid_ld = hid_ld; p.hid_mask = hid_mask;
  for (int i = 0; i < nbranch; ++i) {
    p.out[i] = out[i]; p.out_ctot[i] = out_ctot[i]; p.out_nch[i] = out_nch[i]; p.hid_col[i] = hid_col[i];
    if (out_nch[i] > 32) { set_error("head_fused: branch %d has %d > 32 output channels", i, out_nch[i]); return -1; }
  }
  CUtensorMap tx, tw, tw2;
  {
    cuuint64_t gdim[4] = {static_cast<cuuint64_t>(Cin), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(B)};
    cuuint64_t gstr[3] = {static_cast<cuuint64_t>(x_ld) * 2, static_cast<cuuint64_t>(x_ld) * 2 * W, static_cast<cuuint64_t>(x_ld) * 2 * W * H};
    int lower[2] = {-1, -1}, upper[2] = {-1, -1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    if (enc2(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(x), gdim, gstr, lower, upper, 64, HBM, estr,
             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) { set_error("head_fused: im2col map failed"); return -1; }
  }
  auto tiled2d = [&](CUtensorMap* m, const void* ptr, int inner, int rows, int ld_elems, int box_inner, int box_rows) {
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(inner), static_cast<cuuint64_t>(rows)};
    cuuint64_t gstr[1] = {static_cast<cuuint64_t>(ld_elems) * 2};
    cuuint32_t box[2] = {static_cast<cuuint32_t>(box_inner), static_cast<cuuint32_t>(box_rows)};
    cuuint32_t estr[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  };
  const int K3 = 9 * Cin;
  if (!tiled2d(&tw, w3, K3, nbranch * 256, K3, 64, HBN) || !tiled2d(&tw2, w2, 256, nbranch * 32, 256, 64, 32)) {
    set_error("head_fused: tiled tensor map failed");
    return -1;
  }
  static bool attr = false;
  if (!attr) {
    if (check_cuda(cudaFuncSetAttribute(head_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, H_SMEM), "head smem")) return -1;
    attr = true;
  }
  int dev = 0, nsm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  const int ntm = (p.M + HBM - 1) / HBM;
  const int grid = ntm < nsm ? ntm : nsm;
  return check_cuda(launch_k(head_fused_kernel, dim3(grid), dim3(H_THREADS), H_SMEM, st, tx, tw, tw2, p), "head_fused launch");
}

}  // namespace mf
