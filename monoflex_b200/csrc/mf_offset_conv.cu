// The DCN offset/mask convolutions (DCN.conv_offset_mask, dcn_v2.py:106-122): 3x3, stride 1, pad 1, Cin % 64 == 0 -> 27
// outputs, written as fp32 [M, 32] rows (offsets 0-17, sigmoid masks 18-26, 27-31 the sigmoid of the zero columns) that
// the fused DCN gathers from. Each input element crosses L2 -> SM about once per tile instead of once per tap:
//
//   * a tile is R output rows x S output pixels of one image; per 64-channel chunk the A-TMA warp loads the (R + 2) x
//     (S + 2) input pixels the tile needs as ONE tiled 4-D box {64 ch, S + 2, R + 2, 1} (SWIZZLE_128B: a pixel is one
//     128-byte row of the box, the TMA's zero fill is the padding, at image borders and past W). Strict precision loads the
//     lo halves of the same pixels as a second box at channel coordinate x_lo + c0.
//   * stage pixel q = ry (S + 2) + px. Output (r, x) of the tile is the "flat" row f = r (S + 2) + x, and tap (ky, kx)
//     reads stage pixel f + ky (S + 2) + kx: 64 consecutive flat rows are one K-major wgmma A operand whose descriptor
//     starts (ky (S + 2) + kx) x 128 B further on. The rows x >= S of that range are computed and not stored. The start is
//     moved by whole rows, so it lies off the 1024-byte swizzle atom; the wgmma unit swizzles by absolute address, as the
//     TMA wrote the box, with the descriptor's base-offset field 0 (tests/test_gpu_offset_conv.py checks this on the GPU).
//   * weights come straight from the packed [32, k_pad] rows of mf_pack_conv_weight(_split): per (chunk, kernel row ky)
//     the W-TMA warp loads the three taps' [32 outputs x 64 channels] boxes, strict: W_hi into B rows 0-31 and W_lo into
//     rows 32-63 of each tap. When all of them fit beside the A ring they are loaded once per CTA and stay resident.
//   * strict: A_hi x [W_hi | W_lo] is one m64n64 MMA and A_lo x W_hi one m64n32 MMA into the first 32 columns of the same
//     accumulator; the epilogue adds the column halves in fp32 (A_hi W_hi + A_lo W_hi) + A_hi W_lo before scale / shift.
//   * two consumer warpgroups take alternate 64-row blocks of a tile, NBW blocks each (a template parameter: a runtime
//     block count puts a predicate around the MMAs, and ptxas then fences every one of them); the A and W producers run
//     ahead on separate rings.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include <cstring>

namespace mf {

static constexpr int OC_NWG = 2;             // consumer warpgroups
static constexpr int OC_MAX_BLK = 4;         // 64-row blocks per consumer warpgroup (NBW <= 4)
static constexpr int OC_MAX_AS = 4;          // A ring depth cap
static constexpr int OC_MAX_WS = 24;         // W stages: 3 per chunk when resident (Cin <= 512), else a ring of 3
static constexpr int OC_THREADS = OC_NWG * 128 + 64;
static constexpr int OC_SMEM_MAX = 232448;

struct OffConvParams {
  int B, H, W, nch;              // nch = Cin / 64
  int R, S, P, nblk;             // tile: R rows x S pixels; stage pitch P = S + 2; nblk = 2 NBW 64-row blocks of f = r P + x
  int segs, bands;               // tiles per image row band, bands per image
  int x_lo;                      // strict: channel coordinate of the lo halves
  int a_half, nas;               // bytes of one A box region (1024-aligned); A ring depth (a stage = 1 or 2 boxes)
  int nws, w_resident;           // W stages (one kernel row of one chunk each); resident: 3 nch stages, loaded once
  const float* scale;
  const float* shift;
  float* y;                      // [B H W][32] fp32
};

// strict: A_hi x [W_hi | W_lo] (m64n64) then A_lo x W_hi (m64n32) into columns 0-31 of the same accumulator. One asm block:
// as two statements, the second reading a 16-register slice of the first one's accumulator, ptxas fences every pair.
MF_DEVINL void mma_pair(float (&d)[32], uint64_t a_hi, uint64_t a_lo, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n.reg .pred p;\n.reg .pred q;\nsetp.ne.b32 p, %35, 0;\nsetp.eq.b32 q, %35, %35;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %34, p, 1, 1, 0, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %33, %34, q, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a_hi), "l"(a_lo), "l"(b), "r"(acc));
}

template <bool PAIR, int NBW>
__global__ void __launch_bounds__(OC_THREADS, 1)
offset_conv_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                   const __grid_constant__ OffConvParams p) {
  constexpr int NB = PAIR ? 64 : 32;         // B rows of one tap: W_hi (| W_lo)
  constexpr int TAP_BYTES = NB * 128;
  constexpr int W_STAGE = 3 * TAP_BYTES;
  constexpr int NHL = PAIR ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const uint32_t w_u = smem_u32(smem);
  const int a_stage = NHL * p.a_half;
  const uint32_t a_u = w_u + p.nws * W_STAGE;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(smem + p.nws * W_STAGE + p.nas * a_stage);
  uint64_t* a_empty = a_full + OC_MAX_AS;
  uint64_t* w_full = a_empty + OC_MAX_AS;
  uint64_t* w_empty = w_full + OC_MAX_WS;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
  const int ntiles = p.B * p.bands * p.segs;
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < p.nas; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4 * OC_NWG); }
    for (int s = 0; s < p.nws; ++s) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], 4 * OC_NWG); }
    fence_mbar_init();
  }
  __syncthreads();
  auto tile_origin = [&](int t, int& b, int& oy0, int& ox0) {
    const int band = t / p.segs;
    ox0 = (t - band * p.segs) * p.S;
    b = band / p.bands;
    oy0 = (band - b * p.bands) * p.R;
  };

  if (warp == 4 * OC_NWG) {
    // ================================================================ A: one box per (tile, chunk, hi | lo)
    const uint32_t box_bytes = static_cast<uint32_t>((p.R + 2) * p.P * 128);
    int s = 0;
    uint32_t ph = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      int b, oy0, ox0;
      tile_origin(t, b, oy0, ox0);
      for (int c = 0; c < p.nch; ++c) {
        mbar_wait(&a_empty[s], ph ^ 1);
        if (elect_one()) {
          mbar_arrive_expect_tx(&a_full[s], NHL * box_bytes);
#pragma unroll
          for (int hl = 0; hl < NHL; ++hl)
            tma_load_4d(a_u + s * a_stage + hl * p.a_half, &tmap_x, &a_full[s], c * 64 + hl * p.x_lo, ox0 - 1, oy0 - 1, b);
        }
        __syncwarp();
        if (++s == p.nas) { s = 0; ph ^= 1; }
      }
    }
  } else if (warp == 4 * OC_NWG + 1) {
    // ================================================================ W: the three taps of kernel row ky, chunk c
    auto load = [&](int st, int c, int ky) {
      if (elect_one()) {
        mbar_arrive_expect_tx(&w_full[st], W_STAGE);
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const int kb = (3 * ky + kx) * p.nch + c;             // (tap, chunk) K block of the packed rows
          const uint32_t dst = w_u + st * W_STAGE + kx * TAP_BYTES;
          if (PAIR) {                                           // split packing: [W_hi | W_hi | W_lo] per (tap, chunk)
            tma_load_2d(dst, &tmap_w, &w_full[st], 3 * kb * 64, 0);
            tma_load_2d(dst + 32 * 128, &tmap_w, &w_full[st], (3 * kb + 2) * 64, 0);
          } else {
            tma_load_2d(dst, &tmap_w, &w_full[st], kb * 64, 0);
          }
        }
      }
      __syncwarp();
    };
    if (p.w_resident) {
      for (int c = 0; c < p.nch; ++c)
        for (int ky = 0; ky < 3; ++ky) load(3 * c + ky, c, ky);
    } else {
      int s = 0;
      uint32_t ph = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x)
        for (int c = 0; c < p.nch; ++c)
          for (int ky = 0; ky < 3; ++ky) {
            mbar_wait(&w_empty[s], ph ^ 1);
            load(s, c, ky);
            if (++s == p.nws) { s = 0; ph ^= 1; }
          }
    }
  } else {
    // ================================================================ consumers: warpgroup g owns blocks g, g + 2, ...
    const int g = warp >> 2, w = warp & 3, tq = lane & 3;
    float sc[8], sh[8];                          // columns 8 j + 2 tq + e
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        sc[2 * j + e] = __ldg(p.scale + 8 * j + 2 * tq + e);
        sh[2 * j + e] = __ldg(p.shift + 8 * j + 2 * tq + e);
      }
    float acc[NBW][NB / 2];
    const uint64_t a_d0 = gmma_desc_sw128(a_u), w_d0 = gmma_desc_sw128(w_u);
    int as = 0, ws = 0;
    uint32_t aph = 0, wph = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      int b, oy0, ox0;
      tile_origin(t, b, oy0, ox0);
      for (int c = 0; c < p.nch; ++c) {
        mbar_wait(&a_full[as], aph);
        const uint64_t a_s = a_d0 + static_cast<uint64_t>((as * a_stage) >> 4);
        for (int ky = 0; ky < 3; ++ky) {
          const int wst = p.w_resident ? 3 * c + ky : ws;
          mbar_wait(&w_full[wst], p.w_resident ? 0u : wph);
          const uint64_t w_s = w_d0 + static_cast<uint64_t>((wst * W_STAGE) >> 4);
          gmma_fence();
#pragma unroll
          for (int kx = 0; kx < 3; ++kx)
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4) {
              const uint64_t bd = w_s + static_cast<uint64_t>((kx * TAP_BYTES + k4 * 32) >> 4);
              const uint32_t acc_in = (c | ky | kx | k4) != 0 ? 1u : 0u;
#pragma unroll
              for (int i = 0; i < NBW; ++i) {
                const uint64_t ad = a_s + static_cast<uint64_t>((((g + 2 * i) * 64 + ky * p.P + kx) * 128 + k4 * 32) >> 4);
                if constexpr (PAIR)
                  mma_pair(acc[i], ad, ad + (p.a_half >> 4), bd, acc_in);
                else
                  Gmma<NB>::template mma<0, 0>(acc[i], ad, bd, acc_in);
              }
            }
          gmma_commit();
          gmma_wait<0>();
#pragma unroll
          for (int i = 0; i < NBW; ++i) gmma_hold(acc[i]);
          if (!p.w_resident) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&w_empty[ws]);
            if (++ws == p.nws) { ws = 0; wph ^= 1; }
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&a_empty[as]);
        if (++as == p.nas) { as = 0; aph ^= 1; }
      }
      // ---- epilogue: d[4 j + 2 h + e] is flat row (g + 2 i) 64 + 16 w + lane / 4 + 8 h, column 8 j + 2 tq + e
#pragma unroll
      for (int i = 0; i < NBW; ++i) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int f = (g + 2 * i) * 64 + 16 * w + (lane >> 2) + 8 * h;
          const int r = f / p.P, x = f - r * p.P;
          const int oy = oy0 + r, ox = ox0 + x;
          if (r >= p.R || x >= p.S || oy >= p.H || ox >= p.W) continue;
          float* dst = p.y + (static_cast<long long>(b * p.H + oy) * p.W + ox) * 32 + 2 * tq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float v[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              float a = acc[i][4 * j + 2 * h + e];
              if constexpr (PAIR) a += acc[i][4 * (j + 4) + 2 * h + e];
              a = a * sc[2 * j + e] + sh[2 * j + e];
              v[e] = 8 * j + 2 * tq + e >= 18 ? 1.f / (1.f + __expf(-a)) : a;
            }
            *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(v[0], v[1]);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiledO)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiledO offconv_encode_fn() {
  static PFN_encodeTiledO fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
      set_error("cuTensorMapEncodeTiled entry point unavailable");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiledO>(ptr);
  }
  return fn;
}

// The tile for one layer shape: S from the even splits of W, R and the W residency from what fits in shared memory, chosen by
// an estimate of the per-SM time (waves x the larger of the tensor time and the L2 -> SM time of a tile; H100 SXM: about
// 26 ns per m64n64k16 + m64n32k16 pair, 9 ns per m64n32k16, about 30 B/ns of L2 -> SM bandwidth per SM under full load).
// The same selection, and the L2 -> SM bytes it implies, is restated in tools/bench_dcn.py (offset_conv_traffic).
bool offset_conv_pick(int B, int H, int W, int Cin, bool pair, int nsm, OffConvParams& p) {
  const int nch = Cin / 64, nhl = pair ? 2 : 1;
  const int w_stage = 3 * (pair ? 64 : 32) * 128;
  double best = 1e30;
  bool found = false;
  for (int nseg = 1; nseg <= W; ++nseg) {
    const int S = (W + nseg - 1) / nseg;
    if (nseg > 1 && S < 8) break;                              // narrower segments only add halo
    if (S + 2 > 256) continue;
    if ((W + S - 1) / S != nseg) continue;                     // same S as a smaller nseg
    const int P = S + 2;
    for (int R = 1; R <= H && R + 2 <= 256; ++R) {
      const int nblk = ((R * P - 2 + 127) / 128) * 2;            // even: both warpgroups run NBW = nblk / 2 blocks
      if (nblk > OC_NWG * OC_MAX_BLK) break;
      const int a_half = ((nblk * 64 + 2 * P + 2) * 128 + 1023) & ~1023;
      const int fixed = 2048;
      const bool res = 3 * nch <= OC_MAX_WS && 3 * nch * w_stage + 2 * nhl * a_half + fixed <= OC_SMEM_MAX;
      const int nws = res ? 3 * nch : 3;
      int nas = (OC_SMEM_MAX - fixed - nws * w_stage) / (nhl * a_half);
      if (nas > OC_MAX_AS) nas = OC_MAX_AS;
      if (nas < 2) continue;
      const long long ntiles = static_cast<long long>(B) * ((H + R - 1) / R) * nseg;
      const double mma_ns = nch * nblk * 36.0 * (pair ? 26.2 : 8.7);
      const double load_ns = nch * (nhl * (R + 2.0) * P * 128 + (res ? 0.0 : 3.0 * w_stage)) / 30.0;
      const double cost = static_cast<double>((ntiles + nsm - 1) / nsm) * ((mma_ns > load_ns ? mma_ns : load_ns) + 300.0);
      if (cost < best) {
        best = cost;
        found = true;
        p.nch = nch; p.R = R; p.S = S; p.P = P; p.nblk = nblk; p.segs = nseg; p.bands = (H + R - 1) / R;
        p.a_half = a_half; p.nas = nas; p.nws = nws; p.w_resident = res ? 1 : 0;
      }
    }
  }
  return found;
}

int launch_offset_conv(const __half* x, int x_ld, int x_lo, int B, int H, int W, int Cin, const __half* wp, int n_pad, int k_pad,
                       const float* scale, const float* shift, float* y, int y_ld, bool pair, cudaStream_t st) {
  if (Cin % 64 != 0 || Cin > 512 || n_pad != 32 || k_pad != (pair ? 3 : 1) * 9 * Cin || y_ld != 32 || x_ld % 8 != 0 ||
      (reinterpret_cast<uintptr_t>(x) & 15) != 0 || (pair && (x_lo % 8 != 0 || x_lo < Cin || x_lo + Cin > x_ld)) ||
      (!pair && Cin > x_ld)) {
    set_error("offset_conv: unsupported configuration (Cin %d, x_ld %d, x_lo %d, n_pad %d, k_pad %d, y_ld %d)", Cin, x_ld, x_lo,
              n_pad, k_pad, y_ld);
    return -1;
  }
  PFN_encodeTiledO enc = offconv_encode_fn();
  if (!enc) return -1;
  static int nsm = 0;
  if (nsm == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
    if (nsm <= 0) nsm = 132;
  }
  OffConvParams p;
  memset(&p, 0, sizeof(p));
  if (!offset_conv_pick(B, H, W, Cin, pair, nsm, p)) { set_error("offset_conv: no tile fits (H %d, W %d)", H, W); return -1; }
  p.B = B; p.H = H; p.W = W; p.x_lo = pair ? x_lo : 0;
  p.scale = scale; p.shift = shift; p.y = y;
  CUtensorMap tx, tw;
  {
    cuuint64_t gdim[4] = {static_cast<cuuint64_t>(pair ? x_lo + Cin : Cin), static_cast<cuuint64_t>(W),
                          static_cast<cuuint64_t>(H), static_cast<cuuint64_t>(B)};
    cuuint64_t gstr[3] = {static_cast<cuuint64_t>(x_ld) * 2, static_cast<cuuint64_t>(x_ld) * 2 * W,
                          static_cast<cuuint64_t>(x_ld) * 2 * W * H};
    cuuint32_t box[4] = {64, static_cast<cuuint32_t>(p.P), static_cast<cuuint32_t>(p.R + 2), 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(x), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("offset_conv: cuTensorMapEncodeTiled(x) failed (%d)", static_cast<int>(r)); return -1; }
  }
  {
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(k_pad), 32};
    cuuint64_t gstr[1] = {static_cast<cuuint64_t>(k_pad) * 2};
    cuuint32_t box[2] = {64, 32};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tw, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(wp), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("offset_conv: cuTensorMapEncodeTiled(w) failed (%d)", static_cast<int>(r)); return -1; }
  }
  const int w_stage = 3 * (pair ? 64 : 32) * 128;
  const int smem = p.nws * w_stage + p.nas * (pair ? 2 : 1) * p.a_half + 2048;
  const long long ntiles = static_cast<long long>(B) * p.bands * p.segs;
  const int grid = ntiles < nsm ? static_cast<int>(ntiles) : nsm;
  static void (*const kerns[2][OC_MAX_BLK])(CUtensorMap, CUtensorMap, OffConvParams) = {
      {offset_conv_kernel<false, 1>, offset_conv_kernel<false, 2>, offset_conv_kernel<false, 3>, offset_conv_kernel<false, 4>},
      {offset_conv_kernel<true, 1>, offset_conv_kernel<true, 2>, offset_conv_kernel<true, 3>, offset_conv_kernel<true, 4>}};
  static bool attr[2][OC_MAX_BLK] = {};
  auto kern = kerns[pair][p.nblk / 2 - 1];
  if (!attr[pair][p.nblk / 2 - 1]) {
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, OC_SMEM_MAX), "offset_conv smem"))
      return -1;
    attr[pair][p.nblk / 2 - 1] = true;
  }
  return check_cuda(launch_k(kern, dim3(grid), dim3(OC_THREADS), smem, st, tx, tw, p), "offset_conv launch");
}

}  // namespace mf
