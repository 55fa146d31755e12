// Persistent, warp-specialised implicit-GEMM convolution / fused DCNv2 for sm_90a.
//
//   D[m, n] = sum_k A[m, k] * Wp[n, k]      m = output pixel, n = output channel, k = (tap, cin) cin fastest
//
// One CTA per SM (two for the narrow-N tiles) loops over 128 x BLOCK_N output tiles, n fastest:
//   warps [0, NPW)        A producers. MODE_CONV: 16-byte cp.async gathers of the zero-padded taps into the 128B-swizzled
//                         K-major stage (Cin < 64 layers). MODE_DCN: per (pixel, tap) 4 neighbour NHWC vectors, fp32
//                         bilinear blend * mask, fp16, st.shared; a tile is an 8x16 pixel block so its neighbourhood
//                         stays L1-resident. MODE_CONV_TMA (Cin % 64 == 0): no producer warps at all - the TMA warp
//                         fetches each (tap, 64-channel) A block with ONE im2col-mode cp.async.bulk.tensor.4d (zero
//                         padding, strides and row/image wrap-around done by the TMA unit) and these warps become a
//                         second epilogue group.
//   warps [NPW, NPW+8)    two consumer warpgroups: wgmma (m64 x BLOCK_N x k16, fp32 accumulators in registers), warpgroup
//                         wg owning rows [64 wg, 64 wg + 64) of the tile; at the end of a tile they hand the accumulators
//                         over in 32-column chunks through one fp32 smem slot and go on with the next tile's main loop
//   warp NPW+8            weight tiles by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B), same mbarrier ring as A
//   warps [NPW+9, NPW+13) epilogue: chunk slot -> scale/shift (+residual) -> activation -> fp16 -> swizzled smem staging
//                         -> one TMA store per 64-channel sub-tile (fp32 NHWC / NCHW outputs: direct stores)
// Registers + the chunk slot act as a double buffer: the epilogue of tile i overlaps the main loop of tile i+1; the smem ring
// and the barriers persist across tiles, so the per-tile cost is the MMA time, not a pipeline fill + drain.
// HEAD2 (strict predictor, EPI == 2) has neither producer nor epilogue warps: the consumers contract the 1x1 heads from their
// own accumulators on the tensor cores and store the results (see IgemmParams).
// MODE_DCN with 64-column tiles (NPW == 16, "wide gather", igemm2_wide): 16 producer warps (2 pixel rows per thread and K
// block instead of 4) and ONE consumer warpgroup, which issues two m64n64k16 wgmmas per k16 step (rows [0, 64) and [64, 128))
// and finishes its own tiles from the accumulator fragments; no epilogue warps and no chunk slot, whose shared memory goes to
// the ring. At 64 columns a gathered A element feeds only 64 x 3 MACs, so the gather bounds the kernel, not the tensor pipe.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"

namespace mf {

static constexpr int BM = 128;
static constexpr int BK = 64;
static constexpr int A_STAGE = BM * BK * 2;   // 16 KB

// SPLIT: the fp16 NHWC output is a hi/lo pair (strict-precision mode): two staging tiles per 64-channel sub-tile, paid for
// with one pipeline stage (the K loop of a split layer is 3x longer, so the shallower ring costs nothing measurable).
// EPI (see igemm2_kernel): 1 = SPLIT doubles the staging; 2 = HEAD2 has no output staging and no chunk slot, its staging area
// holds the two slots of 1x1 head weights instead. HEAD2 at BLOCK_N = 128: FIXED = 32768 + 384 + 1024 + 1024 = 35200 B, and
// (232448 - 35200) / (16384 + 16384) = 6.02, so a sixth ring stage fits (SMEM = 6 x 32768 + 35200 = 231808 B).
// WIDE (the wide-gather DCN, see igemm2_wide): no chunk slot. Strict: FIXED = 32768 + 384 + 512 + 36864 + 1024 = 71552 B, and
// (232448 - 71552) / (16384 + 8192) = 6.5 stages would fit, but the ring keeps the DCN's 4: measured on one H100 80GB HBM3
// (700 W), 6 stages made the strict 64 -> 64 layer at 96 x 320, B = 8, 4 % slower (0.313 against 0.301 ms).
template <int BLOCK_N, int MODE, int EPI = 0, bool WIDE = false>
struct Cfg2 {
  static constexpr bool SPLIT = EPI == 1;
  static constexpr int CTAS_PER_SM = BLOCK_N >= 64 ? 1 : 2;
  static constexpr int LAG = BLOCK_N >= 64 ? 3 : (BLOCK_N >= 32 ? 3 : 4);   // cp.async groups in flight per producer thread
  static constexpr int B_STAGE = BLOCK_N * BK * 2;
  static constexpr int OUT_HALF = BLOCK_N >= 64 ? (BLOCK_N / 64) * A_STAGE : 0;     // staging of one fp16 tile
  // HEAD2: one slot of split 1x1 head weights = 4 boxes [32 outputs][64 hidden channels] fp16, 128B-swizzled:
  // W_hi of the tile's two 64-channel chunks, then W_lo of both
  static constexpr int W1_BOX = 32 * BK * 2;
  static constexpr int W1_STAGE = 4 * W1_BOX;
  static constexpr int OUT_STAGE = EPI == 2 ? 2 * W1_STAGE : (SPLIT ? 2 * OUT_HALF : OUT_HALF);
  static constexpr int BAR_BYTES = 384;                         // barriers
  static constexpr int PRM_BYTES = MODE == MODE_DCN ? 9 * BM * 32 : 0;   // DCN sampling records
  static constexpr int CHUNK = BLOCK_N >= 32 ? 32 : 16;         // accumulator hand-over unit (columns)
  static constexpr int ACC_LD = CHUNK + 4;                      // fp32 row stride of the chunk slot (conflict-free, see gmma_store_cols)
  static constexpr int ACC_BYTES = (EPI == 2 || WIDE) ? 0 : BM * ACC_LD * 4;
  static constexpr int BUDGET = (CTAS_PER_SM == 2 ? 113 : 227) * 1024;
  static constexpr int FIXED = OUT_STAGE + BAR_BYTES + 2 * BLOCK_N * 4 + PRM_BYTES + ACC_BYTES + 1024;
  // ring depth: the shallower of the preferred depth and what the shared-memory budget leaves
  static constexpr int STAGES0 = (MODE == MODE_DCN ? 4 : (EPI == 2 ? 6 : (BLOCK_N >= 128 ? 5 : (BLOCK_N >= 64 ? 6 : (BLOCK_N >= 32 ? 5 : 6)))));
  static constexpr int STAGES1 = (SPLIT && BLOCK_N >= 64) ? ((MODE == MODE_DCN && BLOCK_N < 128) ? STAGES0 : STAGES0 - 1) : STAGES0;
  static constexpr int FIT = (BUDGET - FIXED) / (A_STAGE + B_STAGE);
  static constexpr int STAGES = STAGES1 < FIT ? STAGES1 : FIT;
  static_assert(STAGES >= 2, "at least a double-buffered ring");
  static constexpr int SMEM = STAGES * (A_STAGE + B_STAGE) + FIXED;
  static_assert(SMEM <= BUDGET, "shared memory budget");
};

// fragment columns [8 j0, 8 j0 + 8 NJ) of a m64 x N accumulator -> chunk slot rows [64][ld] fp32 (see gmma_store_rows)
template <int N, int J0, int NJ>
MF_DEVINL void gmma_store_cols(const float (&d)[N / 2], uint32_t base, int ld) {
  const int t = threadIdx.x & 127, w = t >> 5, l = t & 31;
  const uint32_t r0 = base + ((16 * w + (l >> 2)) * ld + 2 * (l & 3)) * 4;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + j * 32), "f"(d[4 * (J0 + j)]), "f"(d[4 * (J0 + j) + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + (8 * ld + 8 * j) * 4), "f"(d[4 * (J0 + j) + 2]),
                 "f"(d[4 * (J0 + j) + 3]) : "memory");
  }
}
template <int N, int CHUNK, int CH>
struct ChunkDump {                         // compile-time walk over the chunks of the accumulator
  template <typename F>
  MF_DEVINL static void run(const float (&d)[N / 2], F&& f) {
    if constexpr (CH * CHUNK < N) {
      f(CH, [&](uint32_t base, int ld) { gmma_store_cols<N, CH * CHUNK / 8, CHUNK / 8>(d, base, ld); });
      ChunkDump<N, CHUNK, CH + 1>::run(d, f);
    }
  }
};

// the wide-gather DCN configuration (64-column tiles): 16 producer warps and one self-finishing consumer warpgroup
__host__ __device__ constexpr bool igemm2_wide(int mode, int npw) { return mode == MODE_DCN && npw == 16; }

// warps of a CTA: NPW producers, 8 consumers, the weight-TMA warp (MODE_DCN: the producers issue the weight loads, which
// keeps 640 threads and 96 registers for the consumers' 64 accumulators), 4 epilogue warps (none for HEAD2, whose consumers
// finish their own tiles). Wide-gather DCN: 16 producers + 4 consumers, the same 640 threads.
__host__ __device__ constexpr int igemm2_warps(int mode, int npw, int epi) {
  return igemm2_wide(mode, npw) ? npw + 4 : npw + 8 + (mode == MODE_DCN ? 0 : 1) + (epi == 2 ? 0 : 4);
}

template <int N>
MF_DEVINL void act_chunk(float (&v)[N], int act) {
  if (act == ACT_RELU) {
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = fmaxf(v[i], 0.f);
  } else if (act == ACT_LEAKY) {
#pragma unroll
    for (int i = 0; i < N; ++i) v[i] = fmaxf(v[i], 0.01f * v[i]);      // == v > 0 ? v : 0.01 v
  }
}

// EPI: 0 = plain epilogue, 1 = SPLIT (staged hi/lo output tiles), 2 = HEAD2 (the consumers contract the 1x1 heads on the
// tensor cores, see IgemmParams; no epilogue warps, NPW = 0). tmap_y: the output tiles, or for HEAD2 the split 1x1 weights.
template <int BLOCK_N, int MODE, int NPW, int EPI>
__global__ void __launch_bounds__(igemm2_warps(MODE, NPW, EPI) * 32, Cfg2<BLOCK_N, MODE, EPI>::CTAS_PER_SM)
igemm2_kernel(const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ CUtensorMap tmap_y,
              const __grid_constant__ CUtensorMap tmap_x, const IgemmParams p, const int use_tma_store) {
  constexpr bool PTILE = MODE == MODE_DCN;               // m-tile = 16 x 8 patch of one image
  constexpr bool A_TMA = MODE == MODE_CONV_TMA;
  constexpr int EPI_THREADS = A_TMA ? 128 + NPW * 32 : 128;
  constexpr bool SPLIT = EPI == 1;
  constexpr bool HEAD2 = EPI == 2;
  static_assert(!HEAD2 || (A_TMA && NPW == 0 && BLOCK_N == 128), "HEAD2: TMA-only warps, 128-column tiles");
  constexpr bool WIDE = igemm2_wide(MODE, NPW);
  static_assert(!WIDE || BLOCK_N == 64, "wide-gather DCN: 64-column tiles (two m64n64 accumulators per consumer thread)");
  using C = Cfg2<BLOCK_N, MODE, EPI, WIDE>;
  constexpr int STAGES = C::STAGES;
  constexpr int LAG = C::LAG;
  const bool split_out = SPLIT || p.split_out != 0;      // SPLIT == staged hi/lo tiles; narrow tiles store both halves directly
  constexpr int B_STAGE = C::B_STAGE;
  constexpr int NPT = NPW * 32;
  constexpr int RPP = NPT > 0 ? NPT / 8 : 1;
  constexpr int PASSES = BM / RPP;
  constexpr int W_TMA = NPW + 8;                                   // weight-TMA warp (not in MODE_DCN)
  constexpr int W_EPI = NPW + 8 + (MODE == MODE_DCN ? 0 : 1);      // first warp of epilogue group 0

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* a_smem = smem;
  uint8_t* b_smem = smem + STAGES * A_STAGE;
  uint8_t* o_smem = b_smem + STAGES * B_STAGE;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(o_smem + C::OUT_STAGE);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* acc_full = empty_bar + STAGES;     // [2] chunk slot written (chunk parity)
  uint64_t* acc_empty = acc_full + 2;          // [1] chunk slot read
  uint64_t* w1_full = acc_empty + 1;           // HEAD2: [2] 1x1 weight slot loaded
  uint64_t* w1_empty = w1_full + 2;            // HEAD2: [2] 1x1 weight slot read by both consumer warpgroups
  float* sc_s = reinterpret_cast<float*>(o_smem + C::OUT_STAGE + C::BAR_BYTES);
  float* sh_s = sc_s + BLOCK_N;
  uint8_t* prm_smem = reinterpret_cast<uint8_t*>(sh_s + BLOCK_N);      // MODE_DCN only: 9*128 sampling records (36 KB)
  const uint32_t acc_u = smem_u32(prm_smem + C::PRM_BYTES);           // chunk slot [128][ACC_LD] fp32
  const uint32_t w1_u = smem_u32(o_smem);                              // HEAD2: two 1x1 weight slots (Cfg2::W1_STAGE)

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);      // warp-uniform for the compiler as well
  const int lane = threadIdx.x & 31;
  const int ntn = (p.Cout + BLOCK_N - 1) / BLOCK_N;
  const int tiles_x = (p.W + 15) >> 4, tiles_y = (p.H + 7) >> 3;
  const int ntm = PTILE ? p.B * tiles_x * tiles_y : (p.M + BM - 1) / BM;
  const int ntiles = ntn * ntm;
  const int nkb = p.nkb;
  const int HoWo = p.Ho * p.Wo;

  if (warp == NPW && lane == 0) {
    tma_prefetch_desc(&tmap_w);
    if (use_tma_store || HEAD2) tma_prefetch_desc(&tmap_y);
    if (A_TMA) tma_prefetch_desc(&tmap_x);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], A_TMA ? 1 : NPT + 1);
      mbar_init(&empty_bar[s], WIDE ? 4 : 8);                      // released by every consumer warp
    }
    mbar_init(&acc_full[0], 8);
    mbar_init(&acc_full[1], 8);
    mbar_init(&acc_empty[0], 128);                                 // a chunk is read by one epilogue group
    for (int s = 0; s < 2; ++s) {
      mbar_init(&w1_full[s], 1);
      mbar_init(&w1_empty[s], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();

  // ================================================================ epilogue body (run by 1 or 2 warp groups)
  auto run_epilogue = [&](const int group, const int et) {
    const int quad = warp & 3;                          // a permutation of 0..3 over the 4 warps of either group
    const int row = quad * 32 + lane;
    constexpr int CHUNK = C::CHUNK;
    constexpr int NCHUNK = BLOCK_N / CHUNK;
    int use[2] = {0, 0};                                // completed waits per chunk-parity barrier
    constexpr int NGROUPS = EPI_THREADS / 128;
    const bool staged = use_tma_store != 0;             // host guarantees OUT_F16_NHWC && BLOCK_N >= 64
    const uint32_t sc_u = smem_u32(sc_s), sh_u = smem_u32(sh_s), o_u = smem_u32(o_smem);
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
      const int n0 = (t % ntn) * BLOCK_N;
      const int m_tile = t / ntn;
      int m = m_tile * BM + row;
      bool mvalid = m < p.M;
      int tile_b = 0, tile_y0 = 0, tile_x0 = 0;
      if (PTILE) {
        tile_b = m_tile / (tiles_x * tiles_y);
        const int tile_t = m_tile - tile_b * (tiles_x * tiles_y);
        tile_y0 = (tile_t / tiles_x) << 3;
        tile_x0 = (tile_t % tiles_x) << 4;
        const int yy = tile_y0 + (row >> 4), xx = tile_x0 + (row & 15);
        mvalid = yy < p.H && xx < p.W;
        m = (tile_b * p.H + yy) * p.W + xx;
      }
      if (staged && et == 0) bulk_wait_read0();         // previous tile's TMA store has finished reading the staging
      if (et < BLOCK_N) {
        sts32f(sc_u + et * 4, __ldg(p.scale + n0 + et));
        sts32f(sh_u + et * 4, __ldg(p.shift + n0 + et));
      }
      bar_sync_named(1, EPI_THREADS);
#pragma unroll
      for (int ch0 = 0; ch0 < NCHUNK; ch0 += NGROUPS) {
        const int ch = ch0 + group;
        if (ch >= NCHUNK) break;
        float v[CHUNK];
        mbar_wait(&acc_full[ch & 1], use[ch & 1] & 1);
        ++use[ch & 1];
#pragma unroll
        for (int i = 0; i < CHUNK; i += 4) {
          const float4 a4 = lds128f(acc_u + (row * C::ACC_LD + i) * 4);
          v[i] = a4.x; v[i + 1] = a4.y; v[i + 2] = a4.z; v[i + 3] = a4.w;
        }
        mbar_arrive(acc_empty);                          // chunk slot free for the next hand-over
        const int nb = n0 + ch * CHUNK;
#pragma unroll
        for (int i = 0; i < CHUNK; i += 4) {
          const float4 s4 = lds128f(sc_u + (ch * CHUNK + i) * 4);
          const float4 h4 = lds128f(sh_u + (ch * CHUNK + i) * 4);
          v[i] = v[i] * s4.x + h4.x;
          v[i + 1] = v[i + 1] * s4.y + h4.y;
          v[i + 2] = v[i + 2] * s4.z + h4.z;
          v[i + 3] = v[i + 3] * s4.w + h4.w;
        }
        if (p.res != nullptr && mvalid) {
          const __half* rp = p.res + static_cast<long long>(m) * p.res_ld + nb;
#pragma unroll
          for (int i = 0; i < CHUNK; i += 8) {
            if (nb + i < p.Cout) {
              const uint4 rv = __ldg(reinterpret_cast<const uint4*>(rp + i));
              const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(rh[e]);
                v[i + 2 * e] += f.x;
                v[i + 2 * e + 1] += f.y;
              }
              if (split_out) {                                   // residual = hi + lo
                const uint4 rl = __ldg(reinterpret_cast<const uint4*>(rp + p.res_lo + i));
                const __half2* rlh = reinterpret_cast<const __half2*>(&rl);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const float2 f = __half22float2(rlh[e]);
                  v[i + 2 * e] += f.x;
                  v[i + 2 * e + 1] += f.y;
                }
              }
            }
          }
        }
        act_chunk<CHUNK>(v, p.act);
        if (p.out_mode == OUT_F16_NHWC) {
          if (staged) {
            if constexpr (BLOCK_N >= 64) {
              const uint32_t sub = o_u + (ch >> 1) * A_STAGE;
#pragma unroll
              for (int i = 0; i < CHUNK; i += 8) {
                __half2 o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = __floats2half2_rn(v[i + 2 * e], v[i + 2 * e + 1]);
                sts128(sub + sw128_off(row, (ch & 1) * 4 + (i >> 3)), *reinterpret_cast<uint4*>(o));
                if constexpr (SPLIT) {
                  __half2 l[4];
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 h = __half22float2(o[e]);
                    l[e] = __floats2half2_rn(v[i + 2 * e] - h.x, v[i + 2 * e + 1] - h.y);
                  }
                  sts128(sub + C::OUT_HALF + sw128_off(row, (ch & 1) * 4 + (i >> 3)), *reinterpret_cast<uint4*>(l));
                }
              }
            }
          } else if (mvalid) {
            __half* yp = reinterpret_cast<__half*>(p.y) + static_cast<long long>(m) * p.y_ld + nb;
#pragma unroll
            for (int i = 0; i < CHUNK; i += 8) {
              if (nb + i < p.Cout) {
                __half2 o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) o[e] = __floats2half2_rn(v[i + 2 * e], v[i + 2 * e + 1]);
                *reinterpret_cast<uint4*>(yp + i) = *reinterpret_cast<uint4*>(o);
                if (split_out) {
                  __half2 l[4];
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 h = __half22float2(o[e]);
                    l[e] = __floats2half2_rn(v[i + 2 * e] - h.x, v[i + 2 * e + 1] - h.y);
                  }
                  *reinterpret_cast<uint4*>(yp + p.y_lo + i) = *reinterpret_cast<uint4*>(l);
                }
              }
            }
          }
        } else if (mvalid) {
          if (p.out_mode == OUT_F32_NHWC) {
            float* yp = reinterpret_cast<float*>(p.y) + static_cast<long long>(m) * p.y_ld + nb;
#pragma unroll
            for (int i = 0; i < CHUNK; i += 4) {
              if (nb + i < p.y_ld) *reinterpret_cast<float4*>(yp + i) = make_float4(v[i], v[i + 1], v[i + 2], v[i + 3]);
            }
          } else {
            const int b = m / HoWo, pix = m - b * HoWo;
            float* yp = reinterpret_cast<float*>(p.y) + (static_cast<long long>(b) * p.y_ld + nb) * HoWo + pix;
#pragma unroll
            for (int i = 0; i < CHUNK; ++i) {
              if (nb + i < p.Cout) yp[static_cast<long long>(i) * HoWo] = v[i];
            }
          }
        }
      }
      if (staged) {
        fence_proxy_async();
        bar_sync_named(1, EPI_THREADS);
        if (et == 0) {
          if constexpr (BLOCK_N >= 64) {
#pragma unroll
            for (int sidx = 0; sidx < BLOCK_N / 64; ++sidx) {
              if (n0 + sidx * 64 < p.Cout) {
#pragma unroll
                for (int hl = 0; hl < (SPLIT ? 2 : 1); ++hl) {
                  const uint32_t src = smem_u32(o_smem + hl * C::OUT_HALF + sidx * A_STAGE);
                  const int col = n0 + sidx * 64 + hl * p.y_lo;
                  if (PTILE)
                    tma_store_4d(&tmap_y, src, col, tile_x0, tile_y0, tile_b);
                  else
                    tma_store_2d(&tmap_y, src, col, m_tile * BM);
                }
              }
            }
          }
          bulk_commit();
        }
      } else {
        bar_sync_named(1, EPI_THREADS);       // sc_s / sh_s are rewritten by the next tile
      }
    }
    if (staged && et == 0) bulk_wait0();                 // all stores complete before the CTA exits
  };

  if (warp < NPW && A_TMA) {
    run_epilogue(1, 128 + threadIdx.x);                   // second epilogue group (odd 32-column chunks)
  } else if (warp < NPW) {
    // ================================================================ A producers
    const int tid = threadIdx.x;
    const int j = tid & 7;
    const int rsub = tid >> 3;
    int it = 0;                       // running K-block counter (stage = it % STAGES)
    if (MODE == MODE_CONV) {
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int m0 = (t / ntn) * BM;
        int iy0[PASSES], ix0[PASSES];
        long long base[PASSES];
#pragma unroll
        for (int q = 0; q < PASSES; ++q) {
          const int m = m0 + q * RPP + rsub;
          if (m < p.M) {
            const int b = m / HoWo, rem = m - b * HoWo;
            const int oy = rem / p.Wo, ox = rem - oy * p.Wo;
            iy0[q] = oy * p.stride - p.pad;
            ix0[q] = ox * p.stride - p.pad;
            base[q] = (static_cast<long long>(b * p.H + iy0[q]) * p.W + ix0[q]) * p.x_ld;
          } else {
            iy0[q] = -100000; ix0[q] = -100000; base[q] = 0;
          }
        }
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty_bar[s], ((it / STAGES) & 1) ^ 1);
          const int k = kb * BK + j * 8;
          int tap, c0;
          if (p.split_in) {                 // virtual K order: ((tap, chunk), which in {hi.Whi, lo.Whi, hi.Wlo}, channel)
            const int unit = k / p.cw, c = k - unit * p.cw;
            const int tc = unit / 3, which = unit - tc * 3;
            const int nch = p.Cin / p.cw;
            tap = tc / nch;
            c0 = (tc - tap * nch) * p.cw + c + (which == 1 ? p.x_lo : 0);
          } else {
            tap = k / p.Cin;
            c0 = k - tap * p.Cin;
          }
          const int ky = tap / p.kw, kx = tap - ky * p.kw;
          const bool kvalid = k < p.K_real;
          const long long koff = static_cast<long long>(ky * p.W + kx) * p.x_ld + c0;
          const uint32_t a_stage = smem_u32(a_smem + s * A_STAGE);
#pragma unroll
          for (int q = 0; q < PASSES; ++q) {
            const int r = q * RPP + rsub;
            const int iy = iy0[q] + ky, ix = ix0[q] + kx;
            const bool ok = kvalid && iy >= 0 && iy < p.H && ix >= 0 && ix < p.W;
            const __half* src = ok ? p.x + base[q] + koff : p.x;
            cp_async16_ca(a_stage + sw128_off(r, j), src, ok ? 16u : 0u);
          }
          cp_async_commit();
          if (it >= LAG) {
            cp_async_wait<LAG>();
            fence_proxy_async();
            mbar_arrive(&full_bar[(it - LAG) % STAGES]);
          }
        }
      }
      cp_async_wait<0>();
      fence_proxy_async();
      for (int i = (it > LAG ? it - LAG : 0); i < it; ++i) mbar_arrive(&full_bar[i % STAGES]);
    } else {
      // ---------------------------------------------------------- DCNv2 (3x3, stride 1, pad 1, dil 1, dg 1)
      // Phase P, once per tile: every (pixel, tap) gets its sampling record - 4 bilinear weights already multiplied by
      // the modulation mask (0 for corners / samples outside the image, dcn_v2_im2col_cuda.cu:37-48,180) and the 4
      // corner pixel indices (clamped, so the gather needs no predication). The reference recomputes this per channel;
      // the first version of this kernel per 8-channel chunk. Phase G then is pure load / blend / store.
      const uint32_t prm_w = smem_u32(prm_smem);                    // [9*128] float4 weights
      const uint32_t prm_o = prm_w + 9 * BM * 16;                    // [9*128] int4 corner pixel indices
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int m_tile = t / ntn;
        const int n0 = (t % ntn) * BLOCK_N;
        // weight tile of K block kbb into `stage` (thread 0; its arrive_expect_tx is the extra arrival of full_bar)
        auto load_w = [&](int kbb) {
          if (tid == 0) {
            mbar_arrive_expect_tx(&full_bar[stage], B_STAGE);
            const int wk = p.pair ? (3 * (kbb >> 1) + ((kbb & 1) << 1)) : kbb;    // see the weight-TMA warp
            tma_load_2d(smem_u32(b_smem + stage * B_STAGE), &tmap_w, &full_bar[stage], wk * BK, n0);
          }
        };
        const int tile_b = m_tile / (tiles_x * tiles_y);
        const int tile_t = m_tile - tile_b * (tiles_x * tiles_y);
        const int tile_y0 = (tile_t / tiles_x) << 3, tile_x0 = (tile_t % tiles_x) << 4;
        bar_sync_named(2, NPT);                              // previous tile's gather no longer reads the records
        for (int item = tid; item < 9 * BM; item += NPT) {
          const int tap = item >> 7, r = item & (BM - 1);
          const int yy = tile_y0 + (r >> 4), xx = tile_x0 + (r & 15);
          float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
          int4 o = make_int4(0, 0, 0, 0);
          if (yy < p.H && xx < p.W) {
            const float* om = p.offmask + (static_cast<long long>(tile_b * p.H + yy) * p.W + xx) * p.om_ld;
            const int ky = tap / 3, kx = tap - ky * 3;
            const float h_im = static_cast<float>(yy - 1 + ky) + __ldg(om + 2 * tap);
            const float w_im = static_cast<float>(xx - 1 + kx) + __ldg(om + 2 * tap + 1);
            if (h_im > -1.f && w_im > -1.f && h_im < static_cast<float>(p.H) && w_im < static_cast<float>(p.W)) {
              const float mk = __ldg(om + 18 + tap);
              const float hlf = floorf(h_im), wlf = floorf(w_im);
              const float lh = h_im - hlf, lw = w_im - wlf, hh = 1.f - lh, hw = 1.f - lw;
              const int hl = static_cast<int>(hlf), wl = static_cast<int>(wlf), hi = hl + 1, wi = wl + 1;
              const bool tp = hl >= 0, bt = hi <= p.H - 1, lf = wl >= 0, rt = wi <= p.W - 1;
              w.x = (tp && lf) ? hh * hw * mk : 0.f;
              w.y = (tp && rt) ? hh * lw * mk : 0.f;
              w.z = (bt && lf) ? lh * hw * mk : 0.f;
              w.w = (bt && rt) ? lh * lw * mk : 0.f;
              const int hlc = max(hl, 0), hic = min(hi, p.H - 1), wlc = max(wl, 0), wic = min(wi, p.W - 1);
              const int pb = p.x_ld * 2;                      // bytes per pixel: records hold 32-bit BYTE offsets
              o = make_int4((hlc * p.W + wlc) * pb, (hlc * p.W + wic) * pb, (hic * p.W + wlc) * pb, (hic * p.W + wic) * pb);
            }
          }
          sts128f(prm_w + item * 16, w);
          sts128(prm_o + item * 16, make_uint4(o.x, o.y, o.z, o.w));
        }
        bar_sync_named(2, NPT);
        const char* x_img = reinterpret_cast<const char*>(p.x + static_cast<long long>(tile_b) * p.H * p.W * p.x_ld + j * 8);
        int tap = 0, c0 = 0;
        uint32_t dst_off[PASSES];
#pragma unroll
        for (int q = 0; q < PASSES; ++q) dst_off[q] = sw128_off(q * RPP + rsub, j);
        if constexpr (SPLIT) {
          // strict precision: hi and lo halves of the four corners are blended in fp32 ONCE per (tap, 64-channel chunk) and
          // fill the two stages of the pair schedule, (A_hi, W_hi) and (A_lo, W_lo) (see IgemmParams::pair).
          const int lo_bytes = p.x_lo * 2;
          for (int kb = 0; kb < nkb; kb += 2) {
            const char* xb = x_img + c0 * 2;
            const uint32_t rec = (tap * BM + rsub) * 16;
            uint4 hi4[PASSES], lo4[PASSES];
#pragma unroll
            for (int q = 0; q < PASSES; ++q) {
              const float4 wq = lds128f(prm_w + rec + q * RPP * 16);
              const uint4 o = lds128(prm_o + rec + q * RPP * 16);
              uint4 vh[4], vl[4];
              vh[0] = __ldg(reinterpret_cast<const uint4*>(xb + o.x));
              vh[1] = __ldg(reinterpret_cast<const uint4*>(xb + o.y));
              vh[2] = __ldg(reinterpret_cast<const uint4*>(xb + o.z));
              vh[3] = __ldg(reinterpret_cast<const uint4*>(xb + o.w));
              vl[0] = __ldg(reinterpret_cast<const uint4*>(xb + o.x + lo_bytes));
              vl[1] = __ldg(reinterpret_cast<const uint4*>(xb + o.y + lo_bytes));
              vl[2] = __ldg(reinterpret_cast<const uint4*>(xb + o.z + lo_bytes));
              vl[3] = __ldg(reinterpret_cast<const uint4*>(xb + o.w + lo_bytes));
              const float wv[4] = {wq.x, wq.y, wq.z, wq.w};
              // the lo halves are 2^-11 of the value: their blend needs 11 bits only and runs in packed fp16 (HFMA2, no
              // conversions, error 2^-22 of the value); the hi halves are blended in fp32 with the fp32 weights
              __half2 wh2[4];
#pragma unroll
              for (int cn = 0; cn < 4; ++cn) wh2[cn] = __float2half2_rn(wv[cn]);
              __half2* oh = reinterpret_cast<__half2*>(&hi4[q]);
              __half2* ol = reinterpret_cast<__half2*>(&lo4[q]);
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                float2 acc = make_float2(0.f, 0.f);
                __half2 lacc = __hmul2(wh2[0], reinterpret_cast<const __half2*>(&vl[0])[e]);
#pragma unroll
                for (int cn = 0; cn < 4; ++cn) {
                  const float2 fh = __half22float2(reinterpret_cast<const __half2*>(&vh[cn])[e]);
                  acc = f2_fma(make_float2(wv[cn], wv[cn]), fh, acc);
                  if (cn > 0) lacc = __hfma2(wh2[cn], reinterpret_cast<const __half2*>(&vl[cn])[e], lacc);
                }
                float2 r2 = acc;
                const float2 lf = __half22float2(lacc);
                r2.x += lf.x;
                r2.y += lf.y;
                oh[e] = __floats2half2_rn(r2.x, r2.y);
                const float2 hf = __half22float2(oh[e]);
                ol[e] = __floats2half2_rn(r2.x - hf.x, r2.y - hf.y);
              }
            }
#pragma unroll
            for (int which = 0; which < 2; ++which) {
              mbar_wait(&empty_bar[stage], phase ^ 1);
              load_w(kb + which);
              const uint32_t a_stage = smem_u32(a_smem + stage * A_STAGE);
#pragma unroll
              for (int q = 0; q < PASSES; ++q) sts128(a_stage + dst_off[q], which == 1 ? lo4[q] : hi4[q]);
              fence_proxy_async();
              mbar_arrive(&full_bar[stage]);
              if (++stage == STAGES) { stage = 0; phase ^= 1; }
            }
            c0 += BK;
            if (c0 >= p.Cin) { c0 = 0; ++tap; }
          }
        } else
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          load_w(kb);
          const uint32_t a_stage = smem_u32(a_smem + stage * A_STAGE);
          uint4 v[PASSES][4];
          float4 wq[PASSES];
          const char* xb = x_img + c0 * 2;
          const uint32_t rec = (tap * BM + rsub) * 16;
#pragma unroll
          for (int q = 0; q < PASSES; ++q) {               // all loads of the K block first (memory-level parallelism)
            wq[q] = lds128f(prm_w + rec + q * RPP * 16);
            const uint4 o = lds128(prm_o + rec + q * RPP * 16);
            v[q][0] = __ldg(reinterpret_cast<const uint4*>(xb + o.x));
            v[q][1] = __ldg(reinterpret_cast<const uint4*>(xb + o.y));
            v[q][2] = __ldg(reinterpret_cast<const uint4*>(xb + o.z));
            v[q][3] = __ldg(reinterpret_cast<const uint4*>(xb + o.w));
          }
#pragma unroll
          for (int q = 0; q < PASSES; ++q) {
            const __half2* h1 = reinterpret_cast<const __half2*>(&v[q][0]);
            const __half2* h2 = reinterpret_cast<const __half2*>(&v[q][1]);
            const __half2* h3 = reinterpret_cast<const __half2*>(&v[q][2]);
            const __half2* h4 = reinterpret_cast<const __half2*>(&v[q][3]);
            const float2 w1 = make_float2(wq[q].x, wq[q].x), w2 = make_float2(wq[q].y, wq[q].y);
            const float2 w3 = make_float2(wq[q].z, wq[q].z), w4 = make_float2(wq[q].w, wq[q].w);
            __half2 o2[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {                  // two channels per step
              const float2 f1 = __half22float2(h1[e]), f2 = __half22float2(h2[e]);
              const float2 f3 = __half22float2(h3[e]), f4 = __half22float2(h4[e]);
              float2 acc = f2_mul(w1, f1);
              acc = f2_fma(w2, f2, acc);
              acc = f2_fma(w3, f3, acc);
              acc = f2_fma(w4, f4, acc);
              const float2 r2 = acc;
              o2[e] = __floats2half2_rn(r2.x, r2.y);
            }
            sts128(a_stage + dst_off[q], *reinterpret_cast<uint4*>(o2));
          }
          fence_proxy_async();
          mbar_arrive(&full_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
          c0 += BK;
          if (c0 >= p.Cin) { c0 = 0; ++tap; }
        }
      }
    }
  } else if (warp == W_TMA && MODE != MODE_DCN) {
    // ================================================================ weight tiles by TMA (all lanes walk, one issues)
    {
      int stage = 0;
      uint32_t phase = 0;
      int tl = 0;                                       // HEAD2: tiles of this CTA so far (1x1 weight slot = tl & 1)
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int n0 = (t % ntn) * BLOCK_N;
        if constexpr (HEAD2) {
          // the branch's split 1x1 weights for the tile's 128 hidden channels (K blocks 3c = W_hi and 3c + 2 = W_lo of the
          // two 64-channel chunks c, rows = the branch's 32 outputs), before the tile's first K block
          const int slot = tl & 1;
          mbar_wait(&w1_empty[slot], ((tl >> 1) & 1) ^ 1);
          if (elect_one()) {
            mbar_arrive_expect_tx(&w1_full[slot], C::W1_STAGE);
            const int kc = 3 * ((n0 & 255) >> 6), row = (n0 >> 8) * 32;
#pragma unroll
            for (int q = 0; q < 4; ++q)                  // q = 2 lo + chunk
              tma_load_2d(w1_u + slot * C::W1_STAGE + q * C::W1_BOX, &tmap_y, &w1_full[slot],
                          (kc + 3 * (q & 1) + 2 * (q >> 1)) * BK, row);
          }
          __syncwarp();
          ++tl;
        }
        int cw = 0, chh = 0, cn = 0;
        if (A_TMA) {                              // coordinates of the tile's first output pixel in input space (incl. -pad)
          const int m0 = (t / ntn) * BM;
          cn = m0 / HoWo;
          const int rem = m0 - cn * HoWo;
          const int oy = rem / p.Wo, ox = rem - oy * p.Wo;
          cw = ox * p.stride - p.pad;
          chh = oy * p.stride - p.pad;
        }
        int c0 = 0, kx = 0, ky = 0;                     // running (tap, channel) cursor: no divisions in the K loop
        int lo = 0;                                     // pair schedule: 0 = the A_hi stage, 1 = the A_lo stage
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          const bool issuer = elect_one();
          if (issuer) mbar_arrive_expect_tx(&full_bar[stage], A_TMA ? A_STAGE + B_STAGE : B_STAGE);
          if (A_TMA) {
            if (issuer)
              tma_load_im2col_4d(smem_u32(a_smem + stage * A_STAGE), &tmap_x, &full_bar[stage], c0 + (lo ? p.x_lo : 0), cw, chh,
                                 cn, static_cast<uint16_t>(kx), static_cast<uint16_t>(ky));
            if (!p.split_in || ++lo == 2) {
              lo = 0;
              c0 += BK;
              if (c0 >= p.Cin) {
                c0 = 0;
                if (++kx == p.kw) { kx = 0; ++ky; }
              }
            }
          }
          // weight K coordinate: plain = K block kb; pair schedule = block 3*(kb/2) (W_hi) for the hi stage and 3*(kb/2)+2
          // (W_lo) for the lo stage of the same (tap, chunk)
          const int wk = p.pair ? (3 * (kb >> 1) + ((kb & 1) << 1)) : kb;
          if (issuer) tma_load_2d(smem_u32(b_smem + stage * B_STAGE), &tmap_w, &full_bar[stage], wk * BK, n0);
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp < NPW + 8) {
    // ================================================================ consumers: warpgroup wg issues the wgmmas of tile rows
    // [64 wg, 64 wg + 64) and hands its accumulators to the epilogue chunk by chunk. Every MMA batch is waited for before
    // the stage it read is released (empty barriers count the consumer warps). WIDE: the one warpgroup issues every MMA
    // twice, rows [0, 64) into d and rows [64, 128) into d1, so each row sees the MMA sequence of the two-warpgroup kernel.
    {
      const int wg = (warp - NPW) >> 2;
      float d[BLOCK_N / 2];
      float d1[WIDE ? BLOCK_N / 2 : 1];
      auto mma = [&](uint64_t ad, uint64_t bd, uint32_t accum) {
        Gmma<BLOCK_N>::template mma<0, 0>(d, ad, bd, accum);
        if constexpr (WIDE) Gmma<BLOCK_N>::template mma<0, 0>(d1, ad + ((64 * 128) >> 4), bd, accum);
      };
      auto done = [&]() {
        gmma_commit();
        gmma_wait<0>();
        gmma_hold(d);
        if constexpr (WIDE) gmma_hold(d1);
        __syncwarp();
      };
      auto release = [&](uint64_t* bar) { if (lane == 0) mbar_arrive(bar); };
      // Descriptors are "base + small delta": everything except the 14-bit start-address field is loop invariant, and
      // the field is linear in the byte address, so the hot loop only does 64-bit adds.
      uint64_t a_d0[BK / 16];
      const uint32_t b0 = smem_u32(b_smem);
      const uint32_t a0 = smem_u32(a_smem) + wg * 64 * 128;           // this warpgroup's rows
#pragma unroll
      for (int k4 = 0; k4 < BK / 16; ++k4) a_d0[k4] = gmma_desc_sw128(a0 + k4 * 32);
      const uint64_t b_d0 = gmma_desc_sw128(b0);
      int stage = 0, fills = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        gmma_fence();
        if (p.pair) {
          // pair schedule: stage s0 = (A_hi, W_hi), stage s1 = (A_lo, W_lo) of one (tap, 64-channel chunk); three products
          for (int kb = 0; kb < nkb; kb += 2) {
            const int s0 = stage;
            mbar_wait(&full_bar[s0], phase);
            const uint64_t a0s = static_cast<uint64_t>((s0 * A_STAGE) >> 4), b0s = static_cast<uint64_t>((s0 * B_STAGE) >> 4);
#pragma unroll
            for (int k4 = 0; k4 < BK / 16; ++k4)                                     // A_hi W_hi
              mma(a_d0[k4] + a0s, b_d0 + b0s + 2 * k4, (kb | k4) != 0 ? 1u : 0u);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
            const int s1 = stage;
            mbar_wait(&full_bar[s1], phase);
            const uint64_t a1 = static_cast<uint64_t>((s1 * A_STAGE) >> 4), b1s = static_cast<uint64_t>((s1 * B_STAGE) >> 4);
#pragma unroll
            for (int k4 = 0; k4 < BK / 16; ++k4)                                     // A_lo W_hi
              mma(a_d0[k4] + a1, b_d0 + b0s + 2 * k4, 1u);
#pragma unroll
            for (int k4 = 0; k4 < BK / 16; ++k4)                                     // A_hi W_lo
              mma(a_d0[k4] + a0s, b_d0 + b1s + 2 * k4, 1u);
            done();
            release(&empty_bar[s0]);
            release(&empty_bar[s1]);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        } else
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint64_t a_off = static_cast<uint64_t>((stage * A_STAGE) >> 4);
          const uint64_t b_off = static_cast<uint64_t>((stage * B_STAGE) >> 4);
#pragma unroll
          for (int k4 = 0; k4 < BK / 16; ++k4) mma(a_d0[k4] + a_off, b_d0 + b_off + 2 * k4, (kb | k4) != 0 ? 1u : 0u);
          done();
          release(&empty_bar[stage]);
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
        if constexpr (HEAD2) {
          // ---- 1x1 heads on the tensor cores, straight from the accumulators: IABN affine + leaky ReLU, split into fp16
          // pairs (the same expressions the hi/lo output of every strict layer uses), then per 16-channel k slice
          // A_hi W_hi + A_lo W_hi + A_hi W_lo as m64n32k16 with A in registers (Gmma<32>::mma_rs), over the slot the
          // weight-TMA warp filled at the tile's start
          const int n0 = (t % ntn) * BLOCK_N, m_tile = t / ntn;
          const int branch = n0 >> 8, nout = p.h2_nch[branch];
          const int tq = lane & 3;
          const int row0 = m_tile * BM + wg * 64 + ((warp - NPW) & 3) * 16 + (lane >> 2);   // rows row0 and row0 + 8
          uint32_t ahi[BLOCK_N / 16][4], alo[BLOCK_N / 16][4];
#pragma unroll
          for (int j = 0; j < BLOCK_N / 8; ++j) {
            const float2 s2 = __ldg(reinterpret_cast<const float2*>(p.scale + n0 + 8 * j + 2 * tq));
            const float2 h2 = __ldg(reinterpret_cast<const float2*>(p.shift + n0 + 8 * j + 2 * tq));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float v0 = d[4 * j + 2 * h] * s2.x + h2.x, v1 = d[4 * j + 2 * h + 1] * s2.y + h2.y;
              v0 = fmaxf(v0, 0.01f * v0);
              v1 = fmaxf(v1, 0.01f * v1);
              const __half2 hi = __floats2half2_rn(v0, v1);
              const float2 hf = __half22float2(hi);
              const __half2 lo = __floats2half2_rn(v0 - hf.x, v1 - hf.y);
              ahi[j >> 1][2 * (j & 1) + h] = *reinterpret_cast<const uint32_t*>(&hi);
              alo[j >> 1][2 * (j & 1) + h] = *reinterpret_cast<const uint32_t*>(&lo);
            }
          }
          // the next tile's first MMA does not read d (scale-d = 0), but its asm operands do: without this the old
          // accumulators stay live through the tail, and ptxas spills and serializes every wgmma of the kernel
#pragma unroll
          for (int i = 0; i < BLOCK_N / 2; ++i) d[i] = 0.f;
          const int slot = fills & 1;
          mbar_wait(&w1_full[slot], (fills >> 1) & 1);
          const uint32_t wb = w1_u + slot * C::W1_STAGE;
          float o[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) o[i] = 0.f;
          gmma_fence();
#pragma unroll
          for (int s = 0; s < BLOCK_N / 16; ++s) {
            const uint32_t bw = wb + (s >> 2) * C::W1_BOX + (s & 3) * 32;
            const uint64_t bhi = gmma_desc_sw128(bw), blo = gmma_desc_sw128(bw + 2 * C::W1_BOX);
            Gmma<32>::mma_rs<0>(o, ahi[s], bhi, s != 0 ? 1u : 0u);
            Gmma<32>::mma_rs<0>(o, alo[s], bhi, 1u);
            Gmma<32>::mma_rs<0>(o, ahi[s], blo, 1u);
          }
          gmma_commit();
          gmma_wait<0>();
          gmma_hold(o);
          __syncwarp();
          if (lane == 0) mbar_arrive(&w1_empty[slot]);
          ++fills;
          // partial sums of the tile's 128 hidden channels -> plane (n0 & 255) >> 7; o[4 j + 2 h + e] is output 8 j + 2 tq + e
          // of row row0 + 8 h, so a quad's 8 rows fill one 32-byte sector of each output's plane
          float* part = p.h2_part + (static_cast<long long>((n0 & 255) >> 7) * p.B * p.h2_ntot + p.h2_ch0[branch]) * HoWo;
          const int hc = p.h2_hid_col[branch];
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int m = row0 + 8 * h;
            if (m < p.M) {
              const int bimg = m / HoWo, pix = m - bimg * HoWo;
              float* dst = part + static_cast<long long>(bimg) * p.h2_ntot * HoWo + pix;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                  const int oc = 8 * j + 2 * tq + e;
                  if (oc < nout) dst[static_cast<long long>(oc) * HoWo] = o[4 * j + 2 * h + e];
                }
              }
              // hidden pair rows for the edge fusion: two branches only, border pixels only
              if (hc >= 0 && p.h2_mask[m] != 0) {
                __half* yp = reinterpret_cast<__half*>(p.y) + static_cast<long long>(m) * p.y_ld + hc + (n0 & 255) + 2 * tq;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                  *reinterpret_cast<uint32_t*>(yp + 8 * j) = ahi[j >> 1][2 * (j & 1) + h];
                  *reinterpret_cast<uint32_t*>(yp + p.y_lo + 8 * j) = alo[j >> 1][2 * (j & 1) + h];
                }
              }
            }
          }
        } else if constexpr (WIDE) {
          // ---- the tile's epilogue from the accumulator fragments: scale/shift, activation, fp16 (strict: the hi/lo pair,
          // the expressions of run_epilogue), then the swizzled staging and one 4-D TMA store per half, or direct stores
          // (no residual: the DCN entry points have none). d[4 j + 2 h + e] is row 16 w + l / 4 + 8 h, column 8 j + 2 tq + e.
          const int n0 = (t % ntn) * BLOCK_N, m_tile = t / ntn;
          const int tile_b = m_tile / (tiles_x * tiles_y);
          const int tile_t = m_tile - tile_b * (tiles_x * tiles_y);
          const int tile_y0 = (tile_t / tiles_x) << 3, tile_x0 = (tile_t % tiles_x) << 4;
          const int et = threadIdx.x & 127, tq = lane & 3;
          const bool staged = SPLIT || use_tma_store != 0;    // host guarantees OUT_F16_NHWC (strict: always staged)
          const uint32_t sc_u = smem_u32(sc_s), sh_u = smem_u32(sh_s), o_u = smem_u32(o_smem);
          if (staged && et == 0) bulk_wait_read0();           // previous tile's TMA store has finished reading the staging
          if (et < BLOCK_N) {
            sts32f(sc_u + et * 4, __ldg(p.scale + n0 + et));
            sts32f(sh_u + et * 4, __ldg(p.shift + n0 + et));
          }
          bar_sync_named(1, 128);
          // one walk over the fragments per output form (the form is chosen outside the loop, so the rarely used direct
          // stores cost the staged path no registers); store(row, j, nb, v) writes columns nb, nb + 1 of tile row `row`
          auto finish = [&](auto&& store) {
#pragma unroll
            for (int mh = 0; mh < 2; ++mh) {
              float(&dh)[BLOCK_N / 2] = mh == 0 ? d : d1;
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const int row = 64 * mh + 16 * (warp - NPW) + (lane >> 2) + 8 * h;
#pragma unroll
                for (int j = 0; j < BLOCK_N / 8; ++j) {
                  const int nb = n0 + 8 * j + 2 * tq;
                  const float2 s2 = lds64f(sc_u + (nb - n0) * 4), h2 = lds64f(sh_u + (nb - n0) * 4);
                  float v[2];
                  v[0] = dh[4 * j + 2 * h] * s2.x + h2.x;
                  v[1] = dh[4 * j + 2 * h + 1] * s2.y + h2.y;
                  // the next tile's first MMA does not read the accumulators (scale-d = 0), but its asm operands do:
                  // zeroed, they need no registers through the rest of the epilogue (see HEAD2)
                  dh[4 * j + 2 * h] = 0.f;
                  dh[4 * j + 2 * h + 1] = 0.f;
                  act_chunk<2>(v, p.act);
                  store(row, j, nb, v);
                }
              }
            }
          };
          // pixel of tile row r: image tile_b, (y, x) = (tile_y0 + r / 16, tile_x0 + r % 16); false outside the image
          auto pixel = [&](int r, long long& m, int& yx) {
            const int yy = tile_y0 + (r >> 4), xx = tile_x0 + (r & 15);
            yx = yy * p.W + xx;
            m = static_cast<long long>(tile_b) * HoWo + yx;
            return yy < p.H && xx < p.W;
          };
          if (staged) {
            finish([&](int row, int j, int nb, const float (&v)[2]) {
              const __half2 hi = __floats2half2_rn(v[0], v[1]);
              const uint32_t off = sw128_off(row, j) + 4 * tq;
              sts32(o_u + off, *reinterpret_cast<const uint32_t*>(&hi));
              if constexpr (SPLIT) {
                const float2 hf = __half22float2(hi);
                const __half2 lo = __floats2half2_rn(v[0] - hf.x, v[1] - hf.y);
                sts32(o_u + C::OUT_HALF + off, *reinterpret_cast<const uint32_t*>(&lo));
              }
            });
            fence_proxy_async();
            bar_sync_named(1, 128);
            if (et == 0) {
              if (n0 < p.Cout) {
#pragma unroll
                for (int hl = 0; hl < (SPLIT ? 2 : 1); ++hl)
                  tma_store_4d(&tmap_y, o_u + hl * C::OUT_HALF, n0 + hl * p.y_lo, tile_x0, tile_y0, tile_b);
              }
              bulk_commit();
            }
          } else if constexpr (!SPLIT) {
            // the column guards of run_epilogue: fp16 per 8-column group, fp32 NHWC per 4-column group against the row
            // stride, fp32 NCHW per column
            if (p.out_mode == OUT_F16_NHWC) {
              finish([&](int row, int j, int nb, const float (&v)[2]) {
                long long m;
                int yx;
                if (pixel(row, m, yx) && n0 + 8 * j < p.Cout)
                  *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(p.y) + m * p.y_ld + nb) = __floats2half2_rn(v[0], v[1]);
              });
            } else if (p.out_mode == OUT_F32_NHWC) {
              finish([&](int row, int j, int nb, const float (&v)[2]) {
                long long m;
                int yx;
                if (pixel(row, m, yx) && (nb & ~3) < p.y_ld)
                  *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.y) + m * p.y_ld + nb) = make_float2(v[0], v[1]);
              });
            } else {
              finish([&](int row, int j, int nb, const float (&v)[2]) {
                long long m;
                int yx;
                if (pixel(row, m, yx)) {
                  float* yp = reinterpret_cast<float*>(p.y) + (static_cast<long long>(tile_b) * p.y_ld + nb) * HoWo + yx;
                  if (nb < p.Cout) yp[0] = v[0];
                  if (nb + 1 < p.Cout) yp[HoWo] = v[1];
                }
              });
            }
            bar_sync_named(1, 128);                           // sc_s / sh_s are rewritten by the next tile
          }
        } else {
          // hand-over: one chunk slot, chunk parity selects the full barrier (with two epilogue groups each waits on its own)
          ChunkDump<BLOCK_N, C::CHUNK, 0>::run(d, [&](int ch, auto store) {
            mbar_wait(acc_empty, (fills & 1) ^ 1);
            store(acc_u + wg * 64 * C::ACC_LD * 4, C::ACC_LD);
            __syncwarp();
            if (lane == 0) mbar_arrive(&acc_full[ch & 1]);
            ++fills;
          });
        }
      }
      if constexpr (WIDE) {
        if (use_tma_store && (threadIdx.x & 127) == 0) bulk_wait0();   // all stores complete before the CTA exits
      }
    }
  } else if constexpr (!HEAD2 && !WIDE) {
    run_epilogue(0, (warp - W_EPI) * 32 + lane);          // first epilogue group (even chunks, or all of them)
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled2 encode_fn() {
  static PFN_encodeTiled2 fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
      set_error("cuTensorMapEncodeTiled entry point unavailable");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiled2>(ptr);
  }
  return fn;
}

typedef CUresult (*PFN_encodeIm2col)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                     CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                     CUtensorMapFloatOOBfill);

static PFN_encodeIm2col encode_im2col_fn() {
  static PFN_encodeIm2col fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
      set_error("cuTensorMapEncodeIm2col entry point unavailable");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeIm2col>(ptr);
  }
  return fn;
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

template <int BLOCK_N, int MODE, int NPW, int EPI = 0>
static int launch2_cfg(const CUtensorMap& tw, const CUtensorMap& ty, const CUtensorMap& tx, const IgemmParams& p,
                       int use_tma_store, cudaStream_t st) {
  using C = Cfg2<BLOCK_N, MODE, EPI, igemm2_wide(MODE, NPW)>;
  auto kern = igemm2_kernel<BLOCK_N, MODE, NPW, EPI>;
  static bool attr = false;
  if (!attr) {
    if (check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM), "smem attr")) return -1;
    attr = true;
  }
  const int ntn = (p.Cout + BLOCK_N - 1) / BLOCK_N;
  const int ntm = MODE == MODE_DCN ? p.B * ((p.H + 7) / 8) * ((p.W + 15) / 16) : (p.M + BM - 1) / BM;
  int grid = num_sms() * C::CTAS_PER_SM;
  if (grid > ntn * ntm) grid = ntn * ntm;
  return check_cuda(launch_k(kern, dim3(grid), dim3(igemm2_warps(MODE, NPW, EPI) * 32), C::SMEM, st, tw, ty, tx, p,
                             use_tma_store),
                    "igemm2 launch");
}

// out[b, ch, pix] = bias[ch] + plane 0 + plane 1 (fixed order: deterministic), ch < ncls -> cls, else reg
__global__ void head2_reduce_kernel(const float* __restrict__ part, const float* __restrict__ bias, float* __restrict__ cls,
                                    float* __restrict__ reg, int B, int ncls, int nreg, int HW) {
  const int ntot = ncls + nreg;
  const long long plane = static_cast<long long>(B) * ntot * HW;
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i >= plane) return;
  float4 s = __ldg(reinterpret_cast<const float4*>(part + i));
  const float4 t = __ldg(reinterpret_cast<const float4*>(part + plane + i));
  s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
  const long long row = i / HW;                       // HW % 4 == 0 is checked by the launcher: 4 elements share (b, ch)
  const int ch = static_cast<int>(row % ntot), b = static_cast<int>(row / ntot);
  const int pix = static_cast<int>(i - row * HW);
  const float bv = __ldg(bias + ch);
  s.x += bv; s.y += bv; s.z += bv; s.w += bv;
  float* dst = ch < ncls ? cls + (static_cast<long long>(b) * ncls + ch) * HW + pix
                         : reg + (static_cast<long long>(b) * nreg + (ch - ncls)) * HW + pix;
  *reinterpret_cast<float4*>(dst) = s;
}

int launch_igemm2(const IgemmParams& p, const __half* wp, int n_pad, int k_pad, int mode, cudaStream_t st) {
  PFN_encodeTiled2 enc = encode_fn();
  if (!enc) return -1;
  // HEAD2 tiles: 128 columns (a 256-column tile would need 128 accumulator registers per consumer thread)
  const int bn = p.h2_w != nullptr ? 128 : mf_conv_block_n(p.Cout);
  const bool store_ok = p.out_mode == OUT_F16_NHWC && bn >= 64 && (reinterpret_cast<uintptr_t>(p.y) & 15) == 0 && p.y_ld % 8 == 0;
  if (p.act == ACT_OFFMASK) { set_error("igemm2: the offset/mask convolution runs in mf_offset_conv.cu"); return -1; }
  if (n_pad % bn != 0 || k_pad % BK != 0 || k_pad < p.nkb * BK) {
    set_error("igemm: packed weight shape [%d,%d] incompatible with block_n=%d nkb=%d", n_pad, k_pad, bn, p.nkb);
    return -1;
  }
  if (mode == MODE_DCN && (p.Cin % 64 != 0 || p.kh != 3 || p.kw != 3 || p.stride != 1 || p.pad != 1)) {
    set_error("dcn igemm: only 3x3 s1 p1 with Cin %% 64 == 0 is built (got Cin=%d)", p.Cin);
    return -1;
  }
  if (mode == MODE_DCN && (p.split_in != p.split_out || (p.split_in && p.out_mode != OUT_F16_NHWC))) {
    set_error("dcn igemm: strict precision needs split input AND split fp16 output");
    return -1;
  }
  if (p.split_in && (p.cw <= 0 || p.Cin % p.cw != 0 || (p.cw != 64 && 64 % p.cw != 0) || p.x_lo % 8 != 0)) {
    set_error("igemm: split input needs Cin %% 64 == 0 or Cin in {8,16,32} and an 8-aligned lo offset (Cin=%d cw=%d)", p.Cin, p.cw);
    return -1;
  }
  if (p.split_out && (p.out_mode != OUT_F16_NHWC || p.y_lo % 8 != 0 || (p.res != nullptr && p.res_lo % 8 != 0))) {
    set_error("igemm: split output needs fp16 NHWC rows and 8-aligned lo offsets");
    return -1;
  }
  if (mode == MODE_CONV && (p.Cin % 8 != 0 || p.x_ld % 8 != 0)) {
    set_error("conv igemm: Cin and pixel stride must be multiples of 8 (got %d, %d)", p.Cin, p.x_ld);
    return -1;
  }
  CUtensorMap tw, ty;
  {
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(k_pad), static_cast<cuuint64_t>(n_pad)};
    cuuint64_t gstr[1] = {static_cast<cuuint64_t>(k_pad) * 2};
    cuuint32_t box[2] = {BK, static_cast<cuuint32_t>(bn)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tw, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(wp), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weights) failed (%d)", static_cast<int>(r)); return -1; }
  }
  int use_tma_store = 0;
  ty = tw;
  if (store_ok) {
    CUresult r;
    if (mode == MODE_DCN) {
      cuuint64_t gdim[4] = {static_cast<cuuint64_t>(p.Cout + (p.split_out ? p.y_lo : 0)), static_cast<cuuint64_t>(p.W),
                            static_cast<cuuint64_t>(p.H), static_cast<cuuint64_t>(p.B)};
      cuuint64_t gstr[3] = {static_cast<cuuint64_t>(p.y_ld) * 2, static_cast<cuuint64_t>(p.y_ld) * 2 * p.W,
                            static_cast<cuuint64_t>(p.y_ld) * 2 * p.W * p.H};
      cuuint32_t box[4] = {64, 16, 8, 1};
      cuuint32_t estr[4] = {1, 1, 1, 1};
      r = enc(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, p.y, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    } else {
      cuuint64_t gdim[2] = {static_cast<cuuint64_t>(p.Cout + (p.split_out ? p.y_lo : 0)), static_cast<cuuint64_t>(p.M)};
      cuuint64_t gstr[1] = {static_cast<cuuint64_t>(p.y_ld) * 2};
      cuuint32_t box[2] = {64, BM};
      cuuint32_t estr[2] = {1, 1};
      r = enc(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, p.y, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
              CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    }
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(output) failed (%d)", static_cast<int>(r)); return -1; }
    use_tma_store = 1;
  }
  // A operand by im2col-mode TMA whenever a K block is one (tap, 64-channel) box. Narrower im2col boxes are request-bound
  // inside the TMA unit (measured: the 7x7 stem 1.8x slower than the cp.async gather), so Cin < 64 layers stay on the gather
  // producers.
  CUtensorMap tx = tw;
  bool a_tma = false;
  IgemmParams pp = p;
  if (mode == MODE_CONV && p.Cin % 64 == 0 && (reinterpret_cast<uintptr_t>(p.x) & 15) == 0 && p.kw <= 16 && p.kh <= 16 &&
      p.stride <= 8) {
    PFN_encodeIm2col enc2 = encode_im2col_fn();
    if (!enc2) return -1;
    cuuint64_t gdim[4] = {static_cast<cuuint64_t>(p.Cin + (p.split_in ? p.x_lo : 0)), static_cast<cuuint64_t>(p.W),
                          static_cast<cuuint64_t>(p.H), static_cast<cuuint64_t>(p.B)};
    cuuint64_t gstr[3] = {static_cast<cuuint64_t>(p.x_ld) * 2, static_cast<cuuint64_t>(p.x_ld) * 2 * p.W,
                          static_cast<cuuint64_t>(p.x_ld) * 2 * p.W * p.H};
    int lower[2] = {-p.pad, -p.pad};
    int upper[2] = {p.pad - (p.kw - 1), p.pad - (p.kh - 1)};
    cuuint32_t estr[4] = {1, static_cast<cuuint32_t>(p.stride), static_cast<cuuint32_t>(p.stride), 1};
    CUresult r = enc2(&tx, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<__half*>(p.x), gdim, gstr, lower, upper, BK, BM, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeIm2col failed (%d)", static_cast<int>(r)); return -1; }
    a_tma = true;
  }
  if (p.split_in && (mode == MODE_DCN || a_tma)) {
    pp.pair = 1;                                                   // see IgemmParams::pair
    pp.nkb = 2 * p.kh * p.kw * (p.Cin / 64);
  }
  if (p.h2_w != nullptr) {                     // HEAD2: the strict-precision predictor GEMM (see IgemmParams)
    if (!(a_tma && pp.pair && p.Cout % 256 == 0 && p.h2_part != nullptr && p.Cout / 256 <= 12 && p.act == ACT_LEAKY)) {
      set_error("igemm2 HEAD2: needs the pair-schedule TMA path, Cout a multiple of 256 and the leaky activation");
      return -1;
    }
    // the split 1x1 head weights [nbranch * 32][768]: boxes of 64 K x 32 outputs, 128B-swizzled like the B operand
    cuuint64_t gdim[2] = {3 * 256, static_cast<cuuint64_t>(p.Cout / 256 * 32)};
    cuuint64_t gstr[1] = {3 * 256 * 2};
    cuuint32_t box[2] = {BK, 32};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&ty, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(p.h2_w), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(1x1 head weights) failed (%d)", static_cast<int>(r)); return -1; }
    return launch2_cfg<128, MODE_CONV_TMA, 0, 2>(tw, ty, tx, pp, 0, st);
  }
  if (p.split_out && use_tma_store) {          // staged hi/lo tiles: the SPLIT instantiations (N tiles of 64 / 128 only)
    if (mode == MODE_DCN && bn == 64) return launch2_cfg<64, MODE_DCN, 16, 1>(tw, ty, tx, pp, use_tma_store, st);
    if (mode == MODE_DCN && bn == 128) return launch2_cfg<128, MODE_DCN, 8, 1>(tw, ty, tx, pp, use_tma_store, st);
    if (a_tma && bn == 64) return launch2_cfg<64, MODE_CONV_TMA, 4, 1>(tw, ty, tx, pp, use_tma_store, st);
    if (a_tma && bn == 128) return launch2_cfg<128, MODE_CONV_TMA, 4, 1>(tw, ty, tx, pp, use_tma_store, st);
    if (bn == 64) return launch2_cfg<64, MODE_CONV, 4, 1>(tw, ty, tx, pp, use_tma_store, st);
    if (bn == 128) return launch2_cfg<128, MODE_CONV, 4, 1>(tw, ty, tx, pp, use_tma_store, st);
  }
  if (mode == MODE_DCN && p.split_in) { set_error("dcn igemm: strict precision needs the staged TMA-store epilogue"); return -1; }
  // DCN producer warps: 16 (the wide-gather configuration) for 64-column tiles, 8 otherwise
#define MF_DISPATCH2(BN, DCN_NPW)                                                                        \
  if (bn == BN) {                                                                                        \
    if (mode == MODE_DCN) return launch2_cfg<BN, MODE_DCN, DCN_NPW>(tw, ty, tx, pp, use_tma_store, st);  \
    if (a_tma) return launch2_cfg<BN, MODE_CONV_TMA, 4>(tw, ty, tx, pp, use_tma_store, st);               \
    return launch2_cfg<BN, MODE_CONV, 4>(tw, ty, tx, pp, use_tma_store, st);                              \
  }
  MF_DISPATCH2(16, 8)
  MF_DISPATCH2(32, 8)
  MF_DISPATCH2(64, 16)
  MF_DISPATCH2(128, 8)
#undef MF_DISPATCH2
  set_error("igemm2: unsupported block_n %d", bn);
  return -1;
}

}  // namespace mf

using namespace mf;

extern "C" {

int mf_head2_reduce(const float* part, const float* bias, float* cls, float* reg, int B, int ncls, int nreg, int HW, void* stream) {
  if (HW % 4 != 0) { set_error("head2_reduce: H*W must be a multiple of 4"); return -1; }
  const long long n4 = static_cast<long long>(B) * (ncls + nreg) * HW / 4;
  (void)launch_k(head2_reduce_kernel, dim3(static_cast<unsigned>((n4 + 255) / 256)), dim3(256), 0, MF_STREAM(stream), part, bias,
                 cls, reg, B, ncls, nreg, HW);
  return check_cuda(cudaGetLastError(), "head2_reduce");
}

}  // extern "C"
