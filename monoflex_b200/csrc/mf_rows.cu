// "Row-segment" convolution for the full-resolution stem (base_layer 7x7 3->16, level0 3x3 16->16, level1 3x3/2 16->32,
// dla_dcn.py:268-282): tensors whose pixels are 16 bytes (8 fp16 channels) are kept as planes [B][H][G][Wg][8]
// (G = channel-planes x column-parities), and the implicit-GEMM A operand is never materialised:
//
//   * a tile is R consecutive output rows (R = 1..4, picked on the host per layer) x 128 consecutive pixels of one image;
//     the TMA warp loads each input row segment the R rows need ONCE ((R - 1) * stride + kh rows per plane and parity,
//     144 pixels x 16 B, two tiled cp.async.bulk.tensor boxes of 8-byte elements per segment, zero fill outside the image);
//   * a consumer warpgroup reads the im2col matrix *through descriptors* (wgmma, two 64-pixel halves per row): with the
//     no-swizzle K-major layout a core matrix is 8 rows x 16 B with rows 16 B apart, which is exactly "8 consecutive
//     pixels" of a segment, so
//       A[r, tap kx] = segment[(r + kx) * 16 B]      -> start address + kx*16, SBO = 128 (8 pixels)
//     and the second 16-byte K chunk of an MMA (the next tap for Cin = 8, the second channel plane for Cin = 16) is
//     reached through LBO. A 7x7 conv is 25 MMAs per row, a 3x3 one 9 - no 49x / 9x copies through L1/L2. Output row r
//     of the tile runs the same MMA table with every A start moved by r x `row_bytes` (its input rows lie stride rows
//     further down the stage);
//   * stride 2 works on column-parity planes (pixel 2*ox + kx - 1 = parity (kx+1)&1, index ox + (kx-1)>>1);
//   * the whole packed weight matrix stays resident in smem (<= 40 KB); two consumer warpgroups take alternate tiles, each
//     with its accumulators in registers: while one runs the epilogue of a row (scale/shift + ReLU -> the planar layout of
//     the next stem layer or plain NHWC rows), the other issues its MMAs, and the TMA warp fetches the next tiles'
//     segments. (One warpgroup that commits row r + 1's MMAs before row r's epilogue, wgmma.wait_group 1, is what ptxas
//     serialises: its accumulator reads fall between the start and end of a wgmma pipeline stage.)
//   * MERGE (strict precision): the tap sets that read the same A rows are stacked along N and issued as ONE MMA per A
//     operand; columns [0, NOUT) and [NOUT, 2 NOUT) of the accumulator are two partial sums of the same outputs, added in
//     fp32 (first half + second half) before scale/shift.
#include "mf_common.cuh"
#include "mf_kernels.h"
#include "../../include/monoflex_b200.h"
#include <cstring>

namespace mf {

static constexpr int RBM = 128;
static constexpr int SEG_PIX = 144;                // 128 + 2 x 4 halo, rounded so that half a segment is a multiple of 128 B
static constexpr int SEG_BYTES = SEG_PIX * 16;     // 2304 = 18 * 128
static constexpr int R_STAGES = 6;
static constexpr int MAX_ROWS = 4;          // output rows per tile
static constexpr int MAX_SEG = 40;          // stride 2 at 2 rows: 5 input rows x 4 planes (hi0 hi1 lo0 lo1) x 2 column parities
static constexpr int MAX_MMA = 56;          // MMA table entries per output row (7x7: 25, strict 3x3: 18)
static constexpr int NWG = 2;               // consumer warpgroups per CTA, on alternating tiles; the TMA warp follows them
static constexpr int ROWS_THREADS = NWG * 128 + 32;
static_assert(R_STAGES % NWG == 0, "the ring depth cap must keep every stage with one consumer warpgroup");

struct RowsParams {
  int B, H, Gin, Wg_in;          // input planes [B][H][Gin][Wg_in][8]
  int Ho, Wo, stride, pad;
  int rows;                      // output rows per tile; bands of `rows` rows never cross into the next image
  int row_bytes;                 // stage bytes from the segments of output row r to those of row r + 1
  int nseg, nmma, nkb;           // nkb = k_pad / 64 weight K blocks
  int nstages;                   // row-segment ring depth (<= R_STAGES), sized on the host
  int seg_g[MAX_SEG], seg_dy[MAX_SEG], seg_dx[MAX_SEG];      // group, input row = oy0*stride + dy, start index = ox0 + dx
  int mma_a[MAX_MMA], mma_lbo[MAX_MMA], mma_b[MAX_MMA];      // byte offsets (output row 0): A start in the stage, LBO, B start
  int Cout;
  const float* scale;
  const float* shift;
  int act;
  int out_planar;                // 1: y = [B][Ho][Cout/8 * out_npar][Wo/out_npar][8]; 0: NHWC rows with y_ld
  int out_npar;
  __half* y;
  int y_ld;
  int split_out;                 // strict precision: output = fp16 pair (hi planes then lo planes / lo block y_lo after hi)
  int y_lo;
};

template <int BLOCK_N, bool MERGE>
__global__ void __launch_bounds__(ROWS_THREADS, BLOCK_N == 64 ? 1 : 2)
rows_conv_kernel(const __grid_constant__ CUtensorMap tmap_x, const __grid_constant__ CUtensorMap tmap_w,
                 const __grid_constant__ RowsParams p) {
  constexpr int NOUT = MERGE ? BLOCK_N / 2 : BLOCK_N;        // output channels covered by the tile's columns
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int stage_bytes = p.nseg * SEG_BYTES;                 // multiple of 128
  const int stage_stride = (stage_bytes + 1023) & ~1023;
  uint8_t* b_smem = smem;                                     // [nkb][BLOCK_N][128 B] swizzled weight blocks
  uint8_t* a_smem = smem + ((p.nkb * BLOCK_N * 128 + 1023) & ~1023);
  const int NST = p.nstages;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(a_smem + NST * stage_stride);
  uint64_t* empty_bar = full_bar + R_STAGES;
  uint64_t* w_bar = empty_bar + R_STAGES;
  uint64_t* desc_tab = w_bar + 2;                              // [2 * MAX_MMA]

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;      // warp-uniform for the compiler
  const int R = p.rows;
  const int tiles_x = (p.Wo + RBM - 1) / RBM;
  const int bands = (p.Ho + R - 1) / R;
  const int ntiles = p.B * bands * tiles_x;

  if (warp == 4 * NWG && lane == 0) {
    tma_prefetch_desc(&tmap_x);
    tma_prefetch_desc(&tmap_w);
    for (int s = 0; s < NST; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 4); }
    mbar_init(w_bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4 * NWG) {
    // ================================================================ TMA: resident weights, then row segments per tile
    // (all lanes walk the loop, one elected lane issues)
    {
      if (elect_one()) {
        mbar_arrive_expect_tx(w_bar, p.nkb * BLOCK_N * 128);
        for (int kb = 0; kb < p.nkb; ++kb)
          tma_load_2d(smem_u32(b_smem + kb * BLOCK_N * 128), &tmap_w, w_bar, kb * 64, 0);
      }
      __syncwarp();
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const int tx = t % tiles_x, band = t / tiles_x;
        const int oy0 = (band % bands) * R, b = band / bands;
        const int ox0 = tx * RBM;
        mbar_wait(&empty_bar[stage], phase ^ 1);
        const uint32_t dst = smem_u32(a_smem + stage * stage_stride);
        if (elect_one()) {
          mbar_arrive_expect_tx(&full_bar[stage], stage_bytes);
          for (int sgi = 0; sgi < p.nseg; ++sgi) {             // a segment = two boxes of 144 eight-byte elements (see host)
            const int xe = 2 * (ox0 + p.seg_dx[sgi]), yy = oy0 * p.stride + p.seg_dy[sgi];   // rows >= H: zero fill
            tma_load_4d(dst + sgi * SEG_BYTES, &tmap_x, &full_bar[stage], xe, p.seg_g[sgi], yy, b);
            tma_load_4d(dst + sgi * SEG_BYTES + SEG_BYTES / 2, &tmap_x, &full_bar[stage], xe + SEG_PIX, p.seg_g[sgi], yy, b);
          }
        }
        __syncwarp();
        if (++stage == NST) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ================================================================ consumer warpgroups (warps 0..4 NWG - 1): warpgroup g
    // takes tiles g, g + NWG, ... of this CTA's sequence; while one runs its epilogue the other issues MMAs
    const int t = threadIdx.x & 127, w = t >> 5, g = warp >> 2;
    const uint32_t a0 = smem_u32(a_smem), b0 = smem_u32(b_smem);
    // descriptor tables in smem (stage 0, output row 0 addresses): the issue loop is ld.shared + 64-bit add per MMA
    for (int i = threadIdx.x; i < p.nmma; i += NWG * 128) {
      desc_tab[2 * i] = gmma_desc(a0 + p.mma_a[i], p.mma_lbo[i], 128, 0);
      desc_tab[2 * i + 1] = gmma_desc_sw128(b0 + p.mma_b[i]);
    }
    bar_sync_named(1, NWG * 128);
    float sc[NOUT / 4], sh[NOUT / 4];                   // tile-invariant affine of this thread's columns 8 j + 2 (lane % 4) + e
#pragma unroll
    for (int j = 0; j < NOUT / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        sc[2 * j + e] = __ldg(p.scale + 8 * j + 2 * (lane & 3) + e);
        sh[2 * j + e] = __ldg(p.shift + 8 * j + 2 * (lane & 3) + e);
      }
    const bool relu = p.act == ACT_RELU;
    mbar_wait(w_bar, 0);
    const int nmma = p.nmma;
    const uint64_t row_step = static_cast<uint64_t>(p.row_bytes >> 4);

    // one output row: both 64-pixel halves, the whole MMA table, one commit group
    auto issue = [&](float (&acc)[2][BLOCK_N / 2], uint64_t a_off) {
      gmma_fence();
#pragma unroll 7
      for (int i = 0; i < nmma; ++i) {
        const uint64_t ad = desc_tab[2 * i] + a_off, bd = desc_tab[2 * i + 1];
        Gmma<BLOCK_N>::template mma<0, 0>(acc[0], ad, bd, i != 0 ? 1u : 0u);
        Gmma<BLOCK_N>::template mma<0, 0>(acc[1], ad + (1024 >> 4), bd, i != 0 ? 1u : 0u);     // pixels 64..127: +64 x 16 B
      }
      gmma_commit();
    };
    auto epilogue = [&](float (&acc)[2][BLOCK_N / 2], int b, int oy, int ox0) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
          const int ox = ox0 + 64 * h + 16 * w + (lane >> 2) + 8 * hh;
          if (ox >= p.Wo) continue;
          __half2 o[NOUT / 8], ol[NOUT / 8];
#pragma unroll
          for (int j = 0; j < NOUT / 8; ++j) {
            float v0 = acc[h][4 * j + 2 * hh], v1 = acc[h][4 * j + 2 * hh + 1];
            if (MERGE) {                                   // second partial sum of the same columns
              v0 += acc[h][4 * (j + NOUT / 8) + 2 * hh];
              v1 += acc[h][4 * (j + NOUT / 8) + 2 * hh + 1];
            }
            float f0 = v0 * sc[2 * j] + sh[2 * j];
            float f1 = v1 * sc[2 * j + 1] + sh[2 * j + 1];
            if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
            o[j] = __floats2half2_rn(f0, f1);
            const float2 hf = __half22float2(o[j]);
            ol[j] = __floats2half2_rn(f0 - hf.x, f1 - hf.y);          // lo half of the pair (dead code unless split_out)
          }
          const int c2 = 2 * (lane & 3);                 // this thread's channel pair inside each 8-channel plane
          if (p.out_planar) {
            const int npar = p.out_npar, Wg = p.Wo / npar;
            const int par = npar == 2 ? (ox & 1) : 0, xi = npar == 2 ? (ox >> 1) : ox;
            const int Ghalf = (p.Cout / 8) * npar, G = p.split_out ? 2 * Ghalf : Ghalf;
#pragma unroll
            for (int pl = 0; pl < NOUT / 8; ++pl) {
              if (pl * 8 < p.Cout) {
                __half* dst = p.y + ((static_cast<long long>(b * p.Ho + oy) * G + (pl * npar + par)) * Wg + xi) * 8 + c2;
                *reinterpret_cast<__half2*>(dst) = o[pl];
                if (p.split_out) *reinterpret_cast<__half2*>(dst + static_cast<long long>(Ghalf) * Wg * 8) = ol[pl];
              }
            }
          } else {
            __half* dst = p.y + (static_cast<long long>(b * p.Ho + oy) * p.Wo + ox) * p.y_ld + c2;
#pragma unroll
            for (int pl = 0; pl < NOUT / 8; ++pl)
              if (pl * 8 < p.Cout) {
                *reinterpret_cast<__half2*>(dst + pl * 8) = o[pl];
                if (p.split_out) *reinterpret_cast<__half2*>(dst + p.y_lo + pl * 8) = ol[pl];
              }
          }
        }
    };

    float d[2][BLOCK_N / 2];
    for (int q = g, tt = blockIdx.x + g * gridDim.x; tt < ntiles; q += NWG, tt += NWG * gridDim.x) {
      // q = index of the tile in this CTA's sequence (the TMA warp's order); NST % NWG == 0 (host), so stage q % NST is only
      // ever used by this warpgroup and phase q / NST of its barriers is the next one this warpgroup has not waited for
      const int stage = q % NST;
      const uint32_t phase = (q / NST) & 1;
      const int tx = tt % tiles_x, band = tt / tiles_x;
      const int oy0 = (band % bands) * R, b = band / bands;
      const int ox0 = tx * RBM;
      const int nr = p.Ho - oy0 < R ? p.Ho - oy0 : R;     // rows past Ho are neither computed nor stored
      mbar_wait(&full_bar[stage], phase);
      const uint64_t a_off = static_cast<uint64_t>((stage * stage_stride) >> 4);
      for (int r = 0; r < nr; ++r) {
        issue(d, a_off + r * row_step);
        gmma_wait<0>();
        gmma_hold(d[0]);
        gmma_hold(d[1]);
        if (r == nr - 1) {                               // the stage's last MMAs are done: hand it back to the TMA warp
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[stage]);
        }
        epilogue(d, b, oy0 + r, ox0);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
typedef CUresult (*PFN_encodeTiledR)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiledR rows_encode_fn() {
  static PFN_encodeTiledR fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
      set_error("cuTensorMapEncodeTiled entry point unavailable");
      return nullptr;
    }
    fn = reinterpret_cast<PFN_encodeTiledR>(ptr);
  }
  return fn;
}

template <int BLOCK_N, bool MERGE>
static int rows_conv_launch(int grid, int smem, cudaStream_t st, const CUtensorMap& tx, const CUtensorMap& tw,
                            const RowsParams& p) {
  static int attr = 0;
  if (smem > attr) {
    if (check_cuda(cudaFuncSetAttribute(rows_conv_kernel<BLOCK_N, MERGE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem),
                   "rows smem"))
      return -1;
    attr = smem;
  }
  return check_cuda(launch_k(rows_conv_kernel<BLOCK_N, MERGE>, dim3(grid), dim3(ROWS_THREADS), smem, st, tx, tw, p), "rows_conv launch");
}

// x: planes [B][H][Gin][Wg_in][8] fp16 with Gin = (Cin/8) * in_npar; wp: packed weights [n_pad, k_pad] fp16 whose K order is
// (ky, kx, c) with c over Cin (Cin = 16) or (tap = ky * kw + kx, c over 8) with one zero tap after an odd tap count (Cin = 8).
// in_mode 0: plain fp16 planes, n_pad >= Cout. Strict precision (fp16 pairs), n_pad = 2 Cout: the weight rows are two
// products of the same outputs, stacked along N and added by the epilogue:
//   in_mode 1 (Cin = 8): the image pair plane [hi3 | lo3 | 0 0]; rows [0, Cout) = [W_hi | W_hi | 0 0] (A_hi W_hi + A_lo W_hi
//              in one K = 8 slot), rows [Cout, 2 Cout) = [W_lo | 0 ...] (A_hi W_lo), one K set of kh x kw taps;
//   in_mode 2 (Cin = 16): pair planes [hi0 hi1 lo0 lo1]; TWO K sets stacked along ky, set 0 read from the hi planes, set 1
//              from the lo planes: rows [0, Cout) = [W_hi ; W_hi], rows [Cout, 2 Cout) = [W_lo ; 0].
// So every A operand is read by ONE MMA (N = 2 Cout): the same three products A_hi W_hi + A_lo W_hi + A_hi W_lo over the
// same resident row segments.
static int launch_rows_conv(const __half* x, int B, int H, int W, int Cin, int in_npar, const __half* wp, int n_pad, int k_pad,
                     int kh, int kw, int stride, int pad, int Cout, const float* scale, const float* shift, int act,
                     int out_planar, int out_npar, __half* y, int y_ld, cudaStream_t st, int in_mode, int split_out,
                     int y_lo) {
  PFN_encodeTiledR enc = rows_encode_fn();
  if (!enc) return -1;
  RowsParams p;
  memset(&p, 0, sizeof(p));
  const int P = Cin / 8;
  const bool merge = in_mode != 0;
  const int nsets = in_mode == 2 ? 2 : 1;                // K sets stacked along ky
  const int Ptot = in_mode == 2 ? 2 * P : P;             // planes in memory (hi planes, then lo planes)
  const int npar_in = stride == 2 ? 2 : 1;
  if (in_mode < 0 || in_mode > 2 || (in_mode == 1 && Cin != 8) || (in_mode == 2 && Cin != 16) ||
      (merge && n_pad != 2 * Cout) || (split_out && !out_planar && y_lo % 8 != 0)) {
    set_error("rows_conv: unsupported strict-precision configuration (in_mode %d, Cin %d, stride %d, n_pad %d)", in_mode, Cin,
              stride, n_pad);
    return -1;
  }
  if ((Cin != 8 && Cin != 16) || (stride != 1 && stride != 2) || (stride == 2 && (in_npar != 2 || kw != 3 || pad != 1)) ||
      (stride == 1 && in_npar != 1) || (merge ? (n_pad != 32 && n_pad != 64) : (n_pad != 16 && n_pad != 32)) ||
      Cout > (merge ? n_pad / 2 : n_pad) || k_pad % 64 != 0 || W % in_npar != 0 || (Cin == 8 && kw > 8) || pad > 3 ||
      kw - 1 - pad > 4) {
    set_error("rows_conv: unsupported configuration Cin=%d stride=%d in_npar=%d kw=%d pad=%d n_pad=%d", Cin, stride, in_npar,
              kw, pad, n_pad);
    return -1;
  }
  p.B = B; p.H = H; p.Gin = Ptot * in_npar; p.Wg_in = W / in_npar;
  p.split_out = split_out; p.y_lo = y_lo;
  p.Ho = (H + 2 * pad - kh) / stride + 1;
  p.Wo = (W + 2 * pad - kw) / stride + 1;
  p.stride = stride; p.pad = pad; p.nkb = k_pad / 64;
  p.Cout = Cout; p.scale = scale; p.shift = shift; p.act = act;
  p.out_planar = out_planar; p.out_npar = out_npar; p.y = y; p.y_ld = y_ld;
  if (out_planar && (Cout % 8 != 0 || p.Wo % out_npar != 0)) { set_error("rows_conv: planar output needs Cout %% 8 == 0"); return -1; }
  // ---- rows per tile and ring depth: the most rows for which two stages fit next to the resident weights with two CTAs
  // per SM (one CTA's epilogue and TMA waits overlap the other's MMAs); failing that, one CTA per SM. The depth is a multiple
  // of NWG: tile q of the CTA uses stage q % nst, so every stage then belongs to ONE consumer warpgroup, which waits for
  // each of its phases in turn. (With an odd depth a warpgroup would skip the phase of the other warpgroup's tile, and a
  // parity wait cannot tell "that phase still pending" from "my phase complete".)
  const int w_bytes = (p.nkb * n_pad * 128 + 1023) & ~1023;
  auto stage_of = [&](int rows) { return (((rows - 1) * stride + kh) * Ptot * npar_in * SEG_BYTES + 1023) & ~1023; };
  int rows = 0, nst = 0;
  auto pick = [&](int ctas_per_sm) {
    for (int r = MAX_ROWS; r >= 1; --r) {
      const int n = ((ctas_per_sm == 2 ? 113 : 226) * 1024 - w_bytes - 3072) / stage_of(r) / NWG * NWG;
      if (n >= NWG && ((r - 1) * stride + kh) * Ptot * npar_in <= MAX_SEG) { rows = r; nst = n; return true; }
    }
    return false;
  };
  const int ctas = n_pad != 64 && pick(2) ? 2 : 1;        // N = 64 accumulators: one CTA of 288 threads per SM
  if (ctas == 1 && !pick(1)) { set_error("rows_conv: row segments do not fit in shared memory"); return -1; }
  if (nst > R_STAGES) nst = R_STAGES;
  p.rows = rows; p.nstages = nst;
  p.row_bytes = stride * Ptot * npar_in * SEG_BYTES;
  // ---- segments (input row ry of the band, plane, parity) and the MMA table of output row 0
  int nseg = 0, nmma = 0;
  auto seg_index = [&](int ry, int plane, int par) { return (ry * Ptot + plane) * npar_in + par; };
  for (int ry = 0; ry < (rows - 1) * stride + kh; ++ry)
    for (int plane = 0; plane < Ptot; ++plane)
      for (int par = 0; par < npar_in; ++par) {
        p.seg_g[nseg] = plane * in_npar + par;
        p.seg_dy[nseg] = ry - pad;
        p.seg_dx[nseg] = stride == 2 ? -1 : -pad;
        ++nseg;
      }
  const int ntap = kh * kw;
  if (k_pad < (Cin == 8 ? (ntap + 1) / 2 * 16 : nsets * ntap * Cin)) { set_error("rows_conv: k_pad too small"); return -1; }
  if (Cin == 8) {
    // the kh x kw taps in (ky, kx) order, two per MMA: the second one's 16-byte chunk is reached through LBO = its distance
    // in the stage (the next pixel, or a tap at the start of the next row's segment); an odd last tap gets a zero-weight
    // partner one pixel further. 25 MMAs for a 7x7, where taps padded to 8 per row would take 28.
    auto tap_a = [&](int tp) { return seg_index(tp / kw, 0, 0) * SEG_BYTES + (tp % kw) * 16; };
    for (int m = 0; 2 * m < ntap; ++m) {
      if (nmma >= MAX_MMA) { set_error("rows_conv: too many MMAs"); return -1; }
      p.mma_a[nmma] = tap_a(2 * m);
      p.mma_lbo[nmma] = 2 * m + 1 < ntap ? tap_a(2 * m + 1) - tap_a(2 * m) : 16;
      const int koff = 2 * m * 8;
      p.mma_b[nmma] = (koff / 64) * n_pad * 128 + ((koff % 64) / 16) * 32;
      ++nmma;
    }
  }
  for (int set = 0; set < nsets && Cin == 16; ++set)
  for (int ky = 0; ky < kh; ++ky) {
    const int kyw = set * kh + ky;                      // row of the stacked weight tap sets
    const int pl0 = set == 1 ? P : 0;                   // strict: the second K set reads the lo planes
    for (int kx = 0; kx < kw; ++kx) {                   // one tap per MMA, second channel plane through LBO
      if (nmma >= MAX_MMA) { set_error("rows_conv: too many MMAs"); return -1; }
      int par = 0, shift_px = kx;
      if (stride == 2) { par = (kx == 1) ? 0 : 1; shift_px = (kx == 0) ? 0 : 1; }
      p.mma_a[nmma] = seg_index(ky, pl0, par) * SEG_BYTES + shift_px * 16;
      p.mma_lbo[nmma] = (seg_index(ky, pl0 + 1, par) - seg_index(ky, pl0, par)) * SEG_BYTES;
      const int koff = (kyw * kw + kx) * 16;
      p.mma_b[nmma] = (koff / 64) * n_pad * 128 + ((koff % 64) / 16) * 32;
      ++nmma;
    }
  }
  p.nseg = nseg; p.nmma = nmma;
  // ---- tensor maps
  CUtensorMap tx, tw;
  {
    // A plane row is contiguous (Wg pixels x 16 B). Described with its natural {8 ch, Wg, ..} dimensions the TMA unit issues
    // one 16-byte request per pixel and a tile's 7-12 segments cost ~1000-1600 requests (the kernel was request-bound:
    // 2.5 us per 128-pixel tile). As 8-byte elements a row is ONE dimension of 2*Wg elements; a box holds <= 256 elements,
    // so a 144-pixel segment is two boxes of 144 elements (1152 B each, TMA needs 128-byte aligned smem destinations).
    // Out-of-range elements are zero-filled as before.
    cuuint64_t gdim[4] = {static_cast<cuuint64_t>(p.Wg_in) * 2, static_cast<cuuint64_t>(p.Gin), static_cast<cuuint64_t>(H),
                          static_cast<cuuint64_t>(B)};
    cuuint64_t gstr[3] = {static_cast<cuuint64_t>(p.Wg_in) * 16, static_cast<cuuint64_t>(p.Wg_in) * 16 * p.Gin,
                          static_cast<cuuint64_t>(p.Wg_in) * 16 * p.Gin * H};
    cuuint32_t box[4] = {SEG_PIX, 1, 1, 1};
    cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(&tx, CU_TENSOR_MAP_DATA_TYPE_UINT64, 4, const_cast<__half*>(x), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("rows_conv: cuTensorMapEncodeTiled(x) failed (%d)", static_cast<int>(r)); return -1; }
  }
  {
    cuuint64_t gdim[2] = {static_cast<cuuint64_t>(k_pad), static_cast<cuuint64_t>(n_pad)};
    cuuint64_t gstr[1] = {static_cast<cuuint64_t>(k_pad) * 2};
    cuuint32_t box[2] = {64, static_cast<cuuint32_t>(n_pad)};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&tw, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(wp), gdim, gstr, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("rows_conv: cuTensorMapEncodeTiled(w) failed (%d)", static_cast<int>(r)); return -1; }
  }
  const int smem = w_bytes + nst * stage_of(rows) + 1024 + 2048;
  const int tiles = B * ((p.Ho + rows - 1) / rows) * ((p.Wo + RBM - 1) / RBM);
  int dev = 0, nsm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
  const int grid = tiles < ctas * nsm ? tiles : ctas * nsm;
  int rc;
  if (n_pad == 16)
    rc = rows_conv_launch<16, false>(grid, smem, st, tx, tw, p);
  else if (n_pad == 32)
    rc = merge ? rows_conv_launch<32, true>(grid, smem, st, tx, tw, p) : rows_conv_launch<32, false>(grid, smem, st, tx, tw, p);
  else
    rc = rows_conv_launch<64, true>(grid, smem, st, tx, tw, p);
  if (rc) return -1;
  return check_cuda(cudaGetLastError(), "rows_conv launch");
}

}  // namespace mf

using namespace mf;

extern "C" {

int mf_conv2d_rows_f16(const void* x, int B, int H, int W, int Cin, int in_npar, const void* w_packed, int n_pad, int k_pad,
                       int kh, int kw, int stride, int pad, int Cout, const float* scale, const float* shift, int act,
                       int out_planar, int out_npar, void* y, int y_ld, void* stream) {
  return launch_rows_conv(static_cast<const __half*>(x), B, H, W, Cin, in_npar, static_cast<const __half*>(w_packed), n_pad,
                          k_pad, kh, kw, stride, pad, Cout, scale, shift, act, out_planar, out_npar, static_cast<__half*>(y),
                          y_ld, MF_STREAM(stream), 0, 0, 0);
}

int mf_conv2d_rows_f16x2(const void* x, int B, int H, int W, int Cin, int in_npar, int in_mode, const void* w_packed, int n_pad,
                         int k_pad, int kh, int kw, int stride, int pad, int Cout, const float* scale, const float* shift, int act,
                         int out_planar, int out_npar, void* y, int y_ld, int y_lo, void* stream) {
  return launch_rows_conv(static_cast<const __half*>(x), B, H, W, Cin, in_npar, static_cast<const __half*>(w_packed), n_pad,
                          k_pad, kh, kw, stride, pad, Cout, scale, shift, act, out_planar, out_npar, static_cast<__half*>(y),
                          y_ld, MF_STREAM(stream), in_mode, 1, y_lo);
}

}  // extern "C"
