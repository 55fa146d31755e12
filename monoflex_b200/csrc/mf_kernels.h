// Internal declarations shared by the .cu files of libmonoflex_b200.so (not part of the public C ABI, which is
// include/monoflex_b200.h): the implicit-GEMM parameters and the launchers one file calls in another.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace mf {

enum { MODE_CONV = 0, MODE_DCN = 1, MODE_CONV_TMA = 2 };
enum { ACT_NONE = 0, ACT_RELU = 1, ACT_LEAKY = 2, ACT_OFFMASK = 3 };
enum { OUT_F16_NHWC = 0, OUT_F32_NHWC = 1, OUT_F32_NCHW = 2 };

struct IgemmParams {
  // A operand: NHWC fp16 activations, `x_ld` elements between consecutive pixels (>= Cin: channel-slice views)
  const __half* x;
  int x_ld;
  int B, H, W, Cin;
  int Ho, Wo, kh, kw, stride, pad;
  int M;        // B*Ho*Wo
  int K_real;   // kh*kw*Cin
  int nkb;      // ceil(K_real / 64)
  // DCN: per output pixel 18 offsets (dy,dx per tap) + 9 masks (already sigmoid-ed), fp32, row stride om_ld
  const float* offmask;
  int om_ld;
  // epilogue: y = act(acc*scale[n] + shift[n] (+ res[m,n]))
  int Cout;
  const float* scale;
  const float* shift;
  const __half* res;
  int res_ld;
  int act;
  int out_mode;
  void* y;
  int y_ld;
  // strict-precision ("split") operands: an fp32-grade value v is stored as two fp16 numbers hi = fp16(v), lo = fp16(v - hi)
  // in the same pixel row, the lo block `*_lo` elements after the hi block. split_in: A and the packed weights are split and
  // the K axis is the concatenation, per (tap, 64-channel chunk), of the three products A_hi W_hi, A_lo W_hi, A_hi W_lo
  // (K_real / nkb already count that tripling). split_out: the fp16 NHWC output (and the residual) are hi/lo pairs.
  int split_in, split_out;
  int x_lo, res_lo, y_lo;
  int cw;       // split_in: channels per chunk = min(Cin, 64)
  // pair schedule (set by launch_igemm2 for split_in with 64-channel K blocks): per (tap, chunk) only TWO stages are filled,
  // (A_hi, W_hi) and (A_lo, W_lo), and the consumer warpgroups issue the three products A_hi W_hi, A_lo W_hi, A_hi W_lo across them -
  // one third less operand traffic into shared memory than the K-concatenation (which loads A_hi and W_hi twice).
  // nkb then counts stage fills = 2 * taps * Cin / 64.
  int pair;
  // HEAD2 (strict-precision predictor, EPI == 2 instantiation): this GEMM is the nine 3x3 head branches (N = nbranch x 256,
  // 128-column tiles, IABN + leaky folded into scale / shift / act). Instead of storing the hidden tile, each consumer warpgroup
  // turns its 64 x 128 accumulator into fp16 hi/lo pairs and contracts them with the branch's split 1x1 head weights (<= 32
  // outputs) on the tensor cores, three products per k slice like every strict GEMM. The partial sums over the tile's 128
  // hidden channels go to plane (n0 & 255) >> 7 of `h2_part` [2][B][h2_ntot][Ho*Wo]; mf_head2_reduce adds the two planes in a
  // fixed order (+ bias) into the fp32 NCHW cls / reg maps. The hidden pair rows are stored only for the branches the edge
  // fusion gathers (h2_hid_col >= 0) and only at the pixels flagged in h2_mask.
  const __half* h2_w;            // [nbranch * 32][768] fp16 pairs (mf_pack_conv_weight_split of [nbranch * 32, 256, 1, 1]),
                                 // rows >= h2_nch[b] of a branch zero
  float* h2_part;
  int h2_ntot;                   // channels of the combined output (cls + reg = 53)
  int h2_nch[12], h2_ch0[12], h2_hid_col[12];
  const unsigned char* h2_mask;
};

int launch_igemm2(const IgemmParams& p, const __half* wp, int n_pad, int k_pad, int mode, cudaStream_t st);
int launch_offset_conv(const __half* x, int x_ld, int x_lo, int B, int H, int W, int Cin, const __half* wp, int n_pad, int k_pad,
                       const float* scale, const float* shift, float* y, int y_ld, bool pair, cudaStream_t st);
int launch_simt_gemm(const IgemmParams& p, const __half* wp, int n_pad, int k_pad, int mode, cudaStream_t st);
int launch_conv_wgrad_narrow(const __half* x, int x_ld, int B, int H, int W, const __half* dy, int dy_ld, int k, float* dw,
                             cudaStream_t st);
int launch_draw_heatmap(const int* obj, int B, int max_objs, int ncls, int H, int W, float* hm, cudaStream_t st);
int launch_focal_loss(const float* pred, const float* tgt, long long n, float* out2, cudaStream_t st);
int launch_focal_loss_backward(const float* pred, const float* tgt, long long n, const float* scale, float* grad,
                               cudaStream_t st);

#define MF_LOSS_OBJ_COLS 64   /* floats per (image, object slot) row of the packed label table (mf_loss.cu, mf_targets.cu) */

}  // namespace mf
