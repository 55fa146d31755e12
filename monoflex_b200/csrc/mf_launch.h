// Launcher prototypes of the HBM-bound kernels (internal; the public C ABI is include/monoflex_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>

namespace mf {
int launch_pack_image(const float* x, __half* y, int B, int C, int H, int W, cudaStream_t st);
int launch_nchw_to_nhwc(const float* x, __half* y, int B, int C, int HW, int y_ld, cudaStream_t st);
int launch_nhwc_to_nchw(const __half* x, float* y, int B, int C, int HW, int x_ld, cudaStream_t st);
int launch_pack_offmask(const float* off, const float* mask, float* y, int B, int HW, cudaStream_t st);
int launch_maxpool2(const __half* x, __half* y, int B, int H, int W, int C, int x_ld, int y_ld, cudaStream_t st);
int launch_upsample_add(const __half* x, const float* w, const __half* skip, __half* y, int B, int Hi, int Wi, int C,
                        int f, int x_ld, int skip_ld, int y_ld, cudaStream_t st);
int launch_edge_gather(const __half* feat, int feat_ld, int ch_a, int ch_b, const long long* edge_idx, __half* ea,
                       __half* eb, int B, int H, int W, int K, int out_w, int out_h, cudaStream_t st);
int launch_edge_head_add(const __half* t, const float* w, const float* bias, int n_out, const long long* edge_idx,
                         const long long* edge_len, float* out, int out_ctot, int out_ch0, int B, int K, int H, int W,
                         cudaStream_t st);
int launch_sigmoid_clamp(float* x, long long n, cudaStream_t st);
int launch_edge_mask(const long long* edge_idx, unsigned char* mask, int B, int K, int H, int W, int out_w, int out_h,
                     cudaStream_t st);
int launch_focal_loss(const float* pred, const float* tgt, long long n, float* out2, cudaStream_t st);
#define MF_LOSS_OBJ_COLS 64   /* floats per (image, object slot) row of the packed label table (mf_loss.cu) */
int launch_loss_forward(const float* pred_cls, const float* hm, const float* pred_reg, const float* obj, const float* img,
                        const float* weights11, const float* dim_mean9, int B, int ncls, int M, int H, int W, int C,
                        float* out48, float* ws64, cudaStream_t st);
int launch_loss_backward(const float* pred_cls, const float* hm, const float* pred_reg, const float* obj, const float* img,
                         const float* weights11, const float* dim_mean9, int B, int ncls, int M, int H, int W, int C,
                         const float* ws64, const float* grad_losses11, float* grad_cls, float* grad_reg, cudaStream_t st);
int launch_mn_major_selftest(const __half* a_km, const __half* b_kn, float* d_mn, cudaStream_t st);
int launch_maxpool2_bwd(const __half* x, const __half* dy, __half* dx, int B, int H, int W, int C, int x_ld, int dy_ld,
                        int dx_ld, cudaStream_t st);
size_t upsample_bwd_workspace_floats(int B, int Hi, int Wi, int C, int f);
int launch_upsample_bwd(const __half* x, const float* w, const __half* dy, __half* dx, float* dw, int B, int Hi, int Wi, int C,
                        int f, int x_ld, int dy_ld, int dx_ld, float* workspace, cudaStream_t st);
int launch_sigmoid_clamp_bwd(const float* y, const float* dy, float* dx, long long n, cudaStream_t st);
size_t column_sum_workspace_floats(long long M, int C);
int launch_column_sum(const __half* x, int x_ld, long long M, int C, float* out, float* workspace, cudaStream_t st);
int launch_edge_gather_bwd(const __half* d_ea, const __half* d_eb, int ch_a, int ch_b, const long long* edge_idx, __half* d_feat,
                           int feat_ld, int B, int H, int W, int K, int out_w, int out_h, cudaStream_t st);
int launch_edge_head_add_bwd(const __half* t, const float* w, int n_out, const long long* edge_idx, const long long* edge_len,
                             const float* d_out, int out_ctot, int out_ch0, __half* d_t, float* dw, float* dbias, int B, int K,
                             int H, int W, cudaStream_t st);
int launch_add_rows(__half* dst, int dst_ld, const __half* src, int src_ld, long long M, int C, cudaStream_t st);
int launch_interleave2x2(const __half* p00, const __half* p01, const __half* p10, const __half* p11, int part_ld, __half* out,
                         int out_ld, int B, int Hh, int Wh, int C, cudaStream_t st);
int launch_dcn_sample_cols(const __half* x, int x_ld, const float* om, int om_ld, __half* cols, int B, int H, int W, int C,
                           cudaStream_t st);
int launch_dcn_col2im(const __half* x, int x_ld, const float* om, int om_ld, const __half* gcol, __half* dx, int dx_ld, float* dom,
                      int B, int H, int W, int C, cudaStream_t st);
size_t bn_train_workspace_floats(long long M, int C);
int launch_bn_train_forward(const __half* x, int x_ld, long long M, int C, const float* gamma, const float* beta, float eps,
                            float momentum, int abs_gamma, float* running_mean, float* running_var, const __half* res,
                            int res_ld, int act, __half* y, int y_ld, float* mean, float* rstd, float* scale, float* shift,
                            float* workspace, cudaStream_t st);
int launch_bn_train_backward(const __half* x, int x_ld, const __half* dy, int dy_ld, const __half* y, int y_ld, long long M, int C,
                             const float* mean, const float* rstd, const float* scale, int act, __half* dx, int dx_ld,
                             __half* dres, int dres_ld, float* dgamma, float* dbeta, float* workspace, cudaStream_t st);
#define MF_MAX_PEERS 16
int launch_adamw_p2p(const unsigned long long* param_ptrs, const unsigned long long* grad_ptrs, int world, int rank,
                     unsigned long long mc_params, unsigned long long mc_grads, float* m, float* v, const float* chunk_lr,
                     long long n_chunks, float beta1, float beta2, float eps, float wd, long long step, float lr_scale,
                     cudaStream_t st);
#define MF_ADAMW_CHUNK 512   /* arena granularity (elements) of the per-chunk lr table */
#define MF_OPTIM_ADAMW 0     /* update rules of mf_optim_step_dyn: decoupled weight decay (AdamW, fastai true_wd) */
#define MF_OPTIM_ADAM 1      /* coupled L2 weight decay (torch.optim.Adam) */
int launch_focal_loss_backward(const float* pred, const float* tgt, long long n, const float* scale, float* grad,
                               cudaStream_t st);
int launch_adamw_arena(float* p, const float* g, float* m, float* v, const float* chunk_lr, long long n_chunks,
                       float beta1, float beta2, float eps, float wd, long long step, float grad_scale, float lr_scale,
                       cudaStream_t st);
int launch_adamw_arena_dyn(float* p, float* g, float* m, float* v, const float* chunk_lr, long long n_chunks,
                           float beta1, float beta2, float eps, float wd, float grad_scale, float lr_scale, long long* state4,
                           void* dyn16, int check_finite, float max_norm, double* partials, float* total_norm_out,
                           int rule, const double* hyper, cudaStream_t st);
// OUTPUT_DEPTH estimators of the decode (detector_infer.py:148-209); the values are the C ABI's `depth_mode`
enum {
  MF_DEPTH_SOFT = 0, MF_DEPTH_HARD = 1, MF_DEPTH_MEAN = 2, MF_DEPTH_ORACLE = 3, MF_DEPTH_DIRECT = 4,
  MF_DEPTH_KEYPOINTS_AVG = 5, MF_DEPTH_KEYPOINTS_CENTER = 6, MF_DEPTH_KEYPOINTS_02 = 7, MF_DEPTH_KEYPOINTS_13 = 8,
  MF_DEPTH_MODES = 9
};
int launch_decode(const float* heat, const float* reg, const float* calib, const float* pad, const float* size,
                  const float* dim_mean, int B, int C, int H, int W, int R, int K, float thresh, int apply_sigmoid,
                  int depth_mode, const float* gt, int G, float* s1_score, int* s1_idx, float* scores, long long* inds,
                  float* clses, float* ys, float* xs, float* pois, float* result, int* count, float* depth_err,
                  float* proj, int* min_unc, cudaStream_t st);
int launch_nms_hm(const float* hm, float* out, int planes, int H, int W, cudaStream_t st);
int launch_pack_conv_weight_dgrad(const float* w, int Cout, int Cin, int kh, int kw, int cout_pad, int n_pad, int k_pad,
                                  __half* out, cudaStream_t st);
int launch_pack_conv_weight(const float* w, int Cout, int Cin, int kh, int kw, int cin_pad, int n_pad, int k_pad,
                            __half* out, cudaStream_t st);
// SyncBatchNorm halves (mf_bn_train.cu)
int launch_bn_sync_forward_stats(const __half* x, int x_ld, long long M, int C, float* workspace, double* sums, cudaStream_t st);
int launch_bn_sync_forward_apply(const __half* x, int x_ld, long long M, int C, const double* sums, double count, const float* gamma,
                                 const float* beta, float eps, float momentum, int abs_gamma, float* running_mean,
                                 float* running_var, const __half* res, int res_ld, int act, __half* y, int y_ld, float* mean,
                                 float* rstd, float* scale, float* shift, cudaStream_t st);
int launch_bn_sync_backward_stats(const __half* x, int x_ld, const __half* dy, int dy_ld, const __half* y, int y_ld, long long M,
                                  int C, const float* mean, const float* rstd, int act, float* workspace, double* sums,
                                  float* dgamma, float* dbeta, cudaStream_t st);
int launch_bn_sync_backward_apply(const __half* x, int x_ld, const __half* dy, int dy_ld, const __half* y, int y_ld, long long M,
                                  int C, const float* mean, const float* rstd, const float* scale, const double* sums, double count,
                                  int act, __half* dx, int dx_ld, __half* dres, int dres_ld, float* workspace, cudaStream_t st);
// GPU input pipeline (mf_input.cu)
int launch_preprocess_u8(const unsigned char* const* src, const int* hw, const int* flip, int B, int H, int W,
                         const float* mean3, const float* std3, int to_bgr, float* out, cudaStream_t st);
int launch_draw_heatmap(const int* obj, int B, int max_objs, int ncls, int H, int W, float* hm, cudaStream_t st);
// strict-precision (hi/lo fp16 pairs) companions, mf_split.cu
int launch_pack_conv_weight_split(const float* w, int Cout, int Cin, int kh, int kw, int n_pad, int k_pad, __half* out,
                                  cudaStream_t st);
int launch_pack_image_pair8(const float* x, __half* y, int B, int C, int H, int W, cudaStream_t st);
int launch_pack_image_split(const float* x, __half* y, int B, int C, int H, int W, cudaStream_t st);
int launch_maxpool2_split(const __half* x, int x_lo, __half* y, int y_lo, int B, int H, int W, int C, int x_ld, int y_ld,
                          cudaStream_t st);
int launch_upsample_add_split(const __half* x, int x_lo, const float* w, const __half* skip, int skip_lo, __half* y, int y_lo,
                              int B, int Hi, int Wi, int C, int f, int x_ld, int skip_ld, int y_ld, cudaStream_t st);
int launch_edge_gather_split(const __half* feat, int feat_ld, int feat_lo, int ch_a, int ch_b, const long long* edge_idx,
                             __half* ea, __half* eb, int B, int H, int W, int K, int out_w, int out_h, cudaStream_t st);
int launch_edge_head_add_split(const __half* t, int t_ld, int t_lo, const float* w, const float* bias, int n_out,
                               const long long* edge_idx, const long long* edge_len, float* out, int out_ctot, int out_ch0, int B,
                               int K, int H, int W, cudaStream_t st);
int launch_split_to_nchw(const __half* x, int x_ld, int x_lo, float* y, int B, int C, int HW, cudaStream_t st);
int launch_dcn_v2_forward_f32(const float* x, const float* w, const float* bias, const float* off, const float* mask,
                              float* y, int B, int Cin, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph,
                              int pw, int dh, int dw, int dg, cudaStream_t st);
size_t dcn_v2_backward_f32_workspace(int B, int Cin, int H, int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                                     int dh, int dw, int dg);
int launch_dcn_v2_backward_f32(const float* x, const float* w, const float* off, const float* mask, const float* dy,
                               float* gx, float* goff, float* gmask, float* gw, float* gb, int B, int Cin, int H, int W,
                               int Cout, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int dg,
                               void* workspace, size_t ws_bytes, cudaStream_t st);
}  // namespace mf
