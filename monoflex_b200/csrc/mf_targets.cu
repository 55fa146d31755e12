// Training-target encoding of KITTIDataset.__getitem__ (data/datasets/kitti.py:126-179, 335-521) and its horizontal-flip
// augmentation (data/augmentations/augmentations.py:28-77) for the runs/monoflex.yaml configuration, from raw label rows.
//
//   encode_objects_kernel : one thread per (image, object slot): flip, 3D box corners and their projection, choice between the
//                           projected and the label 2D box, the annotation filter, the projected centre and its border
//                           intersection for outside objects, key-point visibility, down-sampling and rounding, the heat-map
//                           radii and the multi-bin orientation -> the loss's packed object table, the per-image calibration
//                           table, the remaining per-slot fields and the (valid, class, cx, cy, rx, ry) table the heat-map
//                           kernel of mf_input.cu draws.
//   encode_edges_kernel   : one thread per (image, border index): the edge-fusion border walk of get_edge_utils.
//
// The float64 arithmetic uses explicit round-to-nearest operations in the reference's order (no FMA contraction, which could
// move a rounded centre at a tie). Where the reference's box is its float32 label box, the arithmetic on it is float32 too.
// The reference raises for an edge object with two non-zero radii (kitti.py:457) and for an outside object whose 2D box centre
// lies outside the image (approx_proj_center returns None); such objects are counted in the status word and left out.
#include "mf_common.cuh"
#include "mf_launch.h"
#include "../../include/monoflex_b200.h"
#include <math.h>

namespace mf {
namespace {

constexpr double PI = 3.141592653589793;
constexpr int NCLS = 3;
constexpr int DOWN = 4;

// label row columns (MF_TARGET_LABEL_COLS)
enum { L_VALID = 0, L_CLS, L_TRUNC, L_OCC, L_X1, L_Y1, L_X2, L_Y2, L_H, L_W, L_L, L_TX, L_TY, L_TZ, L_RY };
// loss object table columns (OBJ_FIELDS of detector_loss.py / mf_loss.cu)
enum { O_CLS = 0, O_TC = 1, O_BOX = 3, O_REG = 7, O_TRUNC = 8, O_DIM = 9, O_LOC = 12, O_ROTY = 15, O_OFF = 16, O_ORI = 18,
       O_KPD = 26, O_KP = 29 };

struct TargetOut {
  float* obj; float* img; float* alphas; float* gt_bboxes; float* reg_weight; double* occlusions; double* truncations;
  int* obj6; double* P2; int* status;
};

MF_DEVINL double dadd(double a, double b) { return __dadd_rn(a, b); }
MF_DEVINL double dsub(double a, double b) { return __dsub_rn(a, b); }
MF_DEVINL double dmul(double a, double b) { return __dmul_rn(a, b); }
MF_DEVINL double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// Calibration.project_rect_to_image: [x y z 1] . P^T, then u /= w, v /= w
MF_DEVINL void project(const double* P, double x, double y, double z, double& u, double& v) {
  const double a = dadd(dadd(dadd(dmul(x, P[0]), dmul(y, P[1])), dmul(z, P[2])), dmul(1.0, P[3]));
  const double b = dadd(dadd(dadd(dmul(x, P[4]), dmul(y, P[5])), dmul(z, P[6])), dmul(1.0, P[7]));
  const double c = dadd(dadd(dadd(dmul(x, P[8]), dmul(y, P[9])), dmul(z, P[10])), dmul(1.0, P[11]));
  u = ddiv(a, c);
  v = ddiv(b, c);
}

MF_DEVINL double wrap_pi(double a) {         // the while-loops of convertRot2Alpha and the flip
  while (a > PI) a = dsub(a, PI * 2);
  while (a < -PI) a = dadd(a, PI * 2);
  return a;
}

// model/heatmap_coder.py:37-56 on float64 operands (the projected box)
MF_DEVINL double gaussian_radius_f64(double h, double w) {
  const double o = 0.7;
  const double b1 = dadd(h, w);
  const double c1 = ddiv(dmul(dmul(w, h), 1 - o), 1 + o);
  const double r1 = dadd(b1, __dsqrt_rn(dsub(dmul(b1, b1), dmul(4.0, c1)))) / 2;
  const double b2 = dmul(2.0, dadd(h, w));
  const double c2 = dmul(dmul(1 - o, w), h);
  const double r2 = dadd(b2, __dsqrt_rn(dsub(dmul(b2, b2), dmul(16.0, c2)))) / 2;
  const double a3 = 4 * o;
  const double b3 = dmul(-2 * o, dadd(h, w));
  const double c3 = dmul(dmul(o - 1, w), h);
  const double r3 = dadd(b3, __dsqrt_rn(dsub(dmul(b3, b3), dmul(4 * a3, c3)))) / 2;
  return fmin(fmin(r1, r2), r3);
}

// the same on float32 operands (the label box): numpy keeps float32 and rounds the Python-float constants to float32
MF_DEVINL float gaussian_radius_f32(float h, float w) {
  const double o = 0.7;
  const float b1 = __fadd_rn(h, w);
  const float c1 = __fdiv_rn(__fmul_rn(__fmul_rn(w, h), static_cast<float>(1 - o)), static_cast<float>(1 + o));
  const float r1 = __fdiv_rn(__fadd_rn(b1, __fsqrt_rn(__fsub_rn(__fmul_rn(b1, b1), __fmul_rn(4.f, c1)))), 2.f);
  const float b2 = __fmul_rn(2.f, __fadd_rn(h, w));
  const float c2 = __fmul_rn(__fmul_rn(static_cast<float>(1 - o), w), h);
  const float r2 = __fdiv_rn(__fadd_rn(b2, __fsqrt_rn(__fsub_rn(__fmul_rn(b2, b2), __fmul_rn(16.f, c2)))), 2.f);
  const float b3 = __fmul_rn(static_cast<float>(-2 * o), __fadd_rn(h, w));
  const float c3 = __fmul_rn(__fmul_rn(static_cast<float>(o - 1), w), h);
  const float r3 = __fdiv_rn(__fadd_rn(b3, __fsqrt_rn(__fsub_rn(__fmul_rn(b3, b3),
                                                                __fmul_rn(static_cast<float>(4 * (4 * o)), c3)))), 2.f);
  return fminf(fminf(r1, r2), r3);
}

MF_DEVINL int py_int_nonneg(double r) { return r > 0 ? static_cast<int>(r) : 0; }     // max(0, int(r))

// Object3d.generate_corners3d: R . [x; y; z] + t for the eight corners
MF_DEVINL void box_corners(double ry, float tx, float ty, float tz, double oh_, double ow_, double ol_, double* X, double* Y,
                           double* Z) {
  const double cr = cos(ry), sr = sin(ry);
  const double hl = ol_ / 2, hw = ow_ / 2;
  const double xc[8] = {hl, hl, -hl, -hl, hl, hl, -hl, -hl};
  const double yc[8] = {0, 0, 0, 0, -oh_, -oh_, -oh_, -oh_};
  const double zc[8] = {hw, -hw, -hw, hw, hw, -hw, -hw, hw};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    X[k] = dadd(dadd(dadd(dmul(cr, xc[k]), dmul(0.0, yc[k])), dmul(sr, zc[k])), static_cast<double>(tx));
    Y[k] = dadd(dadd(dadd(dmul(0.0, xc[k]), dmul(1.0, yc[k])), dmul(0.0, zc[k])), static_cast<double>(ty));
    Z[k] = dadd(dadd(dadd(dmul(-sr, xc[k]), dmul(0.0, yc[k])), dmul(cr, zc[k])), static_cast<double>(tz));
  }
}

// The right-camera label box (kitti.py:243-249), before the flip: the projected corners' extent under the unflipped P3,
// clamped with Python's max(x, 0) / min(x, img - 1), rounded to float32 (Object3d.box2d and its np.float32 elements)
MF_DEVINL void right_view_box(const double* P, double ry, float tx, float ty, float tz, double oh_, double ow_, double ol_,
                              int img_w, int img_h, float* box) {
  double X[8], Y[8], Z[8];
  box_corners(ry, tx, ty, tz, oh_, ow_, ol_, X, Y, Z);
  double u, v;
  project(P, X[0], Y[0], Z[0], u, v);
  double umin = u, umax = u, vmin = v, vmax = v;
#pragma unroll
  for (int k = 1; k < 8; ++k) {
    project(P, X[k], Y[k], Z[k], u, v);
    umin = fmin(umin, u); umax = fmax(umax, u);
    vmin = fmin(vmin, v); vmax = fmax(vmax, v);
  }
  const double wm1 = img_w - 1, hm1 = img_h - 1;
  box[0] = static_cast<float>(0 > umin ? 0.0 : umin);
  box[1] = static_cast<float>(0 > vmin ? 0.0 : vmin);
  box[2] = static_cast<float>(wm1 < umax ? wm1 : umax);
  box[3] = static_cast<float>(hm1 < vmax ? hm1 : vmax);
}

__global__ void __launch_bounds__(128) encode_objects_kernel(const double* __restrict__ lab, const double* __restrict__ P2,
                                                             const int* __restrict__ sizes, const int* __restrict__ flips,
                                                             const int* __restrict__ rights, int B, int M, int H, int W,
                                                             TargetOut o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * M) return;
  const int b = i / M;
  const int slot = i - b * M;
  float* ob = o.obj + static_cast<long long>(i) * MF_LOSS_OBJ_COLS;
  for (int c = 0; c < MF_LOSS_OBJ_COLS; ++c) ob[c] = 0.f;
  for (int c = 0; c < 6; ++c) o.obj6[6 * i + c] = 0;
  for (int c = 0; c < 4; ++c) o.gt_bboxes[4 * i + c] = 0.f;
  o.alphas[i] = 0.f;
  o.reg_weight[i] = 0.f;
  o.occlusions[i] = 0.0;
  o.truncations[i] = 0.0;

  const int img_w = sizes[2 * b], img_h = sizes[2 * b + 1];
  const bool size_ok = img_w >= 1 && img_h >= 1 && img_w <= W && img_h <= H;
  const bool flip = flips != nullptr && flips[b] != 0;
  const bool right = rights != nullptr && rights[b] != 0;
  double P[12];
  for (int k = 0; k < 12; ++k) P[k] = P2[12 * b + k];
  if (flip) {                                                          // augmentations.py:69-73
    P[2] = dsub(dsub(static_cast<double>(img_w), P[2]), 1.0);
    P[3] = -P[3];
  }
  const int pad_x = size_ok ? (W - img_w) / 2 : 0, pad_y = size_ok ? (H - img_h) / 2 : 0;
  if (slot == 0) {
    for (int k = 0; k < 12; ++k) o.P2[12 * b + k] = P[k];
    float* im = o.img + 8 * b;                                         // Loss_Computation.prepare_targets' calibration row
    im[0] = static_cast<float>(P[0]);
    im[1] = static_cast<float>(P[5]);
    im[2] = static_cast<float>(P[2]);
    im[3] = static_cast<float>(P[6]);
    im[4] = static_cast<float>(ddiv(P[3], -P[0]));
    im[5] = static_cast<float>(ddiv(P[7], -P[5]));
    im[6] = static_cast<float>(pad_x);
    im[7] = static_cast<float>(pad_y);
    if (!size_ok) atomicAdd(o.status, 1);
  }
  const double* L = lab + static_cast<long long>(i) * MF_TARGET_LABEL_COLS;
  if (!size_ok || L[L_VALID] == 0.0) return;
  const int cls = static_cast<int>(L[L_CLS]);
  if (cls < 0 || cls >= NCLS || static_cast<double>(cls) != L[L_CLS]) { atomicAdd(o.status, 1); return; }
  const double trunc = L[L_TRUNC], occ = L[L_OCC];
  const double oh_ = L[L_H], ow_ = L[L_W], ol_ = L[L_L];
  float tx = static_cast<float>(L[L_TX]);
  const float ty = static_cast<float>(L[L_TY]), tz = static_cast<float>(L[L_TZ]);
  double ry = L[L_RY];
  float lbox[4];
  if (right) {                                                         // the box columns of the row are not used
    right_view_box(P2 + 12 * b, ry, tx, ty, tz, oh_, ow_, ol_, img_w, img_h, lbox);
    if (flip) {                                                        // augmentations.py:42-44 on np.float32 scalars
      const float bw = __fsub_rn(lbox[2], lbox[0]);
      lbox[0] = __fsub_rn(__fsub_rn(static_cast<float>(img_w), lbox[2]), 1.f);
      lbox[2] = __fadd_rn(lbox[0], bw);
    }
  } else {
    double xmin = L[L_X1], xmax = L[L_X2];
    if (flip) {                                                        // augmentations.py:42-44 on Python floats
      const double bw = dsub(xmax, xmin);
      xmin = dsub(dsub(static_cast<double>(img_w), xmax), 1.0);
      xmax = dadd(xmin, bw);
    }
    lbox[0] = static_cast<float>(xmin);
    lbox[1] = static_cast<float>(L[L_Y1]);
    lbox[2] = static_cast<float>(xmax);
    lbox[3] = static_cast<float>(L[L_Y2]);
  }
  if (flip) {                                                          // augmentations.py:47-65
    ry = wrap_pi(ry < 0 ? dsub(-PI, ry) : dsub(PI, ry));
    tx = -tx;
  }
  const double alpha = wrap_pi(dsub(ry, atan2(static_cast<double>(tx), static_cast<double>(tz))));   // convertRot2Alpha

  const float locy = __fsub_rn(ty, static_cast<float>(oh_ / 2));      // float32 locs[1] - obj.h / 2
  if (tz <= 0.f) return;                                               // behind the camera

  // generate_corners3d, then the two face centres; projected with P
  double X[10], Y[10], Z[10], U[10], V[10];
  box_corners(ry, tx, ty, tz, oh_, ow_, ol_, X, Y, Z);
#pragma unroll
  for (int f = 0; f < 2; ++f) {                                        // corners_3d[:4].mean(0), corners_3d[4:].mean(0)
    const int k0 = 4 * f;
    X[8 + f] = dadd(dadd(dadd(X[k0], X[k0 + 1]), X[k0 + 2]), X[k0 + 3]) / 4;
    Y[8 + f] = dadd(dadd(dadd(Y[k0], Y[k0 + 1]), Y[k0 + 2]), Y[k0 + 3]) / 4;
    Z[8 + f] = dadd(dadd(dadd(Z[k0], Z[k0 + 1]), Z[k0 + 2]), Z[k0 + 3]) / 4;
  }
#pragma unroll
  for (int k = 0; k < 10; ++k) project(P, X[k], Y[k], Z[k], U[k], V[k]);
  double pminx = U[0], pmaxx = U[0], pminy = V[0], pmaxy = V[0];
  for (int k = 1; k < 8; ++k) {
    pminx = fmin(pminx, U[k]); pmaxx = fmax(pmaxx, U[k]);
    pminy = fmin(pminy, V[k]); pmaxy = fmax(pmaxy, V[k]);
  }
  const double wm1 = img_w - 1, hm1 = img_h - 1;
  // box2d: the projected box (float64) when it lies inside the image, else the label box (float32)
  const bool proj_box = pminx >= 0 && pminy >= 0 && pmaxx <= wm1 && pmaxy <= hm1;
  double bd[4] = {pminx, pminy, pmaxx, pmaxy};
  float bf[4] = {lbox[0], lbox[1], lbox[2], lbox[3]};
  const double min_dim = proj_box ? fmin(dsub(bd[2], bd[0]), dsub(bd[3], bd[1]))
                                  : static_cast<double>(fminf(__fsub_rn(bf[2], bf[0]), __fsub_rn(bf[3], bf[1])));
  if (trunc >= 0.9 && min_dim <= 20) return;                           // FILTER_ANNOS [0.9, 20]

  double pcu, pcv;
  project(P, static_cast<double>(tx), static_cast<double>(locy), static_cast<double>(tz), pcu, pcv);
  const bool inside = pcu >= 0 && pcu <= wm1 && pcv >= 0 && pcv <= hm1;
  double tpu = pcu, tpv = pcv;
  if (!inside) {                                                       // approx_proj_center (kitti_utils.py:990-1028)
    double cx, cy;
    if (proj_box) { cx = dadd(bd[0], bd[2]) / 2; cy = dadd(bd[1], bd[3]) / 2; }
    else { cx = __fdiv_rn(__fadd_rn(bf[0], bf[2]), 2.f); cy = __fdiv_rn(__fadd_rn(bf[1], bf[3]), 2.f); }
    if (!(cx >= 0 && cy >= 0 && cx <= wm1 && cy <= hm1) || cx == pcu) { atomicAdd(o.status, 1); return; }
    const double a = ddiv(dsub(cy, pcv), dsub(cx, pcu));                // the line through both points, y = a x + b
    const double bb = dsub(pcv, dmul(a, pcu));
    double cand[4][2];
    int n = 0;
    const double left_y = bb;
    if (0 <= left_y && left_y <= hm1) { cand[n][0] = 0; cand[n][1] = left_y; ++n; }
    const double right_y = dadd(dmul(wm1, a), bb);
    if (0 <= right_y && right_y <= hm1) { cand[n][0] = wm1; cand[n][1] = right_y; ++n; }
    const double top_x = ddiv(-bb, a);
    if (0 <= top_x && top_x <= wm1) { cand[n][0] = top_x; cand[n][1] = 0; ++n; }
    const double bottom_x = ddiv(dsub(hm1, bb), a);
    if (0 <= bottom_x && bottom_x <= wm1) { cand[n][0] = bottom_x; cand[n][1] = hm1; ++n; }
    if (n == 0) { atomicAdd(o.status, 1); return; }
    int best = 0;
    double best_d = 0;
    for (int k = 0; k < n; ++k) {
      const double dx = dsub(cand[k][0], pcu), dy = dsub(cand[k][1], pcv);
      const double d = __dsqrt_rn(dadd(dmul(dx, dx), dmul(dy, dy)));
      if (k == 0 || d < best_d) { best = k; best_d = d; }
    }
    tpu = cand[best][0];
    tpv = cand[best][1];
  }

  // key-point visibility with KEYPOINT_VISIBLE_MODIFY
  bool vis[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) vis[k] = U[k] >= 0 && U[k] <= wm1 && V[k] >= 0 && V[k] <= hm1 && Z[k] > 0;
  bool mv[10];
#pragma unroll
  for (int k = 0; k < 8; ++k) mv[k] = vis[k & 3] || vis[(k & 3) + 4];
  mv[8] = mv[9] = vis[8] || vis[9];
  const float kpd[3] = {static_cast<float>(mv[8] && mv[9]), static_cast<float>(mv[0] && mv[2] && mv[4] && mv[6]),
                        static_cast<float>(mv[1] && mv[3] && mv[5] && mv[7])};

  // to the feature map (stride 4)
  const double px = pad_x, py = pad_y;
  tpu = dadd(tpu, px) / DOWN; tpv = dadd(tpv, py) / DOWN;
  pcu = dadd(pcu, px) / DOWN; pcv = dadd(pcv, py) / DOWN;
  double box[4], dimx, dimy;
  if (proj_box) {
    for (int k = 0; k < 4; ++k) bd[k] = dadd(bd[k], (k & 1) ? py : px) / DOWN;
    for (int k = 0; k < 4; ++k) box[k] = bd[k];
    dimx = dsub(bd[2], bd[0]); dimy = dsub(bd[3], bd[1]);
  } else {
    for (int k = 0; k < 4; ++k) bf[k] = __fdiv_rn(__fadd_rn(bf[k], static_cast<float>((k & 1) ? pad_y : pad_x)), 4.f);
    for (int k = 0; k < 4; ++k) box[k] = bf[k];
    dimx = __fsub_rn(bf[2], bf[0]); dimy = __fsub_rn(bf[3], bf[1]);
  }
  const int x_min = (pad_x + DOWN - 1) / DOWN, y_min = (pad_y + DOWN - 1) / DOWN;
  const int x_max = (pad_x + img_w - 1) / DOWN, y_max = (pad_y + img_h - 1) / DOWN;
  // numpy .round() is half-to-even; then np.clip to the un-padded border
  const int tcx = min(max(static_cast<int>(rint(tpu)), x_min), x_max);
  const int tcy = min(max(static_cast<int>(rint(tpv)), y_min), y_max);
  const bool pred_2d = tcx >= box[0] && tcy >= box[1] && tcx <= box[2] && tcy <= box[3];
  if (!(dimx > 0 && dimy > 0 && tcx >= 0 && tcx <= W / DOWN - 1 && tcy >= 0 && tcy <= H / DOWN - 1)) return;

  int rx, ryad;
  if (!inside) {                                                       // one-sided Gaussian for outside objects
    const double bw = fmin(tcx - box[0], box[2] - tcx), bh = fmin(tcy - box[1], box[3] - tcy);
    rx = py_int_nonneg(dmul(bw, 0.5));
    ryad = py_int_nonneg(dmul(bh, 0.5));
    if (min(rx, ryad) != 0) { atomicAdd(o.status, 1); return; }
  } else {
    const double r = proj_box ? gaussian_radius_f64(dimy, dimx)
                              : static_cast<double>(gaussian_radius_f32(static_cast<float>(dimy), static_cast<float>(dimx)));
    rx = ryad = py_int_nonneg(r);
  }

  ob[O_CLS] = static_cast<float>(cls);
  ob[O_TC] = static_cast<float>(tcx);
  ob[O_TC + 1] = static_cast<float>(tcy);
  if (pred_2d)
    for (int k = 0; k < 4; ++k) ob[O_BOX + k] = static_cast<float>(box[k]);
  ob[O_REG] = 1.f;
  ob[O_TRUNC] = inside ? 0.f : 1.f;
  ob[O_DIM] = static_cast<float>(ol_);
  ob[O_DIM + 1] = static_cast<float>(oh_);
  ob[O_DIM + 2] = static_cast<float>(ow_);
  ob[O_LOC] = tx;
  ob[O_LOC + 1] = locy;
  ob[O_LOC + 2] = tz;
  ob[O_ROTY] = static_cast<float>(ry);
  ob[O_OFF] = static_cast<float>(dsub(pcu, tcx));
  ob[O_OFF + 1] = static_cast<float>(dsub(pcv, tcy));
  {                                                                    // encode_alpha_multibin, 4 bins, margin 1/6
    const double bin = 2 * PI / 4;
    const double range = dadd(bin / 2, dmul(bin, 1.0 / 6));
    const double centers[4] = {0, PI / 2, PI, -PI / 2};
    for (int k = 0; k < 4; ++k) {
      double off = dsub(alpha, centers[k]);
      if (off > PI) off = dsub(off, 2 * PI);
      if (off < -PI) off = dadd(off, 2 * PI);
      if (fabs(off) < range) { ob[O_ORI + k] = 1.f; ob[O_ORI + 4 + k] = static_cast<float>(off); }
    }
  }
  for (int k = 0; k < 3; ++k) ob[O_KPD + k] = kpd[k];
  for (int k = 0; k < 10; ++k) {
    ob[O_KP + 3 * k] = static_cast<float>(dsub(dadd(U[k], px) / DOWN, tcx));
    ob[O_KP + 3 * k + 1] = static_cast<float>(dsub(dadd(V[k], py) / DOWN, tcy));
    ob[O_KP + 3 * k + 2] = mv[k] ? 1.f : 0.f;
  }
  for (int k = 0; k < 4; ++k) o.gt_bboxes[4 * i + k] = lbox[k];
  o.alphas[i] = static_cast<float>(alpha);
  o.reg_weight[i] = 1.f;
  o.occlusions[i] = occ;
  o.truncations[i] = trunc;
  int* h6 = o.obj6 + 6 * i;
  h6[0] = 1; h6[1] = cls; h6[2] = tcx; h6[3] = tcy; h6[4] = rx; h6[5] = ryad;
}

// get_edge_utils (kitti.py:126-179): left (top to bottom), bottom (left to right), right (bottom to top), top (right to left,
// both corners), zero padded to K = 2 (W/4 + H/4) entries; edge_len = count - 1 (kitti.py:285)
__global__ void __launch_bounds__(256) encode_edges_kernel(const int* __restrict__ sizes, int B, int H, int W, int K,
                                                           long long* __restrict__ edge, long long* __restrict__ edge_len) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * K) return;
  const int b = i / K, k = i - b * K;
  const int img_w = sizes[2 * b], img_h = sizes[2 * b + 1];
  const int pad_x = (W - img_w) / 2, pad_y = (H - img_h) / 2;
  const int x_min = (pad_x + DOWN - 1) / DOWN, y_min = (pad_y + DOWN - 1) / DOWN;
  const int x_max = (pad_x + img_w - 1) / DOWN, y_max = (pad_y + img_h - 1) / DOWN;
  const int ny = max(y_max - y_min, 0), nx = max(x_max - x_min, 0), nt = max(x_max - x_min + 1, 0);
  long long x = 0, y = 0;
  int j = k;
  if (j < ny) { x = x_min; y = y_min + j; }
  else if ((j -= ny) < nx) { x = x_min + j; y = y_max; }
  else if ((j -= nx) < ny) { x = x_max; y = y_max - j; }
  else if ((j -= ny) < nt) { x = x_max - j; y = y_min; }
  edge[2LL * i] = x;
  edge[2LL * i + 1] = y;
  if (k == 0) edge_len[b] = 2 * ny + nx + nt - 1;
}

int launch_edges(const int* sizes, int B, int H, int W, long long* edge, long long* edge_len, cudaStream_t st) {
  const int K = 2 * (W / DOWN + H / DOWN);
  const long long n = static_cast<long long>(B) * K;
  (void)launch_k(encode_edges_kernel, dim3(static_cast<unsigned>((n + 255) / 256)), dim3(256), 0, st, sizes, B, H, W, K, edge,
                 edge_len);
  return check_cuda(cudaGetLastError(), "encode_edges");
}

}  // namespace
}  // namespace mf

using namespace mf;

extern "C" {

int mf_encode_targets_views(const double* labels, const double* P2, const int* sizes, const int* flips, const int* right, int B,
                            int M, int H, int W, float* hm, float* obj, float* img, float* alphas, float* gt_bboxes,
                            float* reg_weight, double* occlusions, double* truncations, int* obj6, double* P2_out,
                            long long* edge_indices, long long* edge_len, int* status, void* stream) {
  if (B < 1 || M < 1 || H < DOWN || W < DOWN || H % DOWN || W % DOWN) {
    set_error("mf_encode_targets_views: B=%d M=%d H=%d W=%d (H and W multiples of %d)", B, M, H, W, DOWN);
    return -1;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cudaError_t e = cudaMemsetAsync(status, 0, sizeof(int), st);
  if (e != cudaSuccess) return check_cuda(e, "encode_targets status");
  TargetOut o{obj, img, alphas, gt_bboxes, reg_weight, occlusions, truncations, obj6, P2_out, status};
  const int n = B * M;
  (void)launch_k(encode_objects_kernel, dim3(static_cast<unsigned>((n + 127) / 128)), dim3(128), 0, st, labels, P2, sizes, flips,
                 right, B, M, H, W, o);
  int rc = check_cuda(cudaGetLastError(), "encode_objects");
  if (rc) return rc;
  rc = launch_draw_heatmap(obj6, B, M, NCLS, H / DOWN, W / DOWN, hm, st);
  if (rc) return rc;
  return launch_edges(sizes, B, H, W, edge_indices, edge_len, st);
}

int mf_encode_targets(const double* labels, const double* P2, const int* sizes, const int* flips, int B, int M, int H, int W,
                      float* hm, float* obj, float* img, float* alphas, float* gt_bboxes, float* reg_weight,
                      double* occlusions, double* truncations, int* obj6, double* P2_out, long long* edge_indices,
                      long long* edge_len, int* status, void* stream) {
  if (B < 1 || M < 1 || H < DOWN || W < DOWN || H % DOWN || W % DOWN) {
    set_error("mf_encode_targets: B=%d M=%d H=%d W=%d (H and W multiples of %d)", B, M, H, W, DOWN);
    return -1;
  }
  return mf_encode_targets_views(labels, P2, sizes, flips, nullptr, B, M, H, W, hm, obj, img, alphas, gt_bboxes, reg_weight,
                                 occlusions, truncations, obj6, P2_out, edge_indices, edge_len, status, stream);
}

int mf_encode_edges(const int* sizes, int B, int H, int W, long long* edge_indices, long long* edge_len, void* stream) {
  if (B < 1 || H < DOWN || W < DOWN || H % DOWN || W % DOWN) {
    set_error("mf_encode_edges: B=%d H=%d W=%d (H and W multiples of %d)", B, H, W, DOWN);
    return -1;
  }
  return launch_edges(sizes, B, H, W, edge_indices, edge_len, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
