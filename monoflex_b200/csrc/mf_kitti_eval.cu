// KITTI official 3D-detection metric (data/datasets/evaluation/kitti_object_eval_python/eval.py, rotate_iou.py):
// 2D / BEV / 3D precision-recall tables, AOS and AP|R40 / AP|R11 for every (metric, class, difficulty, overlap set) at once.
//
// Objects are CSR-packed per image as float64 rows of MF_KITTI_OBJ values (see include/monoflex_b200.h). Stages:
//   overlaps    one CTA per image: the detection x ground-truth blocks of metric 0 (2D), 1 (BEV) and 2 (3D);
//   statistics  flags (clean_data), the compute_fp=False pass, a segmented sort of the true-positive scores, get_thresholds
//               (sequential per configuration), the compute_fp=True pass per (configuration, threshold) over all images;
//   ap          recall / precision / AOS, their suffix maxima and both AP sums.
// The launch count depends on neither the number of images nor of configurations. Greedy matching is sequential inside one
// (image, threshold) as in the reference, and parallel across them; the AOS similarity is summed over images in image
// order like the reference's pr[t, 3], the integer counts in any order. No floating-point atomics.
#include "mf_common.cuh"
#include "../../include/monoflex_b200.h"
#include <cub/device/device_segmented_radix_sort.cuh>
#include <math.h>

namespace mf {
namespace {

constexpr int OBJ = MF_KITTI_OBJ;
constexpr int NPTS = 41;                   // N_SAMPLE_PTS
constexpr int MAX_DT = MF_KITTI_MAX_DT;    // detections per image: the assigned-detection bitmask lives in registers
constexpr int MAX_CLS = 8;
constexpr int STAT_THREADS = 128;
constexpr int THR_THREADS = 256;
constexpr double NO_DETECTION = -10000000.0;

// object columns
enum { C_CLS = 0, C_TRUNC, C_OCC, C_ALPHA, C_X1, C_Y1, C_X2, C_Y2, C_L, C_H, C_W, C_X, C_Y, C_Z, C_RY, C_SCORE };

struct Classes { int c[MAX_CLS]; };

// get_official_eval_result's min_overlaps[k][metric][class] (overlap_0_7, overlap_0_5)
__constant__ double c_min_overlap[2][3][6] = {
    {{0.7, 0.5, 0.5, 0.7, 0.5, 0.7}, {0.7, 0.5, 0.5, 0.7, 0.5, 0.7}, {0.7, 0.5, 0.5, 0.7, 0.5, 0.7}},
    {{0.7, 0.5, 0.5, 0.7, 0.5, 0.5}, {0.5, 0.25, 0.25, 0.5, 0.25, 0.5}, {0.5, 0.25, 0.25, 0.5, 0.25, 0.5}}};
__constant__ double c_min_height[3] = {40, 25, 25};
__constant__ double c_max_occlusion[3] = {0, 1, 2};
__constant__ double c_max_truncation[3] = {0.15, 0.3, 0.5};

// Python's min / max: the first argument unless the second is strictly smaller / larger
MF_DEVINL double pmin(double a, double b) { return b < a ? b : a; }
MF_DEVINL double pmax(double a, double b) { return b > a ? b : a; }

// image_box_overlap for one pair, criterion -1 (IoU) or 0 (over the first box's area), float64 without contraction
MF_DEVINL double box_overlap(const double* b, const double* q, bool iou) {
  const double iw = __dsub_rn(pmin(b[2], q[2]), pmax(b[0], q[0]));
  if (!(iw > 0)) return 0.0;
  const double ih = __dsub_rn(pmin(b[3], q[3]), pmax(b[1], q[1]));
  if (!(ih > 0)) return 0.0;
  const double barea = __dmul_rn(__dsub_rn(b[2], b[0]), __dsub_rn(b[3], b[1]));
  const double inter = __dmul_rn(iw, ih);
  double ua = barea;
  if (iou) ua = __dsub_rn(__dadd_rn(barea, __dmul_rn(__dsub_rn(q[2], q[0]), __dsub_rn(q[3], q[1]))), inter);
  return __ddiv_rn(inter, ua);
}

// ---------------------------------------------------------------------------------------------------- rotated BEV boxes
// rotate_iou.py in numba's types: float32 corners, clipping and vertex sort; trangle_area's `/ 2.0` makes the triangle-fan
// area and the IoU ratio float64, rounded once to float32 where the reference stores them into dev_iou.
MF_DEVINL void rbox_corners(float x, float z, float l, float w, float ry, float* c) {
  // cos / sin of the float32 angle correctly rounded to float32, as math.cos / math.sin meet the float32 corners
  const float ca = static_cast<float>(cos(static_cast<double>(ry))), sa = static_cast<float>(sin(static_cast<double>(ry)));
  const float cx[4] = {-l / 2, -l / 2, l / 2, l / 2};
  const float cy[4] = {-w / 2, w / 2, w / 2, -w / 2};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    c[2 * i] = __fadd_rn(__fadd_rn(__fmul_rn(ca, cx[i]), __fmul_rn(sa, cy[i])), x);
    c[2 * i + 1] = __fadd_rn(__fadd_rn(__fmul_rn(-sa, cx[i]), __fmul_rn(ca, cy[i])), z);
  }
}

MF_DEVINL bool point_in_quad(float px, float py, const float* c) {
  const float ab0 = c[2] - c[0], ab1 = c[3] - c[1];
  const float ad0 = c[6] - c[0], ad1 = c[7] - c[1];
  const float ap0 = px - c[0], ap1 = py - c[1];
  const float abab = __fadd_rn(__fmul_rn(ab0, ab0), __fmul_rn(ab1, ab1));
  const float abap = __fadd_rn(__fmul_rn(ab0, ap0), __fmul_rn(ab1, ap1));
  const float adad = __fadd_rn(__fmul_rn(ad0, ad0), __fmul_rn(ad1, ad1));
  const float adap = __fadd_rn(__fmul_rn(ad0, ap0), __fmul_rn(ad1, ap1));
  return abab >= abap && abap >= 0 && adad >= adap && adap >= 0;
}

MF_DEVINL bool segment_intersection(const float* p1, const float* p2, int i, int j, float* out) {
  const float A0 = p1[2 * i], A1 = p1[2 * i + 1];
  const float B0 = p1[2 * ((i + 1) % 4)], B1 = p1[2 * ((i + 1) % 4) + 1];
  const float C0 = p2[2 * j], C1 = p2[2 * j + 1];
  const float D0 = p2[2 * ((j + 1) % 4)], D1 = p2[2 * ((j + 1) % 4) + 1];
  const float BA0 = B0 - A0, BA1 = B1 - A1, DA0 = D0 - A0, CA0 = C0 - A0, DA1 = D1 - A1, CA1 = C1 - A1;
  const bool acd = __fmul_rn(DA1, CA0) > __fmul_rn(CA1, DA0);
  const bool bcd = __fmul_rn(D1 - B1, C0 - B0) > __fmul_rn(C1 - B1, D0 - B0);
  if (acd == bcd) return false;
  const bool abc = __fmul_rn(CA1, BA0) > __fmul_rn(BA1, CA0);
  const bool abd = __fmul_rn(DA1, BA0) > __fmul_rn(BA1, DA0);
  if (abc == abd) return false;
  const float DC0 = D0 - C0, DC1 = D1 - C1;
  const float ABBA = __fsub_rn(__fmul_rn(A0, B1), __fmul_rn(B0, A1));
  const float CDDC = __fsub_rn(__fmul_rn(C0, D1), __fmul_rn(D0, C1));
  const float DH = __fsub_rn(__fmul_rn(BA1, DC0), __fmul_rn(BA0, DC1));
  const float Dx = __fsub_rn(__fmul_rn(ABBA, DC0), __fmul_rn(BA0, CDDC));
  const float Dy = __fsub_rn(__fmul_rn(ABBA, DC1), __fmul_rn(BA1, CDDC));
  out[0] = __fdiv_rn(Dx, DH);
  out[1] = __fdiv_rn(Dy, DH);
  return true;
}

// intersection area of two rotated rectangles (x, z, l, w, ry): clip points, sort around their centre, fan of triangles
__device__ double rbox_inter(const float* r1, const float* r2) {
  float c1[8], c2[8], pts[48], vs[24];
  rbox_corners(r1[0], r1[1], r1[2], r1[3], r1[4], c1);
  rbox_corners(r2[0], r2[1], r2[2], r2[3], r2[4], c2);
  int n = 0;
  for (int i = 0; i < 4; ++i) {
    if (point_in_quad(c1[2 * i], c1[2 * i + 1], c2)) { pts[2 * n] = c1[2 * i]; pts[2 * n + 1] = c1[2 * i + 1]; ++n; }
    if (point_in_quad(c2[2 * i], c2[2 * i + 1], c1)) { pts[2 * n] = c2[2 * i]; pts[2 * n + 1] = c2[2 * i + 1]; ++n; }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j)
      if (segment_intersection(c1, c2, i, j, pts + 2 * n)) ++n;
  if (n > 0) {
    float cx = 0.f, cy = 0.f;
    for (int i = 0; i < n; ++i) { cx += pts[2 * i]; cy += pts[2 * i + 1]; }
    cx = __fdiv_rn(cx, static_cast<float>(n));
    cy = __fdiv_rn(cy, static_cast<float>(n));
    for (int i = 0; i < n; ++i) {
      float v0 = pts[2 * i] - cx, v1 = pts[2 * i + 1] - cy;
      const float d = sqrtf(__fadd_rn(__fmul_rn(v0, v0), __fmul_rn(v1, v1)));
      v0 = __fdiv_rn(v0, d);
      v1 = __fdiv_rn(v1, d);
      if (v1 < 0) v0 = -2 - v0;
      vs[i] = v0;
    }
    for (int i = 1; i < n; ++i) {
      if (vs[i - 1] > vs[i]) {
        const float t = vs[i], tx = pts[2 * i], ty = pts[2 * i + 1];
        int j = i;
        while (j > 0 && vs[j - 1] > t) {
          vs[j] = vs[j - 1];
          pts[2 * j] = pts[2 * j - 2];
          pts[2 * j + 1] = pts[2 * j - 1];
          --j;
        }
        vs[j] = t;
        pts[2 * j] = tx;
        pts[2 * j + 1] = ty;
      }
    }
  }
  double area = 0.0;
  for (int i = 0; i + 2 < n; ++i) {
    const float* a = pts;
    const float* b = pts + 2 * i + 2;
    const float* c = pts + 2 * i + 4;
    const float t = __fsub_rn(__fmul_rn(a[0] - c[0], b[1] - c[1]), __fmul_rn(a[1] - c[1], b[0] - c[0]));
    area = __dadd_rn(area, fabs(static_cast<double>(t) / 2.0));
  }
  return area;
}

// ------------------------------------------------------------------------------------------------------------ overlaps
// ov[metric][pair_off[i] + d * ng + g]: the reference's diagonal block overlaps[i] of calculate_iou_partly(dt, gt, metric)
__global__ void overlaps_kernel(const double* __restrict__ gt, const int* __restrict__ gt_off, const double* __restrict__ dt,
                                const int* __restrict__ dt_off, const long long* __restrict__ pair_off, long long n_pair,
                                double* __restrict__ ov) {
  const int img = blockIdx.x;
  const int g0 = gt_off[img], ng = gt_off[img + 1] - g0, d0 = dt_off[img], nd = dt_off[img + 1] - d0;
  const long long base = pair_off[img];
  for (int q = threadIdx.x; q < nd * ng; q += blockDim.x) {
    const int d = q / ng, g = q - d * ng;
    const double* D = dt + static_cast<long long>(d0 + d) * OBJ;
    const double* G = gt + static_cast<long long>(g0 + g) * OBJ;
    ov[base + q] = box_overlap(D + C_X1, G + C_X1, true);
    // rotate_iou_gpu_eval(dt, gt): the kernel evaluates devRotateIoUEval(gt box, dt box) in float32
    const float rg[5] = {static_cast<float>(G[C_X]), static_cast<float>(G[C_Z]), static_cast<float>(G[C_L]),
                         static_cast<float>(G[C_W]), static_cast<float>(G[C_RY])};
    const float rd[5] = {static_cast<float>(D[C_X]), static_cast<float>(D[C_Z]), static_cast<float>(D[C_L]),
                         static_cast<float>(D[C_W]), static_cast<float>(D[C_RY])};
    const double inter = rbox_inter(rg, rd);
    const float area_sum = __fadd_rn(__fmul_rn(rg[2], rg[3]), __fmul_rn(rd[2], rd[3]));   // area1 + area2 in float32
    ov[n_pair + base + q] = static_cast<double>(static_cast<float>(
        __ddiv_rn(inter, __dsub_rn(static_cast<double>(area_sum), inter))));
    // d3_box_overlap: criterion-2 area (stored as float32), y-overlap and union in float64, ratio stored as float32
    const float rinc = static_cast<float>(inter);
    double r3 = rinc;
    if (rinc > 0) {
      const double iw = __dsub_rn(pmin(D[C_Y], G[C_Y]), pmax(__dsub_rn(D[C_Y], D[C_H]), __dsub_rn(G[C_Y], G[C_H])));
      if (iw > 0) {
        const double a1 = __dmul_rn(__dmul_rn(D[C_L], D[C_H]), D[C_W]);
        const double a2 = __dmul_rn(__dmul_rn(G[C_L], G[C_H]), G[C_W]);
        const double inc = __dmul_rn(iw, static_cast<double>(rinc));
        r3 = static_cast<double>(static_cast<float>(__ddiv_rn(inc, __dsub_rn(__dadd_rn(a1, a2), inc))));
      } else {
        r3 = 0.0;
      }
    }
    ov[2 * n_pair + base + q] = r3;
  }
}

// ------------------------------------------------------------------------------------------------------------ statistics
struct StatArgs {
  const double* gt; const int* gt_off; const double* dt; const int* dt_off; const long long* pair_off; const double* ov;
  int n_img, n_gt, n_dt, ncls; long long n_pair;
  Classes cls;
  signed char* fg; signed char* fd;   // clean_data flags [ncls * 3][n_gt] / [ncls * 3][n_dt]
  int* seg;                           // [C + 1] segment offsets of the score sort
  double* tps; double* tps_sorted;    // [C][n_gt] true-positive scores of the first pass, -inf padded
  double* thr; int* nthr;             // [C][41], [C]
  double* pr;                         // [C][41][4] tp, fp, fn, similarity
  int* aos;                           // [2]: compute_aos of get_official_eval_result, largest over-limit image (0: none)
};

// configuration c = ((metric * ncls + m) * 3 + difficulty) * 2 + k
struct Cfg { int metric, m, l, k; double min_overlap; };
MF_DEVINL Cfg config(const StatArgs& a, int c) {
  Cfg f;
  f.k = c % 2; f.l = (c / 2) % 3; f.m = (c / 6) % a.ncls; f.metric = c / (6 * a.ncls);
  f.min_overlap = c_min_overlap[f.k][f.metric][a.cls.c[f.m]];
  return f;
}

__global__ void flags_kernel(StatArgs a) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  const int C = 18 * a.ncls;
  if (x <= C) a.seg[x] = x * a.n_gt;
  if (x == 0) { a.aos[0] = a.n_dt > 0 && a.dt[C_ALPHA] != -10.0; a.aos[1] = 0; }
  if (x < a.n_gt) {
    const double* o = a.gt + static_cast<long long>(x) * OBJ;
    const int code = static_cast<int>(o[C_CLS]);
    const double h = __dsub_rn(o[C_Y2], o[C_Y1]);
    for (int m = 0; m < a.ncls; ++m) {
      const int cls = a.cls.c[m];
      const int valid = code == cls ? 1 : ((cls == 1 && code == 4) || (cls == 0 && code == 3)) ? 0 : -1;
      for (int l = 0; l < 3; ++l) {
        const bool ignore = o[C_OCC] > c_max_occlusion[l] || o[C_TRUNC] > c_max_truncation[l] || h <= c_min_height[l];
        a.fg[static_cast<long long>(m * 3 + l) * a.n_gt + x] =
            (valid == 1 && !ignore) ? 0 : (valid == 0 || (ignore && valid == 1)) ? 1 : -1;
      }
    }
  } else if (x < a.n_gt + a.n_dt) {
    const int y = x - a.n_gt;
    const double* o = a.dt + static_cast<long long>(y) * OBJ;
    const int code = static_cast<int>(o[C_CLS]);
    const double h = fabs(__dsub_rn(o[C_Y2], o[C_Y1]));
    for (int m = 0; m < a.ncls; ++m)
      for (int l = 0; l < 3; ++l)
        a.fd[static_cast<long long>(m * 3 + l) * a.n_dt + y] = h < c_min_height[l] ? 1 : code == a.cls.c[m] ? 0 : -1;
  }
}

MF_DEVINL bool bit(const unsigned* s, int j) { return (s[j >> 5] >> (j & 31)) & 1u; }
MF_DEVINL void set_bit(unsigned* s, int j) { s[j >> 5] |= 1u << (j & 31); }

// compute_statistics_jit(compute_fp=False, thresh=0) per (configuration, image): the scores of the true positives, in order
__global__ void first_pass_kernel(StatArgs a) {
  const long long x = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (x >= static_cast<long long>(18 * a.ncls) * a.n_img) return;
  const int c = static_cast<int>(x / a.n_img), img = static_cast<int>(x % a.n_img);
  const Cfg f = config(a, c);
  const int g0 = a.gt_off[img], ng = a.gt_off[img + 1] - g0, d0 = a.dt_off[img], nd = a.dt_off[img + 1] - d0;
  double* out = a.tps + static_cast<long long>(c) * a.n_gt + g0;
  if (nd > MAX_DT) {                                     // never truncated: reported through the AP stage's output
    atomicMax(a.aos + 1, nd);
    for (int g = 0; g < ng; ++g) out[g] = -INFINITY;
    return;
  }
  const signed char* fg = a.fg + static_cast<long long>(f.m * 3 + f.l) * a.n_gt + g0;
  const signed char* fd = a.fd + static_cast<long long>(f.m * 3 + f.l) * a.n_dt + d0;
  const double* ov = a.ov + f.metric * a.n_pair + a.pair_off[img];
  const double* dts = a.dt + static_cast<long long>(d0) * OBJ;
  unsigned assigned[MAX_DT / 32] = {};
  int ntp = 0;
  for (int g = 0; g < ng; ++g) {
    if (fg[g] == -1) continue;
    int det = -1;
    double valid = NO_DETECTION;
    for (int j = 0; j < nd; ++j) {
      if (fd[j] == -1 || bit(assigned, j)) continue;
      const double s = dts[j * OBJ + C_SCORE];
      if (ov[j * ng + g] > f.min_overlap && s > valid) { det = j; valid = s; }
    }
    if (valid == NO_DETECTION) continue;                 // a false negative when fg == 0
    if (fg[g] == 0 && fd[det] != 1) out[ntp++] = dts[det * OBJ + C_SCORE];
    set_bit(assigned, det);
  }
  for (int g = ntp; g < ng; ++g) out[g] = -INFINITY;
}

// get_thresholds per configuration: the number of valid ground-truth objects, then the float64 recall recurrence
__global__ void thresholds_kernel(StatArgs a) {
  const int c = blockIdx.x;
  const Cfg f = config(a, c);
  const signed char* fg = a.fg + static_cast<long long>(f.m * 3 + f.l) * a.n_gt;
  const double* s = a.tps_sorted + static_cast<long long>(c) * a.n_gt;
  int num_gt = 0, n = 0;
  for (int b = 0; b < a.n_gt; b += blockDim.x) {
    const int x = b + threadIdx.x;
    num_gt += __syncthreads_count(x < a.n_gt && fg[x] == 0);
    n += __syncthreads_count(x < a.n_gt && s[x] != -INFINITY);
  }
  if (threadIdx.x != 0) return;
  double* thr = a.thr + c * NPTS;
  double current = 0.0;
  int nt = 0;
  for (int i = 0; i < n; ++i) {
    const double l_recall = static_cast<double>(i + 1) / num_gt;
    const double r_recall = i < n - 1 ? static_cast<double>(i + 2) / num_gt : l_recall;
    if ((r_recall - current) < (current - l_recall) && i < n - 1) continue;
    if (nt < NPTS) thr[nt++] = s[i];
    current += 1.0 / (NPTS - 1.0);
  }
  a.nthr[c] = nt;
}

// compute_statistics_jit(compute_fp=True) for every image at one (configuration, threshold), summed over the images
__global__ void __launch_bounds__(STAT_THREADS) second_pass_kernel(StatArgs a) {
  const int c = blockIdx.x / NPTS, t = blockIdx.x % NPTS;
  if (t >= a.nthr[c]) return;
  const Cfg f = config(a, c);
  const double thresh = a.thr[c * NPTS + t];
  const bool aos = f.metric == 0 && a.aos[0];
  long long tp = 0, fp = 0, fn = 0;
  double sim = 0.0;                                       // thread 0: pr[t, 3] += similarity in image order
  __shared__ double s_sim[STAT_THREADS];
  for (int base = 0; base < a.n_img; base += blockDim.x) {
    const int img = base + threadIdx.x;
    double img_sim = 0.0;
    if (img < a.n_img) {
      const int g0 = a.gt_off[img], ng = a.gt_off[img + 1] - g0, d0 = a.dt_off[img], nd = a.dt_off[img + 1] - d0;
      if (nd <= MAX_DT) {                                 // larger images are reported by the first pass
        const signed char* fg = a.fg + static_cast<long long>(f.m * 3 + f.l) * a.n_gt + g0;
        const signed char* fd = a.fd + static_cast<long long>(f.m * 3 + f.l) * a.n_dt + d0;
        const double* ov = a.ov + f.metric * a.n_pair + a.pair_off[img];
        const double* dts = a.dt + static_cast<long long>(d0) * OBJ;
        const double* gts = a.gt + static_cast<long long>(g0) * OBJ;
        unsigned assigned[MAX_DT / 32] = {}, below[MAX_DT / 32] = {};
        for (int j = 0; j < nd; ++j)
          if (dts[j * OBJ + C_SCORE] < thresh) set_bit(below, j);
        int itp = 0, ifp = 0, ifn = 0;
        double isim = 0.0;
        for (int g = 0; g < ng; ++g) {
          if (fg[g] == -1) continue;
          int det = -1;
          bool found = false, assigned_ignored = false;
          double max_overlap = 0.0;
          for (int j = 0; j < nd; ++j) {
            if (fd[j] == -1 || bit(assigned, j) || bit(below, j)) continue;
            const double o = ov[j * ng + g];
            if (o > f.min_overlap && (o > max_overlap || assigned_ignored) && fd[j] == 0) {
              max_overlap = o; det = j; found = true; assigned_ignored = false;
            } else if (o > f.min_overlap && !found && fd[j] == 1) {
              det = j; found = true; assigned_ignored = true;
            }
          }
          if (!found) {
            if (fg[g] == 0) ++ifn;
            continue;
          }
          if (fg[g] == 0 && fd[det] != 1) {
            ++itp;
            if (aos) isim += (1.0 + cos(__dsub_rn(gts[g * OBJ + C_ALPHA], dts[det * OBJ + C_ALPHA]))) / 2.0;
          }
          set_bit(assigned, det);
        }
        for (int j = 0; j < nd; ++j)
          if (!bit(assigned, j) && fd[j] == 0 && !bit(below, j)) ++ifp;
        if (f.metric == 0) {                              // detections on DontCare regions are not false positives
          for (int g = 0; g < ng; ++g) {
            if (static_cast<int>(gts[g * OBJ + C_CLS]) != MF_KITTI_DONTCARE) continue;
            for (int j = 0; j < nd; ++j) {
              if (bit(assigned, j) || fd[j] != 0 || bit(below, j)) continue;
              if (box_overlap(dts + j * OBJ + C_X1, gts + g * OBJ + C_X1, false) > f.min_overlap) { set_bit(assigned, j); --ifp; }
            }
          }
        }
        tp += itp; fp += ifp; fn += ifn;
        if (aos && (itp > 0 || ifp > 0)) img_sim = isim;  // similarity -1 (no tp, no fp) is not added
      }
    }
    s_sim[threadIdx.x] = img_sim;
    __syncthreads();
    if (threadIdx.x == 0)
      for (int i = 0; i < STAT_THREADS && base + i < a.n_img; ++i) sim += s_sim[i];
    __syncthreads();
  }
  // the integer counts do not depend on the order: a tree over the threads
  __shared__ long long s_i[3][STAT_THREADS];
  s_i[0][threadIdx.x] = tp; s_i[1][threadIdx.x] = fp; s_i[2][threadIdx.x] = fn;
  __syncthreads();
  for (int w = STAT_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
      for (int q = 0; q < 3; ++q) s_i[q][threadIdx.x] += s_i[q][threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double* p = a.pr + (static_cast<long long>(c) * NPTS + t) * 4;
    p[0] = static_cast<double>(s_i[0][0]); p[1] = static_cast<double>(s_i[1][0]); p[2] = static_cast<double>(s_i[2][0]);
    p[3] = sim;
  }
}

// ------------------------------------------------------------------------------------------------------------ AP
// eval_class's tail and get_mAP_R40 / get_mAP; NaN from 0/0 propagates through the suffix maximum like np.max
MF_DEVINL double nanmax(double a, double b) { return (isnan(a) || isnan(b)) ? NAN : (b > a ? b : a); }

__global__ void ap_kernel(const double* __restrict__ pr, const int* __restrict__ nthr, const int* __restrict__ aos_flag,
                          int ncls, double* __restrict__ out) {
  const int C = 18 * ncls, c = threadIdx.x;
  if (c >= C) return;
  const int metric = c / (6 * ncls), rest = c % (6 * ncls);   // rest = (m * 3 + l) * 2 + k
  const bool aos = metric == 0 && aos_flag[0];
  double rec[NPTS], prec[NPTS], ori[NPTS];
  for (int i = 0; i < NPTS; ++i) {
    rec[i] = prec[i] = ori[i] = 0.0;
    if (i < nthr[c]) {
      const double* p = pr + (static_cast<long long>(c) * NPTS + i) * 4;
      rec[i] = p[0] / (p[0] + p[2]);
      prec[i] = p[0] / (p[0] + p[1]);
      if (aos) ori[i] = p[3] / (p[0] + p[1]);
    }
  }
  for (int i = NPTS - 2; i >= 0; --i) {
    rec[i] = nanmax(rec[i + 1], rec[i]);
    prec[i] = nanmax(prec[i + 1], prec[i]);
    ori[i] = nanmax(ori[i + 1], ori[i]);
  }
  const long long tab = static_cast<long long>(C) * NPTS;
  for (int i = 0; i < NPTS; ++i) {
    out[c * NPTS + i] = rec[i];
    out[tab + c * NPTS + i] = prec[i];
    out[2 * tab + c * NPTS + i] = ori[i];
  }
  // ap[R40, R11][bbox, bev, 3d, aos][ncls][3][2]
  double* ap = out + 3 * tab;
  const int per = 6 * ncls;
  double s40 = 0.0, s11 = 0.0, o40 = 0.0, o11 = 0.0;
  for (int i = 1; i < NPTS; ++i) { s40 = s40 + prec[i]; o40 = o40 + ori[i]; }
  for (int i = 0; i < NPTS; i += 4) { s11 = s11 + prec[i]; o11 = o11 + ori[i]; }
  ap[metric * per + rest] = s40 / 40 * 100;
  ap[4 * per + metric * per + rest] = s11 / 11 * 100;
  if (metric == 0) {
    ap[3 * per + rest] = o40 / 40 * 100;
    ap[4 * per + 3 * per + rest] = o11 / 11 * 100;
    if (rest == 0) { ap[8 * per] = aos_flag[0]; ap[8 * per + 1] = aos_flag[1]; }
  }
}

// generate_kitti_3d_detection's rows: np.round(x, 4) in float32, widened; (l, h, w) from the decode's (h, w, l)
__global__ void pack_results_kernel(const float* __restrict__ rows, int n, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double r[14];
  for (int q = 0; q < 14; ++q) r[q] = __fdiv_rn(rintf(__fmul_rn(rows[i * 14 + q], 1e4f)), 1e4f);
  const int cls = static_cast<int>(r[0]);
  const double o[OBJ] = {cls >= 0 && cls <= 2 ? static_cast<double>(cls) : -1.0, 0.0, 0.0, r[1], r[2], r[3], r[4], r[5],
                         r[8], r[6], r[7], r[9], r[10], r[11], r[12], r[13]};
  for (int q = 0; q < OBJ; ++q) out[static_cast<long long>(i) * OBJ + q] = o[q];
}

// workspace carve-up shared by the size query and the stages
struct Layout {
  size_t fg, fd, seg, tps, tps_sorted, thr, nthr, pr, aos, cub, cub_bytes, total;
};
size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }
Layout layout(int n_gt, int n_dt, int ncls) {
  const size_t C = 18 * static_cast<size_t>(ncls);
  Layout L;
  size_t o = 0;
  L.fg = o; o = align256(o + ncls * 3 * static_cast<size_t>(n_gt));
  L.fd = o; o = align256(o + ncls * 3 * static_cast<size_t>(n_dt));
  L.seg = o; o = align256(o + (C + 1) * sizeof(int));
  L.tps = o; o = align256(o + C * n_gt * sizeof(double));
  L.tps_sorted = o; o = align256(o + C * n_gt * sizeof(double));
  L.thr = o; o = align256(o + C * NPTS * sizeof(double));
  L.nthr = o; o = align256(o + C * sizeof(int));
  L.pr = o; o = align256(o + C * NPTS * 4 * sizeof(double));
  L.aos = o; o = align256(o + 2 * sizeof(int));
  L.cub_bytes = 0;
  cub::DeviceSegmentedRadixSort::SortKeysDescending(nullptr, L.cub_bytes, static_cast<const double*>(nullptr),
                                                    static_cast<double*>(nullptr), static_cast<int>(C * n_gt),
                                                    static_cast<int>(C), static_cast<const int*>(nullptr),
                                                    static_cast<const int*>(nullptr));
  L.cub = o; o = align256(o + L.cub_bytes);
  L.total = o;
  return L;
}

}  // namespace
}  // namespace mf

using namespace mf;

extern "C" {

size_t mf_kitti_eval_workspace(int n_gt, int n_dt, int ncls) {
  if (n_gt < 0 || n_dt < 0 || ncls < 1 || ncls > MAX_CLS) return 0;
  return layout(n_gt, n_dt, ncls).total;
}

int mf_kitti_pack_results(const float* rows, int n, double* out, void* stream) {
  if (n < 0) { set_error("mf_kitti_pack_results: n = %d", n); return -1; }
  if (n == 0) return 0;
  pack_results_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(rows, n, out);
  return check_cuda(cudaGetLastError(), "kitti_pack_results");
}

int mf_kitti_eval_overlaps(const double* gt, const int* gt_off, const double* dt, const int* dt_off,
                           const long long* pair_off, int n_img, long long n_pair, double* overlaps, void* stream) {
  if (n_img < 1 || n_pair < 0) { set_error("mf_kitti_eval_overlaps: %d images, %lld pairs", n_img, n_pair); return -1; }
  overlaps_kernel<<<n_img, 128, 0, static_cast<cudaStream_t>(stream)>>>(gt, gt_off, dt, dt_off, pair_off, n_pair, overlaps);
  return check_cuda(cudaGetLastError(), "kitti_eval_overlaps");
}

int mf_kitti_eval_statistics(const double* gt, const int* gt_off, const double* dt, const int* dt_off,
                             const long long* pair_off, int n_img, int n_gt, int n_dt, int max_dt, const double* overlaps,
                             long long n_pair, const int* classes, int ncls, void* workspace, size_t ws_bytes,
                             void* stream) {
  if (n_img < 1 || n_gt < 0 || n_dt < 0) { set_error("mf_kitti_eval_statistics: %d images", n_img); return -1; }
  if (ncls < 1 || ncls > MAX_CLS) { set_error("mf_kitti_eval_statistics: %d classes (1..%d)", ncls, MAX_CLS); return -1; }
  if (max_dt > MAX_DT) {
    set_error("mf_kitti_eval_statistics: an image has %d detections, more than the %d per image this kernel matches",
              max_dt, MAX_DT);
    return -1;
  }
  const Layout L = layout(n_gt, n_dt, ncls);
  if (workspace == nullptr || ws_bytes < L.total) {
    set_error("mf_kitti_eval_statistics: workspace of %zu bytes, %zu needed", ws_bytes, L.total);
    return -1;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  char* ws = static_cast<char*>(workspace);
  StatArgs a;
  a.gt = gt; a.gt_off = gt_off; a.dt = dt; a.dt_off = dt_off; a.pair_off = pair_off; a.ov = overlaps;
  a.n_img = n_img; a.n_gt = n_gt; a.n_dt = n_dt; a.ncls = ncls; a.n_pair = n_pair;
  for (int m = 0; m < MAX_CLS; ++m) {
    a.cls.c[m] = m < ncls ? classes[m] : -1;
    if (m < ncls && (classes[m] < 0 || classes[m] > 5)) {
      set_error("mf_kitti_eval_statistics: class %d is not one of 0..5", classes[m]);
      return -1;
    }
  }
  a.fg = reinterpret_cast<signed char*>(ws + L.fg); a.fd = reinterpret_cast<signed char*>(ws + L.fd);
  a.seg = reinterpret_cast<int*>(ws + L.seg);
  a.tps = reinterpret_cast<double*>(ws + L.tps); a.tps_sorted = reinterpret_cast<double*>(ws + L.tps_sorted);
  a.thr = reinterpret_cast<double*>(ws + L.thr); a.nthr = reinterpret_cast<int*>(ws + L.nthr);
  a.pr = reinterpret_cast<double*>(ws + L.pr); a.aos = reinterpret_cast<int*>(ws + L.aos);
  const int C = 18 * ncls;
  const long long nflag = static_cast<long long>(n_gt) + n_dt + C + 1;
  flags_kernel<<<static_cast<unsigned>((nflag + 255) / 256), 256, 0, st>>>(a);
  if (check_cuda(cudaGetLastError(), "kitti_eval_flags")) return -1;
  const long long npass = static_cast<long long>(C) * n_img;
  first_pass_kernel<<<static_cast<unsigned>((npass + 127) / 128), 128, 0, st>>>(a);
  if (check_cuda(cudaGetLastError(), "kitti_eval_first_pass")) return -1;
  if (n_gt > 0) {
    size_t bytes = L.cub_bytes;
    if (check_cuda(cub::DeviceSegmentedRadixSort::SortKeysDescending(ws + L.cub, bytes, a.tps, a.tps_sorted, C * n_gt, C,
                                                                      a.seg, a.seg + 1, 0, 64, st),
                   "kitti_eval_sort"))
      return -1;
  }
  thresholds_kernel<<<C, THR_THREADS, 0, st>>>(a);
  if (check_cuda(cudaGetLastError(), "kitti_eval_thresholds")) return -1;
  second_pass_kernel<<<C * NPTS, STAT_THREADS, 0, st>>>(a);
  return check_cuda(cudaGetLastError(), "kitti_eval_second_pass");
}

int mf_kitti_eval_ap(const void* workspace, int n_gt, int n_dt, int ncls, double* out, void* stream) {
  if (ncls < 1 || ncls > MAX_CLS || workspace == nullptr) { set_error("mf_kitti_eval_ap: %d classes", ncls); return -1; }
  const Layout L = layout(n_gt, n_dt, ncls);
  const char* ws = static_cast<const char*>(workspace);
  ap_kernel<<<1, 18 * ncls, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const double*>(ws + L.pr),
                                                                      reinterpret_cast<const int*>(ws + L.nthr),
                                                                      reinterpret_cast<const int*>(ws + L.aos), ncls, out);
  return check_cuda(cudaGetLastError(), "kitti_eval_ap");
}

}  // extern "C"
