// 3D IoU of two boxes given by their 8 corners: get_iou_3d model/layers/iou_loss.py:99-136, one box pair per call.
// Shared by the standalone op (mf_iou3d.cu) and the '3D_IoU' log of the fused loss (mf_loss.cu).
//
// Corners are [8][3] float32 in encode_box3d's order (anno_encoder.py:88-122): 0-3 the bottom face (y = +h/2, y points
// down), 4-7 the top face. The reference takes
//   * the height extents in float32: min_h = -sum(y of corners 0-3) / 4 (torch's CPU sum: left to right), max_h likewise
//     from corners 4-7, h_overlap = max(0, min(max_h) - max(min_h));
//   * the BEV rings Polygon(corners[0:4, [x, z]]) and, when both are is_valid, the area of their intersection (GEOS, float64);
//   * overlap3d = f32(area_ab) * h_overlap and union3d = f32(area_a) * (max_h_a - min_h_a) + f32(area_b) * (...) - overlap3d,
//     float32 in this order (a Python float times a 0-dim float32 tensor is rounded to float32 first), iou = overlap / union.
// Here the intersection is one Sutherland-Hodgman clip of the two convex quadrilaterals in float64 (at most 8 vertices, 16
// slots, every loop bounded) followed by the shoelace area; the float32 steps use explicit round-to-nearest operations so
// that no FMA contraction changes them.
//
// Validity: a ring counts as is_valid when its four turn cross products are all non-zero with one sign. That rejects what
// GEOS rejects for encode_box3d's rings: zero-size and collapsed boxes (repeated corners) and self-intersecting (bow-tie)
// rings. Deviation: a simple but NON-convex quadrilateral is invalid here, while shapely accepts it; encode_box3d only builds
// rectangles, so it never produces one. NaN corners give NaN, as in the reference (the area and the height extent are NaN,
// so are the union and the IoU).
#pragma once
#include <cuda_runtime.h>

namespace mf {

namespace iou3d {

constexpr int kMaxVerts = 16;   // a convex quad clipped by 4 half-planes has <= 8 vertices; the rest is headroom

// exact-zero cross product: no FMA, so a x b - b x a is exactly 0 for a vertex on its own edge
__device__ __forceinline__ double cross(double ax, double az, double bx, double bz) {
  return __dsub_rn(__dmul_rn(ax, bz), __dmul_rn(az, bx));
}

// the four turns of the ring share one strict sign; returns +1 (counter-clockwise in (x, z)), -1 (clockwise) or 0 (invalid,
// also for NaN, where every comparison is false)
__device__ __forceinline__ int ring_orientation(const double* x, const double* z) {
  int pos = 0, neg = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int km = (k + 3) & 3, kp = (k + 1) & 3;
    const double c = cross(x[k] - x[km], z[k] - z[km], x[kp] - x[k], z[kp] - z[k]);
    pos += c > 0.0;
    neg += c < 0.0;
  }
  return pos == 4 ? 1 : (neg == 4 ? -1 : 0);
}

// twice the signed shoelace area
__device__ __forceinline__ double shoelace2(const double* x, const double* z, int n) {
  double s = 0.0;
  for (int k = 0; k < n; ++k) {
    const int kp = k + 1 == n ? 0 : k + 1;
    s += cross(x[k], z[k], x[kp], z[kp]);
  }
  return s;
}

// area of the intersection of two valid (convex) rings, each given counter-clockwise
__device__ __forceinline__ double clip_area(const double* ax, const double* az, const double* bx, const double* bz) {
  double px[kMaxVerts], pz[kMaxVerts], qx[kMaxVerts], qz[kMaxVerts];
  int n = 4;
#pragma unroll
  for (int k = 0; k < 4; ++k) { px[k] = ax[k]; pz[k] = az[k]; }
#pragma unroll 1
  for (int j = 0; j < 4; ++j) {                                     // keep the left side of the clip edge b[j] -> b[j+1]
    const double ox = bx[j], oz = bz[j], ex = bx[(j + 1) & 3] - ox, ez = bz[(j + 1) & 3] - oz;
    int m = 0;
    double sx = px[n - 1], sz = pz[n - 1];
    double ds = cross(ex, ez, sx - ox, sz - oz);
#pragma unroll 1
    for (int k = 0; k < n; ++k) {
      const double cx = px[k], cz = pz[k];
      const double dc = cross(ex, ez, cx - ox, cz - oz);
      if ((dc >= 0.0) != (ds >= 0.0) && m < kMaxVerts) {            // the edge crosses the line: t in [0, 1], so the point
        const double t = ds / (ds - dc);                            // stays on the segment even for near-parallel edges
        qx[m] = sx + t * (cx - sx);
        qz[m] = sz + t * (cz - sz);
        ++m;
      }
      if (dc >= 0.0 && m < kMaxVerts) { qx[m] = cx; qz[m] = cz; ++m; }
      sx = cx; sz = cz; ds = dc;
    }
    n = m;
    if (n < 3) return 0.0;
#pragma unroll 1
    for (int k = 0; k < n; ++k) { px[k] = qx[k]; pz[k] = qz[k]; }
  }
  return 0.5 * fabs(shoelace2(px, pz, n));
}

__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fffffff) : fmaxf(a, b); }
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? __int_as_float(0x7fffffff) : fminf(a, b); }

}  // namespace iou3d

// a, b: the two boxes' corners, [8][3] float32 each (x, y, z per corner); returns the reference's float32 IoU
__device__ __forceinline__ float iou3d_corners(const float* a, const float* b) {
  using namespace iou3d;
  // heights (float32, left-to-right sums like torch's CPU reduction over 4 elements)
  const float min_h_a = __fdiv_rn(-__fadd_rn(__fadd_rn(__fadd_rn(a[1], a[4]), a[7]), a[10]), 4.f);
  const float max_h_a = __fdiv_rn(-__fadd_rn(__fadd_rn(__fadd_rn(a[13], a[16]), a[19]), a[22]), 4.f);
  const float min_h_b = __fdiv_rn(-__fadd_rn(__fadd_rn(__fadd_rn(b[1], b[4]), b[7]), b[10]), 4.f);
  const float max_h_b = __fdiv_rn(-__fadd_rn(__fadd_rn(__fadd_rn(b[13], b[16]), b[19]), b[22]), 4.f);
  const float h_overlap = nan_max(0.f, __fsub_rn(nan_min(max_h_a, max_h_b), nan_max(min_h_a, min_h_b)));
  // BEV rings in float64, moved to b's first corner (float differences are exact in float64), so the shoelace does not
  // cancel large coordinates
  const double ox = b[0], oz = b[2];
  double ax[4], az[4], bx[4], bz[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    ax[k] = static_cast<double>(a[3 * k]) - ox; az[k] = static_cast<double>(a[3 * k + 2]) - oz;
    bx[k] = static_cast<double>(b[3 * k]) - ox; bz[k] = static_cast<double>(b[3 * k + 2]) - oz;
  }
  const double area_a = 0.5 * fabs(shoelace2(ax, az, 4)), area_b = 0.5 * fabs(shoelace2(bx, bz, 4));
  const int oa = ring_orientation(ax, az), ob = ring_orientation(bx, bz);
  double overlap = 0.0;
  if (oa != 0 && ob != 0) {
    if (oa < 0) { double t = ax[1]; ax[1] = ax[3]; ax[3] = t; t = az[1]; az[1] = az[3]; az[3] = t; }   // both counter-
    if (ob < 0) { double t = bx[1]; bx[1] = bx[3]; bx[3] = t; t = bz[1]; bz[1] = bz[3]; bz[3] = t; }   // clockwise
    overlap = clip_area(ax, az, bx, bz);
  }
  const float overlap3d = __fmul_rn(static_cast<float>(overlap), h_overlap);
  const float union3d = __fsub_rn(__fadd_rn(__fmul_rn(static_cast<float>(area_a), __fsub_rn(max_h_a, min_h_a)),
                                            __fmul_rn(static_cast<float>(area_b), __fsub_rn(max_h_b, min_h_b))),
                                  overlap3d);
  return __fdiv_rn(overlap3d, union3d);
}

}  // namespace mf
