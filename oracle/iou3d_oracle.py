"""TEST INFRASTRUCTURE ONLY — CPU restatement of the reference's get_iou_3d (model/layers/iou_loss.py:99-136) and of the
'3D_IoU' log of Loss_Computation (model/head/detector_loss.py:333), pinned to tests/golden/iou3d.npz
(oracle/make_golden_iou3d.py).

`ExactPolygon` stands in for shapely.geometry.Polygon (not installable here) where get_iou_3d uses it: `is_valid`, `area` and
`.intersection(other).area`. It computes them EXACTLY with fractions.Fraction on the float64 values of the coordinates and
rounds once to float64, the value GEOS approximates to about 1e-16 relative. Validity follows csrc/mf_iou3d.cuh: the ring's
turn cross products are all non-zero with one sign (convex, simple, no repeated corner). Shapely also accepts simple
non-convex rings; encode_box3d never builds one (DESIGN.md §9). Non-finite coordinates give is_valid False and a NaN area,
as in GEOS."""
from fractions import Fraction
import math

import numpy as np
import torch


def _cross(ox, oz, ax, az, bx, bz):
    return (ax - ox) * (bz - oz) - (az - oz) * (bx - ox)


class ExactPolygon(object):
    def __init__(self, shell=None, _exact=None):
        if _exact is not None:                                       # an intersection result: exact rational vertices
            self._finite, self._v = True, _exact
            return
        c = np.asarray(shell, dtype=np.float64).reshape(-1, 2)
        self._finite = bool(np.isfinite(c).all())
        self._v = [(Fraction(float(x)), Fraction(float(z))) for x, z in c] if self._finite else None

    def _signed2(self):
        v, s = self._v, Fraction(0)
        for k in range(len(v)):
            (x0, z0), (x1, z1) = v[k], v[(k + 1) % len(v)]
            s += x0 * z1 - z0 * x1
        return s

    def _turns(self):
        v, n = self._v, len(self._v)
        return [_cross(*v[k - 1], *v[k], *v[(k + 1) % n]) for k in range(n)]

    @property
    def is_valid(self):
        if not self._finite or len(self._v) < 3:
            return False
        t = self._turns()
        return all(c > 0 for c in t) or all(c < 0 for c in t)

    @property
    def area(self):
        if not self._finite:
            return math.nan
        return float(abs(self._signed2()) / 2)

    def _ccw(self):
        return self._v if self._signed2() > 0 else self._v[::-1]

    def intersection(self, other):
        """exact Sutherland-Hodgman clip of two valid (convex) rings"""
        if not (self.is_valid and other.is_valid):
            raise ValueError("ExactPolygon.intersection is only defined for two valid rings")
        poly, clip = self._ccw(), other._ccw()
        for j in range(len(clip)):
            (ox, oz), (ex, ez) = clip[j], clip[(j + 1) % len(clip)]
            d = [_cross(ox, oz, ex, ez, x, z) for x, z in poly]
            out = []
            for k in range(len(poly)):
                s, e, ds, de = poly[k - 1], poly[k], d[k - 1], d[k]
                if (de >= 0) != (ds >= 0):
                    t = ds / (ds - de)
                    out.append((s[0] + t * (e[0] - s[0]), s[1] + t * (e[1] - s[1])))
                if de >= 0:
                    out.append(e)
            poly = out
            if len(poly) < 3:
                return ExactPolygon(_exact=[])
        return ExactPolygon(_exact=poly)

    @property
    def vertex_count(self):
        """distinct corners of the ring: repeated points and points on a straight run are not counted"""
        v = []
        for p in self._v:
            if not v or p != v[-1]:
                v.append(p)
        while len(v) > 1 and v[0] == v[-1]:
            v.pop()
        changed = True
        while changed and len(v) >= 3:
            changed = False
            for k in range(len(v)):
                if _cross(*v[k - 1], *v[k], *v[(k + 1) % len(v)]) == 0:
                    del v[k]
                    changed = True
                    break
        return len(v) if len(v) >= 3 else 0


def _heights(C):
    y = C[:, :, 1]
    lo = -(((y[:, 0] + y[:, 1]) + y[:, 2]) + y[:, 3]) / np.float32(4.0)     # torch's CPU sum over 4: left to right
    hi = -(((y[:, 4] + y[:, 5]) + y[:, 6]) + y[:, 7]) / np.float32(4.0)
    return lo, hi


def get_iou_3d(pred_corners, target_corners, polygon=ExactPolygon):
    """float32-faithful get_iou_3d: [N, 8, 3] corners (numpy or torch) -> [N] float32 numpy."""
    A = np.asarray(torch.as_tensor(pred_corners).detach().cpu(), dtype=np.float32)
    B = np.asarray(torch.as_tensor(target_corners).detach().cpu(), dtype=np.float32)
    N = A.shape[0]
    iou3d = np.zeros(N, np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        min_h_a, max_h_a = _heights(A)
        min_h_b, max_h_b = _heights(B)
        h_overlap = np.maximum(np.float32(0), np.minimum(max_h_a, max_h_b) - np.maximum(min_h_a, min_h_b))
        for i in range(N):
            bottom_a, bottom_b = polygon(A[i, 0:4][:, [0, 2]]), polygon(B[i, 0:4][:, [0, 2]])
            if bottom_a.is_valid and bottom_b.is_valid:
                bottom_overlap = bottom_a.intersection(bottom_b).area
            else:
                bottom_overlap = 0.0
            overlap3d = np.float32(bottom_overlap) * h_overlap[i]
            union3d = (np.float32(bottom_a.area) * (max_h_a[i] - min_h_a[i]) + np.float32(bottom_b.area) * (max_h_b[i] - min_h_b[i])
                       - overlap3d)
            iou3d[i] = overlap3d / union3d
    return iou3d


def loss_iou3d(pred_cls, pred_reg, fields, calibs_P):
    """the '3D_IoU' log of Loss_Computation (detector_loss.py:333) from the oracle's own corners: the label and predicted
    corners monoflex_oracle.loss_computation builds for corner_loss. Returns (mean as a float32 scalar, per-object IoUs)."""
    from oracle import monoflex_oracle as mo
    seen = []
    build = mo.encode_box3d

    def record(*args):
        c = build(*args)
        seen.append(c.detach())
        return c

    mo.encode_box3d = record
    try:
        with torch.no_grad():
            mo.loss_computation(pred_cls, pred_reg, fields, calibs_P)
    finally:
        mo.encode_box3d = build
    t_corners, p_corners = seen                                      # built in this order by loss_computation
    iou = get_iou_3d(p_corners, t_corners)
    return np.float32(torch.from_numpy(iou).mean().item()), iou
