"""TEST TOOLING — tests/golden/iou3d.npz: the UNMODIFIED reference get_iou_3d (model/layers/iou_loss.py:99-136) with
shapely.geometry.Polygon provided by oracle.iou3d_oracle.ExactPolygon through oracle/ref_shims.py's module mocks (shapely is
not installed here). Build container only:  python -m oracle.make_golden_iou3d

(a) seeded box pairs whose corners come from the reference's own Anno_Encoder.encode_box3d: disjoint pairs, pairs without
    height overlap, containment, identical boxes, boxes turned by pi and pi/2, partial overlaps whose intersection has each
    vertex count from 3 to 8, pairs touching at an edge or a corner, nearly parallel edges, a zero-size box and a NaN box.
    Sizes stay >= 1 mm, so float32 rounding cannot fold a ring.
(b) the unmodified Loss_Computation on the inputs of tests/golden/loss_4x96x320.npz (monoflex_b200/synthetic.py, batch 4,
    seeds of oracle/make_golden_loss.py): its '3D_IoU' log, the per-object IoUs and the corners they were computed from."""
import math
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims as rs                # noqa: E402
from oracle.iou3d_oracle import ExactPolygon      # noqa: E402
from oracle.make_golden_loss import ref_train_targets  # noqa: E402
from monoflex_b200 import synthetic as syn        # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
CASES = ["disjoint", "no_height_overlap", "contains", "identical", "rot_pi", "rot_half_pi", "partial", "edge_touch",
         "corner_touch", "near_parallel", "zero_size", "nan"]


def reference():
    cfg = rs.reference_cfg()
    sys.modules["shapely.geometry"].Polygon = ExactPolygon
    import model.layers.iou_loss as il
    il.Polygon = ExactPolygon                    # bound by `from shapely.geometry import Polygon` at import time
    from model.anno_encoder import Anno_Encoder
    return cfg, il, Anno_Encoder(cfg)


def encode(enc, boxes):
    """boxes: rows (ry, l, h, w, x, y, z) -> [N, 8, 3] float32 corners from the reference's encode_box3d"""
    b = torch.tensor(np.asarray(boxes, np.float64), dtype=torch.float32)
    return enc.encode_box3d(b[:, 0].contiguous(), b[:, 1:4].contiguous(), b[:, 4:7].contiguous()).contiguous()


def bev_vertices(a, b):
    """vertex count of the exact BEV intersection of two corner sets (0 when empty or a ring is invalid)"""
    pa, pb = ExactPolygon(a[0:4][:, [0, 2]]), ExactPolygon(b[0:4][:, [0, 2]])
    if not (pa.is_valid and pb.is_valid):
        return 0
    return pa.intersection(pb).vertex_count


def make_pairs(enc, rng):
    A, B, case = [], [], []

    def add(name, a, b):
        A.append(a)
        B.append(b)
        case.append(name)

    def rand_box(x=0.0, z=20.0):
        return [rng.uniform(-math.pi, math.pi), rng.uniform(1.0, 5.0), rng.uniform(0.8, 2.5), rng.uniform(0.5, 2.5),
                x + rng.uniform(-10, 10), rng.uniform(0.5, 2.0), z + rng.uniform(-10, 30)]

    for _ in range(16):                                              # BEV far apart
        a = rand_box()
        b = rand_box()
        b[4], b[6] = a[4] + rng.choice([-1, 1]) * rng.uniform(7, 20), a[6] + rng.uniform(-20, 20)
        add("disjoint", a, b)
    for _ in range(10):                                              # overlapping footprint, stacked in height
        a = rand_box()
        b = list(a)
        b[0] += rng.uniform(-0.5, 0.5)
        b[5] = a[5] + rng.choice([-1, 1]) * ((a[2] + b[2]) / 2 + rng.uniform(0.01, 1.0))
        add("no_height_overlap", a, b)
    for k in range(16):                                              # one box inside the other (both ways)
        a = rand_box()
        b = list(a)
        b[1], b[2], b[3] = a[1] * rng.uniform(0.2, 0.5), a[2] * rng.uniform(0.3, 0.9), a[3] * rng.uniform(0.2, 0.4)
        b[0] = a[0] + rng.choice([0.0, rng.uniform(-0.1, 0.1)])
        add("contains", a, b) if k % 2 == 0 else add("contains", b, a)
    for _ in range(8):
        a = rand_box()
        add("identical", a, list(a))
    for _ in range(8):
        a = rand_box()
        b = list(a)
        b[0] = a[0] + math.pi
        add("rot_pi", a, b)
    for k in range(8):
        a = rand_box()
        if k < 3:
            a[3] = a[1]                                              # square footprint: the turned box covers the same area
        b = list(a)
        b[0] = a[0] + math.pi / 2
        add("rot_half_pi", a, b)
    # partial overlaps: sample until every vertex count 3..8 of the exact intersection has its quota
    quota = {n: 10 for n in range(3, 9)}
    while any(quota.values()):
        cand = []
        for _ in range(400):
            a = rand_box()
            b = rand_box()
            if rng.uniform() < 0.35:                                 # similar boxes around one centre: 7 and 8 vertices
                b[1:4] = [a[1] * rng.uniform(0.8, 1.25), a[2], a[3] * rng.uniform(0.8, 1.25)]
                b[0] = a[0] + rng.uniform(0.3, 1.3)
                b[4], b[6] = a[4] + rng.uniform(-0.3, 0.3), a[6] + rng.uniform(-0.3, 0.3)
            else:
                r = (a[1] + b[1]) / 2
                b[4], b[6] = a[4] + rng.uniform(-r, r), a[6] + rng.uniform(-r, r)
            b[5] = a[5] + rng.uniform(-0.4, 0.4)
            cand.append((a, b))
        ca, cb = encode(enc, [c[0] for c in cand]).numpy(), encode(enc, [c[1] for c in cand]).numpy()
        for (a, b), x, y in zip(cand, ca, cb):
            n = bev_vertices(x, y)
            if n in quota and quota[n] > 0:
                quota[n] -= 1
                add("partial", a, b)
    # exact contact: axis-aligned (ry = 0 makes cos/sin exactly 1/0) with dyadic sizes and centres
    for k in range(6):
        l, w, h = [1.0, 2.5, 4.0][k % 3], [0.5, 1.5, 2.0][k % 3], 1.5
        x, z = -3.0 + k, 12.0 + 4 * k
        a = [0.0, l, h, w, x, 1.0, z]
        b = [0.0, l * 0.5, h, w * 2, x + l * 0.75, 1.25, z + 0.25] if k % 2 else [0.0, l, h, w, x, 1.25, z + w]
        add("edge_touch", a, b)
        add("corner_touch", a, [0.0, l, h, w * 0.5, x + l, 0.75, z + w * 0.75])
    for k in range(10):                                              # nearly parallel edges
        a = rand_box()
        b = list(a)
        b[0] = a[0] + [1e-7, -1e-7, 1e-6, -1e-6, 1e-5][k % 5]
        b[4] += [0.0, 0.3, 1e-4, 0.5, 0.0][k % 5] * math.cos(a[0])
        b[6] += [0.0, 0.3, 1e-4, 0.5, 1e-3][k % 5] * math.sin(a[0])
        if k >= 5:
            b[1] *= 1.0 + 1e-6
        add("near_parallel", a, b)
    a = rand_box()
    add("zero_size", [a[0], 0.0, 0.0, 0.0] + a[4:], rand_box())
    add("zero_size", a, [a[0], 0.0, 0.0, 0.0] + a[4:])
    add("zero_size", [0.3, 0.0, 0.0, 0.0, 1.0, 1.0, 10.0], [0.3, 0.0, 0.0, 0.0, 1.0, 1.0, 10.0])   # 0 / 0
    a = rand_box()
    add("nan", [a[0], a[1], a[2], a[3], float("nan"), a[5], a[6]], a)
    add("nan", a, [float("nan")] + a[1:])
    return encode(enc, A), encode(enc, B), np.array(case)


def loss_case(cfg, il):
    import model.head.detector_loss as dl
    per_object = []

    def recorded(a, b):
        per_object.append((a.detach().clone(), b.detach().clone()))
        return il.get_iou_3d(a, b)

    dl.get_iou_3d = recorded
    lc = dl.Loss_Computation(cfg)
    fields = syn.make_train_targets(4)
    cls, reg = syn.make_train_predictions(4, fields)
    with torch.no_grad():
        _, log = lc({"cls": cls, "reg": reg}, ref_train_targets(fields))
    (pc, tc), = per_object
    return log["3D_IoU"], pc, tc, il.get_iou_3d(pc, tc)


def main():
    cfg, il, enc = reference()
    rng = np.random.default_rng(20261016)
    A, B, case = make_pairs(enc, rng)
    iou = il.get_iou_3d(A, B)
    log, pc, tc, iou_obj = loss_case(cfg, il)
    out = dict(pred=A.numpy(), target=B.numpy(), iou=iou.numpy().astype(np.float32), case=case,
               loss_pred=pc.numpy(), loss_target=tc.numpy(), loss_iou=iou_obj.numpy().astype(np.float32),
               log_3D_IoU=np.float32(log))
    np.savez_compressed(os.path.join(OUT, "iou3d.npz"), **out)
    for c in CASES:
        v = out["iou"][case == c]
        print("%-18s %3d pairs  IoU %s .. %s" % (c, len(v), np.nanmin(v) if np.isfinite(v).any() else "nan",
                                                 np.nanmax(v) if np.isfinite(v).any() else "nan"))
    print("loss: %d objects, log 3D_IoU = %r" % (len(iou_obj), float(log)))


if __name__ == "__main__":
    main()
