"""Generates tests/golden/kitti_targets.npz by running the UNMODIFIED reference KITTIDataset (/root/reference,
data/datasets/kitti.py with runs/monoflex.yaml, through oracle/ref_shims) on a throwaway KITTI-layout directory of
seeded labels: ImageSets, zero PNGs of KITTI sizes, label_2 and calib (P0-P3, R0_rect, Tr_velo_to_cam, Tr_imu_to_velo).
random.random is patched so that both branches of the horizontal flip occur. The labels cover every branch of the
encoding: projections inside and partly outside the image (label-box fallback), projected centres beyond each of the four
borders, objects behind the camera, the truncation / size filter, Van / DontCare / Misc rows, slot holes, pred_2D = False,
empty 2D boxes, key points partly outside, ry near +-pi, alphas at the multi-bin margins, an empty image and an image
with 40 objects. Objects on which the reference raises are not written (the oracle finds them first).

Run in the build container (needs /root/reference):  python oracle/make_golden_targets.py"""
import math
import os
import sys
import tempfile
from unittest import mock

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
from oracle import target_oracle as to  # noqa: E402
from monoflex_b200 import targets as tg  # noqa: E402

SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370), (1234, 376), (1242, 374)]
DIMS = {"Car": (1.53, 1.63, 3.88), "Pedestrian": (1.76, 0.66, 0.84), "Cyclist": (1.74, 0.60, 1.76),
        "Van": (2.2, 1.9, 5.1), "Misc": (1.5, 1.2, 2.0)}
N_TRAIN, N_TEST = 26, 6


def calib_text(P2):
    P0 = P2.copy()
    P0[:, 3] = 0
    P3 = P2.copy()
    P3[0, 3] = -339.5
    R0 = np.array([[0.9999239, 0.00983776, -0.007445048], [-0.009869795, 0.9999421, -0.004278459],
                   [0.007402527, 0.004351614, 0.9999631]])
    V2C = np.array([[7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03],
                    [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
                    [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01]])
    I2V = np.array([[9.999976e-01, 7.553071e-04, -2.035826e-03, -8.086759e-01],
                    [-7.854027e-04, 9.998898e-01, -1.482298e-02, 3.195559e-01],
                    [2.024406e-03, 1.482454e-02, 9.998881e-01, -7.997231e-01]])
    f = lambda a: " ".join("%.12e" % v for v in np.asarray(a).ravel())
    return "P0: %s\nP1: %s\nP2: %s\nP3: %s\nR0_rect: %s\nTr_velo_to_cam: %s\nTr_imu_to_velo: %s\n" % (
        f(P0), f(P0), f(P2), f(P3), f(R0), f(V2C), f(I2V))


def make_P2(g, w, h):
    f = 721.5377 + g.uniform(-14, 14)
    return np.array([[f, 0, w / 2 - 11.5 + g.uniform(-3, 3), 44.85728 + g.uniform(-2, 2)],
                     [0, f, h / 2 - 14.6 + g.uniform(-3, 3), 0.2163791 + g.uniform(-0.1, 0.1)],
                     [0, 0, 1, 0.002745884]], dtype=np.float64)


def project_box(P, cls, t, ry, dims):
    h, w, l = dims
    c, s = math.cos(ry), math.sin(ry)
    xs = np.array([l / 2, l / 2, -l / 2, -l / 2] * 2)
    ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
    zs = np.array([w / 2, -w / 2, -w / 2, w / 2] * 2)
    X, Y, Z = c * xs + s * zs + t[0], ys + t[1], -s * xs + c * zs + t[2]
    p = np.stack([X, Y, Z, np.ones(8)], 1) @ P.T
    return p[:, 0] / p[:, 2], p[:, 1] / p[:, 2], Z


def line(cls, trunc, occ, box, dims, t, ry, fine=False):
    fmt = "%.6f" if fine else "%.2f"
    vals = [trunc, occ, -10.0] + list(box) + list(dims) + list(t) + [ry]
    s = "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f " % tuple([cls] + vals[:13])
    return s + (fmt % vals[13])


def random_object(g, P, w, h, kind):
    """one label line; kind picks the geometry (see the module docstring)."""
    cls = g.choice(["Car", "Car", "Car", "Pedestrian", "Cyclist"])
    dims = tuple(d * g.uniform(0.85, 1.15) for d in DIMS[cls])
    ry = g.uniform(-math.pi, math.pi)
    fine = False
    if kind == "inside":
        t = (g.uniform(-10, 10), g.uniform(1.4, 1.9), g.uniform(12, 60))
    elif kind in ("left", "right"):
        z = g.uniform(3.5, 9)
        sgn = -1 if kind == "left" else 1
        t = (sgn * z * g.uniform(0.85, 1.05), g.uniform(1.3, 1.9), z)
    elif kind == "top":
        z = g.uniform(3, 6)
        t = (g.uniform(-2, 2), -z * g.uniform(0.22, 0.35) + dims[0] / 2, z)
    elif kind == "bottom":
        z = g.uniform(2.2, 4)
        t = (g.uniform(-2, 2), z * g.uniform(0.36, 0.5) + dims[0] / 2, z)
    elif kind == "behind":
        t = (g.uniform(-5, 5), 1.6, g.uniform(-6, 0))
    elif kind == "pi":
        t = (g.uniform(-8, 8), 1.6, g.uniform(10, 40))
        ry = (math.pi - g.uniform(1e-5, 1e-3)) * (1 if g.uniform() < 0.5 else -1)
        fine = True
    elif kind == "margin":
        t = tuple(float("%.2f" % v) for v in (g.uniform(-8, 8), 1.6, g.uniform(10, 40)))
        a = g.choice([0, math.pi / 2, math.pi, -math.pi / 2]) + g.choice([-1, 1]) * (math.pi / 4 + math.pi / 12)
        a += g.choice([-1, 1]) * 1e-5
        ry = a + math.atan2(np.float32(t[0]), np.float32(t[2]))
        ry = (ry + math.pi) % (2 * math.pi) - math.pi
        fine = True
    else:
        raise ValueError(kind)
    t = tuple(float("%.2f" % v) for v in t)
    u, v, _ = project_box(P, cls, t, float(fine and ry or "%.2f" % ry), dims)
    box = [max(u.min(), 0), max(v.min(), 0), min(u.max(), w - 1), min(v.max(), h - 1)]
    box = [b + g.uniform(-1.5, 1.5) for b in box]
    trunc = 0.0 if kind == "inside" else g.uniform(0, 0.85)
    return line(cls, trunc, int(g.integers(0, 4)), box, dims, t, ry, fine)


def special_objects(g, P, w, h):
    """rows for the branches random sampling rarely reaches"""
    out = []
    # truncation filter: truncated and small -> dropped
    out.append(line("Car", 0.95, 2, (1180.0, 160.0, 1195.0, 180.0), DIMS["Car"], (22.0, 1.6, 30.0), 0.3))
    # truncated but large -> kept
    out.append(line("Car", 0.92, 1, (0.0, 150.0, 200.0, 300.0), DIMS["Car"], (-6.8, 1.6, 6.0), 1.4))
    # pred_2D = False: partly outside (label box), the centre lands outside a wrong label box
    out.append(line("Car", 0.3, 0, (0.0, 170.0, 25.0, 230.0), DIMS["Car"], (-6.0, 1.7, 11.0), -1.2))
    # empty label box on the label-box branch
    out.append(line("Cyclist", 0.2, 0, (0.0, 160.0, 0.0, 260.0), DIMS["Cyclist"], (-4.6, 1.7, 5.0), 0.5))
    # rows of other classes: never take a slot
    for cls in ("Van", "DontCare", "Misc", "Truck", "Person_sitting", "Tram"):
        out.append(line(cls, 0.0, 0, (500.0, 170.0, 560.0, 210.0), DIMS.get(cls, (1.5, 1.6, 3.9)), (1.0, 1.6, 25.0), 0.1))
    return out


def image_labels(g, P, w, h, b):
    if b == 3:
        return []                                                          # an empty image
    if b == 5:
        n = 40                                                             # a crowded image (plus rows of other classes)
        rows = [random_object(g, P, w, h, g.choice(["inside"] * 5 + ["left", "right", "behind"])) for _ in range(n + 14)]
        rows += [line("DontCare", -1, -1, (10.0, 10.0, 40.0, 40.0), (-1, -1, -1), (-1000, -1000, -1000), -10)] * 3
        return rows
    kinds = ["inside"] * int(g.integers(2, 9)) + ["left", "right", "top", "bottom", "behind", "pi", "margin"]
    if b % 2 == 0:
        kinds += ["margin", "margin", "pi"]
    rows = [random_object(g, P, w, h, k) for k in kinds]
    g.shuffle(rows)
    if b % 3 == 0:
        rows += special_objects(g, P, w, h)
    return rows


def keep_encodable(lines, P2, size, flip, max_objs=40):
    """drop, one at a time, rows the reference would raise on (the oracle's status), and rows beyond max_objs"""
    lines = list(lines)
    while True:
        rows = tg.read_kitti_label(lines)
        bad = None
        for n in range(1, rows.shape[0] + 1):
            if to.encode_image(rows[:n], P2, size, flip, max_objs=max(n, max_objs))[1]:
                bad = n - 1
                break
        kept = [i for i, l in enumerate(lines) if l.split(" ")[0] in tg.CLASSES]
        if bad is None:
            return [l for i, l in enumerate(lines) if i not in kept[max_objs:]]
        lines = [l for i, l in enumerate(lines) if i != kept[bad]]


def main():
    g = np.random.default_rng(20261015)
    if not os.path.exists(ref_shims._REF_SO):               # the DCN op is never called here
        ref_shims._load_ref_so = lambda: None
    cfg = ref_shims.reference_cfg()
    from data.datasets.kitti import KITTIDataset
    from PIL import Image
    fields = ["cls_ids", "target_centers", "keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_mask",
              "reg_weight", "offset_3D", "2d_bboxes", "pad_size", "rotys", "trunc_mask", "alphas", "orientations", "hm",
              "gt_bboxes", "occlusions", "truncations", "edge_len", "edge_indices"]
    out = {}
    with tempfile.TemporaryDirectory() as root:
        for d in ("ImageSets", "image_2", "label_2", "calib"):
            os.makedirs(os.path.join(root, d))
        ids = ["%06d" % i for i in range(N_TRAIN + N_TEST)]
        sizes = [SIZES[int(g.integers(0, len(SIZES)))] for _ in ids]
        P2s = [make_P2(g, w, h) for (w, h) in sizes]
        flips = [bool(b % 2) if b < 4 else bool(g.integers(0, 2)) for b in range(N_TRAIN)]
        labels = []
        for b, i in enumerate(ids):
            w, h = sizes[b]
            Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(os.path.join(root, "image_2", i + ".png"))
            with open(os.path.join(root, "calib", i + ".txt"), "w") as f:
                f.write(calib_text(P2s[b]))
            lines = []
            if b < N_TRAIN:
                lines = keep_encodable(image_labels(g, P2s[b], w, h, b), P2s[b], (w, h), flips[b])
            labels.append(lines)
            with open(os.path.join(root, "label_2", i + ".txt"), "w") as f:
                f.write("".join(l + "\n" for l in lines))
        with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
            f.write("".join(i + "\n" for i in ids[:N_TRAIN]))
        with open(os.path.join(root, "ImageSets", "test.txt"), "w") as f:
            f.write("".join(i + "\n" for i in ids[N_TRAIN:]))

        ds = KITTIDataset(cfg, root, is_train=True)
        rec = {k: [] for k in fields + ["P2_flipped"]}
        for b in range(N_TRAIN):
            with mock.patch("random.random", return_value=0.0 if flips[b] else 0.9):
                _, target, _ = ds[b]
            for k in fields:
                rec[k].append(np.asarray(target.get_field(k)))
            rec["P2_flipped"].append(np.asarray(target.get_field("calib").P))
        # the reference's Object3d values after filtrate_objects, before the flip: what read_kitti_label must return
        rows =[np.array([[float(tg.CLASSES.index(o.type)), o.truncation, float(o.occlusion), o.xmin, o.ymin, o.xmax, o.ymax,
                           o.h, o.w, o.l] + [float(v) for v in o.t] + [o.ry]
                          for o in ds.filtrate_objects(ds.get_label_objects(b))], dtype=np.float64).reshape(-1, 14)
                for b in range(N_TRAIN)]
        out["rows_packed"] = tg.pack_labels(rows, 40)
        for k, v in rec.items():
            out["train_" + k] = np.stack(v)
        out["train_labels"] = np.array(["\n".join(l) for l in labels[:N_TRAIN]])
        out["train_P2"] = np.stack([ds.get_calibration(b).P for b in range(N_TRAIN)])     # as parsed from the text
        out["train_calib_text"] = np.array([calib_text(P) for P in P2s[:N_TRAIN]])
        out["train_sizes"] = np.array(sizes[:N_TRAIN], dtype=np.int64)
        out["train_flips"] = np.array(flips, dtype=np.int64)

        # the test split (kitti.py:287-299): the reference reaches it only for a split named 'test', whose (absent) labels it
        # still filters; an empty list stands in for them
        ds_t = KITTIDataset(cfg, root, is_train=False)
        with mock.patch.object(KITTIDataset, "filtrate_objects", lambda self, objs: [] if objs is None else objs):
            tt = [ds_t[b][1] for b in range(N_TEST)]
        out["test_P2"] = np.stack([ds_t.get_calibration(b).P for b in range(N_TEST)])
        out["test_sizes"] = np.array(sizes[N_TRAIN:], dtype=np.int64)
        for k in ("pad_size", "edge_len", "edge_indices"):
            out["test_" + k] = np.stack([np.asarray(t.get_field(k)) for t in tt])
        out["test_P2_calib"] = np.stack([np.asarray(t.get_field("calib").P) for t in tt])
    for k in sorted(out):
        print(k, out[k].shape, out[k].dtype)
    counts = out["train_reg_mask"].sum(1)
    print("objects per image", counts.tolist(), "flips", out["train_flips"].tolist())
    print("trunc_mask", int(out["train_trunc_mask"].sum()), "pred_2D False",
          int(((out["train_2d_bboxes"] == 0).all(-1) & (out["train_reg_mask"] == 1)).sum()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "kitti_targets.npz"), **out)


if __name__ == "__main__":
    main()
