"""Generates tests/golden/kitti_targets_right.npz by running the UNMODIFIED reference KITTIDataset
(data/datasets/kitti.py with runs/monoflex.yaml and DATASETS.USE_RIGHT_IMAGE = True, i.e. runs/monoflex_right.yaml, through
oracle/ref_shims) on a throwaway KITTI-layout directory: ImageSets, zero PNGs in image_2 AND image_3 (a right image may have
another size than its left one), label_2 and calib. The labels and calibration files come from the builders of
oracle/make_golden_targets.py; its calib_text writes a P3 whose baseline is b_x = 339.5 / f_u, about +0.47 m.

Both halves of the dataset are indexed (left items 0..N-1, right items N..2N-1), with random.random patched so that both
branches of the horizontal flip occur on left and on right items. Rows on which the reference raises in either view
(oracle/target_oracle_right.py finds them first) are not written. Right views move objects by about f * 0.53 / z px to the
left, so the left-border objects of the label builder reach the clamped and inverted boxes of kitti.py:246-247.

Run where the reference checkout is present:  python oracle/make_golden_targets_right.py"""
import os
import sys
import tempfile
from unittest import mock

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shims  # noqa: E402
from oracle import target_oracle_right as tor  # noqa: E402
from oracle.make_golden_targets import SIZES, DIMS, calib_text, image_labels, line, make_P2  # noqa: E402
from monoflex_b200 import targets as tg  # noqa: E402

N = 14
FIELDS = ["cls_ids", "target_centers", "keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_mask",
          "reg_weight", "offset_3D", "2d_bboxes", "pad_size", "rotys", "trunc_mask", "alphas", "orientations", "hm",
          "gt_bboxes", "occlusions", "truncations", "edge_len", "edge_indices"]


def left_border_objects(g):
    """objects the right camera sees wholly beyond the left border (a clamped, inverted box), truncated ones that the
    annotation filter then drops silently, and a near one across the right image's left border"""
    out = []
    for _ in range(2):
        z = g.uniform(4, 7)
        out.append(line("Pedestrian", 0.95, 1, (0.0, 160.0, 30.0, 250.0), DIMS["Pedestrian"], (-0.78 * z - 1.8, 1.6, z),
                        g.uniform(-3, 3)))
    out.append(line("Pedestrian", 0.5, 0, (0.0, 150.0, 60.0, 260.0), DIMS["Pedestrian"], (-3.8, 1.7, 4.5), 0.2))
    return out


def keep_encodable(lines, views, max_objs=40):
    """drop, one at a time, rows the reference would raise on in any of the views (P, size, flip, right), and rows beyond
    max_objs"""
    lines = list(lines)
    while True:
        rows = tg.read_kitti_label(lines)
        bad = None
        for n in range(1, rows.shape[0] + 1):
            if any(tor.encode_image(rows[:n], P, size, flip, right, max_objs=max(n, max_objs))[1]
                   for P, size, flip, right in views):
                bad = n - 1
                break
        kept = [i for i, l in enumerate(lines) if l.split(" ")[0] in tg.CLASSES]
        if bad is None:
            return [l for i, l in enumerate(lines) if i not in kept[max_objs:]]
        lines = [l for i, l in enumerate(lines) if i != kept[bad]]


def main():
    g = np.random.default_rng(20261016)
    if not os.path.exists(ref_shims._REF_SO):               # the DCN op is never called here
        ref_shims._load_ref_so = lambda: None
    cfg = ref_shims.reference_cfg()
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    from data.datasets.kitti import KITTIDataset
    from PIL import Image
    out = {}
    with tempfile.TemporaryDirectory() as root:
        for d in ("ImageSets", "image_2", "image_3", "label_2", "calib"):
            os.makedirs(os.path.join(root, d))
        ids = ["%06d" % i for i in range(N)]
        sizes_l = [SIZES[int(g.integers(0, len(SIZES)))] for _ in ids]
        # KITTI's rectified pairs share a size; every third frame gets another right size here
        sizes_r = [SIZES[int(g.integers(0, len(SIZES)))] if b % 3 == 1 else sizes_l[b] for b in range(N)]
        P2s = [make_P2(g, w, h) for (w, h) in sizes_l]
        P3s = []
        flips = [bool(b % 2) if b < 4 else bool(g.integers(0, 2)) for b in range(2 * N)]
        flips[N:N + 4] = [False, True, True, False]
        labels = []
        for b, i in enumerate(ids):
            w, h = sizes_l[b]
            Image.fromarray(np.zeros((h, w, 3), np.uint8)).save(os.path.join(root, "image_2", i + ".png"))
            wr, hr = sizes_r[b]
            Image.fromarray(np.zeros((hr, wr, 3), np.uint8)).save(os.path.join(root, "image_3", i + ".png"))
            text = calib_text(P2s[b])
            with open(os.path.join(root, "calib", i + ".txt"), "w") as f:
                f.write(text)
            P3 = np.array([float(x) for x in text.split("P3:")[1].split("\n")[0].split()]).reshape(3, 4)
            P3s.append(P3)
            lines = image_labels(g, P2s[b], w, h, b)
            if b % 2 == 0 and b != 4:
                lines += left_border_objects(g)
            views = [(P2s[b], (w, h), flips[b], False), (P3, (wr, hr), flips[N + b], True)]
            lines = keep_encodable(lines, views)
            labels.append(lines)
            with open(os.path.join(root, "label_2", i + ".txt"), "w") as f:
                f.write("".join(l + "\n" for l in lines))
        with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
            f.write("".join(i + "\n" for i in ids))

        ds = KITTIDataset(cfg, root, is_train=True)
        assert ds.num_samples == N and len(ds) == 2 * N
        rec = {k: [] for k in FIELDS + ["P2_flipped"]}
        for idx in range(2 * N):
            with mock.patch("random.random", return_value=0.0 if flips[idx] else 0.9):
                _, target, _ = ds[idx]
            for k in FIELDS:
                rec[k].append(np.asarray(target.get_field(k)))
            rec["P2_flipped"].append(np.asarray(target.get_field("calib").P))
        # the reference's Object3d values after filtrate_objects, before the flip (the left item's rows; a right item
        # overwrites only the box columns, on the device)
        rows = [np.array([[float(tg.CLASSES.index(o.type)), o.truncation, float(o.occlusion), o.xmin, o.ymin, o.xmax, o.ymax,
                           o.h, o.w, o.l] + [float(v) for v in o.t] + [o.ry]
                          for o in ds.filtrate_objects(ds.get_label_objects(b))], dtype=np.float64).reshape(-1, 14)
                for b in range(N)]
        packed = tg.pack_labels(rows, 40)
        out["rows_packed"] = np.concatenate([packed, packed])
        for k, v in rec.items():
            out[k] = np.stack(v)
        out["labels"] = np.array(["\n".join(l) for l in labels])
        out["P2_parsed"] = np.stack([ds.get_calibration(b).P for b in range(N)])
        out["P3_parsed"] = np.stack([ds.get_calibration(b, use_right_cam=True).P for b in range(N)])
        out["P"] = np.concatenate([out["P2_parsed"], out["P3_parsed"]])          # the matrix each item is encoded from
        out["calib_text"] = np.array([calib_text(P) for P in P2s])
        out["sizes"] = np.array(sizes_l + sizes_r, dtype=np.int64)
        out["flips"] = np.array(flips, dtype=np.int64)
        out["right"] = np.array([0] * N + [1] * N, dtype=np.int64)
        out["frame"] = np.array(list(range(N)) * 2, dtype=np.int64)
        out["num_samples"] = np.array(ds.num_samples, dtype=np.int64)
        out["dataset_len"] = np.array(len(ds), dtype=np.int64)
        assert np.array_equal(out["P3_parsed"], np.stack(P3s))
    for k in sorted(out):
        print(k, out[k].shape, out[k].dtype)
    reg = out["reg_mask"] == 1
    print("objects per item", reg.sum(1).tolist())
    print("flips", out["flips"].tolist())
    print("right trunc_mask", int(out["trunc_mask"][N:].sum()), "left trunc_mask", int(out["trunc_mask"][:N].sum()))
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "kitti_targets_right.npz"), **out)


if __name__ == "__main__":
    main()
