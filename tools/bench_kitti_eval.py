"""Time the KITTI official metric (monoflex_b200/evaluation.py) at KITTI-val size and check it on known answers.

    python tools/bench_kitti_eval.py [--images 3769] [--repeat 5] [--seed 0]

A seeded set of KITTI-like labels (3,769 images as in the val split, about 7 objects per image over Car / Van / Truck /
Pedestrian / Person_sitting / Cyclist / DontCare) and detections (perturbed copies plus false positives, up to 50 per
image, the decode's K) is written as text files to a temporary directory. Timed, median of --repeat runs after a warm-up:
from_label_dir (parse and upload, host clock ending in a synchronise), the overlaps / statistics / AP stages (CUDA events)
and the whole evaluate_python call (host clock; it ends in the copy of the result tables). Checked at that size:
detections equal to the ground truth (their 3D boxes turned by 0.01 rad, see below) give AP 100 wherever valid ground
truth exists, detections moved 100 m (and 5000 px)
away give 0 everywhere, and two runs are bit-identical. Prints one JSON line, with the card's name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200 import evaluation as E  # noqa: E402

NAMES = np.array(["Car", "Van", "Truck", "Pedestrian", "Person_sitting", "Cyclist", "DontCare"])
P_NAMES = np.array([0.55, 0.06, 0.02, 0.1, 0.01, 0.04, 0.22])
HWL = np.array([[1.5, 1.6, 3.9], [2.2, 1.9, 5.0], [3.2, 2.5, 10.0], [1.75, 0.65, 0.85], [1.3, 0.6, 0.8], [1.75, 0.6, 1.75],
                [-1, -1, -1]])


def make_labels(rng, n):
    k = rng.choice(len(NAMES), n, p=P_NAMES)
    hwl = HWL[k] * rng.uniform(0.85, 1.15, (n, 3))
    z = rng.uniform(4, 70, n)
    x, y = rng.uniform(-0.5, 0.5, n) * z, rng.uniform(1.4, 1.9, n)
    h2d = np.clip(720 * hwl[:, 0] / z, 12, 300)
    w2d = h2d * rng.uniform(0.4, 2.5, n)
    cx = 610 + 720 * x / z
    box = np.stack([cx - w2d / 2, 175 - h2d / 2, cx + w2d / 2, 175 + h2d / 2], 1)
    return dict(name=NAMES[k], trunc=rng.choice([0.0, 0.0, 0.1, 0.2, 0.4, 0.7], n), occ=rng.choice(4, n, p=(.5, .25, .2, .05)),
                alpha=rng.uniform(-np.pi, np.pi, n), box=box, hwl=hwl, loc=np.stack([x, y, z], 1),
                ry=rng.uniform(-np.pi, np.pi, n))


def gt_line(o, i):
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        o["name"][i], o["trunc"][i], o["occ"][i], o["alpha"][i], *o["box"][i], *o["hwl"][i], *o["loc"][i], o["ry"][i])


def dt_line(o, i, score):
    vals = np.round(np.array([o["alpha"][i], *o["box"][i], *o["hwl"][i], *o["loc"][i], o["ry"][i], score], np.float32), 4)
    name = {"Van": "Car", "Truck": "Car", "Person_sitting": "Pedestrian", "DontCare": "Car"}.get(o["name"][i], o["name"][i])
    return " ".join([name, "0", "0"] + [repr(v) for v in vals.tolist()])


def write_set(root, n_img, seed):
    rng = np.random.default_rng(seed)
    for d in ("label", "pred"):
        os.makedirs(os.path.join(root, d))
    n_obj = n_det = 0
    for i in range(n_img):
        n = int(rng.poisson(7.5))
        g = make_labels(rng, n)
        keep = [j for j in range(n) if g["name"][j] != "DontCare" and rng.random() < 0.85]
        n_fp = max(0, min(50 - len(keep), int(rng.integers(5, 45))))
        f = make_labels(rng, n_fp)
        for key in ("loc", "box"):
            g_copy = g[key][keep] + rng.normal(0, 0.03, g[key][keep].shape) * (1 if key == "loc" else 10)
            f[key] = np.concatenate([g_copy, f[key]])
        for key in ("name", "trunc", "occ", "alpha", "hwl", "ry"):
            f[key] = np.concatenate([g[key][keep], f[key]])
        scores = rng.uniform(0.01, 1.0, len(keep) + n_fp)
        with open(os.path.join(root, "label", "%06d.txt" % i), "w") as fh:
            fh.write("".join(gt_line(g, j) + "\n" for j in range(n)))
        with open(os.path.join(root, "pred", "%06d.txt" % i), "w") as fh:
            fh.write("".join(dt_line(f, j, scores[j]) + "\n" for j in range(len(scores))) or "\n")
        n_obj += n
        n_det += len(scores)
    with open(os.path.join(root, "split.txt"), "w") as fh:
        fh.write("".join("%d\n" % i for i in range(n_img)))
    return n_obj, n_det


def valid_gt_exists(gt, classes):
    """[ncls, 3]: clean_data's num_valid_gt > 0, restated on the host"""
    obj = gt.objects.cpu().numpy()
    h = obj[:, 7] - obj[:, 5]
    out = np.zeros((len(classes), 3), bool)
    for m, c in enumerate(classes):
        for l, (hmin, occ, trunc) in enumerate(((40, 0, 0.15), (25, 1, 0.3), (25, 2, 0.5))):
            out[m, l] = ((obj[:, 0] == c) & (obj[:, 2] <= occ) & (obj[:, 1] <= trunc) & (h > hmin)).any()
    return out


def median(xs):
    return float(np.median(xs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_kitti_eval needs a GPU"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    classes = [0, 1, 2]
    with tempfile.TemporaryDirectory() as root:
        n_obj, n_det = write_set(root, args.images, args.seed)
        label, pred, split = (os.path.join(root, p) for p in ("label", "pred", "split.txt"))
        E.evaluate_python(label, pred, split, classes, "R40")             # warm-up: module load, allocator
        t_parse, t_stage, t_all = [], [], []
        for _ in range(args.repeat):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            gt = E.KittiAnnos.from_label_dir(label, list(range(args.images)))
            dt = E.KittiAnnos.from_label_dir(pred)
            torch.cuda.synchronize()
            t_parse.append(time.perf_counter() - t0)
            ev = []
            tables, _ = E.eval_tables(gt, dt, classes, events=ev)
            t_stage.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            result, _ = E.evaluate_python(label, pred, split, classes, "R40")
            torch.cuda.synchronize()
            t_all.append(time.perf_counter() - t0)
        again, _ = E.eval_tables(gt, dt, classes)
        identical = all(tables[k].tobytes() == again[k].tobytes() for k in ("recall", "precision", "orientation", "ap"))
        # known answers: detections equal to the ground truth, and moved far away. The equal detections are turned by
        # 0.01 rad about their centre: rotate_iou.py's clipping is degenerate for two coincident rectangles (corners on
        # edges; the reference's own kernel returns 0 or 1/3 for a box against itself), a copy turned this little keeps
        # an IoU above 0.99 in BEV and 3D and no decision on an edge.
        obj = gt.objects.clone()
        obj[:, 14] += 0.01
        obj[:, 15] = torch.arange(obj.shape[0], device=obj.device, dtype=torch.float64) / obj.shape[0] + 0.5
        perfect, _ = E.eval_tables(gt, E.KittiAnnos(obj, gt.counts), classes)
        far = obj.clone()
        far[:, 11] += 100.0
        far[:, [4, 6]] += 5000.0
        away, _ = E.eval_tables(gt, E.KittiAnnos(far, gt.counts), classes)
        aps = perfect["ap"][:, :3]                                        # [R40 / R11][bbox, bev, 3d][cls][diff][k]
        want = np.where(valid_gt_exists(gt, classes), 100.0, 0.0)[None, None, :, :, None]
        off_perfect = [(r, m, c, l, k, float(aps[r, m, c, l, k])) for r, m, c, l, k in zip(*np.nonzero(aps != want))]
        ok_perfect = not off_perfect
        ok_away = bool(np.all(away["ap"] == 0.0))
    st = np.array(t_stage)
    print(json.dumps({
        "gpu": q, "images": args.images, "gt_objects": n_obj, "detections": n_det, "repeat": args.repeat,
        "from_label_dir_ms": round(median(t_parse) * 1e3, 2),
        "overlaps_ms": round(median(st[:, 0]), 3), "statistics_ms": round(median(st[:, 1]), 3),
        "ap_ms": round(median(st[:, 2]), 3), "evaluate_python_ms": round(median(t_all) * 1e3, 2),
        "ap_100_where_valid_gt": ok_perfect, "off_perfect": [[int(v) for v in o[:5]] + [o[5]] for o in off_perfect[:12]],
        "ap_0_when_moved_away": ok_away, "two_runs_bit_identical": identical,
        "car_3d_moderate_R40": float(tables["ap"][0, 2, 0, 1, 0])}))
    print(result)
    if not (ok_perfect and ok_away and identical):
        sys.exit(1)


if __name__ == "__main__":
    main()
