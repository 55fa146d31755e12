"""Golden fixture of the KITTI official metric from the UNMODIFIED reference: tests/golden/kitti_eval.npz.

    NUMBA_ENABLE_CUDASIM=1 python -m oracle.make_golden_kitti_eval

numba's CUDA simulator runs the reference's rotated-IoU kernel (rotate_iou.py) on the CPU, so eval.py and evaluate.py
run as they are; skimage and fire are mocked (visualiser / CLI imports only). The simulator's float arithmetic is not
the GPU's, so BEV / 3D overlaps may differ from a float32 kernel in the last bits. Every detection is therefore resampled
until none of its 2D, BEV, 3D or DontCare overlaps lies within MARGIN of an overlap threshold and none of its BEV corners
lies within CORNER_MARGIN metres of an edge line of a box it overlaps (or the other way round); a float32 decision cannot
flip on such a set.

The seeded set: KITTI-like labels over N_IMG images (Car, Pedestrian, Cyclist, Van, Person_sitting, Truck, DontCare;
occlusion and truncation over all three difficulties; heights on both sides of 25 and 40; every Cyclist occluded, so
Cyclist/easy has no valid ground truth), detections that are perturbed copies, class swaps, duplicates, false positives,
boxes under MIN_HEIGHT and boxes on DontCare regions, images without ground truth and images without detections (the
reference writer's lone "\\n"), and four crowded images with 40, 70, 100 and 128 detections. A second, small set has
alpha = -10 on every detection, so AOS is off."""
import os
import sys
import tempfile
from unittest import mock

import numpy as np

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")
from oracle.ref_shims import REF_ROOT  # noqa: E402

EVAL_DIR = os.path.join(REF_ROOT, "data", "datasets", "evaluation")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "kitti_eval.npz")
THRESHOLDS = (0.25, 0.5, 0.7)
MARGIN = 1e-3
CORNER_MARGIN = 1e-4
N_IMG, N_IMG_NOAOS = 240, 24
CROWDED = {5: 40, 60: 70, 120: 100, 180: 128}    # images whose assigned-detection masks span 2, 3 and 4 words
FIELDS = ("truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")


def reference():
    for n in ("skimage", "skimage.io", "fire"):
        sys.modules.setdefault(n, mock.MagicMock())
    if EVAL_DIR not in sys.path:
        sys.path.insert(0, EVAL_DIR)
    from kitti_object_eval_python import eval as ev, evaluate as evl, kitti_common as kc
    return ev, evl, kc


# ---------------------------------------------------------------------------------------------------- label synthesis
def gt_object(rng, name):
    if name == "DontCare":
        x1, y1 = rng.uniform(0, 1100), rng.uniform(120, 250)
        return dict(name=name, trunc=-1.0, occ=-1, alpha=-10.0, box=(x1, y1, x1 + rng.uniform(20, 120), y1 + rng.uniform(15, 60)),
                    hwl=(-1.0, -1.0, -1.0), loc=(-1000.0, -1000.0, -1000.0), ry=-10.0)
    hwl = {"Car": (1.5, 1.6, 3.9), "Van": (2.2, 1.9, 5.0), "Truck": (3.2, 2.5, 10.0), "Pedestrian": (1.75, 0.65, 0.85),
           "Person_sitting": (1.3, 0.6, 0.8), "Cyclist": (1.75, 0.6, 1.75)}[name]
    hwl = tuple(v * rng.uniform(0.85, 1.15) for v in hwl)
    z = rng.uniform(4, 65)
    x, y = rng.uniform(-0.5, 0.5) * z, rng.uniform(1.4, 1.9)
    h2d = float(np.clip(720 * hwl[0] / z * rng.uniform(0.9, 1.1), 12, 250))   # both sides of 25 and 40
    w2d = h2d * rng.uniform(0.4, 2.5)
    cx = 610 + 720 * x / z
    box = (cx - w2d / 2, 175 - h2d / 2, cx + w2d / 2, 175 + h2d / 2)
    occ = int(rng.integers(1, 3)) if name == "Cyclist" else int(rng.choice(4, p=(0.5, 0.25, 0.2, 0.05)))
    return dict(name=name, trunc=float(rng.choice((0.0, 0.0, 0.1, 0.2, 0.4, 0.7))), occ=occ, alpha=rng.uniform(-np.pi, np.pi),
                box=box, hwl=hwl, loc=(x, y, z), ry=rng.uniform(-np.pi, np.pi))


def make_gt(rng):
    names = ("Car", "Car", "Car", "Car", "Pedestrian", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "DontCare")
    n = 0 if rng.random() < 0.06 else int(rng.integers(1, 12))
    return [gt_object(rng, names[int(rng.integers(len(names)))]) for _ in range(n)]


DT_NAMES = ("Car", "Pedestrian", "Cyclist")
SWAP = {"Car": "Pedestrian", "Van": "Car", "Truck": "Car", "Pedestrian": "Cyclist", "Person_sitting": "Pedestrian",
        "Cyclist": "Pedestrian"}


def det_maker(kind, g=None):
    """a closure drawing one detection of the given kind; called again to resample it"""
    def draw(rng):
        if kind in ("copy", "swap", "dup"):
            bw, bh = g["box"][2] - g["box"][0], g["box"][3] - g["box"][1]
            box = tuple(np.add(g["box"], rng.normal(0, 0.06, 4) * (bw, bh, bw, bh)))
            name = g["name"] if kind != "swap" else SWAP[g["name"]]
            name = {"Van": "Car", "Truck": "Car", "Person_sitting": "Pedestrian"}.get(name, name)
            return dict(name=name, trunc=0.0, occ=0, alpha=g["alpha"] + rng.normal(0, 0.3), box=box,
                        hwl=tuple(np.multiply(g["hwl"], rng.uniform(0.85, 1.15, 3))),
                        loc=tuple(np.add(g["loc"], rng.normal(0, 0.04, 3) * (1, 1, g["loc"][2] / 4))),
                        ry=g["ry"] + rng.normal(0, 0.15))
        if kind == "dontcare":        # a detection on a DontCare region
            bw, bh = g["box"][2] - g["box"][0], g["box"][3] - g["box"][1]
            box = tuple(np.add(g["box"], rng.normal(0, 0.1, 4) * (bw, bh, bw, bh)))
            d = gt_object(rng, DT_NAMES[int(rng.integers(2))])
            d.update(box=box, trunc=0.0, occ=0)
            return d
        d = gt_object(rng, DT_NAMES[int(rng.integers(3))])            # false positive anywhere
        d.update(trunc=0.0, occ=0)
        if kind == "small":
            y = d["box"][1]
            d["box"] = (d["box"][0], y, d["box"][2], y + rng.uniform(8, 24))
        return d
    return draw


def make_dt(rng, gts):
    makers = []
    for g in gts:
        if g["name"] == "DontCare":
            if rng.random() < 0.6:
                makers.append(det_maker("dontcare", g))
            continue
        if rng.random() < 0.85:
            makers.append(det_maker("swap" if rng.random() < 0.1 else "copy", g))
        if rng.random() < 0.15:
            makers.append(det_maker("dup", g))
    makers += [det_maker("fp") for _ in range(int(rng.integers(0, 4)))]
    makers += [det_maker("small") for _ in range(int(rng.random() < 0.3))]
    return makers


def fmt_gt(o):
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        o["name"], o["trunc"], o["occ"], o["alpha"], *o["box"], *o["hwl"], *o["loc"], o["ry"])


def fmt_dt(o, score):
    # generate_kitti_3d_detection's row: class, 0, 0, then np.round(4) values written by repr
    vals = np.round(np.array([o["alpha"], *o["box"], *o["hwl"], *o["loc"], o["ry"], score], np.float32), 4).tolist()
    return " ".join([o["name"], "0", "0"] + [repr(v) for v in vals])


def text(lines):
    return "".join(l + "\n" for l in lines) if lines else "\n"


def parse(kc, s):
    with tempfile.NamedTemporaryFile("w", suffix=".txt", delete=False) as f:
        f.write(s)
    try:
        return kc.get_label_anno(f.name)
    finally:
        os.unlink(f.name)


# -------------------------------------------------------------------------------------------------------- margins
def bev_corners(x, z, l, w, ry):
    c, s = np.cos(ry), np.sin(ry)
    px, py = np.array([-l, -l, l, l]) / 2, np.array([-w, w, w, -w]) / 2
    return np.stack([c * px + s * py + x, -s * px + c * py + z], 1)


def near_edge(a, b):
    """a corner of box a within CORNER_MARGIN of an edge line of box b"""
    for k in range(4):
        p, q = b[k], b[(k + 1) % 4]
        n = np.array([q[1] - p[1], p[0] - q[0]])
        nn = np.linalg.norm(n)
        if nn > 0 and (np.abs((a - p) @ n) / nn < CORNER_MARGIN).any():
            return True
    return False


def bad_detections(ev, gt, dt):
    """indices of detections with an overlap near a threshold or a corner near an edge"""
    bad = set()
    if len(dt["name"]) == 0:
        return bad
    if len(gt["name"]):
        ovs = [ev.calculate_iou_partly([dt], [gt], m, 1)[0][0] for m in range(3)]
        for ov in ovs:
            for t in THRESHOLDS:
                bad |= set(np.nonzero((np.abs(ov - t) < MARGIN).any(1))[0].tolist())
        for d in range(len(dt["name"])):
            cd = bev_corners(dt["location"][d, 0], dt["location"][d, 2], dt["dimensions"][d, 0], dt["dimensions"][d, 2],
                             dt["rotation_y"][d])
            for g in range(len(gt["name"])):
                if ovs[1][d, g] > 0 or np.abs(dt["location"][d, [0, 2]] - gt["location"][g, [0, 2]]).max() < 12:
                    cg = bev_corners(gt["location"][g, 0], gt["location"][g, 2], gt["dimensions"][g, 0],
                                     gt["dimensions"][g, 2], gt["rotation_y"][g])
                    if near_edge(cd, cg) or near_edge(cg, cd):
                        bad.add(d)
    dc = gt["bbox"][gt["name"] == "DontCare"] if len(gt["name"]) else np.zeros((0, 4))
    if len(dc):
        ov = ev.image_box_overlap(dt["bbox"], dc, 0)
        for t in THRESHOLDS:
            bad |= set(np.nonzero((np.abs(ov - t) < MARGIN).any(1))[0].tolist())
    return bad


def crowd(rng, gts, makers, n):
    """top the detections up to n with duplicates of the image's objects and false positives"""
    objs = [g for g in gts if g["name"] != "DontCare"]
    while len(makers) < n:
        makers.append(det_maker("dup", objs[int(rng.integers(len(objs)))]) if rng.random() < 0.6 else det_maker("fp"))
    return makers


def make_set(ev, kc, rng, n_img, no_alpha=False, crowded=None):
    """crowded: {image index: detection count} for images with more detections than one 32-bit mask word"""
    crowded = crowded or {}
    ids = np.sort(rng.choice(7481, n_img, replace=False))
    labels, results, n_dropped = [], [], 0
    pool = list(rng.permutation(np.arange(500, 10000)) / 1e4)     # distinct 4-decimal scores
    for i in range(n_img):
        gts = make_gt(rng)
        while i in crowded and sum(g["name"] != "DontCare" for g in gts) < 6:
            gts = make_gt(rng)
        gt_txt = text([fmt_gt(o) for o in gts])
        gt = parse(kc, gt_txt)
        makers = [] if rng.random() < 0.05 and i not in crowded else make_dt(rng, gts)
        if i in crowded:
            makers = crowd(rng, gts, makers, crowded[i])
        dets = [m(rng) for m in makers]
        scores = np.array([pool.pop() for _ in dets])
        for _ in range(60):
            if no_alpha:
                for d in dets:
                    d["alpha"] = -10.0
            dt_txt = text([fmt_dt(d, s) for d, s in zip(dets, scores)])
            dt = parse(kc, dt_txt)
            bad = bad_detections(ev, gt, dt)
            if not bad:
                break
            for d in bad:
                dets[d] = makers[d](rng)
        else:
            keep = [d for d in range(len(dets)) if d not in bad]
            n_dropped += len(dets) - len(keep)
            dets, scores = [dets[d] for d in keep], scores[keep]
            dt_txt = text([fmt_dt(d, s) for d, s in zip(dets, scores)])
            assert not bad_detections(ev, gt, parse(kc, dt_txt))
        labels.append(gt_txt)
        results.append(dt_txt)
    # distinct scores over the whole set: the first pass keeps the highest-scoring match
    allsc = np.concatenate([parse(kc, r)["score"] for r in results])
    assert len(np.unique(allsc)) == len(allsc), "score collision; change the seed"
    return ids, labels, results, n_dropped


def pack(annos, prefix, z):
    z[prefix + "count"] = np.array([len(a["name"]) for a in annos], np.int64)
    z[prefix + "name"] = np.concatenate([a["name"] for a in annos]).astype("U16")
    for f in FIELDS:
        z[prefix + f] = np.concatenate([a[f] for a in annos], 0)


def evaluate_set(ev, evl, kc, ids, labels, results, z, tag):
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "label"))
        os.makedirs(os.path.join(d, "pred"))
        for i, l, r in zip(ids, labels, results):
            open(os.path.join(d, "label", "%06d.txt" % i), "w").write(l)
            open(os.path.join(d, "pred", "%06d.txt" % i), "w").write(r)
        open(os.path.join(d, "split.txt"), "w").write("".join("%d\n" % i for i in ids))
        gt = kc.get_label_annos(os.path.join(d, "label"), [int(i) for i in ids])
        dt = kc.get_label_annos(os.path.join(d, "pred"))
        for metric in ("R40", "R11"):
            res, ret = evl.evaluate(os.path.join(d, "label"), os.path.join(d, "pred"), os.path.join(d, "split.txt"),
                                    current_class=["Car", "Pedestrian", "Cyclist"], metric=metric)
            res2, ret2 = ev.get_official_eval_result(gt, dt, [0, 1, 2], metric=metric)
            assert res == res2 and list(ret) == list(ret2)
            z["%s_result_%s" % (tag, metric)] = np.array(res)
            z["%s_ret_keys_%s" % (tag, metric)] = np.array(list(ret))
            z["%s_ret_values_%s" % (tag, metric)] = np.array([float(v) for v in ret.values()])
    z[tag + "_ids"] = ids
    z[tag + "_label_text"] = np.array(labels)
    z[tag + "_result_text"] = np.array(results)
    return gt, dt


def main(seed=20261015):
    ev, evl, kc = reference()
    rng = np.random.default_rng(seed)
    z = {}
    ids, labels, results, dropped = make_set(ev, kc, rng, N_IMG, crowded=CROWDED)
    gt, dt = evaluate_set(ev, evl, kc, ids, labels, results, z, "main")
    pack(gt, "gt_", z)
    pack(dt, "dt_", z)
    min_overlaps = np.stack([np.array([[0.7, 0.5, 0.5]] * 3), np.array([[0.7, 0.5, 0.5], [0.5, 0.25, 0.25], [0.5, 0.25, 0.25]])])
    for m in range(3):
        ov, _, _, _ = ev.calculate_iou_partly(dt, gt, m, 100)
        z["overlaps_%d" % m] = np.concatenate([o.reshape(-1) for o in ov])
        ret = ev.eval_class(gt, dt, [0, 1, 2], [0, 1, 2], m, min_overlaps, compute_aos=(m == 0))
        for k, v in ret.items():
            z["%s_%d" % (k, m)] = v
    ids2, labels2, results2, dropped2 = make_set(ev, kc, rng, N_IMG_NOAOS, no_alpha=True)
    evaluate_set(ev, evl, kc, ids2, labels2, results2, z, "noaos")
    np.savez_compressed(OUT, **z)
    print("wrote %s: %d + %d images, %d / %d objects, %d detections dropped after 60 resamples"
          % (OUT, N_IMG, N_IMG_NOAOS, len(z["gt_name"]), len(z["dt_name"]), dropped + dropped2))


if __name__ == "__main__":
    main()
