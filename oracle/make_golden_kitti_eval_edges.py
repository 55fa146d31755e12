"""Golden fixture of the KITTI official metric at its decision edges, from the UNMODIFIED reference:
tests/golden/kitti_eval_edges.npz.

    NUMBA_ENABLE_CUDASIM=1 python -m oracle.make_golden_kitti_eval_edges

tests/golden/kitti_eval.npz keeps every overlap clear of the thresholds and every score unique, so it never exercises
the metric's tie and boundary rules. This set is built from them, on values whose outcome does not depend on how numba's
CUDA simulator rounds (integer 2D boxes, axis-aligned BEV boxes on dyadic coordinates, exact duplicates):
  - 2D IoUs and DontCare overlaps (criterion 0) of exactly 0.5 and exactly the double 0.7, next to boxes one ulp above;
  - BEV / 3D IoUs of exactly 0.25 and 0.5 (nested boxes sharing edges), and ones within 4e-5 above / below 0.7;
  - equal scores and equal overlaps where which detection wins changes the counts; exact duplicate detections; tied
    true-positive scores across images (repeated thresholds); scores on 1e-2 and 1e-4 grids;
  - ground-truth and detection 2D heights of exactly 25 and 40, negative detection heights, truncation 0.15 / 0.3 / 0.5,
    occlusion 0..3, Van / Person_sitting / Truck / Tram / Misc / lower-case dontcare;
  - images of 31, 32, 33, 63, 64, 65, 95, 96, 97, 127 and 128 detections whose matching and DontCare-suppressed
    detections sit at mask bits 31 / 32, 63 / 64, 95 / 96 and 127;
  - more than 41 true positives of one configuration at full recall, 300 images (not a multiple of 128, more than 256),
    the first image without detections.
The rest of the images are make_golden_kitti_eval's seeded random images (margins kept, scores rounded to 2 or 4
decimals). A second small set has its first image empty and alpha = -10 on the first detection of the next, so AOS is
off by the reference's rule although later detections have alphas.

Recorded: the inputs as the reference parses them, the three overlaps, eval_class's tables for the class lists [0, 1, 2],
[2, 0] and [5, 4, 3, 2, 1, 0], the `result` text and `ret_dict` of R40 and R11 for each list (evaluate and
get_official_eval_result agree), and the label and result text of both sets. The reference's rotate_iou_gpu_eval is
memoised on its inputs, so repeated evaluations of one set simulate the rotated-IoU kernel once."""
import io
import os
import zipfile

import numpy as np

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")
from oracle import make_golden_kitti_eval as base  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "kitti_eval_edges.npz")
CLASS_LISTS = ((0, 1, 2), (2, 0), (5, 4, 3, 2, 1, 0))
CROWDED = (31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128)
N_IMG, N_IMG_NOAOS = 300, 12
# nested lengths l next to 2.8: BEV / 3D IoU l / 4 about 3e-5 below and above 0.7, clear of the reference's float32
# segment-intersection error (4e-6 here)
F32_BELOW_07, F32_ABOVE_07 = 45874 / 2 ** 14, 45877 / 2 ** 14


def obj(name, box, x=0.0, z=20.0, hwl=(1.5, 2.0, 4.0), ry=0.0, alpha=0.25, trunc=0.0, occ=0, y=1.5, score=None):
    return dict(name=name, trunc=trunc, occ=occ, alpha=alpha, box=tuple(float(v) for v in box), hwl=tuple(hwl),
                loc=(x, y, z), ry=ry, score=score)


def dontcare(box):
    return dict(name="DontCare", trunc=-1.0, occ=-1, alpha=-10.0, box=tuple(float(v) for v in box), hwl=(-1.0, -1.0, -1.0),
                loc=(-1000.0, -1000.0, -1000.0), ry=-10.0, score=None)


def line(o):
    vals = (o["trunc"], o["occ"], o["alpha"], *o["box"], *o["hwl"], *o["loc"], o["ry"])
    if o["score"] is not None:
        vals = (0, 0) + vals[2:] + (o["score"],)
    return " ".join([o["name"]] + [repr(v) if isinstance(v, float) else str(v) for v in vals])


def copy(g, score, **kw):
    """a detection equal to a ground-truth object (2D box, 3D box, alpha), renamed / changed by kw"""
    d = dict(g, trunc=0.0, occ=0, score=score)
    d.update(kw)
    return d


def box_at(i, h=100.0, w=60.0, y1=100.0):
    """the i-th slot of a row of disjoint integer 2D boxes, with its 3D box in a disjoint BEV slot"""
    x1 = 10.0 + 70.0 * (i % 17)
    return (x1, y1 + 120.0 * (i // 17), x1 + w, y1 + 120.0 * (i // 17) + h), dict(x=-40.0 + 5.0 * (i % 17), z=10.0 + 5.0 * (i // 17))


# ------------------------------------------------------------------------------------------------------ edge images
def img_2d_thresholds():
    """2D IoU exactly 0.5 and 0.7 (and one ulp above), DontCare overlaps exactly 0.5 and 0.7 (and one ulp above)"""
    g0, g1, g2 = obj("Car", (100, 100, 200, 200), x=-8.0), obj("Car", (300, 100, 400, 200), x=0.0), \
        obj("Car", (500, 100, 600, 200), x=8.0)
    gts = [g0, g1, g2, dontcare((700, 100, 800, 150)), dontcare((900, 100, 1000, 170))]
    below = float(np.nextafter(200.0, 100.0))
    dts = [copy(g0, 0.61, box=(100.0, 100.0, 200.0, 150.0)),            # IoU 0.5
           copy(g1, 0.62, box=(300.0, 100.0, 400.0, 170.0)),            # IoU 0.7
           copy(g2, 0.63, box=(500.0, 100.0, 600.0, float(np.nextafter(170.0, 200.0)))),   # just above 0.7
           copy(g0, 0.64, box=(700.0, 100.0, 800.0, 200.0), x=20.0),    # DontCare overlap 0.5
           copy(g0, 0.65, box=(700.0, 100.0, 800.0, below), x=26.0),    # DontCare overlap just above 0.5
           copy(g0, 0.66, box=(900.0, 100.0, 1000.0, 200.0), x=32.0),   # DontCare overlap 0.7
           copy(g0, 0.67, box=(900.0, 100.0, 1000.0, below), x=38.0)]   # just above 0.7
    return gts, dts


def img_2d_thresholds_iou_up():
    """IoU one ulp above 0.5"""
    g = obj("Car", (100, 100, 200, 200))
    return [g], [copy(g, 0.5, box=(100.0, 100.0, 200.0, float(np.nextafter(150.0, 200.0))))]


def img_bev_thresholds():
    """axis-aligned nested BEV / 3D boxes sharing edges: IoU exactly 0.5 and 0.25, and just below / above 0.7 after
    0.7 by 3e-5 (2D boxes identical, so only BEV / 3D decide)"""
    gts, dts = [], []
    for i, (cls, gl, gw, dl) in enumerate((("Car", 4.0, 2.0, 2.0), ("Pedestrian", 1.0, 0.5, 0.5),
                                          ("Pedestrian", 1.0, 0.5, 0.25), ("Car", 4.0, 2.0, F32_BELOW_07),
                                          ("Car", 4.0, 2.0, F32_ABOVE_07), ("Cyclist", 2.0, 0.5, 0.5))):
        box, p = box_at(i)
        g = obj(cls, box, hwl=(1.5, gw, gl), **p)
        gts.append(g)
        dts.append(copy(g, round(0.7 - 0.01 * i, 2), hwl=(1.5, gw, dl)))
    return gts, dts


def img_ties():
    """equal scores and equal overlaps where the first detection and the last give different counts: A and B overlap
    the first object equally (and tie on score), only A overlaps the second above 0.7"""
    g1, g2 = obj("Car", (100, 100, 200, 200)), obj("Car", (120, 100, 220, 200), x=8.0)
    a = copy(g1, 0.8, box=(110.0, 100.0, 210.0, 200.0))
    b = copy(g1, 0.8, box=(90.0, 100.0, 190.0, 200.0))
    return [g1, g2], [a, b]


def img_ties_second_pass():
    """as img_ties, the overlap tie alone: distinct scores, the higher-scored B listed second"""
    g1, g2 = obj("Car", (100, 100, 200, 200)), obj("Car", (120, 100, 220, 200), x=8.0)
    a = copy(g1, 0.85, box=(110.0, 100.0, 210.0, 200.0))
    b = copy(g1, 0.9, box=(90.0, 100.0, 190.0, 200.0))
    return [g1, g2], [a, b]


def img_duplicates():
    g = obj("Car", (100, 100, 200, 200))
    d = copy(g, 0.75, box=(102.0, 100.0, 200.0, 200.0))
    return [g], [d, dict(d), dict(d)]


def img_heights():
    """2D heights exactly 25 and 40 (ground truth and detections), a negative detection height, truncation written
    0.15 / 0.3 / 0.5 and occlusion 0..3"""
    gts, dts = [], []
    spec = ((25.0, 0.0, 0, 25.0), (40.0, 0.0, 0, 40.0), (40.5, 0.0, 0, 40.0), (25.5, 0.0, 1, 25.0),
            (60.0, 0.15, 0, 60.0), (60.0, 0.3, 1, 60.0), (60.0, 0.5, 2, 60.0), (60.0, 0.0, 3, 60.0), (41.0, 0.0, 0, 25.0))
    for i, (gh, tr, oc, dh) in enumerate(spec):
        box, p = box_at(i, h=gh)
        g = obj("Car", box, trunc=tr, occ=oc, **p)
        gts.append(g)
        b = box[:3] + (box[1] + dh,)
        dts.append(copy(g, round(0.55 + 0.01 * i, 2), box=b))
    box, p = box_at(len(spec), h=50.0)
    dts.append(obj("Car", (box[0], box[3], box[2], box[1]), score=0.5, **p))          # height -50: a false positive
    box, p = box_at(len(spec) + 1, h=30.0)
    dts.append(obj("Car", (box[0], box[3], box[2], box[1]), score=0.52, **p))         # height -30
    return gts, dts


def img_names():
    names = ("Van", "Person_sitting", "Truck", "Tram", "Misc", "dontcare", "Pedestrian", "Cyclist")
    gts, dts = [], []
    for i, n in enumerate(names):
        box, p = box_at(i)
        g = obj(n, box, **p)
        gts.append(g)
        dn = {"Van": "Car", "Person_sitting": "Pedestrian", "Truck": "Car", "Tram": "Car", "Misc": "Cyclist",
              "dontcare": "Car"}.get(n, n)
        dts.append(copy(g, round(0.45 + 0.01 * i, 2), name=dn))
    return gts, dts


def img_crowded(n, rng):
    """n detections: the matches of ground-truth objects at mask bits 31, 32, 63, 64, 95, 96, 127 and n - 1 (those below
    n), a DontCare-suppressed detection at n - 2, the rest false positives in their own slots"""
    bits = sorted({b for b in (31, 32, 63, 64, 95, 96, 127, n - 1) if b < n})
    gts, dts = [], [None] * n
    for s, b in enumerate(bits):
        box, p = box_at(s)
        g = obj("Car", box, **p)
        gts.append(g)
        dts[b] = copy(g, round(float(rng.uniform(0.3, 0.9)), 2))
    box, p = box_at(len(bits))
    gts.append(dontcare(box))
    sup = n - 2 if n - 2 not in bits else n - 3
    dts[sup] = obj("Car", box, score=round(float(rng.uniform(0.3, 0.9)), 2), x=30.0, z=60.0)
    k = len(bits) + 1
    for j in range(n):
        if dts[j] is None:
            box, p = box_at(k, h=float(rng.integers(20, 60)))
            k += 1
            dts[j] = obj("Car", box, score=round(float(rng.uniform(0.05, 0.95)), 2), **p)
    return gts, dts


def img_full_recall(i, score):
    """one Cyclist and its exact copy: every Cyclist of the random images is occluded, so with over 41 of these
    Cyclist / easy has more than 41 true positives at full recall"""
    box, p = box_at(i % 17)
    g = obj("Cyclist", box, **p)
    return [g], [copy(g, score)]


def edge_images(rng):
    imgs = [([obj("Car", (100, 100, 200, 200))], [])]          # first image: no detections
    imgs += [img_2d_thresholds(), img_2d_thresholds_iou_up(), img_bev_thresholds(), img_ties(), img_ties_second_pass(),
             img_duplicates(), img_heights(), img_names()]
    imgs += [img_crowded(n, rng) for n in CROWDED]
    # tied true-positive scores across images: repeated thresholds
    imgs += [img_full_recall(i, 0.5 if i % 3 else 0.75) for i in range(24)]
    imgs += [img_full_recall(i, round(0.3 + 0.0123 * i, 4)) for i in range(30)]
    return imgs


# ---------------------------------------------------------------------------------------------------------- the sets
def texts(imgs):
    return [base.text([line(o) for o in g]) for g, d in imgs], [base.text([line(o) for o in d]) for g, d in imgs]


def random_images(ev, kc, rng, n):
    """make_golden_kitti_eval's random images with their scores rounded to 2 (even images) or 4 decimals"""
    ids, labels, results, _ = base.make_set(ev, kc, rng, n)
    out = []
    for i, r in enumerate(results):
        if r == "\n":
            out.append(r)
            continue
        rows = [l.split(" ") for l in r.splitlines()]
        for w in rows:
            w[-1] = repr(round(float(w[-1]), 2 if i % 2 == 0 else 4))
        out.append("".join(" ".join(w) + "\n" for w in rows))
    return labels, out


def memoise(ev):
    """rotate_iou_gpu_eval is a pure function of its inputs: simulate it once per distinct input"""
    fn, cache = ev.rotate_iou_gpu_eval, {}

    def cached(boxes, query_boxes, criterion=-1, device_id=0):
        key = (boxes.astype(np.float32).tobytes(), query_boxes.astype(np.float32).tobytes(), boxes.shape[0],
               query_boxes.shape[0], criterion)
        if key not in cache:
            cache[key] = fn(boxes, query_boxes, criterion, device_id)
        return cache[key].copy()
    ev.rotate_iou_gpu_eval = cached


def evaluate(ev, evl, kc, ids, labels, results, z, tag):
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        for sub in ("label", "pred"):
            os.makedirs(os.path.join(d, sub))
        for i, l, r in zip(ids, labels, results):
            open(os.path.join(d, "label", "%06d.txt" % i), "w").write(l)
            open(os.path.join(d, "pred", "%06d.txt" % i), "w").write(r)
        open(os.path.join(d, "split.txt"), "w").write("".join("%d\n" % i for i in ids))
        gt = kc.get_label_annos(os.path.join(d, "label"), [int(i) for i in ids])
        dt = kc.get_label_annos(os.path.join(d, "pred"))
        for cl in CLASS_LISTS:
            name = "".join(map(str, cl))
            names = [base_names[c] for c in cl]
            for metric in ("R40", "R11"):
                res, ret = evl.evaluate(os.path.join(d, "label"), os.path.join(d, "pred"), os.path.join(d, "split.txt"),
                                        current_class=names, metric=metric)
                res2, ret2 = ev.get_official_eval_result(gt, dt, list(cl), metric=metric)
                assert res == res2 and list(ret) == list(ret2)
                z["%s_result_%s_%s" % (tag, name, metric)] = np.array(res)
                z["%s_ret_keys_%s_%s" % (tag, name, metric)] = np.array(list(ret))
                z["%s_ret_values_%s_%s" % (tag, name, metric)] = np.array([float(v) for v in ret.values()])
    z[tag + "_ids"] = np.asarray(ids)
    z[tag + "_label_text"] = np.array(labels)
    z[tag + "_result_text"] = np.array(results)
    return gt, dt


base_names = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting", 5: "Truck"}


def save(path, arrays):
    """np.savez_compressed with fixed member timestamps, so a rerun writes the same bytes"""
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as f:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            f.writestr(zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0)), buf.getvalue(), zipfile.ZIP_DEFLATED)


def main(seed=20261018):
    ev, evl, kc = base.reference()
    memoise(ev)
    rng = np.random.default_rng(seed)
    z = {}
    edges = edge_images(rng)
    labels, results = texts(edges)
    rl, rr = random_images(ev, kc, rng, N_IMG - len(edges))
    labels, results = labels + rl, results + rr
    ids = np.sort(rng.choice(7481, N_IMG, replace=False))
    gt, dt = evaluate(ev, evl, kc, ids, labels, results, z, "main")
    base.pack(gt, "gt_", z)
    base.pack(dt, "dt_", z)
    for m in range(3):
        ov, _, _, _ = ev.calculate_iou_partly(dt, gt, m, 100)
        z["overlaps_%d" % m] = np.concatenate([o.reshape(-1) for o in ov])
    for cl in CLASS_LISTS:
        name = "".join(map(str, cl))
        mo = np.stack([np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3),
                       np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5],
                                 [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]])])[:, :, list(cl)]
        for m in range(3):
            ret = ev.eval_class(gt, dt, list(cl), [0, 1, 2], m, mo, compute_aos=(m == 0))
            for k, v in ret.items():
                z["%s_%s_%d" % (k, name, m)] = v
    # AOS off: the first image has no detections, the next one's first detection has alpha -10
    noaos = edge_images(rng)[:N_IMG_NOAOS]
    noaos[1] = (noaos[1][0], [dict(noaos[1][1][0], alpha=-10.0)] + noaos[1][1][1:])
    l2, r2 = texts(noaos)
    evaluate(ev, evl, kc, np.arange(N_IMG_NOAOS) * 7 + 3, l2, r2, z, "noaos")
    save(OUT, z)
    print("wrote %s: %d + %d images, %d / %d objects" % (OUT, N_IMG, N_IMG_NOAOS, len(z["gt_name"]), len(z["dt_name"])))


if __name__ == "__main__":
    main()
