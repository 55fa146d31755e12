"""Golden fixture of the KITTI COCO-style AP from the UNMODIFIED reference: tests/golden/kitti_coco.npz.

    NUMBA_ENABLE_CUDASIM=1 python -m oracle.make_golden_kitti_coco

Runs the reference's get_coco_eval_result (kitti_object_eval_python/eval.py:626-643, 729-788) and its evaluate() entry
(evaluate.py:14-32) with coco=True and with score_thresh > 0, under numba's CUDA simulator as
oracle/make_golden_kitti_eval.py does. One shim, nothing else patched: do_coco_style_eval calls
np.linspace(start, stop, 10.0) with a float count, which NumPy 2 refuses (TypeError: 'numpy.float64' object cannot be
interpreted as an integer); np.linspace is wrapped to pass int(num) and is otherwise numpy's own, so the threshold table
holds exactly the doubles the reference meant (0.8999999999999999, 0.44999999999999996 and 0.6499999999999999 among them).

The labels and detections are make_golden_kitti_eval's synthesis, resampled against every threshold of the
0.25:0.05:0.95 grid (the values both COCO ranges take) instead of the official three, so no 2D, BEV, 3D or DontCare
overlap lies within MARGIN of a threshold and no BEV corner near a box edge: a float32 decision cannot flip. The main
set has images without ground truth, images without detections and a crowded image of 128 detections; a small second
set has alpha = -10 on every detection, so AOS is off. SCORE_THRESH cases use a threshold equal to one detection's
score (filter_annos_low_score keeps it: `>=`)."""
import os
import tempfile

import numpy as np

os.environ.setdefault("NUMBA_ENABLE_CUDASIM", "1")
from oracle import make_golden_kitti_eval as base  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "kitti_coco.npz")
N_IMG, N_IMG_NOAOS = 140, 16
CROWDED = {9: 128, 70: 48}
CLASS_LISTS = ((0, 1, 2), (3, 4, 0))
GRID = tuple(sorted(set(np.linspace(0.5, 0.95, 10).tolist()) | set(np.linspace(0.25, 0.7, 10).tolist())))


def shim_linspace():
    """np.linspace with an integer count: the one change the reference's COCO path needs under NumPy 2"""
    linspace = np.linspace
    if getattr(linspace, "_int_count", False):
        return

    def int_count(start, stop, num=50, *args, **kwargs):
        return linspace(start, stop, int(num), *args, **kwargs)
    int_count._int_count = True
    np.linspace = int_count


def coco_min_overlaps(classes):
    """do_coco_style_eval's [10, 3 metric, ncls] table from get_coco_eval_result's class_to_range"""
    rng = {0: [0.5, 0.95, 10], 1: [0.25, 0.7, 10], 2: [0.25, 0.7, 10], 3: [0.5, 0.95, 10], 4: [0.25, 0.7, 10]}
    out = np.zeros([10, 3, len(classes)])
    for j, c in enumerate(classes):
        for i in range(3):
            out[:, i, j] = np.linspace(*rng[c])
    return out


def write_set(d, ids, labels, results):
    os.makedirs(os.path.join(d, "label"))
    os.makedirs(os.path.join(d, "pred"))
    for i, l, r in zip(ids, labels, results):
        open(os.path.join(d, "label", "%06d.txt" % i), "w").write(l)
        open(os.path.join(d, "pred", "%06d.txt" % i), "w").write(r)
    open(os.path.join(d, "split.txt"), "w").write("".join("%d\n" % i for i in ids))
    return os.path.join(d, "label"), os.path.join(d, "pred"), os.path.join(d, "split.txt")


def evaluate_set(ev, evl, kc, ids, labels, results, z, tag, score_thresh):
    with tempfile.TemporaryDirectory() as d:
        label, pred, split = write_set(d, ids, labels, results)
        gt = kc.get_label_annos(label, [int(i) for i in ids])
        dt = kc.get_label_annos(pred)
        for classes in CLASS_LISTS:
            name = "".join(map(str, classes))
            res = ev.get_coco_eval_result(gt, dt, list(classes))
            assert res == evl.evaluate(label, pred, split, current_class=list(classes), coco=True)
            z["%s_coco_%s" % (tag, name)] = np.array(res)
        names = ["Car", "Pedestrian", "Cyclist"]
        z["%s_coco_score" % tag] = np.array(evl.evaluate(label, pred, split, current_class=names, coco=True,
                                                          score_thresh=score_thresh))
        res, ret = evl.evaluate(label, pred, split, current_class=names, score_thresh=score_thresh, metric="R40")
        z["%s_score_result" % tag] = np.array(res)
        z["%s_score_ret_keys" % tag] = np.array(list(ret))
        z["%s_score_ret_values" % tag] = np.array([float(v) for v in ret.values()])
    z[tag + "_ids"] = ids
    z[tag + "_label_text"] = np.array(labels)
    z[tag + "_result_text"] = np.array(results)
    return gt, dt


def main(seed=20261018):
    shim_linspace()
    base.THRESHOLDS = GRID                     # resample against every COCO threshold
    ev, evl, kc = base.reference()
    rng = np.random.default_rng(seed)
    z = {"grid": np.array(GRID)}
    ids, labels, results, dropped = base.make_set(ev, kc, rng, N_IMG, crowded=CROWDED)
    scores = np.sort(np.concatenate([base.parse(kc, r)["score"] for r in results]))
    thresh = float(scores[len(scores) // 2])   # a detection's own score: kept by `>=`
    z["score_thresh"] = np.array(thresh)
    gt, dt = evaluate_set(ev, evl, kc, ids, labels, results, z, "main", thresh)
    base.pack(gt, "gt_", z)
    base.pack(dt, "dt_", z)
    for m in range(3):
        ov, _, _, _ = ev.calculate_iou_partly(dt, gt, m, 100)
        z["overlaps_%d" % m] = np.concatenate([o.reshape(-1) for o in ov])
    for classes in CLASS_LISTS:
        name = "".join(map(str, classes))
        mo = coco_min_overlaps(classes)
        z["min_overlaps_" + name] = mo
        for m in range(3):
            ret = ev.eval_class(gt, dt, list(classes), [0, 1, 2], m, mo, compute_aos=(m == 0))
            for k, v in ret.items():
                z["%s_%s_%d" % (k, name, m)] = v
    ids2, labels2, results2, dropped2 = base.make_set(ev, kc, rng, N_IMG_NOAOS, no_alpha=True)
    evaluate_set(ev, evl, kc, ids2, labels2, results2, z, "noaos", thresh)
    np.savez_compressed(OUT, **z)
    print("wrote %s: %d + %d images, %d / %d objects, score_thresh %r, %d detections dropped after 60 resamples"
          % (OUT, N_IMG, N_IMG_NOAOS, len(z["gt_name"]), len(z["dt_name"]), thresh, dropped + dropped2))


if __name__ == "__main__":
    main()
