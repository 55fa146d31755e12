"""TEST TOOLING — tests/golden/decode_depth.npz: the UNMODIFIED reference PostProcessor (model/head/detector_infer.py, via
oracle/ref_shims.py) for every OUTPUT_DEPTH estimator, oracle included, on the decode workload of oracle/make_golden.py
(syn.make_head_logits(2, 80, 24) with make_targets calibration), at thresholds 0.0 and 0.2. Build container only:

    python -m oracle.make_golden_depth

The oracle estimator needs ground truth. It is built here from a seed and stored in the fixture (gt_* fields, 40 slots per
image like DATASETS.MAX_OBJECTS):
  * perturbed copies of detections' decoded boxes at several IoUs (some below 0.5, so the match is rejected), with a depth
    next to a different estimator each time, so that every estimator index is chosen;
  * unmatched boxes, copies of detections' boxes under another class, and invalid slots (reg_mask 0) holding garbage;
  * when a detection's box is clamped to zero area, a zero-area GT box on it: the reference's box_iou is then 0 / 0 = NaN,
    which is not < 0.5, so the match is accepted.
Every detection's decision is kept away from its thresholds (IoU vs 0.5, nearest-centre distance, |d - z| between the
estimators), so boxes that differ in the last bits cannot flip it. Per method / image / threshold the fixture holds the
reference's `result`, `estimated_depth_error` and `proj_center`."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims as rs            # noqa: E402
from oracle.make_golden import ref_targets    # noqa: E402
from monoflex_b200 import synthetic as syn    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
METHODS = ('soft', 'hard', 'mean', 'oracle', 'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02', 'keypoints_13')
SINGLE = ('direct', 'keypoints_center', 'keypoints_02', 'keypoints_13')      # the four estimators, in ensemble order
G = 40
IOUS = (0.95, 0.8, 0.65, 0.56, 0.44, 0.3)


def box_iou(a, b):
    """engine/visualize_infer.py:23-27 in fp32"""
    a, b = a.astype(np.float32), b.astype(np.float32)
    inter = max(min(a[2], b[2]) - max(a[0], b[0]), 0) * max(min(a[3], b[3]) - max(a[1], b[1]), 0)
    union = (a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.float32(inter) / np.float32(union)


def decisions(boxes, clses, deps, gt):
    """-> per detection (chosen estimator or -1, ok): ok is False when a decision sits near one of its thresholds"""
    valid = gt[:, 0] != 0
    g = gt[valid]
    out = []
    for i in range(boxes.shape[0]):
        c = (boxes[i, :2] + boxes[i, 2:]) / 2
        dis = (((g[:, 2:4] + g[:, 4:6]) / 2 - c) ** 2).sum(1)
        dis[g[:, 1] != clses[i]] = 9999
        order = np.argsort(dis, kind='stable')
        near = order[0]
        ok = True
        if len(order) > 1 and dis[near] != 9999 and dis[order[1]] - dis[near] < 1e-3 * max(1.0, dis[near]):
            ok = False
        if dis[near] != 9999 and abs(dis[near] - 9999) < 10:
            ok = False
        iou = box_iou(boxes[i], g[near, 2:6])
        if not np.isnan(iou) and abs(iou - 0.5) < 0.02:
            ok = False
        if not iou < 0.5:
            d = np.abs(deps[i] - g[near, 6])
            o = np.argsort(d, kind='stable')
            if deps[i, o[1]] != deps[i, o[0]] and d[o[1]] - d[o[0]] < 1e-3 * max(1.0, g[near, 6]):
                ok = False
            out.append((int(o[0]), ok))
        else:
            out.append((-1, ok))
    return out


def make_gt(rng, boxes, clses, deps, n_hi, size):
    """one image's 40 GT slots (valid, class, x1, y1, x2, y2, z)"""
    gt = np.zeros((G, 7), np.float32)
    rows = []
    wh = boxes[:, 2:] - boxes[:, :2]
    zero = [i for i in range(len(boxes)) if wh[i, 0] == 0 or wh[i, 1] == 0]
    picks, targets = [], []
    for j in range(4):                  # for every estimator j, detections whose j-th depth stands apart from the others
        cand = [i for i in range(n_hi) if wh[i, 0] > 2 and wh[i, 1] > 2 and i not in picks
                and np.abs(np.delete(deps[i], j) - deps[i, j]).min() > 1.0]
        for i in rng.choice(cand, size=min(len(cand), 3), replace=False):
            picks.append(int(i))
            targets.append(j)
    for k, (i, j) in enumerate(zip(picks, targets)):                  # perturbed copies of detections
        s = 1.0 / np.sqrt(IOUS[k % len(IOUS)])
        c, h = (boxes[i, :2] + boxes[i, 2:]) / 2, wh[i] / 2 * s
        c = c + rng.uniform(-0.05, 0.05, 2) * wh[i]
        others = np.abs(np.delete(deps[i], j) - deps[i, j]).min()
        z = deps[i, j] + rng.choice((-1, 1)) * rng.uniform(0.05, 0.2) * max(others, 1e-2)
        rows.append((1, clses[i], c[0] - h[0], c[1] - h[1], c[0] + h[0], c[1] + h[1], z))
    for i in zero[:1]:                                                # zero-area box: NaN IoU, match accepted
        j = int(rng.integers(4))
        rows.append((1, clses[i], *boxes[i], deps[i, j] + 1e-3 * max(1.0, deps[i, j])))
    rest = np.setdiff1d(np.arange(len(boxes)), picks)
    for i in rng.choice(rest, size=3, replace=False):                 # copies under another class
        rows.append((1, (clses[i] + 1 + rng.integers(2)) % 3, *boxes[i], rng.uniform(5, 60)))
    for _ in range(6):                                                # unmatched boxes anywhere
        c = rng.uniform((0, 0), size)
        h = rng.uniform(10, 80, 2)
        rows.append((1, rng.integers(3), c[0] - h[0], c[1] - h[1], c[0] + h[0], c[1] + h[1], rng.uniform(5, 60)))
    slots = rng.permutation(G)[:len(rows)]
    gt[:, 1:] = rng.uniform(0, 300, (G, 6))                           # garbage in the invalid slots
    gt[:, 1] = rng.integers(3, size=G)
    for s, r in zip(slots, rows):
        gt[s] = r
    for s in range(G):                                                # an invalid slot right on a detection's box
        if gt[s, 0] == 0:
            gt[s, 1:6] = (clses[0], *boxes[0])
            break
    return gt


def depth_inputs():
    """(heat, reg, targets) of the fixture: the maps of syn.make_head_logits(2, 80, 24) with the 2D box channels (0:4)
    scaled by 4 and the key-point channels (6:26) by 8. Unscaled, every key-point depth of this map clamps at 100 and
    the three key-point estimators are indistinguishable; scaled, they spread over the depth range."""
    cl, rgm = syn.make_head_logits(2, 80, 24)
    rgm[:, 0:4] *= 4
    rgm[:, 6:26] *= 8
    return torch.sigmoid(cl).clamp(1e-4, 1 - 1e-4), rgm, syn.make_targets(2, 80, 24)


def main():
    torch.set_num_threads(8)
    cfg = rs.reference_cfg(width=320, height=96)
    pp = rs.build_reference_model(cfg).eval().heads.post_processor
    heat, rgm, tg = depth_inputs()
    targets = ref_targets(tg)

    def run(b, method, thr):
        pp.output_depth, pp.det_threshold = method, thr
        with torch.no_grad():
            return pp({'cls': heat[b:b + 1].clone(), 'reg': rgm[b:b + 1].clone()}, targets[b:b + 1], test=True)

    rng = np.random.Generator(np.random.PCG64(31))
    out = {}
    for b in range(2):
        res0 = run(b, 'direct', 0.0)[0].numpy()
        boxes, clses = res0[:, 2:6].astype(np.float32), res0[:, 0]
        deps = np.stack([run(b, m, 0.0)[0].numpy()[:, 11] for m in SINGLE], 1).astype(np.float32)
        n_hi = run(b, 'direct', 0.2)[0].shape[0]
        for attempt in range(200):
            gt = make_gt(rng, boxes, clses, deps, n_hi, tg['size'][b])
            dec = decisions(boxes, clses, deps, gt)
            chosen = {e for e, _ in dec[:n_hi] if e >= 0}
            if all(ok for _, ok in dec) and chosen == {0, 1, 2, 3} and any(e < 0 for e, _ in dec[:n_hi]):
                break
        else:
            raise RuntimeError("no ground truth with safe margins for image %d" % b)
        print("image %d: attempt %d, estimator per detection %s" % (b, attempt, [e for e, _ in dec]))
        targets[b].add_field('reg_mask', torch.from_numpy((gt[:, 0] != 0).astype(np.uint8)))
        targets[b].add_field('cls_ids', torch.from_numpy(gt[:, 1].astype(np.int64)))
        targets[b].add_field('gt_bboxes', torch.from_numpy(gt[:, 2:6].copy()))
        locs = rng.uniform(-10, 10, (G, 3)).astype(np.float32)
        locs[:, 2] = gt[:, 6]
        targets[b].add_field('locations', torch.from_numpy(locs))
        out['gt_reg_mask_b%d' % b] = targets[b].get_field('reg_mask').numpy()
        out['gt_cls_ids_b%d' % b] = targets[b].get_field('cls_ids').numpy()
        out['gt_bboxes_b%d' % b] = targets[b].get_field('gt_bboxes').numpy()
        out['gt_locations_b%d' % b] = locs
        for m in METHODS:
            for thr in (0.0, 0.2):
                res, ev, vis = run(b, m, thr)
                tag = '%s_b%d_thr%s' % (m, b, thr)
                out['result_' + tag] = res.numpy()
                out['depth_err_' + tag] = ev['estimated_depth_error'].numpy()
                out['proj_' + tag] = vis['proj_center'].numpy()
    np.savez_compressed(os.path.join(OUT, "decode_depth.npz"), **out)
    print("decode_depth.npz", os.path.getsize(os.path.join(OUT, "decode_depth.npz")))


if __name__ == "__main__":
    main()
