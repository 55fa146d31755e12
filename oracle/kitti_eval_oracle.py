"""TEST INFRASTRUCTURE ONLY — float64 CPU restatement of the KITTI official metric of monoflex_b200/evaluation.py
(kitti_object_eval_python/eval.py of the reference), pinned to tests/golden/kitti_eval.npz and kitti_eval_edges.npz.

`eval_tables(gt, dt, classes)` takes the same KittiAnnos rows as evaluation.eval_tables and returns what it returns:
(tables, overlaps [3, n_pair]). The two halves are separate so the statistics can be fed the overlaps the kernel
computed and compared with its tables exactly:
  overlaps    2D: image_box_overlap in float64 in the kernel's operation order (equal bit for bit). BEV / 3D: the
              float32 corners of both boxes (as rotate_iou builds them) intersected EXACTLY with iou3d_oracle.ExactPolygon
              and rounded once to float64, then the reference's float32 / float64 mix of the IoU ratio and d3_box_overlap.
  statistics  clean_data, the compute_fp=False pass, get_thresholds, the compute_fp=True pass with the DontCare
              suppression and the AOS similarity (summed in ground-truth order per image, images in order, nothing
              added for an image without tp and fp), recall / precision / AOS with NaN-propagating suffix maxima, and the
              R40 / R11 sums. Both passes run for all configurations of one metric at once (numpy rows), the second
              pass for every (configuration, threshold) row, so 400 images x 3 classes take seconds.

`flip` names one matching rule to get wrong on purpose (FLIPS); the suite uses it to show that its fixtures can tell."""
import math

import numpy as np

from oracle.iou3d_oracle import ExactPolygon

NPTS = 41
DONTCARE = 6
MIN_HEIGHT = (40.0, 25.0, 25.0)
MAX_OCCLUSION = (0.0, 1.0, 2.0)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
# min_overlaps[k, metric, class] of get_official_eval_result
MIN_OVERLAPS = np.array([[[0.7, 0.5, 0.5, 0.7, 0.5, 0.7]] * 3,
                         [[0.7, 0.5, 0.5, 0.7, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5],
                          [0.5, 0.25, 0.25, 0.5, 0.25, 0.5]]])
# one rule each, wrong: `>=` on min_overlap; the last of equal scores (first pass) / overlaps (second pass) wins;
# ground truth ignored below MIN_HEIGHT only (`<`); detections ignored at MIN_HEIGHT too (`<=`); DontCare with `>=`
FLIPS = ("overlap_ge", "score_last", "overlap_last", "gt_height_lt", "dt_height_le", "dontcare_ge")
# object columns (include/monoflex_b200.h)
C_CLS, C_TRUNC, C_OCC, C_ALPHA, C_X1, C_Y1, C_X2, C_Y2, C_L, C_H, C_W, C_X, C_Y, C_Z, C_RY, C_SCORE = range(16)


def _rows(a):
    """(objects [N, 16] float64 numpy, offsets [n_img + 1]) of a KittiAnnos"""
    obj = a.objects.detach().cpu().numpy().astype(np.float64, copy=False)
    off = np.zeros(len(a.counts) + 1, np.int64)
    np.cumsum(a.counts, out=off[1:])
    return obj, off


def pair_offsets(gcount, dcount):
    pairs = np.asarray(gcount, np.int64) * np.asarray(dcount, np.int64)
    return np.concatenate([[0], np.cumsum(pairs)])


# ---------------------------------------------------------------------------------------------------------- overlaps
def box_overlap(D, G, iou):
    """image_box_overlap of D [nd, 4] against G [ng, 4] -> [nd, ng]: criterion -1 (IoU) or 0 (over D's area); Python's
    min / max keep the first argument unless the second is strictly smaller / larger"""
    b, q = D[:, None, :], G[None, :, :]
    iw = np.where(q[..., 2] < b[..., 2], q[..., 2], b[..., 2]) - np.where(q[..., 0] > b[..., 0], q[..., 0], b[..., 0])
    ih = np.where(q[..., 3] < b[..., 3], q[..., 3], b[..., 3]) - np.where(q[..., 1] > b[..., 1], q[..., 1], b[..., 1])
    barea = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    inter = iw * ih
    ua = (barea + (q[..., 2] - q[..., 0]) * (q[..., 3] - q[..., 1])) - inter if iou else np.broadcast_to(barea, inter.shape)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = inter / ua
    return np.where((iw > 0) & (ih > 0), r, 0.0)


def bev_corners(x, z, l, w, ry):
    """rotate_iou's rbbox_to_corners in float32: cos / sin of the float32 angle rounded to float32"""
    f = np.float32
    x, z, l, w, ry = f(x), f(z), f(l), f(w), f(ry)
    ca, sa = f(math.cos(float(ry))), f(math.sin(float(ry)))
    cx = (-l / f(2), -l / f(2), l / f(2), l / f(2))
    cy = (-w / f(2), w / f(2), w / f(2), -w / f(2))
    return np.array([[(ca * cx[i] + sa * cy[i]) + x, (-sa * cx[i] + ca * cy[i]) + z] for i in range(4)], np.float32)


def bev_inter(a, b):
    """exact intersection area of the float32 corner rings of two BEV boxes (x, z, l, w, ry), rounded once"""
    ca, cb = bev_corners(*a), bev_corners(*b)
    # disjoint bounding boxes cannot overlap; skip the exact clip
    if (ca[:, 0].max() < cb[:, 0].min() or cb[:, 0].max() < ca[:, 0].min() or ca[:, 1].max() < cb[:, 1].min()
            or cb[:, 1].max() < ca[:, 1].min()):
        return 0.0
    pa, pb = ExactPolygon(ca.astype(np.float64)), ExactPolygon(cb.astype(np.float64))
    if not (pa.is_valid and pb.is_valid):
        return 0.0
    return pa.intersection(pb).area


def pair_overlaps(D, G):
    """BEV and 3D overlaps of one detection row and one ground-truth row (the kernel's evaluation of rotate_iou and
    d3_box_overlap with the intersection area exact)"""
    f = np.float32
    rg = (G[C_X], G[C_Z], G[C_L], G[C_W], G[C_RY])
    rd = (D[C_X], D[C_Z], D[C_L], D[C_W], D[C_RY])
    inter = bev_inter(rg, rd)
    area_sum = f(f(rg[2]) * f(rg[3])) + f(f(rd[2]) * f(rd[3]))
    with np.errstate(invalid="ignore", divide="ignore"):
        bev = float(f(np.float64(inter) / (np.float64(area_sum) - inter)))
    rinc = f(inter)
    r3 = float(rinc)
    if rinc > 0:
        iw = min(D[C_Y], G[C_Y]) - max(D[C_Y] - D[C_H], G[C_Y] - G[C_H])
        if iw > 0:
            a1 = D[C_L] * D[C_H] * D[C_W]
            a2 = G[C_L] * G[C_H] * G[C_W]
            inc = iw * float(rinc)
            r3 = float(f(inc / ((a1 + a2) - inc)))
        else:
            r3 = 0.0
    return bev, r3


def overlaps(gt, dt):
    """[3, n_pair] float64, image i's block at pair_off[i] as [nd, ng] row-major: calculate_iou_partly(dt, gt, metric)"""
    G, goff = _rows(gt)
    D, doff = _rows(dt)
    poff = pair_offsets(np.diff(goff), np.diff(doff))
    out = np.zeros((3, int(poff[-1])))
    for i in range(len(goff) - 1):
        gi, di = G[goff[i]:goff[i + 1]], D[doff[i]:doff[i + 1]]
        if len(gi) == 0 or len(di) == 0:
            continue
        out[0, poff[i]:poff[i + 1]] = box_overlap(di[:, C_X1:C_Y2 + 1], gi[:, C_X1:C_Y2 + 1], True).reshape(-1)
        b = [pair_overlaps(d, g) for d in di for g in gi]
        out[1, poff[i]:poff[i + 1]] = [v[0] for v in b]
        out[2, poff[i]:poff[i + 1]] = [v[1] for v in b]
    return out


# -------------------------------------------------------------------------------------------------------- statistics
def clean_flags(G, D, classes, flip=None):
    """clean_data for every (class, difficulty): fg [ncls, 3, n_gt], fd [ncls, 3, n_dt] in {-1, 0, 1}"""
    gcode, dcode = G[:, C_CLS].astype(np.int64), D[:, C_CLS].astype(np.int64)
    gh = G[:, C_Y2] - G[:, C_Y1]
    dh = np.abs(D[:, C_Y2] - D[:, C_Y1])
    fg = np.empty((len(classes), 3, len(G)), np.int8)
    fd = np.empty((len(classes), 3, len(D)), np.int8)
    for m, cls in enumerate(classes):
        valid = np.where(gcode == cls, 1, np.where(((cls == 1) & (gcode == 4)) | ((cls == 0) & (gcode == 3)), 0, -1))
        for l in range(3):
            low = gh < MIN_HEIGHT[l] if flip == "gt_height_lt" else gh <= MIN_HEIGHT[l]
            ignore = (G[:, C_OCC] > MAX_OCCLUSION[l]) | (G[:, C_TRUNC] > MAX_TRUNCATION[l]) | low
            fg[m, l] = np.where((valid == 1) & ~ignore, 0, np.where((valid == 0) | (ignore & (valid == 1)), 1, -1))
            small = dh <= MIN_HEIGHT[l] if flip == "dt_height_le" else dh < MIN_HEIGHT[l]
            fd[m, l] = np.where(small, 1, np.where(dcode == cls, 0, -1))
    return fg, fd


def get_thresholds(scores, num_gt):
    """get_thresholds on the true-positive scores, with the kernel's cap of N_SAMPLE_PTS values"""
    s = np.sort(np.asarray(scores, np.float64))[::-1]
    n, current, out = len(s), 0.0, []
    for i in range(n):
        l_recall = (i + 1) / num_gt
        r_recall = (i + 2) / num_gt if i < n - 1 else l_recall
        if (r_recall - current) < (current - l_recall) and i < n - 1:
            continue
        if len(out) < NPTS:
            out.append(s[i])
        current += 1 / (NPTS - 1.0)
    return out


def _first_max(v, last):
    """index of the first (or last) maximum along axis 1"""
    if last:
        return v.shape[1] - 1 - np.argmax(v[:, ::-1], axis=1)
    return np.argmax(v, axis=1)


def _gt_over(ov, mo, flip):
    return ov >= mo if flip == "overlap_ge" else ov > mo


def first_pass(ov_img, fg, fd, scores, mo, flip):
    """compute_statistics_jit(compute_fp=False) for rows of configurations of one image: fg [R, ng], fd [R, nd],
    mo [R, 1], ov_img [nd, ng]. Returns a list per row of the true-positive scores in order."""
    R, ng = fg.shape
    nd = fd.shape[1]
    assigned = np.zeros((R, nd), bool)
    out = [[] for _ in range(R)]
    rows = np.arange(R)
    for g in range(ng):
        live = fg[:, g] != -1
        if not live.any() or nd == 0:
            continue
        cand = (fd != -1) & ~assigned & _gt_over(ov_img[:, g][None, :], mo, flip) & live[:, None]
        # s > valid from valid = -1e7: the first (last, when flipped) of the highest scores
        s = np.where(cand, scores[None, :], -np.inf)
        det = _first_max(s, flip == "score_last")
        found = cand.any(1)
        for r in np.nonzero(found & (fg[:, g] == 0) & (fd[rows, det] != 1))[0]:
            out[r].append(scores[det[r]])
        assigned[rows[found], det[found]] = True
    return out


def second_pass(ov_img, dc_ov, fg, fd, scores, galpha, dalpha, mo, thresh, metric, aos, flip):
    """compute_statistics_jit(compute_fp=True) of one image for rows of (configuration, threshold): tp, fp, fn [R] and
    the similarity [R] (NaN where the reference's -1 is not added)"""
    R, ng = fg.shape
    nd = fd.shape[1]
    tp, fn = np.zeros(R, np.int64), np.zeros(R, np.int64)
    sim = np.zeros(R)
    below = scores[None, :] < thresh[:, None]
    assigned = np.zeros((R, nd), bool)
    rows = np.arange(R)
    for g in range(ng):
        live = fg[:, g] != -1
        if not live.any():
            continue
        if nd:
            elig = (fd != -1) & ~assigned & ~below & _gt_over(ov_img[:, g][None, :], mo, flip) & live[:, None]
            m0, m1 = elig & (fd == 0), elig & (fd == 1)
            # every eligible overlap exceeds min_overlap > 0 = the initial max_overlap, so the first (last, when
            # flipped) largest overlap of a kept detection wins; else the first ignored detection
            d0 = _first_max(np.where(m0, ov_img[:, g][None, :], -np.inf), flip == "overlap_last")
            has0, has1 = m0.any(1), m1.any(1)
            det = np.where(has0, d0, np.argmax(m1, axis=1))
            found = has0 | has1
        else:
            det, found = np.zeros(R, np.int64), np.zeros(R, bool)
        fn += live & ~found & (fg[:, g] == 0)
        hit = live & found & (fg[:, g] == 0)
        if nd:
            hit &= fd[rows, det] != 1
        tp += hit
        if aos and hit.any():
            sim = np.where(hit, sim + (1.0 + np.cos(galpha[g] - dalpha[det])) / 2.0, sim)
        live_found = live & found
        assigned[rows[live_found], det[live_found]] = True
    fp = (~assigned & (fd == 0) & ~below).sum(1)
    if metric == 0:
        for q in range(dc_ov.shape[1]):
            cand = ~assigned & (fd == 0) & ~below
            cand &= (dc_ov[:, q][None, :] >= mo) if flip == "dontcare_ge" else (dc_ov[:, q][None, :] > mo)
            fp -= cand.sum(1)
            assigned |= cand
    sim = np.where((tp > 0) | (fp > 0), sim, np.nan)
    return tp, fp, fn, sim


def statistics(gt, dt, classes, ov, flip=None):
    """the tables of evaluation.eval_tables from given overlaps [3, n_pair] (the kernel's, or overlaps())"""
    assert flip is None or flip in FLIPS, flip
    G, goff = _rows(gt)
    D, doff = _rows(dt)
    n_img, ncls = len(goff) - 1, len(classes)
    assert len(doff) - 1 == n_img and n_img > 0
    assert np.diff(doff).max(initial=0) <= 128, "the kernel refuses images of more than 128 detections"
    ov = np.asarray(ov, np.float64)
    poff = pair_offsets(np.diff(goff), np.diff(doff))
    fg, fd = clean_flags(G, D, classes, flip)
    num_valid = (fg == 0).sum(2)                                              # [ncls, 3]
    compute_aos = len(D) > 0 and D[0, C_ALPHA] != -10.0
    dc = [np.nonzero(G[goff[i]:goff[i + 1], C_CLS] == DONTCARE)[0] for i in range(n_img)]
    dc_ov = [box_overlap(D[doff[i]:doff[i + 1], C_X1:C_Y2 + 1], G[goff[i] + dc[i]][:, C_X1:C_Y2 + 1], False)
             for i in range(n_img)]
    shape = (3, ncls, 3, 2, NPTS)
    rec, prec, ori = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    thresholds = np.full((3, ncls, 3, 2, NPTS), np.nan)
    # rows of one metric: (m, l, k)
    cfg = [(m, l, k) for m in range(ncls) for l in range(3) for k in range(2)]
    for metric in range(3):
        aos = metric == 0 and compute_aos
        mo = np.array([MIN_OVERLAPS[k, metric, classes[m]] for m, l, k in cfg])[:, None]
        blocks = [ov[metric, poff[i]:poff[i + 1]].reshape(doff[i + 1] - doff[i], goff[i + 1] - goff[i])
                  for i in range(n_img)]
        tps = [[] for _ in cfg]
        for i in range(n_img):
            fgi = np.stack([fg[m, l, goff[i]:goff[i + 1]] for m, l, k in cfg])
            fdi = np.stack([fd[m, l, doff[i]:doff[i + 1]] for m, l, k in cfg])
            for r, s in enumerate(first_pass(blocks[i], fgi, fdi, D[doff[i]:doff[i + 1], C_SCORE], mo, flip)):
                tps[r] += s
        thr = [get_thresholds(tps[r], num_valid[m, l]) for r, (m, l, k) in enumerate(cfg)]
        # second-pass rows (configuration, threshold); thresholds past a configuration's count are +inf (inactive)
        T = np.full((len(cfg), NPTS), np.inf)
        for r, t in enumerate(thr):
            T[r, :len(t)] = t
        rr = np.repeat(np.arange(len(cfg)), NPTS)
        mo2, T2 = mo[rr], T.reshape(-1)
        pr = np.zeros((len(rr), 4))
        for i in range(n_img):
            fgi = np.stack([fg[m, l, goff[i]:goff[i + 1]] for m, l, k in cfg])[rr]
            fdi = np.stack([fd[m, l, doff[i]:doff[i + 1]] for m, l, k in cfg])[rr]
            tp, fp, fn, sim = second_pass(blocks[i], dc_ov[i], fgi, fdi, D[doff[i]:doff[i + 1], C_SCORE],
                                          G[goff[i]:goff[i + 1], C_ALPHA], D[doff[i]:doff[i + 1], C_ALPHA], mo2, T2,
                                          metric, aos, flip)
            pr[:, 0] += tp
            pr[:, 1] += fp
            pr[:, 2] += fn
            if aos:
                pr[:, 3] = np.where(np.isnan(sim), pr[:, 3], pr[:, 3] + sim)
        pr = pr.reshape(len(cfg), NPTS, 4)
        with np.errstate(invalid="ignore", divide="ignore"):
            r_, p_ = pr[..., 0] / (pr[..., 0] + pr[..., 2]), pr[..., 0] / (pr[..., 0] + pr[..., 1])
            o_ = pr[..., 3] / (pr[..., 0] + pr[..., 1]) if aos else np.zeros_like(r_)
        for r, (m, l, k) in enumerate(cfg):
            n = len(thr[r])
            thresholds[metric, m, l, k, :n] = thr[r]
            for tab, v in ((rec, r_), (prec, p_), (ori, o_)):
                x = np.zeros(NPTS)
                x[:n] = v[r, :n]
                # suffix maximum; np.maximum propagates NaN like np.max
                tab[metric, m, l, k] = np.maximum.accumulate(x[::-1])[::-1]
    ap = np.zeros((2, 4, ncls, 3, 2))
    for metric, tab in ((0, prec), (1, prec), (2, prec), (3, ori)):
        t = tab[0 if metric == 3 else metric]
        s40, s11 = 0.0, 0.0
        for i in range(1, NPTS):
            s40 = s40 + t[..., i]
        for i in range(0, NPTS, 4):
            s11 = s11 + t[..., i]
        ap[0, metric], ap[1, metric] = s40 / 40 * 100, s11 / 11 * 100
    return {"recall": rec, "precision": prec, "orientation": ori, "ap": ap, "compute_aos": bool(compute_aos),
            "thresholds": thresholds}


def float32_tolerance(gt, dt):
    """[n_pair] bound on |BEV / 3D overlap of the reference's float32 clipping - the exact one|: its segment
    intersections are determinants of corner coordinates, so their error grows with the coordinates' squares s^2 and the
    overlap's with 1 / the smaller footprint a. 16 eps32 s^2 / a is twice the largest ratio on tests/golden/kitti_eval.npz
    (pedestrians at z = 50 differ by 3e-4)."""
    G, goff = _rows(gt)
    D, doff = _rows(dt)
    out = []
    for i in range(len(goff) - 1):
        gi, di = G[goff[i]:goff[i + 1]], D[doff[i]:doff[i + 1]]
        s = np.maximum(np.abs(di[:, [C_X, C_Z]]).max(1)[:, None], np.abs(gi[:, [C_X, C_Z]]).max(1)[None, :])
        a = np.minimum(np.abs(di[:, C_L] * di[:, C_W])[:, None], np.abs(gi[:, C_L] * gi[:, C_W])[None, :])
        out.append((1e-6 + 16 * 2.0 ** -23 * s ** 2 / np.maximum(a, 1e-3)).reshape(-1))
    return np.concatenate(out) if out else np.zeros(0)


def eval_tables(gt, dt, classes, flip=None):
    """(tables, overlaps) as evaluation.eval_tables returns them, from the oracle's own overlaps"""
    ov = overlaps(gt, dt)
    return statistics(gt, dt, classes, ov, flip), ov
