"""TEST INFRASTRUCTURE ONLY — the float64 KITTI-metric oracle of oracle/kitti_eval_oracle.py over any table of overlap
thresholds, as evaluation.eval_tables(..., min_overlaps=table) computes it; pinned to tests/golden/kitti_coco.npz with
get_coco_eval_result's ten-set table.

`statistics(gt, dt, classes, ov, min_overlaps)` takes eval_class's table [n_sets][3 metric][ncls] (by class position, as
the kernel does) and returns kitti_eval_oracle.statistics' tables with an overlap-set axis of length n_sets. It runs the
same clean_data flags, compute_statistics passes, get_thresholds and AP sums: kitti_eval_oracle's functions, with the
configuration rows (class, difficulty, set) of one metric read from the table instead of the official two sets."""
import numpy as np

from oracle import kitti_eval_oracle as K


def statistics(gt, dt, classes, ov, min_overlaps):
    """the tables of evaluation.eval_tables(gt, dt, classes, min_overlaps=min_overlaps) from given overlaps [3, n_pair]"""
    table = np.asarray(min_overlaps, np.float64)
    n_sets, ncls = table.shape[0], len(classes)
    assert table.shape == (n_sets, 3, ncls) and n_sets > 0, table.shape
    G, goff = K._rows(gt)
    D, doff = K._rows(dt)
    n_img = len(goff) - 1
    assert len(doff) - 1 == n_img and n_img > 0
    assert np.diff(doff).max(initial=0) <= 128, "the kernel refuses images of more than 128 detections"
    ov = np.asarray(ov, np.float64)
    poff = K.pair_offsets(np.diff(goff), np.diff(doff))
    fg, fd = K.clean_flags(G, D, classes)
    num_valid = (fg == 0).sum(2)                                              # [ncls, 3]
    compute_aos = len(D) > 0 and D[0, K.C_ALPHA] != -10.0
    dc = [np.nonzero(G[goff[i]:goff[i + 1], K.C_CLS] == K.DONTCARE)[0] for i in range(n_img)]
    dc_ov = [K.box_overlap(D[doff[i]:doff[i + 1], K.C_X1:K.C_Y2 + 1], G[goff[i] + dc[i]][:, K.C_X1:K.C_Y2 + 1], False)
             for i in range(n_img)]
    shape = (3, ncls, 3, n_sets, K.NPTS)
    rec, prec, ori = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    thresholds = np.full(shape, np.nan)
    cfg = [(m, l, k) for m in range(ncls) for l in range(3) for k in range(n_sets)]    # rows of one metric
    for metric in range(3):
        aos = metric == 0 and compute_aos
        mo = np.array([table[k, metric, m] for m, l, k in cfg])[:, None]
        blocks = [ov[metric, poff[i]:poff[i + 1]].reshape(doff[i + 1] - doff[i], goff[i + 1] - goff[i])
                  for i in range(n_img)]
        flags = [(np.stack([fg[m, l, goff[i]:goff[i + 1]] for m, l, k in cfg]),
                  np.stack([fd[m, l, doff[i]:doff[i + 1]] for m, l, k in cfg])) for i in range(n_img)]
        tps = [[] for _ in cfg]
        for i in range(n_img):
            for r, s in enumerate(K.first_pass(blocks[i], *flags[i], D[doff[i]:doff[i + 1], K.C_SCORE], mo, None)):
                tps[r] += s
        thr = [K.get_thresholds(tps[r], num_valid[m, l]) for r, (m, l, k) in enumerate(cfg)]
        # second-pass rows (configuration, threshold); thresholds past a configuration's count are +inf (inactive)
        T = np.full((len(cfg), K.NPTS), np.inf)
        for r, t in enumerate(thr):
            T[r, :len(t)] = t
        rr = np.repeat(np.arange(len(cfg)), K.NPTS)
        pr = np.zeros((len(rr), 4))
        for i in range(n_img):
            tp, fp, fn, sim = K.second_pass(blocks[i], dc_ov[i], flags[i][0][rr], flags[i][1][rr],
                                            D[doff[i]:doff[i + 1], K.C_SCORE], G[goff[i]:goff[i + 1], K.C_ALPHA],
                                            D[doff[i]:doff[i + 1], K.C_ALPHA], mo[rr], T.reshape(-1), metric, aos, None)
            pr[:, 0] += tp
            pr[:, 1] += fp
            pr[:, 2] += fn
            if aos:
                pr[:, 3] = np.where(np.isnan(sim), pr[:, 3], pr[:, 3] + sim)
        pr = pr.reshape(len(cfg), K.NPTS, 4)
        with np.errstate(invalid="ignore", divide="ignore"):
            r_, p_ = pr[..., 0] / (pr[..., 0] + pr[..., 2]), pr[..., 0] / (pr[..., 0] + pr[..., 1])
            o_ = pr[..., 3] / (pr[..., 0] + pr[..., 1]) if aos else np.zeros_like(r_)
        for r, (m, l, k) in enumerate(cfg):
            n = len(thr[r])
            thresholds[metric, m, l, k, :n] = thr[r]
            for tab, v in ((rec, r_), (prec, p_), (ori, o_)):
                x = np.zeros(K.NPTS)
                x[:n] = v[r, :n]
                tab[metric, m, l, k] = np.maximum.accumulate(x[::-1])[::-1]        # NaN-propagating suffix maximum
    ap = np.zeros((2, 4, ncls, 3, n_sets))
    for metric, tab in ((0, prec), (1, prec), (2, prec), (3, ori)):
        t = tab[0 if metric == 3 else metric]
        s40, s11 = 0.0, 0.0
        for i in range(1, K.NPTS):
            s40 = s40 + t[..., i]
        for i in range(0, K.NPTS, 4):
            s11 = s11 + t[..., i]
        ap[0, metric], ap[1, metric] = s40 / 40 * 100, s11 / 11 * 100
    return {"recall": rec, "precision": prec, "orientation": ori, "ap": ap, "compute_aos": bool(compute_aos),
            "thresholds": thresholds}
