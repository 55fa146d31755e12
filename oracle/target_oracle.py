"""TEST INFRASTRUCTURE ONLY (oracle) - CPU restatement of the training-target encoding of KITTIDataset.__getitem__
(data/datasets/kitti.py:126-179, 335-521) and its horizontal flip (data/augmentations/augmentations.py:28-77) for the
runs/monoflex.yaml configuration, working from the rows of monoflex_b200.targets.read_kitti_label. Pinned against the
unmodified reference by oracle/make_golden_targets.py -> tests/golden/kitti_targets.npz (tests/test_targets_host.py); the GPU
tests compare csrc/mf_targets.cu against it on random batches. Only tests and tools import this file.

numpy semantics it restates (numpy >= 2, NEP 50): a float32 scalar combined with a Python float stays float32, so the label
box branch (Object3d.box2d is float32) computes its filter, its centre and its gaussian_radius in float32; the projected-box
branch is float64. The border intersection of approx_proj_center is the closed form of the line through the two points where
the reference calls np.polyfit (the two differ in the last bits of a double)."""
import math

import numpy as np

from oracle import input_oracle as io

PI = np.pi
ALPHA_CENTERS = np.array([0, PI / 2, PI, -PI / 2])


def _wrap(a):
    while a > math.pi:
        a -= math.pi * 2
    while a < -math.pi:
        a += math.pi * 2
    return a


def _project(P, pts):
    hom = np.hstack((pts, np.ones((pts.shape[0], 1))))
    p = np.dot(hom, np.transpose(P))
    p[:, 0] /= p[:, 2]
    p[:, 1] /= p[:, 2]
    return p[:, 0:2]


def _gaussian_radius(height, width, min_overlap=0.7):
    r1 = ((height + width) + np.sqrt((height + width) ** 2 - 4 * 1 * (width * height * (1 - min_overlap) / (1 + min_overlap)))) / 2
    b2 = 2 * (height + width)
    r2 = (b2 + np.sqrt(b2 ** 2 - 4 * 4 * ((1 - min_overlap) * width * height))) / 2
    a3 = 4 * min_overlap
    b3 = -2 * min_overlap * (height + width)
    r3 = (b3 + np.sqrt(b3 ** 2 - 4 * a3 * ((min_overlap - 1) * width * height))) / 2
    return min(r1, r2, r3)


def _border_point(pc, c, img_w, img_h):
    """approx_proj_center: the nearest intersection of the line through pc and the box centre c with the image border, or
    None where the reference raises (c outside the image; the kernel also refuses a vertical line)."""
    if not (c[0] >= 0 and c[1] >= 0 and c[0] <= img_w - 1 and c[1] <= img_h - 1) or float(c[0]) == pc[0]:
        return None
    a = (float(c[1]) - pc[1]) / (float(c[0]) - pc[0])
    b = pc[1] - a * pc[0]
    cand = []
    if 0 <= b <= img_h - 1:
        cand.append((0.0, b))
    y = (img_w - 1) * a + b
    if 0 <= y <= img_h - 1:
        cand.append((float(img_w - 1), y))
    x = -b / a
    if 0 <= x <= img_w - 1:
        cand.append((x, 0.0))
    x = (img_h - 1 - b) / a
    if 0 <= x <= img_w - 1:
        cand.append((x, float(img_h - 1)))
    if not cand:
        return None
    cand = np.array(cand)
    d = np.sqrt((cand[:, 0] - pc[0]) ** 2 + (cand[:, 1] - pc[1]) ** 2)
    return cand[int(np.argmin(d))]


def encode_image(rows, P2, size, flip, W=1280, H=384, max_objs=40, down=4, ncls=3):
    """rows: float64 [n, 14] of read_kitti_label; P2 float64 [3, 4]; size (w, h); flip bool. Returns (fields, status): the
    reference's per-image target fields (without ori_img / calib: 'P2' is the flipped matrix) and the number of objects the
    reference would raise on (left out here)."""
    img_w, img_h = int(size[0]), int(size[1])
    P = np.array(P2, dtype=np.float64).reshape(3, 4).copy()
    if flip:
        P[0, 2] = img_w - P[0, 2] - 1
        P[0, 3] = -P[0, 3]
    pad = np.array([(W - img_w) // 2, (H - img_h) // 2])
    ow, oh = W // down, H // down
    x_min, y_min = int(np.ceil(pad[0] / down)), int(np.ceil(pad[1] / down))
    x_max, y_max = (pad[0] + img_w - 1) // down, (pad[1] + img_h - 1) // down
    f = dict(cls_ids=np.zeros(max_objs, np.int32), target_centers=np.zeros((max_objs, 2), np.int32),
             keypoints=np.zeros((max_objs, 10, 3), np.float32), keypoints_depth_mask=np.zeros((max_objs, 3), np.float32),
             dimensions=np.zeros((max_objs, 3), np.float32), locations=np.zeros((max_objs, 3), np.float32),
             reg_mask=np.zeros(max_objs, np.uint8), reg_weight=np.zeros(max_objs, np.float32),
             offset_3D=np.zeros((max_objs, 2), np.float32), bboxes=np.zeros((max_objs, 4), np.float32),
             rotys=np.zeros(max_objs, np.float32), trunc_mask=np.zeros(max_objs, np.uint8), alphas=np.zeros(max_objs, np.float32),
             orientations=np.zeros((max_objs, 8), np.float32), gt_bboxes=np.zeros((max_objs, 4), np.float32),
             occlusions=np.zeros(max_objs), truncations=np.zeros(max_objs), obj6=np.zeros((max_objs, 6), np.int32))
    status = 0
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 14)
    for i, r in enumerate(rows):
        cls, trunc, occ = int(r[0]), float(r[1]), float(r[2])
        xmin, ymin, xmax, ymax = (float(v) for v in r[3:7])
        h, w, l = (float(v) for v in r[7:10])
        t = r[10:13].astype(np.float32)
        ry = float(r[13])
        if flip:
            bw = xmax - xmin
            xmin = img_w - xmax - 1
            xmax = xmin + bw
            ry = _wrap((-math.pi - ry) if ry < 0 else (math.pi - ry))
            t[0] = -t[0]
        label_box = np.array([xmin, ymin, xmax, ymax], dtype=np.float32)
        alpha = _wrap(ry - math.atan2(t[0], t[2]))
        locs = t.copy()
        locs[1] = locs[1] - h / 2
        if locs[2] <= 0:
            continue
        R = np.array([[np.cos(ry), 0, np.sin(ry)], [0, 1, 0], [-np.sin(ry), 0, np.cos(ry)]])
        corners = np.dot(R, np.vstack([[l / 2, l / 2, -l / 2, -l / 2] * 2, [0, 0, 0, 0, -h, -h, -h, -h],
                                       [w / 2, -w / 2, -w / 2, w / 2] * 2])).T + t
        uv = _project(P, corners)
        pbox = np.array([uv[:, 0].min(), uv[:, 1].min(), uv[:, 0].max(), uv[:, 1].max()])
        inside_box = pbox[0] >= 0 and pbox[1] >= 0 and pbox[2] <= img_w - 1 and pbox[3] <= img_h - 1
        box = pbox.copy() if inside_box else label_box.copy()
        if trunc >= 0.9 and (box[2:] - box[:2]).min() <= 20:
            continue
        pc = _project(P, locs.reshape(-1, 3))[0]
        inside = (0 <= pc[0] <= img_w - 1) and (0 <= pc[1] <= img_h - 1)
        if inside:
            tp = pc.copy()
        else:
            tp = _border_point(pc, (box[:2] + box[2:]) / 2, img_w, img_h)
            if tp is None:
                status += 1
                continue
        kp3 = np.concatenate((corners, np.stack((corners[:4].mean(axis=0), corners[4:].mean(axis=0)))), axis=0)
        kp2 = _project(P, kp3)
        vis = (kp2[:, 0] >= 0) & (kp2[:, 0] <= img_w - 1) & (kp2[:, 1] >= 0) & (kp2[:, 1] <= img_h - 1) & (kp3[:, 2] > 0)
        vis = np.append(np.tile(vis[:4] | vis[4:8], 2), np.tile(vis[8] | vis[9], 2))
        kpd = np.array([vis[[8, 9]].all(), vis[[0, 2, 4, 6]].all(), vis[[1, 3, 5, 7]].all()], dtype=np.float32)
        kp2 = (kp2 + pad.reshape(1, 2)) / down
        tp = (tp + pad) / down
        pc = (pc + pad) / down
        box[0::2] += pad[0]
        box[1::2] += pad[1]
        box /= down
        dim = box[2:] - box[:2]
        tc = np.rint(tp).astype(np.int64)
        tc[0] = np.clip(tc[0], x_min, x_max)
        tc[1] = np.clip(tc[1], y_min, y_max)
        pred_2d = tc[0] >= box[0] and tc[1] >= box[1] and tc[0] <= box[2] and tc[1] <= box[3]
        if not ((dim > 0).all() and 0 <= tc[0] <= ow - 1 and 0 <= tc[1] <= oh - 1):
            continue
        if not inside:
            rx = max(0, int(min(tc[0] - box[0], box[2] - tc[0]) * 0.5))
            ryad = max(0, int(min(tc[1] - box[1], box[3] - tc[1]) * 0.5))
            if min(rx, ryad) != 0:
                status += 1
                continue
        else:
            rx = ryad = max(0, int(_gaussian_radius(dim[1], dim[0])))
        f["cls_ids"][i] = cls
        f["target_centers"][i] = tc
        f["offset_3D"][i] = pc - tc
        f["gt_bboxes"][i] = label_box
        if pred_2d:
            f["bboxes"][i] = box
        f["keypoints"][i] = np.concatenate((kp2 - tc.reshape(1, -1), vis[:, None].astype(np.float32)), axis=1)
        f["keypoints_depth_mask"][i] = kpd
        f["dimensions"][i] = np.array([l, h, w])
        f["locations"][i] = locs
        f["rotys"][i] = ry
        f["alphas"][i] = alpha
        off = alpha - ALPHA_CENTERS
        off[off > PI] -= 2 * PI
        off[off < -PI] += 2 * PI
        half = (2 * PI / 4) / 2 + (2 * PI / 4) * (1 / 6)
        for k in range(4):
            if abs(off[k]) < half:
                f["orientations"][i, k] = 1
                f["orientations"][i, k + 4] = off[k]
        f["reg_mask"][i] = 1
        f["reg_weight"][i] = 1
        f["trunc_mask"][i] = int(not inside)
        f["occlusions"][i] = occ
        f["truncations"][i] = trunc
        f["obj6"][i] = (1, cls, tc[0], tc[1], rx, ryad)
    f["hm"] = io.draw_heatmaps(f["obj6"][None], ncls, oh, ow)[0]
    f["pad_size"] = pad
    f["P2"] = P
    f["edge_indices"], f["edge_len"] = edge_indices((img_w, img_h), pad, W, H, down)
    return f, status


def edge_indices(size, pad, W, H, down=4):
    """get_edge_utils (kitti.py:126-179) zero-padded to 2 (W/4 + H/4) rows, and edge_len = count - 1 (kitti.py:280-285)."""
    img_w, img_h = size
    x_min, y_min = int(np.ceil(pad[0] / down)), int(np.ceil(pad[1] / down))
    x_max, y_max = (pad[0] + img_w - 1) // down, (pad[1] + img_h - 1) // down
    pts = ([(x_min, y) for y in range(y_min, y_max)] + [(x, y_max) for x in range(x_min, x_max)]
           + [(x_max, y) for y in range(y_max, y_min, -1)] + [(x, y_min) for x in range(x_max, x_min - 1, -1)])
    out = np.zeros((2 * (W // down + H // down), 2), dtype=np.int64)
    out[:len(pts)] = np.array(pts, dtype=np.int64).reshape(-1, 2)
    return out, len(pts) - 1


def encode_batch(labels, P2, sizes, flips, W=1280, H=384):
    """labels float64 [B, M, 16] (monoflex_b200.targets.pack_labels) -> dict of stacked fields, total status."""
    B, M = labels.shape[:2]
    outs, status = [], 0
    for b in range(B):
        rows = labels[b, labels[b, :, 0] != 0, 1:15]
        f, s = encode_image(rows, P2[b], sizes[b], bool(flips[b]), W, H, M)
        outs.append(f)
        status += s
    return {k: np.stack([o[k] for o in outs]) for k in outs[0]}, status
