"""TEST INFRASTRUCTURE ONLY (oracle) - the right-camera items of KITTIDataset.__getitem__ (DATASETS.USE_RIGHT_IMAGE,
runs/monoflex_right.yaml; data/datasets/kitti.py:232-252) on top of oracle/target_oracle.py, which restates the left items
and the encoding both share. Pinned against the unmodified reference by oracle/make_golden_targets_right.py ->
tests/golden/kitti_targets_right.npz (tests/test_targets_right_host.py); the GPU tests compare csrc/mf_targets.cu against it on
random batches that mix left and right items. Only tests and tools import this file.

A right item differs from a left one before the class filter and the flip:
  1. P is the calibration's P3;
  2. every label's 2D box is replaced by the extent of its eight corners projected with the unflipped P3, clamped with
     Python's max(x, 0) / min(x, img - 1) and stored as np.float32 (Object3d.box2d and its elements);
  3. the flip then works on those np.float32 scalars: under numpy >= 2 (NEP 50) `img_w - xmax - 1` and `xmin + w` stay
     float32, where a left item's Python floats are float64.
Everything after that is the left encoding with P3 in place of P2, so the right item is handed to
target_oracle.encode_image already flipped (P, ry, tx and the float32 box exactly as the flip leaves them) with flip=False."""
import math

import numpy as np

from oracle import target_oracle as to


def right_view_box(row, P3, size):
    """kitti.py:243-249 for one read_kitti_label row: the float32 [4] box from generate_corners3d projected with P3."""
    h, w, l = (float(v) for v in row[7:10])
    t = np.asarray(row[10:13]).astype(np.float32)
    ry = float(row[13])
    R = np.array([[np.cos(ry), 0, np.sin(ry)], [0, 1, 0], [-np.sin(ry), 0, np.cos(ry)]])
    corners = np.dot(R, np.vstack([[l / 2, l / 2, -l / 2, -l / 2] * 2, [0, 0, 0, 0, -h, -h, -h, -h],
                                   [w / 2, -w / 2, -w / 2, w / 2] * 2])).T + t
    uv = to._project(np.asarray(P3, dtype=np.float64).reshape(3, 4), corners)
    img_w, img_h = int(size[0]), int(size[1])
    return np.array([max(uv[:, 0].min(), 0), max(uv[:, 1].min(), 0), min(uv[:, 0].max(), img_w - 1),
                     min(uv[:, 1].max(), img_h - 1)], dtype=np.float32)


def flip_right_box(box, img_w):
    """augmentations.py:42-45 on np.float32 scalars, written out in float32 (what numpy >= 2 computes)."""
    xmin, ymin, xmax, ymax = (np.float32(v) for v in box)
    w = np.float32(xmax - xmin)
    xmin = np.float32(np.float32(np.float32(img_w) - xmax) - np.float32(1))
    xmax = np.float32(xmin + w)
    return np.array([xmin, ymin, xmax, ymax], dtype=np.float32)


def encode_image(rows, P2, size, flip, right=False, W=1280, H=384, max_objs=40, down=4, ncls=3):
    """target_oracle.encode_image with right: for a right item P2 is the calibration's P3 and size the right image's; the
    rows' box columns are not read. Returns (fields, status); fields['P2'] is the flipped P3."""
    if not right:
        return to.encode_image(rows, P2, size, flip, W, H, max_objs, down, ncls)
    img_w = int(size[0])
    P = np.array(P2, dtype=np.float64).reshape(3, 4).copy()
    rows = np.array(rows, dtype=np.float64).reshape(-1, 14)
    for r in rows:
        box = right_view_box(r, P, size)
        if flip:
            box = flip_right_box(box, img_w)
            r[13] = to._wrap((-math.pi - r[13]) if r[13] < 0 else (math.pi - r[13]))
            r[10] = -r[10]
        r[3:7] = box
    if flip:
        P[0, 2] = img_w - P[0, 2] - 1
        P[0, 3] = -P[0, 3]
    return to.encode_image(rows, P, size, False, W, H, max_objs, down, ncls)


def encode_batch(labels, P2, sizes, flips, right=None, W=1280, H=384):
    """target_oracle.encode_batch with per-image right flags (None: all left)."""
    B, M = labels.shape[:2]
    right = np.zeros(B, dtype=bool) if right is None else np.asarray(right).astype(bool)
    outs, status = [], 0
    for b in range(B):
        rows = labels[b, labels[b, :, 0] != 0, 1:15]
        f, s = encode_image(rows, P2[b], sizes[b], bool(flips[b]), bool(right[b]), W, H, M)
        outs.append(f)
        status += s
    return {k: np.stack([o[k] for o in outs]) for k in outs[0]}, status
