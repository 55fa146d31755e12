"""CPU: the right-camera items of KITTIDataset (DATASETS.USE_RIGHT_IMAGE, runs/monoflex_right.yaml): the host half of the GPU
target encoding (monoflex_b200/targets.py) and oracle/target_oracle_right.py against the unmodified reference's
__getitem__ recorded in tests/golden/kitti_targets_right.npz (oracle/make_golden_targets_right.py)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from monoflex_b200 import targets as tg
from monoflex_b200.config import default_cfg
from oracle import target_oracle_right as tor

INT_FIELDS = ["cls_ids", "target_centers", "reg_mask", "trunc_mask", "pad_size", "edge_len", "edge_indices"]
FLOAT_FIELDS = ["keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_weight", "offset_3D", "rotys",
                "alphas", "orientations", "gt_bboxes", "2d_bboxes", "occlusions", "truncations", "hm"]


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "kitti_targets_right.npz")) as z:
        return {k: z[k] for k in z.files}


def right_cfg():
    cfg = default_cfg()
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    return cfg


def test_oracle_reproduces_reference_right_items(gold):
    """every field bit for bit, left and right items, flipped and not, in one batch"""
    f, status = tor.encode_batch(gold["rows_packed"], gold["P"], gold["sizes"], gold["flips"], gold["right"])
    assert status == 0
    f["2d_bboxes"] = f.pop("bboxes")
    for k in INT_FIELDS + FLOAT_FIELDS:
        assert np.array_equal(f[k], gold[k]), k
    assert np.array_equal(f["P2"], gold["P2_flipped"])


def test_fixture_covers_right_items(gold):
    right, flips, reg = gold["right"] == 1, gold["flips"] == 1, gold["reg_mask"] == 1
    n = int(gold["num_samples"])
    assert right.sum() == n and (gold["frame"][right] == np.arange(n)).all()
    for fl in (False, True):                                       # both flip branches carry right-view objects
        assert reg[right & (flips == fl)].sum() > 50
    assert (gold["trunc_mask"][right] == 1).sum() >= 20            # outside centres in the right view
    sz = gold["sizes"]
    assert (sz[right] != sz[~right]).any(-1).sum() >= 3            # right images of another size than their left one
    # the right view moves objects: same frame, same object, other boxes and centres
    assert not np.array_equal(gold["gt_bboxes"][right], gold["gt_bboxes"][~right])
    # P3's baseline b_x = P[0, 3] / -f_u is about +0.47 m (P2: about -0.06 m)
    P3 = gold["P3_parsed"]
    bx = P3[:, 0, 3] / -P3[:, 0, 0]
    assert (bx > 0.44).all() and (bx < 0.5).all()


def test_fixture_tells_float32_flip_from_float64(gold, monkeypatch):
    """The right item's flip runs on np.float32 scalars (numpy >= 2): a float64 flip of the same box gives other
    label boxes in the fixture, so the fixture pins the rounding."""
    def flip64(box, img_w):
        x1, y1, x2, y2 = (float(v) for v in box)
        w = x2 - x1
        x1 = img_w - x2 - 1
        return np.array([x1, y1, x1 + w, y2], dtype=np.float32)
    monkeypatch.setattr(tor, "flip_right_box", flip64)
    f, _ = tor.encode_batch(gold["rows_packed"], gold["P"], gold["sizes"], gold["flips"], gold["right"])
    assert (f["gt_bboxes"] != gold["gt_bboxes"]).any()


def test_right_view_box_ignores_label_box_columns(gold):
    rows = gold["rows_packed"][gold["right"] == 1]
    P, sizes = gold["P"][gold["right"] == 1], gold["sizes"][gold["right"] == 1]
    b = int(np.argmax(rows[:, :, 0].sum(1)))
    r = rows[b, 0, 1:15].copy()
    box = tor.right_view_box(r, P[b], sizes[b])
    r[3:7] = [-5.0, 1e4, 3.0, -7.0]
    assert np.array_equal(tor.right_view_box(r, P[b], sizes[b]), box)
    assert box.dtype == np.float32 and box[0] >= 0 and box[1] >= 0


def test_label_parser_reproduces_reference_objects(gold):
    rows = [tg.read_kitti_label(str(s).split("\n") if str(s) else []) for s in gold["labels"]]
    packed = tg.pack_labels(rows, 40)
    n = int(gold["num_samples"])
    assert np.array_equal(packed, gold["rows_packed"][:n]) and np.array_equal(packed, gold["rows_packed"][n:])


def test_calib_parser_right_camera(gold, tmp_path):
    for text, P2, P3 in zip(gold["calib_text"], gold["P2_parsed"], gold["P3_parsed"]):
        p = tmp_path / "calib.txt"
        p.write_text(str(text))
        assert np.array_equal(tg.read_kitti_calib(str(p), use_right_cam=True), P3)
        assert np.array_equal(tg.read_kitti_calib(str(p)), P2)
        assert np.array_equal(tg.read_kitti_calib(str(p), use_right_cam=False), P2)


def test_dataset_index_rule(gold):
    n = int(gold["num_samples"])
    cfg = right_cfg()
    assert tg.dataset_len(n, cfg) == int(gold["dataset_len"]) == 2 * n
    for idx in range(2 * n):
        assert tg.dataset_view(idx, n, cfg) == (int(gold["frame"][idx]), bool(gold["right"][idx]))
    for bad in (-1, 2 * n):
        with pytest.raises(IndexError):
            tg.dataset_view(bad, n, cfg)
    # USE_RIGHT_IMAGE & is_train: the test split and runs/monoflex.yaml have no right items
    assert tg.dataset_len(n, cfg, is_train=False) == n
    assert tg.dataset_len(n, default_cfg()) == n
    assert tg.dataset_view(n - 1, n, cfg, is_train=False) == (n - 1, False)
    with pytest.raises(IndexError):
        tg.dataset_view(n, n, default_cfg())


def test_encoder_accepts_right_image_config():
    """GpuTargetEncoder(cfg) serves runs/monoflex_right.yaml; the left-view check of a cfg still refuses it, and every
    other option other than runs/monoflex.yaml's still raises with right views on"""
    tg.GpuTargetEncoder(right_cfg())
    tg.GpuTargetEncoder(default_cfg())
    tg.GpuTargetEncoder._check_config(right_cfg(), right_views=True)
    tg.GpuTargetEncoder._check_config(default_cfg(), right_views=True)
    with pytest.raises(NotImplementedError):
        tg.GpuTargetEncoder._check_config(right_cfg())
    for node, key, value in (("INPUT", "HEATMAP_CENTER", '2D'), ("INPUT", "ORIENTATION", 'head-axis'),
                             ("DATASETS", "FILTER_ANNOS", [0.8, 20]), ("DATASETS", "USE_RIGHT_IMAGE", 'both')):
        cfg = right_cfg()
        setattr(getattr(cfg, node), key, value)
        with pytest.raises(NotImplementedError):
            tg.GpuTargetEncoder(cfg)
        with pytest.raises(NotImplementedError):
            tg.GpuTargetEncoder._check_config(cfg, right_views=True)
