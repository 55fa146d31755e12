"""CPU: the host half of the GPU target encoding (monoflex_b200/targets.py) and the target oracle against the unmodified
reference's KITTIDataset.__getitem__ recorded in tests/golden/kitti_targets.npz (oracle/make_golden_targets.py)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from monoflex_b200 import targets as tg
from monoflex_b200.config import default_cfg
from oracle import target_oracle as to

INT_FIELDS = ["cls_ids", "target_centers", "reg_mask", "trunc_mask", "pad_size", "edge_len", "edge_indices"]
FLOAT_FIELDS = ["keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_weight", "offset_3D", "rotys",
                "alphas", "orientations", "gt_bboxes", "occlusions", "truncations"]


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "kitti_targets.npz")) as z:
        return {k: z[k] for k in z.files}


def ulp32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_label_parser_reproduces_reference_objects(gold):
    rows = [tg.read_kitti_label(str(s).split("\n") if str(s) else []) for s in gold["train_labels"]]
    packed = tg.pack_labels(rows, 40)
    assert np.array_equal(packed, gold["rows_packed"])            # bit for bit, float32 location rounding included


def test_calib_parser(gold, tmp_path):
    for text, P in zip(gold["train_calib_text"], gold["train_P2"]):
        p = tmp_path / "calib.txt"
        p.write_text(str(text))
        assert np.array_equal(tg.read_kitti_calib(str(p)), P)


def test_pack_labels_limits():
    row = np.zeros((41, 14))
    with pytest.raises(ValueError):
        tg.pack_labels([row], 40)
    out = tg.pack_labels([row[:3], row[:0]], 40)
    assert out.shape == (2, 40, 16) and out[0, :, 0].sum() == 3 and out[1].sum() == 0


def test_fixture_covers_the_branches(gold):
    lab = gold["rows_packed"]
    present = lab[..., 0] == 1
    reg = gold["train_reg_mask"] == 1
    flips = gold["train_flips"]
    assert set(flips.tolist()) == {0, 1}
    assert (present & ~reg).any()                                 # skipped objects leave slot holes
    assert (lab[..., 13][present] <= 0).any()                     # behind the camera
    assert (gold["train_trunc_mask"] == 1).sum() >= 20            # outside centres
    assert ((gold["train_2d_bboxes"] == 0).all(-1) & reg).any()   # pred_2D = False
    assert present.sum(1).max() == 40 and present.sum(1).min() == 0
    kp_vis = gold["train_keypoints"][..., 2]
    assert ((kp_vis[reg] == 0).any(-1) & (kp_vis[reg] == 1).any(-1)).any()
    lines = "\n".join(str(s) for s in gold["train_labels"])
    for cls in ("Van", "DontCare", "Misc"):
        assert cls + " " in lines
    # outside centres on every border: the intersection of the feature-map centre with each clipped border
    tc, pad, sizes = gold["train_target_centers"], gold["train_pad_size"], gold["train_sizes"]
    tm = gold["train_trunc_mask"] == 1
    sides = set()
    for b in range(tc.shape[0]):
        x_min, y_min = -(-pad[b, 0] // 4), -(-pad[b, 1] // 4)
        x_max, y_max = (pad[b, 0] + sizes[b, 0] - 1) // 4, (pad[b, 1] + sizes[b, 1] - 1) // 4
        for (x, y) in tc[b][tm[b]]:
            sides |= {s for s, hit in (("l", x == x_min), ("r", x == x_max), ("t", y == y_min), ("b", y == y_max)) if hit}
    assert sides == {"l", "r", "t", "b"}, sides
    ori = gold["train_orientations"][reg]
    assert (ori[:, :4].sum(1) == 2).any() and (ori[:, :4].sum(1) == 1).any()    # overlapping bins and single bins


def test_oracle_reproduces_reference(gold):
    f, status = to.encode_batch(gold["rows_packed"], gold["train_P2"], gold["train_sizes"], gold["train_flips"])
    assert status == 0
    for k in INT_FIELDS:
        assert np.array_equal(f[k], gold["train_" + k]), k
    assert np.array_equal(f["P2"], gold["train_P2_flipped"])
    # the reference reaches the border intersection through np.polyfit (an SVD least-squares fit), the oracle through the
    # closed form of the line: the two doubles differ in the last bits, which can move a float32 key point or offset of an
    # outside object by one ulp. Every other value goes through the same numpy operations and is bit-identical.
    outside = (gold["train_trunc_mask"] == 1)
    for k in FLOAT_FIELDS + ["bboxes"]:
        ref = gold["train_" + ("2d_bboxes" if k == "bboxes" else k)]
        d = ulp32(f[k], ref) if ref.dtype == np.float32 else (f[k] != ref).astype(np.int64)
        d = d.reshape(d.shape[0], d.shape[1], -1).max(-1)
        assert d[~outside].max() == 0, k
        assert d.max() <= 1, (k, d.max())
    hm = f["hm"]
    assert np.array_equal(hm, gold["train_hm"])


def test_oracle_test_split_edges(gold):
    for P, s, pad, el, ei in zip(gold["test_P2"], gold["test_sizes"], gold["test_pad_size"], gold["test_edge_len"],
                                 gold["test_edge_indices"]):
        assert np.array_equal(pad, [(1280 - s[0]) // 2, (384 - s[1]) // 2])
        e, n = to.edge_indices(tuple(s), pad, 1280, 384)
        assert n == el and np.array_equal(e, ei)
    assert np.array_equal(gold["test_P2_calib"], gold["test_P2"])


def test_encoder_config_checks():
    cfg = default_cfg()
    tg.GpuTargetEncoder._check_config(cfg)                        # runs/monoflex.yaml values (or absent) are accepted
    cfg.INPUT.HEATMAP_CENTER = '2D'
    with pytest.raises(NotImplementedError):
        tg.GpuTargetEncoder._check_config(cfg)
    cfg = default_cfg()
    cfg.DATASETS.FILTER_ANNOS = [0.8, 20]
    with pytest.raises(NotImplementedError):
        tg.GpuTargetEncoder._check_config(cfg)
    cfg = default_cfg()
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    with pytest.raises(NotImplementedError):
        tg.GpuTargetEncoder._check_config(cfg)
