"""CPU: the 3D IoU oracle (oracle/iou3d_oracle.py) against the unmodified reference's get_iou_3d and Loss_Computation
'3D_IoU' log recorded in tests/golden/iou3d.npz (oracle/make_golden_iou3d.py), the exact polygon stand-in, and what the
fixture covers."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import iou3d_oracle as io
from oracle import monoflex_oracle as mo


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "iou3d.npz")) as z:
        return {k: z[k] for k in z.files}


def same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def test_oracle_reproduces_reference_pairs(gold):
    assert same_bits(io.get_iou_3d(gold["pred"], gold["target"]), gold["iou"])


def test_oracle_reproduces_reference_loss_log(gold):
    iou = io.get_iou_3d(gold["loss_pred"], gold["loss_target"])
    assert same_bits(iou, gold["loss_iou"])
    assert same_bits(torch.from_numpy(iou).mean().item(), gold["log_3D_IoU"])
    # the same log from the oracle's own loss corners (monoflex_oracle.loss_computation's) on the fixture's loss inputs
    from monoflex_b200 import synthetic as syn
    fields = syn.make_train_targets(4)
    cls, reg = syn.make_train_predictions(4, fields)
    mean, per_object = io.loss_iou3d(cls, reg, fields, [syn.KITTI_P2] * 4)
    assert per_object.shape == gold["loss_iou"].shape
    assert abs(mean - gold["log_3D_IoU"]) <= 1e-5 * abs(gold["log_3D_IoU"])


def test_loss_oracle_leaves_loss_computation_alone():
    from monoflex_b200 import synthetic as syn
    build = mo.encode_box3d
    fields = syn.make_train_targets(1, empty_image=-1)
    cls, reg = syn.make_train_predictions(1, fields)
    io.loss_iou3d(cls, reg, fields, [syn.KITTI_P2])
    assert mo.encode_box3d is build
    _, log = mo.loss_computation(cls, reg, fields, [syn.KITTI_P2])
    assert "3D_IoU" not in log


def _box(ry, l, w, x, z):
    c = mo.encode_box3d(torch.tensor([ry]), torch.tensor([[l, 1.5, w]]), torch.tensor([[x, 1.0, z]]))[0].numpy()
    return io.ExactPolygon(c[0:4][:, [0, 2]])


def test_exact_polygon_sanity():
    a, b = _box(0.3, 4.0, 1.6, 1.0, 20.0), _box(-0.9, 3.0, 2.0, 2.0, 21.0)
    assert a.is_valid and b.is_valid
    assert a.intersection(b).area == b.intersection(a).area > 0
    assert a.intersection(a).area == a.area
    assert abs(a.area - 6.4) < 1e-5                                  # float32 corners of a 4 x 1.6 rectangle
    far = _box(0.3, 4.0, 1.6, 30.0, 20.0)
    assert a.intersection(far).area == 0.0 and far.intersection(a).area == 0.0
    # GEOS validity for what encode_box3d can build: repeated corners, a bow-tie and NaN are invalid
    assert not io.ExactPolygon([[0, 0], [0, 0], [0, 0], [0, 0]]).is_valid
    assert not io.ExactPolygon([[0, 0], [1, 1], [1, 0], [0, 1]]).is_valid
    nan = io.ExactPolygon([[0, 0], [0, 1], [float("nan"), 1], [1, 0]])
    assert not nan.is_valid and np.isnan(nan.area)
    assert io.ExactPolygon([[0, 0], [0, 2], [3, 2], [3, 0]]).area == 6.0


def test_fixture_covers_every_case(gold):
    case, iou = gold["case"], gold["iou"]
    need = {"disjoint": 8, "no_height_overlap": 5, "contains": 8, "identical": 4, "rot_pi": 4, "rot_half_pi": 4,
            "partial": 30, "edge_touch": 3, "corner_touch": 3, "near_parallel": 5, "zero_size": 2, "nan": 2}
    for c, n in need.items():
        assert (case == c).sum() >= n, c
    counts = {}
    for a, b in zip(gold["pred"][case == "partial"], gold["target"][case == "partial"]):
        pa, pb = io.ExactPolygon(a[0:4][:, [0, 2]]), io.ExactPolygon(b[0:4][:, [0, 2]])
        n = pa.intersection(pb).vertex_count
        counts[n] = counts.get(n, 0) + 1
    assert all(counts.get(n, 0) >= 3 for n in range(3, 9)), counts
    for c in ("disjoint", "no_height_overlap", "edge_touch", "corner_touch"):
        assert (iou[case == c] == 0).all(), c

    def inside(p, r):                                                 # closed axis-aligned rectangle (ry = 0)
        return r[:4, 0].min() <= p[0] <= r[:4, 0].max() and r[:4, 2].min() <= p[2] <= r[:4, 2].max()

    for c in ("edge_touch", "corner_touch"):                          # they do touch: a corner of one lies on the other
        for a, b in zip(gold["pred"][case == c], gold["target"][case == c]):
            assert any(inside(p, b) for p in a[:4]) or any(inside(p, a) for p in b[:4]), c
    assert (iou[case == "identical"] == 1).all()
    assert np.isnan(iou[case == "nan"]).all()
    z = iou[case == "zero_size"]
    assert (z[:2] == 0).all() and np.isnan(z[2])                     # zero-size vs a box: 0; two zero-size boxes: 0 / 0
    assert ((iou[case == "contains"] > 0) & (iou[case == "contains"] < 1)).all()
    assert (iou[case == "near_parallel"] > 0.5).all()
    assert np.isfinite(gold["loss_iou"]).all() and 0 < gold["log_3D_IoU"] < 1
