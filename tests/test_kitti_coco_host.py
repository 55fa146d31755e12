"""The KITTI COCO-style AP (evaluation.get_coco_eval_result, evaluate(coco=True)) on the host: the threshold table, the
float64 oracle over a threshold table (oracle/kitti_sets_oracle.py) against the official oracle and, with the COCO
table, against the unmodified reference's tables and text (oracle/make_golden_kitti_coco.py ->
tests/golden/kitti_coco.npz), what the fixture covers, the class rules and the C entry points' bindings. CPU only."""
import ctypes
import os

import numpy as np
import pytest

from conftest import GOLDEN
from monoflex_b200 import evaluation as E
from oracle import kitti_eval_oracle as K
from oracle import kitti_sets_oracle as S
from test_kitti_eval import unpack

CLASS_LISTS = ((0, 1, 2), (3, 4, 0))


@pytest.fixture(scope="module")
def z():
    with np.load(os.path.join(GOLDEN, "kitti_coco.npz")) as f:
        z = {k: f[k] for k in f.files}
    z["gt"] = E.KittiAnnos.from_annos(unpack(z, "gt_"), device="cpu")
    z["dt"] = E.KittiAnnos.from_annos(unpack(z, "dt_"), device="cpu")
    z["ov"] = np.stack([z["overlaps_%d" % m] for m in range(3)])
    return z


def name(classes):
    return "".join(map(str, classes))


def golden_tables(z, classes):
    """eval_class's tables of one class list as [3 metric][ncls][3][10][41]"""
    return {k: np.stack([z["%s_%s_%d" % (k, name(classes), m)] for m in range(3)])
            for k in ("recall", "precision", "orientation")}


def test_threshold_table_is_numpys_linspace(z):
    for classes in CLASS_LISTS:
        mo = E.coco_min_overlaps(list(classes))
        assert mo.shape == (10, 3, 3)
        assert mo.tobytes() == z["min_overlaps_" + name(classes)].tobytes()
    mo = E.coco_min_overlaps([0, 1])
    assert np.array_equal(mo[:, 0, 0], np.linspace(0.5, 0.95, 10)) and np.array_equal(mo[:, 2, 1], np.linspace(0.25, 0.7, 10))
    # three thresholds are not the decimal literals they print as
    assert mo[8, 0, 0] == 0.8999999999999999 and mo[4, 1, 1] == 0.44999999999999996 and mo[8, 1, 1] == 0.6499999999999999
    assert mo[4, 0, 0] == 0.7 and (mo[4, :, 0] == E.MIN_OVERLAPS[0, :, 0]).all()


@pytest.mark.parametrize("classes", CLASS_LISTS)
def test_oracle_with_the_coco_table_reproduces_the_golden(z, classes):
    mo = z["min_overlaps_" + name(classes)]
    got = S.statistics(z["gt"], z["dt"], list(classes), z["ov"], mo)
    ref = golden_tables(z, classes)
    for k in ("recall", "precision"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    np.testing.assert_allclose(got["orientation"], ref["orientation"], rtol=1e-12, atol=0)
    # the reference's text from the oracle's AP per set, averaged over the sets on the host
    assert E.coco_result_text(list(classes), got["ap"][0], got["compute_aos"]) == str(z["main_coco_" + name(classes)])


@pytest.mark.parametrize("classes", [(0, 2), (5, 4, 3, 2, 1, 0)])
def test_set_oracle_with_the_official_table_equals_the_official_oracle(z, classes):
    a = K.statistics(z["gt"], z["dt"], list(classes), z["ov"])
    b = S.statistics(z["gt"], z["dt"], list(classes), z["ov"], E.MIN_OVERLAPS[:, :, list(classes)])
    for k in ("recall", "precision", "orientation", "ap", "thresholds"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_fixture_covers_the_cases(z):
    assert (z["gt_count"] == 0).any() and (z["dt_count"] == 0).any()
    assert z["dt_count"].max() == 128
    for tag in ("main", "noaos"):
        text = str(z[tag + "_coco_012"])
        assert text.startswith("Car coco AP@0.50:0.05:0.95:\n") and "Pedestrian coco AP@0.25:0.05:0.70:\n" in text
    assert "aos  AP" in str(z["main_coco_012"]) and "aos" not in str(z["noaos_coco_012"])
    assert "Van coco AP@0.50:0.05:0.95:" in str(z["main_coco_340"])
    # the score threshold is a detection's own score (kept), and drops some detections
    t = float(z["score_thresh"])
    assert (z["dt_score"] == t).sum() == 1 and (z["dt_score"] < t).any()
    assert str(z["main_coco_score"]) != str(z["main_coco_012"])
    # every float32 overlap is clear of every threshold of the grid
    for m in range(3):
        assert np.abs(z["overlaps_%d" % m][:, None] - z["grid"][None, :]).min() >= 1e-3, m


def test_truck_has_no_coco_range():
    with pytest.raises(KeyError):
        E.get_coco_eval_result([], [], "Truck")
    with pytest.raises(KeyError):
        E.get_coco_eval_result([], [], [0, 5])


def test_annos_off_the_gpu_are_refused(z):
    gt = E.KittiAnnos.from_annos(unpack(z, "gt_")[:3], device="cpu")
    dt = E.KittiAnnos.from_annos(unpack(z, "dt_")[:3], device="cpu")
    with pytest.raises(ValueError, match="CUDA tensors only"):
        E.get_coco_eval_result(gt, dt, [0, 1, 2])


def test_command_line_classes():
    assert E.parse_classes("0,1,2") == [0, 1, 2]
    assert E.parse_classes("Car, Pedestrian") == ["Car", "Pedestrian"]
    assert E.parse_classes("4") == [4]


def test_sets_entry_point_types():
    from monoflex_b200 import _lib
    sig, proto = _lib.SIGNATURES, _lib._PROTOTYPES
    assert sig["mf_kitti_eval_sets_workspace_size"] == [ctypes.c_int] * 4 + [ctypes.c_void_p]
    stats = sig["mf_kitti_eval_sets_statistics"]
    assert stats[:13] == sig["mf_kitti_eval_statistics"][:13]
    assert stats[13:] == [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_size_t, ctypes.c_void_p]
    assert sig["mf_kitti_eval_sets_ap"] == [ctypes.c_void_p] + [ctypes.c_int] * 4 + [ctypes.c_void_p] * 2
    for n in ("mf_kitti_eval_sets_workspace_size", "mf_kitti_eval_sets_statistics", "mf_kitti_eval_sets_ap"):
        assert proto[n][0] is ctypes.c_int


@pytest.mark.parametrize("args,msg", [((10, 10, 3, 0), b"0 overlap sets"), ((10, 10, 9, 2), b"9 classes"),
                                      ((10, 10, 8, 1 << 24), b"overlap sets")])
def test_workspace_size_refuses_bad_counts(args, msg):
    from monoflex_b200 import _lib
    lib = _lib.load()
    size = ctypes.c_size_t(7)
    assert lib.mf_kitti_eval_sets_workspace_size(*args, ctypes.byref(size)) == -1
    assert msg in lib.mf_last_error() and size.value == 7
