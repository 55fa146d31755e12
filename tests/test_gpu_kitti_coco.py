"""The KITTI COCO-style AP on the GPU (csrc/mf_kitti_eval.cu's overlap-set entry points, evaluation.get_coco_eval_result
and evaluate()): the text and the tables against the unmodified reference (tests/golden/kitti_coco.npz) and against the
float64 oracle (oracle/kitti_sets_oracle.py) on the kernel's own overlaps, evaluate() and the command line on written result folders, determinism,
the official table through the new entry points, and the limits.

The statistics are compared exactly (AOS within 1e-12 relative: the device's cos against numpy's)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import ROOT
from monoflex_b200 import evaluation as E
from oracle import kitti_eval_oracle as K
from oracle import kitti_sets_oracle as S
from test_gpu_kitti_eval_edges import assert_equal_tables
from test_kitti_coco_host import CLASS_LISTS, golden_tables, name, z  # noqa: F401 (z is a fixture)
from test_kitti_eval import assert_same_result, unpack, write_set

pytestmark = pytest.mark.gpu
NAMES = ["Car", "Pedestrian", "Cyclist"]


def cuda(a):
    return E.KittiAnnos(a.objects.cuda(), a.counts)


def assert_same_score_result(got, z, tag):
    """evaluate(score_thresh=...)'s (result, ret_dict) against the golden, as assert_same_result does"""
    keyed = {"%s_result_R40" % tag: z["%s_score_result" % tag], "%s_ret_keys_R40" % tag: z["%s_score_ret_keys" % tag],
             "%s_ret_values_R40" % tag: z["%s_score_ret_values" % tag]}
    assert_same_result(got, keyed, "%s_@R40" % tag)


@pytest.mark.parametrize("classes", CLASS_LISTS)
def test_coco_text_equals_the_reference(z, classes):
    assert E.get_coco_eval_result(unpack(z, "gt_"), unpack(z, "dt_"), list(classes)) == str(z["main_coco_" + name(classes)])


def test_evaluate_on_result_folders_equals_the_reference(z, tmp_path):
    t = float(z["score_thresh"])
    for tag in ("main", "noaos"):
        root = tmp_path / tag
        root.mkdir()
        label, pred, split = write_set(z, tag, root)
        for classes in CLASS_LISTS:
            assert E.evaluate(label, pred, split, list(classes), coco=True) == str(z["%s_coco_%s" % (tag, name(classes))])
        assert E.evaluate(label, pred, split, NAMES, coco=True, score_thresh=t) == str(z[tag + "_coco_score"])
        assert_same_score_result(E.evaluate(label, pred, split, NAMES, score_thresh=t, metric="R40"), z, tag)


def test_command_line_prints_the_reference_table(z, tmp_path):
    label, pred, split = write_set(z, "main", tmp_path)
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "monoflex_b200.evaluation", "--label_path", label, "--result_path", pred, "--label_split_file", split]
    out = subprocess.run(base + ["--current_class", "0,1,2", "--coco"], cwd=ROOT, env=env, capture_output=True,
                         text=True, check=True).stdout
    assert out == str(z["main_coco_012"])
    out = subprocess.run(base + ["--current_class", "Car,Pedestrian,Cyclist", "--score_thresh", repr(float(z["score_thresh"]))],
                         cwd=ROOT, env=env, capture_output=True, text=True, check=True).stdout
    assert out == str(z["main_score_result"])


@pytest.mark.parametrize("classes", CLASS_LISTS)
def test_per_set_tables_equal_the_golden_and_the_oracle(z, classes):
    mo = E.coco_min_overlaps(list(classes))
    tables, ov = E.eval_tables(cuda(z["gt"]), cuda(z["dt"]), list(classes), min_overlaps=mo)
    assert tables["recall"].shape == (3, 3, 3, 10, K.NPTS) and tables["ap"].shape == (2, 4, 3, 3, 10)
    ov = ov.cpu().numpy()
    assert np.array_equal(ov[0], z["ov"][0])
    for m in (1, 2):
        assert np.abs(ov[m] - z["ov"][m]).max() <= 1e-5, m
    ref = golden_tables(z, classes)
    for k in ("recall", "precision"):
        np.testing.assert_array_equal(tables[k], ref[k], err_msg=k)
    np.testing.assert_allclose(tables["orientation"], ref["orientation"], rtol=1e-12, atol=0)
    assert_equal_tables(tables, S.statistics(z["gt"], z["dt"], list(classes), ov, mo))


@pytest.mark.parametrize("n_sets", [1, 3, 16])
def test_any_number_of_sets_equals_the_oracle(z, n_sets):
    """arbitrary tables: every (set, metric, class) its own threshold"""
    classes = [2, 0, 1, 3]
    mo = np.random.default_rng(n_sets).uniform(0.2, 0.9, (n_sets, 3, len(classes)))
    tables, ov = E.eval_tables(cuda(z["gt"]), cuda(z["dt"]), classes, min_overlaps=mo)
    assert tables["precision"].shape[3] == n_sets
    assert_equal_tables(tables, S.statistics(z["gt"], z["dt"], classes, ov.cpu().numpy(), mo))


def test_two_runs_are_bit_identical(z):
    classes = [0, 1, 2, 3, 4]
    mo = E.coco_min_overlaps(classes)
    a, oa = E.eval_tables(cuda(z["gt"]), cuda(z["dt"]), classes, min_overlaps=mo)
    b, ob = E.eval_tables(cuda(z["gt"]), cuda(z["dt"]), classes, min_overlaps=mo)
    assert torch.equal(oa, ob)
    for k in ("recall", "precision", "orientation", "ap"):
        assert a[k].tobytes() == b[k].tobytes()


@pytest.mark.parametrize("classes", [(0, 1, 2), (2, 0), (5, 4, 3, 2, 1, 0)])
def test_official_table_through_the_sets_entry_points_equals_the_official_ones(z, classes):
    gt, dt = cuda(z["gt"]), cuda(z["dt"])
    a, _ = E.eval_tables(gt, dt, list(classes))
    b, _ = E.eval_tables(gt, dt, list(classes), min_overlaps=E.MIN_OVERLAPS[:, :, list(classes)])
    for k in ("recall", "precision", "orientation", "ap"):
        assert a[k].shape == b[k].shape and a[k].tobytes() == b[k].tobytes(), k
    assert a["compute_aos"] == b["compute_aos"]


def test_car_at_the_0_7_set_equals_the_official_first_set(z):
    gt, dt = cuda(z["gt"]), cuda(z["dt"])
    mo = E.coco_min_overlaps([0, 1, 2])
    assert (mo[4, :, 0] == 0.7).all() and np.linspace(0.5, 0.95, 10)[4] == 0.7
    coco, _ = E.eval_tables(gt, dt, [0, 1, 2], min_overlaps=mo)
    official, _ = E.eval_tables(gt, dt, [0, 1, 2])
    for k in ("recall", "precision", "orientation"):
        assert coco[k][:, 0, :, 4].tobytes() == official[k][:, 0, :, 0].tobytes(), k
    assert coco["ap"][:, :, 0, :, 4].tobytes() == official["ap"][:, :, 0, :, 0].tobytes()


def test_truck_too_many_classes_and_bad_tables_raise(z):
    gts, dts = unpack(z, "gt_"), unpack(z, "dt_")
    with pytest.raises(KeyError):
        E.get_coco_eval_result(gts, dts, ["Car", "Truck"])
    with pytest.raises(KeyError):
        E.get_coco_eval_result(gts, dts, 5)
    with pytest.raises(ValueError, match="9 classes"):
        E.get_coco_eval_result(gts, dts, [0, 1, 2, 3, 4, 0, 1, 2, 3])
    with pytest.raises(ValueError, match="min_overlaps"):
        E.eval_tables(gts, dts, [0, 1], min_overlaps=np.full((10, 3, 3), 0.5))
    with pytest.raises(ValueError, match="min_overlaps"):
        E.eval_tables(gts, dts, [0], min_overlaps=np.zeros((0, 3, 1)))
    big = {k: np.concatenate([v] * (129 // max(len(v), 1) + 1))[:129] for k, v in dts[int(np.argmax(z["dt_count"]))].items()}
    with pytest.raises(RuntimeError, match="129 detections"):
        E.get_coco_eval_result(gts[:3], [dts[1], big, dts[2]], [0])
