"""The float64 restatement of the KITTI metric (oracle/kitti_eval_oracle.py) against both goldens of the unmodified
reference (kitti_eval.npz, kitti_eval_edges.npz), what the edge fixture covers, and which wrong rules each fixture can
tell from the right ones. CPU only."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from monoflex_b200 import evaluation as E
from oracle import kitti_eval_oracle as K
from test_kitti_eval import unpack

CLASS_LISTS = ((0, 1, 2), (2, 0), (5, 4, 3, 2, 1, 0))
EDGE_BITS = (31, 32, 63, 64, 95, 96, 127)


def load(name):
    with np.load(os.path.join(GOLDEN, name)) as f:
        z = {k: f[k] for k in f.files}
    z["gt"] = E.KittiAnnos.from_annos(unpack(z, "gt_"), device="cpu")
    z["dt"] = E.KittiAnnos.from_annos(unpack(z, "dt_"), device="cpu")
    z["ov"] = np.stack([z["overlaps_%d" % m] for m in range(3)])
    return z


@pytest.fixture(scope="module")
def old():
    return load("kitti_eval.npz")


@pytest.fixture(scope="module")
def edges():
    return load("kitti_eval_edges.npz")


def tables_of(z, classes):
    """the golden's eval_class tables of one class list as [3 metric][ncls][3][2][41]"""
    name = "" if "precision_0" in z else "_" + "".join(map(str, classes))
    return {k: np.stack([z["%s%s_%d" % (k, name, m)] for m in range(3)]) for k in ("recall", "precision", "orientation")}


def assert_tables(got, ref):
    for k in ("recall", "precision"):
        np.testing.assert_array_equal(got[k], ref[k], err_msg=k)
    np.testing.assert_allclose(got["orientation"], ref["orientation"], rtol=1e-12, atol=0)


def test_statistics_reproduce_the_old_golden(old):
    assert_tables(K.statistics(old["gt"], old["dt"], [0, 1, 2], old["ov"]), tables_of(old, (0, 1, 2)))


@pytest.mark.parametrize("classes", CLASS_LISTS)
def test_statistics_reproduce_the_edge_golden(edges, classes):
    assert_tables(K.statistics(edges["gt"], edges["dt"], list(classes), edges["ov"]), tables_of(edges, classes))


@pytest.mark.parametrize("fixture", ["old", "edges"])
def test_overlaps_equal_the_golden(fixture, request):
    """2D bit for bit; BEV / 3D: the reference clips in float32, so they are within its rounding of the exact values"""
    z = request.getfixturevalue(fixture)
    ov = K.overlaps(z["gt"], z["dt"])
    assert ov.shape == z["ov"].shape
    assert np.array_equal(ov[0], z["ov"][0])
    tol = K.float32_tolerance(z["gt"], z["dt"])
    for m in (1, 2):
        err = np.abs(ov[m] - z["ov"][m])
        assert (err <= tol).all(), (m, err.max(), tol[np.argmax(err - tol)])


def dc_overlaps(z):
    """criterion-0 overlaps of every detection with the DontCare boxes of its image"""
    out = []
    for g, d in zip(unpack(z, "gt_"), unpack(z, "dt_")):
        dc = g["bbox"][g["name"] == "DontCare"]
        if len(d["name"]) and len(dc):
            out.append(K.box_overlap(d["bbox"], dc, False).reshape(-1))
    return np.concatenate(out)


def test_edge_fixture_exercises_every_rule(edges):
    z = edges
    ov0, ov1, ov2 = z["ov"]
    # overlaps exactly at a threshold, and just past it
    dc = dc_overlaps(z)
    for t in (0.5, 0.7):
        assert (ov0 == t).any() and ((ov0 > t) & (ov0 < t + 1e-12)).any(), t
        assert (dc == t).any() and ((dc > t) & (dc < t + 1e-12)).any(), t
    for ov in (ov1, ov2):
        assert (ov == 0.5).any() and (ov == 0.25).any()
        assert ((ov < 0.7) & (ov > 0.7 - 4e-5)).any() and ((ov > 0.7) & (ov < 0.7 + 4e-5)).any()
    # score ties inside an image and across images, exact duplicate detections
    dts = unpack(z, "dt_")
    assert sum(len(d["score"]) - len(np.unique(d["score"])) for d in dts) > 20
    assert any(len(np.unique(np.c_[d["bbox"], d["score"]], axis=0)) < len(d["score"]) - 1 for d in dts)
    sc = z["dt_score"]
    assert np.array_equal(sc, np.round(sc, 4)) and (sc != np.round(sc, 2)).any() and (sc == np.round(sc, 2)).mean() > 0.5
    # heights at the difficulty edges, truncation and occlusion levels, class names
    valid = z["gt_name"] != "DontCare"
    h = (z["gt_bbox"][:, 3] - z["gt_bbox"][:, 1])[valid]
    dh = z["dt_bbox"][:, 3] - z["dt_bbox"][:, 1]
    for v in (25.0, 40.0):
        assert (h == v).any() and (dh == v).any()
    assert (dh < -40).any() and ((dh < -25) & (dh > -40)).any()
    assert {0.15, 0.3, 0.5} <= set(z["gt_truncated"][valid].tolist())
    assert set(z["gt_occluded"][valid].tolist()) >= {0, 1, 2, 3}
    assert {"Van", "Person_sitting", "Truck", "Tram", "Misc", "dontcare", "DontCare"} <= set(z["gt_name"])
    # the crowded images: a match at each edge bit, a DontCare-suppressed detection next to the last
    off = np.concatenate([[0], np.cumsum(z["dt_count"])])
    poff = K.pair_offsets(z["gt_count"], z["dt_count"])
    for n in (31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128):
        i = int(np.nonzero(z["dt_count"] == n)[0][0])
        block = ov0[poff[i]:poff[i + 1]].reshape(n, z["gt_count"][i])
        for b in [b for b in EDGE_BITS if b < n] + [n - 1]:
            assert block[b].max() > 0.7, (n, b)
        g = unpack(z, "gt_")[i]
        sup = K.box_overlap(z["dt_bbox"][off[i]:off[i + 1]], g["bbox"][g["name"] == "DontCare"], False)
        assert sup[n - 2 if n - 2 not in EDGE_BITS else n - 3].max() > 0.7, n
    # image count, the first image without detections, AOS on here and off in the second set
    assert len(z["gt_count"]) > 256 and len(z["gt_count"]) % 128 and z["dt_count"][0] == 0
    assert "aos  AP" in str(z["main_result_012_R40"]) and "aos" not in str(z["noaos_result_012_R40"])
    assert str(z["noaos_result_text"][0]) == "\n" and " -10.0 " in str(z["noaos_result_text"][1]).splitlines()[0]
    assert " -10.0 " not in str(z["noaos_result_text"][1]).splitlines()[1]


def test_edge_fixture_reaches_41_and_repeated_thresholds(edges):
    t = K.statistics(edges["gt"], edges["dt"], [0, 1, 2], edges["ov"])["thresholds"]
    n = (~np.isnan(t)).sum(-1)
    assert n.max() == K.NPTS
    assert (t[..., :-1] == t[..., 1:]).any()


@pytest.mark.parametrize("flip", K.FLIPS)
def test_each_wrong_rule_changes_the_edge_tables(edges, flip):
    """the fixture tells each rule from its flip: at least one table entry moves"""
    ok = K.statistics(edges["gt"], edges["dt"], [0, 1, 2], edges["ov"])
    bad = K.statistics(edges["gt"], edges["dt"], [0, 1, 2], edges["ov"], flip=flip)
    assert any(not np.array_equal(ok[k], bad[k], equal_nan=True) for k in ("recall", "precision", "orientation"))


def test_no_wrong_rule_changes_the_old_tables(old):
    """kitti_eval.npz keeps overlaps off the thresholds, scores unique and heights off 25 and 40, so it cannot tell
    any of these rules from its flip: what the edge fixture adds"""
    ok = K.statistics(old["gt"], old["dt"], [0, 1, 2], old["ov"])
    for flip in K.FLIPS:
        bad = K.statistics(old["gt"], old["dt"], [0, 1, 2], old["ov"], flip=flip)
        assert all(np.array_equal(ok[k], bad[k], equal_nan=True) for k in ("recall", "precision", "orientation")), flip
