"""KITTI official metric (monoflex_b200/evaluation.py, csrc/mf_kitti_eval.cu) against the unmodified reference's
kitti_object_eval_python (oracle/make_golden_kitti_eval.py -> tests/golden/kitti_eval.npz).

CPU: parsing, and what the fixture covers. GPU (-m gpu): overlaps, precision / recall / AOS tables, the `result` text and
`ret_dict` through get_official_eval_result and evaluate_python, determinism, limits, and from_results against the text
files the reference writes."""
import csv
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import evaluation as E

FIELDS = ("truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")
THRESHOLDS = (0.25, 0.5, 0.7)


@pytest.fixture(scope="module")
def z():
    with np.load(os.path.join(GOLDEN, "kitti_eval.npz")) as f:
        return {k: f[k] for k in f.files}


def unpack(z, prefix):
    """the reference-parsed per-image dicts"""
    off = np.concatenate([[0], np.cumsum(z[prefix + "count"])])
    return [{"name": z[prefix + "name"][a:b], **{f: z[prefix + f][a:b] for f in FIELDS}} for a, b in zip(off[:-1], off[1:])]


def write_set(z, tag, root):
    label, pred = root / "label", root / "pred"
    label.mkdir()
    pred.mkdir()
    for i, l, r in zip(z[tag + "_ids"], z[tag + "_label_text"], z[tag + "_result_text"]):
        (label / ("%06d.txt" % i)).write_text(str(l))
        (pred / ("%06d.txt" % i)).write_text(str(r))
    split = root / "split.txt"
    split.write_text("".join("%d\n" % i for i in z[tag + "_ids"]))
    return str(label), str(pred), str(split)


def packed(annos):
    return E.KittiAnnos.from_annos(annos, device="cpu").objects.numpy()


# ------------------------------------------------------------------------------------------------------------- CPU
def test_from_label_dir_parses_like_the_reference(z, tmp_path):
    label, pred, _ = write_set(z, "main", tmp_path)
    ids = [int(i) for i in z["main_ids"]]
    for path, prefix, image_ids in ((label, "gt_", ids), (pred, "dt_", None)):
        got = E.KittiAnnos.from_label_dir(path, image_ids, device="cpu")
        ref = unpack(z, prefix)
        assert np.array_equal(got.counts, z[prefix + "count"])
        assert np.array_equal(got.objects.numpy(), packed(ref))
        names = [n for a in ref for n in a["name"]]
        assert got.objects[:, 0].tolist() == [E.class_code(n) for n in names]
        for i in (0, 7, len(ids) - 1):
            a = E.get_label_anno(os.path.join(path, "%06d.txt" % ids[i]))
            for f in FIELDS:
                assert np.array_equal(a[f], ref[i][f]), f


def test_class_codes():
    assert [E.class_code(n) for n in ("Car", "car", "VAN", "Person_sitting", "Truck", "DontCare", "dontcare", "Tram",
                                      "Misc")] == [0, 0, 3, 4, 5, 6, -1, -1, -1]


def box_overlap(a, b, iou):
    iw = min(a[2], b[2]) - max(a[0], b[0])
    ih = min(a[3], b[3]) - max(a[1], b[1])
    if iw <= 0 or ih <= 0:
        return 0.0
    ua = (a[2] - a[0]) * (a[3] - a[1]) + ((b[2] - b[0]) * (b[3] - b[1]) - iw * ih if iou else 0)
    return iw * ih / ua


def test_fixture_exercises_every_branch(z):
    gts, dts = unpack(z, "gt_"), unpack(z, "dt_")
    names = set(z["gt_name"])
    assert {"Car", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "DontCare"} <= names
    valid = z["gt_name"] != "DontCare"
    h = z["gt_bbox"][:, 3] - z["gt_bbox"][:, 1]
    for lo, hi in ((0, 25), (25, 40), (40, 1e9)):
        assert ((h[valid] > lo) & (h[valid] <= hi)).any()
    assert set(z["gt_occluded"][valid]) >= {0, 1, 2, 3}
    assert (z["gt_truncated"][valid] > 0.5).any() and ((z["gt_truncated"] > 0.15) & (z["gt_truncated"] <= 0.3)).any()
    dh = np.abs(z["dt_bbox"][:, 3] - z["dt_bbox"][:, 1])
    assert (dh < 25).any() and ((dh >= 25) & (dh < 40)).any()                 # the detection height filter
    assert (z["gt_count"] == 0).any()
    empty = [str(t) for t, c in zip(z["main_result_text"], z["dt_count"]) if c == 0]
    assert empty and all(t == "\n" for t in empty)
    on_dc = swapped_in = 0
    for g, d in zip(gts, dts):
        for k in range(len(d["name"])):
            for q in range(len(g["name"])):
                if g["name"][q] == "DontCare" and box_overlap(d["bbox"][k], g["bbox"][q], False) > 0.7:
                    on_dc += 1
                if g["name"][q] in ("Van", "Person_sitting") and box_overlap(d["bbox"][k], g["bbox"][q], True) > 0.7 \
                        and d["name"][k] == {"Van": "Car", "Person_sitting": "Pedestrian"}[g["name"][q]]:
                    swapped_in += 1
    assert on_dc > 5 and swapped_in > 5                                        # DontCare suppression, Van / Person_sitting
    assert len(np.unique(z["dt_score"])) == len(z["dt_score"])
    # Cyclist / easy has no valid ground truth: AP 0 there, non-zero elsewhere
    assert not z["precision_0"][2, 0].any() and z["precision_0"][0].any() and z["precision_0"][1].any()
    assert "aos  AP" in str(z["main_result_R40"]) and "aos" not in str(z["noaos_result_R40"])
    assert all(str(t).startswith(tuple(E.ID_TYPE_CONVERSION.values())) or str(t) == "\n" for t in z["noaos_result_text"])


def test_float32_overlaps_are_clear_of_every_threshold(z):
    for m in range(3):
        ov = z["overlaps_%d" % m]
        assert ov.size and (ov > 0.5).any()
        for t in THRESHOLDS:
            assert np.abs(ov - t).min() >= 1e-3, (m, t)


def test_objects_must_be_float64_rows_of_16():
    for bad in (torch.zeros(2, 16, dtype=torch.float32), torch.zeros(2, 15, dtype=torch.float64), torch.zeros(32)):
        with pytest.raises(ValueError, match="float64"):
            E.KittiAnnos(bad, [2])
    strided = E.KittiAnnos(torch.zeros(16, 2, dtype=torch.float64).t(), [1, 1])
    assert strided.objects.is_contiguous()


def test_annos_off_the_gpu_are_refused_before_any_launch(z):
    gt = E.KittiAnnos.from_annos(unpack(z, "gt_")[:3], device="cpu")
    dt = E.KittiAnnos.from_annos(unpack(z, "dt_")[:3], device="cpu")
    with pytest.raises(ValueError, match="CUDA tensors only"):
        E.get_official_eval_result(gt, dt, [0])
    with pytest.raises(ValueError, match="CUDA tensors only"):
        E.eval_tables(gt, dt, [0, 1, 2])


def test_fixture_has_images_over_one_mask_word(z):
    """the assigned / below-threshold masks of the matching kernels span 2, 3 and 4 32-bit words on these images"""
    n = z["dt_count"]
    assert n.max() <= 128
    for lo, hi in ((33, 64), (65, 96), (97, 128)):
        assert ((n >= lo) & (n <= hi)).any(), (lo, hi)


def test_unknown_metric_raises_before_any_work():
    with pytest.raises(ValueError):
        E.get_official_eval_result([], [], [0], metric="R20")


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_overlaps_and_tables_match_the_reference(z):
    gt, dt = E.KittiAnnos.from_annos(unpack(z, "gt_")), E.KittiAnnos.from_annos(unpack(z, "dt_"))
    tables, ov = E.eval_tables(gt, dt, [0, 1, 2])
    ov = ov.cpu().numpy()
    assert np.array_equal(ov[0], z["overlaps_0"])                              # 2D: bit for bit
    for m in (1, 2):
        assert np.abs(ov[m] - z["overlaps_%d" % m]).max() <= 1e-5
    for m in range(3):
        np.testing.assert_array_equal(tables["precision"][m], z["precision_%d" % m])
        np.testing.assert_array_equal(tables["recall"][m], z["recall_%d" % m])
        np.testing.assert_allclose(tables["orientation"][m], z["orientation_%d" % m], rtol=1e-12, atol=0)
    assert tables["compute_aos"]


def assert_same_result(got, z, key):
    result, ret = got
    assert result == str(z[key.replace("@", "result_")])
    assert list(ret) == list(z[key.replace("@", "ret_keys_")])
    ref = z[key.replace("@", "ret_values_")]
    for (k, v), r in zip(ret.items(), ref):
        if "aos" in k:
            assert v == pytest.approx(r, rel=1e-12, abs=0), k
        else:
            assert (v == r) or (np.isnan(v) and np.isnan(r)), k


@pytest.mark.gpu
@pytest.mark.parametrize("metric", ["R40", "R11"])
def test_official_result_text_and_dict(z, tmp_path, metric):
    gts, dts = unpack(z, "gt_"), unpack(z, "dt_")
    detail = {}
    got = E.get_official_eval_result(gts, dts, ["Car", "Pedestrian", "Cyclist"], PR_detail_dict=detail, metric=metric)
    assert_same_result(got, z, "main_@" + metric)
    assert set(detail) == {"bbox", "aos", "bev", "3d"}
    np.testing.assert_array_equal(detail["bev"], z["precision_1"])
    for tag in ("main", "noaos"):
        root = tmp_path / tag
        root.mkdir()
        label, pred, split = write_set(z, tag, root)
        assert_same_result(E.evaluate_python(label, pred, split, ["Car", "Pedestrian", "Cyclist"], metric), z,
                           "%s_@%s" % (tag, metric))


@pytest.mark.gpu
def test_two_runs_are_bit_identical(z):
    gt, dt = E.KittiAnnos.from_annos(unpack(z, "gt_")), E.KittiAnnos.from_annos(unpack(z, "dt_"))
    a, oa = E.eval_tables(gt, dt, [0, 1, 2, 3, 4, 5])
    b, ob = E.eval_tables(gt, dt, [0, 1, 2, 3, 4, 5])
    assert torch.equal(oa, ob)
    for k in ("recall", "precision", "orientation", "ap"):
        assert a[k].tobytes() == b[k].tobytes()


@pytest.mark.gpu
def test_over_limit_image_and_unknown_metric_raise(z):
    gts, dts = unpack(z, "gt_"), unpack(z, "dt_")
    big = {k: np.concatenate([v] * (129 // len(v) + 1))[:129] for k, v in dts[0].items()}
    with pytest.raises(RuntimeError, match="129 detections"):
        E.get_official_eval_result(gts[:3], [dts[1], big, dts[2]], [0])
    at_limit = {k: v[:128] for k, v in big.items()}
    E.get_official_eval_result(gts[:3], [dts[1], at_limit, dts[2]], [0])
    with pytest.raises(ValueError):
        E.get_official_eval_result(gts, dts, [0], metric="R41")


def write_reference_rows(rows, path):
    """generate_kitti_3d_detection: np.round(4) on the float32 row, class name, 0, 0, the values; a lone newline for none"""
    with open(path, "w", newline="") as f:
        w = csv.writer(f, delimiter=" ", lineterminator="\n")
        if len(rows) == 0:
            w.writerow([])
        for p in rows:
            p = p.numpy().round(4)
            w.writerow([E.ID_TYPE_CONVERSION[int(p[0])], 0, 0] + p[1:].tolist())


@pytest.mark.gpu
def test_from_results_equals_the_text_route(tmp_path):
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.detector import KeypointDetector
    H, W, B = 384, 1280, 3
    m = KeypointDetector(default_cfg(width=W, height=H))
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval()
    m.heads.post_processor.det_threshold = 0.0
    x = syn.make_images(B, H, W).cuda()
    targets = [t.to("cuda") for t in syn.make_param_lists(syn.make_targets(B, W // 4, H // 4))]
    with torch.no_grad():
        result, eval_utils, _ = m(x, targets)
    counts = [int(c) for c in eval_utils["counts"]]
    counts[-1] = 0                                                  # an image without detections
    result = result[:sum(counts)]
    rows = result.cpu().split(counts)
    pred, label = tmp_path / "pred", tmp_path / "label"
    pred.mkdir()
    label.mkdir()
    for i, r in enumerate(rows):
        write_reference_rows(r, pred / ("%06d.txt" % i))
    # ground truth derived from the rows: every other detection as a labelled object
    for i, r in enumerate(rows):
        lines = []
        for p in r.double().tolist()[::2]:
            lines.append("%s 0.00 0 %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f" % (
                E.ID_TYPE_CONVERSION[int(p[0])], *p[1:13]))
        (label / ("%06d.txt" % i)).write_text("".join(s + "\n" for s in lines))
    text = E.KittiAnnos.from_label_dir(str(pred))
    direct = E.KittiAnnos.from_results(result, counts)
    assert np.array_equal(direct.counts, text.counts)
    assert torch.equal(direct.objects, text.objects)
    gt = E.KittiAnnos.from_label_dir(str(label))
    split = tmp_path / "split.txt"
    split.write_text("".join("%d\n" % i for i in range(B)))
    result, ret = E.get_official_eval_result(gt, direct, [0, 1, 2])
    result_t, ret_t = E.evaluate_python(str(label), str(pred), str(split), [0, 1, 2], "R40")
    assert result == result_t and list(ret) == list(ret_t)
    assert np.array_equal(list(ret.values()), list(ret_t.values()), equal_nan=True)
    assert max(np.nan_to_num(list(ret.values()))) > 0, result
