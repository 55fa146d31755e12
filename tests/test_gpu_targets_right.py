"""GPU: right-camera items (DATASETS.USE_RIGHT_IMAGE, runs/monoflex_right.yaml) in the training-target encoder
(csrc/mf_targets.cu behind monoflex_b200/targets.py) against the unmodified reference's KITTIDataset.__getitem__
(tests/golden/kitti_targets_right.npz) and against oracle/target_oracle_right.py on random batches that mix left / right and
flipped / unflipped images in one call; the unchanged left path, the status word, CUDA-graph capture, the loss on P3's
baseline and a captured Trainer fed right-image targets."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import targets as tg
from monoflex_b200._lib import call, stream
from monoflex_b200.config import default_cfg
from oracle import target_oracle_right as tor

pytestmark = pytest.mark.gpu

INT_FIELDS = ["cls_ids", "target_centers", "reg_mask", "trunc_mask", "pad_size", "edge_len", "edge_indices"]
FLOAT_FIELDS = ["keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_weight", "offset_3D", "rotys",
                "alphas", "orientations", "gt_bboxes", "2d_bboxes"]
SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370), (1234, 376)]
DIMS = [(1.53, 1.63, 3.88), (1.76, 0.66, 0.84), (1.74, 0.60, 1.76)]
OUTPUTS = ("edge_indices", "edge_len", "alphas", "gt_bboxes", "reg_weight", "occlusions", "truncations", "obj6", "P2", "status")


def right_cfg():
    cfg = default_cfg()
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    return cfg


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "kitti_targets_right.npz")) as z:
        return {k: z[k] for k in z.files}


def ulp32(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def fields_of(enc):
    """the encoder's outputs as the reference's per-image fields, stacked (through the drop-in ParamsLists)"""
    pl = enc.param_lists()
    out = {}
    for k in pl[0].fields():
        if k == "calib":
            out["P2"] = np.stack([np.array(t.get_field(k).P) for t in pl])
        else:
            out[k] = torch.stack([t.get_field(k) for t in pl]).cpu().numpy()
    return out


def assert_matches(got, ref, n_status_got, n_status_ref):
    """integer / mask fields exact; float fields within 1 fp32 ulp (the reference's float64 goes through BLAS and libm
    sin / cos / atan2, the kernel through CUDA's); float64 fields exact; heat maps with identical support and peaks"""
    assert n_status_got == n_status_ref
    for k in INT_FIELDS:
        assert np.array_equal(got[k].astype(np.int64), np.asarray(ref[k]).astype(np.int64)), k
    for k in FLOAT_FIELDS:
        d = ulp32(got[k], ref[k])
        assert d.max() <= 1, (k, d.max(), np.argwhere(d > 1)[:4])
    for k in ("occlusions", "truncations"):
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got["P2"], ref["P2"])
    hm, rhm = got["hm"], ref["hm"]
    assert np.array_equal(hm == 0, rhm == 0) and np.array_equal(hm == 1, rhm == 1)
    assert ulp32(hm, rhm).max() <= 1


def random_batch(seed, B=8, M=40, right=None):
    """seeded KITTI-like frames seen by either camera: labels in the left camera's frame (objects inside, across every
    border, behind the camera, truncated), P3 = P2 with a baseline of about 0.47 m, a right image that may have another
    size, random flips and (unless given) random right flags. A right item's label box columns hold garbage: the
    encoder must not read them. Returns labels, P (P2 or P3 per image), sizes, flips, right."""
    g = np.random.default_rng(seed)
    sizes = np.array([SIZES[int(i)] for i in g.integers(0, len(SIZES), B)], dtype=np.int64)
    right = g.integers(0, 2, B) if right is None else np.asarray(right, dtype=np.int64)
    P = np.zeros((B, 3, 4))
    rows = []
    for b in range(B):
        w, h = sizes[b]
        f = 721.5377 + g.uniform(-14, 14)
        P2 = np.array([[f, 0, w / 2 - 11 + g.uniform(-3, 3), 44.857 + g.uniform(-2, 2)],
                       [0, f, h / 2 - 15 + g.uniform(-3, 3), 0.216 + g.uniform(-0.1, 0.1)], [0, 0, 1, 0.0027]])
        P[b] = P2
        lines = []
        for _ in range(int(g.integers(0, M + 1))):
            c = int(g.integers(0, 3))
            hh, ww, ll = (d * g.uniform(0.85, 1.15) for d in DIMS[c])
            z = g.uniform(-4, 70)
            x = g.uniform(-1.1, 1.1) * max(z, 2.0)
            y = g.uniform(0.8, 2.4) if g.uniform() < 0.8 else g.uniform(-3, 4)
            ry = g.uniform(-math.pi, math.pi)
            cr, sr = math.cos(ry), math.sin(ry)
            xs = np.array([ll / 2, ll / 2, -ll / 2, -ll / 2] * 2)
            zs = np.array([ww / 2, -ww / 2, -ww / 2, ww / 2] * 2)
            ys = np.array([0, 0, 0, 0, -hh, -hh, -hh, -hh])
            pts = np.stack([cr * xs + sr * zs + x, ys + y, -sr * xs + cr * zs + z, np.ones(8)], 1) @ P2.T
            u, v = pts[:, 0] / np.maximum(pts[:, 2], 1e-3), pts[:, 1] / np.maximum(pts[:, 2], 1e-3)
            box = [min(max(u.min(), 0), w - 1), min(max(v.min(), 0), h - 1), min(max(u.max(), 0), w - 1),
                   min(max(v.max(), 0), h - 1)]
            box = [q + g.uniform(-2, 2) for q in box]
            if right[b]:
                box = list(g.uniform(-500, 1500, 4))
            lines.append("%s %.2f %d -10 %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                tg.CLASSES[c], g.uniform(0, 1), int(g.integers(0, 4)), *box, hh, ww, ll, x, y, z, ry))
        rows.append(tg.read_kitti_label(lines))
        if right[b]:
            P[b, 0, 3] = -339.5 + g.uniform(-5, 5)
            if g.uniform() < 0.3:
                sizes[b] = SIZES[int(g.integers(0, len(SIZES)))]
    flips = g.integers(0, 2, B)
    return tg.pack_labels(rows, M), P, sizes, flips, right


def oracle_fields(labels, P, sizes, flips, right):
    f, status = tor.encode_batch(labels, P, sizes, flips, right)
    f["2d_bboxes"] = f.pop("bboxes")
    return f, status


def test_encoder_vs_reference_golden_right(gold):
    """the 2N items of a USE_RIGHT_IMAGE dataset (left and right, flipped and not) in one call"""
    enc = tg.GpuTargetEncoder(right_cfg())
    e = enc.encode(gold["rows_packed"], gold["P"], gold["sizes"], gold["flips"], right=gold["right"])
    got = fields_of(e)
    ref = {k: gold[k] for k in INT_FIELDS + FLOAT_FIELDS + ["occlusions", "truncations", "hm"]}
    ref["P2"] = gold["P2_flipped"]
    assert_matches(got, ref, int(e.status.item()), 0)
    right = gold["right"] == 1
    for flip in (0, 1):                                            # both flip branches of the right view carry objects
        assert got["reg_mask"][right & (gold["flips"] == flip)].sum() > 50
    e.check()


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_encoder_vs_oracle_mixed_batches(seed):
    enc = tg.GpuTargetEncoder(right_cfg())
    labels, P, sizes, flips, right = random_batch(seed, right=[1, 1, 0, 1, 0, 1, 1, 0])
    flips[:4] = [0, 1, 0, 1]                                       # right unflipped, right flipped, left, right flipped
    e = enc.encode(labels, P, sizes, flips, right=right)
    ref, status = oracle_fields(labels, P, sizes, flips, right)
    got = fields_of(e)
    assert_matches(got, ref, int(e.status.item()), status)
    r = right == 1
    assert got["reg_mask"][r].sum() > 20 and got["trunc_mask"][r].sum() > 0
    # b_x of P3 in the loss's calibration rows: about +0.47 m, and -0.47 m once the flip has negated P[0, 3]
    bx = e.prepared[2][:, 4].cpu().numpy()
    assert (np.abs(bx[r]) > 0.4).all() and (np.sign(bx[r]) == np.where(flips[r] == 1, -1, 1)).all()


def test_left_batch_identical_across_entry_points():
    """right=None, right = all zeros and the old mf_encode_targets entry point: the same bits for a left batch"""
    enc = tg.GpuTargetEncoder(right_cfg())
    labels, P2, sizes, flips, _ = random_batch(41, right=[0] * 8)
    e0 = enc.encode(labels, P2, sizes, flips)
    e1 = enc.encode(labels, P2, sizes, flips, right=np.zeros(8, np.int64))
    e2 = enc.encode(labels, P2, sizes, flips, right=torch.zeros(8, dtype=torch.int32, device="cuda"))
    for t in list(e2.prepared) + [getattr(e2, n) for n in OUTPUTS]:
        t.fill_(7)
    lab, p2, sz, fl, _ = e2.inputs
    hm, obj, img = e2.prepared
    call("mf_encode_targets", lab.data_ptr(), p2.data_ptr(), sz.data_ptr(), fl.data_ptr(), 8, enc.max_objs, enc.H, enc.W,
         hm.data_ptr(), obj.data_ptr(), img.data_ptr(), e2.alphas.data_ptr(), e2.gt_bboxes.data_ptr(),
         e2.reg_weight.data_ptr(), e2.occlusions.data_ptr(), e2.truncations.data_ptr(), e2.obj6.data_ptr(), e2.P2.data_ptr(),
         e2.edge_indices.data_ptr(), e2.edge_len.data_ptr(), e2.status.data_ptr(), stream())
    for e in (e1, e2):
        for a, b in zip(e.prepared, e0.prepared):
            assert torch.equal(a, b)
        for name in OUTPUTS:
            assert torch.equal(getattr(e, name), getattr(e0, name)), name
    assert int(e0.reg_weight.sum()) > 20


def test_status_word_counts_right_view_objects():
    """A pedestrian 3.72 m left of a camera 4 m away: the left view encodes it, the right view (0.53 m further right) sees
    it wholly beyond the left border, a clamped and inverted box whose centre lies outside the image, where the reference
    raises (approx_proj_center returns None). Counted, left out, and check() raises; the other objects are unaffected."""
    enc = tg.GpuTargetEncoder(right_cfg())
    f = 721.5377
    P2 = np.array([[f, 0, 609.5593, 44.85728], [0, f, 172.854, 0.2163791], [0, 0, 1, 0.002745884]])
    P3 = P2.copy()
    P3[0, 3] = -339.5
    labels, P, sizes, flips, right = random_batch(21, B=2, right=[1, 1])
    n = int(labels[0, :, 0].sum())
    assert n < 40
    bad = tg.read_kitti_label(["Pedestrian 0.00 0 -10 0.00 150.00 60.00 300.00 1.76 0.66 0.84 -3.72 1.70 4.00 0.00"])
    labels_bad = labels.copy()
    labels_bad[0, n, 0] = 1
    labels_bad[0, n, 1:15] = bad[0]
    sizes[0] = (1242, 375)
    for rt, P0 in ((1, P3), (0, P2)):
        right[0], P[0] = rt, P0
        for fl in (0, 1):
            flips[0] = fl
            e0 = enc.encode(labels, P, sizes, flips, right=right)
            good, n0 = fields_of(e0), int(e0.status.item())
            e = enc.encode(labels_bad, P, sizes, flips, right=right)
            ref, status = oracle_fields(labels_bad, P, sizes, flips, right)
            assert int(e.status.item()) == status == n0 + rt, (rt, fl)
            got = fields_of(e)
            if rt:
                with pytest.raises(RuntimeError):
                    e.check()
                for k in good:
                    assert np.array_equal(got[k], good[k]), k          # the other objects are unaffected
            else:
                assert got["reg_mask"][0, n] == 1                      # the left view encodes it
                assert_matches(got, ref, int(e.status.item()), status)


def test_encode_right_captured_in_cuda_graph():
    enc = tg.GpuTargetEncoder(right_cfg())
    labels, P, sizes, flips, right = random_batch(31)
    dev = torch.device("cuda")
    s_lab, s_p = torch.from_numpy(labels).to(dev), torch.from_numpy(P).to(dev)
    s_sz, s_fl = torch.from_numpy(sizes).to(dev, torch.int32), torch.from_numpy(flips).to(dev, torch.int32)
    s_rt = torch.from_numpy(right).to(dev, torch.int32)
    static = tuple(t.clone() for t in enc.encode(s_lab, s_p, s_sz, s_fl, right=s_rt).prepared)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                                  # a host synchronisation inside would fail the capture
        e = enc.encode(s_lab, s_p, s_sz, s_fl, out=static, right=s_rt)
    for seed in (32, 33, 34):
        labels2, P_2, sizes2, flips2, right2 = random_batch(seed, right=[seed % 2] * 4 + [1 - seed % 2] * 4)
        s_lab.copy_(torch.from_numpy(labels2))
        s_p.copy_(torch.from_numpy(P_2))
        s_sz.copy_(torch.from_numpy(sizes2))
        s_fl.copy_(torch.from_numpy(flips2))
        s_rt.copy_(torch.from_numpy(right2))
        graph.replay()
        ref = enc.encode(labels2, P_2, sizes2, flips2, right=right2)
        for a, b in zip(e.prepared, ref.prepared):
            assert torch.equal(a, b)
        for name in OUTPUTS:
            assert torch.equal(getattr(e, name), getattr(ref, name)), name


def test_loss_on_right_targets_matches_oracle():
    """Loss_Computation on right-image targets (the drop-in ParamsLists and prepared=) against the CPU oracle's loss with
    each image's flipped P3: the loss kernel's calibration rows carry b_x of about +0.47 m, where P2 gives about -0.06 m."""
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    from oracle import monoflex_oracle as mo
    cfg = right_cfg()
    enc = tg.GpuTargetEncoder(cfg)
    labels, P, sizes, flips, right = random_batch(51, B=4, right=[1, 1, 1, 1])
    flips[:] = [0, 1, 0, 1]
    e = enc.encode(labels, P, sizes, flips, right=right)
    pl = e.param_lists()
    fields = []
    for t in pl:
        d = {k: t.get_field(k).cpu().numpy() for k in t.fields() if k != "calib"}
        d["bboxes"] = d.pop("2d_bboxes")
        fields.append(d)
    assert all(f["reg_mask"].sum() > 0 for f in fields)
    Pf = [np.array(t.get_field("calib").P) for t in pl]
    assert all(abs(p[0, 3] / -p[0, 0]) > 0.4 for p in Pf)                 # +-0.47 m: the flip negates P[0, 3]
    cls, reg = syn.make_train_predictions(4, fields, seed=52)
    lc = Loss_Computation(cfg)
    la, loga = lc({"cls": cls.cuda(), "reg": reg.cuda()}, pl)
    lb, logb = lc({"cls": cls.cuda(), "reg": reg.cuda()}, e.edge_targets(), prepared=e.prepared)
    ref, ref_log = mo.loss_computation(cls, reg, fields, Pf)
    assert list(la) == mo.LOSS_NAMES
    for k in mo.LOSS_NAMES:
        b = ref[k].item()
        for got in (la, lb):
            assert abs(got[k].item() - b) <= 1e-5 * max(1.0, abs(b)), (k, got[k].item(), b)
    for k, v in ref_log.items():
        for log in (loga, logb):
            assert abs(log[k] - v.item()) <= 1e-5 * max(1.0, abs(v.item())), (k, log[k], v.item())


def test_captured_trainer_fed_right_targets_matches_eager():
    """A captured Trainer fed right-image EncodedTargets (new labels, flips and right flags every step) against an eager
    Trainer fed the equivalent ParamsLists, with the tolerances of the left-image test in test_gpu_targets.py."""
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.train import Trainer
    cfg = right_cfg()
    B = 2
    models = []
    for _ in range(2):
        m = KeypointDetector(cfg).cuda()
        m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        models.append(m)
    images = syn.make_images(B, 384, 1280, seed=1).cuda()
    ta = Trainer(models[0], cfg, loss_scale=128.0)
    tb = Trainer(models[1], cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    enc = tg.GpuTargetEncoder(cfg)
    logs_a, logs_b = [], []
    for step in range(4):
        labels, P, sizes, flips, right = random_batch(100 + step, B=B, right=[1, step % 2])
        e = enc.encode(labels, P, sizes, flips, right=right)
        logs_a.append(ta.step(images, e.param_lists())[1])
        logs_b.append(tb.step(images, e, sync_log=False)[1])
    assert tb._graph is not None
    logs_b = [l.resolve() for l in logs_b]
    for k, v in logs_a[0].items():
        assert abs(v - logs_b[0][k]) <= 1e-5 * max(abs(v), 1e-3), (k, v, logs_b[0][k])
    for i, (la, lb) in enumerate(zip(logs_a, logs_b)):
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(ta_tot) and np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
    assert logs_b[2] != logs_b[3]
