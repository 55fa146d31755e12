"""GPU: the training-target encoder (csrc/mf_targets.cu behind monoflex_b200/targets.py) against the unmodified reference's
KITTIDataset.__getitem__ (tests/golden/kitti_targets.npz) and against oracle/target_oracle.py on random batches; the drop-in
ParamsLists, the status word, CUDA-graph capture, and a captured Trainer fed encoded targets."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import targets as tg
from monoflex_b200.config import default_cfg
from oracle import target_oracle as to

pytestmark = pytest.mark.gpu

INT_FIELDS = ["cls_ids", "target_centers", "reg_mask", "trunc_mask", "pad_size", "edge_len", "edge_indices"]
FLOAT_FIELDS = ["keypoints", "keypoints_depth_mask", "dimensions", "locations", "reg_weight", "offset_3D", "rotys",
                "alphas", "orientations", "gt_bboxes", "2d_bboxes"]
SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370), (1234, 376)]
DIMS = [(1.53, 1.63, 3.88), (1.76, 0.66, 0.84), (1.74, 0.60, 1.76)]


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


def random_batch(seed, B=8, M=40):
    """seeded KITTI-like labels: objects inside, across every border, behind the camera, truncated; random flips"""
    g = np.random.default_rng(seed)
    sizes = np.array([SIZES[int(i)] for i in g.integers(0, len(SIZES), B)], dtype=np.int64)
    P2 = np.zeros((B, 3, 4))
    rows = []
    for b in range(B):
        w, h = sizes[b]
        f = 721.5377 + g.uniform(-14, 14)
        P2[b] = [[f, 0, w / 2 - 11 + g.uniform(-3, 3), 44.857 + g.uniform(-2, 2)],
                 [0, f, h / 2 - 15 + g.uniform(-3, 3), 0.216 + g.uniform(-0.1, 0.1)], [0, 0, 1, 0.0027]]
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
            pts = np.stack([cr * xs + sr * zs + x, ys + y, -sr * xs + cr * zs + z, np.ones(8)], 1) @ P2[b].T
            u, v = pts[:, 0] / np.maximum(pts[:, 2], 1e-3), pts[:, 1] / np.maximum(pts[:, 2], 1e-3)
            box = [min(max(u.min(), 0), w - 1), min(max(v.min(), 0), h - 1), min(max(u.max(), 0), w - 1),
                   min(max(v.max(), 0), h - 1)]
            box = [q + g.uniform(-2, 2) for q in box]
            lines.append("%s %.2f %d -10 %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                tg.CLASSES[c], g.uniform(0, 1), int(g.integers(0, 4)), *box, hh, ww, ll, x, y, z, ry))
        rows.append(tg.read_kitti_label(lines))
    flips = g.integers(0, 2, B)
    return tg.pack_labels(rows, M), P2, sizes, flips


def oracle_fields(labels, P2, sizes, flips):
    f, status = to.encode_batch(labels, P2, sizes, flips)
    f["2d_bboxes"] = f.pop("bboxes")
    return f, status


def test_encoder_vs_reference_golden(gold):
    enc = tg.GpuTargetEncoder(default_cfg())
    e = enc.encode(gold["rows_packed"], gold["train_P2"], gold["train_sizes"], gold["train_flips"])
    got = fields_of(e)
    ref = {k[len("train_"):]: v for k, v in gold.items() if k.startswith("train_")}
    ref["P2"] = ref["P2_flipped"]
    assert_matches(got, ref, int(e.status.item()), 0)
    for flip in (0, 1):                                            # both flip branches carry objects
        sel = gold["train_flips"] == flip
        assert got["reg_mask"][sel].sum() > 50
    e.check()
    # the test split (kitti.py:287-299)
    tl = enc.encode_inference(gold["test_P2"], gold["test_sizes"])
    for b, t in enumerate(tl):
        assert np.array_equal(t.get_field("pad_size").numpy(), gold["test_pad_size"][b])
        assert int(t.get_field("edge_len")) == gold["test_edge_len"][b]
        assert np.array_equal(t.get_field("edge_indices").cpu().numpy(), gold["test_edge_indices"][b])
        assert np.array_equal(np.array(t.get_field("calib").P), gold["test_P2_calib"][b])


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_encoder_vs_oracle_random_batches(seed):
    enc = tg.GpuTargetEncoder(default_cfg())
    labels, P2, sizes, flips = random_batch(seed)
    e = enc.encode(labels, P2, sizes, flips)
    ref, status = oracle_fields(labels, P2, sizes, flips)
    got = fields_of(e)
    assert_matches(got, ref, int(e.status.item()), status)
    assert got["reg_mask"].sum() > 40 and got["trunc_mask"].sum() > 0


def test_param_lists_drop_in_for_prepare_targets_and_loss(gold):
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    cfg = default_cfg()
    enc = tg.GpuTargetEncoder(cfg)
    labels, P2, sizes, flips = random_batch(11, B=4)
    e = enc.encode(labels, P2, sizes, flips)
    lossev = Loss_Computation(cfg)
    prep = lossev.prepare_targets(e.param_lists(), torch.device("cuda"))
    for a, b in zip(prep, e.prepared):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    g = torch.Generator(device="cuda").manual_seed(0)
    cls = torch.rand(4, 3, 96, 320, device="cuda", generator=g).clamp(1e-4, 1 - 1e-4)
    reg = torch.randn(4, 50, 96, 320, device="cuda", generator=g) * 0.5
    la, loga = lossev({'cls': cls, 'reg': reg}, e.param_lists())
    lb, logb = lossev({'cls': cls, 'reg': reg}, e.edge_targets(), prepared=e.prepared)
    # the focal-loss sum is accumulated with float atomics (mf_elementwise.cu), so hm_loss varies in its last bits from run to
    # run even on identical inputs; every other loss and logged value is bit-identical
    for k in la:
        if k == "hm_loss":
            assert abs(float(la[k]) - float(lb[k])) <= 1e-5 * abs(float(la[k])), (float(la[k]), float(lb[k]))
        else:
            assert torch.equal(la[k], lb[k]), k
    for k in loga:
        assert loga[k] == logb[k] or (k == "hm_loss" and abs(loga[k] - logb[k]) <= 1e-5 * abs(loga[k])), k


def test_status_word_counts_bad_objects():
    enc = tg.GpuTargetEncoder(default_cfg())
    labels, P2, sizes, flips = random_batch(21, B=2)
    n = int(labels[0, :, 0].sum())
    assert n < 40
    bad = tg.read_kitti_label(["Car 0.00 0 -10 -100.00 150.00 -20.00 200.00 1.50 1.60 3.90 -12.00 1.60 8.00 0.30"])
    labels_bad = labels.copy()
    labels_bad[0, n, 0] = 1
    labels_bad[0, n, 1:15] = bad[0]
    for fl in (0, 1):
        flips[0] = fl
        e0 = enc.encode(labels, P2, sizes, flips)
        good, n0 = fields_of(e0), int(e0.status.item())
        e = enc.encode(labels_bad, P2, sizes, flips)
        assert int(e.status.item()) == n0 + 1
        with pytest.raises(RuntimeError):
            e.check()
        got = fields_of(e)
        for k in good:
            assert np.array_equal(got[k], good[k]), k                # the other objects are unaffected


def test_encode_captured_in_cuda_graph():
    enc = tg.GpuTargetEncoder(default_cfg())
    labels, P2, sizes, flips = random_batch(31)
    dev = torch.device("cuda")
    s_lab, s_p2 = torch.from_numpy(labels).to(dev), torch.from_numpy(P2).to(dev)
    s_sz, s_fl = torch.from_numpy(sizes).to(dev, torch.int32), torch.from_numpy(flips).to(dev, torch.int32)
    static = tuple(t.clone() for t in enc.encode(s_lab, s_p2, s_sz, s_fl).prepared)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):                                  # a host synchronisation inside would fail the capture
        e = enc.encode(s_lab, s_p2, s_sz, s_fl, out=static)
    for seed in (32, 33):
        labels2, P22, sizes2, flips2 = random_batch(seed)
        s_lab.copy_(torch.from_numpy(labels2))
        s_p2.copy_(torch.from_numpy(P22))
        s_sz.copy_(torch.from_numpy(sizes2))
        s_fl.copy_(torch.from_numpy(flips2))
        graph.replay()
        ref = enc.encode(labels2, P22, sizes2, flips2)
        for a, b in zip(e.prepared, ref.prepared):
            assert torch.equal(a, b)
        for name in ("edge_indices", "edge_len", "alphas", "gt_bboxes", "occlusions", "truncations", "obj6", "P2", "status"):
            assert torch.equal(getattr(e, name), getattr(ref, name)), name


def test_captured_trainer_fed_encoded_targets_matches_eager_param_lists():
    """A captured Trainer fed EncodedTargets (new labels and flips every step) against an eager Trainer fed the equivalent
    ParamsLists: the first step's logged losses agree to fp32 rounding, later ones within the captured-step tolerances of
    test_gpu_train.py (the DCN backward's scatter atomics make two runs drift apart in the last bits)."""
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.train import Trainer
    cfg = default_cfg()
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
        labels, P2, sizes, flips = random_batch(100 + step, B=B)
        e = enc.encode(labels, P2, sizes, flips)
        logs_a.append(ta.step(images, e.param_lists())[1])
        logs_b.append(tb.step(images, e, sync_log=False)[1])
    assert tb._graph is not None
    logs_b = [l.resolve() for l in logs_b]
    # the focal-loss sum is accumulated with float atomics (mf_elementwise.cu): hm_loss differs in its last bits from run to
    # run, so the first step's logged values are compared to 1e-5
    for k, v in logs_a[0].items():
        assert abs(v - logs_b[0][k]) <= 1e-5 * max(abs(v), 1e-3), (k, v, logs_b[0][k])
    for i, (la, lb) in enumerate(zip(logs_a, logs_b)):
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
    assert logs_b[2] != logs_b[3]
