"""-m gpu: the CUDA get_iou_3d (csrc/mf_iou3d.cu, monoflex_b200/model/layers/iou_loss.py) and the '3D_IoU' log of the fused
loss against the unmodified reference (tests/golden/iou3d.npz, oracle/make_golden_iou3d.py) and the exact CPU oracle
(oracle/iou3d_oracle.py)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200.config import default_cfg
from monoflex_b200.model.layers.iou_loss import get_iou_3d
from oracle import iou3d_oracle as io
from oracle import monoflex_oracle as mo

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "iou3d.npz")) as z:
        return {k: z[k] for k in z.files}


def assert_close(got, want):
    """every value within 1 float32 ulp of the reference's, or within 1e-9; NaN exactly where the reference has NaN"""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(got), nan), np.nonzero(np.isnan(got) != nan)
    g, w = got[~nan], want[~nan]
    ulp = np.spacing(np.abs(w).astype(np.float32))
    bad = ~((np.abs(g.astype(np.float64) - w) <= ulp) | (np.abs(g.astype(np.float64) - w) <= 1e-9))
    assert not bad.any(), list(zip(g[bad][:5], w[bad][:5]))


def op(a, b):
    return get_iou_3d(torch.as_tensor(a).cuda(), torch.as_tensor(b).cuda()).cpu().numpy()


def test_op_matches_reference_fixture(gold):
    assert_close(op(gold["pred"], gold["target"]), gold["iou"])
    assert_close(op(gold["loss_pred"], gold["loss_target"]), gold["loss_iou"])


def random_pairs(n, seed):
    """seeded encode_box3d pairs: random overlaps, boxes around one centre, and near-coincident copies (the same box moved
    by up to a few float32 ulps of its coordinates, turned by up to 1e-6 rad or scaled by 1 + 1e-6)"""
    g = np.random.Generator(np.random.PCG64(seed))

    def boxes(m):
        return (g.uniform(-np.pi, np.pi, m), np.stack([g.uniform(0.05, 5, m), g.uniform(0.05, 2.5, m), g.uniform(0.05, 2.5, m)], 1),
                np.stack([g.uniform(-20, 20, m), g.uniform(0, 2.5, m), g.uniform(2, 60, m)], 1))

    ra, da, la = boxes(n)
    rb, db, lb = boxes(n)
    kind = g.integers(0, 4, n)
    near = kind == 0                                                   # near-coincident copies
    rb[near] = ra[near] + g.choice([0.0, 1e-7, -1e-6, 1e-6], near.sum())
    db[near] = da[near] * g.choice([1.0, 1.0 + 1e-6, 1.0 - 1e-6], (near.sum(), 1))
    lb[near] = la[near] + g.choice([0.0, 1e-6, -3e-6], (near.sum(), 3))
    centre = kind == 1                                                 # one centre, similar sizes: 6-8 vertex overlaps
    rb[centre] = ra[centre] + g.uniform(-1.5, 1.5, centre.sum())
    db[centre] = da[centre] * g.uniform(0.7, 1.4, (centre.sum(), 3))
    lb[centre] = la[centre] + g.uniform(-0.3, 0.3, (centre.sum(), 3))
    part = kind == 2                                                   # partial overlaps
    lb[part] = la[part] + g.uniform(-3, 3, (part.sum(), 3)) * np.array([1.0, 0.3, 1.0])
    f = lambda r, d, l: mo.encode_box3d(torch.tensor(r, dtype=torch.float32), torch.tensor(d, dtype=torch.float32),
                                        torch.tensor(l, dtype=torch.float32))
    return f(ra, da, la), f(rb, db, lb)


def test_op_matches_oracle_on_random_pairs():
    a, b = random_pairs(10000, seed=31)
    want = io.get_iou_3d(a, b)
    assert (want > 0).mean() > 0.5 and (want > 0.99).sum() > 100      # most pairs overlap, many near-coincident ones
    assert_close(op(a, b), want)


def test_empty_and_input_rejection():
    z = torch.zeros(0, 8, 3, device="cuda")
    out = get_iou_3d(z, z)
    assert out.shape == (0,) and out.is_cuda and out.dtype == torch.float32
    x = torch.zeros(4, 8, 3, device="cuda")
    with pytest.raises(RuntimeError):
        get_iou_3d(x.cpu(), x.cpu())
    with pytest.raises(RuntimeError):
        get_iou_3d(x, x.cpu())
    with pytest.raises(TypeError):
        get_iou_3d(x.double(), x.double())
    with pytest.raises(TypeError):
        get_iou_3d(x.half(), x)
    with pytest.raises(ValueError):
        get_iou_3d(x[:, :, :2], x[:, :, :2])
    with pytest.raises(ValueError):
        get_iou_3d(x.view(4, 24), x.view(4, 24))
    with pytest.raises(ValueError):
        get_iou_3d(x, x[:3])
    from monoflex_b200._lib import call                                # the C entry checks its own arguments
    with pytest.raises(RuntimeError, match="N = -1"):
        call("mf_iou3d_corners", x.data_ptr(), x.data_ptr(), -1, x.data_ptr(), None)


# ------------------------------------------------------------------------------------------------ the loss's '3D_IoU' log
def _loss_case(batch, seed=5):
    from monoflex_b200 import synthetic as syn
    if batch == 1:
        fields = syn.make_train_targets(1, empty_image=-1)
        cls, reg = syn.make_train_predictions(1, fields)
    else:
        fields = syn.make_train_targets(batch, seed=seed)
        cls, reg = syn.make_train_predictions(batch, fields, seed=seed + 1)
    return syn, fields, cls, reg


def _cuda_log(syn, fields, cls, reg):
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    lc = Loss_Computation(default_cfg())
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    _, log = lc({"cls": cls.cuda(), "reg": reg.cuda()}, targets)
    return log


def test_loss_log_matches_reference_fixture(gold):
    from monoflex_b200 import synthetic as syn
    fields = syn.make_train_targets(4)
    cls, reg = syn.make_train_predictions(4, fields)
    log = _cuda_log(syn, fields, cls, reg)
    want = float(gold["log_3D_IoU"])
    assert list(log)[:2] == ["2D_IoU", "3D_IoU"]                       # the reference's log_loss_dict order
    assert abs(log["3D_IoU"] - want) <= 1e-5 * abs(want), (log["3D_IoU"], want)


@pytest.mark.parametrize("batch", [1, 4, 8])
def test_loss_log_matches_oracle(batch):
    syn, fields, cls, reg = _loss_case(batch)
    log = _cuda_log(syn, fields, cls, reg)
    want, per_object = io.loss_iou3d(cls, reg, fields, [syn.KITTI_P2] * batch)
    assert len(per_object) > 0 and np.isfinite(want)
    assert abs(log["3D_IoU"] - want) <= 1e-5 * max(abs(want), 1e-3), (log["3D_IoU"], want)


def test_loss_log_is_deterministic():
    syn, fields, cls, reg = _loss_case(8)
    a = _cuda_log(syn, fields, cls, reg)["3D_IoU"]
    b = _cuda_log(syn, fields, cls, reg)["3D_IoU"]
    assert np.float32(a).view(np.int32) == np.float32(b).view(np.int32)


def test_loss_log_without_objects_is_zero():
    syn, fields, cls, reg = _loss_case(4)
    for f in fields:
        f["reg_mask"] = np.zeros_like(f["reg_mask"])
    assert _cuda_log(syn, fields, cls, reg)["3D_IoU"] == 0.0


def test_captured_train_step_reports_3d_iou():
    """a captured Trainer step carries '3D_IoU' through DeferredLog.snapshot() read late; on the first replay it agrees with
    an eager twin within the tolerance the captured-step test holds the losses to (the DCN backward's atomics make the
    twins' parameters drift apart after the first update, so not bit for bit)"""
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.train import Trainer
    cfg = default_cfg()
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    trainers = []
    for graph in (False, True):
        model = KeypointDetector(cfg).cuda()
        model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        trainers.append(Trainer(model, cfg, loss_scale=128.0, use_cuda_graph=graph, graph_warmup=2))
    ta, tb = trainers
    logs_a, logs_b = [], []
    for _ in range(4):
        logs_a.append(ta.step(images, targets)[1])
        logs_b.append(tb.step(images, targets, sync_log=False)[1])
    assert tb._graph is not None
    logs_b = [l.resolve() for l in logs_b]                             # read after the later replays overwrote the buffer
    for la, lb in zip(logs_a, logs_b):
        assert "3D_IoU" in la and "3D_IoU" in lb
        assert np.isfinite(lb["3D_IoU"]) and 0.0 <= lb["3D_IoU"] <= 1.0
    a, b = logs_a[2]["3D_IoU"], logs_b[2]["3D_IoU"]                    # step 2: the first replay
    assert abs(a - b) <= 0.03 * abs(a) + 1e-6, (a, b)
