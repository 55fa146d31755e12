"""CPU: pin oracle.loss_computation against the UNMODIFIED reference Loss_Computation at the loss's branch points
(oracle/loss_edge_cases.py -> oracle/make_golden_loss_edges.py -> tests/golden/loss_edges.npz): clamps, relus, ties, wraps,
per-image calibrations, full images, shared centres and the degenerate normalisers, in float32 and float64. The GPU test
(tests/test_gpu_loss_edges.py) then uses the float64 oracle as its reference."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import iou3d_oracle
from oracle import loss_edge_cases as le
from oracle import monoflex_oracle as mo

LOG_KEYS = ['2D_IoU', '3D_IoU', 'depth_loss', 'keypoint_depth_loss', 'depth_MAE', 'center_MAE', '02_MAE', '13_MAE',
            'lower_MAE', 'hard_MAE', 'soft_MAE', 'mean_MAE']


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "loss_edges.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def cases():
    return {}


def get(cases, name):
    if name not in cases:
        cases[name] = le.build(name)
    return cases[name]


def close(a, b, rtol):
    """same NaN positions, elsewhere |a - b| <= rtol |b| (1e-30 absolute floor for exact zeros)"""
    a, b = np.float64(a), np.float64(b)
    if np.isnan(b):
        return bool(np.isnan(a))
    return bool(abs(a - b) <= rtol * abs(b) + 1e-30)


def oracle_run(case, dtype):
    cls = case["cls"].to(dtype).requires_grad_(True)
    reg = case["reg"].to(dtype).requires_grad_(True)
    loss, log = mo.loss_computation(cls, reg, case["fields"], case["calibs_P"])
    return cls, reg, loss, log


@pytest.mark.parametrize("name", le.CASES + le.KERNEL_ONLY)
def test_builder_is_deterministic_and_keeps_its_margins(name, cases, gold):
    case = get(cases, name)
    le.check_margins(case)
    assert le.checksum(le.build(name)) == le.checksum(case)
    if name in le.CASES:
        assert str(gold[name + "/checksum"]) == le.checksum(case), "the builder drifted from tests/golden/loss_edges.npz"
        assert gold[name + "/grad_reg"].shape == (11, len(case["table"]), 50)


def test_builder_covers_every_branch(cases):
    branches = {t[2] for t in get(cases, "kinks")["table"]}
    want = {r.__name__[2:] for r in le.KINKS} | {"corner", "plain+shared_centre"}
    assert want <= branches, want - branches
    full = get(cases, "full")
    assert len(le._objects(full["fields"][0])) == le.M and le._objects(full["fields"][6]) == [le.M - 1]
    assert sum(t[2].endswith("shared_centre") for t in full["table"]) == 3
    calib = get(cases, "calib")
    assert [bool(f["reg_mask"].any()) for f in calib["fields"]] == [False, True, False, True, True]
    fu = [P[0][0] for P in calib["calibs_P"]]
    assert len(set(fu)) == 5 and len({tuple(f["pad_size"]) for f in calib["fields"]}) == 5
    assert all(f["trunc_mask"][f["reg_mask"] == 1].all() for f in get(cases, "all_trunc")["fields"])
    assert all(f["keypoints_depth_mask"].sum() == 0 for f in get(cases, "no_valid_kd")["fields"])


def test_margin_check_rejects_values_near_a_boundary(cases):
    """an undeclared near-tie (predicted direct depth within 1e-5 of the label) and a declared tie that is not exact"""
    case = dict(get(cases, "calib"))
    b, i = 1, le._objects(case["fields"][1])[0]
    x, y = case["fields"][b]["target_centers"][i]
    reg = case["reg"].clone()
    reg[b, 48, y, x] = -float(np.log(case["fields"][b]["locations"][i, 2] * (1 + 1e-5)))
    with pytest.raises(AssertionError, match="abs_depth"):
        le.check_margins(dict(case, reg=reg))
    with pytest.raises(AssertionError, match="declared tie is not exact"):
        le.check_margins(dict(case, ties={(b, i): {"abs_off0"}}))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("name", le.CASES)
def test_oracle_matches_reference_at_edges(name, dtype, cases, gold):
    """the 11 losses, the 11 logged metrics the oracle states, the per-loss gradients at every centre and the heat-map
    gradient vs the reference's float32 run; NaN exactly where the reference has it. float32: same arithmetic up to
    summation order; float64: the fixture's own float32 rounding is the error"""
    case = get(cases, name)
    cls, reg, loss, log = oracle_run(case, dtype)
    rtol = 1e-5
    for k in mo.LOSS_NAMES:
        assert close(loss[k].item(), gold["%s/loss_%s" % (name, k)], rtol), (k, loss[k].item(), gold["%s/loss_%s" % (name, k)])
    for k in LOG_KEYS:
        if k == "3D_IoU":
            continue
        assert close(log[k].item(), gold["%s/log_%s" % (name, k)], rtol), (k, log[k].item(), gold["%s/log_%s" % (name, k)])
    ref = gold[name + "/grad_reg"].astype(np.float64)
    for n, k in enumerate(mo.LOSS_NAMES):
        if not torch.isfinite(loss[k]):
            assert np.all(ref[n] == 0)
            continue
        g, = torch.autograd.grad(loss[k], reg, retain_graph=True, allow_unused=True)
        g = le.grads_at_centres(torch.zeros_like(reg) if g is None else g, case)
        tol = 1e-5 * np.abs(ref[n]).max(axis=1, keepdims=True) + 1e-9       # per object row: its own gradient's scale
        err = np.abs(g - ref[n])
        row = int((err / tol).max(axis=1).argmax())
        assert np.all(err <= tol), (k, "object row", row, g[row], ref[n, row])
    gc, = torch.autograd.grad(loss["hm_loss"], cls)
    ref = gold[name + "/grad_cls_sample"]
    assert np.abs(gc.reshape(-1)[::97].double().numpy() - ref).max() <= 1e-5 * np.abs(ref).max()


@pytest.mark.parametrize("name", le.CASES)
def test_iou3d_oracle_matches_reference_at_edges(name, cases, gold):
    case = get(cases, name)
    iou, _ = iou3d_oracle.loss_iou3d(case["cls"], case["reg"], case["fields"], case["calibs_P"])
    assert close(iou, gold[name + "/log_3D_IoU"], 1e-5), (iou, gold[name + "/log_3D_IoU"])


def test_degenerate_sets_are_nan_in_the_reference(gold):
    """what the GPU test holds the kernel to: a NaN offset_loss with every other loss finite when every object is
    truncated, a NaN logged keypoint_depth_loss with a finite loss when no key-point-depth group is valid"""
    want = {"all_trunc": {"loss_offset_loss"}, "no_valid_kd": {"log_keypoint_depth_loss"}}
    for name in le.CASES:
        nan = {k.split("/")[1] for k in gold if k.startswith(name + "/l") and np.isnan(gold[k])}
        assert nan == want.get(name, set()), (name, nan)
