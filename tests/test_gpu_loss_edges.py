"""-m gpu: the fused training loss (csrc/mf_loss.cu) at its branch points (oracle/loss_edge_cases.py) against float64
autograd through the CPU oracle (pinned to the unmodified reference at the same inputs by tests/test_loss_edges_host.py)
and against the reference's own float32 numbers (tests/golden/loss_edges.npz).

Backward is checked loss by loss (one-hot upstream gradient) on the whole [B, 50, H, W] gradient, so a wrong
sub-gradient on one channel of one object cannot hide under a larger term: |g - ref| <= 1e-5 max|ref_k[n]| + 1e-9 on
every object's row n of centre channels (each row's tolerance from its own gradient), exactly 0 on every other pixel and wherever a branch cuts the float64 gradient (clamped depths and uncertainties,
relu at 0, detached invalid key-point depths; oracle/loss_edge_cases.ZEROS), non-zero on a closed clamp bound. Ties
are built exactly, so the kernel has to split the gradient like torch's min / max (half to each side) to stay within the tolerance."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200.config import default_cfg
from oracle import iou3d_oracle
from oracle import loss_edge_cases as le
from oracle import monoflex_oracle as mo

pytestmark = pytest.mark.gpu

LOG_KEYS = ['2D_IoU', '3D_IoU', 'depth_loss', 'keypoint_depth_loss', 'depth_MAE', 'center_MAE', '02_MAE', '13_MAE',
            'lower_MAE', 'hard_MAE', 'soft_MAE', 'mean_MAE']


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "loss_edges.npz")) as z:
        return {k: z[k] for k in z.files}


def targets_of(case):
    from monoflex_b200.structures import Calibration, ParamsList
    out = []
    for f, P in zip(case["fields"], case["calibs_P"]):
        t = ParamsList((1280, 384), is_train=True)
        for k, v in f.items():
            t.add_field("2d_bboxes" if k == "bboxes" else k, torch.from_numpy(np.ascontiguousarray(v)))
        t.add_field("calib", Calibration(P))
        out.append(t.to("cuda"))
    return out


def run_kernel(case, cls_grad=True):
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    lc = Loss_Computation(default_cfg())
    c = case["cls"].clone().cuda().requires_grad_(cls_grad)
    r = case["reg"].clone().cuda().requires_grad_(True)
    loss, log = lc({"cls": c, "reg": r}, targets_of(case))
    return loss, log, c, r


def run_oracle(case):
    c = case["cls"].double().requires_grad_(True)
    r = case["reg"].double().requires_grad_(True)
    loss, log = mo.loss_computation(c, r, case["fields"], case["calibs_P"])
    return loss, log, c, r


def close(a, b, rtol=1e-5):
    a, b = np.float64(a), np.float64(b)
    if np.isnan(b):
        return bool(np.isnan(a))
    return bool(abs(a - b) <= rtol * abs(b) + 1e-30)


def grads(loss, inputs, k):
    gs = torch.autograd.grad(loss[k], inputs, retain_graph=True, allow_unused=True)
    return [torch.zeros_like(x) if g is None else g for x, g in zip(inputs, gs)]


def assert_grad_matches(g, ref, what):
    """per object row n of the gradient at the labelled centres: |g[n] - ref[n]| <= 1e-5 max|ref[n]| + 1e-9, so no row's
    tolerance is set by another object's (clamped uncertainties and the F.normalize eps give 1e4..1e12 gradients)"""
    g, ref = np.asarray(g, np.float64), np.asarray(ref, np.float64)
    assert np.isfinite(g).all(), what
    tol = 1e-5 * np.abs(ref).max(axis=1, keepdims=True) + 1e-9
    err = np.abs(g - ref)
    n, ch = np.unravel_index(int((err / tol).argmax()), err.shape)
    assert np.all(err <= tol), (what, "object row", n, "channel", ch, g[n, ch], ref[n, ch], tol[n, 0])


def assert_cls_grad_matches(g, ref, what):
    """the heat-map gradient is one focal term: |g - ref| <= 1e-5 max|ref| + 1e-9"""
    g, ref = g.detach().cpu().double().numpy(), ref.detach().cpu().double().numpy()
    assert np.abs(g - ref).max() <= 1e-5 * np.abs(ref).max() + 1e-9, what


def assert_branch_zeros(g, ref, case, k):
    """exact zeros where a branch cuts the gradient (oracle/loss_edge_cases.ZEROS), non-zero on a closed clamp bound"""
    rows = {(b, i): n for n, (b, i) in enumerate((b, i) for b, f in enumerate(case["fields"]) for i in le._objects(f))}
    for b, i, branch in case["table"]:
        for table, want_zero in ((le.ZEROS, True), (le.NONZERO, False)):
            for losses, chans in table.get(branch, []):
                if losses is None or k in losses:
                    n = rows[(b, i)]
                    if want_zero:
                        assert np.all(ref[n, chans] == 0) and np.all(g[n, chans] == 0), (branch, k, g[n, chans])
                    else:
                        assert np.all(ref[n, chans] != 0) and np.all(g[n, chans] != 0), (branch, k, g[n, chans])


def at_centres(case, shape):
    m = torch.zeros(shape, dtype=torch.bool)
    for b, x, y in le.centers_of(case):
        m[b, :, y, x] = True
    return m


def check_case(case, gold=None):
    loss, log, c, r = run_kernel(case)
    rl, rlog, rc, rr = run_oracle(case)
    name = case["name"]
    for k in mo.LOSS_NAMES:
        assert close(loss[k].item(), rl[k].item()), (k, loss[k].item(), rl[k].item())
        if gold is not None:
            assert close(loss[k].item(), gold["%s/loss_%s" % (name, k)]), (k, loss[k].item(), gold["%s/loss_%s" % (name, k)])
    iou, _ = iou3d_oracle.loss_iou3d(case["cls"], case["reg"], case["fields"], case["calibs_P"])
    for k in LOG_KEYS:
        ref = iou if k == "3D_IoU" else rlog[k].item()
        assert close(log[k], ref), (k, log[k], ref)
        if gold is not None:
            assert close(log[k], gold["%s/log_%s" % (name, k)]), (k, log[k], gold["%s/log_%s" % (name, k)])
    off = ~at_centres(case, r.shape).cuda()
    for k in mo.LOSS_NAMES:
        gc, gr = grads(loss, [c, r], k)
        assert gr[off].abs().sum().item() == 0, (name, k)         # nothing off the centres
        if not torch.isfinite(rl[k]):                 # a NaN loss (mean of an empty set) sends no gradient
            assert gr.abs().sum().item() == 0 and gc.abs().sum().item() == 0, k
            continue
        rgc, rgr = grads(rl, [rc, rr], k)
        g, ref = le.grads_at_centres(gr, case), le.grads_at_centres(rgr, case)
        assert_grad_matches(g, ref, (name, k, "reg"))
        assert_branch_zeros(g, ref, case, k)
        assert_cls_grad_matches(gc, rgc, (name, k, "cls"))
    return loss, log, r


@pytest.mark.parametrize("name", le.CASES)
def test_loss_edges_vs_float64_oracle_and_reference(name, gold):
    check_case(le.build(name), gold)


def test_shared_centre_gradient_is_the_sum():
    """three objects on one pixel of a full image: the kernel's gradient there is the float64 autograd sum over the three
    objects, and each of them contributes (without objects 17 and 33 the pixel's gradient moves far beyond tolerance)"""
    case = le.build("full")
    b, x, y = le.centers_of(case)[5]
    assert [le.centers_of(case)[i] for i in (17, 33)] == [(b, x, y)] * 2

    def pixel_grad(cs, run):
        loss, _, _, r = run(cs)
        g, = torch.autograd.grad(sum(v for k, v in loss.items() if k != "hm_loss"), r)
        return g[b, :, y, x].detach().cpu().double()

    got, want = pixel_grad(case, run_kernel), pixel_grad(case, run_oracle)
    assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()
    alone = dict(case, fields=[dict(f) for f in case["fields"]])
    alone["fields"][0]["reg_mask"] = case["fields"][0]["reg_mask"].copy()
    alone["fields"][0]["reg_mask"][[17, 33]] = 0
    one = pixel_grad(alone, run_oracle)
    assert (got - one).abs().max().item() > 1e-2 * want.abs().max().item()


def test_grad_cls_absent_without_requires_grad():
    case = le.build("calib")
    loss, _, c, r = run_kernel(case, cls_grad=False)
    sum(loss.values()).backward()
    assert c.grad is None and r.grad is not None and r.grad.abs().sum().item() > 0


def test_kernel_only_no_object():
    """no labelled object in the batch (the reference crashes): every regression loss and its gradient is exactly 0,
    hm_loss is the focal term; the logged means are 0 except keypoint_depth_loss, the mean over no valid group (NaN)"""
    case = le.build("no_object")
    loss, log, c, r = run_kernel(case)
    hl, npos = mo.focal_loss(case["cls"].double(), torch.stack([torch.from_numpy(f["hm"]) for f in case["fields"]]))
    assert close(loss["hm_loss"].item(), (hl / torch.clamp(npos, 1)).item())
    assert all(loss[k].item() == 0 for k in mo.LOSS_NAMES[1:])
    assert all(log[k] == 0 for k in LOG_KEYS if k != "keypoint_depth_loss") and np.isnan(log["keypoint_depth_loss"])
    g, = torch.autograd.grad(sum(loss.values()), r)
    assert g.abs().sum().item() == 0


def test_kernel_only_no_box2d():
    """no object has a 2D box (the reference raises NameError): bbox_loss and 2D_IoU are 0 and send no gradient, every
    other loss and log matches the float64 oracle"""
    case = le.build("no_box2d")
    loss, log, c, r = run_kernel(case)
    rl, rlog, rc, rr = run_oracle(case)
    assert loss["bbox_loss"].item() == 0 and log["2D_IoU"] == 0
    for k in mo.LOSS_NAMES[2:]:
        assert close(loss[k].item(), rl[k].item()), k
    for k in LOG_KEYS[2:]:
        assert close(log[k], rlog[k].item()), k
    gb, = torch.autograd.grad(loss["bbox_loss"], r, retain_graph=True)
    assert gb.abs().sum().item() == 0
    for k in mo.LOSS_NAMES[2:]:
        g, ref = grads(loss, [r], k)[0], grads(rl, [rr], k)[0]
        assert_grad_matches(le.grads_at_centres(g, case), le.grads_at_centres(ref, case), k)


def test_batch_of_64_and_the_limit():
    """B = 64 (2560 object slots, ranks far from the image index, a different f_u per image) matches the float64
    oracle; B = 65 is refused with a RuntimeError before any launch, and the same batch then evaluates as before"""
    case = le.wide_batch(64)
    loss, log, c, r = run_kernel(case)
    rl, rlog, rc, rr = run_oracle(case)
    for k in mo.LOSS_NAMES:
        assert close(loss[k].item(), rl[k].item()), (k, loss[k].item(), rl[k].item())
    w = torch.tensor([0.3, 1.7, 0.9, 2.0, 0.5, 1.1, 3.0, 0.7, 1.3, 4.0, 0.2], dtype=torch.float64)
    g, = torch.autograd.grad(sum(float(wk) * loss[k] for wk, k in zip(w, mo.LOSS_NAMES)), r)
    ref, = torch.autograd.grad(sum(wk * rl[k] for wk, k in zip(w, mo.LOSS_NAMES)), rr)
    assert_grad_matches(le.grads_at_centres(g, case), le.grads_at_centres(ref, case), "B=64")
    assert g[~at_centres(case, g.shape).cuda()].abs().sum().item() == 0
    big = le.wide_batch(65)
    with pytest.raises(RuntimeError, match="batch 65"):
        run_kernel(big)
    torch.cuda.synchronize()
    again, _, _, _ = run_kernel(case)
    assert all(close(again[k].item(), loss[k].item()) for k in mo.LOSS_NAMES)   # hm_loss sums with atomics: not bitwise


def test_workspace_stays_in_bounds_at_b64():
    """the C entry points at B = 64 with a workspace of exactly LOSS_WS_FLOATS floats and a 48-float output, each followed
    by a sentinel-filled guard region: nothing past either is written, and the per-image key-point f_u (by rank among
    the images with objects, anno_encoder.py:186) sits in ws[24 + b] for all 64 images"""
    from monoflex_b200._lib import call
    from monoflex_b200.model.head.detector_loss import LOSS_WS_FLOATS, Loss_Computation
    case = le.wide_batch(64)
    lc = Loss_Computation(default_cfg())
    hm, obj, img = lc.prepare_targets(targets_of(case), torch.device("cuda"))
    cls, reg = case["cls"].cuda().contiguous(), case["reg"].cuda().contiguous()
    B, C, H, W = reg.shape
    sentinel = -7.25
    out = torch.full((48 + 256,), sentinel, device="cuda")
    out[:48] = 0
    ws = torch.full((LOSS_WS_FLOATS + 256,), sentinel, device="cuda")
    ws[:LOSS_WS_FLOATS] = 0
    st = torch.cuda.current_stream().cuda_stream
    args = (cls.data_ptr(), hm.data_ptr(), reg.data_ptr(), obj.data_ptr(), img.data_ptr(), ctypes.addressof(lc._w11),
            ctypes.addressof(lc._dm9), B, cls.shape[1], lc.max_objs, H, W, C)
    call("mf_loss_forward", *args, out.data_ptr(), ws.data_ptr(), st)
    gl = torch.ones(11, device="cuda")
    gc, gr = torch.empty_like(cls), torch.empty_like(reg)
    call("mf_loss_backward", *args, ws.data_ptr(), gl.data_ptr(), gc.data_ptr(), gr.data_ptr(), st)
    torch.cuda.synchronize()
    assert (ws[LOSS_WS_FLOATS:] == sentinel).all() and (out[48:] == sentinel).all()
    assert (ws[:LOSS_WS_FLOATS] != sentinel).all()
    owners = [b for b, f in enumerate(case["fields"]) if f["reg_mask"].any()]
    fu = img[:, 0].cpu()
    want = torch.stack([fu[sum(1 for o in owners if o < b)] for b in range(B)])
    assert torch.equal(ws[24:24 + B].cpu(), want) and owners[-1] == B - 1
