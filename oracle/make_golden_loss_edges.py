"""TEST TOOLING — tests/golden/loss_edges.npz: the UNMODIFIED reference Loss_Computation (model/head/detector_loss.py, via
oracle/ref_shims.py) on CPU in float32 on every case of oracle/loss_edge_cases.py that the reference can run (all but the
kernel-only ones). Build container only:  python -m oracle.make_golden_loss_edges

Per case `<c>`: `<c>/loss_<name>` (11) and `<c>/log_<key>` (the 12 logged metrics; '3D_IoU' through
oracle.iou3d_oracle.ExactPolygon in place of shapely, as oracle/make_golden_iou3d.py does), `<c>/grad_reg` [11, N_obj, 50]:
the gradient of each loss alone w.r.t. `reg` at every labelled centre, `<c>/grad_cls_sample`: the gradient of hm_loss
w.r.t. `cls` at every 97th element, `<c>/checksum`: the builder's input checksum (a drifting builder fails loudly).

The reference stops in pdb.set_trace() on a NaN or Inf loss (detector_loss.py:485-489); all_trunc has a NaN offset_loss
by construction, so set_trace is stubbed and the cases that may reach it are listed in NAN_LOSS."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims as rs                     # noqa: E402
from oracle import loss_edge_cases as le               # noqa: E402
from oracle.iou3d_oracle import ExactPolygon           # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "loss_edges.npz")
NAN_LOSS = ("all_trunc",)
LOG_KEYS = ['2D_IoU', '3D_IoU', 'depth_loss', 'keypoint_depth_loss', 'depth_MAE', 'center_MAE', '02_MAE', '13_MAE',
            'lower_MAE', 'hard_MAE', 'soft_MAE', 'mean_MAE']
LOSS_NAMES = ['hm_loss', 'bbox_loss', 'depth_loss', 'offset_loss', 'orien_loss', 'dims_loss', 'corner_loss',
              'keypoint_loss', 'keypoint_depth_loss', 'trunc_offset_loss', 'weighted_avg_depth_loss']


def ref_targets(fields, calibs_P):
    """reference ParamsLists with each image's own Calibration (data/datasets/kitti_utils.py:211-218 fields)"""
    from structures.params_3d import ParamsList
    from data.datasets.kitti_utils import Calibration
    out = []
    for f, P in zip(fields, calibs_P):
        t = ParamsList((1280, 384), is_train=True)
        for k, v in f.items():
            t.add_field("2d_bboxes" if k == "bboxes" else k, torch.from_numpy(np.ascontiguousarray(v)))
        c = Calibration.__new__(Calibration)
        P = np.array(P, np.float64)
        c.P = P
        c.c_u, c.c_v, c.f_u, c.f_v = P[0, 2], P[1, 2], P[0, 0], P[1, 1]
        c.b_x, c.b_y = P[0, 3] / (-c.f_u), P[1, 3] / (-c.f_v)
        t.add_field("calib", c)
        out.append(t)
    return out


def run_case(lc, dl, name):
    case = le.build(name)
    stops = []
    dl.pdb.set_trace = lambda: stops.append(name)
    cls, reg = case["cls"].clone().requires_grad_(True), case["reg"].clone().requires_grad_(True)
    loss, log = lc({"cls": cls, "reg": reg}, ref_targets(case["fields"], case["calibs_P"]))
    assert bool(stops) == (name in NAN_LOSS), (name, stops)
    out = {"checksum": np.array(le.checksum(case))}
    out.update({"loss_" + k: np.float32(loss[k].item()) for k in LOSS_NAMES})
    out.update({"log_" + k: np.float32(log[k]) for k in LOG_KEYS})
    rows = []
    for k in LOSS_NAMES:
        g, = torch.autograd.grad(loss[k], reg, retain_graph=True, allow_unused=True)
        rows.append(le.grads_at_centres(torch.zeros_like(reg) if g is None else g, case).astype(np.float32))
    out["grad_reg"] = np.stack(rows)
    gc, = torch.autograd.grad(loss["hm_loss"], cls)
    out["grad_cls_sample"] = gc.reshape(-1)[::97].numpy().astype(np.float32)
    return out


def main():
    cfg = rs.reference_cfg()
    sys.modules["shapely.geometry"].Polygon = ExactPolygon
    import model.layers.iou_loss as il
    il.Polygon = ExactPolygon                         # bound by `from shapely.geometry import Polygon` at import time
    import model.head.detector_loss as dl
    dl.get_iou_3d = il.get_iou_3d
    lc = dl.Loss_Computation(cfg)
    torch.manual_seed(0)
    out = {}
    for name in le.CASES:
        res = run_case(lc, dl, name)
        out.update({"%s/%s" % (name, k): v for k, v in res.items()})
        print("%-12s %2d objects  total %s  NaN: %s" % (
            name, res["grad_reg"].shape[1], sum(res["loss_" + k] for k in LOSS_NAMES),
            [k for k, v in res.items() if np.ndim(v) == 0 and v.dtype != np.dtype("<U64") and np.isnan(v)]))
    np.savez_compressed(OUT, **out)


if __name__ == "__main__":
    main()
