"""Loss_Computation (reference: model/head/detector_loss.py:18-493) on two hand-written kernels (csrc/mf_loss.cu).

Same constructor / call interface as the reference: ``loss_dict, log_loss_dict = Loss_Computation(cfg)(predictions,
targets)`` with ``predictions = {'cls': sigmoid-ed heat map [B,3,H,W], 'reg': [B,50,H,W]}`` and ``targets`` the list of
per-image ``ParamsList`` objects of data/datasets/kitti.py:496-521. ``loss_dict`` holds the 11 differentiable loss tensors
of runs/monoflex.yaml:45 (views of one device buffer; ``sum(loss_dict.values()).backward()`` as in engine/trainer.py:109-117
runs the fused backward kernel), ``log_loss_dict`` the reference's logged scalars.

Differences, on purpose:
  * ONE device->host copy per call for the logged scalars instead of the reference's 14+ ``.item()`` syncs;
  * '3D_IoU' (detector_loss.py:333: the mean over the labelled objects of get_iou_3d of the predicted and the label corners,
    shapely polygons in a Python loop there) is computed inside the forward loss kernel from the corners it already builds
    for corner_loss, with the clip of csrc/mf_iou3d.cuh (float64 bird's-eye-view clip, the reference's float32 steps); no
    extra launch, no host read. A simple non-convex ring counts as invalid there, valid in shapely (DESIGN.md §9);
    encode_box3d never builds one. Without any labelled object the value is 0, like the other logged means;
  * a batch without any labelled object (the reference crashes in prepare_predictions) gives 0 for every regression loss
    and gradient and for the logged means, except the logged keypoint_depth_loss: the mean over no valid key-point-depth
    group, NaN as in the reference whenever no group is valid; a batch without any 2D box (the reference raises NameError
    at detector_loss.py:291) gives bbox_loss = 2D_IoU = 0;
  * only the runs/monoflex.yaml loss configuration is built - anything else raises NotImplementedError (no fallback).
"""
import ctypes

import torch

from ..._lib import call, load
from ..layers.utils import Converter_key2channel

LOG_KEYS = ['2D_IoU', '3D_IoU', 'depth_loss', 'keypoint_depth_loss', 'depth_MAE', 'center_MAE', '02_MAE', '13_MAE',
            'lower_MAE', 'hard_MAE', 'soft_MAE', 'mean_MAE']                  # the reference's log_loss_dict order
LOSS_WS_FLOATS = 96                                      # ws96 of mf_loss_forward / mf_loss_backward, include/monoflex_b200.h
LOG_SLOTS = [0, 11, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10]        # out[16 + slot] of each LOG_KEYS entry, include/monoflex_b200.h
OBJ_FIELDS = [("cls_ids", 1), ("target_centers", 2), ("2d_bboxes", 4), ("reg_mask", 1), ("trunc_mask", 1), ("dimensions", 3),
              ("locations", 3), ("rotys", 1), ("offset_3D", 2), ("orientations", 8), ("keypoints_depth_mask", 3),
              ("keypoints", 30)]          # column order of the packed label table, include/monoflex_b200.h


def make_loss_evaluator(cfg):
    return Loss_Computation(cfg=cfg)


def _get(ns, name, default):
    return getattr(ns, name, default)


class _FusedLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, cls, reg, hm, obj, img, owner):
        B, C, H, W = reg.shape
        out = torch.zeros(48, dtype=torch.float32, device=reg.device)
        ws = torch.zeros(LOSS_WS_FLOATS, dtype=torch.float32, device=reg.device)
        st = torch.cuda.current_stream().cuda_stream
        call("mf_loss_forward", cls.data_ptr(), hm.data_ptr(), reg.data_ptr(), obj.data_ptr(), img.data_ptr(),
             ctypes.addressof(owner._w11), ctypes.addressof(owner._dm9), B, cls.shape[1], owner.max_objs, H, W, C,
             out.data_ptr(), ws.data_ptr(), st)
        ctx.save_for_backward(cls, reg, hm, obj, img, ws)
        ctx.owner = owner
        return out                                                # [0..10] losses, [16..] logged metrics and counts

    @staticmethod
    def backward(ctx, g_out):
        cls, reg, hm, obj, img, ws = ctx.saved_tensors
        owner = ctx.owner
        B, C, H, W = reg.shape
        g = g_out[:11].contiguous().float()
        need_cls, need_reg = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        grad_cls = torch.empty_like(cls) if need_cls else None
        grad_reg = torch.empty_like(reg) if need_reg else None
        st = torch.cuda.current_stream().cuda_stream
        call("mf_loss_backward", cls.data_ptr(), hm.data_ptr(), reg.data_ptr(), obj.data_ptr(), img.data_ptr(),
             ctypes.addressof(owner._w11), ctypes.addressof(owner._dm9), B, cls.shape[1], owner.max_objs, H, W, C,
             ws.data_ptr(), g.data_ptr(), grad_cls.data_ptr() if need_cls else None,
             grad_reg.data_ptr() if need_reg else None, st)
        return grad_cls, grad_reg, None, None, None, None


class Loss_Computation(object):
    def __init__(self, cfg):
        head = cfg.MODEL.HEAD
        self.key2channel = Converter_key2channel(keys=head.REGRESSION_HEADS, channels=head.REGRESSION_CHANNELS)
        self.max_objs = cfg.DATASETS.MAX_OBJECTS
        self.loss_keys = list(_get(head, "LOSS_NAMES", REF_LOSS_NAMES))
        weights = list(_get(head, "INIT_LOSS_WEIGHT", REF_LOSS_WEIGHTS))
        self.loss_weights = dict(zip(self.loss_keys, weights))
        self._check_config(cfg)
        self._w11 = (ctypes.c_float * 11)(*[float(self.loss_weights[k]) for k in REF_LOSS_NAMES])
        dm = [float(v) for row in head.DIMENSION_MEAN for v in row]
        self._dm9 = (ctypes.c_float * 9)(*dm)

    def _check_config(self, cfg):
        head = cfg.MODEL.HEAD
        want = dict(LOSS_TYPE=["Penalty_Reduced_FocalLoss", "L1", "giou", "L1"], HEATMAP_TYPE='centernet',
                    CORNER_LOSS_DEPTH='soft_combine', TRUNCATION_OFFSET_LOSS='log', MODIFY_INVALID_KEYPOINT_DEPTH=True,
                    UNCERTAINTY_RANGE=[-10, 10], DIMENSION_WEIGHT=[1, 1, 1], LOSS_PENALTY_ALPHA=2, LOSS_BETA=4,
                    DEPTH_MODE='inv_sigmoid', DEPTH_RANGE=[0.1, 100], DIMENSION_REG=['exp', True, False])
        for k, v in want.items():
            got = _get(head, k, v)
            got = list(got) if isinstance(got, (list, tuple)) else got
            if got != v:
                raise NotImplementedError("Loss_Computation: MODEL.HEAD.%s = %r; only %r (runs/monoflex.yaml) is built" % (k, got, v))
        if sorted(self.loss_keys) != sorted(REF_LOSS_NAMES):
            raise NotImplementedError("Loss_Computation: LOSS_NAMES %r; only the 11 losses of runs/monoflex.yaml:45 are built"
                                      % (self.loss_keys,))
        if cfg.INPUT.ORIENTATION != 'multi-bin' or cfg.INPUT.ORIENTATION_BIN_SIZE != 4:
            raise NotImplementedError("Loss_Computation: only 4-bin multi-bin orientation is built")
        if list(self.key2channel.keys) != ['2d_dim', '3d_offset', 'corner_offset', 'corner_uncertainty', '3d_dim', 'ori_cls',
                                           'ori_offset', 'depth', 'depth_uncertainty']:
            raise NotImplementedError("Loss_Computation: regression heads differ from runs/monoflex.yaml:27")

    def prepare_targets(self, targets, device):
        """detector_loss.py:88-114: stack the per-image fields; here additionally packed into the kernel's label table."""
        B = len(targets)

        def st(name):
            return torch.stack([t.get_field(name) for t in targets]).to(device=device, dtype=torch.float32, non_blocking=True)

        hm = st("hm").contiguous()
        cols = [st(name).reshape(B * self.max_objs, n) for name, n in OBJ_FIELDS]
        used = sum(n for _, n in OBJ_FIELDS)
        width = load().mf_loss_obj_cols()
        cols.append(torch.zeros(B * self.max_objs, width - used, dtype=torch.float32, device=device))
        obj = torch.cat(cols, 1).contiguous()
        # per-image calibration (host scalars, cached by value) + pad_size (stacked on the device: no host sync when the
        # targets already live there)
        rows = []
        for t in targets:
            c = t.get_field("calib")
            rows.append((float(c.f_u), float(c.f_v), float(c.c_u), float(c.c_v), float(c.b_x), float(c.b_y)))
        key = (tuple(rows), str(device))
        cache = getattr(self, "_calib_cache", None)
        if cache is None or cache[0] != key:
            rows = torch.tensor(rows, dtype=torch.float32)
            if torch.device(device).type == "cuda":       # through pinned memory: a new batch's cameras do not block the host
                rows = rows.pin_memory().to(device, non_blocking=True)
            cache = self._calib_cache = (key, rows.to(device))
        pad = torch.stack([torch.as_tensor(t.get_field("pad_size")) for t in targets]).to(device=device, dtype=torch.float32,
                                                                                         non_blocking=True).view(B, 2)
        img = torch.cat([cache[1], pad], 1).contiguous()
        return hm, obj, img

    def __call__(self, predictions, targets, prepared=None, sync_log=True):
        """prepared: (hm, obj, img) from `prepare_targets` already on the device (static buffers of a captured training step);
        sync_log=False: no host read here - log_loss_dict is a `DeferredLog` whose `resolve()` does the step's single D2H copy
        when the caller wants the numbers (a CUDA-graph capture cannot contain it)."""
        cls, reg = predictions['cls'], predictions['reg']
        if not (cls.is_cuda and reg.is_cuda):
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        cls, reg = cls.float().contiguous(), reg.float().contiguous()
        if len(targets) != reg.shape[0]:
            raise ValueError("Loss_Computation: %d target lists for a batch of %d" % (len(targets), reg.shape[0]))
        hm, obj, img = prepared if prepared is not None else self.prepare_targets(targets, reg.device)
        if hm.shape != cls.shape:
            raise ValueError("Loss_Computation: heat-map label %s vs prediction %s" % (tuple(hm.shape), tuple(cls.shape)))
        out = _FusedLoss.apply(cls, reg, hm, obj, img, self)
        loss_dict = {k: out[i] for i, k in enumerate(REF_LOSS_NAMES)}
        log = DeferredLog(out.detach())
        return loss_dict, (log.resolve() if sync_log else log)


class DeferredLog(object):
    """the logged scalars of one loss evaluation, still on the device; resolve() -> the reference's log_loss_dict"""

    def __init__(self, out):
        self.out = out
        self._host = None
        self._event = None

    def snapshot(self):
        """Enqueue this evaluation's D2H read now (pinned, asynchronous) and return a log whose resolve() only waits for that
        copy: a captured training step re-uses one device buffer, so a log that is read one step late (the host prepares
        batch i+1 while step i runs) has to be copied out before the next replay overwrites it."""
        snap = DeferredLog(self.out)
        dev = torch.cat([self.out[:11], self.out[16:16 + len(LOG_KEYS)]])
        snap._host = torch.empty(dev.shape, dtype=dev.dtype, pin_memory=True)
        snap._host.copy_(dev, non_blocking=True)
        snap._event = torch.cuda.Event()
        snap._event.record()
        return snap

    def resolve(self):
        out = self.out
        if self._host is not None:
            self._event.synchronize()
            host = self._host
        else:
            host = torch.cat([out[:11], out[16:16 + len(LOG_KEYS)]]).cpu()                # the step's single D2H read
        log_loss_dict = {k: float(host[11 + j]) for k, j in zip(LOG_KEYS, LOG_SLOTS)}
        for i, k in enumerate(REF_LOSS_NAMES):                                            # detector_loss.py:478-480
            if k not in log_loss_dict:
                log_loss_dict[k] = float(host[i])
        return log_loss_dict


REF_LOSS_NAMES = ['hm_loss', 'bbox_loss', 'depth_loss', 'offset_loss', 'orien_loss', 'dims_loss', 'corner_loss',
                  'keypoint_loss', 'keypoint_depth_loss', 'trunc_offset_loss', 'weighted_avg_depth_loss']   # runs/monoflex.yaml:45
REF_LOSS_WEIGHTS = [1, 1, 1, 0.5, 1, 1, 0.2, 1.0, 0.2, 0.1, 0.2]                                           # runs/monoflex.yaml:47
