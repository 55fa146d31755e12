"""Heat-map helpers with the reference's names (model/layers/utils.py:22-145), backed by the fused CUDA decode kernel.
`select_topk` uses floor division for ys / class ids (torch-1.4 semantics the reference relies on, SURVEY H5) and the
tie rule (score desc, index asc)."""
import ctypes

import torch

from ..._lib import call, stream


class Converter_key2channel(object):
    def __init__(self, keys, channels):
        self.keys = [k for group in keys for k in group]
        self.channels = [c for group in channels for c in group]

    def __call__(self, key):
        i = self.keys.index(key)
        s = sum(self.channels[:i])
        return slice(s, s + self.channels[i], 1)


def sigmoid_hm(hm_features):
    x = hm_features.float().contiguous()
    call("mf_sigmoid_clamp", x.data_ptr(), x.numel(), stream())
    return x


class DecodeWorkspace(object):
    """Caller-owned output / scratch buffers of mf_decode_detections for a fixed (B, C, K, R). With `n_modes` (the
    number of estimators of one mf_decode_detections_depths call) the per-mode outputs result, depth_err and min_unc
    take a leading mode dimension: [n_modes, B, K, ...]. With `eval_slots` = M > 0 it also holds the outputs of
    mf_eval_depth_errors for M object slots per image: depth_errors [13, B*M] and depth_counts [B], the second row of
    `counts` [2, B] whose first row is `count`, so one device-to-host copy reads both."""

    def __init__(self, B, C, K, R, device, n_modes=None, eval_slots=0):
        f = dict(dtype=torch.float32, device=device)
        self.B, self.C, self.K, self.R, self.n_modes, self.eval_slots = B, C, K, R, n_modes, eval_slots
        lead = () if n_modes is None else (n_modes,)
        slabs = 8     # MF_DECODE_SLABS: stage 1 splits every (image, class) plane into 8 pixel ranges
        self.ws_score = torch.empty(B * C * K * slabs, **f)
        self.ws_idx = torch.empty(B * C * K * slabs, dtype=torch.int32, device=device)
        self.scores, self.clses = torch.empty(B, K, **f), torch.empty(B, K, **f)
        self.ys, self.xs = torch.empty(B, K, **f), torch.empty(B, K, **f)
        self.inds = torch.empty(B, K, dtype=torch.long, device=device)
        self.pois = torch.empty(B, K, R, **f)
        self.result = torch.empty(*lead, B, K, 14, **f)
        if eval_slots:
            self.counts = torch.empty(2, B, dtype=torch.int32, device=device)
            self.count, self.depth_counts = self.counts[0], self.counts[1]
            self.depth_errors = torch.empty(len(EVAL_DEPTH_KEYS), B * eval_slots, **f)
        else:
            self.count = torch.empty(B, dtype=torch.int32, device=device)
            self.counts = self.depth_counts = self.depth_errors = None
        self.depth_err = torch.empty(*lead, B, K, **f)
        self.proj = torch.empty(B, K, 2, **f)
        self.min_unc = torch.empty(*lead, B, K, dtype=torch.int32, device=device)


# OUTPUT_DEPTH estimators of the decode kernel (detector_infer.py:148-209), in the order of the C ABI's `depth_mode`
DEPTH_MODES = ('soft', 'hard', 'mean', 'oracle', 'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02',
               'keypoints_13')
ENSEMBLE_DEPTH_MODES = DEPTH_MODES[:4]
# keys of PostProcessor.evaluate_3D_depths' dict (detector_infer.py:341-357), in the row order of mf_eval_depth_errors
EVAL_DEPTH_KEYS = ('direct', 'direct_sigma', 'keypoint_center', 'keypoint_02', 'keypoint_13', 'keypoint_center_sigma',
                   'keypoint_02_sigma', 'keypoint_13_sigma', 'sigma_min', 'sigma_weighted', 'mean', 'min', 'target')


def decode_detections(heat, reg, calib, pad, size, dim_mean, K, thresh, apply_sigmoid=False, ws=None, depth_mode='soft',
                      gt=None):
    """nms_hm + select_topk + select_point_of_interest + 3D decode in two kernels. All arguments are CUDA tensors.
    `depth_mode` is one of DEPTH_MODES; 'oracle' needs `gt` [B, G, 7] fp32 = (valid, class, x1, y1, x2, y2, z) per
    ground-truth slot of every image. A tuple of distinct DEPTH_MODES decodes all of them from one NMS / top-k / POI
    gather: the workspace's result, depth_err and min_unc then hold one [B, K, ...] block per mode, in the tuple's order,
    each equal to the single-mode decode of that mode."""
    B, C, H, W = heat.shape
    R = reg.shape[1]
    several = isinstance(depth_mode, (tuple, list))
    modes = tuple(depth_mode) if several else (depth_mode,)
    for m in modes:
        if m not in DEPTH_MODES:
            raise ValueError("depth_mode %r is not one of %s" % (m, DEPTH_MODES))
    if not modes or len(set(modes)) != len(modes):
        raise ValueError("depth_mode %r: give one or more distinct modes" % (depth_mode,))
    if 'oracle' in modes:
        if gt is None or gt.dim() != 3 or tuple(gt.shape[::2]) != (B, 7) or gt.dtype != torch.float32 \
                or not gt.is_contiguous():
            raise ValueError("the oracle depth needs gt as a contiguous float32 [B, G, 7] tensor")
    n_modes = len(modes) if several else None
    if ws is None or (ws.B, ws.C, ws.K, ws.R, getattr(ws, 'n_modes', None)) != (B, C, K, R, n_modes):
        ws = DecodeWorkspace(B, C, K, R, heat.device, n_modes)
    gt_ptr, G = (gt.data_ptr(), gt.shape[1]) if gt is not None else (None, 0)
    if n_modes is None:
        name, mode_args = "mf_decode_detections", (DEPTH_MODES.index(depth_mode),)
    else:
        name, mode_args = "mf_decode_detections_depths", ((ctypes.c_int * n_modes)(*map(DEPTH_MODES.index, modes)), n_modes)
    call(name, heat.data_ptr(), reg.data_ptr(), calib.data_ptr(), pad.data_ptr(), size.data_ptr(), dim_mean.data_ptr(),
         B, C, H, W, R, K, float(thresh), 1 if apply_sigmoid else 0, *mode_args, gt_ptr, G, ws.ws_score.data_ptr(),
         ws.ws_idx.data_ptr(), ws.scores.data_ptr(), ws.inds.data_ptr(), ws.clses.data_ptr(), ws.ys.data_ptr(),
         ws.xs.data_ptr(), ws.pois.data_ptr(), ws.result.data_ptr(), ws.count.data_ptr(), ws.depth_err.data_ptr(),
         ws.proj.data_ptr(), ws.min_unc.data_ptr(), stream())
    return ws


def eval_depth_errors(reg, calib, dim_mean, gt, out=None, counts=None):
    """PostProcessor.evaluate_3D_depths at the ground-truth centres in one kernel (asynchronous). reg [B, 50, H, W],
    calib [B, 6], dim_mean [C, 3] and gt [B, M, 5] = (reg_mask, cls_id, x, y, z) are float32 CUDA tensors. Returns
    (out [13, B*M], counts [B] int32): the valid slots' errors compacted in the order of reg_mask.view(-1), one row per
    key of EVAL_DEPTH_KEYS, and the valid slots of each image. Slots past sum(counts) are not written."""
    B, R, H, W = reg.shape
    if gt.dim() != 3 or gt.shape[0] != B or gt.shape[2] != 5 or gt.dtype != torch.float32 or not gt.is_contiguous():
        raise ValueError("eval_depth_errors needs gt as a contiguous float32 [B, M, 5] tensor, got %s %s"
                         % (tuple(gt.shape), gt.dtype))
    M = gt.shape[1]
    if out is None:
        out = torch.empty(len(EVAL_DEPTH_KEYS), B * M, dtype=torch.float32, device=reg.device)
        counts = torch.empty(B, dtype=torch.int32, device=reg.device)
    call("mf_eval_depth_errors", reg.data_ptr(), calib.data_ptr(), dim_mean.data_ptr(), gt.data_ptr(), B, M,
         dim_mean.shape[0], H, W, R, out.data_ptr(), counts.data_ptr(), stream())
    return out, counts


def depth_error_dict(table, counts):
    """{key: 1-D tensor} of the first sum(counts) columns of an eval_depth_errors table: one copy, the keys are its rows"""
    rows = table[:, :sum(counts)].clone()
    return {k: rows[i] for i, k in enumerate(EVAL_DEPTH_KEYS)}


def _dummy_decode_inputs(heat):
    B = heat.shape[0]
    dev = heat.device
    calib = torch.ones(B, 6, device=dev)
    z2 = torch.zeros(B, 2, device=dev)
    return calib, z2, torch.ones(B, 2, device=dev), torch.ones(heat.shape[1], 3, device=dev)


def nms_hm(heat_map, kernel=3, reso=1):
    """heat * (max_pool2d(heat, 3, 1, 1) == heat) (utils.py:45-58). The fused decode applies the same test itself; NMS
    is idempotent, so select_topk(nms_hm(x)) == select_topk(x)."""
    if int(kernel / reso) != 3:
        raise NotImplementedError("only the 3x3 NMS of the reference configuration is built")
    heat = heat_map.float().contiguous()
    out = torch.empty_like(heat)
    call("mf_nms_hm", heat.data_ptr(), out.data_ptr(), heat.shape[0] * heat.shape[1], heat.shape[2], heat.shape[3], stream())
    return out


def select_topk(heat_map, K=100):
    """[N,C,H,W] -> (scores [N,K], inds int64 [N,K], clses, ys, xs); the 3x3 NMS is fused into the selection kernel."""
    heat = heat_map.float().contiguous()
    reg = torch.zeros(heat.shape[0], 50, heat.shape[2], heat.shape[3], device=heat.device)
    ws = decode_detections(heat, reg, *_dummy_decode_inputs(heat), K=K, thresh=0.0)
    return ws.scores, ws.inds, ws.clses, ws.ys, ws.xs


def select_point_of_interest(batch, index, feature_maps):
    """[N,C,H,W] gathered at flat indices [N,K] -> [N,K,C] (utils.py:120-145). Tiny gather; done with torch indexing
    here because the fused decode kernel already returns the POIs on the hot path."""
    w = feature_maps.shape[3]
    if index.dim() == 3:
        index = index[:, :, 1] * w + index[:, :, 0]
    index = index.view(batch, -1).long()
    fm = feature_maps.reshape(batch, feature_maps.shape[1], -1)
    return fm.gather(2, index.unsqueeze(1).expand(-1, fm.shape[1], -1)).permute(0, 2, 1).contiguous()
