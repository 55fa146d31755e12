"""Heat-map helpers with the reference's names (model/layers/utils.py:22-145), backed by the fused CUDA decode kernel.
`select_topk` uses floor division for ys / class ids (torch-1.4 semantics the reference relies on, SURVEY H5) and the
tie rule (score desc, index asc)."""
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
    """Caller-owned output / scratch buffers of mf_decode_detections for a fixed (B, C, K, R)."""

    def __init__(self, B, C, K, R, device):
        f = dict(dtype=torch.float32, device=device)
        self.B, self.C, self.K, self.R = B, C, K, R
        slabs = 8     # MF_DECODE_SLABS: stage 1 splits every (image, class) plane into 8 pixel ranges
        self.ws_score = torch.empty(B * C * K * slabs, **f)
        self.ws_idx = torch.empty(B * C * K * slabs, dtype=torch.int32, device=device)
        self.scores, self.clses = torch.empty(B, K, **f), torch.empty(B, K, **f)
        self.ys, self.xs = torch.empty(B, K, **f), torch.empty(B, K, **f)
        self.inds = torch.empty(B, K, dtype=torch.long, device=device)
        self.pois = torch.empty(B, K, R, **f)
        self.result = torch.empty(B, K, 14, **f)
        self.count = torch.empty(B, dtype=torch.int32, device=device)
        self.depth_err = torch.empty(B, K, **f)
        self.proj = torch.empty(B, K, 2, **f)
        self.min_unc = torch.empty(B, K, dtype=torch.int32, device=device)


# OUTPUT_DEPTH estimators of the decode kernel (detector_infer.py:148-209), in the order of the C ABI's `depth_mode`
DEPTH_MODES = ('soft', 'hard', 'mean', 'oracle', 'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02',
               'keypoints_13')
ENSEMBLE_DEPTH_MODES = DEPTH_MODES[:4]


def decode_detections(heat, reg, calib, pad, size, dim_mean, K, thresh, apply_sigmoid=False, ws=None, depth_mode='soft',
                      gt=None):
    """nms_hm + select_topk + select_point_of_interest + 3D decode in two kernels. All arguments are CUDA tensors.
    `depth_mode` is one of DEPTH_MODES; 'oracle' needs `gt` [B, G, 7] fp32 = (valid, class, x1, y1, x2, y2, z) per
    ground-truth slot of every image."""
    B, C, H, W = heat.shape
    R = reg.shape[1]
    if depth_mode not in DEPTH_MODES:
        raise ValueError("depth_mode %r is not one of %s" % (depth_mode, DEPTH_MODES))
    if depth_mode == 'oracle':
        if gt is None or gt.dim() != 3 or tuple(gt.shape[::2]) != (B, 7) or gt.dtype != torch.float32 \
                or not gt.is_contiguous():
            raise ValueError("the oracle depth needs gt as a contiguous float32 [B, G, 7] tensor")
    if ws is None or (ws.B, ws.C, ws.K, ws.R) != (B, C, K, R):
        ws = DecodeWorkspace(B, C, K, R, heat.device)
    gt_ptr, G = (gt.data_ptr(), gt.shape[1]) if gt is not None else (None, 0)
    call("mf_decode_detections", heat.data_ptr(), reg.data_ptr(), calib.data_ptr(), pad.data_ptr(), size.data_ptr(),
         dim_mean.data_ptr(), B, C, H, W, R, K, float(thresh), 1 if apply_sigmoid else 0, DEPTH_MODES.index(depth_mode),
         gt_ptr, G, ws.ws_score.data_ptr(), ws.ws_idx.data_ptr(), ws.scores.data_ptr(), ws.inds.data_ptr(),
         ws.clses.data_ptr(), ws.ys.data_ptr(), ws.xs.data_ptr(), ws.pois.data_ptr(), ws.result.data_ptr(),
         ws.count.data_ptr(), ws.depth_err.data_ptr(), ws.proj.data_ptr(), ws.min_unc.data_ptr(), stream())
    return ws


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
