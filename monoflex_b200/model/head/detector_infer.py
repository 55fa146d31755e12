"""PostProcessor (reference: model/head/detector_infer.py:20-278).

forward(predictions, targets, features=None, test=False) -> (result[N,14], eval_utils, visualize_preds) exactly as the
reference for batch size 1. Unlike the reference (valid for B == 1 only: detector_infer.py:211, anno_encoder.py:79) the
CUDA decode takes per-image calibration / padding / size, so for B > 1 `result` is the concatenation of the valid rows
of every image and `eval_utils['batch_idxs']` / `['counts']` say which image each row belongs to (SURVEY H8).

forward_depths(predictions, targets, methods) -> {method: what forward returns with output_depth = method}: one NMS /
top-k / POI gather and one decode kernel for all the methods (engine/inference.py's inference_all_depths in one pass).

Every OUTPUT_DEPTH estimator of the reference is decoded by the kernel: 'soft' (runs/monoflex.yaml), 'hard', 'mean',
'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02', 'keypoints_13' and 'oracle'. `output_depth` is read at
every forward, so engine/inference.py's inference_all_depths can switch it between passes. The oracle matches every
detection against its own image's ground truth (reg_mask, cls_ids, gt_bboxes, locations); the reference matches the
whole batch against targets[0], which is the same thing for B = 1. An image without valid ground truth keeps the mean
of the four estimators, where the reference raises (argmin of an empty tensor).

TEST.EVAL_DEPTH (--eval_depth) runs evaluate_3D_depths in one more kernel after the decode (inside the captured graph
of KeypointDetector): eval_utils['depth_errors'] is the reference's dict of 13 per-object tensors, with the rows of
every image in (image, slot) order, and eval_utils['depth_error_counts'] the valid objects of each image. The reference
is batch-1 only there too. The --eval_iou diagnostic (TEST.EVAL_DIS_IOUS) is out of scope (DESIGN.md §9)."""
import torch
from torch import nn

from ..layers.utils import (DEPTH_MODES, ENSEMBLE_DEPTH_MODES, Converter_key2channel, DecodeWorkspace, decode_detections,
                            depth_error_dict, eval_depth_errors)

ORACLE_FIELDS = ('reg_mask', 'cls_ids', 'gt_bboxes', 'locations')
EVAL_DEPTH_FIELDS = ('target_centers', 'reg_mask', 'cls_ids', 'locations')


def make_post_processor(cfg):
    key2channel = Converter_key2channel(keys=cfg.MODEL.HEAD.REGRESSION_HEADS, channels=cfg.MODEL.HEAD.REGRESSION_CHANNELS)
    return PostProcessor(cfg=cfg, key2channel=key2channel)


class PostProcessor(nn.Module):
    def __init__(self, cfg, anno_encoder=None, key2channel=None):
        super(PostProcessor, self).__init__()
        self.key2channel = key2channel
        self.det_threshold = cfg.TEST.DETECTIONS_THRESHOLD
        self.max_detection = cfg.TEST.DETECTIONS_PER_IMG
        self.eval_dis_iou = cfg.TEST.EVAL_DIS_IOUS
        self.eval_depth = cfg.TEST.EVAL_DEPTH
        self.output_width = cfg.INPUT.WIDTH_TRAIN // cfg.MODEL.BACKBONE.DOWN_RATIO
        self.output_height = cfg.INPUT.HEIGHT_TRAIN // cfg.MODEL.BACKBONE.DOWN_RATIO
        self.output_depth = cfg.MODEL.HEAD.OUTPUT_DEPTH
        self.uncertainty_as_conf = cfg.TEST.UNCERTAINTY_AS_CONFIDENCE
        self.down_ratio = cfg.MODEL.BACKBONE.DOWN_RATIO
        self.register_buffer("dim_mean", torch.tensor(cfg.MODEL.HEAD.DIMENSION_MEAN, dtype=torch.float32),
                             persistent=False)
        expected = ['2d_dim', '3d_offset', 'corner_offset', 'corner_uncertainty', '3d_dim', 'ori_cls', 'ori_offset',
                    'depth', 'depth_uncertainty']
        if key2channel.keys != expected or key2channel.channels != [4, 2, 20, 3, 3, 8, 8, 1, 1]:
            raise NotImplementedError("decode kernel is built for the runs/monoflex.yaml regression layout")
        if cfg.MODEL.HEAD.DEPTH_MODE != 'inv_sigmoid' or list(cfg.MODEL.HEAD.DIMENSION_REG) != ['exp', True, False] \
                or not self.uncertainty_as_conf or self.down_ratio != 4:
            raise NotImplementedError("decode kernel is built for the runs/monoflex.yaml decode settings")
        self._ws = None
        self._ws_depths = None
        self._meta_cache = None

    def prepare_targets(self, targets, test, device, methods=None):
        """calib / pad_size / size of every image as three small device tensors (detector_infer.py:53-58). The host-side
        scalars (calibration, image size) are cached BY VALUE; pad_size is stacked on the device like the reference
        does, so a CUDA `pad_size` field costs no host sync. The oracle table is appended when `methods` (default: the
        output_depth alone) include 'oracle', then the depth_table when TEST.EVAL_DEPTH is set."""
        calib, size = [], []
        for t in targets:
            c = t.get_field("calib")
            calib.append((float(c.f_u), float(c.f_v), float(c.c_u), float(c.c_v), float(c.b_x), float(c.b_y)))
            size.append((float(t.size[0]), float(t.size[1])))
        key = (tuple(calib), tuple(size), str(device))
        if self._meta_cache is None or self._meta_cache[0] != key:     # copied up without waiting for the device
            self._meta_cache = (key, torch.tensor(calib, dtype=torch.float32).to(device, non_blocking=True),
                                torch.tensor(size, dtype=torch.float32).to(device, non_blocking=True))
        pad = torch.stack([torch.as_tensor(t.get_field("pad_size")) for t in targets]).to(device=device, dtype=torch.float32,
                                                                                         non_blocking=True).view(-1, 2)
        meta = (self._meta_cache[1], pad, self._meta_cache[2])
        if 'oracle' in ((self.output_depth,) if methods is None else methods):
            meta += (self.oracle_table(targets, device),)
        if self.eval_depth:
            meta += (self.depth_table(targets, device),)
        return meta

    @staticmethod
    def oracle_table(targets, device):
        """Ground truth of every image for the oracle depth (detector_infer.py:239-252) as one [B, G, 7] device tensor:
        (valid, class, x1, y1, x2, y2, z) per object slot, from the label fields the training loader attaches."""
        missing = [f for f in ORACLE_FIELDS if not all(t.has_field(f) for t in targets)]
        if missing:
            raise RuntimeError("OUTPUT_DEPTH='oracle' matches detections to the ground truth, but the targets lack %s "
                               "(a TEST_SPLIT='test' loader attaches no labels)" % ", ".join(missing))
        rows = []
        for t in targets:
            f = [torch.as_tensor(t.get_field(k)).to(device=device, dtype=torch.float32, non_blocking=True)
                 for k in ORACLE_FIELDS]
            n = f[0].numel()
            rows.append(torch.cat([f[0].view(n, 1), f[1].view(n, 1), f[2].view(n, 4), f[3].view(n, 3)[:, 2:]], 1))
        return torch.stack(rows).contiguous()

    @staticmethod
    def depth_table(targets, device):
        """Ground truth of every image for evaluate_3D_depths (detector_infer.py:280-359) as one [B, M, 5] device tensor:
        (reg_mask, cls_id, target centre x, y, location z) per object slot, from the label fields the training loader
        attaches."""
        missing = [f for f in EVAL_DEPTH_FIELDS if not all(t.has_field(f) for t in targets)]
        if missing:
            raise RuntimeError("TEST.EVAL_DEPTH measures the depths at the ground-truth centres, but the targets lack %s "
                               "(a TEST_SPLIT='test' loader attaches no labels)" % ", ".join(missing))
        return _depth_table(*(torch.stack([torch.as_tensor(t.get_field(k)) for t in targets]) for k in EVAL_DEPTH_FIELDS),
                            device=device)

    def launch(self, heat, reg, meta, methods=None):
        """the two decode kernels (asynchronous; no host sync) for the output_depth or, given a tuple of `methods`, for all
        of them into a workspace of one block per method; with TEST.EVAL_DEPTH the depth-error kernel after them"""
        calib, pad, size = meta[:3]
        B, K = heat.shape[0], self.max_detection
        n_modes = None if methods is None else len(methods)
        modes = (self.output_depth,) if methods is None else methods
        table = meta[-1] if self.eval_depth else None
        eval_slots = 0 if table is None else table.shape[1]
        ws = self._ws if methods is None else self._ws_depths
        if ws is None or (ws.B, ws.C, ws.n_modes, ws.eval_slots) != (B, heat.shape[1], n_modes, eval_slots) \
                or ws.scores.device != heat.device:
            ws = DecodeWorkspace(B, heat.shape[1], K, reg.shape[1], heat.device, n_modes, eval_slots)
            if methods is None:
                self._ws = ws
            else:
                self._ws_depths = ws
        ws = decode_detections(heat, reg, calib, pad, size, self.dim_mean, K, self.det_threshold, False, ws,
                               depth_mode=self.output_depth if methods is None else methods,
                               gt=meta[3] if 'oracle' in modes else None)
        if table is not None:
            eval_depth_errors(reg, calib, self.dim_mean, table, ws.depth_errors, ws.depth_counts)
        return ws

    def finish(self, ws, heat, reg):
        """host side: read the valid counts (the reference syncs at `valid_mask.sum() == 0`, :106) and slice."""
        return self.finish_depths(ws, heat, reg, (self.output_depth,))[self.output_depth]

    def finish_depths(self, ws, heat, reg, methods):
        """finish() of every method of `methods`, the estimators of the workspace's result blocks in order (a
        single-mode workspace holds one block without the mode dimension). The counts are read once; the tensors that do
        not depend on the estimator are shared between the methods' dicts."""
        B = heat.shape[0]
        depth_errors = None
        if ws.depth_errors is None:
            counts = ws.count.tolist()
        else:                                  # the decode's and the depth errors' counts in one copy
            counts, depth_counts = ws.counts.tolist()
            depth_errors = depth_error_dict(ws.depth_errors, depth_counts)

        def rows(t):
            """the valid rows of every image of a [B, K, ...] workspace tensor, concatenated"""
            if B == 1:
                return t[0, :counts[0]]
            if all(n == ws.K for n in counts):
                return t.reshape(B * ws.K, *t.shape[2:])
            return torch.cat([t[b, :n] for b, n in enumerate(counts)], 0)
        batch_idxs = torch.cat([torch.full((n,), b, dtype=torch.long, device=heat.device) for b, n in enumerate(counts)], 0)
        # detections are tiny: hand out copies, not views of the (re-used) decode workspace
        vis_scores, pois = rows(ws.scores).clone(), rows(ws.pois).clone()
        keypoints = pois[:, self.key2channel('corner_offset')].reshape(-1, 10, 2)
        proj_center = rows(ws.proj).clone()                                                             # :125
        depth_uncertainty = reg[:, self.key2channel('depth_uncertainty')].squeeze(1)                    # :136
        out = {}
        for m, method in enumerate(methods):
            block = (lambda t: t) if ws.n_modes is None else (lambda t: t[m])
            result, depth_err = rows(block(ws.result)).clone(), rows(block(ws.depth_err)).clone()
            visualize_preds = {'heat_map': heat, 'keypoints': keypoints, 'proj_center': proj_center,
                               'depth_uncertainty': depth_uncertainty}
            if method in ENSEMBLE_DEPTH_MODES:
                visualize_preds['min_uncertainty'] = rows(block(ws.min_unc)).long()                     # :185
            conf = result[:, 13] / vis_scores.clamp_min(1e-12) if result.shape[0] else result.new_zeros(0)
            eval_utils = {'dis_ious': None, 'depth_errors': depth_errors, 'uncertainty_conf': conf,
                          'estimated_depth_error': depth_err, 'vis_scores': vis_scores, 'batch_idxs': batch_idxs,
                          'counts': counts, 'topk': (ws.scores, ws.inds, ws.clses, ws.ys, ws.xs),
                          'padded_result': block(ws.result)}
            if depth_errors is not None:
                eval_utils['depth_error_counts'] = depth_counts
            out[method] = (result, eval_utils, visualize_preds)
        return out

    def check_config(self, methods=None):
        """the output_depth, or every method of `methods` (a non-empty sequence of distinct names) -> the tuple of them"""
        names = (self.output_depth,) if methods is None else methods
        if isinstance(names, str) or not isinstance(names, (tuple, list)) or not names or len(set(names)) != len(names):
            raise ValueError("methods must be a non-empty list of distinct OUTPUT_DEPTH names, got %r" % (methods,))
        for name in names:
            if name not in DEPTH_MODES:
                if isinstance(name, str) and name.find('keypoints') >= 0:                            # :172-173
                    raise ValueError("unknown key-point depth OUTPUT_DEPTH=%r" % (name,))
                raise ValueError("OUTPUT_DEPTH=%r is not one of %s" % (name, ", ".join(DEPTH_MODES)))
        if self.eval_dis_iou:
            raise NotImplementedError("the --eval_iou diagnostic (TEST.EVAL_DIS_IOUS) is out of scope")
        return tuple(names)

    def evaluate_3D_depths(self, targets, pred_regression):
        """detector_infer.py:280-359: {key: 1-D float32 CUDA tensor} of the depth errors of every estimator at the
        ground-truth centres, one entry per valid object in the order of targets['reg_mask'].view(-1). `targets` is the
        dict of the reference's prepare_targets(test=False): calib (a list), target_centers [B, M, 2], reg_mask [B, M],
        cls_ids [B, M], locations [B, M, 3]. Each image uses its own calibration. Synchronises once, to read the count."""
        reg = pred_regression.float().contiguous()
        if not reg.is_cuda:
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        missing = [f for f in EVAL_DEPTH_FIELDS if f not in targets]
        if missing:
            raise RuntimeError("evaluate_3D_depths needs the label fields %s" % ", ".join(missing))
        calib = torch.tensor([(float(c.f_u), float(c.f_v), float(c.c_u), float(c.c_v), float(c.b_x), float(c.b_y))
                              for c in targets['calib']], dtype=torch.float32).to(reg.device)
        table = _depth_table(*(torch.as_tensor(targets[k]) for k in EVAL_DEPTH_FIELDS), device=reg.device)
        out, counts = eval_depth_errors(reg, calib, self.dim_mean, table)
        return depth_error_dict(out, counts.tolist())

    def forward(self, predictions, targets, features=None, test=False, refine_module=None):
        self.check_config()
        heat, reg = predictions['cls'], predictions['reg']
        if not heat.is_cuda:
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        heat, reg = heat.float().contiguous(), reg.float().contiguous()
        ws = self.launch(heat, reg, self.prepare_targets(targets, test, heat.device))
        return self.finish(ws, heat, reg)

    def forward_depths(self, predictions, targets, methods, test=False):
        """{method: forward(predictions, targets) with output_depth = method} for every method of `methods`, from one
        decode launch; the oracle table is built once, and only when 'oracle' is among the methods."""
        methods = self.check_config(methods)
        heat, reg = predictions['cls'], predictions['reg']
        if not heat.is_cuda:
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        heat, reg = heat.float().contiguous(), reg.float().contiguous()
        ws = self.launch(heat, reg, self.prepare_targets(targets, test, heat.device, methods), methods)
        return self.finish_depths(ws, heat, reg, methods)


def _depth_table(target_centers, reg_mask, cls_ids, locations, device):
    """the [B, M, 5] depth_table (reg_mask, cls_id, x, y, z) from the stacked label fields [B, M, ...]: a handful of
    launches whatever B is"""
    f = [v.to(device=device, dtype=torch.float32, non_blocking=True) for v in (target_centers, reg_mask, cls_ids, locations)]
    B, M = f[1].shape[0], f[1][0].numel()
    return torch.cat([f[1].view(B, M, 1), f[2].view(B, M, 1), f[0].view(B, M, 2), f[3].view(B, M, 3)[..., 2:]], 2)
