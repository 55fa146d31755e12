"""PostProcessor (reference: model/head/detector_infer.py:20-278).

forward(predictions, targets, features=None, test=False) -> (result[N,14], eval_utils, visualize_preds) exactly as the
reference for batch size 1. Unlike the reference (valid for B == 1 only: detector_infer.py:211, anno_encoder.py:79) the
CUDA decode takes per-image calibration / padding / size, so for B > 1 `result` is the concatenation of the valid rows
of every image and `eval_utils['batch_idxs']` / `['counts']` say which image each row belongs to (SURVEY H8).

Every OUTPUT_DEPTH estimator of the reference is decoded by the kernel: 'soft' (runs/monoflex.yaml), 'hard', 'mean',
'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02', 'keypoints_13' and 'oracle'. `output_depth` is read at
every forward, so engine/inference.py's inference_all_depths can switch it between passes. The oracle matches every
detection against its own image's ground truth (reg_mask, cls_ids, gt_bboxes, locations); the reference matches the
whole batch against targets[0], which is the same thing for B = 1. An image without valid ground truth keeps the mean
of the four estimators, where the reference raises (argmin of an empty tensor). The --eval_iou / --eval_depth
diagnostics are out of scope (DESIGN.md §9)."""
import torch
from torch import nn

from ..layers.utils import DEPTH_MODES, ENSEMBLE_DEPTH_MODES, Converter_key2channel, DecodeWorkspace, decode_detections

ORACLE_FIELDS = ('reg_mask', 'cls_ids', 'gt_bboxes', 'locations')


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
        self._meta_cache = None

    def prepare_targets(self, targets, test, device):
        """calib / pad_size / size of every image as three small device tensors (detector_infer.py:53-58). The host-side
        scalars (calibration, image size) are cached BY VALUE; pad_size is stacked on the device like the reference
        does, so a CUDA `pad_size` field costs no host sync."""
        calib, size = [], []
        for t in targets:
            c = t.get_field("calib")
            calib.append((float(c.f_u), float(c.f_v), float(c.c_u), float(c.c_v), float(c.b_x), float(c.b_y)))
            size.append((float(t.size[0]), float(t.size[1])))
        key = (tuple(calib), tuple(size), str(device))
        if self._meta_cache is None or self._meta_cache[0] != key:
            self._meta_cache = (key, torch.tensor(calib, dtype=torch.float32).to(device),
                                torch.tensor(size, dtype=torch.float32).to(device))
        pad = torch.stack([torch.as_tensor(t.get_field("pad_size")) for t in targets]).to(device=device, dtype=torch.float32,
                                                                                         non_blocking=True).view(-1, 2)
        if self.output_depth != 'oracle':
            return self._meta_cache[1], pad, self._meta_cache[2]
        return self._meta_cache[1], pad, self._meta_cache[2], self.oracle_table(targets, device)

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

    def launch(self, heat, reg, meta):
        """the two decode kernels (asynchronous; no host sync)"""
        calib, pad, size = meta[:3]
        B, K = heat.shape[0], self.max_detection
        if self._ws is None or (self._ws.B, self._ws.C) != (B, heat.shape[1]) or self._ws.scores.device != heat.device:
            self._ws = DecodeWorkspace(B, heat.shape[1], K, reg.shape[1], heat.device)
        return decode_detections(heat, reg, calib, pad, size, self.dim_mean, K, self.det_threshold, False, self._ws,
                                 depth_mode=self.output_depth, gt=meta[3] if len(meta) > 3 else None)

    def finish(self, ws, heat, reg):
        """host side: read the valid counts (the reference syncs at `valid_mask.sum() == 0`, :106) and slice."""
        B = heat.shape[0]
        visualize_preds = {'heat_map': heat}
        counts = ws.count.tolist()

        def rows(t):
            """the valid rows of every image of a [B, K, ...] workspace tensor, concatenated"""
            if B == 1:
                return t[0, :counts[0]]
            if all(n == ws.K for n in counts):
                return t.reshape(B * ws.K, *t.shape[2:])
            return torch.cat([t[b, :n] for b, n in enumerate(counts)], 0)
        batch_idxs = torch.cat([torch.full((n,), b, dtype=torch.long, device=heat.device) for b, n in enumerate(counts)], 0)
        # detections are tiny: hand out copies, not views of the (re-used) decode workspace
        result, vis_scores, pois = rows(ws.result).clone(), rows(ws.scores).clone(), rows(ws.pois).clone()
        depth_err = rows(ws.depth_err).clone()
        visualize_preds['keypoints'] = pois[:, self.key2channel('corner_offset')].reshape(-1, 10, 2)
        visualize_preds['proj_center'] = rows(ws.proj).clone()                                          # :125
        visualize_preds['depth_uncertainty'] = reg[:, self.key2channel('depth_uncertainty')].squeeze(1)  # :136
        if self.output_depth in ENSEMBLE_DEPTH_MODES:
            visualize_preds['min_uncertainty'] = rows(ws.min_unc).long()                                # :185
        conf = result[:, 13] / vis_scores.clamp_min(1e-12) if result.shape[0] else result.new_zeros(0)
        eval_utils = {'dis_ious': None, 'depth_errors': None, 'uncertainty_conf': conf,
                      'estimated_depth_error': depth_err, 'vis_scores': vis_scores, 'batch_idxs': batch_idxs,
                      'counts': counts, 'topk': (ws.scores, ws.inds, ws.clses, ws.ys, ws.xs), 'padded_result': ws.result}
        return result, eval_utils, visualize_preds

    def check_config(self):
        if self.output_depth not in DEPTH_MODES:
            if isinstance(self.output_depth, str) and self.output_depth.find('keypoints') >= 0:     # :172-173
                raise ValueError("unknown key-point depth OUTPUT_DEPTH=%r" % (self.output_depth,))
            raise ValueError("OUTPUT_DEPTH=%r is not one of %s" % (self.output_depth, ", ".join(DEPTH_MODES)))
        if self.eval_dis_iou or self.eval_depth:
            raise NotImplementedError("--eval_iou / --eval_depth diagnostics are out of scope")

    def forward(self, predictions, targets, features=None, test=False, refine_module=None):
        self.check_config()
        heat, reg = predictions['cls'], predictions['reg']
        if not heat.is_cuda:
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        heat, reg = heat.float().contiguous(), reg.float().contiguous()
        ws = self.launch(heat, reg, self.prepare_targets(targets, test, heat.device))
        return self.finish(ws, heat, reg)
