"""KeypointDetector (reference: model/detector.py:11-37): backbone -> heads, same constructor and forward signature so
engine/trainer.py:109 and engine/inference.py:38 call it unchanged.

Training mode (engine/trainer.py:103-126): `loss_dict, log_loss_dict = model(images, targets)` runs the train-mode plans
(batch-statistics BatchNorm, running statistics updated) and the fused loss; `sum(loss_dict.values()).backward()` then
reaches `_TapeBridge.backward`, which replays the backward tape of the two plans (monoflex_b200/tape.py)
and ACCUMULATES the gradient of every parameter the forward used into `p.grad` - exactly what autograd does for the
reference, so `optimizer.zero_grad(); losses.backward(); optimizer.step()` works unchanged with torch.optim.AdamW or with
solver.FusedAdamW (whose `.grad`s are views of one arena).

Eval forwards are replayed from a CUDA graph (SURVEY §8f N3): shapes are static (384x1280 zero-padded images), so the
~135 kernel launches of a forward are captured once per (input shape, parameter version) and replayed with one
cudaGraphLaunch; per call only the image batch and the per-image target fields are copied into static buffers.
`MF_CUDA_GRAPH=0` (or `model.use_cuda_graph = False`) runs the same launches eagerly.

`forward_depths(images, targets, methods)` decodes several OUTPUT_DEPTH estimators from one backbone + predictor pass
(captured in a graph of its own, next to the forward's)."""
import os

import torch
from torch import nn

from .. import engine
from ..structures import to_image_list
from .backbone import build_backbone
from .head.detector_head import bulid_head
from .layers.utils import depth_error_dict


class _TapeBridge(torch.autograd.Function):
    """Autograd boundary between the predictor outputs (fp32 `cls`, `reg`, produced by hand-written kernels outside autograd)
    and the reference-side loss: forward hands the two maps to autograd, backward receives dL/dcls, dL/dreg and runs the
    whole-network backward tape. `anchor` is a dummy leaf that makes autograd schedule this node."""

    @staticmethod
    def forward(ctx, anchor, cls, reg, model):
        ctx.model = model
        return cls.detach(), reg.detach()

    @staticmethod
    def backward(ctx, g_cls, g_reg):
        ctx.model._tape_backward(g_cls, g_reg)
        return None, None, None, None


class KeypointDetector(nn.Module):
    def __init__(self, cfg):
        super(KeypointDetector, self).__init__()
        self.backbone = build_backbone(cfg)
        self.heads = bulid_head(cfg, self.backbone.out_channels)
        self.test = cfg.DATASETS.TEST_SPLIT == 'test'
        self.use_cuda_graph = os.environ.get("MF_CUDA_GRAPH", "1") != "0"
        self._graph = None
        self._graph_depths = None
        self.set_precision(engine.default_precision())
        # fp16 gradient flow of the backward tape: dL/dcls, dL/dreg are multiplied by `loss_scale` before they enter the
        # tape and every parameter gradient is divided by it again before it is accumulated into p.grad (fp32)
        # MF_LOSS_SCALE=dynamic selects a loss_scale.DynamicLossScale in the Trainer; the static value then stays 128 and
        # is not used. loss_scaler: a DynamicLossScale (device scale, GradScaler's rule) or None for the static scale.
        env_scale = os.environ.get("MF_LOSS_SCALE", "128")
        self.loss_scale = 128.0 if env_scale.strip().lower() == "dynamic" else float(env_scale)
        self.loss_scaler = None
        self._anchor = None

    def set_precision(self, mode):
        """'strict' (default): hi/lo fp16 pair arithmetic, fp32-grade results - the mode that meets the 1e-3 parity contract
        with the fp32 reference; 'fast': single fp16 tensor-core pass (2-4e-3 end to end). Inference only; training plans
        always run the fp16 kernels with fp32 master weights."""
        if mode not in engine.PRECISIONS:
            raise ValueError("precision must be one of %s" % (engine.PRECISIONS,))
        self.precision = self.backbone.precision = mode
        self._graph = self._graph_depths = None
        return self

    def forward(self, images, targets=None):
        if self.training and targets is None:
            raise ValueError("In training mode, targets should be passed")
        images = to_image_list(images)
        if self.training:
            return self._forward_train(images.tensors, targets)
        x = images.tensors
        if not self.use_cuda_graph or not x.is_cuda:
            features = self.backbone(x)
            return self.heads(features, targets, test=self.test)
        return self._forward_graph(x, targets)

    # ------------------------------------------------------------------ training path
    def _forward_train(self, x, targets, prepared=None, sync_log=True):
        """model/detector.py:32-34 + detector_head.py:17-25 in training mode -> (loss_dict, log_loss_dict)."""
        if not x.is_cuda:
            raise RuntimeError("monoflex_b200 trains on sm_90a GPUs only; no CPU fallback")
        features = self.backbone.train_forward(x)
        pred = self.heads.predictor.train_forward(features, targets)
        engine.bump_buffers(self)               # running statistics were updated by the bn_train kernels
        if self._anchor is None or self._anchor.device != x.device:
            self._anchor = torch.zeros(1, device=x.device, requires_grad=True)
        cls, reg = _TapeBridge.apply(self._anchor, pred['cls'], pred['reg'], self)
        return self.heads.loss_evaluator({'cls': cls, 'reg': reg}, targets, prepared=prepared, sync_log=sync_log)

    def train_forward_losses(self, images, targets):
        """explicit name of the training-mode forward (kept from round 1; same as `model.train(); model(images, targets)`)"""
        if not self.training:
            raise RuntimeError("train_forward_losses needs model.train()")
        return self._forward_train(to_image_list(images).tensors, targets)

    @torch.no_grad()
    def _tape_backward(self, g_cls, g_reg):
        """dL/dcls, dL/dreg -> accumulate dL/dp into p.grad for every parameter the forward used (the backward tape)."""
        from ..tape import backbone_backward, predictor_backward
        pred_mod, S, scaler = self.heads.predictor, self.loss_scale, self.loss_scaler
        if scaler is not None:
            if scaler.optimizer is None:
                raise RuntimeError("model.loss_scaler is set, but no fused optimiser updates it: a dynamic loss scale needs "
                                   "solver.FusedAdamW / FusedAdam / FusedOneCycleAdam .step(loss_scaler=...) after every "
                                   "backward (Trainer(loss_scale='dynamic') does this; by hand: loss_scaler.attach(optimizer))")
            S = scaler.scale                 # 0-d device tensor: the seeding multiply reads the current scale on the GPU
        plan_h, plan_b = pred_mod.last_plan, self.backbone.last_plan
        if g_cls is None:
            g_cls = torch.zeros_like(plan_h.cls)
        if g_reg is None:
            g_reg = torch.zeros_like(plan_h.reg)
        hgrads, d_feat = predictor_backward(pred_mod, plan_h, g_cls * S, g_reg * S)
        bgrads = backbone_backward(self.backbone, plan_b, d_feat)
        params = getattr(self, "_param_by_name", None)
        if params is None:
            params = self._param_by_name = dict(self.named_parameters())
        inv = None if scaler is not None else 1.0 / S
        used = set()
        acc_dst, acc_src, acc_assign = [], [], []
        for prefix, grads in (("heads.predictor.", hgrads), ("backbone.", bgrads)):
            for name, g in grads.items():
                p = params[prefix + name]
                used.add(prefix + name)
                if not p.requires_grad:
                    continue
                if scaler is not None:       # every p.grad in the one unscale launch below; a first gradient is assigned
                    assign = p.grad is None
                    if assign:
                        p.grad = torch.empty_like(p)
                    acc_dst.append(p.grad)
                    acc_assign.append(assign)
                    g = g.view_as(p)
                    acc_src.append(g if g.is_contiguous() and g.dtype == p.grad.dtype else g.contiguous().to(p.grad.dtype))
                elif p.grad is None:
                    p.grad = (g * inv).view_as(p)
                else:
                    acc_dst.append(p.grad)
                    g = g.view_as(p)
                    # the multi-tensor kernel needs dense operands; ONE strided gradient would send the whole list down the
                    # per-tensor slow path (285 tiny add kernels per step in the ncu launch list)
                    acc_src.append(g if g.is_contiguous() and g.dtype == p.grad.dtype else g.contiguous().to(p.grad.dtype))
        if scaler is not None:               # p.grad += g * inv_scale, inv_scale read from the device scale, one launch
            scaler.unscale_accumulate(acc_dst, acc_src, acc_assign)
        elif acc_dst:                        # one multi-tensor kernel instead of ~280 tiny adds (p.grad += g / loss_scale)
            torch._foreach_add_(acc_dst, acc_src, alpha=inv)
        self.last_grad_names = used          # parameters outside the forward graph (the reference leaves their .grad None)

    def forward_async(self, images, targets):
        """Enqueue one eval forward (graph replay) and return a handle; `handle.result()` waits for it and returns what
        `forward` returns. Lets a caller overlap the host-side read of step i with the GPU work of step i+1 (the decode
        workspace is re-used by the next forward, so call `result()` - or at least `stage()` - before the forward after
        next). With TEST.EVAL_DEPTH, `result()` also sets `handle.eval_utils['depth_errors']` /
        `['depth_error_counts']` as forward fills them."""
        if self.training:
            raise RuntimeError("forward_async is an inference API")
        x = to_image_list(images).tensors
        if not x.is_cuda:
            raise RuntimeError("monoflex_b200 runs on sm_90a GPUs only; no CPU fallback")
        g = self._enqueue_graph(x, targets)
        return PendingDetections(self.heads.post_processor, g['ws'], g['plan_h'].cls)

    def forward_depths(self, images, targets, methods):
        """Eval mode: {method: what forward(images, targets) returns with heads.post_processor.output_depth = method} for
        every OUTPUT_DEPTH name of `methods`, from one backbone + predictor pass and one decode launch. Only the depth, the
        location, alpha / ry and the score differ between the methods; the detections are the same."""
        if self.training:
            raise RuntimeError("forward_depths is an inference API: call model.eval() first")
        post = self.heads.post_processor
        methods = post.check_config(methods)
        x = to_image_list(images).tensors
        if not self.use_cuda_graph or not x.is_cuda:
            pred = self.heads.predictor(self.backbone(x), targets)
            return post.forward_depths(pred, targets, methods, test=self.test)
        g = self._enqueue_graph(x, targets, methods)
        return post.finish_depths(g['ws'], g['plan_h'].cls, g['plan_h'].reg, methods)

    # ------------------------------------------------------------------ CUDA-graph path
    def _forward_graph(self, x, targets):
        g = self._enqueue_graph(x, targets)
        return self.heads.post_processor.finish(g['ws'], g['plan_h'].cls, g['plan_h'].reg)

    def _enqueue_graph(self, x, targets, methods=None):
        """replay the forward's graph or, given a tuple of `methods`, the graph of forward_depths (each kept in its own
        slot, so alternating the two does not capture again)"""
        pred, post = self.heads.predictor, self.heads.post_processor
        post.check_config(methods)
        x = x.float().contiguous()
        k_edge = targets[0].get_field("edge_indices").shape[0]
        # per-call target fields of the decode: calib / pad / size and, for the oracle depth and for TEST.EVAL_DEPTH, the
        # ground-truth tables
        meta = post.prepare_targets(targets, self.test, x.device, methods)
        key = (tuple(x.shape), x.device, k_edge, engine.fingerprint(self), post.det_threshold, post.max_detection, self.precision,
               post.output_depth if methods is None else methods, post.eval_depth, tuple(tuple(m.shape) for m in meta))
        g = self._graph if methods is None else self._graph_depths
        if g is None or g['key'] != key:
            g = self._capture(x, targets, key, meta, methods)
            if methods is None:
                self._graph = g
            else:
                self._graph_depths = g
        g['x'].copy_(x, non_blocking=True)
        pred.load_targets(g['plan_h'], targets)
        for dst, src in zip(g['meta'], meta):
            if dst.data_ptr() != src.data_ptr():
                dst.copy_(src, non_blocking=True)
        g['graph'].replay()
        return g

    def _capture(self, x, targets, key, meta, methods=None):
        pred, post = self.heads.predictor, self.heads.post_processor
        xs = x.clone()
        plan_b = self.backbone._plan_for(xs)
        plan_h = pred.plan_for(plan_b.output, key[2])
        pred.load_targets(plan_h, targets)
        meta = tuple(t.clone() for t in meta)

        def body():
            self.backbone.run_plan(plan_b, xs)
            plan_h.run()
            return post.launch(plan_h.cls, plan_h.reg, meta, methods)
        body()                                   # eager warm-up: func attributes, tensor-map driver entry points, workspaces
        torch.cuda.synchronize()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            ws = body()
        return {'key': key, 'graph': graph, 'x': xs, 'plan_b': plan_b, 'plan_h': plan_h, 'meta': meta, 'ws': ws}


class PendingDetections(object):
    """Handle of an enqueued forward: `stage()` starts the device->host copy of the padded detections + counts into
    pinned buffers (asynchronous, stream ordered), `result()` waits for it and slices on the host. With TEST.EVAL_DEPTH
    the same copy carries the depth errors' counts, and `stage()` copies their table on the device into a buffer of its
    own; `result()` then sets `eval_utils` = {'depth_errors': the dict forward returns, 'depth_error_counts': [B]}
    (before it, and without EVAL_DEPTH, eval_utils['depth_errors'] is None)."""

    def __init__(self, post, ws, heat):
        self.post, self.ws, self.heat = post, ws, heat
        self._staged = None
        self.eval_utils = {'depth_errors': None}

    def stage(self):
        if self._staged is None:
            ws = self.ws
            host = getattr(ws, "_pinned", None)
            if host is None:
                cnt = ws.count if ws.depth_errors is None else ws.counts
                host = ws._pinned = [(torch.empty(ws.result.shape).pin_memory(), torch.empty(cnt.shape, dtype=torch.int32).pin_memory(),
                                      torch.cuda.Event(), None if ws.depth_errors is None else torch.empty_like(ws.depth_errors))
                                     for _ in range(2)]
                ws._pin_i = 0
            res_h, cnt_h, ev, errs = host[ws._pin_i]
            ws._pin_i ^= 1
            res_h.copy_(ws.result, non_blocking=True)
            cnt_h.copy_(ws.count if errs is None else ws.counts, non_blocking=True)
            if errs is not None:
                errs.copy_(ws.depth_errors)
            ev.record()
            self._staged = (res_h, cnt_h, ev, errs)
        return self

    def result(self):
        """-> (result[N,14] on the HOST, counts list): the rows `forward` would return, read through pinned memory."""
        res_h, cnt_h, ev, errs = self.stage()._staged
        ev.synchronize()
        counts = cnt_h.tolist()
        if errs is not None:
            counts, depth_counts = counts
            self.eval_utils = {'depth_errors': depth_error_dict(errs, depth_counts), 'depth_error_counts': depth_counts}
        rows = [res_h[b, :n] for b, n in enumerate(counts)]
        return (torch.cat(rows, 0) if len(rows) > 1 else rows[0].clone()), counts
