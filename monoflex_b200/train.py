"""Training step on the CUDA kernels, driven exactly like the reference loop (engine/trainer.py:103-126):

    loss_dict, log = model(images, targets); losses = sum(loss_dict.values())
    optimizer.zero_grad(); losses.backward(); [clip_grad_norm_]; optimizer.step(); scheduler.step()

`model(images, targets)` in training mode runs the train-mode plans + the fused loss; `losses.backward()` reaches the
backward tape through `model/detector.py::_TapeBridge` and accumulates into `p.grad`. `Trainer` is that loop as an object:
it owns the `FusedAdamW` arena optimiser, performs the data-parallel gradient exchange the reference gets from
DistributedDataParallel (tools/plain_train_net.py:100-104: mean over ranks) - bucketed NCCL all-reduce of the gradient arena
with the 1/world folded into the AdamW kernel, or the fused peer-memory kernel when built with `symmetric_group` - and guards
the update with a device-side finite check of the gradient arena (fp16 gradient flow under a fixed loss scale: a non-finite
gradient skips the step instead of poisoning params and moments; the reference trains in fp32 and stops on NaN losses,
detector_loss.py:485-489).

`use_cuda_graph=True` (SURVEY §8f N3): shapes are static (384x1280 padded images, 40 object slots), train-mode plans read
every parameter from its live storage, and nothing between the image copy and the optimiser update needs the host, so after
`graph_warmup` eager steps the whole step - forward plans, fused loss, loss backward, the backward tape with all its
temporaries, zero_grad and (single GPU) the guarded AdamW update - is captured ONCE in a CUDA graph and replayed; per step
the host copies the batch and its labels into static buffers and launches one graph (multi-GPU: graph, NCCL all-reduce,
AdamW).

`cfg.SOLVER.GRAD_NORM_CLIP > 0` (the reference's clip_grad_norm_ between backward and step, engine/trainer.py:119): the eager
step calls torch's `clip_grad_norm_` over the parameters, line for line like the reference. The captured step clips on the
device instead (`FusedAdamW.step(max_grad_norm=...)`: the norm is accumulated by the scan of the gradient arena that also
serves as the finite guard, and the coefficient is applied in the AdamW kernel, no host read), inside the graph on one GPU
and in the update that follows the NCCL all-reduce on several, so it clips the rank mean as DDP + clip_grad_norm_ does.
`optimizer.last_grad_norm` holds the norm of the last captured step. Not available with `symmetric_group` in the captured
step (raises NotImplementedError): the fused peer-memory exchange has no cross-rank norm between its reduce and update.

`cfg.SOLVER.OPTIMIZER` picks the optimiser through `solver.build_optimizer`: 'adamw' (FusedAdamW, as before), 'adam'
(FusedAdam) or 'adam_onecycle' (FusedOneCycleAdam); the last two only without `symmetric_group` (the peer-memory exchange
kernel is AdamW only). With `LR_WARMUP` or a one-cycle optimiser the schedules step as the reference's do_train steps them
(engine/trainer.py:123-126): `warmup.step(i)` while i < WARMUP_STEPS, then `scheduler.step(i)`, i the 0-based index of the
step just taken; 'adam_onecycle' with LR_WARMUP raises (the reference asserts a warm-up scheduler it never builds). The
plain adamw / LambdaLR case keeps calling `scheduler.step()` without an index. The captured step refreshes the optimiser's
device lr table and hyper-parameter block (lr, beta1 and weight decay a schedule moves) before every replay, so the
one-GPU update stays inside the graph for every optimiser.
"""
import torch
import torch.distributed as dist

from . import solver
from .targets import EncodedTargets


class Trainer(object):
    def __init__(self, model, cfg, loss_scale=None, symmetric_group=None, process_group=None, bucket_bytes=32 << 20,
                 use_cuda_graph=False, graph_warmup=2):
        if not next(model.parameters()).is_cuda:
            raise RuntimeError("monoflex_b200 trains on sm_90a GPUs only; no CPU fallback")
        self.grad_norm_clip = getattr(cfg.SOLVER, "GRAD_NORM_CLIP", -1)
        name = cfg.SOLVER.OPTIMIZER
        if name not in solver.OPTIMIZERS:
            raise NotImplementedError("optimizer %r: the fused optimisers are %s" % (name, ", ".join(solver.OPTIMIZERS)))
        if name != "adamw" and symmetric_group is not None:
            raise NotImplementedError("optimizer %r with symmetric_group: the fused peer-memory exchange kernel runs AdamW "
                                      "only; use the NCCL exchange (no symmetric_group)" % name)
        onecycle = name.find("onecycle") >= 0
        if onecycle and cfg.SOLVER.LR_WARMUP:
            raise ValueError("optimizer %r with LR_WARMUP: the one-cycle schedule has no warm-up scheduler (the reference's "
                             "do_train asserts one)" % name)
        if use_cuda_graph and self.grad_norm_clip > 0 and symmetric_group is not None:
            raise NotImplementedError("GRAD_NORM_CLIP > 0 with symmetric_group: the fused peer-memory exchange (step_exchange) "
                                      "has no cross-rank gradient norm between its reduce and its update; use the NCCL "
                                      "exchange (no symmetric_group) or use_cuda_graph=False")
        self.model = model.train()
        if loss_scale is not None:
            model.loss_scale = float(loss_scale)
        self.cfg = cfg
        self.group = process_group
        self.bucket_bytes = bucket_bytes
        self.optimizer = solver.build_optimizer(model, cfg, symmetric_group=symmetric_group)
        self._arena_opt = getattr(self.optimizer, "opt", self.optimizer)    # FusedOneCycleAdam wraps its arena optimiser
        self.scheduler, self.warmup_scheduler = solver.build_scheduler(self.optimizer, cfg.SOLVER)
        # indexed stepping of do_train (engine/trainer.py:123-126) with a warm-up or one-cycle schedule
        self._indexed_schedule = onecycle or self.warmup_scheduler is not None
        self.warmup_iters = solver.solver_value(cfg.SOLVER, "WARMUP_STEPS") if cfg.SOLVER.LR_WARMUP else -1
        self.iteration = 0
        self._unused_marked = False
        self.use_cuda_graph = bool(use_cuda_graph)
        self.graph_warmup = int(graph_warmup)
        self._graph = None

    @property
    def world(self):
        return dist.get_world_size(self.group) if (dist.is_available() and dist.is_initialized()) else 1

    # ------------------------------------------------------------------ eager step (the reference loop, line by line)
    def step(self, images, targets, sync_log=True):
        """one optimisation step on a batch -> (loss_dict, log_loss_dict) of the forward that produced the gradients.
        targets: the per-image ParamsLists, or the EncodedTargets of GpuTargetEncoder.encode"""
        if self.use_cuda_graph and self.iteration >= self.graph_warmup:
            return self._step_graph(images, targets, sync_log)
        model, opt = self.model, self.optimizer
        model.train()
        if isinstance(targets, EncodedTargets):
            loss_dict, log = model._forward_train(images, targets.edge_targets(), prepared=targets.prepared, sync_log=sync_log)
        else:
            loss_dict, log = model._forward_train(images, targets, sync_log=sync_log)
        losses = sum(loss_dict.values())
        opt.zero_grad()
        losses.backward()                                            # fused loss backward -> tape bridge -> p.grad (arena views)
        if not self._unused_marked:                                  # parameters outside the forward graph: the reference's
            opt.mark_unused({n for n, _ in model.named_parameters()} - set(model.last_grad_names), model)   # AdamW skips grad None
            self._unused_marked = True
        if self.grad_norm_clip > 0:
            torch.nn.utils.clip_grad_norm_(model.parameters(), self.grad_norm_clip)
        self._exchange_and_update()
        self._schedule_step()
        self.iteration += 1
        return {k: v.detach() for k, v in loss_dict.items()}, log

    def _schedule_step(self):
        if not self._indexed_schedule:
            self.scheduler.step()
        elif self.iteration < self.warmup_iters:
            self.warmup_scheduler.step(self.iteration)
        else:
            self.scheduler.step(self.iteration)

    def _exchange_and_update(self, max_grad_norm=None):
        opt, world = self.optimizer, self.world
        if self._arena_opt._symm is not None:
            opt.step_exchange()                                      # reduce + AdamW + broadcast in one peer-memory kernel
        else:
            if world > 1:
                solver.allreduce_grads(opt.arena, self.bucket_bytes, self.group)
            opt.step(grad_scale=1.0 / world, max_grad_norm=max_grad_norm)   # clips the rank mean, as DDP + clip_grad_norm_

    # ------------------------------------------------------------------ captured step
    def _capture(self, images, targets):
        model, opt = self.model, self._arena_opt
        dev = images.device
        pred, lossev = model.heads.predictor, model.heads.loss_evaluator
        if isinstance(targets, EncodedTargets):
            prep, targets = targets.prepared, targets.edge_targets()
        else:
            prep = lossev.prepare_targets(targets, dev)
        g = {"x": images.clone(), "prep": tuple(t.clone() for t in prep), "update_inside": self.world == 1 and opt._symm is None}
        opt._lr_table()                        # table and hyper-parameter block current: the captured step() copies nothing
        pred._targets_preloaded = True
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        try:
            with torch.cuda.graph(graph):
                loss_dict, log = model._forward_train(g["x"], targets, prepared=g["prep"], sync_log=False)
                losses = sum(loss_dict.values())
                opt.zero_grad()
                losses.backward()
                if g["update_inside"]:
                    self.optimizer.step(grad_scale=1.0, max_grad_norm=self.grad_norm_clip)
        finally:
            pred._targets_preloaded = False
        if g["update_inside"]:                 # capture only records: undo the host-side bookkeeping of the captured step()
            opt.step_count -= 1
            opt._step_t -= 1
        g.update(graph=graph, loss_dict={k: v.detach() for k, v in loss_dict.items()}, log=log, plan_h=pred.last_plan)
        self._graph = g
        return g

    def _step_graph(self, images, targets, sync_log=True):
        model, opt = self.model, self._arena_opt
        g = self._graph
        if g is None:
            g = self._capture(images, targets)
        if tuple(images.shape) != tuple(g["x"].shape):
            raise RuntimeError("captured training step: batch shape changed from %s to %s" % (tuple(g["x"].shape), tuple(images.shape)))
        g["x"].copy_(images, non_blocking=True)
        if isinstance(targets, EncodedTargets):               # encoded straight into the step's static buffers
            targets.encode_into(g["prep"], (g["plan_h"].edge_idx, g["plan_h"].edge_len))
        else:
            for dst, src in zip(g["prep"], model.heads.loss_evaluator.prepare_targets(targets, images.device)):
                dst.copy_(src, non_blocking=True)
            model.heads.predictor.load_targets(g["plan_h"], targets)
        opt._lr_table()                              # in-place refresh of the lr table / hyper block the schedule moved
        g["graph"].replay()
        if g["update_inside"]:
            opt.step_count += 1
            opt._step_t += 1
            for p in opt.arena.tensors:
                torch.autograd.graph.increment_version(p)
        else:
            self._exchange_and_update(max_grad_norm=self.grad_norm_clip)
        self._schedule_step()
        self.iteration += 1
        return g["loss_dict"], (g["log"].resolve() if sync_log else g["log"].snapshot())
