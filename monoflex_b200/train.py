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

`loss_scale`: a float is the static loss scale of the fp16 backward (`model.loss_scale`, default 128 or MF_LOSS_SCALE);
"dynamic" (or MF_LOSS_SCALE=dynamic) or a `loss_scale.DynamicLossScale` turns on the dynamic scale: `model.loss_scaler`
seeds the backward with the device scale, unscales into p.grad on the device, and every optimiser step (eager or
captured, after the NCCL all-reduce on several GPUs, so every rank keeps the same scale) updates it by GradScaler's rule
from the finite guard's skip decision. `trainer.scaler` is the DynamicLossScale, None for a static scale. Not available
with `symmetric_group` (the peer-memory exchange kernel has no finite guard).
"""
import collections
import datetime
import logging
import os
import time

import torch
import torch.distributed as dist

from . import loss_scale as _loss_scale
from . import parallel
from . import solver
from .targets import EncodedTargets


class Trainer(object):
    def __init__(self, model, cfg, loss_scale=None, symmetric_group=None, process_group=None, bucket_bytes=32 << 20,
                 use_cuda_graph=False, graph_warmup=2, optimizer=None, scheduler=None, warmup_scheduler=None,
                 start_iteration=0):
        if optimizer is not None:
            solver.check_fused(optimizer)
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
        static_scale, self.scaler = _loss_scale.resolve(loss_scale)
        if self.scaler is not None and symmetric_group is not None:
            raise NotImplementedError("a dynamic loss scale with symmetric_group: the fused peer-memory exchange kernel has "
                                      "no finite guard to update the scale from; use the NCCL exchange (no symmetric_group)")
        self.model = model.train()
        if static_scale is not None:
            model.loss_scale = static_scale
        self.cfg = cfg
        self.group = process_group
        self.bucket_bytes = bucket_bytes
        given = optimizer is not None
        self.optimizer = optimizer if given else solver.build_optimizer(model, cfg, symmetric_group=symmetric_group)
        self._arena_opt = getattr(self.optimizer, "opt", self.optimizer)    # FusedOneCycleAdam wraps its arena optimiser
        if self.scaler is not None:
            self.scaler.attach(self._arena_opt)
        model.loss_scaler = self.scaler
        if given:
            if scheduler is None or (cfg.SOLVER.LR_WARMUP and warmup_scheduler is None):
                raise ValueError("Trainer(optimizer=...): pass its scheduler%s too (build_scheduler's)"
                                 % (" and warmup_scheduler" if cfg.SOLVER.LR_WARMUP else ""))
            self.scheduler, self.warmup_scheduler = scheduler, warmup_scheduler
        else:
            self.scheduler, self.warmup_scheduler = solver.build_scheduler(self.optimizer, cfg.SOLVER)
        # indexed stepping of do_train (engine/trainer.py:123-126) with a warm-up or one-cycle schedule, or with the
        # caller's schedulers
        self._indexed_schedule = given or onecycle or self.warmup_scheduler is not None
        self.warmup_iters = solver.solver_value(cfg.SOLVER, "WARMUP_STEPS") if cfg.SOLVER.LR_WARMUP else -1
        self.iteration = int(start_iteration)      # the 0-based index of the next step, which the indexed schedules read
        self._eager_steps = 0
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
        if self.use_cuda_graph and self._eager_steps >= self.graph_warmup:
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
        self._eager_steps += 1
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
            opt.step(grad_scale=1.0 / world, max_grad_norm=max_grad_norm,   # clips the rank mean, as DDP + clip_grad_norm_
                     loss_scaler=self.scaler)

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
                    self.optimizer.step(grad_scale=1.0, max_grad_norm=self.grad_norm_clip, loss_scaler=self.scaler)
        finally:
            pred._targets_preloaded = False
        if g["update_inside"]:                 # capture only records: undo the host-side bookkeeping of the captured step()
            opt.step_count -= 1
            opt._step_t -= 1
        # the graph owns the plans whose buffers it reads: an eval forward between steps (do_eval) replaces the backbone's
        # and the predictor's cached plan, which would otherwise free the train plans' buffers under the graph
        g.update(graph=graph, loss_dict={k: v.detach() for k, v in loss_dict.items()}, log=log, plan_h=pred.last_plan,
                 plan_b=model.backbone.last_plan)
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


# ---------------------------------------------------------------------------------------------------------------- do_train
class SmoothedValue(object):
    """utils/metric_logger.py's meter: the last `window` values as float32 (`value`, `avg`) and a float64 running mean"""

    def __init__(self, window=10):
        self.deque = collections.deque(maxlen=window)
        self.total = 0.0
        self.count = 0

    def update(self, value):
        self.deque.append(value)
        self.count += 1
        self.total += value

    @property
    def value(self):
        return torch.tensor(list(self.deque))[-1].item()

    @property
    def avg(self):
        return torch.tensor(list(self.deque)).mean().item()

    @property
    def global_avg(self):
        return self.total / self.count


class MetricLogger(object):
    """utils/metric_logger.py's MetricLogger on host floats: meters in first-update order, str() their windowed means"""

    def __init__(self, delimiter=" "):
        self.meters = collections.OrderedDict()
        self.delimiter = delimiter

    def update(self, **kwargs):
        for k, v in kwargs.items():
            self.meters.setdefault(k, SmoothedValue()).update(float(v))

    def __str__(self):
        return self.delimiter.join("{}: {:.4f}".format(name, m.avg) for name, m in self.meters.items())


LOSS_SCALE_KEY = "mf_loss_scale"       # the dynamic loss scale's state in a checkpoint's extra data (`arguments`)


def do_eval(cfg, model, data_loaders_val, iteration):
    """engine/trainer.py's do_eval on monoflex_b200.inference.inference: OUTPUT_DIR/<DATASETS.TEST[0]>/inference_<iter>"""
    from .inference import inference
    dataset_name = cfg.DATASETS.TEST[0]
    output_folder = os.path.join(cfg.OUTPUT_DIR, dataset_name, "inference_{}".format(iteration))
    os.makedirs(output_folder, exist_ok=True)
    ret = inference(model, data_loaders_val, dataset_name=dataset_name, eval_types=("detection",),
                    device=cfg.MODEL.DEVICE, output_folder=output_folder)
    parallel.barrier()
    return ret


class _PendingSteps(object):
    """The host side of do_train's per-iteration records, in iteration order, each with its step's DeferredLog snapshot.
    `resolve(keep)` waits for the copies of all but the last `keep` steps - steps enqueued at least `keep` iterations ago,
    which the GPU has usually finished - and feeds them to the meters, TensorBoard and the log as the reference's loop
    does at the end of each iteration."""

    def __init__(self, emit):
        self.items = collections.deque()
        self.emit = emit

    def push(self, **item):
        self.items.append(item)

    def resolve(self, keep=0):
        while len(self.items) > keep:
            item = self.items.popleft()
            item["log_loss_dict"] = item.pop("log").resolve()
            self.emit(**item)


def do_train(cfg, distributed, model, data_loader, data_loaders_val, optimizer, scheduler, warmup_scheduler, checkpointer,
             device, arguments, lag=2, graph_warmup=2):
    """engine/trainer.py:do_train with the same signature and side effects, each step one replay of the captured Trainer
    step (use_cuda_graph=True). `optimizer` is a fused optimiser of solver.build_optimizer and `scheduler` /
    `warmup_scheduler` those of solver.build_scheduler, the objects `checkpointer` saves; they are stepped as do_train
    steps them. A DistributedDataParallel `model` is unwrapped: the gradient exchange is the Trainer's.

    The logged scalars of each step are DeferredLog snapshots read `lag` iterations late, so the host never waits for the
    step it has just enqueued; the meters, the TensorBoard scalars and the log lines are written from them at the
    reference's global steps and in its order. At a checkpoint or an evaluation every pending step is resolved first.
    A dynamic loss scale is saved with the checkpoints under arguments[LOSS_SCALE_KEY] and restored from it."""
    from torch.utils.tensorboard import SummaryWriter
    solver.check_fused(optimizer)
    logger = logging.getLogger("monoflex.trainer")
    logger.info("Start training")
    net = model.module if isinstance(model, torch.nn.parallel.DistributedDataParallel) else model
    meters = MetricLogger(delimiter=" ")
    max_iter = cfg.SOLVER.MAX_ITERATION
    start_iter = arguments["iteration"]
    if cfg.SOLVER.LR_WARMUP and warmup_scheduler is None:
        raise ValueError("do_train: SOLVER.LR_WARMUP needs the warm-up scheduler of build_scheduler")
    trainer = Trainer(net, cfg, use_cuda_graph=True, graph_warmup=graph_warmup, optimizer=optimizer, scheduler=scheduler,
                      warmup_scheduler=warmup_scheduler, start_iteration=start_iter)
    if trainer.scaler is not None and LOSS_SCALE_KEY in arguments:
        trainer.scaler.load_state_dict(arguments[LOSS_SCALE_KEY])
    rank = dist.get_rank() if (dist.is_available() and dist.is_initialized()) else 0
    local_rank = int(os.environ.get("LOCAL_RANK", rank % max(torch.cuda.device_count(), 1)))
    default_depth_method = cfg.MODEL.HEAD.OUTPUT_DEPTH
    by_epoch = getattr(cfg.SOLVER, "EVAL_AND_SAVE_EPOCH", False)
    writer = None
    best = dict(mAP=0, result_str=None, iteration=0, eval_iteration=0)
    record_metrics = ['Car_bev_', 'Car_3d_']
    if local_rank == 0:
        writer = SummaryWriter(os.path.join(cfg.OUTPUT_DIR, 'writer/{}/'.format(cfg.START_TIME)))

    def emit(iteration, log_loss_dict, batch_time, data_time, lr):
        """the reference loop's bookkeeping of one iteration (engine/trainer.py: from meters.update on)"""
        meters.update(loss=sum(loss for key, loss in log_loss_dict.items() if key.find('loss') >= 0), **log_loss_dict)
        meters.update(time=batch_time, data=data_time)
        eta_string = str(datetime.timedelta(seconds=int(meters.meters["time"].global_avg * (max_iter - iteration))))
        if rank == 0:
            writer.add_scalars('train_metric/depth_errors',
                               {k: m.value for k, m in meters.meters.items() if k.find('MAE') >= 0}, iteration)
            writer.add_scalar('stat/lr', lr, iteration)
            for name, meter in meters.meters.items():
                if name.find('MAE') >= 0:
                    continue
                writer.add_scalar(("stat/{}" if name in ('time', 'data') else "train_metric/{}").format(name), meter.value,
                                  iteration)
        if iteration % 10 == 0 or iteration == max_iter:
            logger.info(meters.delimiter.join(["eta: {eta}", "iter: {iter}", "{meters}", "lr: {lr:.8f} \n"]).format(
                eta=eta_string, iter=iteration, meters=str(meters), lr=lr))

    def save(name):
        if trainer.scaler is not None:
            arguments[LOSS_SCALE_KEY] = trainer.scaler.state_dict()
        checkpointer.save(name, **arguments)

    pending = _PendingSteps(emit)
    net.train()
    start_training_time = time.time()
    end = time.time()
    for iteration, data in zip(range(start_iter, max_iter), data_loader):
        data_time = time.time() - end
        if "encoded" in data:                       # a KittiTrainLoader batch: targets already encoded on the device
            images, targets = data["images"].tensors, data["encoded"]
        else:
            images = data["images"].to(device, non_blocking=True)     # pinned host batches go up without blocking
            images = getattr(images, "tensors", images)
            targets = [target.to(device) for target in data["targets"]]
        _, log = trainer.step(images, targets, sync_log=False)
        if log._event is None:                      # an eager warm-up step: its buffers are its own, copy them out too
            log = log.snapshot()
        iteration += 1
        arguments["iteration"] = iteration
        batch_time = time.time() - end
        end = time.time()
        pending.push(iteration=iteration, log=log, batch_time=batch_time, data_time=data_time,
                     lr=optimizer.param_groups[0]["lr"])
        ckpt = iteration % cfg.SOLVER.SAVE_CHECKPOINT_INTERVAL == 0
        evaluate = iteration % cfg.SOLVER.EVAL_INTERVAL == 0
        pending.resolve(0 if (ckpt or evaluate or iteration == max_iter) else lag)
        if ckpt:
            logger.info('iteration = {}, saving checkpoint ...'.format(iteration))
            if rank == 0:
                save("model_checkpoint")
        if iteration == max_iter and rank == 0:
            save("model_final")
        if evaluate:
            if by_epoch:
                cur_epoch = iteration // arguments["iter_per_epoch"]
                logger.info('epoch = {}, evaluate model on validation set with depth {}'.format(cur_epoch,
                                                                                                default_depth_method))
            else:
                logger.info('iteration = {}, evaluate model on validation set with depth {}'.format(
                    iteration, default_depth_method))
            result_dict, result_str, dis_ious = do_eval(cfg, net, data_loaders_val, iteration)
            if rank == 0:
                result_dict = result_dict[0]            # the R40 results
                for key, value in result_dict.items():
                    for metric in record_metrics:
                        if key.find(metric) >= 0:
                            threshold = key[len(metric): len(metric) + 4]
                            writer.add_scalar("eval_{}_{}/{}".format(default_depth_method, threshold, key), float(value),
                                              best["eval_iteration"] + 1)
                for key, value in dis_ious.items():
                    writer.add_scalar("IoUs_{}/{}".format(key, default_depth_method), value, best["eval_iteration"] + 1)
                eval_mAP = float(result_dict['{}_3d_{:.2f}/moderate'.format('Car', 0.7)])
                if eval_mAP >= best["mAP"]:
                    best.update(mAP=eval_mAP, iteration=iteration, result_str=result_str)
                    save("model_moderate_best_{}".format(default_depth_method))
                    if by_epoch:
                        logger.info('epoch = {}, best_mAP = {:.2f}, updating best checkpoint for depth {} \n'.format(
                            cur_epoch, eval_mAP, default_depth_method))
                    else:
                        logger.info('iteration = {}, best_mAP = {:.2f}, updating best checkpoint for depth {} \n'.format(
                            iteration, eval_mAP, default_depth_method))
                best["eval_iteration"] += 1
            net.train()
            parallel.barrier()
    pending.resolve(0)
    total_training_time = time.time() - start_training_time
    total_time_str = str(datetime.timedelta(seconds=total_training_time))
    if writer is not None:
        writer.flush()
    if rank == 0:
        logger.info("Total training time: {} ({:.4f} s / it), best model is achieved at iteration = {}".format(
            total_time_str, total_training_time / (max_iter), best["iteration"]))
        logger.info('The best performance is as follows')
        if best["result_str"] is None:       # the reference's '\n' + None raises here
            logger.info('no evaluation ran before iteration {}'.format(max_iter))
        else:
            logger.info('\n' + best["result_str"])
    return trainer
