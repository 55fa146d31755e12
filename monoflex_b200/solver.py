"""Optimiser side of the training step (SURVEY §8 row R13; reference solver/__init__.py:10-37, engine/trainer.py:103-126).

The reference builds ``torch.optim.AdamW`` with ONE param group per tensor (``get_model_params``: lr = BASE_LR, or
BASE_LR * BIAS_LR_FACTOR when "bias" is in the parameter name) - ~280 groups, so eager torch runs ~1000 tiny kernels per
step - and DDP all-reduces 280 gradient tensors (83.8 MB) in its own buckets.

Here every trainable tensor lives in ONE flat fp32 arena (``ParamArena``): ``p.data`` and ``p.grad`` become views of the
parameter / gradient arenas, each tensor padded to ``mf_adamw_chunk()`` elements so a per-chunk lr table can stand in for
the param groups. ``FusedAdamW.step()`` is then a single hand-written kernel launch (``mf_adamw_step``, 28 B/parameter),
``zero_grad()`` one memset and the gradient all-reduce a few large chunk-aligned buckets of the same arena
(``allreduce_grads``; NCCL SUM, the 1/world_size of the mean is folded into the AdamW kernel's ``grad_scale``).

``FusedAdamW`` subclasses ``torch.optim.Optimizer`` so the reference's ``LambdaLR`` / ``CosineWarmupLR`` schedulers and
``state_dict()`` checkpointing (utils/check_point.py) keep working: ``param_groups`` has the reference's one-group-per-
tensor layout and ``state[p]`` exposes ``step / exp_avg / exp_avg_sq`` (views of the moment arenas).
There is no CPU fallback: ``step()`` raises if the arena is not on a CUDA device.

The reference's other ``SOLVER.OPTIMIZER`` values run on the same arena and the same guarded, clipping, capturable step
(``mf_optim_step_dyn``: one update pass, 28 B/parameter), with the hyper-parameters a schedule moves every step (lr
multiplier, beta1, weight decay) in a small device block the host rewrites in place before each launch or graph replay:

* ``'adam'`` -> ``FusedAdam``: ``torch.optim.Adam`` (coupled L2 weight decay, ``g + wd * p``) over the same groups as
  ``'adamw'``; its ``state_dict`` loads into ``torch.optim.Adam`` and back.
* ``'adam_onecycle'`` -> ``FusedOneCycleAdam``: fastai's ``OptimWrapper`` over ``Adam(betas=(0.9, 0.99))`` with
  ``true_wd=True, bn_wd=True`` (solver/__init__.py:45-58, fastai_optim.py:101-233): two groups (non-BN leaf modules, BN
  leaf modules) at one shared lr, every grouped tensor decayed by ``1 - wd * lr`` - also those whose gradient is None, which
  Adam then skips - and Adam with ``betas = (mom, 0.99)``. Parameters owned by a module that has children (every ``DCN``:
  its ``weight`` / ``bias`` beside the ``conv_offset_mask`` child) are in no group and never change, as in the reference.
* ``build_scheduler``: ``OneCycle`` for the one-cycle optimiser, ``LambdaLR`` (+ ``CosineWarmupLR`` with ``LR_WARMUP``)
  otherwise (learning_schedules_fastai.py:12-91), restated here.
"""
import math

import numpy as np
import torch
import torch.distributed as dist

ADAMW_CHUNK = 512          # must equal mf_adamw_chunk(); checked when the library is loaded in FusedAdamW.__init__


def get_model_params(model, cfg):
    """solver/__init__.py:10-24: one group per trainable tensor, bias tensors at BASE_LR * BIAS_LR_FACTOR."""
    base_lr = cfg.SOLVER.BASE_LR
    params = []
    for key, value in model.named_parameters():
        if not value.requires_grad:
            continue
        key_lr = [base_lr]
        if "bias" in key:
            key_lr.append(base_lr * cfg.SOLVER.BIAS_LR_FACTOR)
        params.append({"params": [value], "lr": max(key_lr)})
    return params


class ParamArena:
    """Flat fp32 storage for a list of parameters: `.params`, `.grads` (and the AdamW moments) share one layout in which
    tensor i occupies [offset_i, offset_i + numel_i) and offset_i is a multiple of `chunk` elements."""

    def __init__(self, tensors, chunk=ADAMW_CHUNK, alloc=None):
        """alloc(numel, device) -> flat fp32 tensor; default torch.zeros (FusedAdamW passes a symmetric-memory allocator
        when the fused NVLink gradient exchange is requested)."""
        tensors = list(tensors)
        if not tensors:
            raise ValueError("ParamArena: no parameters")
        dev = tensors[0].device
        for p in tensors:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("ParamArena: all parameters must be fp32 on one device")
        self.chunk = int(chunk)
        self.tensors = tensors
        self.offsets, off = [], 0
        for p in tensors:
            self.offsets.append(off)
            off += -(-p.numel() // self.chunk) * self.chunk
        self.numel = off
        self.n_chunks = off // self.chunk
        if alloc is None:
            alloc = lambda n, d: torch.zeros(n, dtype=torch.float32, device=d)
        self.params = alloc(off, dev)
        self.grads = alloc(off, dev)
        with torch.no_grad():
            for p, o in zip(tensors, self.offsets):
                n = p.numel()
                self.params[o:o + n].copy_(p.detach().reshape(-1))
                if p.grad is not None:
                    self.grads[o:o + n].copy_(p.grad.reshape(-1))
                p.data = self.params[o:o + n].view(p.shape)
                p.grad = self.grads[o:o + n].view(p.shape)

    def view(self, flat, i):
        o, p = self.offsets[i], self.tensors[i]
        return flat[o:o + p.numel()].view(p.shape)

    def chunk_table(self, per_tensor_values):
        """fp32 [n_chunks] table holding tensor i's value on each of its chunks."""
        t = torch.zeros(self.n_chunks, dtype=torch.float32)
        for (o, p, v) in zip(self.offsets, self.tensors, per_tensor_values):
            t[o // self.chunk: (o + p.numel() + self.chunk - 1) // self.chunk] = float(v)
        return t

    def buckets(self, bucket_bytes):
        """chunk-aligned [lo, hi) element ranges of at most bucket_bytes covering the arena (last bucket first: gradients
        of the head are produced first by backward, so it can be reduced while the backbone's are still being computed)."""
        per = max(self.chunk, (int(bucket_bytes) // 4) // self.chunk * self.chunk)
        spans = [(lo, min(lo + per, self.numel)) for lo in range(0, self.numel, per)]
        return spans[::-1]


def allreduce_grads(arena, bucket_bytes=32 << 20, group=None, async_op=False):
    """SUM-all-reduce the gradient arena in a few large buckets (DDP's job in the reference, tools/plain_train_net.py:100-104).
    Returns (world_size, handles): pass 1/world_size as `grad_scale` to FusedAdamW.step for DDP's gradient mean."""
    if not (dist.is_available() and dist.is_initialized()):
        return 1, []
    world = dist.get_world_size(group)
    if world == 1:
        return 1, []
    handles = []
    for lo, hi in arena.buckets(bucket_bytes):
        h = dist.all_reduce(arena.grads[lo:hi], op=dist.ReduceOp.SUM, group=group, async_op=True)
        handles.append(h)
    if not async_op:
        for h in handles:
            h.wait()
        handles = []
    return world, handles


class FusedAdamW(torch.optim.Optimizer):
    """torch.optim.AdamW(model_params, lr, betas=(0.9, 0.99), weight_decay) (solver/__init__.py:36-37) with the update of
    ALL tensors in one kernel launch over a ParamArena."""

    _rule = None            # None: the mf_adamw_step* entry points; MF_OPTIM_* rule of mf_optim_step_dyn in the subclasses

    def __init__(self, params, lr=3e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-5, symmetric_group=None,
                 capturable=True, check_finite=True, outside_params=()):
        """capturable (default): `step()` keeps the step count on the device and guards the update with a finite scan of the
        gradient arena (`mf_adamw_step_dyn`: a non-finite gradient skips the update, `skipped_steps()` counts them), so a
        whole training step can be captured in one CUDA graph; capturable=False is the host-scalar `mf_adamw_step` launch.
        symmetric_group: a torch.distributed process group (NCCL, one rank per GPU of ONE NVLink domain). When given,
        the parameter and gradient arenas are allocated in symmetric (peer-mapped) memory and `step_exchange()` replaces
        `allreduce_grads(); step(grad_scale=1/world)` by the fused reduce-scatter + AdamW + all-gather kernel.
        outside_params: trainable tensors in no param group. They get arena storage (so zero_grad, the all-reduce and the
        clipping norm cover their gradients, as they cover every model parameter in the reference) but are never updated."""
        # amsgrad / maximize / foreach / capturable / differentiable / fused: the keys torch.optim.AdamW.load_state_dict
        # expects in every param group, so a checkpoint written here loads into the reference's optimiser and vice versa
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                                      foreach=None, capturable=False, differentiable=False, fused=None))
        self.capturable, self.check_finite = bool(capturable), bool(check_finite)
        self.n_grouped = sum(len(g["params"]) for g in self.param_groups)
        tensors = [p for g in self.param_groups for p in g["params"]] + list(outside_params)
        if len({id(p) for p in tensors}) != len(tensors):
            raise ValueError("FusedAdamW: a parameter appears in more than one group")
        for g in self.param_groups:
            g.setdefault("initial_lr", g["lr"])
            if (g["betas"], g["eps"], g["weight_decay"]) != (self.defaults["betas"], self.defaults["eps"],
                                                              self.defaults["weight_decay"]):
                raise NotImplementedError("FusedAdamW: betas / eps / weight_decay must be the same for every group "
                                          "(the reference only varies lr, solver/__init__.py:18-24)")
        self._symm = None
        alloc = None
        if symmetric_group is not None:
            import torch.distributed._symmetric_memory as symm_mem

            def alloc(n, dev):
                t = symm_mem.empty(n, dtype=torch.float32, device=dev)
                t.zero_()
                return t
        self.arena = ParamArena(tensors, alloc=alloc)
        if symmetric_group is not None:
            hp = symm_mem.rendezvous(self.arena.params, symmetric_group)
            hg = symm_mem.rendezvous(self.arena.grads, symmetric_group)
            self._symm = (hp, hg, symmetric_group)
        self.exp_avg = torch.zeros_like(self.arena.params)
        self.exp_avg_sq = torch.zeros_like(self.arena.params)
        self.step_count = 0
        self._lr_key = None
        self._chunk_lr = None
        self._skip = [False] * len(self.arena.tensors)     # tensors outside the forward graph (autograd leaves their grad None)
        dev = self.arena.params.device
        self._state4 = torch.zeros(4, dtype=torch.int64, device=dev)      # [step, found-non-finite, skipped steps, -]
        self._dyn16 = torch.zeros(4, dtype=torch.float32, device=dev)
        # per-CTA sums of squares of the clipping scan (mf_adamw_step_dyn_clip), allocated once so step() stays capturable
        self._norm_partials = torch.empty((self.arena.n_chunks + 1) // 2, dtype=torch.float64, device=dev)
        self.last_grad_norm = torch.full((), float("nan"), dtype=torch.float32, device=dev)
        self._bind_state()

    # -- torch.optim plumbing ---------------------------------------------------------------------------------------
    def _bind_state(self):
        self._step_t = torch.tensor(float(self.step_count))      # ONE tensor shared by every state entry
        for i, p in enumerate(self.arena.tensors[:self.n_grouped]):
            self.state[p] = {"step": self._step_t,
                             "exp_avg": self.arena.view(self.exp_avg, i),
                             "exp_avg_sq": self.arena.view(self.exp_avg_sq, i)}

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        steps = set()
        with torch.no_grad():
            for i, p in enumerate(self.arena.tensors):
                st = self.state.get(p)
                if not st:
                    continue
                self.arena.view(self.exp_avg, i).copy_(st["exp_avg"])
                self.arena.view(self.exp_avg_sq, i).copy_(st["exp_avg_sq"])
                steps.add(int(float(st["step"])))
        if len(steps) > 1:
            raise ValueError("FusedAdamW: per-tensor step counts differ in the checkpoint: %s" % sorted(steps))
        self.step_count = steps.pop() if steps else 0
        self._state4.zero_()
        self._state4[0] = self.step_count
        self._bind_state()
        self._lr_key = None

    def zero_grad(self, set_to_none=False):
        """one memset of the gradient arena; p.grad stays a view of it (set_to_none is ignored on purpose)."""
        self.arena.grads.zero_()

    def _group_of_tensor(self):
        """the param group of each arena tensor, None for outside_params"""
        return [g for g in self.param_groups for _ in g["params"]] + [None] * (len(self.arena.tensors) - self.n_grouped)

    def _lr_table(self):
        lrs = tuple(0.0 if (skip or g is None) else g["lr"] for (g, skip) in zip(self._group_of_tensor(), self._skip))
        self._upload_table(lrs)
        return self._chunk_lr

    def _upload_table(self, lrs):
        if lrs != self._lr_key:
            table = self.arena.chunk_table(lrs).to(self.arena.params.device)
            if self._chunk_lr is None or self._chunk_lr.shape != table.shape:
                self._chunk_lr = table
            else:
                self._chunk_lr.copy_(table)               # in place: a captured graph keeps reading the same buffer
            self._lr_key = lrs

    def mark_unused(self, names, model):
        """Parameters the forward never uses (e.g. the outer `project` of DLA's two-level trees, dla_dcn.py:249) get grad None
        from autograd in the reference and torch's AdamW skips them entirely (no weight decay, no moment update). Their
        arena gradient is always zero here; this marks them so the kernel skips their chunks too - independently of the
        param-group lr the scheduler keeps rewriting."""
        by_id = {id(p): i for i, p in enumerate(self.arena.tensors)}
        for n, p in model.named_parameters():
            if n in names and id(p) in by_id:
                self._skip[by_id[id(p)]] = True
        self._lr_key = None

    def skipped_steps(self):
        """number of optimiser steps skipped because the gradient arena held a non-finite value (host sync)"""
        return int(self._state4[2].item())

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0, max_grad_norm=None):
        """One AdamW update of the whole arena on `grad_scale * grads`.
        max_grad_norm > 0: `torch.nn.utils.clip_grad_norm_(params, max_grad_norm)` first, on the device and inside the same
        three launches (capturable): the norm of `grad_scale * grads` goes to `last_grad_norm` (a 0-d device tensor, the
        value clip_grad_norm_ returns; read it without a sync), the gradient arena is left clipped like p.grad after
        clip_grad_norm_ (still the SUM when grad_scale = 1/world), and a non-finite norm skips the step like any non-finite
        gradient. None or <= 0 (the reference's GRAD_NORM_CLIP = -1): no clipping, `last_grad_norm` is not written."""
        if closure is not None:
            raise NotImplementedError("FusedAdamW: closures are not used by the reference trainer")
        if not self.arena.params.is_cuda:
            raise RuntimeError("FusedAdamW.step: parameters are not on a CUDA device (there is no CPU path)")
        clip = max_grad_norm is not None and float(max_grad_norm) > 0
        if clip and not self.capturable:
            raise NotImplementedError("FusedAdamW.step: max_grad_norm needs the device-side step (capturable=True)")
        from . import _lib
        lib = _lib.load()
        if lib.mf_adamw_chunk() != self.arena.chunk:
            raise RuntimeError("FusedAdamW: arena chunk %d != library chunk %d" % (self.arena.chunk, lib.mf_adamw_chunk()))
        gbase, pbase = self.arena.grads.data_ptr(), self.arena.params.data_ptr()
        for p, o in zip(self.arena.tensors, self.arena.offsets):   # a caller that replaced .grad / .data breaks the arena
            g = p.grad                                              # contract: fail loudly instead of updating stale memory
            if g is None or g.data_ptr() != gbase + 4 * o or p.data_ptr() != pbase + 4 * o:
                raise RuntimeError("FusedAdamW: a parameter's .data / .grad no longer aliases the arena "
                                   "(use optimizer.zero_grad(), not set_to_none)")
        table = self._lr_table()
        self.step_count += 1
        b1, b2 = self.defaults["betas"]
        if self._rule is not None:
            if self.step_count == 1 and int(self._state4[0].item()) != 0:
                raise RuntimeError("%s: device step counter out of sync" % type(self).__name__)
            _lib.call("mf_optim_step_dyn", self._rule, self.arena.params.data_ptr(), self.arena.grads.data_ptr(),
                      self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), table.data_ptr(), self.arena.n_chunks,
                      self._hyper.data_ptr(), b2, self.defaults["eps"], float(grad_scale), self._state4.data_ptr(),
                      self._dyn16.data_ptr(), 1 if self.check_finite else 0, float(max_grad_norm) if clip else 0.0,
                      self._norm_partials.data_ptr(), self.last_grad_norm.data_ptr(), torch.cuda.current_stream().cuda_stream)
            self._step_t += 1
            for p in self.arena.tensors:
                torch.autograd.graph.increment_version(p)
            return None
        if self.capturable:
            if self.step_count == 1 and int(self._state4[0].item()) != 0:
                raise RuntimeError("FusedAdamW: device step counter out of sync")
            args = (self.arena.params.data_ptr(), self.arena.grads.data_ptr(), self.exp_avg.data_ptr(),
                    self.exp_avg_sq.data_ptr(), table.data_ptr(), self.arena.n_chunks, b1, b2, self.defaults["eps"],
                    self.defaults["weight_decay"], float(grad_scale), 1.0, self._state4.data_ptr(), self._dyn16.data_ptr(),
                    1 if self.check_finite else 0)
            if clip:
                _lib.call("mf_adamw_step_dyn_clip", *args, float(max_grad_norm), self._norm_partials.data_ptr(),
                          self.last_grad_norm.data_ptr(), torch.cuda.current_stream().cuda_stream)
            else:
                _lib.call("mf_adamw_step_dyn", *args, torch.cuda.current_stream().cuda_stream)
            self._step_t += 1
            for p in self.arena.tensors:
                torch.autograd.graph.increment_version(p)
            return None
        _lib.call("mf_adamw_step", self.arena.params.data_ptr(), self.arena.grads.data_ptr(), self.exp_avg.data_ptr(),
                  self.exp_avg_sq.data_ptr(), table.data_ptr(), self.arena.n_chunks, b1, b2, self.defaults["eps"],
                  self.defaults["weight_decay"], self.step_count, float(grad_scale), 1.0,
                  torch.cuda.current_stream().cuda_stream)
        self._step_t += 1
        for p in self.arena.tensors:            # cached kernel plans key on parameter versions (engine.fingerprint)
            torch.autograd.graph.increment_version(p)
        return None


def _fused_exchange_step(self, use_multicast=True):
    """DDP all-reduce + optimizer.step() as ONE kernel over NVLink peer memory (csrc/mf_train.cu adamw_p2p_kernel):
    barrier -> every rank reduces, updates and re-broadcasts its 1/world shard -> barrier. Call after backward, on the
    stream that produced the gradients. Needs FusedAdamW(..., symmetric_group=pg)."""
    import ctypes
    if self._symm is None:
        raise RuntimeError("FusedAdamW.step_exchange: construct the optimiser with symmetric_group=<process group>")
    from . import _lib
    hp, hg, _ = self._symm
    world, rank = hp.world_size, hp.rank
    table = self._lr_table()
    self.step_count += 1
    b1, b2 = self.defaults["betas"]
    pp = (ctypes.c_ulonglong * world)(*[int(x) for x in hp.buffer_ptrs])
    gp = (ctypes.c_ulonglong * world)(*[int(x) for x in hg.buffer_ptrs])
    mc_p = int(hp.multicast_ptr or 0) if use_multicast else 0     # 0 when the fabric / driver has no NVLS multicast
    mc_g = int(hg.multicast_ptr or 0) if use_multicast else 0
    if not (mc_p and mc_g):
        mc_p = mc_g = 0
    hg.barrier(channel=0)                       # every rank's backward has finished writing its gradient arena
    _lib.call("mf_adamw_step_p2p", ctypes.addressof(pp), ctypes.addressof(gp), world, rank, mc_p, mc_g,
              self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), table.data_ptr(), self.arena.n_chunks, b1, b2,
              self.defaults["eps"], self.defaults["weight_decay"], self.step_count, 1.0,
              torch.cuda.current_stream().cuda_stream)
    hp.barrier(channel=1)                       # every shard of the new parameters has landed in every arena
    self._step_t += 1
    for p in self.arena.tensors:
        torch.autograd.graph.increment_version(p)
    return bool(mc_p)


FusedAdamW.step_exchange = torch.no_grad()(_fused_exchange_step)


class FusedAdam(FusedAdamW):
    """torch.optim.Adam(params, lr, betas, weight_decay) (the reference's 'adam', solver/__init__.py:33-34) over a
    ParamArena, in the guarded capturable step of FusedAdamW: weight decay is coupled L2 (`g <- g + wd * p`, after any
    clipping), tensors marked unused (grad None in the reference) are not touched at all. `state_dict()` has
    torch.optim.Adam's layout and loads into it and back.

    Device hyper-parameter block (`_hyper`, float64 {lr multiplier, beta1, weight decay, 0}): refreshed in place by
    `_lr_table()`, which `step()` calls and the captured Trainer calls before each replay. When every updated tensor's group
    has the same lr, the chunk table holds 1 (0 / -1 for skipped / decay-only tensors) and the lr itself is the multiplier,
    so a schedule that moves one lr for all groups rewrites 8 bytes, not the table."""

    _rule = 1                       # MF_OPTIM_ADAM
    _unused_decays = False          # mark_unused tensors: skipped entirely (torch's Adam skips grad None)

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.0, check_finite=True,
                 outside_params=()):
        super().__init__(params, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, capturable=True,
                         check_finite=check_finite, outside_params=outside_params)
        self.defaults["decoupled_weight_decay"] = False            # torch.optim.Adam's group key (torch >= 2.6)
        for g in self.param_groups:
            g.setdefault("decoupled_weight_decay", False)
        self._hyper = torch.zeros(4, dtype=torch.float64, device=self.arena.params.device)
        self._hyper_key = None

    def _weight_decay(self):
        wds = {g["weight_decay"] for g in self.param_groups}
        if len(wds) != 1:
            raise NotImplementedError("%s: weight_decay must be the same for every group" % type(self).__name__)
        return float(wds.pop())

    def _lr_table(self):
        groups = self._group_of_tensor()
        betas = {tuple(g["betas"]) for g in self.param_groups}
        if len(betas) != 1 or tuple(betas)[0][1] != self.defaults["betas"][1]:
            raise NotImplementedError("%s: every group needs the same betas, and beta2 stays %r"
                                      % (type(self).__name__, self.defaults["betas"][1]))
        beta1 = float(tuple(betas)[0][0])
        unused = -1.0 if self._unused_decays else 0.0
        active = {float(g["lr"]) for g, skip in zip(groups, self._skip) if g is not None and (not skip or self._unused_decays)}
        if len(active) == 1:                  # one shared lr: it goes to the device block, the table holds its sign pattern
            mult = active.pop()
            vals = tuple(0.0 if g is None else (unused if skip else 1.0) for g, skip in zip(groups, self._skip))
        else:
            mult = 1.0
            vals = tuple(0.0 if g is None else (unused * g["lr"] if skip else g["lr"]) for g, skip in zip(groups, self._skip))
        self._upload_table(vals)
        key = (mult, beta1, self._weight_decay())
        if key != self._hyper_key:
            self._hyper.copy_(torch.tensor(key + (0.0,), dtype=torch.float64))   # in place, like the table
            self._hyper_key = key
        return self._chunk_lr

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._hyper_key = None

    def step_exchange(self, use_multicast=True):
        raise NotImplementedError("%s: the fused peer-memory exchange runs AdamW only" % type(self).__name__)


class _OneCycleInnerAdam(FusedAdam):
    """The inner optimiser of FusedOneCycleAdam: Adam with weight decay 0 after a decoupled decay of every grouped tensor by
    1 - wd * lr (fastai's true_wd step), wd held in `decoupled_wd`; one update pass (rule MF_OPTIM_ADAMW on the device)."""

    _rule = 0                       # MF_OPTIM_ADAMW: p * (1 - lr * wd), then Adam
    _unused_decays = True           # grouped tensors with grad None: decayed, not Adam-updated

    def __init__(self, params, betas, eps, outside_params):
        self.decoupled_wd = 0.0
        super().__init__(params, lr=1e-3, betas=betas, eps=eps, weight_decay=0.0, outside_params=outside_params)

    def _weight_decay(self):
        return float(self.decoupled_wd)


BN_TYPES = (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d, torch.nn.BatchNorm3d, torch.nn.SyncBatchNorm)


def onecycle_param_groups(model):
    """fastai's layer groups of the reference's 'adam_onecycle' (solver/__init__.py:46-53, fastai_optim.py:13-24): the leaf
    modules of `model` (modules without children), split into non-BN and BN leaves (nn.BatchNorm1d/2d/3d, SyncBatchNorm;
    InPlaceABN is not a BN type), each group the trainable parameters of its leaves. Returns ([non_bn, bn], outside): outside
    = the trainable parameters in neither group, those owned by a module that has children (every DCN's weight and bias)."""
    def leaves(m):
        kids = list(m.children())
        return [m] if not kids else [leaf for c in kids for leaf in leaves(c)]

    groups, seen = ([], []), set()
    for leaf in leaves(model):
        for p in leaf.parameters():
            if p.requires_grad and id(p) not in seen:
                seen.add(id(p))
                groups[1 if isinstance(leaf, BN_TYPES) else 0].append(p)
    outside = [p for p in model.parameters() if p.requires_grad and id(p) not in seen]
    return list(groups), outside


class FusedOneCycleAdam(object):
    """The reference's 'adam_onecycle' optimiser: `OptimWrapper.create(partial(Adam, betas=(0.9, 0.99)), lr,
    get_layer_groups(model), wd=wd, true_wd=True, bn_wd=True)` on the arena.

    It has the wrapper interface the reference's OneCycle and trainer touch: the `lr`, `mom`, `wd` and `beta` properties
    (single values, or lists of one: one layer group), `param_groups` (the inner Adam's two groups), `zero_grad()`,
    `step()` and `state_dict()` / `load_state_dict()` in the inner Adam's layout. `step()` is one device pass: every grouped
    tensor is decayed by 1 - wd * lr - those marked unused only that -, then Adam with weight decay 0 and betas
    (mom, beta), bias correction 1 - mom^step from the current mom. Parameters in no group are never changed. Anything else
    (`arena`, `mark_unused`, `skipped_steps`, `last_grad_norm`, ...) is the inner optimiser's (`.opt`)."""

    def __init__(self, model, lr, wd, betas=(0.9, 0.99), eps=1e-8):
        (non_bn, bn), outside = onecycle_param_groups(model)
        self.opt = _OneCycleInnerAdam([{"params": non_bn, "lr": 0.0}, {"params": bn, "lr": 0.0}], betas=betas, eps=eps,
                                      outside_params=outside)
        self.true_wd, self.bn_wd = True, True
        self._mom, self._beta, self._lr = [betas[0]], [betas[1]], [0.0]
        self.wd = wd
        self.lr = lr

    def __getattr__(self, k):
        if k == "opt":
            raise AttributeError(k)
        return getattr(self.opt, k)

    @staticmethod
    def _one(val):
        if isinstance(val, (list, tuple)):
            if len(val) != 1:
                raise ValueError("FusedOneCycleAdam: one layer group, got %d values" % len(val))
            val = val[0]
        return val

    def _set(self, key, val):
        for g in self.opt.param_groups:
            g[key] = val

    @property
    def param_groups(self):
        return self.opt.param_groups

    @property
    def lr(self):
        return self._lr[-1]

    @lr.setter
    def lr(self, val):
        self._lr = [self._one(val)]
        self._set("lr", self._lr[0])

    @property
    def mom(self):
        return self._mom[-1]

    @mom.setter
    def mom(self, val):
        self._mom = [self._one(val)]
        self._set("betas", (self._mom[0], self._beta[0]))

    @property
    def beta(self):
        return self._beta[-1]

    @beta.setter
    def beta(self, val):
        if val is None:
            return
        self._beta = [self._one(val)]
        self._set("betas", (self._mom[0], self._beta[0]))

    @property
    def wd(self):
        return self._wd[-1]

    @wd.setter
    def wd(self, val):
        self._wd = [self._one(val)]
        self.opt.decoupled_wd = float(self._wd[0])

    def zero_grad(self, set_to_none=False):
        self.opt.zero_grad()

    def step(self, closure=None, grad_scale=1.0, max_grad_norm=None):
        self._set("weight_decay", 0)               # true_wd: the decay is outside Adam
        return self.opt.step(closure, grad_scale=grad_scale, max_grad_norm=max_grad_norm)

    def state_dict(self):
        return self.opt.state_dict()

    def load_state_dict(self, state_dict):
        self.opt.load_state_dict(state_dict)
        g = self.opt.param_groups[0]
        self._lr, self._mom, self._beta = [g["lr"]], [g["betas"][0]], [g["betas"][1]]

    def __repr__(self):
        return "FusedOneCycleAdam over %d + %d tensors (%d in no group), true weight decay %r" % (
            len(self.opt.param_groups[0]["params"]), len(self.opt.param_groups[1]["params"]),
            len(self.opt.arena.tensors) - self.opt.n_grouped, self.wd)


OPTIMIZERS = ("adamw", "adam", "adam_onecycle")


def build_optimizer(model, cfg, symmetric_group=None):
    """solver/__init__.py:27-62: 'adamw' -> FusedAdamW, 'adam' -> FusedAdam (both over the one-group-per-tensor params),
    'adam_onecycle' -> FusedOneCycleAdam. 'sgd' (which reads SOLVER.MOMENTUM, a key config/defaults.py does not define)
    is not built. symmetric_group: the fused peer-memory exchange of FusedAdamW (AdamW only)."""
    sc = cfg.SOLVER
    name = sc.OPTIMIZER
    if name not in OPTIMIZERS:
        raise NotImplementedError("optimizer %r: the fused optimisers are %s" % (name, ", ".join(OPTIMIZERS)))
    if name != "adamw" and symmetric_group is not None:
        raise NotImplementedError("optimizer %r with symmetric_group: the fused peer-memory exchange kernel runs AdamW only"
                                  % name)
    if name == "adamw":
        kw = {} if symmetric_group is None else {"symmetric_group": symmetric_group}
        return FusedAdamW(get_model_params(model, cfg), lr=sc.BASE_LR, weight_decay=sc.WEIGHT_DECAY, betas=(0.9, 0.99), **kw)
    if name == "adam":
        return FusedAdam(get_model_params(model, cfg), lr=sc.BASE_LR, weight_decay=sc.WEIGHT_DECAY, betas=(0.9, 0.99))
    return FusedOneCycleAdam(model, sc.BASE_LR, sc.WEIGHT_DECAY, betas=(0.9, 0.99))


# ------------------------------------------------------------------ schedules (learning_schedules_fastai.py:12-91)
# config/defaults.py:255-275 values for the keys a cfg may not carry
SOLVER_DEFAULTS = dict(MAX_ITERATION=30000, MOMS=(0.95, 0.85), PCT_START=0.4, DIV_FACTOR=10, WARMUP_STEPS=-1)


def solver_value(optim_cfg, key):
    return getattr(optim_cfg, key, SOLVER_DEFAULTS[key])


def annealing_cos(start, end, pct):
    """cosine from `start` (pct 0) to `end` (pct 1), in numpy float64 like the reference"""
    return end + (start - end) / 2 * (np.cos(np.pi * pct) + 1)


class OneCycle(object):
    """fastai one-cycle over an optimiser with `lr` / `mom` properties (FusedOneCycleAdam): the constructor sets
    lr = lr_max / div_factor and mom = moms[0]; `step(i)` anneals lr from lr_max / div_factor up to lr_max and mom from
    moms[0] to moms[1] over the first int(total_step * pct_start) steps, then lr down to lr_max / div_factor / 1e4 and mom
    back to moms[0] until total_step (learning_schedules_fastai.py:12-79)."""

    def __init__(self, optimizer, total_step, lr_max, moms, div_factor, pct_start):
        self.optimizer, self.total_step = optimizer, total_step
        self.lr_max, self.moms, self.div_factor, self.pct_start = lr_max, moms, div_factor, pct_start
        low = lr_max / div_factor
        mid = int(total_step * pct_start)
        if not 0 < mid < total_step:
            raise ValueError("OneCycle: int(total_step * pct_start) = %d must lie in (0, %d)" % (mid, total_step))
        # (first step, end step, start value, end value) of each phase; a later phase overrides from its first step on
        self.lr_phases = ((0, mid, low, lr_max), (mid, total_step, lr_max, low / 1e4))
        self.mom_phases = ((0, mid, moms[0], moms[1]), (mid, total_step, moms[1], moms[0]))
        optimizer.lr, optimizer.mom = low, moms[0]

    def step(self, step):
        for attr, phases in (("lr", self.lr_phases), ("mom", self.mom_phases)):
            for lo, hi, a, b in phases:
                if step >= lo:
                    setattr(self.optimizer, attr, annealing_cos(a, b, (step - lo) / (hi - lo)))


class CosineWarmupLR(torch.optim.lr_scheduler.LRScheduler):
    """lr = eta_min + (base_lr - eta_min) * (1 - cos(pi * epoch / T_max)) / 2 (learning_schedules_fastai.py:82-91); the
    constructor's initial step sets every group's lr to eta_min."""

    def __init__(self, optimizer, T_max, eta_min=0, last_epoch=-1):
        self.T_max, self.eta_min = T_max, eta_min
        super().__init__(optimizer, last_epoch)

    def get_lr(self):
        return [self.eta_min + (base - self.eta_min) * (1 - math.cos(math.pi * self.last_epoch / self.T_max)) / 2
                for base in self.base_lrs]


def build_scheduler(optimizer, optim_cfg, last_epoch=-1, total_iters_each_epoch=None):
    """solver/__init__.py:64-92 -> (scheduler, warmup scheduler or None): `OneCycle(optimizer, MAX_ITERATION, BASE_LR, MOMS,
    DIV_FACTOR, PCT_START)` for a one-cycle optimiser, else the multi-step LambdaLR, plus with LR_WARMUP a
    `CosineWarmupLR(T_max=WARMUP_STEPS, eta_min=BASE_LR / DIV_FACTOR)` built after it (which sets every lr to eta_min).
    Keys the cfg lacks take config/defaults.py's values (SOLVER_DEFAULTS). Same keyword interface as the reference
    (`build_scheduler(optimizer, total_iters_each_epoch=..., optim_cfg=...)`, tools/plain_train_net.py:86-90);
    `total_iters_each_epoch` is unused there too. The reference's trainer steps them with the index of the step just taken
    (`warmup.step(i)` while i < WARMUP_STEPS, else `scheduler.step(i)`, engine/trainer.py:123-126)."""
    if str(optim_cfg.OPTIMIZER).find("onecycle") >= 0:
        return OneCycle(optimizer, solver_value(optim_cfg, "MAX_ITERATION"), optim_cfg.BASE_LR,
                        list(solver_value(optim_cfg, "MOMS")), solver_value(optim_cfg, "DIV_FACTOR"),
                        solver_value(optim_cfg, "PCT_START")), None
    decay_steps = optim_cfg.STEPS

    def lr_lbmd(cur_epoch):
        cur_decay = 1
        for decay_step in decay_steps:
            if cur_epoch >= decay_step:
                cur_decay = cur_decay * optim_cfg.LR_DECAY
        return max(cur_decay, optim_cfg.LR_CLIP / optim_cfg.BASE_LR)

    scheduler = torch.optim.lr_scheduler.LambdaLR(optimizer, lr_lbmd, last_epoch=last_epoch)
    warmup = None
    if optim_cfg.LR_WARMUP:
        warmup = CosineWarmupLR(optimizer, T_max=solver_value(optim_cfg, "WARMUP_STEPS"),
                                eta_min=optim_cfg.BASE_LR / solver_value(optim_cfg, "DIV_FACTOR"))
    return scheduler, warmup
