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
"""
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

    def __init__(self, params, lr=3e-4, betas=(0.9, 0.99), eps=1e-8, weight_decay=1e-5, symmetric_group=None,
                 capturable=True, check_finite=True):
        """capturable (default): `step()` keeps the step count on the device and guards the update with a finite scan of the
        gradient arena (`mf_adamw_step_dyn`: a non-finite gradient skips the update, `skipped_steps()` counts them), so a
        whole training step can be captured in one CUDA graph; capturable=False is the host-scalar `mf_adamw_step` launch.
        symmetric_group: a torch.distributed process group (NCCL, one rank per GPU of ONE NVLink domain). When given,
        the parameter and gradient arenas are allocated in symmetric (peer-mapped) memory and `step_exchange()` replaces
        `allreduce_grads(); step(grad_scale=1/world)` by the fused reduce-scatter + AdamW + all-gather kernel."""
        # amsgrad / maximize / foreach / capturable / differentiable / fused: the keys torch.optim.AdamW.load_state_dict
        # expects in every param group, so a checkpoint written here loads into the reference's optimiser and vice versa
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=False, maximize=False,
                                      foreach=None, capturable=False, differentiable=False, fused=None))
        self.capturable, self.check_finite = bool(capturable), bool(check_finite)
        tensors = [p for g in self.param_groups for p in g["params"]]
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
        for i, p in enumerate(self.arena.tensors):
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

    def _lr_table(self):
        lrs = tuple(0.0 if skip else g["lr"] for (g, skip) in zip((g for g in self.param_groups for _ in g["params"]), self._skip))
        if lrs != self._lr_key:
            table = self.arena.chunk_table(lrs).to(self.arena.params.device)
            if self._chunk_lr is None or self._chunk_lr.shape != table.shape:
                self._chunk_lr = table
            else:
                self._chunk_lr.copy_(table)               # in place: a captured graph keeps reading the same buffer
            self._lr_key = lrs
        return self._chunk_lr

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


def build_optimizer(model, cfg):
    """solver/__init__.py:26-62. Only the 'adamw' optimiser of runs/monoflex.yaml:62 is built."""
    name = cfg.SOLVER.OPTIMIZER
    if name != "adamw":
        raise NotImplementedError("optimizer %r: only 'adamw' (runs/monoflex.yaml) is implemented" % name)
    return FusedAdamW(get_model_params(model, cfg), lr=cfg.SOLVER.BASE_LR, weight_decay=cfg.SOLVER.WEIGHT_DECAY,
                      betas=(0.9, 0.99))


def build_scheduler(optimizer, optim_cfg, last_epoch=-1, total_iters_each_epoch=None):
    """solver/__init__.py:64-92 without the fastai one-cycle branch: multi-step LambdaLR (+ no warm-up, LR_WARMUP False).
    Same keyword interface as the reference (`build_scheduler(optimizer, total_iters_each_epoch=..., optim_cfg=...)`,
    tools/plain_train_net.py:86-90); `total_iters_each_epoch` only feeds the one-cycle branch and is ignored."""
    decay_steps = optim_cfg.STEPS

    def lr_lbmd(cur_epoch):
        cur_decay = 1
        for decay_step in decay_steps:
            if cur_epoch >= decay_step:
                cur_decay = cur_decay * optim_cfg.LR_DECAY
        return max(cur_decay, optim_cfg.LR_CLIP / optim_cfg.BASE_LR)

    if optim_cfg.LR_WARMUP:
        raise NotImplementedError("LR_WARMUP (CosineWarmupLR) is not built; runs/monoflex.yaml:65 sets it False")
    return torch.optim.lr_scheduler.LambdaLR(optimizer, lr_lbmd, last_epoch=last_epoch), None
