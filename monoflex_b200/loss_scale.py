"""Dynamic loss scale of the fp16 training backward, kept on the device (torch.amp.GradScaler's rule).

The backward tape (tape.py) carries activation gradients as fp16 rows, so the loss gradients are multiplied by a loss scale
before they enter it and the parameter gradients are divided by it again before they reach `p.grad`. A fixed scale either
leaves small gradients in fp16's subnormal range or overflows on large ones; `DynamicLossScale` moves it the way
`torch.amp.GradScaler` does: halve it on a step whose gradients are not finite (the step is skipped), double it after
`growth_interval` clean steps in a row.

`scale` (0-d float32) and `growth_tracker` (0-d int32) live on the GPU and are only ever changed in place by kernels:

  * the seeding multiply of `KeypointDetector._tape_backward` reads `scale`;
  * `unscale_accumulate` (one `mf_unscale_accumulate` launch) adds `src * inv_scale` into every `p.grad`, inv_scale =
    `scale.double().reciprocal().float()` computed on the device;
  * `update` (one `mf_loss_scale_update` launch) applies `torch._amp_update_scale_` to the skip decision the optimiser's
    finite guard has just published, in the same stream and with no host read.

So a training step captured in a CUDA graph keeps following the scale. Use it through `Trainer(model, cfg,
loss_scale="dynamic")` (or an instance, or `MF_LOSS_SCALE=dynamic`); by hand, `attach()` it to the fused optimiser, set
`model.loss_scaler` and pass it to `optimizer.step(loss_scaler=...)` after every backward.
"""
import torch

_KEYS = ("scale", "growth_factor", "backoff_factor", "growth_interval", "_growth_tracker")


class DynamicLossScale(object):
    def __init__(self, init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        """GradScaler's defaults. The state lives on the current CUDA device (each rank's own GPU)."""
        self.growth_factor, self.backoff_factor, self.growth_interval = self._check(init_scale, growth_factor,
                                                                                    backoff_factor, growth_interval)
        dev = torch.device("cuda", torch.cuda.current_device())
        self.scale = torch.full((), float(init_scale), dtype=torch.float32, device=dev)
        self.growth_tracker = torch.zeros((), dtype=torch.int32, device=dev)
        self.optimizer = None                   # the fused optimiser whose step updates the scale (attach())

    @staticmethod
    def _check(init_scale, growth_factor, backoff_factor, growth_interval):
        def num(name, v):
            if isinstance(v, bool) or not isinstance(v, (int, float)):
                raise ValueError("DynamicLossScale: %s must be a number, got %r" % (name, v))
            return float(v)
        s, g, b = num("init_scale", init_scale), num("growth_factor", growth_factor), num("backoff_factor", backoff_factor)
        if not (0.0 < s < float("inf")) or s > torch.finfo(torch.float32).max:
            raise ValueError("DynamicLossScale: init_scale must be a positive finite float32, got %r" % (init_scale,))
        if not g > 1.0 or g == float("inf"):
            raise ValueError("DynamicLossScale: growth_factor must be a finite number > 1, got %r" % (growth_factor,))
        if not 0.0 < b < 1.0:
            raise ValueError("DynamicLossScale: backoff_factor must lie in (0, 1), got %r" % (backoff_factor,))
        if isinstance(growth_interval, bool) or not isinstance(growth_interval, int) or not 1 <= growth_interval < 2 ** 31:
            raise ValueError("DynamicLossScale: growth_interval must be an int in [1, 2^31), got %r" % (growth_interval,))
        return g, b, int(growth_interval)

    def attach(self, optimizer):
        """bind to the fused optimiser (FusedAdamW / FusedAdam / FusedOneCycleAdam) whose step() will update the scale;
        the detector's backward refuses to run with a scaler no fused optimiser steps"""
        from . import solver
        inner = getattr(optimizer, "opt", optimizer)
        if not isinstance(inner, solver.FusedAdamW):
            raise TypeError("DynamicLossScale: the scale is updated by the fused optimiser step (solver.FusedAdamW, "
                            "FusedAdam, FusedOneCycleAdam), not by %s" % type(optimizer).__name__)
        if inner._symm is not None:
            raise NotImplementedError("DynamicLossScale with symmetric_group: the fused peer-memory exchange kernel has no "
                                      "finite guard to update the scale from; use the NCCL exchange")
        self.optimizer = inner
        return self

    # -- GradScaler's interface -------------------------------------------------------------------------------------
    def get_scale(self):
        """the current scale as a Python float (host read)"""
        return float(self.scale.item())

    def state_dict(self):
        """torch.amp.GradScaler's keys and types; loads into GradScaler("cuda") and back"""
        return {"scale": self.get_scale(), "growth_factor": self.growth_factor, "backoff_factor": self.backoff_factor,
                "growth_interval": self.growth_interval, "_growth_tracker": int(self.growth_tracker.item())}

    def load_state_dict(self, state_dict):
        missing = [k for k in _KEYS if k not in state_dict]
        if missing:
            raise RuntimeError("DynamicLossScale.load_state_dict: missing keys %s" % missing)
        g, b, n = self._check(state_dict["scale"], state_dict["growth_factor"], state_dict["backoff_factor"],
                              state_dict["growth_interval"])
        self.growth_factor, self.backoff_factor, self.growth_interval = g, b, n
        self.scale.fill_(float(state_dict["scale"]))                 # in place: a captured graph keeps reading this memory
        self.growth_tracker.fill_(int(state_dict["_growth_tracker"]))

    # -- device launches --------------------------------------------------------------------------------------------
    def unscale_accumulate(self, dsts, srcs, assign=None):
        """dst += src * inv_scale (or dst = src * inv_scale where assign[i]) for every pair, fp32 and dense, in one launch
        per mf_unscale_max_tensors() pairs"""
        import ctypes
        from . import _lib
        n = len(dsts)
        if len(srcs) != n or (assign is not None and len(assign) != n):
            raise ValueError("unscale_accumulate: %d destinations, %d sources" % (n, len(srcs)))
        dev = self.scale.device
        dptr, sptr, numel = [], [], []
        for d, s in zip(dsts, srcs):
            if (d.dtype != torch.float32 or s.dtype != torch.float32 or d.numel() != s.numel() or not d.is_contiguous()
                    or not s.is_contiguous() or d.device != dev or s.device != dev):
                raise ValueError("unscale_accumulate: dst and src must be dense fp32 tensors of one size on %s" % dev)
            dptr.append(d.data_ptr())
            sptr.append(s.data_ptr())
            numel.append(d.numel())
        cap = _lib.load().mf_unscale_max_tensors()
        stream = torch.cuda.current_stream(dev).cuda_stream
        for lo in range(0, n, cap):
            hi = min(n, lo + cap)
            k = hi - lo
            dp = (ctypes.c_ulonglong * k)(*dptr[lo:hi])
            sp = (ctypes.c_ulonglong * k)(*sptr[lo:hi])
            nn = (ctypes.c_longlong * k)(*numel[lo:hi])
            asg = None if assign is None else (ctypes.c_ubyte * k)(*[1 if a else 0 for a in assign[lo:hi]])
            _lib.call("mf_unscale_accumulate", ctypes.addressof(dp), ctypes.addressof(sp), ctypes.addressof(nn),
                      None if asg is None else ctypes.addressof(asg), k, self.scale.data_ptr(), stream)

    def update(self, dyn16):
        """torch._amp_update_scale_ on the skip flag the optimiser step just enqueued published in dyn16"""
        from . import _lib
        _lib.call("mf_loss_scale_update", dyn16.data_ptr(), self.scale.data_ptr(), self.growth_tracker.data_ptr(),
                  self.growth_factor, self.backoff_factor, self.growth_interval,
                  torch.cuda.current_stream(self.scale.device).cuda_stream)

    def __repr__(self):
        return "DynamicLossScale(growth_factor=%g, backoff_factor=%g, growth_interval=%d)" % (
            self.growth_factor, self.backoff_factor, self.growth_interval)


def resolve(loss_scale):
    """Trainer's `loss_scale` argument -> (static float or None, DynamicLossScale or None): None keeps the model's
    static scale (MF_LOSS_SCALE=dynamic selects the dynamic one), "dynamic" builds a DynamicLossScale with GradScaler's
    defaults, an instance is used as given, anything else is a static float"""
    import os
    if loss_scale is None and os.environ.get("MF_LOSS_SCALE", "").strip().lower() == "dynamic":
        loss_scale = "dynamic"
    if isinstance(loss_scale, DynamicLossScale):
        return None, loss_scale
    if isinstance(loss_scale, str) and loss_scale.strip().lower() == "dynamic":
        return None, DynamicLossScale()
    return (None if loss_scale is None else float(loss_scale)), None
