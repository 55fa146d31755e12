"""TEST INFRASTRUCTURE. Records tests/golden/solver.npz from the UNMODIFIED reference solver package (solver/__init__.py,
fastai_optim.py, learning_schedules_fastai.py), run on the CPU through oracle/ref_shims.py:

  * sched_onecycle_{lr,mom}: OptimWrapper.lr / .mom after the OneCycle constructor (index 0) and after every
    `scheduler.step(i)`, i = 0 .. MAX_ITERATION - 1, as engine/trainer.py:103-126 steps it;
  * sched_warmup_lr: every group's lr after LambdaLR + CosineWarmupLR are built (row 0) and after each do_train step
    (`warmup.step(i)` while i < WARMUP_STEPS, else `scheduler.step(i)`), over the reference's 'adam' groups of toy_net();
  * onecycle_group{0,1}_names / onecycle_nogroup_names: the one-cycle group membership, by parameter name, of the
    reference's KeypointDetector (runs/monoflex.yaml);
  * oc_* / adam_*: seeded trajectories of OptimWrapper + OneCycle ('adam_onecycle') and of torch.optim.Adam with the
    reference's groups ('adam') over toy_net(), from the same initial parameters and gradients (traj_init/*, traj_grad*;
    NEVER_GRADED keeps grad None): parameters / exp_avg / exp_avg_sq / step after every step, and every group's lr and beta1
    after every step's scheduler.step (*_hyper).

    python oracle/make_golden_solver.py        (needs the reference tree; writes tests/golden/solver.npz)
"""
import collections
import collections.abc
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT = os.path.join(ROOT, "tests", "golden", "solver.npz")

# schedule and trajectory settings, read by tests/test_solver_schedules_host.py and tests/test_gpu_optimizers.py
SCHED = dict(BASE_LR=3e-4, MAX_ITERATION=300, MOMS=[0.95, 0.85], PCT_START=0.4, DIV_FACTOR=10, WARMUP_STEPS=50,
             STEPS=(120, 200), LR_DECAY=0.1, LR_CLIP=1e-7, BIAS_LR_FACTOR=2.0)
TRAJ = dict(BASE_LR=3e-3, WEIGHT_DECAY=0.05, MAX_ITERATION=10, PCT_START=0.4, MOMS=[0.95, 0.85], DIV_FACTOR=10, STEPS=6,
            BIAS_LR_FACTOR=2.0, LR_DECAY=0.1, DECAY_AT=3)
NEVER_GRADED = ("head.weight",)              # in a one-cycle group, but autograd leaves its grad None


class _Owner(nn.Module):
    """owns parameters AND has a child, like the reference's DCN (weight / bias beside conv_offset_mask): flatten_model
    skips it, so its own parameters are in no one-cycle group"""

    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(8, 3, 3, 3))
        self.bias = nn.Parameter(torch.empty(8))
        self.offset = nn.Linear(2, 2)


def toy_net():
    """ragged tensor sizes (1, 511, 216, 600, ...) on both sides of the 512-element arena chunk"""
    net = nn.Module()
    net.stem = nn.Conv2d(3, 8, 3)                     # 216 + 8
    net.bn = nn.BatchNorm2d(8)
    net.dcn = _Owner()
    net.mid = nn.Linear(20, 30)                       # 600 + 30
    net.bn1 = nn.BatchNorm1d(30)
    net.one = nn.Linear(511, 1, bias=False)           # 511
    net.tiny = nn.Linear(1, 1)                        # 1 + 1
    net.head = nn.Linear(30, 3)                       # never graded
    return net


def _ref_cfg(**solver):
    import ref_shims
    cfg = ref_shims.reference_cfg()
    for k, v in solver.items():
        setattr(cfg.SOLVER, k, v)
    return cfg


def _schedules(out):
    import solver as ref_solver
    cfg = _ref_cfg(OPTIMIZER="adam_onecycle", **{k: SCHED[k] for k in ("BASE_LR", "MAX_ITERATION", "MOMS", "PCT_START",
                                                                          "DIV_FACTOR")})
    opt = ref_solver.build_optimizer(toy_net(), cfg)
    sched, warm = ref_solver.build_scheduler(opt, None, cfg.SOLVER)
    assert warm is None
    lrs, moms = [opt.lr], [opt.mom]
    for i in range(SCHED["MAX_ITERATION"]):
        sched.step(i)
        lrs.append(opt.lr)
        moms.append(opt.mom)
    out["sched_onecycle_lr"], out["sched_onecycle_mom"] = np.array(lrs, np.float64), np.array(moms, np.float64)

    cfg = _ref_cfg(OPTIMIZER="adam", LR_WARMUP=True, **{k: SCHED[k] for k in SCHED if k not in ("MOMS", "PCT_START")})
    opt = ref_solver.build_optimizer(toy_net(), cfg)
    sched, warm = ref_solver.build_scheduler(opt, None, cfg.SOLVER)
    rows = [[g["lr"] for g in opt.param_groups]]
    for i in range(SCHED["MAX_ITERATION"]):
        if i < SCHED["WARMUP_STEPS"]:
            warm.step(i)
        else:
            sched.step(i)
        rows.append([g["lr"] for g in opt.param_groups])
    out["sched_warmup_lr"] = np.array(rows, np.float64)


def _membership(out):
    import ref_shims
    import solver as ref_solver
    cfg = _ref_cfg(OPTIMIZER="adam_onecycle")
    model = ref_shims.build_reference_model(cfg)
    opt = ref_solver.build_optimizer(model, cfg)
    name_of = {id(p): n for n, p in model.named_parameters()}
    grouped = set()
    for gi, g in enumerate(opt.param_groups):
        names = [name_of[id(p)] for p in g["params"]]
        grouped.update(names)
        out["onecycle_group%d_names" % gi] = np.array(names)
    out["onecycle_nogroup_names"] = np.array([n for n, p in model.named_parameters() if p.requires_grad and n not in grouped])


def _trajectory(out, prefix, optimizer_name):
    import solver as ref_solver
    gen = np.random.Generator(np.random.PCG64(7))
    net = toy_net()
    names = [n for n, _ in net.named_parameters()]
    with torch.no_grad():
        for n, p in net.named_parameters():
            p.copy_(torch.from_numpy(gen.standard_normal(tuple(p.shape)).astype(np.float32) * 0.1))
            out["traj_init/%s" % n] = p.detach().numpy().copy()
    cfg = _ref_cfg(OPTIMIZER=optimizer_name, LR_WARMUP=False, GRAD_NORM_CLIP=-1,
                   STEPS=(TRAJ["DECAY_AT"],), **{k: TRAJ[k] for k in ("BASE_LR", "WEIGHT_DECAY", "MAX_ITERATION", "PCT_START",
                                                                      "MOMS", "DIV_FACTOR", "BIAS_LR_FACTOR", "LR_DECAY")})
    opt = ref_solver.build_optimizer(net, cfg)
    sched, _ = ref_solver.build_scheduler(opt, None, cfg.SOLVER)
    inner = getattr(opt, "opt", None) or opt                 # OptimWrapper's torch.optim.Adam, or the Adam itself
    params = dict(net.named_parameters())
    lrs = []
    for t in range(TRAJ["STEPS"]):
        for n, p in params.items():
            if n in NEVER_GRADED:
                p.grad = None
                continue
            g = torch.from_numpy(gen.standard_normal(tuple(p.shape)).astype(np.float32) * 0.1)
            p.grad = g
            out["traj_grad%d/%s" % (t, n)] = g.numpy().copy()     # the same draws for both trajectories
        opt.step()                                           # engine/trainer.py:121, 123-126 (no warm-up)
        sched.step(t)
        lrs.append([g["lr"] for g in inner.param_groups] + [g["betas"][0] for g in inner.param_groups])
        for n, p in params.items():
            out["%s_p%d/%s" % (prefix, t, n)] = p.detach().numpy().copy()
            st = inner.state.get(p, {})
            if st:
                out["%s_m%d/%s" % (prefix, t, n)] = st["exp_avg"].numpy().copy()
                out["%s_v%d/%s" % (prefix, t, n)] = st["exp_avg_sq"].numpy().copy()
                out["%s_step%d/%s" % (prefix, t, n)] = np.array(float(st["step"]))
    out["traj_names"] = np.array(names)
    out["%s_hyper" % prefix] = np.array(lrs, np.float64)     # per step: every group's lr, then every group's beta1


def main():
    sys.path.insert(0, HERE)
    import ref_shims
    ref_shims.install()
    collections.Iterable = collections.abc.Iterable          # fastai_optim.py:3 (removed from collections in Python 3.10)
    out = {}
    _schedules(out)
    _membership(out)
    _trajectory(out, "oc", "adam_onecycle")
    _trajectory(out, "adam", "adam")
    np.savez_compressed(OUT, **out)
    print("wrote %s (%d arrays)" % (OUT, len(out)))


if __name__ == "__main__":
    main()
