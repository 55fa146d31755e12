"""CPU: the reference's other SOLVER settings (solver/__init__.py:27-92, learning_schedules_fastai.py, engine/trainer.py:81-126)
against tests/golden/solver.npz (oracle/make_golden_solver.py, the unmodified reference solver package): the lr / momentum
sequences of build_scheduler under the Trainer's stepping rule, the one-cycle group membership of KeypointDetector, and the
guards of build_optimizer / Trainer."""
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import solver
from monoflex_b200.config import default_cfg
from monoflex_b200.train import Trainer
from oracle.make_golden_solver import SCHED, TRAJ, NEVER_GRADED, toy_net


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "solver.npz"))


def _cfg(**solver_keys):
    cfg = default_cfg(device="cpu")
    for k, v in solver_keys.items():
        setattr(cfg.SOLVER, k, v)
    return cfg


def _trainer_stepper(optimizer, cfg):
    """the schedule half of a Trainer (its own _schedule_step and the attributes __init__ derives), without a GPU model"""
    sched, warm = solver.build_scheduler(optimizer, cfg.SOLVER)
    t = types.SimpleNamespace(scheduler=sched, warmup_scheduler=warm, iteration=0,
                              _indexed_schedule=cfg.SOLVER.OPTIMIZER.find("onecycle") >= 0 or warm is not None,
                              warmup_iters=solver.solver_value(cfg.SOLVER, "WARMUP_STEPS") if cfg.SOLVER.LR_WARMUP else -1)

    def step():
        Trainer._schedule_step(t)
        t.iteration += 1
    return t, step


def test_onecycle_lr_and_momentum_sequences_equal_reference(gold):
    cfg = _cfg(OPTIMIZER="adam_onecycle", **{k: SCHED[k] for k in ("BASE_LR", "MAX_ITERATION", "MOMS", "PCT_START",
                                                                      "DIV_FACTOR")})
    opt = solver.build_optimizer(toy_net(), cfg)
    assert isinstance(opt, solver.FusedOneCycleAdam)
    t, step = _trainer_stepper(opt, cfg)
    assert t.warmup_scheduler is None and isinstance(t.scheduler, solver.OneCycle)
    lrs, moms = [opt.lr], [opt.mom]
    for _ in range(SCHED["MAX_ITERATION"]):
        step()
        lrs.append(opt.lr)
        moms.append(opt.mom)
        assert all(g["lr"] == opt.lr and g["betas"] == (opt.mom, 0.99) for g in opt.param_groups)
    assert np.array_equal(np.array(lrs, np.float64), gold["sched_onecycle_lr"])
    assert np.array_equal(np.array(moms, np.float64), gold["sched_onecycle_mom"])


def test_warmup_then_lambda_lr_sequence_equals_reference(gold):
    cfg = _cfg(OPTIMIZER="adam", LR_WARMUP=True, **{k: SCHED[k] for k in SCHED if k not in ("MOMS", "PCT_START")})
    opt = solver.build_optimizer(toy_net(), cfg)
    assert type(opt) is solver.FusedAdam
    t, step = _trainer_stepper(opt, cfg)
    assert isinstance(t.warmup_scheduler, solver.CosineWarmupLR)
    rows = [[g["lr"] for g in opt.param_groups]]
    for _ in range(SCHED["MAX_ITERATION"]):
        step()
        rows.append([g["lr"] for g in opt.param_groups])
    want = gold["sched_warmup_lr"]
    assert want[0, 0] == SCHED["BASE_LR"] / SCHED["DIV_FACTOR"]          # the warm-up constructor sets eta_min
    assert np.array_equal(np.array(rows, np.float64), want)


def test_adamw_warmup_uses_the_same_schedule(gold):
    """'adamw' + LR_WARMUP: FusedAdamW (unchanged) under the same CosineWarmupLR / LambdaLR stepping"""
    cfg = _cfg(OPTIMIZER="adamw", LR_WARMUP=True, **{k: SCHED[k] for k in SCHED if k not in ("MOMS", "PCT_START")})
    opt = solver.build_optimizer(toy_net(), cfg)
    assert type(opt) is solver.FusedAdamW
    _, step = _trainer_stepper(opt, cfg)
    rows = [[g["lr"] for g in opt.param_groups]]
    for _ in range(SCHED["MAX_ITERATION"]):
        step()
        rows.append([g["lr"] for g in opt.param_groups])
    assert np.array_equal(np.array(rows, np.float64), gold["sched_warmup_lr"])


def test_missing_solver_keys_take_reference_defaults():
    sc = types.SimpleNamespace(OPTIMIZER="adam_onecycle", BASE_LR=3e-3)
    opt = solver.FusedOneCycleAdam(toy_net(), 3e-3, 1e-5)
    sched, warm = solver.build_scheduler(opt, sc)
    assert warm is None and sched.total_step == 30000 and list(sched.moms) == [0.95, 0.85]
    assert sched.div_factor == 10 and sched.pct_start == 0.4 and opt.lr == 3e-3 / 10
    cfg = default_cfg(device="cpu")
    for k in ("MAX_ITERATION", "MOMS", "PCT_START", "DIV_FACTOR", "WARMUP_STEPS"):
        assert hasattr(cfg.SOLVER, k)


def test_onecycle_groups_of_keypoint_detector_equal_reference(gold):
    from monoflex_b200.model.detector import KeypointDetector
    model = KeypointDetector(default_cfg(device="cpu"))
    name_of = {id(p): n for n, p in model.named_parameters()}
    (non_bn, bn), outside = solver.onecycle_param_groups(model)
    assert [name_of[id(p)] for p in non_bn] == [str(n) for n in gold["onecycle_group0_names"]]
    assert [name_of[id(p)] for p in bn] == [str(n) for n in gold["onecycle_group1_names"]]
    nogroup = [name_of[id(p)] for p in outside]
    assert nogroup == [str(n) for n in gold["onecycle_nogroup_names"]]
    # the quirk: every DCN's own weight / bias (beside its conv_offset_mask child) is in no group
    dcn = [n for n, m in model.named_modules() if type(m).__name__ == "DCN"]
    assert dcn and sorted(nogroup) == sorted(d + s for d in dcn for s in (".weight", ".bias"))
    assert not any("conv_offset_mask" in n for n in nogroup)


def test_onecycle_optimizer_layout_on_cpu(gold):
    """the wrapper's two groups hold the grouped tensors; the arena also holds the no-group ones (their gradient is part of
    the clipping norm) with lr 0; mark_unused makes a grouped tensor decay-only (-1 in the table)"""
    net = toy_net()
    opt = solver.build_optimizer(net, _cfg(OPTIMIZER="adam_onecycle", BASE_LR=TRAJ["BASE_LR"],
                                           WEIGHT_DECAY=TRAJ["WEIGHT_DECAY"]))
    names = {id(p): n for n, p in net.named_parameters()}
    assert len(opt.param_groups) == 2
    assert [names[id(p)] for p in opt.param_groups[1]["params"]] == ["bn.weight", "bn.bias", "bn1.weight", "bn1.bias"]
    assert [names[id(p)] for p in opt.arena.tensors[opt.n_grouped:]] == ["dcn.weight", "dcn.bias"]
    assert opt.wd == TRAJ["WEIGHT_DECAY"] and opt.lr == TRAJ["BASE_LR"] and opt.mom == 0.9 and opt.beta == 0.99
    opt.mark_unused(set(NEVER_GRADED), net)
    table = opt._lr_table()
    a = opt.arena
    for i, p in enumerate(a.tensors):
        c0, c1 = a.offsets[i] // a.chunk, (a.offsets[i] + p.numel() - 1) // a.chunk + 1
        want = 0.0 if i >= opt.n_grouped else (-1.0 if names[id(p)] in NEVER_GRADED else 1.0)
        assert torch.all(table[c0:c1] == want), names[id(p)]
    assert opt._hyper.tolist() == [TRAJ["BASE_LR"], 0.9, TRAJ["WEIGHT_DECAY"], 0.0]
    sd = opt.state_dict()
    assert len(sd["param_groups"]) == 2 and len(sd["state"]) == opt.n_grouped


def test_adam_table_keeps_per_group_lrs():
    """'adam' with BIAS_LR_FACTOR 2: two lrs, so the table holds them and the multiplier is 1; unused tensors are 0"""
    net = toy_net()
    cfg = _cfg(OPTIMIZER="adam", BASE_LR=1e-3, WEIGHT_DECAY=1e-4)
    opt = solver.build_optimizer(net, cfg)
    opt.mark_unused(set(NEVER_GRADED), net)
    table = opt._lr_table()
    assert sorted(set(table.tolist())) == pytest.approx([0.0, 1e-3, 2e-3])
    assert opt._hyper.tolist() == [1.0, 0.9, 1e-4, 0.0]
    for g in opt.param_groups:
        g["lr"] = 5e-4                                            # one shared lr: the table becomes a mask
    table = opt._lr_table()
    assert sorted(set(table.tolist())) == [0.0, 1.0] and opt._hyper[0].item() == 5e-4
    sd = opt.state_dict()
    ref = torch.optim.Adam(solver.get_model_params(net, cfg))
    ref.load_state_dict(sd)                                       # torch.optim.Adam's layout
    assert ref.param_groups[0]["decoupled_weight_decay"] is False


def test_guards():
    net = toy_net()
    with pytest.raises(NotImplementedError, match="sgd"):
        solver.build_optimizer(net, _cfg(OPTIMIZER="sgd"))
    with pytest.raises(NotImplementedError, match="symmetric_group"):
        solver.build_optimizer(net, _cfg(OPTIMIZER="adam"), symmetric_group=object())
    fake = types.SimpleNamespace(parameters=lambda: iter([types.SimpleNamespace(is_cuda=True)]))
    with pytest.raises(NotImplementedError, match="sgd"):
        Trainer(fake, _cfg(OPTIMIZER="sgd"))
    with pytest.raises(ValueError, match="LR_WARMUP"):
        Trainer(fake, _cfg(OPTIMIZER="adam_onecycle", LR_WARMUP=True))
    for name in ("adam", "adam_onecycle"):
        with pytest.raises(NotImplementedError, match="symmetric_group"):
            Trainer(fake, _cfg(OPTIMIZER=name), symmetric_group=object())
