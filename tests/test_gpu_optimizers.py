"""-m gpu: the reference's 'adam' and 'adam_onecycle' optimisers and LR_WARMUP on the device (solver.FusedAdam,
solver.FusedOneCycleAdam, mf_optim_step_dyn) against torch.optim.Adam and against the reference's OptimWrapper + OneCycle
trajectory (tests/golden/solver.npz), eager and replayed from a CUDA graph, and the captured Trainer against the eager one."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import solver
from monoflex_b200.config import default_cfg
from oracle.make_golden_solver import TRAJ, NEVER_GRADED, toy_net

pytestmark = pytest.mark.gpu

SHAPES = [(1,), (511,), (512,), (513,), (16, 3, 7, 7), (27, 64, 3, 3), (27,), (256, 64, 3, 3), (3, 256, 1, 1), (3,)]
NAMES = ["w%d" % i if i % 2 == 0 else "b%d.bias" % i for i in range(len(SHAPES))]
UNUSED = {"w4", "b9.bias"}           # grad None for torch (its Adam skips them), zero in the arena, lr 0 in the chunk table


def _tensors(gen, scale=0.1):
    return [torch.from_numpy(gen.standard_normal(s).astype(np.float32) * scale) for s in SHAPES]


def _close(got, want, what):
    d = (got.detach().cpu() - want).abs().max().item()
    assert d <= 2e-7 + 1e-6 * want.abs().max().item(), (what, d)


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
@pytest.mark.parametrize("clip", [False, True])
def test_fused_adam_matches_torch_adam(clip, grad_scale):
    """FusedAdam == torch.optim.Adam(get_model_params, betas=(0.9, 0.99), weight_decay) (solver/__init__.py:33-34): ragged
    sizes, BIAS_LR_FACTOR 2, an lr decay after step 3, coupled L2 decay large enough to matter (0.05), tensors with grad None
    untouched; clip: clip_grad_norm_ to half the norm first; grad_scale 0.5: the arena holds a two-rank SUM, torch the mean"""
    gen = np.random.Generator(np.random.PCG64(31))
    init = _tensors(gen)
    lrs = [1e-3 * (2.0 if "bias" in n else 1.0) for n in NAMES]
    ref_p = [torch.nn.Parameter(t.clone()) for t in init]
    ref = torch.optim.Adam([{"params": [p], "lr": lr} for p, lr in zip(ref_p, lrs)], lr=1e-3, weight_decay=0.05,
                           betas=(0.9, 0.99))
    our_p = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    ours = solver.FusedAdam([{"params": [p], "lr": lr} for p, lr in zip(our_p, lrs)], lr=1e-3, weight_decay=0.05,
                            betas=(0.9, 0.99))
    holder = torch.nn.Module()
    for n, p in zip(NAMES, our_p):
        holder.register_parameter(n.replace(".", "_"), p)
    ours.mark_unused({n.replace(".", "_") for n in UNUSED}, holder)
    for it in range(5):
        grads = _tensors(gen, 0.1 / grad_scale)
        for n, p, q, g in zip(NAMES, ref_p, our_p, grads):
            q.grad.copy_(torch.zeros_like(g) if n in UNUSED else g)
            p.grad = None if n in UNUSED else g * grad_scale
        if it == 3:
            for opt in (ref, ours):
                for g in opt.param_groups:
                    g["lr"] *= 0.1
        c = None
        if clip:
            c = 0.5 * float(ours.arena.grads.double().norm()) * grad_scale
            want_norm = float(torch.nn.utils.clip_grad_norm_(ref_p, c))
        ref.step()
        ours.step(grad_scale=grad_scale, max_grad_norm=c)
        if clip:
            assert abs(float(ours.last_grad_norm) - want_norm) <= 1e-6 * want_norm
        for n, p, q in zip(NAMES, ref_p, our_p):
            _close(q, p.detach(), (it, n))
    for n, p, q, t in zip(NAMES, ref_p, our_p, init):
        if n in UNUSED:
            assert torch.equal(q.detach().cpu(), t) and p not in ref.state
            continue
        st = ref.state[p]
        assert torch.allclose(ours.state[q]["exp_avg"].cpu(), st["exp_avg"], rtol=1e-5, atol=1e-8)
        assert torch.allclose(ours.state[q]["exp_avg_sq"].cpu(), st["exp_avg_sq"], rtol=1e-5, atol=1e-10)
        assert float(ours.state[q]["step"]) == float(st["step"]) == 5.0
    assert ours.skipped_steps() == 0


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(GOLDEN, "solver.npz"))


def _traj_net(gold):
    net = toy_net()
    with torch.no_grad():
        for n, p in net.named_parameters():
            p.copy_(torch.from_numpy(gold["traj_init/" + n]))
    return net.cuda()


def _run_trajectory(gold, prefix, opt, sched, net, captured):
    """the reference's trajectory: set p.grad, optimizer.step(), scheduler.step(t); from step 1 on, captured replays one
    CUDA graph of step() after refreshing the lr table / hyper-parameter block (what the captured Trainer does)"""
    inner = getattr(opt, "opt", opt)
    params = dict(net.named_parameters())
    graph = None
    for t in range(TRAJ["STEPS"]):
        for n, p in params.items():
            p.grad.copy_(torch.zeros_like(p) if n in NEVER_GRADED else torch.from_numpy(gold["traj_grad%d/%s" % (t, n)]).cuda())
        want_hyper = [g["lr"] for g in inner.param_groups] + [g["betas"][0] for g in inner.param_groups]
        if captured and t >= 1:
            if graph is None:
                inner._lr_table()
                graph = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                with torch.cuda.graph(graph):
                    opt.step()
                inner.step_count -= 1
                inner._step_t -= 1
            inner._lr_table()
            graph.replay()
            inner.step_count += 1
            inner._step_t += 1
        else:
            opt.step()
        sched.step(t)
        assert [g["lr"] for g in inner.param_groups] + [g["betas"][0] for g in inner.param_groups] == \
            gold["%s_hyper" % prefix][t].tolist()
        yield t, params, want_hyper


@pytest.mark.parametrize("captured", [False, True])
def test_fused_onecycle_follows_reference_trajectory(gold, captured):
    """FusedOneCycleAdam + OneCycle against the unmodified OptimWrapper + OneCycle (oracle/make_golden_solver.py): the
    momentum phase change at step 4 falls inside the replays; the never-graded grouped tensor is only decayed, the tensors
    of the non-leaf module (DCN-like) are bit-unchanged though they have gradients"""
    net = _traj_net(gold)
    cfg = default_cfg()
    for k in ("BASE_LR", "WEIGHT_DECAY", "MAX_ITERATION", "PCT_START", "MOMS", "DIV_FACTOR"):
        setattr(cfg.SOLVER, k, TRAJ[k])
    cfg.SOLVER.OPTIMIZER = "adam_onecycle"
    opt = solver.build_optimizer(net, cfg)
    sched, warm = solver.build_scheduler(opt, cfg.SOLVER)
    assert warm is None
    opt.mark_unused(set(NEVER_GRADED), net)
    for t, params, used in _run_trajectory(gold, "oc", opt, sched, net, captured):
        hyper = opt._hyper.tolist()
        assert hyper[:3] == [used[0], used[2], TRAJ["WEIGHT_DECAY"]], (t, hyper, used)     # what the step read
        for n, p in params.items():
            if n.startswith("dcn.") and "offset" not in n:
                assert torch.equal(p.detach().cpu(), torch.from_numpy(gold["traj_init/" + n])), (t, n)
                continue
            _close(p, torch.from_numpy(gold["oc_p%d/%s" % (t, n)]), (t, n))
            st = opt.opt.state[p]
            if n in NEVER_GRADED:
                assert "oc_m%d/%s" % (t, n) not in gold.files
                assert float(st["exp_avg"].abs().max()) == 0.0 and float(st["exp_avg_sq"].abs().max()) == 0.0
                continue
            assert torch.allclose(st["exp_avg"].cpu(), torch.from_numpy(gold["oc_m%d/%s" % (t, n)]), rtol=1e-5, atol=1e-8)
            assert torch.allclose(st["exp_avg_sq"].cpu(), torch.from_numpy(gold["oc_v%d/%s" % (t, n)]), rtol=1e-5, atol=1e-10)
            assert float(st["step"]) == float(gold["oc_step%d/%s" % (t, n)]) == t + 1
    head = params[NEVER_GRADED[0]].detach().cpu()
    assert not torch.equal(head, torch.from_numpy(gold["traj_init/" + NEVER_GRADED[0]]))      # decayed
    assert opt.skipped_steps() == 0 and opt.step_count == TRAJ["STEPS"]


@pytest.mark.parametrize("captured", [False, True])
def test_fused_adam_follows_reference_trajectory(gold, captured):
    """FusedAdam + LambdaLR (decay after step 3, inside the replays) against torch.optim.Adam with the reference's groups"""
    net = _traj_net(gold)
    cfg = default_cfg()
    cfg.SOLVER.OPTIMIZER, cfg.SOLVER.STEPS = "adam", (TRAJ["DECAY_AT"],)
    for k in ("BASE_LR", "WEIGHT_DECAY", "BIAS_LR_FACTOR", "LR_DECAY"):
        setattr(cfg.SOLVER, k, TRAJ[k])
    opt = solver.build_optimizer(net, cfg)
    sched, _ = solver.build_scheduler(opt, cfg.SOLVER)
    opt.mark_unused(set(NEVER_GRADED), net)
    for t, params, _ in _run_trajectory(gold, "adam", opt, sched, net, captured):
        for n, p in params.items():
            if n in NEVER_GRADED:
                assert torch.equal(p.detach().cpu(), torch.from_numpy(gold["traj_init/" + n]))
                continue
            _close(p, torch.from_numpy(gold["adam_p%d/%s" % (t, n)]), (t, n))
            st = opt.state[p]
            assert torch.allclose(st["exp_avg"].cpu(), torch.from_numpy(gold["adam_m%d/%s" % (t, n)]), rtol=1e-5, atol=1e-8)
            assert torch.allclose(st["exp_avg_sq"].cpu(), torch.from_numpy(gold["adam_v%d/%s" % (t, n)]), rtol=1e-5,
                                  atol=1e-10)


def _two_steps(opt, net, gen):
    for _ in range(2):
        for p in net.parameters():
            p.grad.copy_(torch.from_numpy(gen.standard_normal(tuple(p.shape)).astype(np.float32) * 0.1).cuda())
        opt.step()


def _state_equal(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    assert len(sa["state"]) == len(sb["state"]) and len(sa["param_groups"]) == len(sb["param_groups"])
    for i, st in sa["state"].items():
        for k in ("exp_avg", "exp_avg_sq"):
            assert torch.equal(st[k].cpu(), sb["state"][i][k].cpu()), (i, k)
        assert float(st["step"]) == float(sb["state"][i]["step"])
    for ga, gb in zip(sa["param_groups"], sb["param_groups"]):
        assert ga["lr"] == gb["lr"] and tuple(ga["betas"]) == tuple(gb["betas"]) and ga["params"] == gb["params"]


def test_state_dict_round_trips(gold):
    """FusedAdam <-> torch.optim.Adam(get_model_params); FusedOneCycleAdam <-> the reference's inner Adam layout (two groups:
    non-BN leaves, BN leaves); after the round trip the next step of the reloaded optimiser equals the original's"""
    gen = np.random.Generator(np.random.PCG64(5))
    cfg = default_cfg()
    cfg.SOLVER.OPTIMIZER = "adam"
    net = _traj_net(gold)
    ours = solver.build_optimizer(net, cfg)
    _two_steps(ours, net, gen)
    ref = torch.optim.Adam(solver.get_model_params(net, cfg), betas=(0.9, 0.99))
    ref.load_state_dict(ours.state_dict())
    net2 = _traj_net(gold)
    back = solver.build_optimizer(net2, cfg)
    back.load_state_dict(ref.state_dict())
    _state_equal(ours, back)
    assert back.step_count == 2
    with torch.no_grad():
        for p, q in zip(net.parameters(), net2.parameters()):
            q.copy_(p)
    g = np.random.Generator(np.random.PCG64(6))
    _two_steps(ours, net, g)
    _two_steps(back, net2, np.random.Generator(np.random.PCG64(6)))
    for p, q in zip(net.parameters(), net2.parameters()):
        assert torch.equal(p, q)

    cfg.SOLVER.OPTIMIZER = "adam_onecycle"
    net = _traj_net(gold)
    ours = solver.build_optimizer(net, cfg)
    ours.lr, ours.mom = 2e-3, 0.91
    _two_steps(ours, net, gen)
    (non_bn, bn), _ = solver.onecycle_param_groups(net)
    ref = torch.optim.Adam([{"params": non_bn, "lr": 0}, {"params": bn, "lr": 0}], betas=(0.9, 0.99))
    ref.load_state_dict(ours.state_dict())
    assert ref.param_groups[0]["betas"] == (0.91, 0.99) and ref.param_groups[1]["lr"] == 2e-3
    back = solver.build_optimizer(_traj_net(gold), cfg)
    back.load_state_dict(ref.state_dict())
    _state_equal(ours, back)
    assert (back.lr, back.mom, back.beta) == (2e-3, 0.91, 0.99) and back.step_count == 2


# ------------------------------------------------------------------ captured Trainer against the eager Trainer
CASES = {
    # optimiser, extra SOLVER keys, steps: 'adam' decays its lr inside the replays (LambdaLR, unindexed), the one-cycle lr /
    # momentum phases change at step 4 and the warm-up ends at step 3, both inside the replays (graph_warmup 2)
    "adam": ("adam", dict(STEPS=(3,)), 5),
    "adam_onecycle": ("adam_onecycle", dict(MAX_ITERATION=10, PCT_START=0.4), 6),
    "adamw_warmup": ("adamw", dict(LR_WARMUP=True, WARMUP_STEPS=3), 5),
}


def _train_models(n):
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    models = []
    for _ in range(n):
        model = KeypointDetector(default_cfg()).cuda()
        model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        models.append(model)
    return models, images, targets


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm()))


def _lr_state(opt):
    """host lrs and momenta of every group; the lr of every grouped tensor as the update kernel forms it from the device
    table and hyper-parameter block (float32 table entry x float32 multiplier), and the device beta1"""
    inner = getattr(opt, "opt", opt)
    lrs, moms = [g["lr"] for g in inner.param_groups], [g["betas"][0] for g in inner.param_groups]
    if inner._chunk_lr is None:
        return lrs, moms, None, None
    a, table = inner.arena, inner._chunk_lr.cpu().numpy()
    mult, beta1 = inner._hyper.cpu().tolist()[:2] if hasattr(inner, "_hyper") else (1.0, None)
    eff = [abs(float(table[o // a.chunk] * np.float32(mult))) for o in a.offsets[:inner.n_grouped]]
    return lrs, moms, eff, beta1


def _expected_device_lrs(opt, lrs):
    inner = getattr(opt, "opt", opt)
    decays = getattr(inner, "_unused_decays", False)
    per_tensor = [lr for g, lr in zip(inner.param_groups, lrs) for _ in g["params"]]
    return [0.0 if (skip and not decays) else float(np.float32(lr)) for lr, skip in zip(per_tensor, inner._skip)]


@pytest.mark.parametrize("clip", [False, True])
@pytest.mark.parametrize("case", sorted(CASES))
def test_captured_trainer_matches_eager(case, clip):
    """Trainer(use_cuda_graph=True) against an eager Trainer on a twin model, per step: the same lrs / momenta on the host
    and in the device table / hyper block the step read, the same logged losses (the captured-step test's tolerances: the
    DCN backward's scatter atomics make runs drift on this synthetic network), parameter and moment updates pointing the
    same way, the same step count. clip: GRAD_NORM_CLIP below the gradient norm, so every replay clips."""
    from monoflex_b200.train import Trainer
    name, extra, steps = CASES[case]
    cfg = default_cfg()
    cfg.SOLVER.OPTIMIZER = name
    for k, v in extra.items():
        setattr(cfg.SOLVER, k, v)
    if clip:
        cfg.SOLVER.GRAD_NORM_CLIP = 1e-3
    (ma, mb), images, targets = _train_models(2)
    ta = Trainer(ma, cfg, loss_scale=128.0)
    tb = Trainer(mb, cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    oa, ob = ta._arena_opt, tb._arena_opt
    assert type(oa) is type(ob) and type(oa) is {"adam": solver.FusedAdam, "adamw": solver.FusedAdamW,
                                                 "adam_onecycle": solver._OneCycleInnerAdam}[name]
    p0 = oa.arena.params.clone()
    assert torch.equal(p0, ob.arena.params)
    cos = None
    for i in range(steps):
        before = _lr_state(ta.optimizer)[:2]
        assert before == _lr_state(tb.optimizer)[:2], i
        la = ta.step(images, targets)[1]
        lb = tb.step(images, targets)[1]
        assert (tb._graph is not None) == (i >= 2)
        ha, hb = _lr_state(ta.optimizer), _lr_state(tb.optimizer)
        assert ha == hb, i                  # the schedules moved the same way; both steps read the same table / block ...
        assert hb[2] == _expected_device_lrs(tb.optimizer, before[0]), i     # ... holding the lrs of the step just taken
        assert hb[3] in (None, before[1][0]), (i, hb[3], before[1])         # ... and its beta1
        if clip:
            assert float(ob.last_grad_norm) > cfg.SOLVER.GRAD_NORM_CLIP or i < 2, (i, float(ob.last_grad_norm))
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
        if i == 2:
            # the first replay, before the twins drift apart (after 5-6 steps the moments of two EAGER runs of this
            # synthetic network agree no better than cos ~0.5): the update and the moments point the same way
            da, db = oa.arena.params - p0, ob.arena.params - p0
            cos = (_cos(da, db), _cos(oa.exp_avg, ob.exp_avg), _cos(oa.exp_avg_sq, ob.exp_avg_sq))
            assert float(da.norm()) > 0 and min(cos) > 0.5, cos
    print(case, clip, "first-replay cos (update, exp_avg, exp_avg_sq)", cos)
    assert oa.skipped_steps() == ob.skipped_steps() == 0
    assert oa.step_count == ob.step_count == steps and int(ob._state4[0]) == steps
    assert float(oa._step_t) == float(ob._step_t) == steps
