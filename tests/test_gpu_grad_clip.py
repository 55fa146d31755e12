"""-m gpu: gradient-norm clipping on the device (FusedAdamW.step(max_grad_norm=...), mf_optim_step_dyn) against
torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW, and the captured Trainer with the reference's SOLVER.GRAD_NORM_CLIP."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from monoflex_b200 import solver
from monoflex_b200.config import default_cfg

pytestmark = pytest.mark.gpu

SHAPES = [(1,), (511,), (512,), (513,), (16, 3, 7, 7), (27, 64, 3, 3), (27,), (256, 64, 3, 3), (3, 256, 1, 1), (3,)]
UNUSED = {"p1", "p6"}              # outside the forward graph: grad None for torch, zero in the arena, lr 0 in the chunk table


def _tensors(gen, shapes, scale=0.1):
    return [torch.from_numpy(gen.standard_normal(s).astype(np.float32) * scale) for s in shapes]


def _fused(init, lrs, names):
    ps = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    opt = solver.FusedAdamW([{"params": [p], "lr": lr} for p, lr in zip(ps, lrs)], lr=3e-4, weight_decay=1e-5,
                            betas=(0.9, 0.99))
    holder = torch.nn.Module()
    for n, p in zip(names, ps):
        holder.register_parameter(n, p)
    opt.mark_unused(UNUSED, holder)
    return ps, opt


def _setup(seed):
    gen = np.random.Generator(np.random.PCG64(seed))
    names = ["p%d" % i for i in range(len(SHAPES))]
    lrs = [3e-4 * (2.0 if i % 2 else 1.0) for i in range(len(SHAPES))]
    return gen, names, lrs, _tensors(gen, SHAPES)


def _set_grads(ps, names, grads):
    for n, q, g in zip(names, ps, grads):
        q.grad.copy_(torch.zeros_like(g) if n in UNUSED else g)


def _ulp32(x):
    return float(np.spacing(np.float32(x)))


@pytest.mark.parametrize("grad_scale", [1.0, 0.5])
def test_clip_matches_torch_clip_grad_norm_and_adamw(grad_scale):
    """three clipped steps with an lr change in between: the norm, the clipped gradients, the parameters and the moments
    follow clip_grad_norm_ + torch.optim.AdamW on copies. grad_scale 0.5: the arena holds a two-rank SUM, torch the mean."""
    gen, names, lrs, init = _setup(21)
    ref_p = [torch.nn.Parameter(t.clone()) for t in init]
    ref = torch.optim.AdamW([{"params": [p], "lr": lr} for p, lr in zip(ref_p, lrs)], lr=3e-4, weight_decay=1e-5,
                            betas=(0.9, 0.99))
    our_p, ours = _fused(init, lrs, names)
    a = ours.arena
    used = torch.zeros(a.numel, dtype=torch.bool)
    for o, p in zip(a.offsets, a.tensors):
        used[o:o + p.numel()] = True
    for it in range(3):
        grads = _tensors(gen, SHAPES, 0.1 / grad_scale)                   # what the arena holds
        _set_grads(our_p, names, grads)
        for n, p, g in zip(names, ref_p, grads):
            p.grad = None if n in UNUSED else g * grad_scale              # what torch sees (x 0.5 is exact)
        g64 = a.grads.double()
        norm64 = float(g64.norm()) * grad_scale
        c = 0.5 * norm64
        if it == 2:
            for opt in (ref, ours):
                for g in opt.param_groups:
                    g["lr"] *= 0.1
        want_norm = float(torch.nn.utils.clip_grad_norm_(ref_p, c))
        ref.step()
        ours.step(grad_scale=grad_scale, max_grad_norm=c)
        got_norm = float(ours.last_grad_norm)
        assert abs(got_norm - want_norm) <= 1e-6 * want_norm, (it, got_norm, want_norm)
        assert abs(got_norm - norm64) <= _ulp32(norm64), (it, got_norm, norm64)
        for n, p, q in zip(names, ref_p, our_p):
            if n in UNUSED:
                assert float(q.grad.abs().max()) == 0.0
                continue
            want_g = p.grad / grad_scale
            dg = (q.grad.cpu() - want_g).abs().max().item()
            assert dg <= 1e-6 * want_g.abs().max().item(), (it, n, dg)
            d = (q.detach().cpu() - p.detach()).abs().max().item()
            assert d <= 2e-7 + 1e-6 * p.detach().abs().max().item(), (it, n, d)
        assert abs(float(a.grads.double().norm()) * grad_scale - c) <= 1e-5 * c
    for n, p, q, t in zip(names, ref_p, our_p, init):
        if n in UNUSED:                                                    # torch's AdamW skips grad None: so does the kernel
            assert torch.equal(q.detach().cpu(), t) and p not in ref.state
            continue
        st = ref.state[p]
        assert torch.allclose(ours.state[q]["exp_avg"].cpu(), st["exp_avg"], rtol=1e-5, atol=1e-8)
        assert torch.allclose(ours.state[q]["exp_avg_sq"].cpu(), st["exp_avg_sq"], rtol=1e-5, atol=1e-10)
    assert a.params.cpu()[~used].abs().sum() == 0 and a.grads.cpu()[~used].abs().sum() == 0
    assert ours.skipped_steps() == 0


def test_clip_not_triggered_is_a_plain_step():
    """max_grad_norm above the norm: the gradient arena is not written, parameters and moments are bit-identical to step()"""
    gen, names, lrs, init = _setup(22)
    pa, oa = _fused(init, lrs, names)
    pb, ob = _fused(init, lrs, names)
    for _ in range(2):
        grads = _tensors(gen, SHAPES)
        _set_grads(pa, names, grads)
        _set_grads(pb, names, grads)
        g0 = oa.arena.grads.clone()
        c = 2.0 * float(g0.double().norm())
        oa.step(max_grad_norm=c)
        ob.step()
        assert torch.equal(oa.arena.grads, g0)
        assert float(oa.last_grad_norm) < c
        assert torch.equal(oa.arena.params, ob.arena.params)
        assert torch.equal(oa.exp_avg, ob.exp_avg) and torch.equal(oa.exp_avg_sq, ob.exp_avg_sq)


@pytest.mark.parametrize("bad", [float("inf"), float("nan")])
def test_nonfinite_gradient_with_clipping_skips_the_step(bad):
    gen, names, lrs, init = _setup(23)
    ps, opt = _fused(init, lrs, names)
    _set_grads(ps, names, _tensors(gen, SHAPES))
    opt.step(max_grad_norm=0.1)
    torch.cuda.synchronize()
    p0, m0, v0 = opt.arena.params.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone()
    _set_grads(ps, names, _tensors(gen, SHAPES))
    ps[4].grad.view(-1)[17] = bad
    g0 = opt.arena.grads.clone()
    opt.step(max_grad_norm=0.1)
    assert opt.skipped_steps() == 1
    assert not np.isfinite(float(opt.last_grad_norm))
    assert torch.equal(opt.arena.params, p0) and torch.equal(opt.exp_avg, m0) and torch.equal(opt.exp_avg_sq, v0)
    assert torch.equal(opt.arena.grads.nan_to_num(), g0.nan_to_num())
    _set_grads(ps, names, _tensors(gen, SHAPES))                           # the next finite step updates again
    opt.step(max_grad_norm=0.1)
    assert opt.skipped_steps() == 1 and not torch.equal(opt.arena.params, p0)
    assert int(opt._state4[0]) == 2


def test_clip_is_deterministic_at_arena_scale():
    """the same step on the same arena twice (6.2 M elements: more CTAs' worth than the scan grid, so every CTA strides):
    bit-identical norm, clipped gradients and parameters"""
    gen = np.random.Generator(np.random.PCG64(24))
    shapes = [(5_000_000,), (1_234_567,), (77,)]
    init = [torch.from_numpy(gen.standard_normal(s).astype(np.float32) * 0.05) for s in shapes]
    grads = [torch.from_numpy(gen.standard_normal(s).astype(np.float32) * 1e-3) for s in shapes]
    runs = []
    for _ in range(2):
        ps = [torch.nn.Parameter(t.clone().cuda()) for t in init]
        opt = solver.FusedAdamW(ps, lr=3e-4, weight_decay=1e-5, betas=(0.9, 0.99))
        for p, g in zip(ps, grads):
            p.grad.copy_(g.cuda())
        norm64 = float(opt.arena.grads.double().norm())
        opt.step(max_grad_norm=0.25 * norm64)
        runs.append((opt.last_grad_norm.clone(), opt.arena.grads.clone(), opt.arena.params.clone()))
        assert abs(float(opt.last_grad_norm) - norm64) <= _ulp32(norm64)
    for x, y in zip(*runs):
        assert torch.equal(x, y)


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


def test_captured_trainer_clips_grad_norm():
    """Trainer(use_cuda_graph=True) with SOLVER.GRAD_NORM_CLIP = half the smallest gradient norm of four unclipped eager steps
    (on this synthetic network the norm falls about 5x between the first and the third step, so half the first step's norm
    would not clip the replays): the replays clip on the device (the norm is above the clip, the arena's norm after the step
    is the clip) and the per-step losses follow an eager Trainer, which clips with torch's clip_grad_norm_, under the
    captured-step test's tolerances"""
    from monoflex_b200.train import Trainer
    (m0, ma, mb), images, targets = _train_models(3)
    t0 = Trainer(m0, default_cfg(), loss_scale=128.0)
    norms = []
    for _ in range(4):
        t0.step(images, targets)
        norms.append(float(t0.optimizer.arena.grads.double().norm()))
    c = 0.5 * min(norms)
    del t0, m0
    cfg = default_cfg()
    cfg.SOLVER.GRAD_NORM_CLIP = c
    ta = Trainer(ma, cfg, loss_scale=128.0)
    tb = Trainer(mb, cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    for i in range(4):
        la = ta.step(images, targets)[1]
        lb = tb.step(images, targets)[1]
        if i >= 2:
            assert tb._graph is not None
            norm = float(tb.optimizer.last_grad_norm)
            assert norm > c, (i, norm, c)
            got = float(tb.optimizer.arena.grads.double().norm())
            assert abs(got - c * norm / (norm + 1e-6)) <= 1e-5 * c, (i, got, c)
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
    assert tb.optimizer.skipped_steps() == 0 and tb.optimizer.step_count == ta.optimizer.step_count == 4


def test_captured_trainer_clip_refused_with_symmetric_group():
    from monoflex_b200.train import Trainer
    cfg = default_cfg()
    cfg.SOLVER.GRAD_NORM_CLIP = 10.0
    with pytest.raises(NotImplementedError, match="symmetric_group"):       # refused before any rendezvous
        Trainer(torch.nn.Linear(2, 2).cuda(), cfg, symmetric_group=object(), use_cuda_graph=True)


def test_captured_trainer_clips_rank_mean_two_ranks():
    """world >= 2 only (skipped on a 1-GPU box): after the NCCL all-reduce the captured step clips the rank-mean gradient
    to GRAD_NORM_CLIP on every rank, and the replicas stay identical (tools/grad_clip_two_rank_check.py)"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(root, "tools", "grad_clip_two_rank_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert '"ok": true' in r.stdout
