"""-m gpu: the dynamic loss scale of the fp16 training backward (monoflex_b200/loss_scale.py): GradScaler's update rule on
the device, eager and inside a captured graph; the one-launch unscale-and-accumulate kernel against torch._foreach_add_;
that every fp16 overflow of the gradient flow reaches the finite guard; eager and captured trainers; a constant dynamic
scale against the static one; what a larger scale does to the gradients the static 128 leaves in fp16's subnormal range;
checkpoints; refusals."""
import numpy as np
import pytest
import torch

import tape_ref
from monoflex_b200 import engine, solver
from monoflex_b200.config import default_cfg
from monoflex_b200.loss_scale import DynamicLossScale
from oracle import monoflex_oracle as mo

pytestmark = pytest.mark.gpu

# found_inf pattern of the update-rule test (1 = an inf is written into the gradient arena before the step)
PATTERN = [0, 0, 0, 1, 0, 0, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0]


def _toy_opt(seed=0):
    gen = torch.Generator().manual_seed(seed)
    params = [torch.nn.Parameter(torch.randn(s, generator=gen).cuda()) for s in ((37, 5), (300,), (4, 4, 3, 3))]
    return solver.FusedAdamW([{"params": [p], "lr": 1e-3} for p in params], weight_decay=1e-4)


def _fill_grads(opt, gen, bad):
    for p in opt.arena.tensors:
        p.grad.copy_(torch.randn(p.shape, generator=gen).cuda() * 0.1)
    if bad:
        opt.arena.tensors[1].grad[7] = float("inf")


@pytest.mark.parametrize("init_scale", [2.0 ** 16, 2.0 ** 127])
@pytest.mark.parametrize("max_norm", [None, 1.0])
@pytest.mark.parametrize("captured", [False, True])
def test_update_rule_follows_amp_update_scale(init_scale, max_norm, captured):
    """scale and growth tracker after every step equal torch._amp_update_scale_ fed the same found_inf; 2^127 never grows
    to inf; parameters move exactly on the clean steps"""
    opt = _toy_opt()
    s = DynamicLossScale(init_scale=init_scale, growth_interval=3)
    ref_scale = torch.full((1,), init_scale, dtype=torch.float32, device="cuda")
    ref_tracker = torch.zeros(1, dtype=torch.int32, device="cuda")
    gen = torch.Generator().manual_seed(1)
    graph = None
    for t, bad in enumerate(PATTERN):
        _fill_grads(opt, gen, bad)
        before = opt.arena.params.clone()
        if captured and t >= 1:
            if graph is None:
                opt._lr_table()
                graph = torch.cuda.CUDAGraph()
                torch.cuda.synchronize()
                saved = (s.scale.clone(), s.growth_tracker.clone(), opt._state4.clone())
                with torch.cuda.graph(graph):
                    opt.step(max_grad_norm=max_norm, loss_scaler=s)
                opt.step_count -= 1
                opt._step_t -= 1
                assert torch.equal(s.scale, saved[0]) and torch.equal(opt._state4, saved[2])   # capture only records
            graph.replay()
            opt.step_count += 1
            opt._step_t += 1
        else:
            opt.step(max_grad_norm=max_norm, loss_scaler=s)
        torch._amp_update_scale_(ref_scale, ref_tracker, torch.full((1,), float(bad), device="cuda"), 2.0, 0.5, 3)
        torch.cuda.synchronize()
        assert s.scale.item() == ref_scale.item() and s.growth_tracker.item() == ref_tracker.item(), (t, s.state_dict())
        assert torch.equal(opt.arena.params, before) == bool(bad), t
    assert np.isfinite(s.get_scale())
    assert opt.skipped_steps() == sum(PATTERN) and int(opt._state4[0]) == len(PATTERN) - sum(PATTERN)
    if init_scale == 2.0 ** 127:
        assert s.get_scale() <= 2.0 ** 127


def _sizes():
    """every parameter shape of the detector (its ~280 gradients) plus odd and tiny sizes"""
    from monoflex_b200.model.detector import KeypointDetector
    shapes = [tuple(p.shape) for p in KeypointDetector(default_cfg()).parameters()]
    return shapes + [(1,), (3,), (5,), (4095,), (4097,), (8191, 3)]


@pytest.fixture(scope="module")
def pairs():
    gen = torch.Generator(device="cuda").manual_seed(3)
    shapes = _sizes()
    srcs, dsts = [], []
    for i, sh in enumerate(shapes):
        n = int(np.prod(sh))
        if i % 7 == 3:                     # misaligned views: the kernel's scalar path
            srcs.append(torch.randn(n + 1, generator=gen, device="cuda")[1:] * 1e3)
            dsts.append(torch.randn(n + 3, generator=gen, device="cuda")[3:])
        else:
            srcs.append(torch.randn(n, generator=gen, device="cuda") * 1e3)
            dsts.append(torch.randn(n, generator=gen, device="cuda"))
    return shapes, srcs, dsts


def test_unscale_accumulate_bit_identical_to_foreach_add(pairs):
    """dst += src * inv_scale in one launch over every size at once: bit-identical to _foreach_add_ for 2^k, k = 0..24;
    the first-assignment flag gives src * inv_scale"""
    shapes, srcs, dsts = pairs
    assert len(shapes) > 280
    s = DynamicLossScale()
    assign = [i % 11 == 5 for i in range(len(srcs))]
    for k in range(25):
        s.scale.fill_(2.0 ** k)
        inv = s.scale.double().reciprocal().float().item()
        got = [d.clone() for d in dsts]
        want = [d.clone() for d in dsts]
        s.unscale_accumulate(got, srcs)
        torch._foreach_add_(want, srcs, alpha=inv)
        for g, w in zip(got, want):
            assert torch.equal(g, w), k
        got = [d.clone() for d in dsts]
        s.unscale_accumulate(got, srcs, assign)
        for a, g, d, src in zip(assign, got, dsts, srcs):
            assert torch.equal(g, src * inv if a else d + src * inv), k


def test_unscale_accumulate_non_power_of_two_within_one_ulp(pairs):
    shapes, srcs, dsts = pairs
    s = DynamicLossScale(init_scale=1000.0)
    inv = s.scale.double().reciprocal().float().item()
    got = [d.clone() for d in dsts]
    want = [d.clone() for d in dsts]
    s.unscale_accumulate(got, srcs)
    torch._foreach_add_(want, srcs, alpha=inv)
    for g, w in zip(got, want):
        ulp = (torch.nextafter(w.abs(), torch.full_like(w, float("inf"))) - w.abs())
        assert bool(((g - w).abs() <= ulp).all())


# ------------------------------------------------------------------ the seeded two-image batch of the tape tests
def _model():
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    model = KeypointDetector(default_cfg()).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    return model


def _batch():
    from monoflex_b200 import synthetic as syn
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    return images, targets


class _F16Recorder(object):
    """stands in for `torch` inside monoflex_b200.tape: records every fp16 buffer predictor_backward allocates"""

    def __init__(self):
        self.bufs = []

    def __getattr__(self, k):
        return getattr(torch, k)

    def _rec(self, fn, *a, **kw):
        t = fn(*a, **kw)
        if t.dtype == torch.half:
            self.bufs.append(t)
        return t

    def zeros(self, *a, **kw):
        return self._rec(torch.zeros, *a, **kw)

    def empty(self, *a, **kw):
        return self._rec(torch.empty, *a, **kw)


@pytest.fixture(scope="module")
def sweep():
    """one forward of the seeded batch, then the backward and a guarded step (lr 0: nothing moves) at S = 2^k, k = 7, 8,
    ... until three scales in a row overflowed. Per S: whether the fp16 gradient flow overflowed, seen in every gradient
    buffer of the backbone tape (observe hook) and every fp16 buffer of the predictor backward, and whether the step
    was skipped."""
    from monoflex_b200 import tape
    model = _model()
    images, targets = _batch()
    feats = model.backbone.train_forward(images)
    pred_mod = model.heads.predictor
    pred = pred_mod.train_forward(feats, targets)
    c = pred["cls"].detach().clone().requires_grad_(True)
    r = pred["reg"].detach().clone().requires_grad_(True)
    loss_dict, _ = model.heads.loss_evaluator({"cls": c, "reg": r}, targets)
    sum(loss_dict.values()).backward()
    g_cls, g_reg = c.grad.clone(), r.grad.clone()
    opt = solver.FusedAdamW(solver.get_model_params(model, default_cfg()))
    for g in opt.param_groups:
        g["lr"] = 0.0                                          # the guard scans the arena, nothing is updated
    s = DynamicLossScale(growth_interval=10 ** 9).attach(opt)
    model.loss_scaler = s
    orig_bb, orig_torch = tape.backbone_backward, tape.torch
    rows = []
    try:
        for k in range(7, 64):
            flags = []

            def observe(rec, grad, done):
                if done:
                    for a in [rec["y"]] + [rec[n] for n in ("x", "residual", "skip") if rec.get(n) is not None]:
                        if a is not rec["y"] and a is model.backbone.last_plan.input:
                            continue
                        g = grad(a)
                        flags.append(~torch.isfinite(g.buf[:, g.ch_off:g.ch_off + g.C]).all())

            rec16 = _F16Recorder()
            tape.backbone_backward = lambda bb, plan, d, observe_=None: orig_bb(bb, plan, d, observe=observe)
            tape.torch = rec16
            s.scale.fill_(2.0 ** k)
            s.growth_tracker.zero_()
            skipped0 = opt.skipped_steps()
            opt.zero_grad()
            model._tape_backward(g_cls, g_reg)
            tape.backbone_backward, tape.torch = orig_bb, orig_torch
            opt.step(loss_scaler=s)
            overflow = bool(torch.stack(flags).any()) or any(not bool(torch.isfinite(b).all()) for b in rec16.bufs)
            skipped = opt.skipped_steps() > skipped0
            rows.append((k, overflow, skipped, len(rec16.bufs), len(flags)))
            if len(rows) >= 3 and all(r_[1] for r_ in rows[-3:]):
                break
    finally:
        tape.backbone_backward, tape.torch = orig_bb, orig_torch
        model.loss_scaler = None
    return dict(model=model, rows=rows, g_cls=g_cls, g_reg=g_reg)


def test_overflow_is_never_lost(sweep):
    """the step is skipped exactly at the scales whose fp16 gradient flow overflowed, and those scales are upward closed"""
    rows = sweep["rows"]
    print("\nk, overflowed, skipped, predictor fp16 buffers, backbone buffer checks:")
    for row in rows:
        print("  2^%d %s %s %d %d" % row)
    assert rows[0][3] >= 10 and rows[0][4] >= 100              # the recorders saw the buffers
    for k, overflow, skipped, _, _ in rows:
        assert overflow == skipped, (k, overflow, skipped)
    ks = [k for k, _, skipped, _, _ in rows if skipped]
    assert ks, "no overflow up to 2^%d" % rows[-1][0]
    assert ks == list(range(ks[0], rows[-1][0] + 1)), ks
    assert not rows[0][2]                                      # the static default 128 does not overflow on this batch


def _predictor_rel_err(model, plan, g_cls, g_reg, S, monkeypatch):
    """relative L2 error of every predictor parameter gradient at loss scale S against float64 autograd through the
    oracle's predictor at the kernels' forward point (fp16 storage points of the forward modelled, the backward's fp16
    rounding NOT modelled)"""
    from monoflex_b200.tape import predictor_backward
    pred_mod = model.heads.predictor
    ctx = plan.ctx
    pfx = "heads.predictor."
    hid, hc = ctx["hid"], pred_mod.head_conv

    def nchw(a):
        return a.buf[:, a.ch_off:a.ch_off + a.C].reshape(a.B, a.H, a.W, a.C).permute(0, 3, 1, 2).double()

    def iabn(sd, p, x):
        i = 0 if ".class_head." in p else int(p.split("reg_features.")[1].split(".")[0]) + 1
        mask = tape_ref.act_mask(nchw(engine.Act.on(hid.buf, hid.B, hid.H, hid.W, hc, hid.ch_off + i * hc)), tape_ref.ACT_LEAKY)
        return mo.bn_eval(sd, p, x, abs_weight=True) * mask
    monkeypatch.setattr(mo, "iabn", iabn)
    sd = {pfx + n: p.detach().double().requires_grad_(True) for n, p in pred_mod.named_parameters()}
    sd.update({pfx + n: b.double() for n, b in pred_mod.named_buffers()})
    feats = nchw(ctx["x"]).requires_grad_(True)

    def stored(t):
        return t + (t.half().double() - t).detach()
    with mo.training_mode():
        out = mo.predictor(sd, feats, plan.edge_idx, plan.edge_len, out_w=pred_mod.output_width,
                           out_h=pred_mod.output_height, stored=stored)
    torch.autograd.backward([out["cls"], out["reg"]], [g_cls.double(), g_reg.double()])
    pgrads, _ = predictor_backward(pred_mod, plan, g_cls * S, g_reg * S)
    errs = {}
    for name, g in pgrads.items():
        ref = sd[pfx + name].grad
        if ref.norm() > 0:
            errs[name] = ((g.double() / S - ref).norm() / ref.norm()).item()
    monkeypatch.undo()
    return errs


def test_larger_scale_lifts_the_subnormal_gradients(sweep, monkeypatch):
    """at the largest scale that does not overflow this batch, the 2d_dim branch's 3x3 weight gradient - which the
    static 128 moves by ~3e-2 through fp16 subnormals in d_raw - is at least three times closer to float64"""
    rows = sweep["rows"]
    k_max = max(k for k, _, skipped, _, _ in rows if not skipped)
    model = sweep["model"]
    plan = model.heads.predictor.last_plan
    e128 = _predictor_rel_err(model, plan, sweep["g_cls"], sweep["g_reg"], 128.0, monkeypatch)
    emax = _predictor_rel_err(model, plan, sweep["g_cls"], sweep["g_reg"], 2.0 ** k_max, monkeypatch)
    name = "reg_features.0.0.weight"
    print("\n%s rel-L2 vs float64: %.3e at S = 128, %.3e at S = 2^%d (largest non-overflowing scale)"
          % (name, e128[name], emax[name], k_max))
    # the edge Conv1d biases in front of a train-mode BatchNorm1d have an analytically zero gradient: no relative error
    nonzero = [n for n in emax if not (n.startswith("trunc_") and n.endswith(".0.bias"))]
    print("worst other predictor parameter: %.3e at 128, %.3e at 2^%d" % (
        max(e128[n] for n in nonzero), max(emax[n] for n in nonzero), k_max))
    assert k_max > 7, "this batch's largest safe scale does not exceed 128"
    assert emax[name] <= e128[name] / 3, (e128[name], emax[name])


# ------------------------------------------------------------------ trainers
def _twin(**kw):
    from monoflex_b200.train import Trainer
    cfg = default_cfg()
    model = _model()
    images, targets = _batch()
    return Trainer(model, cfg, **kw), images, targets


def _run(tr, images, targets, steps, sync_log=True):
    out = []
    opt = tr.optimizer
    for _ in range(steps):
        p0, m0 = opt.arena.params.clone(), opt.exp_avg.clone()
        sk0 = opt.skipped_steps()
        _, log = tr.step(images, targets, sync_log=sync_log)
        skipped = opt.skipped_steps() > sk0
        if skipped:
            assert torch.equal(opt.arena.params, p0) and torch.equal(opt.exp_avg, m0)
        else:
            assert not torch.equal(opt.arena.params, p0)
        out.append((skipped, tr.scaler.get_scale(), int(tr.scaler.growth_tracker), log))
    return out


def test_eager_and_captured_trainers_agree():
    """twin models from 2^16 with growth_interval 2: the same skips and scale sequence eagerly and replayed from the
    captured step; skipped steps leave parameters and moments alone; the device step counter counts applied updates"""
    ta, images, targets = _twin(loss_scale=DynamicLossScale(growth_interval=2))
    tb, _, _ = _twin(loss_scale=DynamicLossScale(growth_interval=2), use_cuda_graph=True, graph_warmup=2)
    assert ta.scaler is ta.model.loss_scaler and tb.scaler is tb.model.loss_scaler
    ra = _run(ta, images, targets, 8)
    rb = _run(tb, images, targets, 8, sync_log=False)
    assert tb._graph is not None
    print("\nstep: (skipped, scale, tracker) eager | captured")
    for i, (a, b) in enumerate(zip(ra, rb)):
        print("  %d: %s | %s" % (i, a[:3], b[:3]))
    assert [a[:3] for a in ra] == [b[:3] for b in rb]
    assert ra[0][0], "2^16 should back off on this batch"
    assert not all(a[0] for a in ra)
    for opt in (ta.optimizer, tb.optimizer):
        applied = sum(1 for a in ra if not a[0])
        assert int(opt._state4[0]) == applied and opt.skipped_steps() == 8 - applied
    for i, (a, b) in enumerate(zip(ra, rb)):
        if a[0]:
            continue                                       # a skipped step's losses are those of the unchanged model
        la, lb = a[3], b[3].resolve()
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)


def test_constant_dynamic_scale_equals_static():
    """DynamicLossScale(128, never growing) gives the static 128's gradients (up to the DCN backward's scatter atomics)
    and, with clipping on, the same gradient norm"""
    grads, norms = [], []
    for dyn in (False, True):
        model = _model()
        images, targets = _batch()
        opt = solver.build_optimizer(model, default_cfg())
        s = None
        if dyn:
            s = DynamicLossScale(init_scale=128.0, growth_interval=10 ** 9).attach(opt)
            model.loss_scaler = s
        else:
            model.loss_scale = 128.0
        loss_dict, _ = model(images, targets)
        opt.zero_grad()
        sum(loss_dict.values()).backward()
        grads.append(opt.arena.grads.clone())
        opt.step(max_grad_norm=1.0, loss_scaler=s)
        norms.append(opt.last_grad_norm.item())
        if dyn:
            assert s.get_scale() == 128.0 and opt.skipped_steps() == 0
    a, b = grads
    rel = ((a - b).norm() / a.norm()).item()
    print("\nconstant dynamic vs static 128: arena gradient rel-L2 %.3e, grad norm %.6g vs %.6g" % (rel, norms[0], norms[1]))
    assert rel <= 1e-2
    assert abs(norms[0] - norms[1]) <= 1e-2 * norms[0]


def test_checkpoint_round_trip_and_resume():
    """the scaler's state_dict loads into torch.amp.GradScaler("cuda") and back; after skipped steps the optimiser's
    state_dict counts applied updates; a trainer resumed from both continues with the same scale and step"""
    tr, images, targets = _twin(loss_scale=DynamicLossScale(growth_interval=2))
    for _ in range(5):
        tr.step(images, targets)
    skipped = tr.optimizer.skipped_steps()
    applied = 5 - skipped
    assert skipped > 0
    sd_s = tr.scaler.state_dict()
    ref = torch.amp.GradScaler("cuda")
    ref.load_state_dict(sd_s)
    assert ref.state_dict() == sd_s
    back = DynamicLossScale()
    back.load_state_dict(ref.state_dict())
    assert back.state_dict() == sd_s
    sd_o = tr.optimizer.state_dict()
    assert {float(st["step"]) for st in sd_o["state"].values()} == {float(applied)}
    assert tr.optimizer.step_count == applied
    sd_m = {k: v.clone() for k, v in tr.model.state_dict().items()}

    tr2, _, _ = _twin(loss_scale=back)
    tr2.model.load_state_dict(sd_m)
    tr2.optimizer.load_state_dict(sd_o)
    assert int(tr2.optimizer._state4[0]) == applied
    for _ in range(3):
        tr.step(images, targets)
        tr2.step(images, targets)
        assert tr.scaler.state_dict() == tr2.scaler.state_dict()
        assert int(tr.optimizer._state4[0]) == int(tr2.optimizer._state4[0])


def test_refusals():
    """a dynamic scale with the peer-memory exchange, and a dynamic scale no fused optimiser updates (the reference loop
    with torch.optim.AdamW), are refused - the latter at the first backward"""
    from monoflex_b200.train import Trainer
    model = _model()
    with pytest.raises(NotImplementedError, match="symmetric_group"):
        Trainer(model, default_cfg(), loss_scale="dynamic", symmetric_group=object())
    images, targets = _batch()
    model.loss_scaler = DynamicLossScale()
    opt = torch.optim.AdamW(solver.get_model_params(model, default_cfg()), lr=1e-4)
    loss_dict, _ = model(images, targets)
    opt.zero_grad()
    with pytest.raises(RuntimeError, match="no fused optimiser updates it"):
        sum(loss_dict.values()).backward()
    with pytest.raises(TypeError):
        model.loss_scaler.attach(opt)
