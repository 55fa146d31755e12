"""-m gpu: the training backward checked layer by layer at the kernels' own forward point.

Every record of the backbone tape (monoflex_b200/tape.py::backbone_backward) is compared, through the tape's `observe`
hook, with the float64 backward of the same layer (tests/tape_ref.py) taken at the fp16 values the forward recorded
(`x`, `raw`, `y`, `residual`, `skip`, the DCN's offset/mask rows), with the activation mask the kernels used (sign of the
recorded output) and with the upstream gradient the tape held when the record ran. The forward point is the kernels', so
the network's chaotic sensitivity to it never enters: what is left is fp16 rounding. The checks also cover what the tape
adds on top of its operators: which gradient buffer and channel slice each record adds into, that it ADDS (the buffer
already holds the gradients of earlier-replayed consumers), that nothing outside the slice moves, that no gradient
arrives after its consumer ran, and that every parameter the forward uses gets exactly one gradient.

The predictor backward (tape.py::predictor_backward) is compared as a whole with float64 autograd through the oracle's
predictor, fed the recorded fp16 feature map, with the kernels' fp16 storage points modelled by a straight-through round
trip: once with the training step's loss gradients, and once with seeded gradients that are non-zero everywhere, so that
the offset edge-fusion tail (which the seeded targets, with no truncated object, leave without gradient) is checked too.

Error model: every operator writes fp16 rows, d_raw (the BN's input gradient) and the offset/mask gradient are rounded
to fp16 before the convolution backward uses them, and dcn_col2im accumulates with half2 atomics. Expected: ~1e-3 of the
increment's magnitude for data gradients, less for weight gradients, ~1e-2 for the DCN's data and offset/mask
gradients. Every bound is about three times the worst value measured on an H100 (given beside it).
"""
import collections

import pytest
import torch

import tape_ref
from monoflex_b200 import engine
from monoflex_b200.config import default_cfg
from oracle import monoflex_oracle as mo

pytestmark = pytest.mark.gpu

LOSS_SCALE = 128.0                   # the trainer's MF_LOSS_SCALE default: gradients in the fp16 range training uses

# bound per check, about 3x the worst error measured on an NVIDIA H100 80GB HBM3 (700 W) over both geometries (value
# beside it). Data gradients ("dx", "residual"): max over the destination slice of |(after - before) - increment| less
# half an fp16 ulp of `after` (the rounding of the accumulation), over max |increment| - the increment against its own
# scale, however full the buffer already was. Parameter gradients: max|got - want| / max|want| per tensor unless noted.
# Checks not listed here are bit-exact (max-pool routing, the skip gradient of upsample_add, untouched columns).
BOUNDS = {
    "conv_bn dx": 1.2e-3,            # 4.0e-4
    "conv_bn residual": 4e-4,        # 1.2e-4
    "conv_bn dW": 2e-3,              # 5.7e-4
    "bn dgamma/dbeta": 1e-6,         # 3.4e-7: the BN operator's own inputs, no rounded intermediate
    "dcn dx": 7e-3,                  # 2.3e-3: fp16 grad columns, half2 atomics
    "dcn dW": 2e-3,                  # 5.8e-4
    "offmask dW": 2e-3,              # 6.2e-4
    "offmask dbias": 2.5e-3,         # 7.5e-4
    "dcn dbias / sum|d_raw|": 5e-4,  # 1.5e-4: max over channels of |dbias| / sum |d_raw|
    "upsample dx": 5e-5,             # 1.7e-5
    "upsample dW": 4e-7,             # 1.4e-7
}
PRED_BOUNDS = {                      # the predictor as a whole, worst measured over both upstream gradients
    "parameter": 3e-3,               # relative L2 per parameter gradient; 9.2e-4
    "d_feat": 1.5e-3,                # relative L2 of the feature-map gradient, whole map and near the edges; 5.5e-4
    "zero bias": 1.5e-3,             # max over channels of |dbias| / sum |d_raw|; 5.5e-4
}


def _nchw(a, buf=None):
    """float64 NCHW copy of activation `a` (an engine.Act over [M, ld] rows), read from `buf` (a snapshot) if given"""
    b = a.buf if buf is None else buf
    return b[:, a.ch_off:a.ch_off + a.C].reshape(a.B, a.H, a.W, a.C).permute(0, 3, 1, 2).double()


def _rows(t):
    B, C, H, W = t.shape
    return t.permute(0, 2, 3, 1).reshape(B * H * W, C)


def _half_ulp(h):
    """half a unit in the last place of each fp16 value of h (subnormals included), float64"""
    return torch.exp2(torch.floor(torch.log2(h.double().abs())).clamp_min(-14) - 11)


def _rel(got, want):
    return ((got.double() - want).abs().max() / want.abs().max().clamp_min(1e-300)).item()


class _Checker(object):
    """observe(rec, grad, done) for tape.backbone_backward: checks every record against tests/tape_ref.py"""

    def __init__(self, backbone, plan):
        self.plan = plan
        self.index = {id(r): i for i, r in enumerate(plan.tape)}
        self.names = {id(p): n for n, p in backbone.named_parameters()}
        self.errs = collections.defaultdict(list)          # check -> [(error, where)]
        self.ref_params = {}                               # parameter name -> (check, float64 reference)
        self.duplicates = []
        self.visits = collections.Counter()
        self.final = []                                    # (grad(y), its rows when the record ran)
        self.grad_acts = []                                # every gradient buffer the records touch
        self.before = None
        self.tied_windows = 0                              # max-pool windows whose maximum occurs more than once

    def _param(self, p, check, ref):
        name = self.names[id(p)]
        if name in self.ref_params:
            self.duplicates.append(name)
        self.ref_params[name] = (check, ref.reshape(p.shape))

    def _dests(self, rec):
        return [rec[k] for k in ("x", "residual", "skip") if rec.get(k) is not None and rec[k] is not self.plan.input]

    def __call__(self, rec, grad, done):
        y = rec["y"]
        if not done:
            self.visits[id(rec)] += 1
            self.before = {}                               # buffer address -> (live gradient buffer, its copy now)
            for a in [y] + self._dests(rec):
                g = grad(a)
                self.before.setdefault(g.buf.data_ptr(), (g.buf, g.buf.clone()))
                self.grad_acts.append(g)
            gy = grad(y)
            self.final.append((gy, gy.buf[:, gy.ch_off:gy.ch_off + gy.C].clone()))
            return
        where = "#%d %s -> %dx%dx%d" % (self.index[id(rec)], rec["kind"], y.C, y.H, y.W)
        gy = grad(y)
        dy = _nchw(gy, self.before[gy.buf.data_ptr()][1])
        incs, exact = [], []               # (check, destination activation, float64 increment: compared / fp16-exact)
        kind = rec["kind"]
        if kind in ("conv_bn", "dcn"):
            mod = rec["bn"][0][0]
            assert all(e[0] is mod for e in rec["bn"])
            d_raw, g, dgamma, dbeta = tape_ref.bn_backward(_nchw(rec["raw"]), _nchw(y), dy, mod.weight.detach(), mod.eps,
                                                           rec.get("act", engine.ACT_RELU), rec.get("abs_weight", False))
            self._param(mod.weight, "bn dgamma/dbeta", dgamma)
            self._param(mod.bias, "bn dgamma/dbeta", dbeta)
            x = _nchw(rec["x"])
            if kind == "conv_bn":
                w = rec["weight"].detach()
                if rec["x"] is self.plan.input:
                    x = x[:, :w.shape[1]]                  # the packed image: 3 colour channels, zero padding
                dx, dw = tape_ref.conv_backward(x, w, d_raw, rec["stride"], rec["pad"])
                self._param(rec["weight"], "conv_bn dW", dw)
                assert rec["bias"] is None
                if rec["x"] is not self.plan.input:
                    incs.append(("conv_bn dx", rec["x"], dx))
                if rec["residual"] is not None:
                    incs.append(("conv_bn residual", rec["residual"], g))
            else:
                dcn = rec["mod"]
                om = rec["om"].view(y.B, y.H, y.W, 32).permute(0, 3, 1, 2).double()
                dx1, d_off, d_pre, dw, _ = tape_ref.dcn_backward(x, om[:, :18], om[:, 18:27], dcn.weight.detach(), d_raw)
                dom = torch.cat([d_off, d_pre], 1)
                dx2, dw_om = tape_ref.conv_backward(x, dcn.conv_offset_mask.weight.detach(), dom, 1, 1)
                self._param(dcn.weight, "dcn dW", dw)
                # in front of a train-mode BN the bias gradient is analytically zero: bounded by sum |d_raw| per channel
                self._param(dcn.bias, "dcn dbias / sum|d_raw|", d_raw.abs().sum((0, 2, 3)))
                self._param(dcn.conv_offset_mask.weight, "offmask dW", dw_om)
                self._param(dcn.conv_offset_mask.bias, "offmask dbias", dom.sum((0, 2, 3)))
                incs.append(("dcn dx", rec["x"], dx1 + dx2))
                assert dom.abs().max().item() < 3e4, where  # the tape narrows this fp32 gradient to fp16 rows
        elif kind == "maxpool2":
            xv = _nchw(rec["x"])
            win = xv.reshape(xv.shape[0], xv.shape[1], xv.shape[2] // 2, 2, xv.shape[3] // 2, 2)
            self.tied_windows += ((win == win.amax((3, 5), keepdim=True)).sum((3, 5)) > 1).sum().item()
            exact.append(("maxpool2 dx", rec["x"], tape_ref.maxpool2_backward(xv, dy)))
        elif kind == "upsample_add":
            dx, dw, dskip = tape_ref.upsample_backward(_nchw(rec["x"]), rec["weight"].detach(), dy, rec["f"])
            self._param(rec["weight"], "upsample dW", dw)
            incs.append(("upsample dx", rec["x"], dx))
            if rec["skip"] is not None:
                assert grad(rec["skip"]).buf.data_ptr() != grad(rec["x"]).buf.data_ptr()
                exact.append(("upsample dskip", rec["skip"], dskip))
        else:
            raise AssertionError("unknown tape record %r" % kind)
        # every gradient buffer the record could touch: every column outside the destination slices bit-identical; in the
        # slices, what the record added (after - before, exact in float64) against the sum of the float64 increments that
        # land there, relative to the increments' own magnitude. The fp16 rounding of the sum (at most half an ulp of
        # `after`) is the one part of the difference that is not the increment's error, and it is allowed for.
        for ptr, (now, buf0) in self.before.items():
            inc_sum = torch.zeros(buf0.shape, dtype=torch.float64, device=buf0.device)
            covered = torch.zeros(buf0.shape[1], dtype=torch.bool, device=buf0.device)
            compared = []
            for is_exact, (check, a, inc) in [(False, t) for t in incs] + [(True, t) for t in exact]:
                ga = grad(a)
                if ga.buf.data_ptr() != ptr:
                    continue
                sl = slice(ga.ch_off, ga.ch_off + ga.C)
                assert not covered[sl].any() or not is_exact, (check, where)
                covered[sl] = True
                if is_exact:
                    want16 = (buf0[:, sl].float() + _rows(inc).float()).half()     # the fp32 add of mf_add_rows_f16
                    assert torch.equal(now[:, sl], want16), (check, where)
                    self.errs[check].append((0.0, where))
                else:
                    inc_sum[:, sl] += _rows(inc)
                    compared.append((check, sl))
            if compared:
                miss = ((now.double() - buf0.double() - inc_sum).abs() - _half_ulp(now)).clamp_min(0)
                for check, sl in compared:
                    self.errs[check].append(((miss[:, sl].max() / inc_sum[:, sl].abs().max().clamp_min(1e-300)).item(), where))
            assert torch.equal(now[:, ~covered], buf0[:, ~covered]), ("gradient written outside its slice", where)

    def param_errors(self, grads):
        for name, (check, ref) in self.ref_params.items():
            got = grads[name].double()
            assert torch.isfinite(got).all(), name
            if check == "dcn dbias / sum|d_raw|":
                self.errs[check].append(((got.abs() / ref.clamp_min(1e-30)).max().item(), name))
            else:
                self.errs[check].append((_rel(got, ref), name))


def _model():
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    model = KeypointDetector(default_cfg()).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    return model


def _replay_checked(model, d_feat):
    from monoflex_b200.tape import backbone_backward
    plan = model.backbone.last_plan
    chk = _Checker(model.backbone, plan)
    grads = backbone_backward(model.backbone, plan, d_feat, observe=chk)
    torch.cuda.synchronize()
    chk.param_errors(grads)
    return plan, chk, grads


def _check_replay(plan, chk, grads, backbone):
    # every record visited exactly once
    assert len(chk.visits) == len(plan.tape) and set(chk.visits.values()) == {1}
    # finality: no gradient reached an activation after the record consuming it ran
    for gy, rows in chk.final:
        assert torch.equal(gy.buf[:, gy.ch_off:gy.ch_off + gy.C], rows)
    # producers: every activation a record reads is the input image or lies inside the outputs of records
    covered = {}
    for rec in plan.tape:
        y = rec["y"]
        covered.setdefault(y.buf.data_ptr(), torch.zeros(y.buf.shape[1], dtype=torch.bool))[y.ch_off:y.ch_off + y.C] = True
    for rec in plan.tape:
        for k in ("x", "residual", "skip"):
            a = rec.get(k)
            if a is None or a is plan.input:
                continue
            c = covered.get(a.buf.data_ptr())
            assert c is not None and bool(c[a.ch_off:a.ch_off + a.C].all()), ("activation without a producer", rec["kind"], k)
    # completeness: one gradient per parameter the forward uses; the outer `project` of 2-level trees has none
    assert not chk.duplicates, chk.duplicates
    unused = {n for n, _ in backbone.named_parameters() if n.startswith(("base.level3.project", "base.level4.project"))}
    assert len(unused) == 6 and not unused & set(grads)
    assert set(grads) == set(chk.ref_params) == {n for n, _ in backbone.named_parameters()} - unused
    # the max-pool routing check is a tie test: the recorded ReLU outputs must tie in some windows
    print("\ntied max-pool windows: %d" % chk.tied_windows)
    assert chk.tied_windows > 0
    # finite rows in every gradient buffer
    for g in chk.grad_acts:
        assert torch.isfinite(g.buf[:, g.ch_off:g.ch_off + g.C]).all()


def _assert_bounds(chk, tag):
    print("\n%s: worst error per check (bound)" % tag)
    for check, errs in sorted(chk.errs.items()):
        worst = max(errs)
        print("  %-26s %.3e  (%s)  at %s, n=%d" % (check, worst[0], BOUNDS.get(check, "bit-exact"), worst[1], len(errs)))
    for check, errs in chk.errs.items():
        worst = max(errs)
        assert worst[0] <= BOUNDS.get(check, 0.0), (check, worst)


@pytest.fixture(scope="module")
def trained():
    """the seeded two-image training step of the tape tests: forward, loss x 128, predictor backward, observed replay"""
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.tape import predictor_backward
    model = _model()
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    feats = model.backbone.train_forward(images)
    pred_mod = model.heads.predictor
    pred = pred_mod.train_forward(feats, targets)
    c = pred["cls"].detach().clone().requires_grad_(True)
    r = pred["reg"].detach().clone().requires_grad_(True)
    loss_dict, _ = model.heads.loss_evaluator({"cls": c, "reg": r}, targets)
    (LOSS_SCALE * sum(loss_dict.values())).backward()
    pgrads, d_feat = predictor_backward(pred_mod, pred_mod.last_plan, c.grad, r.grad)
    plan, chk, grads = _replay_checked(model, d_feat)
    return dict(model=model, pred_plan=pred_mod.last_plan, grad_cls=c.grad, grad_reg=r.grad, pgrads=pgrads,
                d_feat=d_feat, plan=plan, chk=chk, grads=grads)


def test_backbone_tape_layer_by_layer(trained):
    """B = 2, 384 x 1280, the real feature-map gradient"""
    plan, chk = trained["plan"], trained["chk"]
    kinds = collections.Counter(r["kind"] for r in plan.tape)
    assert (kinds["dcn"], kinds["maxpool2"], kinds["upsample_add"]) == (16, 6, 8), kinds
    _check_replay(plan, chk, trained["grads"], trained["model"].backbone)
    _assert_bounds(chk, "B=2 384x1280")


def test_backbone_tape_layer_by_layer_ragged(trained):
    """B = 1, 128 x 416: level 5 is 4 x 13 (odd width, ragged tiles), BN over one image, a seeded feature-map gradient at
    the real one's rms"""
    from monoflex_b200 import synthetic as syn
    model = _model()
    images = syn.make_images(1, 128, 416, seed=3).cuda()
    model.backbone.train_forward(images)
    assert model.backbone.last_plan.levels[5].W == 13
    rms = trained["d_feat"].float().pow(2).mean().sqrt().item()
    gen = torch.Generator(device="cuda").manual_seed(11)
    out = model.backbone.last_plan.output
    d_feat = (torch.randn(out.M, out.C, generator=gen, device="cuda") * rms).half()
    plan, chk, grads = _replay_checked(model, d_feat)
    _check_replay(plan, chk, grads, model.backbone)
    _assert_bounds(chk, "B=1 128x416")


class _grad_f16(torch.autograd.Function):
    """identity whose backward rounds the gradient to fp16: the InPlaceABN backward writes d_raw as fp16 rows in place.
    This rounding must be modelled here, not only bounded: the 2d_dim branch's loss gradient is non-zero at a few object
    pixels, so the BN backward's mean terms leave d_raw at 1e-6 .. 1e-5 (x 128) over every other pixel, in fp16's subnormal
    range, and they add up coherently in the 3x3 weight gradient (3e-2 relative on reg_features.0.0.weight otherwise)."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.half().double()


@pytest.mark.parametrize("upstream", ["loss", "random"])
def test_predictor_backward_vs_float64_autograd(trained, monkeypatch, upstream):
    """the whole predictor backward against float64 autograd through the oracle's predictor at the kernels' forward point:
    the recorded fp16 feature map, the plan's edge indices, the InPlaceABN's leaky mask from the sign of the recorded
    hidden map, and the hidden maps, gathered edge features and BatchNorm1d outputs rounded to fp16 where the kernels
    store them. upstream="loss": the loss gradients of the training step. The seeded targets hold no truncated object,
    so their 3d_offset gradient is zero at every edge position and the offset edge tail gets none; upstream="random":
    seeded gradients at the loss gradients' rms (the backward is linear in them), non-zero everywhere, so that every
    parameter - the offset edge tail's included - has a non-zero reference gradient."""
    from monoflex_b200.tape import predictor_backward
    pred_mod = trained["model"].heads.predictor
    plan = trained["pred_plan"]
    ctx = plan.ctx
    pfx = "heads.predictor."
    hid, hc = ctx["hid"], pred_mod.head_conv
    if upstream == "loss":
        grad_cls, grad_reg = trained["grad_cls"], trained["grad_reg"]
        pgrads, d_feat = trained["pgrads"], trained["d_feat"]
    else:
        gen = torch.Generator(device="cuda").manual_seed(12)
        grad_cls, grad_reg = [torch.randn(g.shape, generator=gen, device="cuda") * g.pow(2).mean().sqrt()
                              for g in (trained["grad_cls"], trained["grad_reg"])]
        pgrads, d_feat = predictor_backward(pred_mod, plan, grad_cls, grad_reg)
        torch.cuda.synchronize()

    def iabn(sd, p, x):
        """InPlaceABN with the leaky mask the kernels used (the float64 pre-activations straddle zero elsewhere)"""
        i = 0 if ".class_head." in p else int(p.split("reg_features.")[1].split(".")[0]) + 1
        mask = tape_ref.act_mask(_nchw(engine.Act.on(hid.buf, hid.B, hid.H, hid.W, hc, hid.ch_off + i * hc)), tape_ref.ACT_LEAKY)
        return mo.bn_eval(sd, p, _grad_f16.apply(x), abs_weight=True) * mask
    monkeypatch.setattr(mo, "iabn", iabn)
    sd = {pfx + n: p.detach().double().requires_grad_(True) for n, p in pred_mod.named_parameters()}
    sd.update({pfx + n: b.double() for n, b in pred_mod.named_buffers()})
    feats = _nchw(ctx["x"]).requires_grad_(True)
    kept = []

    def stored(t):
        t = t + (t.half().double() - t).detach()
        if t.dim() == 3 and t.shape[1] == pred_mod.head_conv:             # the two BatchNorm1d outputs of the edge tail
            t.retain_grad()
            kept.append(t)
        return t
    with mo.training_mode():
        out = mo.predictor(sd, feats, plan.edge_idx, plan.edge_len, out_w=pred_mod.output_width,
                           out_h=pred_mod.output_height, stored=stored)
    torch.autograd.backward([out["cls"], out["reg"]], [grad_cls.double(), grad_reg.double()])
    assert set(pgrads) == {n for n, _ in pred_mod.named_parameters()}
    errs, zero = {}, []
    for name, g in pgrads.items():
        ref = sd[pfx + name].grad
        assert torch.isfinite(g).all(), name
        if ref.norm() > 0:
            errs[name] = ((g.double() - ref).norm() / ref.norm()).item()
        else:                                     # exactly zero upstream: the kernels must give exact zeros too
            assert upstream == "loss" and name.startswith("trunc_offset_conv.") and not g.any(), name
            zero.append(name)
    assert len(zero) == (6 if upstream == "loss" else 0), zero
    # the edge Conv1d biases sit in front of a train-mode BatchNorm1d: analytically zero, so bounded by the per-channel
    # sum |d_raw| of their BatchNorm1d's input gradient instead
    zero_bias = {}
    for seq, t in zip((pred_mod.trunc_heatmap_conv, pred_mod.trunc_offset_conv), kept):
        [entry] = ctx["bn"][id(seq[1])]
        raw = entry[1]
        B, K = raw.B, raw.W
        rawv = raw.buf[:, raw.ch_off:raw.ch_off + raw.C].reshape(B, K, -1).permute(0, 2, 1).double()
        y = entry[2]
        yv = y.buf[:, y.ch_off:y.ch_off + y.C].reshape(B, K, -1).permute(0, 2, 1).double()
        d_raw = tape_ref.bn_backward(rawv, yv, t.grad, seq[1].weight.detach(), seq[1].eps, tape_ref.ACT_NONE)[0]
        name = [n for n, p in pred_mod.named_parameters() if p is seq[0].bias][0]
        if name in zero:
            continue
        assert d_raw.abs().sum((0, 2)).min() > 0, name
        zero_bias[name] = (pgrads[name].double().abs() / d_raw.abs().sum((0, 2))).max().item()
        del errs[name]
    d_err = ((_rows(feats.grad) - d_feat.double()).norm() / feats.grad.norm()).item()
    # the edge-fusion tail reaches the feature map only within one pixel of the ~830 border positions of each image: its
    # own check, so that an error confined to it cannot hide in the whole map's norm
    B, H, W = hid.B, hid.H, hid.W
    near = torch.zeros(B, 1, H, W, device=feats.device)
    for b in range(B):
        e = plan.edge_idx[b, :int(plan.edge_len[b])]
        near[b, 0, e[:, 1], e[:, 0]] = 1
    near = _rows(torch.nn.functional.max_pool2d(near, 3, 1, 1)).bool().view(-1)
    d_err_edge = ((_rows(feats.grad)[near] - d_feat.double()[near]).norm() / _rows(feats.grad)[near].norm()).item()
    worst = max(errs.items(), key=lambda kv: kv[1])
    print("\npredictor (%s upstream): worst parameter rel-L2 %.3e (%s), d_feat rel-L2 %.3e (%.3e near the edges), zero "
          "biases / sum|d_raw| %s" % (upstream, worst[1], worst[0], d_err, d_err_edge, zero_bias))
    assert worst[1] <= PRED_BOUNDS["parameter"], worst
    assert d_err <= PRED_BOUNDS["d_feat"] and d_err_edge <= PRED_BOUNDS["d_feat"], (d_err, d_err_edge)
    assert max(zero_bias.values()) <= PRED_BOUNDS["zero bias"], zero_bias
