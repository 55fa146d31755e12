"""The backbone plan launch by launch against float64, at pair precision (-m gpu, except the host-side checks of the helpers).

The whole-network tests (tests/test_gpu_model.py) hold the strict backbone to 1e-3 of the fp32 oracle, because rounding
builds up over ~50 layers. A lost or misplaced lo half moves one layer by only a few 1e-4, so it hides under that bound.
Here every op the plan builder emits (Plan.conv, conv_rows_strict, conv_rows, dcn, maxpool2, upsample_add) is recorded
while the real KeypointDetector backbone builds its plan, and after one forward each launch's output is compared with
float64 computed from the values that launch actually read: pairs are read straight from the plan's buffers (concat
slices, lo blocks at the owning buffer's half width, the planar stem layouts), never through a device-side conversion.
So errors do not build up and the strict bound stays at the per-kernel STRICT_TOL, except for the long reductions
(STRICT_DEEP_TOL below).

Each op's reference, in float64 on the recorded inputs and the weights the kernels multiply (param64: the strict packers'
W_hi + W_lo pairs, the fast packers' fp16(W)); the error against the fp32 weights themselves is printed beside it:
  conv       conv2d, eval BatchNorm folded in double, + residual, activation (stem convs on the image pair plane)
  dcn        the offset/mask conv against conv2d + sigmoid; the gather + contract through the oracle's dcn_v2_forward on the
             GPU's own float32 offsets and masks (sampling positions and bilinear weights in float32, as the reference
             computes them), then BatchNorm + ReLU
  maxpool2   max_pool2d, bit for bit (the pair max is lossless)
  upsample   the depth-wise conv_transpose2d + the skip
The errors are per image and per channel, relative to max(max|ref_c|, 0.05 max|ref|), so one wrong 8-channel group cannot
hide behind the tensor's largest channel. The float64 side runs on the GPU (torch's float64 convolutions and the oracle's
gather), so the product geometry B = 8, 384x1280 needs no reduction.

The check is shown to be sharp twice: dropping the lo halves from every op's reference inputs moves that reference by at
least 4x its tolerance, and zeroing the lo block a conv, a DCN and the largest up-sample read on the GPU, then relaunching
just their launches, makes their check fail by at least 4x. The deepest up-sample the product runs is f = 4 (ida_up;
every dla_up stage up-samples by 2), so f = 8 is covered by the per-kernel tests at the end of this file.

Fast precision runs through the same recorder: fp16 inputs as stored, fp16-rounded weights, the DCN blend rounded to fp16
as the kernel stores it, at the per-kernel tolerances of tests/test_gpu_ops.py.

Measured on an H100 80GB HBM3 (700 W power limit), worst per-channel error over both shapes, strict | fast:
  conv (K < 1152) 2.4e-5 | 4.9e-4    conv (K >= 1152) 9.7e-5 | 4.9e-4    stem rows 1.3e-6 | 4.7e-4
  dcn 6.5e-5 (offset conv 2.1e-5) | 1.0e-3    maxpool2 0 | 0    upsample_add 2.4e-7 | 4.8e-4
Dropping the lo halves moves every strict reference by 9.2e-4 or more; zeroing them on the GPU makes the level2 residual
conv, the node DCN after the f = 4 up-sample and that up-sample fail by 1.4e-3, 2.9e-3 and 4.6e-4. Against the fp32
weights the offset convs reading level 5 measure 1.2e-4: the He-initialised weights are ~0.01-0.02 there, so W_lo sits in
fp16's subnormal range and keeps only the bits above 2^-25, the pair format's absolute floor (csrc/mf_split.cu). The
whole file runs in about 20 s, the float64 side included."""
import inspect
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_ops import STRICT_TOL
from monoflex_b200 import engine, synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.model.backbone.dla_dcn import DeformConv
from monoflex_b200.model.detector import KeypointDetector
from oracle import monoflex_oracle as mo

FAST_CONV_TOL = 1e-3     # fp16 output: one rounding is 4.9e-4 of the value
FAST_DCN_TOL = 1.5e-3    # plus the fp16 rounding of the blended samples
# strict convs and DCNs with a reduction K = taps x Cin >= 1152 (levels 4-5 and the DCNs reading them): the three products
# of every K step accumulate in the tensor cores' fp32 accumulator, whose error grows with K; measured up to 9.3e-5
# (level5 3x3 convs, K = 4608) per channel, the same whether the reference multiplies the fp32 weights or their pairs
STRICT_DEEP_TOL = 1.2e-4
DEEP_K = 1152
LO_MARGIN = 4            # a lost lo half must move the check by at least this many tolerances

SHAPES = [(8, 384, 1280), (3, 160, 288)]     # the bench geometry; level 5 is 5x9, every level ragged against the tiles
SHAPE_IDS = ["%dx%dx%d" % s for s in SHAPES]

RECORDED = ("conv", "conv_rows_strict", "conv_rows", "dcn", "maxpool2", "upsample_add")
# the launches each recorded op emits, in order, per precision
LAUNCHES = {
    ("conv", "strict"): ("mf_conv2d_nhwc_f16x2",),
    ("conv", "fast"): ("mf_conv2d_nhwc_f16",),
    ("conv_rows_strict", "strict"): ("mf_conv2d_rows_f16x2",),
    ("conv_rows", "fast"): ("mf_conv2d_rows_f16",),
    ("dcn", "strict"): ("mf_conv2d_nhwc_f16x2", "mf_dcn_nhwc_f16x2"),
    ("dcn", "fast"): ("mf_conv2d_nhwc_f16", "mf_dcn_nhwc_f16"),
    ("maxpool2", "strict"): lambda op: row_format_launch(op, "mf_maxpool2_nhwc_f16", True),
    ("maxpool2", "fast"): lambda op: row_format_launch(op, "mf_maxpool2_nhwc_f16", False),
    ("upsample_add", "strict"): lambda op: row_format_launch(op, "mf_upsample_add_nhwc_f16", True),
    ("upsample_add", "fast"): lambda op: row_format_launch(op, "mf_upsample_add_nhwc_f16", False),
}
# argument positions of the lo offsets of the launches that read and write either row format (include/monoflex_b200.h);
# the up-sample's skip_lo (6) only counts with a skip input (argument 4)
LO_ARGS = {"mf_maxpool2_nhwc_f16": (2, 5), "mf_upsample_add_nhwc_f16": (2, 6, 9)}


def row_format_launch(op, name, pair):
    """(name,) when the op's launch passes pair-row lo offsets (all non-zero) in a strict plan and fp16 rows (all zero) in
    a fast one; otherwise a description of the wrong format, which no launch list matches"""
    args = op.plan.launches[op.first][1]
    lo = [args[i] for i in LO_ARGS[name] if not (name == "mf_upsample_add_nhwc_f16" and i == 6 and args[4] is None)]
    if all((v != 0) == pair for v in lo):
        return (name,)
    return ("%s with lo offsets %s" % (name, lo),)


# ------------------------------------------------------------------------------------------------ recording the plan
class Op(object):
    """one recorded plan-builder call: its kind, bound arguments, returned Act, [first, end) launch range and, for a DCN,
    the fp32 [M, 32] offset/mask rows it keeps; `subs` are the recorded calls it made itself, `kept` the tensors it added
    to plan.keep and `saved` its Plan.bn_saved entries (train plans)"""

    def __init__(self, plan, kind, args, y, first, end, om, subs=(), kept=(), saved=()):
        self.plan, self.kind, self.args, self.y, self.first, self.end, self.om = plan, kind, args, y, first, end, om
        self.subs, self.kept, self.saved = list(subs), list(kept), list(saved)

    def sub(self, kind):
        """the first recorded call of `kind` this op made itself"""
        return next(o for o in self.subs if o.kind == kind)

    @property
    def x(self):
        return self.args["x"]

    @property
    def reads(self):
        """the activations the op's launches read"""
        extra = {"conv": "residual", "upsample_add": "skip"}.get(self.kind)
        return [a for a in (self.x, self.args.get(extra)) if a is not None]


def record(monkeypatch, kinds=RECORDED):
    """wrap the plan builder's op emitters `kinds`; returns the list the outermost wrapped calls are appended to (the
    calls they make themselves go to their `subs`)"""
    ops = []
    frames = [ops]                        # the list the call being recorded is appended to, innermost last

    def wrap(kind, fn):
        sig = inspect.signature(fn)

        def recorded(self, *args, **kw):
            bound = sig.bind(self, *args, **kw)
            bound.apply_defaults()
            first, keep0, saved0 = len(self.ops), len(self.keep), len(self.bn_saved)
            frames.append([])
            try:
                y = fn(self, *args, **kw)
            finally:
                subs = frames.pop()
            a = dict(bound.arguments)
            del a["self"]
            frames[-1].append(Op(self, kind, a, y, first, len(self.ops), self.keep[keep0] if kind == "dcn" else None,
                                 subs, self.keep[keep0:], self.bn_saved[saved0:]))
            return y
        return recorded

    for kind in kinds:
        monkeypatch.setattr(engine.Plan, kind, wrap(kind, getattr(engine.Plan, kind)))
    return ops


def check_coverage(ops, names, precision, launches=None):
    """the recorded launch ranges tile [0, len(names)) and each emits exactly the launches of its kind -> problems.
    `launches` (default LAUNCHES): (kind, precision) -> the launch names, or a function of the op giving them"""
    bad, pos = [], 0
    for op in sorted(ops, key=lambda o: o.first):
        if op.first != pos:
            bad.append("launches %d..%d: %s" % (pos, op.first, names[pos:op.first]))
        want = (LAUNCHES if launches is None else launches).get((op.kind, precision))
        if callable(want):
            want = want(op)
        if want is None or tuple(names[op.first:op.end]) != want:
            bad.append("%s at %d: %s" % (op.kind, op.first, names[op.first:op.end]))
        pos = max(pos, op.end)
    if pos != len(names):
        bad.append("launches %d..%d: %s" % (pos, len(names), names[pos:]))
    return bad


# ------------------------------------------------------------------------------------------------ reading pairs
def halves(a):
    """(hi, lo) of Act `a` as float64 [B, C, H, W] on its buffer's device, read straight from `buf` (NHWC rows with
    ch_off and the lo block `a.lo` elements after hi, or the planar stem layout [B][H][(2) x C/8 x npar][W/npar][8], see
    Act.nchw_view); lo is None for an fp16 activation"""
    s = 2 if a.split else 1
    if a.npar:
        assert a.ch_off == 0
        v = a.buf.view(a.B, a.H, s, a.C // 8, a.npar, a.W // a.npar, 8).double()
        v = v.permute(0, 2, 3, 6, 1, 5, 4).reshape(a.B, s, a.C, a.H, a.W)
        return v[:, 0], (v[:, 1] if a.split else None)
    rows = a.buf.view(a.B, a.H, a.W, a.ld)
    hi = rows[..., a.ch_off:a.ch_off + a.C].permute(0, 3, 1, 2).double()
    if not a.split:
        return hi, None
    return hi, rows[..., a.ch_off + a.lo:a.ch_off + a.lo + a.C].permute(0, 3, 1, 2).double()


def image_halves(x8):
    """the strict row-segment stem's image pair plane [hi3 | lo3 | 0 0] (mf_pack_image_pair8) -> (hi, lo)"""
    v, _ = halves(x8)
    assert not v[:, 6:].any()
    return v[:, 0:3], v[:, 3:6]


def pair_format_errors(hi, lo):
    """-> list of violations of the pair format: non-finite halves, |lo| > ulp(hi) / 2 (hi = fp16(v), lo = fp16(v - hi))"""
    bad = []
    if not (torch.isfinite(hi).all() and torch.isfinite(lo).all()):
        bad.append("non-finite")
    # the fp16 spacing above |hi|, from the next bit pattern: exact on every device (a tie puts lo exactly on ulp/2, and
    # the CUDA pow(2, e) is not exact enough to compare against)
    m = hi.abs().half()
    ulp = (m.view(torch.int16) + 1).view(torch.float16).double() - m.double()
    n = int((lo.abs() > ulp / 2).sum())
    if n:
        bad.append("%d lo halves above ulp(hi)/2" % n)
    return bad


def values(a, keep_lo=True):
    """float64 values of Act `a`: hi + lo for pairs (hi alone when keep_lo is False), the fp16 values otherwise"""
    hi, lo = halves(a)
    return hi + lo if (lo is not None and keep_lo) else hi


# ------------------------------------------------------------------------------------------------ float64 references
def bn_fold(bn):
    s = bn.weight.detach().double() / torch.sqrt(bn.running_var.detach().double() + bn.eps)
    return s, bn.bias.detach().double() - bn.running_mean.detach().double() * s


def activate(y, act):
    return {engine.ACT_RELU: F.relu, engine.ACT_NONE: lambda t: t, engine.ACT_LEAKY: lambda t: F.leaky_relu(t, 0.01)}[act](y)


def param64(w, kind="fp32"):
    """a conv weight in float64: 'fp32' as stored, 'pair' = W_hi + W_lo as the strict packers split it (fp16(W) and
    fp16(W - W_hi): a W_lo below 2^-14 keeps only the bits above 2^-25), 'fp16' = fp16(W) as the fast packer rounds it"""
    w = w.detach().float()
    hi = w.half()
    if kind == "fp16":
        return hi.double()
    if kind == "pair":
        return hi.double() + (w - hi.float()).half().double()
    return w.double()


def conv_ref(x, w, stride, pad, bn, act, residual=None, weights="fp32", bias=None):
    """eval-mode conv (+ bias) + BatchNorm (+ residual) + activation in float64; bn=None: no normalisation (the raw
    convolutions of train plans). A Conv1d weight [O, I, k] runs as [O, I, 1, k] over a [B, I, 1, L] input."""
    w = param64(w, weights).to(x.device)
    if w.dim() == 3:
        w = w.unsqueeze(2)
    y = F.conv2d(x, w, None if bias is None else bias.detach().double().to(x.device), stride, pad)
    if bn is None:
        return activate(y if residual is None else y + residual, act)
    s, t = bn_fold(bn)
    y = y * s.to(y.device).view(1, -1, 1, 1) + t.to(y.device).view(1, -1, 1, 1)
    if residual is not None:
        y = y + residual
    return activate(y, act)


def offset_mask_ref(x, om_conv, weights="fp32"):
    """DCN.conv_offset_mask + the sigmoid of the mask channels: [B, 27, H, W] float64"""
    om = F.conv2d(x, param64(om_conv.weight, weights).to(x.device), om_conv.bias.detach().double().to(x.device), 1, 1)
    return torch.cat([om[:, :18], torch.sigmoid(om[:, 18:27])], 1)


def dcn_ref(x, dcn_mod, bn, off, mask, fp16=False, weights="fp32"):
    """DCNv2 gather + contract + BatchNorm + ReLU on the given offsets/masks. Strict: the oracle's dcn_v2_forward in float64
    (float32 offsets keep the sampling positions and bilinear weights in float32, as the reference computes them). Fast:
    the blend of the fp16 input in float32, rounded to fp16 as the kernel stores it, fp16 weights. bn=None: the raw
    output (gather + contract + bias) a train plan normalises with batch statistics."""
    w, b = dcn_mod.weight.detach(), dcn_mod.bias.detach().double().to(x.device)
    if fp16:
        B, C, H, W = x.shape
        cols = mo.dcn_columns(x.float(), off, mask).half().double().reshape(B, C * 9, H * W)
        out = (torch.matmul(param64(w, "fp16").to(x.device).reshape(w.shape[0], -1), cols) + b.view(1, -1, 1)).view(B, -1, H, W)
    else:
        out = mo.dcn_v2_forward(x, param64(w, weights).to(x.device), b, off, mask)
    if bn is None:
        return out
    s, t = bn_fold(bn)
    return F.relu(out * s.to(x.device).view(1, -1, 1, 1) + t.to(x.device).view(1, -1, 1, 1))


def upsample_ref(x, w, f, skip=None):
    """depth-wise ConvTranspose2d(k = 2f, stride f, pad f/2) + skip in float64"""
    y = F.conv_transpose2d(x, w.detach().double().to(x.device), None, stride=f, padding=f // 2, groups=x.shape[1])
    return y if skip is None else y + skip


def channel_err(got, ref):
    """worst over images and channels of max|got_c - ref_c| / max(max|ref_c|, 0.05 max|ref|), each image on its own"""
    d = (got.double() - ref).abs().amax(dim=(2, 3))
    m = ref.abs().amax(dim=(2, 3))
    den = torch.maximum(m, 0.05 * m.amax(dim=1, keepdim=True)).clamp_min(1e-30)
    return (d / den).max().item()


def om_planes(op):
    """the DCN's recorded [M, 32] rows -> float32 offsets [B, 18, H, W], masks [B, 9, H, W] and the 27 channels"""
    x = op.x
    om = op.om.view(x.B, x.H, x.W, 32).permute(0, 3, 1, 2)
    return om[:, :18].contiguous(), om[:, 18:27].contiguous(), om[:, :27]


# ------------------------------------------------------------------------------------------------ one op
def reference(op, precision, keep_lo=True, weights=None):
    """-> {part: float64 reference} of one recorded op ('y', and 'om' for a DCN), on the weights the kernels multiply
    (see param64) unless `weights` says otherwise. keep_lo=False drops the lo halves of every pair input (the sharpness
    check)."""
    fast = precision == "fast"
    wk = weights or ("fp16" if fast else "pair")
    a = op.args
    k = op.kind
    if k in ("conv_rows_strict", "conv_rows"):
        if a.get("image") or (k == "conv_rows" and a["x"].C == 8):
            if fast:
                x = values(a["x"])[:, 0:3]
            else:
                hi, lo = image_halves(a["x"])
                x = hi + lo if keep_lo else hi
        else:
            x = values(a["x"], keep_lo)
        return {"y": conv_ref(x, a["weight"], a["stride"], a["pad"], a["bn"], engine.ACT_RELU, weights=wk)}
    x = values(a["x"], keep_lo)
    if k == "conv":
        res = values(a["residual"], keep_lo) if a["residual"] is not None else None
        return {"y": conv_ref(x, a["weight"], a["stride"], a["pad"], a["bn"], a["act"], res, weights=wk)}
    if k == "dcn":
        off, mask, _ = om_planes(op)
        mod = a["dcn_mod"]
        return {"om": offset_mask_ref(x, mod.conv_offset_mask, weights=wk),
                "y": dcn_ref(x, mod, a["bn"], off, mask, fp16=fast, weights=wk)}
    if k == "maxpool2":
        return {"y": F.max_pool2d(x, 2, 2)}
    if k == "upsample_add":
        skip = values(a["skip"], keep_lo) if a["skip"] is not None else None
        return {"y": upsample_ref(x, a["up_weight"], a["f"], skip)}
    raise AssertionError("no checker for %s" % k)


def reduction(op):
    a = op.args
    w = a.get("weight")
    if w is None and op.kind == "dcn":
        w = a["dcn_mod"].weight
    return 0 if w is None else w.shape[1] * w.shape[2] * w.shape[3]


def tolerance(op, precision):
    kind = op.kind
    if kind == "maxpool2":
        return 0.0
    if precision == "strict":
        return STRICT_DEEP_TOL if reduction(op) >= DEEP_K else STRICT_TOL
    return FAST_DCN_TOL if kind == "dcn" else FAST_CONV_TOL


def errors(op, refs):
    """{part: error} of the op's current outputs against `refs`"""
    e = {"y": channel_err(values(op.y), refs["y"])}
    if "om" in refs:
        e["om"] = channel_err(om_planes(op)[2].double(), refs["om"])
    return e


def failures(op, precision, e):
    tol = tolerance(op, precision)
    if op.kind == "maxpool2":
        return {k: v for k, v in e.items() if v != 0.0}
    om_tol = tol if precision == "strict" else FAST_CONV_TOL            # the offset/mask conv is a conv
    return {k: v for k, v in e.items() if v >= (om_tol if k == "om" else tol)}


def relaunch(plan, op):
    st = torch.cuda.current_stream().cuda_stream
    for fn, args, name in plan.launches[op.first:op.end]:
        assert fn(*args, st) == 0, name
    torch.cuda.synchronize()


def lo_block(a):
    """the view of `a`'s lo block inside its buffer (NHWC pair rows)"""
    assert a.split and not a.npar
    return a.buf.view(a.M, a.ld)[:, a.ch_off + a.lo:a.ch_off + a.lo + a.C]


# ------------------------------------------------------------------------------------------------ the plan
def label_of(model, op):
    names = {id(p): n for n, p in model.backbone.named_parameters()}
    names.update({id(m): n for n, m in model.backbone.named_modules()})
    a = op.args
    for key in ("weight", "dcn_mod", "up_weight"):
        if key in a and id(a[key]) in names:
            return names[id(a[key])].replace(".weight", "")
    if op.kind == "conv_rows_strict" or op.kind == "conv_rows":
        return "stem"
    return op.kind


def run_recorded(model, x, precision, monkeypatch):
    """build the backbone's plan for `precision` under the recorder and run it once -> (plan, ops)"""
    model.set_precision(precision)
    with monkeypatch.context() as mp:
        ops = record(mp)
        with torch.no_grad():
            model.backbone(x)
    torch.cuda.synchronize()
    plan = model.backbone.last_plan
    assert ops and all(op.plan is plan for op in ops)
    assert not plan.pack_descs and len(plan.launches) == len(plan.ops)     # launch i is plan op i
    return plan, ops


def check_plan(model, plan, ops, precision):
    """every launch covered, every activation in pair format, every op against float64 -> [(label, kind, shape, err)]"""
    names = [name for _, _, name in plan.launches]
    bad = check_coverage(ops, names, precision)
    assert not bad, bad
    print("%s plan: %d ops, %d launches, %s" % (precision, len(ops), len(names), sorted(set(names))))
    rows, fails, lost_lo = [], [], {}
    if precision == "strict":
        assert pair_format_errors(*image_halves(plan.input)) == []
    for op in ops:
        if precision == "strict":
            for a in [op.y] + op.reads:
                if a.split:
                    f = pair_format_errors(*halves(a))
                    assert not f, (label_of(model, op), f)
        refs = reference(op, precision)
        e = errors(op, refs)
        f = failures(op, precision, e)
        if f:
            fails.append((label_of(model, op), op.kind, f))
        if precision == "strict" and op.kind != "maxpool2":
            # the check can see a lost lo half: dropping them from the reference's inputs moves it by LO_MARGIN tolerances
            moved = errors_between(reference(op, precision, keep_lo=False), refs)
            lost_lo[id(op)] = min(moved.values())
            low = {k: v for k, v in moved.items() if v < LO_MARGIN * tolerance(op, precision)}
            if low:
                fails.append((label_of(model, op), op.kind, "lo halves invisible: %s" % low))
        # informational: against the fp32 weights themselves, i.e. with the floor of the pair format's weight split
        w32 = None
        if precision == "strict" and op.kind in ("conv", "conv_rows_strict", "dcn"):
            w32 = "fp32 weights %.2e lost lo %.2e tol %.1e" % (max(errors(op, reference(op, precision, weights="fp32")).values()),
                                                               lost_lo[id(op)], tolerance(op, precision))
        rows.append((label_of(model, op), op.kind, (op.y.B, op.y.C, op.y.H, op.y.W), e, w32))
    return rows, fails


def errors_between(a, b):
    return {k: channel_err(a[k], b[k]) for k in b}


def sharpness(model, plan, ops):
    """zero the lo blocks the chosen ops read on the GPU, relaunch only their launches: their checks fail by LO_MARGIN"""
    convs = [op for op in ops if op.kind == "conv" and op.args["residual"] is not None and
             any(a.ld != 2 * a.C for a in op.reads)]                      # a residual conv reading a concat slice
    ups = [op for op in ops if op.kind == "upsample_add"]
    up = max(ups, key=lambda o: o.args["f"])
    dcns = [op for op in ops if op.kind == "dcn" and op.x is up.y]           # the node DCN after the largest up-sample
    assert convs and dcns
    out = {}
    for op in (convs[0], dcns[0], up):
        refs = reference(op, "strict")
        before = errors(op, refs)
        saved = [(lo_block(a), lo_block(a).clone()) for a in op.reads]
        for blk, _ in saved:
            blk.zero_()
        relaunch(plan, op)
        lost = errors(op, refs)
        for blk, keep in saved:
            blk.copy_(keep)
        relaunch(plan, op)
        assert errors(op, refs) == before                                    # restored, bit for bit
        label = "%s (%s%s)" % (label_of(model, op), op.kind, ", f=%d" % op.args["f"] if op.kind == "upsample_add" else "")
        out[label] = lost["y"]
        assert lost["y"] >= LO_MARGIN * tolerance(op, "strict"), (label, before, lost)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_backbone_plan_launch_by_launch(shape, monkeypatch):
    t0 = time.time()
    B, H, W = shape
    model = KeypointDetector(default_cfg(width=W, height=H))
    model.load_state_dict(syn.make_state_dict(0))
    model = model.cuda().eval()
    x = syn.make_images(B, H, W).cuda()
    table, fails = {}, []
    for precision in ("strict", "fast"):
        plan, ops = run_recorded(model, x, precision, monkeypatch)
        rows, f = check_plan(model, plan, ops, precision)
        fails += [(precision,) + t for t in f]
        table[precision] = rows
        if precision == "strict":
            lost = sharpness(model, plan, ops)
        del plan, ops
        torch.cuda.empty_cache()
    model.set_precision("strict")
    print("\n%s: %d ops; worst per-channel error (strict | fast)" % ("x".join(map(str, shape)), len(table["strict"])))
    fmt = lambda e: " ".join("%s %.2e" % kv for kv in sorted(e.items()))
    for (label, kind, shp, es, w32), (_, kind_f, _, ef, _) in zip(table["strict"], table["fast"]):
        print("  %-30s %-16s %-20s %-28s | %-28s | %s" % (label, kind, shp, fmt(es), fmt(ef),
                                                          w32 or ""))
    for precision in ("strict", "fast"):
        for kind in RECORDED:
            ev = [max(e.values()) for _, k, _, e, _ in table[precision] if k == kind]
            if ev:
                print("  worst %s %-16s %.2e over %d ops" % (precision, kind, max(ev), len(ev)))
    print("  lost lo halves on the GPU: %s" % {k: "%.2e" % v for k, v in lost.items()})
    print("  wall time %.1f s" % (time.time() - t0))
    assert not fails, fails


# ------------------------------------------------------------------------------------------------ per kernel: pairs in slices
UP_CASES = [(f, C, skip) for f in (2, 4, 8) for C in (64, 128, 256) for skip in (True, False)]


def wide_rows(v, pad, split):
    """[B, C, H, W] fp32 values -> (rows buffer `pad` channels wider on each side of every block, NaN there, ch_off):
    pair rows [NaN pad | hi | NaN pad | NaN pad | lo | NaN pad] or fp16 rows [NaN pad | v | NaN pad]"""
    B, C, H, W = v.shape
    r = v.permute(0, 2, 3, 1).reshape(-1, C)
    blocks = [r.half()]
    if split:
        blocks.append((r - blocks[0].float()).half())
    buf = torch.full((r.shape[0], len(blocks) * (C + 2 * pad)), float("nan"), dtype=torch.half)
    for i, blk in enumerate(blocks):
        buf[:, i * (C + 2 * pad) + pad:i * (C + 2 * pad) + pad + C] = blk
    return buf, pad


def slice_act(v, pad, split, device="cuda"):
    buf, off = wide_rows(v, pad, split)
    B, C, H, W = v.shape
    a = engine.Act.on(buf.to(device), B, H, W, C, ch_off=off)
    a.split = split
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("split", [True, False], ids=["split", "f16"])
@pytest.mark.parametrize("f,C,skip", UP_CASES, ids=["f%d-C%d-%s" % (f, C, "skip" if s else "noskip") for f, C, s in UP_CASES])
def test_upsample_add_slices(f, C, skip, split):
    """mf_upsample_add_nhwc_f16 on pair rows and fp16 rows that are channel slices of wider buffers (different offsets
    and lo positions for x and skip, NaN in every column outside the slices), ragged 5x7 maps, against float64"""
    gen = np.random.Generator(np.random.PCG64(100 * f + C + skip))
    B, Hi, Wi = 2, 5, 7
    xv = torch.from_numpy(gen.standard_normal((B, C, Hi, Wi)).astype(np.float32))
    sv = torch.from_numpy(gen.standard_normal((B, C, Hi * f, Wi * f)).astype(np.float32))
    w = torch.from_numpy(gen.uniform(0.0, 1.0, (C, 1, 2 * f, 2 * f)).astype(np.float32))
    P = engine.Plan("cuda", strict=split)
    xa = slice_act(xv, 8, split)
    sa = slice_act(sv, 24, split) if skip else None
    ya = P.upsample_add(xa, w.cuda(), sa, f)
    P.finalize()
    P.run()
    torch.cuda.synchronize()
    ref = upsample_ref(values(xa), w, f, values(sa) if skip else None)
    if split:
        assert pair_format_errors(*halves(ya)) == []
    e = channel_err(values(ya), ref)
    print("f=%d C=%d skip=%s %s: %.2e" % (f, C, skip, "split" if split else "f16", e))
    assert e < (STRICT_TOL if split else FAST_CONV_TOL)


@pytest.mark.gpu
@pytest.mark.parametrize("C", [64, 128, 256])
def test_maxpool2_pair_slices(C):
    """mf_maxpool2_nhwc_f16 on pair rows, from one concat slice into another: bit-exact pair values, every other column
    untouched"""
    gen = np.random.Generator(np.random.PCG64(C))
    B, H, W = 2, 10, 14
    xv = torch.from_numpy(gen.standard_normal((B, C, H, W)).astype(np.float32))
    P = engine.Plan("cuda", strict=True)
    xa = slice_act(xv, 16, True)
    ya = slice_act(torch.zeros(B, C, H // 2, W // 2), 8, True)
    P.maxpool2(xa, out=ya)
    P.finalize()
    P.run()
    torch.cuda.synchronize()
    assert torch.equal(values(ya), F.max_pool2d(values(xa), 2, 2))
    assert pair_format_errors(*halves(ya)) == []
    keep = torch.ones(ya.ld, dtype=torch.bool)
    keep[8:8 + C] = False
    keep[ya.lo + 8:ya.lo + 8 + C] = False
    assert ya.buf[:, keep].isnan().all()


# ------------------------------------------------------------------------------------------------ host side
def test_pair_reading_on_synthetic_buffers():
    """halves() reads NHWC concat slices (lo at the owning buffer's half width) and both planar stem layouts exactly, and
    agrees with Act.nchw_view where that is a pure view"""
    gen = np.random.Generator(np.random.PCG64(1))
    B, H, W = 2, 3, 6
    rnd = lambda *s: torch.from_numpy(gen.standard_normal(s).astype(np.float32))
    # a concat [a (16) | b (24)] of pair rows: b's lo block starts at 40 + 16, not at 24
    a, b = rnd(B, 16, H, W), rnd(B, 24, H, W)
    buf, _ = wide_rows(torch.cat([a, b], 1), 0, True)
    act = engine.Act.on(buf, B, H, W, 24, ch_off=16)
    act.split = True
    assert act.lo == 40
    hi, lo = halves(act)
    assert torch.equal(hi, b.half().double()) and torch.equal(lo, (b - b.half().float()).half().double())
    assert pair_format_errors(hi, lo) == []
    assert torch.equal(values(act, keep_lo=False), hi)
    # planar layouts [B][H][(hi, lo) x C/8 x npar][W/npar][8]
    for npar in (1, 2):
        for split in (False, True):
            v = rnd(B, 16, H, W)
            parts = [v.half()] + ([(v - v.half().float()).half()] if split else [])
            planes = torch.stack([p.view(B, 2, 8, H, W // npar, npar).permute(0, 3, 1, 5, 4, 2) for p in parts], 2)
            pa = engine.Act(B, H, W, 16)
            pa.npar, pa.split, pa.buf = npar, split, planes.reshape(-1, 8).contiguous()
            ph, pl = halves(pa)
            assert torch.equal(ph, parts[0].double())
            assert (pl is None) == (not split) and (not split or torch.equal(pl, parts[1].double()))
            assert torch.equal(values(pa).float(), pa.nchw_view().float())
    # NHWC fp16 slice against its zero-copy view
    buf16, off = wide_rows(rnd(B, 24, H, W), 8, False)
    a16 = engine.Act.on(buf16, B, H, W, 24, ch_off=off)
    assert torch.equal(values(a16), a16.nchw_view().double())


def test_pair_format_check():
    hi = torch.tensor([1.0, -3.0, 0.0, 2.0 ** -20, 1000.0], dtype=torch.float64)
    ok = torch.tensor([2.0 ** -11, -2.0 ** -10, 0.0, 2.0 ** -25, 0.25], dtype=torch.float64)
    assert pair_format_errors(hi, ok) == []
    for i, v in ((0, 2.0 ** -10), (2, 2.0 ** -24), (4, 0.5)):
        bad = ok.clone()
        bad[i] = v
        assert pair_format_errors(hi, bad) == ["1 lo halves above ulp(hi)/2"], i
    assert "non-finite" in pair_format_errors(hi, ok * float("nan"))


def test_channel_err_sees_one_group():
    """a wrong 8-channel group at 1/10 of the tensor's range: per-channel error sees it, the tensor-wide one would not"""
    ref = torch.randn(2, 64, 5, 7, dtype=torch.float64)
    ref[:, 8:16] *= 0.1
    got = ref.clone()
    got[1, 8:16] *= 1 + 1e-4
    assert channel_err(got, ref) > 3 * STRICT_TOL
    assert ((got - ref).abs().max() / ref.abs().max()).item() < STRICT_TOL
    assert channel_err(ref, ref) == 0.0


def test_references_match_oracle():
    """the float64 references against oracle/monoflex_oracle.py (pinned to the reference by tests/test_oracle_golden.py):
    conv + BN + residual, the offset/mask conv, DCN + BN + ReLU, the up-sample + skip"""
    torch.manual_seed(0)
    B, C, H, W = 2, 16, 9, 11
    x = torch.randn(B, C, H, W, dtype=torch.float64)
    sd = {k: v.double() if v.is_floating_point() else v for k, v in syn.make_state_dict(0).items()}
    # a BasicBlock conv2 with its residual, the module parameters as stored
    m = KeypointDetector(default_cfg(width=4 * W, height=4 * H))
    m.load_state_dict(syn.make_state_dict(0))
    blk = m.backbone.base.level2.tree1
    p = "backbone.base.level2.tree1"
    xin = torch.randn(B, 64, H, W, dtype=torch.float64)
    res = torch.randn(B, 64, H, W, dtype=torch.float64)
    got = conv_ref(xin, blk.conv2.weight, 1, 1, blk.bn2, engine.ACT_RELU, res)
    want = mo.conv_bn(sd, p + ".conv2", p + ".bn2", xin, 1, 1, True, res)
    assert (got - want).abs().max().item() < 1e-12
    # DCN (offsets in float64 here, so every step is the oracle's own arithmetic)
    dc = DeformConv(C, 8)
    with torch.no_grad():
        for t in dc.parameters():
            t.copy_(torch.randn_like(t) * 0.3)
        bn = dc.actf[0]
        bn.weight.uniform_(0.5, 1.5), bn.running_mean.normal_(0, 0.1), bn.running_var.uniform_(0.5, 1.5)
    dsd = {"d." + k: v.double() for k, v in dc.state_dict().items() if v.is_floating_point()}
    om = offset_mask_ref(x, dc.conv.conv_offset_mask)
    y = dcn_ref(x, dc.conv, bn, om[:, :18], om[:, 18:27])
    assert (y - mo.deform_conv(dsd, "d", x)).abs().max().item() < 1e-12
    # fast: the fp16-stored blend is within one fp16 rounding of the exact one
    y16 = dcn_ref(x.float().half().double(), dc.conv, bn, om[:, :18].float(), om[:, 18:27].float(), fp16=True)
    assert channel_err(y16, y) < 2e-2
    # up-sample + skip, f = 4
    w = sd["backbone.ida_up.up_2.weight"]
    xu, sk = torch.randn(B, 64, 3, 5, dtype=torch.float64), torch.randn(B, 64, 12, 20, dtype=torch.float64)
    assert (upsample_ref(xu, w, 4, sk) - (mo.up(sd, "backbone.ida_up.up_2", xu, 4) + sk)).abs().max().item() < 1e-12


def test_coverage_check_finds_unchecked_launches():
    """check_coverage reports a launch no recorded op claims, and an op that emitted launches of another kind"""
    class O(object):
        def __init__(self, kind, first, end):
            self.kind, self.first, self.end, self.plan = kind, first, end, plan
    plan = engine.Plan("cpu")
    names = ["mf_conv2d_nhwc_f16x2", "mf_conv2d_nhwc_f16x2", "mf_dcn_nhwc_f16x2", "mf_maxpool2_nhwc_f16"]
    pool_args = (0, 128, 64, 0, 128, 64, 2, 10, 14, 64)        # x, x_ld, x_lo, y, y_ld, y_lo: pair rows
    plan.launches = [(None, (), n) for n in names[:3]] + [(None, pool_args, names[3])]
    ops = [O("conv", 0, 1), O("dcn", 1, 3), O("maxpool2", 3, 4)]
    assert check_coverage(ops, names, "strict") == []
    assert len(check_coverage(ops[:2], names, "strict")) == 1                       # the max-pool launch unclaimed
    assert len(check_coverage([O("conv", 0, 1), O("maxpool2", 3, 4)], names, "strict")) == 1
    assert len(check_coverage(ops, names, "fast")) == 3                              # strict launches in a fast plan
    assert check_coverage([O("new_op", 0, 4)], names, "strict") != []
    # the same launch name on fp16 rows in a strict plan, or with one lo offset missing, is reported
    for lo in ((0, 0), (64, 0)):
        plan.launches[3] = (None, pool_args[:2] + lo[:1] + pool_args[3:5] + lo[1:] + pool_args[6:], names[3])
        assert len(check_coverage(ops, names, "strict")) == 1, lo
    # ... and in a fast plan the fp16-row launch is accepted, the pair-row one reported
    fast = ["mf_conv2d_nhwc_f16", "mf_conv2d_nhwc_f16", "mf_dcn_nhwc_f16", "mf_maxpool2_nhwc_f16"]
    plan.launches[3] = (None, (0, 64, 0, 0, 64, 0, 2, 10, 14, 64), names[3])
    assert check_coverage(ops, fast, "fast") == []
    plan.launches[3] = (None, pool_args, names[3])
    assert len(check_coverage(ops, fast, "fast")) == 1
