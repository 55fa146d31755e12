"""The training forward launch by launch against float64, before and after an in-place parameter update (-m gpu, except
the host-side checks of the helpers and of the plans' launch lists).

The train-mode plans (engine.Plan(train=True)) are built from kernels the inference plans never run: raw convolutions
whose bias is copied into the epilogue's shift by an `add_py` op on every run, mf_bn_train_forward (batch statistics,
running-statistics update, fused residual and activation, issued per 256-channel chunk at `weight + 4 * off`), the head's
nine InPlaceABN modules over column slices of one 2304-wide raw buffer, the edge fusion's Conv1d + BatchNorm1d over the
B x K gathered rows, the generic 7x7 stem on the packed 8-channel image, and the batched live re-pack of every weight
(mf_pack_conv_weights_batched) that keeps a cached plan valid after the optimiser updates the parameters in place. The
whole-network loss test holds the forward to 5 % per loss term, under which a wrong chunk offset, a biased running variance
or a stale packed weight all hide; the backward's layer tests take this forward point as given.

Here every plan-builder call of both train plans (backbone and predictor) is recorded while KeypointDetector's
train_forward_losses builds them, every launch is claimed by exactly one recorded op (the weight re-pack first), and after
the forward each launch is compared with float64 computed on the GPU from the values that launch read (its fp16 input
rows, the live parameters, and the running statistics as they were before the run). The model is then updated in place,
every parameter and running buffer by ~1e-2 relative, and the same plans - not rebuilt - are run and checked again against
the new values. Errors are per image and per channel, relative to max(max|ref_c|, 0.05 max|ref|) (channel_err).

What each op is checked against, bound | worst measured on an H100 80GB HBM3 (700 W) over both shapes and both runs:
  weight re-pack      every packed weight = fp16(live parameter) in the (tap, channel) layout, zero padding  bit-exact
  refreshed copies    conv / DCN / head biases in the epilogue shift, tap-major up-sample weights = live     bit-exact
  image pack          fp16 of the image, channels 3-7 zero                                                   bit-exact
  raw conv (+ bias)   conv2d of the recorded fp16 input with fp16(W) (+ b), finite                     1e-3 | 4.9e-4
  BN statistics       mean, rstd, scale, shift from the fp16 raw rows, per 256-channel chunk           1e-5 | 1.8e-6
  running statistics  (1 - m) r0 + m (mean, var M / (M - 1)), r0 copied before the run            1.2e-6 | 4.1e-7
  BN output           act(raw scale + shift [+ residual])                                              1e-3 | 4.9e-4
  DCN                 offset/mask conv + sigmoid, fp32 rows                                          2.5e-5 | 7.3e-6
                      gather + contract on the GPU's own offsets (dcn_ref, fp16 blend), raw         1.5e-3 | 5.0e-4
                      then the BN rows above
  maxpool2            max_pool2d                                                                             bit-exact
  upsample_add        depth-wise conv_transpose2d + skip                                               1e-3 | 4.8e-4
  head 1x1            each hid slice x fp16(W) + b, fp32 NCHW                                          3e-6 | 8.7e-7
  edge gather         the kernel's fp32 grid_sample (align_corners) of hid at edge_idx, every one of the K rows
                      (zero-padded tail included), replicated into columns 0 and K + 1                        bit-exact
  edge Conv1d + BN1d  raw and BN rows as above, statistics over all B x K rows
  edge head add       cls / reg + (t w2 + b2) at k < edge_len[b] into its channels                     5e-7 | 1.4e-7
                      every other value of cls and reg unmoved                                                bit-exact
  sigmoid clamp       clamp(sigmoid(x), 1e-4, 1 - 1e-4), relative                                     5e-7 | 1.8e-7

The checks are shown to be sharp by swapping the reference, each swap failing by at least SWAP_MARGIN x the bound: the
pre-update parameters and running statistics in the second run's references (every parameterised part of every op),
the biased running variance at the edge fusion's BatchNorm1d (the smallest M), gamma instead of |gamma| + eps at a head
InPlaceABN seeded with negative gammas, the edge BatchNorm1d's statistics over the k < edge_len rows only, and the
parameters of the two 256-channel halves of a 512-channel BatchNorm swapped. Measured margins (smallest over both
shapes): stale raw convolution 10x, stale BN output 14x, stale offset/mask conv 520x, stale head / edge head 1x1
weights 3500x / 5500x, stale running statistics 1.5e4x, biased running variance 17.8x (B = 8, where M / (M - 1) - 1 is
1.5e-4), the others 2e5x or more. The file runs in about 25 s on the GPU.

Per kernel (mf_bn_train_forward against float64): M from 1 to past the 132 x 8-CTA cap, C in {8, 16, 64, 256}, input rows
wider than C with NaN neighbours, a constant channel, mean/std up to 300. The statistics are sums of d = x - x[row 0]
(csrc/mf_bn_train.cu): summed as E[x^2] - E[x]^2 in fp32 they lost ~2^-24 (mean/std)^2 of the variance, and a constant
channel kept a variance of rounding noise instead of 0 (its rstd off by up to ~1e-3 of 1/sqrt(eps)).
"""
import math
import time
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_backbone_layers import (FAST_CONV_TOL, FAST_DCN_TOL, activate, channel_err, check_coverage, conv_ref,
                                      dcn_ref, offset_mask_ref, om_planes, record, upsample_ref, values)
from monoflex_b200 import _lib, engine, synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.model.detector import KeypointDetector

# bounds: about 3x the worst value measured on an NVIDIA H100 80GB HBM3 (700 W), both shapes, both runs (given beside)
# mean, rstd, scale, shift: fp32 per-lane and per-CTA sums of (x - pivot)^2 over up to a few hundred rows; 3.1e-6 per
# kernel (M = 127 rows of 16 channels: one CTA, its 128 row lanes summed in order), 1.8e-6 in the product
STATS_TOL = 1e-5
RUNNING_TOL = 1.2e-6    # 4.1e-7: two fp32 products and a sum, and a tenth of the variance's error
OM_TOL = 2.5e-5         # 7.3e-6: the DCN offset/mask conv, fp32 rows
HEAD_TOL = 3e-6         # 8.7e-7: fp32 NCHW output, fp16 products summed over K = 256 in fp32
EDGE_ADD_TOL = 5e-7     # 1.4e-7: fp32 dot product over 256 channels + the fp32 add, relative to the updated value
SIGMOID_TOL = 5e-7      # 1.8e-7: fp32 expf and division, relative
# raw convolutions, BN outputs, up-samples: one fp16 rounding of the stored value (4.9e-4) under FAST_CONV_TOL; 5.0e-4
# (the DCN's raw output, FAST_DCN_TOL)
SWAP_MARGIN = 4         # a swapped reference must fail its check by at least this many bounds
PERTURB = 1e-2          # relative size of the in-place update between the two runs

SHAPES = [(8, 384, 1280), (3, 160, 288)]     # the bench training geometry; level 5 is 5x9, every level ragged
SHAPE_IDS = ["%dx%dx%d" % s for s in SHAPES]

TRAIN_RECORDED = ("conv", "dcn", "maxpool2", "upsample_add", "conv_to_f32", "bn_train", "add")
IN_PLACE = ("mf_edge_head_add", "mf_sigmoid_clamp")       # launches that update the predictor's cls / reg in place


def bn_chunks(slices):
    """the number of mf_bn_train_forward launches Plan.bn_train emits for `slices`"""
    return sum((c_num + 255) // 256 for _, _, c_num in slices)


def conv_slices(op):
    bn = op.args["bn"]
    return bn if isinstance(bn, list) else [(bn, 0, op.y.C)]


# the launches each recorded op of a train plan emits, in order ("__py__": a refresh of a derived copy of a parameter)
TRAIN_LAUNCHES = {
    ("conv", "train"): lambda op: ((("__py__",) if op.args["bias"] is not None else ()) + ("mf_conv2d_nhwc_f16",) +
                                   ("mf_bn_train_forward",) * bn_chunks(conv_slices(op))),
    ("dcn", "train"): ("__py__", "mf_conv2d_nhwc_f16", "__py__", "mf_dcn_nhwc_f16", "mf_bn_train_forward"),
    ("maxpool2", "train"): ("mf_maxpool2_nhwc_f16",),
    ("upsample_add", "train"): ("__py__", "mf_upsample_add_nhwc_f16"),
    ("conv_to_f32", "train"): ("__py__", "mf_conv2d_nhwc_f16"),
    ("mf_edge_gather", "train"): ("mf_edge_gather",),
    ("mf_edge_head_add", "train"): ("mf_edge_head_add",),
    ("mf_sigmoid_clamp", "train"): ("mf_sigmoid_clamp",),
}


# ------------------------------------------------------------------------------------------------ recording
def plan_ops(ops, plan):
    """the recorded top-level ops of `plan`, direct Plan.add calls named after their kernel"""
    out = []
    for op in ops:
        if op.plan is plan:
            if op.kind == "add":
                op.kind = op.args["fn_name"]
            out.append(op)
    return out


def train_coverage(plan, ops):
    """the weight re-pack is launch 0 and every other launch is claimed by exactly one recorded op -> problems"""
    names = [name for _, _, name in plan.launches]
    if not names or names[0] != "mf_pack_conv_weights_batched":
        return ["the batched weight re-pack is not the first launch: %s" % names[:1]]
    # plan op i is launch i + 1
    return check_coverage(ops, names[1:], "train", TRAIN_LAUNCHES)


def stepping_run(self):
    """Plan.run, keeping a copy of the predictor's cls / reg maps before every launch that updates them in place"""
    st = torch.cuda.current_stream().cuda_stream
    self.snaps = {}
    for i, (fn, args, name) in enumerate(self.launches):
        if name in IN_PLACE:
            self.snaps[i] = (self.cls.clone(), self.reg.clone())
        if args is None:
            fn()
        elif fn(*args, st) != 0:
            raise RuntimeError("%s failed: %s" % (name, _lib.load().mf_last_error().decode()))


# ------------------------------------------------------------------------------------------------ float64 references
def bn_train_ref(raw, gamma, beta, eps, momentum, abs_gamma, r0m, r0v, act, residual=None, rows=None):
    """training-mode BatchNorm over float64 [B, C, H, W] (statistics over B, H, W; `rows`: a 0/1 [B, 1, H, W] mask of
    the rows the statistics take, all by default) -> dict of mean, rstd, scale, shift, running mean / var, y. A single
    row keeps var = 0 for the running update, as the kernel does (torch refuses training statistics of one value)."""
    dev = raw.device
    d64 = lambda t: t.detach().double().to(dev)
    if rows is None:
        rows = torch.ones_like(raw[:, :1])
    n = rows.sum()
    mean = (raw * rows).sum((0, 2, 3)) / n
    var = (((raw - mean.view(1, -1, 1, 1)) ** 2) * rows).sum((0, 2, 3)) / n
    rstd = 1.0 / torch.sqrt(var + eps)
    g = d64(gamma)
    if abs_gamma:
        g = g.abs() + eps
    scale = g * rstd
    shift = d64(beta) - mean * scale
    unb = var * n / (n - 1) if n > 1 else var
    y = raw * scale.view(1, -1, 1, 1) + shift.view(1, -1, 1, 1)
    if residual is not None:
        y = y + residual
    return dict(mean=mean, var=var, rstd=rstd, scale=scale, shift=shift, beta=d64(beta),
                rm=(1 - momentum) * d64(r0m) + momentum * mean, rv=(1 - momentum) * d64(r0v) + momentum * unb,
                rm_size=(1 - momentum) * d64(r0m).abs() + momentum * mean.abs(), y=activate(y, act))


def running_err(rm, rv, r):
    """worst relative error of the updated running statistics, each against the size of its two terms (the running mean
    of a channel can cancel to ~0)"""
    return max(((rm.double() - r["rm"]).abs() / r["rm_size"].clamp_min(1e-30)).max().item(),
               ((rv.double() - r["rv"]).abs() / r["rv"]).max().item())


def stats_err(stats, r):
    """worst relative error of the kernel's (mean, rstd, scale, shift) [4, C], each against the size of what it is made
    of: the mean against |mean| + std, the shift against |beta| + |mean scale|"""
    s = stats.double()
    std = torch.sqrt(r["var"])
    e = [(s[0] - r["mean"]).abs() / (r["mean"].abs() + std).clamp_min(1e-30),
         (s[1] - r["rstd"]).abs() / r["rstd"],
         (s[2] - r["scale"]).abs() / r["scale"].abs().clamp_min(1e-30),
         (s[3] - r["shift"]).abs() / (r["beta"].abs() + (r["mean"] * r["scale"]).abs()).clamp_min(1e-30)]
    return max(t.max().item() for t in e)


def fp32_fma(v, w, acc):
    """fp32 fma(v, w, acc) for fp16 v and fp32 w, acc (the product is exact in float64)"""
    return (v.double() * w.double() + acc.double()).float()


def edge_gather_ref(feat, cols, edge_idx, K, ow, oh):
    """mf_edge_gather as the kernel computes it: the grid_sample coordinates of every edge index (padding_mode='replicate'
    columns 0 and K + 1 repeat the first and last index) and the bilinear corner weights in fp32, the four corners summed
    by fp32 FMAs in order, the result rounded to fp16. feat: fp16 rows [B, H, W, ld]; -> [B, 256, 1, K + 2] per column
    start in `cols`, float64."""
    B, H, W, _ = feat.shape
    e = (torch.arange(K + 2) - 1).clamp(0, K - 1)
    # the coordinates in numpy float32, whose division is IEEE like the kernel's (torch divides by a scalar through its
    # reciprocal)
    idx = edge_idx.cpu()[:, e].numpy().astype(np.float32)                 # [B, K + 2, 2] (x, y)
    f32 = np.float32
    gx = idx[..., 0] / f32(ow - 1) * f32(2) - f32(1)
    gy = idx[..., 1] / f32(oh - 1) * f32(2) - f32(1)
    ix = ((gx + f32(1)) / f32(2)) * f32(W - 1)
    iy = ((gy + f32(1)) / f32(2)) * f32(H - 1)
    x0f, y0f = np.floor(ix), np.floor(iy)
    wx1, wy1 = ix - x0f, iy - y0f
    wx0, wy0 = f32(1) - wx1, f32(1) - wy1
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(feat.device)
    x0, y0 = t(x0f.astype(np.int64)), t(y0f.astype(np.int64))
    wx0, wx1, wy0, wy1 = t(wx0), t(wx1), t(wy0), t(wy1)
    bi = torch.arange(B, device=feat.device).view(B, 1)
    out = []
    for c0 in cols:
        acc = torch.zeros(B, K + 2, 256, dtype=torch.float32, device=feat.device)
        for yy, xx, wgt in ((y0, x0, wy0 * wx0), (y0, x0 + 1, wy0 * wx1), (y0 + 1, x0, wy1 * wx0), (y0 + 1, x0 + 1, wy1 * wx1)):
            inside = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            v = feat[bi, yy.clamp(0, H - 1), xx.clamp(0, W - 1), c0:c0 + 256]
            acc = torch.where(inside[..., None], fp32_fma(v, wgt[..., None].expand_as(acc), acc), acc)
        out.append(acc.half().double().permute(0, 2, 1).unsqueeze(2))
    return out


def edge_add_ref(before, t, w2, b2, edge_idx, edge_len, ch0):
    """float64 `before` (cls or reg) + (t[b, :, 0, e] . w2[o] + b2[o]) at (b, ch0 + o, y_e, x_e) for e < edge_len[b]
    -> (reference, mask of the updated values)"""
    ref = before.double().clone()
    mask = torch.zeros_like(ref, dtype=torch.bool)
    n_out = w2.shape[0]
    for b in range(ref.shape[0]):
        n = int(edge_len[b])
        xs, ys = edge_idx[b, :n, 0], edge_idx[b, :n, 1]
        inc = (w2.double().reshape(n_out, -1) @ t[b, :, 0, :n]) + b2.double().view(-1, 1)   # [n_out, n]
        for o in range(n_out):
            ref[b, ch0 + o].index_put_((ys, xs), inc[o], accumulate=True)
            mask[b, ch0 + o, ys, xs] = True
    return ref, mask


def sigmoid_clamp_ref(x):
    return torch.sigmoid(x.double()).clamp(1e-4, 1 - 1e-4)


# ------------------------------------------------------------------------------------------------ one recorded op
class Values(object):
    """what a reference reads for a parameter or running buffer: the live tensor, or a copy taken earlier"""

    def __init__(self, copies=None):
        self.copies = copies or {}

    def __call__(self, t):
        return self.copies.get(id(t), t.detach())


def ns(mod, pv, *names):
    return types.SimpleNamespace(**{n: pv(getattr(mod, n)) for n in names})


def bn_parts(op_bn, raw64, pv, r0, res64=None, swap=None, rows=None):
    """{(c0, part): (got, ref, tol kind)} for every chunk of one recorded Plan.bn_train call. `swap`: 'biased' (running
    variance without M / (M - 1)), 'plain_gamma' (gamma for |gamma| + eps), 'halves' (the parameters of the other
    256-channel chunk of a 512-channel slice)"""
    a = op_bn.args
    out = {}
    for mod, raw, y, stats, c0, cc in op_bn.saved:
        first = [s for s in a["slices"] if s[0] is mod and s[1] <= c0 < s[1] + s[2]][0]
        off = c0 - first[1]
        if swap == "halves":
            assert first[2] == 512
            off = 256 - off
        sl = slice(off, off + cc)
        eps, m = getattr(mod, "eps", engine.BN_EPS), getattr(mod, "momentum", 0.1)
        r = bn_train_ref(raw64[:, c0:c0 + cc], pv(mod.weight)[sl], pv(mod.bias)[sl], eps, m,
                         a["abs_weight"] and swap != "plain_gamma", r0(mod.running_mean)[sl], r0(mod.running_var)[sl],
                         a["act"], None if res64 is None else res64[:, c0:c0 + cc], rows)
        if swap == "biased":
            r["rv"] = (1 - m) * r0(mod.running_var)[sl].double().to(raw64.device) + m * r["var"]
        off = c0 - first[1]
        out[(c0, "stats")] = (stats_err(stats, r), STATS_TOL)
        run = mod.running_mean[off:off + cc], mod.running_var[off:off + cc]
        out[(c0, "running")] = (running_err(run[0], run[1], r), RUNNING_TOL)
        out[(c0, "y")] = (channel_err(values(y)[:, c0:c0 + cc], r["y"]), FAST_CONV_TOL)
    return out


def check_op(op, pv, r0, swap=None):
    """{part: (error, bound)} of one recorded train-plan op against float64 on the values it read"""
    k, a = op.kind, op.args
    if k == "conv":
        raw_op = op.sub("conv")
        x = values(a["x"])
        w = a["weight"]
        w = torch.cat([pv(t) for t in w]) if isinstance(w, (list, tuple)) else pv(w)
        if x.shape[1] != w.shape[1]:                           # the packed image: 3 colour channels, zero padding
            x = x[:, :w.shape[1]]
        raw = values(raw_op.y)
        bias = pv(a["bias"]) if a["bias"] is not None else None
        ref = conv_ref(x, w, a["stride"], a["pad"], None, engine.ACT_NONE, weights="fp16", bias=bias)
        parts = {"raw": (channel_err(raw, ref) if torch.isfinite(raw).all() else math.inf, FAST_CONV_TOL)}
        rows = None
        if swap == "edge_len":
            rows = torch.zeros_like(raw[:, :1])
            for b, n in enumerate(op.plan.edge_len.tolist()):
                rows[b, :, :, :n] = 1
        res = values(a["residual"]) if a["residual"] is not None else None
        for key, v in bn_parts(op.sub("bn_train"), raw, pv, r0, res, swap, rows).items():
            parts["%s@%d" % (key[1], key[0])] = v
        return parts
    if k == "dcn":
        x = values(a["x"])
        mod = a["dcn_mod"]
        off, mask, om = om_planes(op)
        bn_op = op.sub("bn_train")
        raw = values(bn_op.args["raw"])
        parts = {"om": (channel_err(om.double(), offset_mask_ref(x, ns(mod.conv_offset_mask, pv, "weight", "bias"),
                                                                  weights="fp16")), OM_TOL),
                 "raw": (channel_err(raw, dcn_ref(x, ns(mod, pv, "weight", "bias"), None, off, mask, fp16=True,
                                                  weights="fp16")), FAST_DCN_TOL)}
        for key, v in bn_parts(bn_op, raw, pv, r0, swap=swap).items():
            parts["%s@%d" % (key[1], key[0])] = v
        return parts
    if k == "maxpool2":
        return {"y": (0.0 if torch.equal(values(op.y), F.max_pool2d(values(a["x"]), 2, 2)) else math.inf, 0.0)}
    if k == "upsample_add":
        skip = values(a["skip"]) if a["skip"] is not None else None
        return {"y": (channel_err(values(op.y), upsample_ref(values(a["x"]), pv(a["up_weight"]), a["f"], skip)),
                      FAST_CONV_TOL)}
    raise AssertionError("no checker for %s" % k)


def predictor_checks(plan, ops, pv, edge_swap=None):
    """{(label, part): (error, bound)} of the predictor's head 1x1 convs, edge gather, edge head adds and sigmoid"""
    out = {}
    names = [name for _, _, name in plan.launches]
    adds = [i for i, n in enumerate(names) if n == "mf_edge_head_add"]
    sig = names.index("mf_sigmoid_clamp")
    maps = {"cls": plan.cls, "reg": plan.reg}
    before_heads = dict(zip(("cls", "reg"), plan.snaps[adds[0]]))
    B, _, H, W = plan.cls.shape
    for op in ops:
        if op.kind == "conv_to_f32":
            a = op.args
            dst = a["out_tensor"]
            which = "cls" if dst.data_ptr() == plan.cls.data_ptr() else "reg"
            ch = (dst.data_ptr() - maps[which].data_ptr()) // (4 * H * W)
            w = pv(a["weight"])
            ref = F.conv2d(values(a["x"]), w.half().double(), pv(a["bias"]).double(), 1, 0)
            out[("head %s[%d:%d]" % (which, ch, ch + w.shape[0]), "y")] = (
                channel_err(before_heads[which][:, ch:ch + w.shape[0]], ref), HEAD_TOL)
    # edge fusion: gather, then the two branches' BN rows (checked with the convs) and their head adds
    pred = plan.pred_mod
    hid = plan.hidden
    feat = hid.buf.view(B, H, W, hid.ld)
    K = plan.edge_idx.shape[1]
    ea_ref, eb_ref = edge_gather_ref(feat, plan.edge_cols, plan.edge_idx, K, pred.output_width, pred.output_height)
    for nm, act, ref in (("ea", plan.ea, ea_ref), ("eb", plan.eb, eb_ref)):
        out[("edge gather " + nm, "y")] = (0.0 if torch.equal(values(act), ref) else
                                          (values(act) - ref).abs().max().item() + 1e-30, 0.0)
    for i, (seq, t_op, which, ch0) in enumerate(plan.edge_branches):
        before = dict(zip(("cls", "reg"), plan.snaps[adds[i]]))
        after = dict(zip(("cls", "reg"), plan.snaps[adds[i + 1]] if i + 1 < len(adds) else plan.snaps[sig]))
        t = values(t_op.y)
        ref, mask = edge_add_ref(before[which], t, pv(seq[3].weight), pv(seq[3].bias), plan.edge_idx, plan.edge_len, ch0)
        got = after[which].double()
        err = ((got - ref).abs()[mask].max() / ref.abs()[mask].max()).item()
        untouched = torch.equal(after[which][~mask], before[which][~mask])
        other = "reg" if which == "cls" else "cls"
        untouched = untouched and torch.equal(after[other], before[other])
        out[("edge head add %s[%d]" % (which, ch0), "y")] = (err, EDGE_ADD_TOL)
        out[("edge head add %s[%d]" % (which, ch0), "untouched")] = (0.0 if untouched else math.inf, 0.0)
    pre = plan.snaps[sig][0]
    ref = sigmoid_clamp_ref(pre)
    out[("sigmoid clamp", "y")] = (((plan.cls.double() - ref).abs() / ref).max().item(), SIGMOID_TOL)
    return out


def refresh_checks(plan, pv):
    """the derived copies each run refreshes, against the live parameters, bit for bit -> [problems]: every packed
    weight, every bias copied into an epilogue shift, every tap-major up-sample weight"""
    bad = []
    halves = [t for t in plan.keep if isinstance(t, torch.Tensor) and t.dtype == torch.half]
    for (src, dst, cout, cin, taps, cin_pad, n_pad, k_pad) in plan.pack_descs:
        owner = [t for t in halves if t.data_ptr() <= dst < t.data_ptr() + 2 * t.numel()]
        assert len(owner) == 1
        t = owner[0].view(-1)
        got = t[(dst - owner[0].data_ptr()) // 2:][:cout * k_pad].view(cout, k_pad)
        want = torch.zeros(cout, k_pad, dtype=torch.half, device=got.device)
        want[:, :taps * cin_pad].view(cout, taps, cin_pad)[:, :, :cin] = \
            pv(src).reshape(cout, cin, taps).permute(0, 2, 1).half()
        if not torch.equal(got, want):
            bad.append("packed weight %s" % (tuple(src.shape),))
    return bad


def shift_checks(ops, pv):
    """every bias a train plan copies into an epilogue shift (conv_to_f32, raw conv with a bias, DCN) equals the live
    parameter after the run -> [problems]"""
    bad = []

    def walk(op):
        yield op
        for s in op.subs:
            yield from walk(s)
    for top in ops:
        for op in walk(top):
            a = op.args
            pairs = []
            if op.kind in ("conv", "conv_to_f32") and a.get("bias") is not None and a.get("bn") is None:
                pairs.append((a["bias"], op))
            if op.kind == "dcn":
                pairs.append((a["dcn_mod"].bias, op))
            for bias, o in pairs:
                launch = [n for n in range(o.first, o.end) if o.plan.launches[n + 1][2] in
                          ("mf_conv2d_nhwc_f16", "mf_dcn_nhwc_f16")][-1]
                fn, args, name = o.plan.launches[launch + 1]
                ptr = args[15] if name == "mf_conv2d_nhwc_f16" else args[13]
                shift = [t for t in o.plan.keep if isinstance(t, torch.Tensor) and t.data_ptr() == ptr][0]
                if not torch.equal(shift[:bias.shape[0]], pv(bias)):
                    bad.append("%s bias %s" % (op.kind, tuple(bias.shape)))
            if op.kind == "upsample_add":
                C, k = a["up_weight"].shape[0], a["up_weight"].shape[2]
                wt = op.kept[0]
                if not torch.equal(wt, pv(a["up_weight"]).reshape(C, k * k).t()):
                    bad.append("up-sample taps %s" % (tuple(a["up_weight"].shape),))
    return bad


# ------------------------------------------------------------------------------------------------ the plans
def make_model(shape):
    B, H, W = shape
    sd = syn.make_state_dict(0)
    # negative InPlaceABN gammas in the class head: the kernels must use |gamma| + eps there
    g = sd["heads.predictor.class_head.1.weight"]
    g[::3] = -g[::3]
    model = KeypointDetector(default_cfg(width=W, height=H))
    model.load_state_dict(sd)
    model = model.cuda().train()
    fields = syn.make_train_targets(B, out_w=W // 4, out_h=H // 4, empty_image=1 if B > 1 else -1)
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields, out_w=W // 4, out_h=H // 4)]
    # a shorter border list on the last image: edge_len differs between images
    n = int(targets[-1].get_field("edge_len"))
    targets[-1].add_field("edge_len", torch.tensor(n - 37, dtype=torch.long, device="cuda"))
    images = syn.make_images(B, H, W, seed=2).cuda()
    return model, images, targets


def running_copies(model):
    return Values({id(t): t.detach().clone() for t in model.buffers() if t.is_floating_point()})


def forward_recorded(model, images, targets, monkeypatch):
    """train_forward_losses with the recorder and the stepping run -> (recorded ops, running statistics before the run)"""
    r0 = running_copies(model)
    with monkeypatch.context() as mp:
        ops = record(mp, TRAIN_RECORDED)
        mp.setattr(engine.Plan, "run", stepping_run)
        with torch.no_grad():
            model.train_forward_losses(images, targets)
    torch.cuda.synchronize()
    return ops, r0


def annotate_predictor(model, plan, ops):
    """what predictor_checks needs to find in the plan: the predictor, the gathered columns, the edge branches"""
    pred = model.heads.predictor
    plan.pred_mod = pred
    plan.edge_cols = (0, (pred.offset_index[0] + 1) * pred.head_conv)
    convs = [op for op in ops if op.kind == "conv" and op.args["x"] in (plan.ea, plan.eb)]
    assert len(convs) == 2
    plan.edge_branches = [(pred.trunc_heatmap_conv, convs[0], "cls", 0),
                          (pred.trunc_offset_conv, convs[1], "reg", plan.ctx["off_ch0"])]


def label_of(names, op):
    a = op.args
    w = a.get("weight", a.get("dcn_mod", a.get("up_weight")))
    if isinstance(w, list):
        return "head 3x3"
    return names.get(id(w), "#%d" % op.first).replace(".weight", "")


def check_all(model, images, plans, pv, r0, tag):
    """every op of both plans -> ({(group, label, part): (error, bound)}, [problems])"""
    res, bad = {}, []
    (bplan, bops), (pplan, pops) = plans
    names = {id(m): n for n, m in model.named_modules()}
    names.update({id(p): n for n, p in model.named_parameters()})
    # the image pack, outside the launch list
    x8 = values(bplan.input)
    if not (torch.equal(x8[:, :3], images.half().double()) and not x8[:, 3:].any()):
        bad.append("%s: image pack" % tag)
    bad += ["%s: %s" % (tag, b) for b in refresh_checks(bplan, pv) + refresh_checks(pplan, pv)]
    bad += ["%s: %s" % (tag, b) for b in shift_checks(bops + pops, pv)]
    for plan, ops in plans:
        for op in ops:
            if op.kind in ("conv", "dcn", "maxpool2", "upsample_add"):
                for part, v in check_op(op, pv, r0).items():
                    res[(op.kind, "%s @%d" % (label_of(names, op), op.first), part)] = v
    for (label, part), v in predictor_checks(pplan, pops, pv).items():
        res[(label.split("[")[0], label, part)] = v
    for key, (e, tol) in res.items():
        if not e <= tol:
            bad.append("%s: %s %s %s %.3e > %.1e" % (tag, key[0], key[1], key[2], e, tol))
    return res, bad


def summarize(res, tag):
    worst = {}
    for (group, label, part), (e, tol) in res.items():
        kind = group + " " + part.split("@")[0]
        if e > worst.get(kind, (-1, 0, ""))[0]:
            worst[kind] = (e, tol, label)
    print("\n%s: worst error per check (bound)" % tag)
    for kind, (e, tol, label) in sorted(worst.items()):
        print("  %-28s %.3e (%.1e) at %s" % (kind, e, tol, label))


def margin(parts, keys=None):
    """the largest error / bound over the chosen parts"""
    return max(e / tol for k, (e, tol) in parts.items() if keys is None or k.split("@")[0] in keys)


def perturb(model, seed):
    """the in-place update between the runs: every parameter and running buffer times (1 + PERTURB n), same storage"""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    with torch.no_grad():
        for t in list(model.parameters()) + [b for b in model.buffers() if b.is_floating_point()]:
            ptr = t.data_ptr()
            t.mul_(1 + PERTURB * torch.randn(t.shape, generator=gen, device=t.device))
            assert t.data_ptr() == ptr


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_train_forward_launch_by_launch(shape, monkeypatch):
    t0 = time.time()
    model, images, targets = make_model(shape)
    ops, r0 = forward_recorded(model, images, targets, monkeypatch)
    bplan, pplan = model.backbone.last_plan, model.heads.predictor.last_plan
    bops, pops = plan_ops(ops, bplan), plan_ops(ops, pplan)
    assert len(bops) + len(pops) == len(ops)
    annotate_predictor(model, pplan, pops)
    # 1. every launch claimed, the re-pack first, one BN launch per 256-channel chunk
    for plan, pl_ops in ((bplan, bops), (pplan, pops)):
        bad = train_coverage(plan, pl_ops)
        assert not bad, bad
        for op in pl_ops:
            if op.kind == "conv":
                assert [n for _, _, n in plan.launches[op.first + 1:op.end + 1]].count("mf_bn_train_forward") == \
                    bn_chunks(conv_slices(op))
    assert sum(1 for op in bops if op.kind == "conv" and op.y.C == 512) > 0
    print("\n%s: backbone %d ops / %d launches, predictor %d ops / %d launches" % (
        "x".join(map(str, shape)), len(bops), len(bplan.launches), len(pops), len(pplan.launches)))
    plans = ((bplan, bops), (pplan, pops))
    live = Values()
    # 2. run 1
    res1, bad = check_all(model, images, plans, live, r0, "run 1")
    summarize(res1, "run 1")
    assert not bad, bad
    # 3. the in-place "optimiser step", run 2 on the same plans
    old = Values({id(t): t.detach().clone() for t in list(model.parameters()) + list(model.buffers())
                  if t.is_floating_point()})
    perturb(model, 7)
    ops2, r0_2 = forward_recorded(model, images, targets, monkeypatch)
    assert ops2 == [] and model.backbone.last_plan is bplan and model.heads.predictor.last_plan is pplan
    res2, bad = check_all(model, images, plans, live, r0_2, "run 2")
    summarize(res2, "run 2")
    assert not bad, bad
    # 4. sharpness: each swapped reference fails by SWAP_MARGIN bounds
    margins, weak = {}, []
    for plan, pl_ops in plans:
        for op in pl_ops:
            if op.kind in ("conv", "dcn", "upsample_add"):
                parts = check_op(op, old, old)
                for part in parts:
                    if part.split("@")[0] in ("raw", "om", "y", "running"):
                        m = parts[part][0] / parts[part][1]
                        margins.setdefault("stale " + part.split("@")[0], []).append(m)
                        if m < SWAP_MARGIN:
                            weak.append(("stale parameters", op.kind, op.first, part, m))
    for (label, part), (e, tol) in predictor_checks(pplan, pops, old).items():
        if label.startswith(("head", "edge head add")) and part == "y":
            margins.setdefault("stale " + label.split("[")[0].rsplit(" ", 1)[0], []).append(e / tol)
            if e / tol < SWAP_MARGIN:
                weak.append(("stale parameters", label, e / tol))
    edge_bn = [b for _, b, _, _ in pplan.edge_branches]
    head = [op for op in pops if op.kind == "conv" and isinstance(op.args["weight"], list)][0]
    wide = [op for op in bops if op.kind == "conv" and op.y.C == 512][0]
    swaps = {"biased running variance (edge BatchNorm1d)": margin(check_op(edge_bn[0], live, r0_2, "biased"), ("running",)),
             "gamma for |gamma| + eps (class head)": margin(check_op(head, live, r0_2, "plain_gamma")),
             "statistics over k < edge_len (edge BatchNorm1d)": margin(check_op(edge_bn[0], live, r0_2, "edge_len")),
             "chunk parameters swapped (512-channel BN)": margin(check_op(wide, live, r0_2, "halves"))}
    for k, v in margins.items():
        swaps[k + " (min over ops)"] = min(v)
    print("  swapped references, error / bound: %s" % {k: "%.1f" % v for k, v in swaps.items()})
    print("  wall time %.1f s" % (time.time() - t0))
    assert not weak, weak
    assert all(v >= SWAP_MARGIN for v in swaps.values()), swaps


# ------------------------------------------------------------------------------------------------ per kernel: BatchNorm edges
def bn_case_list():
    cases = []
    for C in (8, 16, 64, 256):
        RL = 256 // (C // 8)
        for M in sorted({1, 7, RL - 1, 4 * RL + 1, 1056 * 4 * RL, 1056 * 4 * RL + 1}):
            cases.append((M, C, 1))
    cases += [(245760, 64, r) for r in (0, 1, 10, 30, 300)]
    return cases


BN_CASES = bn_case_list()


def bn_kernel_inputs(M, C, ratio, seed):
    """fp16 rows [M, C + 16] with the C channels at column 8 and NaN around them; channel 0 constant; the others
    mean = ratio x std; gamma (some negative), beta, running statistics; residual rows like x"""
    gen = np.random.Generator(np.random.PCG64(seed))
    std = 0.25 * gen.uniform(0.5, 2.0, C)
    v = (gen.standard_normal((M, C)) + ratio) * std
    v[:, 0] = 0.3
    x = torch.full((M, C + 16), float("nan"), dtype=torch.half)
    x[:, 8:8 + C] = torch.from_numpy(v.astype(np.float32)).half()
    res = torch.full((M, C + 16), float("nan"), dtype=torch.half)
    res[:, 8:8 + C] = torch.from_numpy(gen.standard_normal((M, C)).astype(np.float32)).half()
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    gamma = t(gen.uniform(0.5, 1.5, C) * np.where(np.arange(C) % 5 == 2, -1, 1))
    beta = t(gen.standard_normal(C) * 0.1)
    beta[0] = 0.25
    return x, res, gamma, beta, t(gen.standard_normal(C) * 0.1), t(gen.uniform(0.5, 1.5, C))


def run_bn_kernel(x, res, gamma, beta, rm, rv, M, C, act, abs_gamma, eps=1e-5, momentum=0.1):
    """mf_bn_train_forward on the column-8 slices -> (y rows [M, C + 16] (NaN outside the slice unless written), stats)"""
    y = torch.full_like(x, float("nan"))
    stats = torch.empty(4, C, dtype=torch.float32, device=x.device)
    ws = torch.empty(max(1, _lib.load().mf_bn_train_workspace(M, C) // 4), dtype=torch.float32, device=x.device)
    ld = C + 16
    _lib.call("mf_bn_train_forward", x.data_ptr() + 16, ld, M, C, gamma.data_ptr(), beta.data_ptr(), eps, momentum,
              abs_gamma, rm.data_ptr(), rv.data_ptr(), None if res is None else res.data_ptr() + 16, ld, act,
              y.data_ptr() + 16, ld, stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), stats[3].data_ptr(),
              ws.data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    return y, stats


def fp16_ulp(v):
    """the spacing of fp16 values at |v| (float64), subnormals included"""
    m = v.abs().half()
    return (m.view(torch.int16) + 1).view(torch.float16).double() - m.double()


@pytest.mark.gpu
@pytest.mark.parametrize("M,C,ratio", BN_CASES, ids=["M%d-C%d-r%d" % c for c in BN_CASES])
def test_bn_train_forward_edges(M, C, ratio):
    """mf_bn_train_forward against float64 at the row-count edges of its CTA split (1 row, fewer rows than one CTA's row
    lanes, one CTA's 4 x RL row group + 1, exactly the 132 x 8-CTA cap and one row past it, where a CTA's slab doubles),
    on rows wider than C whose neighbouring columns are NaN (never read, never written), with a constant channel and
    mean/std up to 300"""
    i = BN_CASES.index((M, C, ratio))
    act, with_res, abs_gamma = i % 3, i % 2 == 0, int(i % 4 == 1)
    x, res, gamma, beta, rm0, rv0 = [t.cuda() for t in bn_kernel_inputs(M, C, ratio, 1000 + i)]
    rm, rv = rm0.clone(), rv0.clone()
    y, stats = run_bn_kernel(x, res if with_res else None, gamma, beta, rm, rv, M, C, act, abs_gamma)
    raw = x[:, 8:8 + C].double().t().reshape(1, C, M, 1)
    r64 = res[:, 8:8 + C].double().t().reshape(1, C, M, 1) if with_res else None
    r = bn_train_ref(raw, gamma, beta, 1e-5, 0.1, abs_gamma, rm0, rv0, act, r64)
    got_y = y[:, 8:8 + C].double().t().reshape(1, C, M, 1)
    e = dict(stats=stats_err(stats, r), running=running_err(rm, rv, r),
             y=channel_err(got_y, r["y"]))
    print("M=%d C=%d mean/std=%d act=%d res=%d abs=%d: %s" % (M, C, ratio, act, with_res, abs_gamma,
                                                             {k: "%.2e" % v for k, v in e.items()}))
    assert e["stats"] <= STATS_TOL and e["running"] <= RUNNING_TOL and e["y"] <= FAST_CONV_TOL, e
    # the columns around the slice: never written
    assert y[:, :8].isnan().all() and y[:, 8 + C:].isnan().all()
    # the constant channel: var = 0 exactly, so mean = its value, rstd = 1/sqrt(eps) and running_var = (1 - m) r0 in fp32;
    # y is act(beta [+ residual]) within one fp16 ulp, plus - with a residual, whose sum can be far smaller than beta -
    # the fp32 rounding of x scale and shift, which round separately (so the result is not bit for bit)
    rstd0 = np.float32(1.0 / math.sqrt(float(np.float32(1e-5))))
    assert stats[1, 0].item() == rstd0 and stats[0, 0].item() == float(x[0, 8])
    assert rv[0].item() == float(np.float32(np.float32(1 - np.float32(0.1)) * np.float32(rv0[0].item())))
    want0 = activate(r["beta"][0] + (r64[0, 0] if with_res else 0.0), act)
    slack = 2.0 ** -22 * abs(float(x[0, 8]) * stats[2, 0].item()) if with_res else 0.0
    assert ((got_y[0, 0] - want0).abs() <= fp16_ulp(want0) + slack).all()
    if M == 1:
        # torch refuses training statistics of one value per channel; the kernel takes var = 0 for the running update too
        # (checked above against bn_train_ref, which does the same)
        with pytest.raises(ValueError):
            F.batch_norm(torch.zeros(1, C, 1, 1), torch.zeros(C), torch.ones(C), training=True)
        assert torch.equal(r["var"], torch.zeros_like(r["var"]))


# ------------------------------------------------------------------------------------------------ host side
def test_bn_train_ref_matches_torch():
    """bn_train_ref against torch's training-mode batch_norm (float64, CPU): output, running statistics, |gamma| + eps"""
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(3, 16, 5, 7, generator=gen, dtype=torch.float64) * 2 + 1
    res = torch.randn(3, 16, 5, 7, generator=gen, dtype=torch.float64)
    g, b = torch.randn(16, generator=gen, dtype=torch.float64), torch.randn(16, generator=gen, dtype=torch.float64)
    rm, rv = torch.randn(16, generator=gen, dtype=torch.float64), torch.rand(16, generator=gen, dtype=torch.float64) + 0.5
    for abs_gamma in (0, 1):
        for act in (engine.ACT_NONE, engine.ACT_RELU, engine.ACT_LEAKY):
            rm_t, rv_t = rm.clone(), rv.clone()
            gw = g.abs() + 1e-5 if abs_gamma else g
            want = activate(F.batch_norm(x, rm_t, rv_t, gw, b, True, 0.1, 1e-5) + res, act)
            r = bn_train_ref(x, g, b, 1e-5, 0.1, abs_gamma, rm, rv, act, res)
            assert (r["y"] - want).abs().max().item() < 1e-12
            assert (r["rm"] - rm_t).abs().max().item() < 1e-14 and (r["rv"] - rv_t).abs().max().item() < 1e-14
    # a row mask selects the statistics' rows
    rows = torch.zeros(3, 1, 5, 7, dtype=torch.float64)
    rows[:, :, :, :4] = 1
    r = bn_train_ref(x, g, b, 1e-5, 0.1, 0, rm, rv, engine.ACT_NONE, rows=rows)
    assert torch.allclose(r["mean"], x[..., :4].mean((0, 2, 3)), atol=1e-14, rtol=0)
    # one row: var = 0 for the running update
    r = bn_train_ref(x[:1, :, :1, :1], g, b, 1e-5, 0.1, 0, rm, rv, engine.ACT_NONE)
    assert torch.equal(r["var"], torch.zeros(16, dtype=torch.float64)) and torch.allclose(r["rv"], 0.9 * rv)


def test_stats_err_sees_each_statistic():
    C = 8
    r = dict(mean=torch.full((C,), 3.0, dtype=torch.float64), var=torch.full((C,), 0.25, dtype=torch.float64),
             rstd=torch.full((C,), 2.0, dtype=torch.float64), scale=torch.full((C,), 1.5, dtype=torch.float64),
             shift=torch.full((C,), -4.4, dtype=torch.float64), beta=torch.full((C,), 0.1, dtype=torch.float64))
    exact = torch.stack([r["mean"], r["rstd"], r["scale"], r["shift"]]).float()
    assert stats_err(exact, r) < 1e-7
    for row in range(4):
        s = exact.clone()
        s[row, 5] *= 1 + 1e-4
        assert stats_err(s, r) > 2e-5, row


def test_edge_gather_ref_is_grid_sample():
    """edge_gather_ref against F.grid_sample(align_corners=True) on the reference's normalised coordinates, replicate
    columns included, to fp16 rounding; integer coordinates that survive the fp32 round trip read one pixel exactly"""
    B, H, W, ld, K = 2, 6, 9, 24, 5
    gen = torch.Generator().manual_seed(4)
    feat = (torch.randn(B, H, W, ld, generator=gen) * 3).half()
    feat = torch.cat([feat] * 11, 3)[..., :264]                           # 256 channels from column 8
    idx = torch.stack([torch.randint(0, W, (B, K), generator=gen), torch.randint(0, H, (B, K), generator=gen)], 2)
    [got] = edge_gather_ref(feat, (8,), idx, K, W, H)
    grid = idx.double().view(B, K, 1, 2).clone()
    grid[..., 0] = grid[..., 0] / (W - 1) * 2 - 1
    grid[..., 1] = grid[..., 1] / (H - 1) * 2 - 1
    fmap = feat[..., 8:264].double().permute(0, 3, 1, 2)
    want = F.grid_sample(fmap, grid, align_corners=True).squeeze(-1)          # [B, 256, K]
    want = torch.cat([want[..., :1], want, want[..., -1:]], 2).unsqueeze(2)
    assert ((got - want).abs() <= fp16_ulp(want)).all()


def test_edge_add_ref():
    B, C, H, W, K = 2, 5, 4, 8, 7
    before = torch.randn(B, C, H, W, dtype=torch.float64)
    t = torch.randn(B, 256, 1, K, dtype=torch.float64)
    w2, b2 = torch.randn(2, 256, 1, dtype=torch.float64), torch.randn(2, dtype=torch.float64)
    idx = torch.tensor([[[x, y] for x, y in zip(range(K), [0, 1, 2, 3, 3, 2, 1])]] * B)
    ln = torch.tensor([K, 3])
    ref, mask = edge_add_ref(before, t, w2, b2, idx, ln, 2)
    assert int(mask.sum()) == 2 * (K + 3) and torch.equal(ref[~mask], before[~mask])
    assert torch.allclose(ref[1, 3, 2, 2], before[1, 3, 2, 2] + w2[1, :, 0] @ t[1, :, 0, 2] + b2[1])
    assert torch.equal(ref[1, 3, 3, 3], before[1, 3, 3, 3])                 # k = 3 >= edge_len[1]


def _cpu_train_plans(H=64, W=128, B=2):
    """both train plans of a KeypointDetector built on the CPU under the recorder (built, never run)"""
    model = KeypointDetector(default_cfg(width=W, height=H))
    model.load_state_dict(syn.make_state_dict(0))
    model.train()
    mp = pytest.MonkeyPatch()
    try:
        ops = record(mp, TRAIN_RECORDED)
        bplan = model.backbone.build_plan(B, H, W, "cpu")
        pplan = model.heads.predictor.build_plan(bplan.output, 2 * (W // 4 + H // 4))
    finally:
        mp.undo()
    return model, bplan, pplan, plan_ops(ops, bplan), plan_ops(ops, pplan)


def test_train_plans_launch_lists():
    """host side: every launch of both train plans is claimed by exactly one recorded op (the weight re-pack first), with
    one BN launch per 256-channel chunk: the 512-channel level-5 convs two, the head's nine InPlaceABN slices nine"""
    model, bplan, pplan, bops, pops = _cpu_train_plans()
    assert train_coverage(bplan, bops) == [] and train_coverage(pplan, pops) == []
    chunks = sorted({bn_chunks(conv_slices(op)) for op in bops + pops if op.kind == "conv"})
    assert chunks == [1, 2, 9], chunks
    kinds = sorted({op.kind for op in pops})
    assert kinds == ["conv", "conv_to_f32", "mf_edge_gather", "mf_edge_head_add", "mf_sigmoid_clamp"], kinds
    # the generic 7x7 stem on the 8-channel packed image, never the row-segment stem
    assert bops[0].kind == "conv" and bops[0].args["cin_pad"] == 8 and bops[0].args["x"] is bplan.input
    # a dropped or an extra launch is reported
    bplan.launches.insert(5, bplan.launches[5])
    assert train_coverage(bplan, bops) != []
    del bplan.launches[5]
    assert train_coverage(bplan, bops) == []
    bplan.launches.append(bplan.launches.pop(0))
    assert train_coverage(bplan, bops) != []
