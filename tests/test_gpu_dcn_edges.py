"""-m gpu: the deformable-convolution kernels at their sampling edges, against the float64 reference of tests/dcn_ref.py
(pinned to the reference's own C loops by tests/test_dcn_edges_host.py). Offsets and masks come from the edge menu
(dcn_ref.edge_menu: samples on the grid, exactly on and just inside the border, far outside, 1e-8 off the grid) or from the
reference's initialisation of the offset conv (all zero), and are written straight into the kernels' offset/mask rows.

  a  zero offset conv (DCN.init_offset): offsets exactly 0, masks exactly 0.5, DCN = 3x3 conv with 0.5 W (fast, strict, train)
  b  column readout: one-hot weights make the fused DCN return its sampled operand, compared element by element
  c  contraction on the edge menu, x and y channel slices of wider buffers
  d  the model's DCN layer shapes at 384x1280, taken from the backbone plan
  e  the fp16 training backward (backward.dcn_backward and the tape's slice call form)
  f  the exact-fp32 operator pair behind dcn_v2.py (_ext.dcn_v2_forward / dcn_v2_backward)
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcn_ref
from gpu_util import FakeBN, to_rows, to_rows_split
from monoflex_b200 import engine
from monoflex_b200._lib import call, stream

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                     # float32 unit roundoff
FAST_TOL, STRICT_TOL = 1.5e-3, 3e-5
MAGNITUDES = (1.0, 2.0, 0.5)       # image b is filled at MAGNITUDES[b]: a sample read from the wrong image shows up


def h16(t):
    return t.half().float()


def images(gen, B, C, H, W):
    x = torch.from_numpy(gen.standard_normal((B, C, H, W)).astype(np.float32))
    return x * torch.tensor(MAGNITUDES[:B] if B <= 3 else [1.0] * B).view(B, 1, 1, 1)


def nchw(rows, B, H, W):
    return rows.reshape(B, H, W, -1).permute(0, 3, 1, 2)


def rows16(x):
    """[B, C, H, W] -> fp16 pixel rows [B*H*W, C] on the tensor's device"""
    return x.permute(0, 2, 3, 1).reshape(-1, x.shape[1]).half().contiguous()


def pair_value(rows, C, lo):
    """hi + lo of pair rows (hi channels [0, C), lo channels [lo, lo + C)) in float64"""
    return rows[:, :C].double() + rows[:, lo:lo + C].double()


def worst(got, want, err=None):
    """where the largest error is, for assertion messages"""
    err = (got.double() - want.double()).abs() if err is None else err
    err = torch.nan_to_num(err, nan=float("inf"))
    i = int(err.argmax())
    at = np.unravel_index(i, tuple(err.shape))
    return "worst at %s: got %r want %r (err %.3e)" % (tuple(int(a) for a in at), got.reshape(-1)[i].item(),
                                                      want.reshape(-1)[i].item(), err.reshape(-1)[i].item())


def rel(got, want):
    got, want = got.double(), want.double()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def ulp16(v):
    """spacing of fp16 at |v| (2^-24 in the subnormal range)"""
    e = torch.floor(torch.log2(v.abs().double().clamp_min(2.0 ** -14)))
    return torch.pow(2.0, e - 10)


class _Mod(object):
    pass


def dcn_module(gen, cin, cout, off_scale=1.5, fp16=False):
    d = _Mod()
    q = h16 if fp16 else (lambda t: t)
    d.weight = q(torch.from_numpy((gen.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32))).cuda()
    d.bias = torch.from_numpy((gen.standard_normal(cout) * 0.1).astype(np.float32)).cuda()
    d.conv_offset_mask = _Mod()
    d.conv_offset_mask.weight = q(torch.from_numpy(
        (gen.standard_normal((27, cin, 3, 3)) * off_scale / np.sqrt(9 * cin)).astype(np.float32))).cuda()
    d.conv_offset_mask.bias = torch.from_numpy((gen.standard_normal(27) * 0.2).astype(np.float32)).cuda()
    return d


def bn_eval64(y, bn, bias):
    """eval BatchNorm after the conv bias, float64"""
    s = bn.weight.double() / torch.sqrt(bn.running_var.double() + bn.eps)
    return (y + bias.double().view(1, -1, 1, 1) - bn.running_mean.double().view(1, -1, 1, 1)) * s.view(1, -1, 1, 1) + \
        bn.bias.double().view(1, -1, 1, 1)


# ----------------------------------------------------------------------------------------------------------- a
@pytest.mark.parametrize("mode", ["fast", "strict", "train"])
def test_reference_init_gives_exact_offmask_and_half_weight_conv(mode):
    """DCN's constructor zeroes conv_offset_mask (the reference's init_offset, dcn_v2.py:114-116): the offset conv must
    produce offsets of exactly 0 and masks of exactly 0.5, and the DCN must then be a plain 3x3 conv with 0.5 W."""
    from monoflex_b200.model.backbone.DCNv2.dcn_v2 import DCN
    B, Cin, Cout, H, W = 2, 128, 64, 13, 41
    gen = np.random.Generator(np.random.PCG64(1))
    mod = DCN(Cin, Cout, (3, 3), stride=1, padding=1).cuda()
    with torch.no_grad():
        mod.weight.copy_(h16(torch.from_numpy((gen.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(9 * Cin)).astype(np.float32))))
        mod.bias.copy_(torch.from_numpy((gen.standard_normal(Cout) * 0.1).astype(np.float32)))
    assert mod.conv_offset_mask.weight.abs().sum().item() == 0 and mod.conv_offset_mask.bias.abs().sum().item() == 0
    x = images(gen, B, Cin, H, W)
    bn = torch.nn.BatchNorm2d(Cout).cuda() if mode == "train" else FakeBN(Cout, gen)
    P = engine.Plan("cuda", strict=mode == "strict", train=mode == "train")
    xa = P.act(B, H, W, Cin)
    ya = P.dcn(xa, mod, bn)
    P.finalize()
    xa.buf.copy_(to_rows_split(x) if mode == "strict" else to_rows(x))
    P.run()
    torch.cuda.synchronize()
    om = P.tape[-1]["om"] if mode == "train" else P.keep[0]
    assert torch.equal(om[:, :18], torch.zeros_like(om[:, :18])), (mode, worst(om[:, :18], torch.zeros_like(om[:, :18])))
    half = torch.full_like(om[:, 18:27], 0.5)
    assert torch.equal(om[:, 18:27], half), (mode, worst(om[:, 18:27], half))
    xv = xa.nchw_view().double()
    conv = F.conv2d(xv, 0.5 * mod.weight.detach().double(), None, padding=1)
    if mode == "train":
        raw = P.tape[-1]["raw"]                                   # the DCN output before the batch-statistics BN
        ref = conv + mod.bias.detach().double().view(1, -1, 1, 1)
        got = raw.nchw_view().double()
        assert rel(got, ref) < FAST_TOL, (mode, rel(got, ref), worst(got, ref))
        return
    ref = F.relu(bn_eval64(conv, bn, mod.bias.detach()))
    got = ya.nchw_view().double()
    tol = STRICT_TOL if mode == "strict" else FAST_TOL
    assert rel(got, ref) < tol, (mode, rel(got, ref), worst(got, ref))


# ----------------------------------------------------------------------------------------------------------- b
def readout_selection(cin):
    """576 (tap, channel) pairs, 64 per tap; at every tap the channels cover every 64-channel chunk of Cin"""
    n = torch.arange(576)
    tap, j, g = n // 64, n % 64, cin // 64
    return tap, j * g + (7 * j + 13 * tap) % g


def one_hot_weights(cin):
    tap, c = readout_selection(cin)
    w = torch.zeros(576, cin, 3, 3)
    w[torch.arange(576), c, tap // 3, tap % 3] = 1.0
    return w


@pytest.mark.parametrize("hw", [(1, 1), (1, 17), (9, 15), (8, 16), (13, 41)])
@pytest.mark.parametrize("cin", [64, 128, 256, 512])
def test_column_readout(cin, hw):
    """one-hot weights (output n = column (tap_n, c_n)), scale 1, shift 0, no activation: the fused DCN returns its sampled
    operand itself, which is compared element by element with float64 on the edge menu (3 images at different magnitudes,
    maps ragged against the 8 x 16 pixel tile)."""
    B, (H, W) = 3, hw
    M = B * H * W
    gen = np.random.Generator(np.random.PCG64(cin + 100 * H + W))
    x = images(gen, B, cin, H, W)
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=cin + H * W)
    offset, mask = offset.cuda(), mask.cuda()
    om = dcn_ref.to_offmask_rows(offset, mask)
    tap, c = readout_selection(cin)
    tap, c = tap.cuda(), c.cuda()
    w = one_hot_weights(cin).cuda()
    P = engine.Plan("cuda")

    def select(cols64):                                         # [B, C, 9, H, W] -> rows [M, 576]
        return cols64[:, c, tap].permute(0, 2, 3, 1).reshape(M, 576)

    # fast: fp16 activations, one fp16 product
    xr = to_rows(x)
    wp, n_pad, k_pad = P.pack_weight(w)
    scale, shift = P.affine(576, n_pad)                          # identity epilogue
    y = torch.full((M, 576), float("nan"), dtype=torch.half, device="cuda")
    call("mf_dcn_nhwc_f16", xr.data_ptr(), cin, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, 576,
         scale.data_ptr(), shift.data_ptr(), engine.ACT_NONE, engine.OUT_F16_NHWC, y.data_ptr(), 576, stream())
    cols = torch.empty(M, 9 * cin, dtype=torch.half, device="cuda")
    call("mf_dcn_sample_cols_nhwc_f16", xr.data_ptr(), cin, om.data_ptr(), 32, cols.data_ptr(), B, H, W, cin, stream())
    torch.cuda.synchronize()
    ref, absum = dcn_ref.columns(nchw(xr, B, H, W).double(), offset, mask, with_abs=True)
    ref, absum = select(ref), select(absum)
    # the blend runs in fp32 (three roundings in a corner weight, four in the sum: < 8 u of the sum of |terms|), then
    # rounds once to fp16: within one fp16 ulp of fp16(exact) plus the fp32 part
    r16 = ref.half().double()
    err = (y.double() - r16).abs()
    bound = torch.maximum(ulp16(r16), ulp16(y)) + 8 * U * absum
    assert (err <= bound).all(), ("fast", cin, hw, worst(y, ref, err - bound))
    # the dW operand of the training backward: same rounding points as the fused producer (signed zeros compare equal)
    sampled = cols[:, tap * cin + c]
    same = sampled.float() == y.float()
    assert same.all(), ("sample_cols vs fused producer", cin, hw, worst(sampled, y))

    # strict: hi/lo pairs, three products
    xs = to_rows_split(x)
    wp2, n_pad2, k_pad2 = P.pack_weight(w, split=True)
    scale, shift = P.affine(576, n_pad2)
    y2 = torch.full((M, 1152), float("nan"), dtype=torch.half, device="cuda")
    call("mf_dcn_nhwc_f16x2", xs.data_ptr(), 2 * cin, cin, B, H, W, cin, om.data_ptr(), 32, wp2.data_ptr(), n_pad2, k_pad2,
         576, scale.data_ptr(), shift.data_ptr(), engine.ACT_NONE, y2.data_ptr(), 1152, 576, stream())
    torch.cuda.synchronize()
    xv = nchw(pair_value(xs, cin, cin), B, H, W)
    ref, absum = dcn_ref.columns(xv, offset, mask, with_abs=True)
    ref, absum = select(ref), select(absum)
    got = pair_value(y2, 576, 576)
    # bound, in units of u = 2^-24 times the sum of |corner terms| S:
    #   hi halves blended in fp32 (3 roundings per weight + 4 in the sum)                                 7
    #   lo halves (<= 2^-11 of the value) blended in fp16 with fp16 weights: weight rounding 2^-22 per
    #   term, four fp16 roundings of a sum <= 2^-11 S                                                      20
    #   fp32 hi + lo, the pair split of the operand (lo rounded: 2^-22), the GEMM's fp32 sum, the pair
    #   split of the output (2^-22)                                                                       1 + 4 + 1 + 4
    # = 37 u S, plus the fp16 subnormal floor of the lo halves (four blend roundings, two splits: 3 u)
    err = (got - ref).abs()
    bound = 37 * U * absum + 3 * U
    assert (err <= bound).all(), ("strict", cin, hw, worst(got, ref, err - bound))


# ----------------------------------------------------------------------------------------------------------- c
CHANNEL_PAIRS = [(512, 256), (256, 256), (256, 128), (128, 128), (128, 64), (64, 64), (256, 64)]


@pytest.mark.parametrize("prec", ["fast", "strict"])
@pytest.mark.parametrize("pair", CHANNEL_PAIRS)
def test_contraction_on_channel_slices(pair, prec):
    """random weights on the edge menu; x is a channel slice of a wider buffer (x_ld > Cin, channel offset 64, strict lo
    block at ld / 2) and y is written into a slice of a wider buffer whose other channels must stay untouched"""
    cin, cout = pair
    B, H, W = 2, 13, 41
    M = B * H * W
    strict = prec == "strict"
    gen = np.random.Generator(np.random.PCG64(cin * 7 + cout))
    x = images(gen, B, cin, H, W)
    wt = torch.from_numpy((gen.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32))
    wt = wt if strict else h16(wt)
    bias = torch.from_numpy((gen.standard_normal(cout) * 0.1).astype(np.float32)).cuda()
    bn = FakeBN(cout, gen)
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=cin + cout)
    offset, mask = offset.cuda(), mask.cuda()
    om = dcn_ref.to_offmask_rows(offset, mask)
    P = engine.Plan("cuda", strict=strict)
    wp, n_pad, k_pad = P.pack_weight(wt.cuda(), split=strict)
    scale, shift = P.affine(cout, n_pad, bn, bias)
    xo, lx, yo, ly = 64, cin + 128, 32, cout + 64                 # slice offsets and widths (channels)
    SENT = 1000.0
    if strict:
        rows = to_rows_split(x)
        xbuf = torch.full((M, 2 * lx), SENT, dtype=torch.half, device="cuda")
        xbuf[:, xo:xo + cin] = rows[:, :cin]
        xbuf[:, lx + xo:lx + xo + cin] = rows[:, cin:]
        ybuf = torch.full((M, 2 * ly), SENT, dtype=torch.half, device="cuda")
        call("mf_dcn_nhwc_f16x2", xbuf.data_ptr() + 2 * xo, 2 * lx, lx, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad,
             k_pad, cout, scale.data_ptr(), shift.data_ptr(), engine.ACT_NONE, ybuf.data_ptr() + 2 * yo, 2 * ly, ly, stream())
        xv = pair_value(rows, cin, cin)
        inside = torch.zeros(2 * ly, dtype=torch.bool, device="cuda")
        inside[yo:yo + cout] = inside[ly + yo:ly + yo + cout] = True
    else:
        xbuf = torch.full((M, lx), SENT, dtype=torch.half, device="cuda")
        xbuf[:, xo:xo + cin] = to_rows(x)
        ybuf = torch.full((M, ly), SENT, dtype=torch.half, device="cuda")
        call("mf_dcn_nhwc_f16", xbuf.data_ptr() + 2 * xo, lx, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad,
             cout, scale.data_ptr(), shift.data_ptr(), engine.ACT_NONE, engine.OUT_F16_NHWC, ybuf.data_ptr() + 2 * yo, ly,
             stream())
        xv = xbuf[:, xo:xo + cin].double()
        inside = torch.zeros(ly, dtype=torch.bool, device="cuda")
        inside[yo:yo + cout] = True
    torch.cuda.synchronize()
    assert (ybuf[:, ~inside] == SENT).all(), (prec, pair, "channels outside the y slice were written")
    got = pair_value(ybuf[:, yo:], cout, ly) if strict else ybuf[:, yo:yo + cout].double()
    cols = dcn_ref.columns(nchw(xv, B, H, W), offset, mask)
    ref = torch.einsum("okt,bkthw->bohw", wt.cuda().double().view(cout, cin, 9), cols)
    ref = ref * scale[:cout].double().view(1, -1, 1, 1) + shift[:cout].double().view(1, -1, 1, 1)
    got = nchw(got, B, H, W)
    tol = STRICT_TOL if strict else FAST_TOL
    assert rel(got, ref) < tol, (prec, pair, rel(got, ref), worst(got, ref))


# ----------------------------------------------------------------------------------------------------------- d
def model_dcn_shapes():
    """(Cin, Cout, H, W) of every distinct DCN layer in the backbone plan of a 384 x 1280 input"""
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.backbone.dla_dcn import build_backbone
    shapes = []
    orig = engine.Plan.dcn

    def record(self, x, dcn_mod, bn, out=None):
        shapes.append((x.C, dcn_mod.weight.shape[0], x.H, x.W))
        return orig(self, x, dcn_mod, bn, out)

    net = build_backbone(default_cfg(width=1280, height=384)).cuda().eval()
    engine.Plan.dcn = record
    try:
        net.build_plan(1, 384, 1280, "cuda")
    finally:
        engine.Plan.dcn = orig
    del net
    torch.cuda.empty_cache()
    return sorted(set(shapes), key=lambda s: (s[2], -s[0], -s[1]))


_SHAPES = []


def full_size_cases():
    if not _SHAPES:
        _SHAPES.extend(model_dcn_shapes())
    cases = [(2,) + s for s in _SHAPES]
    cases += [(8,) + s for s in _SHAPES if (s[2], s[3]) == (96, 320)]
    return cases


def test_model_dcn_shapes_are_the_known_seven():
    """the list the full-size test walks: DLAUp / IDAUp emit seven distinct DCN shapes at 384 x 1280"""
    assert full_size_cases()[:7] == [(2, 512, 256, 12, 40), (2, 256, 256, 24, 80), (2, 256, 128, 24, 80),
                                     (2, 256, 64, 24, 80), (2, 128, 128, 48, 160), (2, 128, 64, 48, 160),
                                     (2, 64, 64, 96, 320)], full_size_cases()


@pytest.mark.parametrize("prec", ["fast", "strict"])
@pytest.mark.parametrize("idx", range(8))
def test_full_size_layers(idx, prec):
    """P.dcn (offset conv + fused DCN + BN + ReLU) at the model's own shapes, B = 2 (and B = 8 at 96 x 320, where the
    persistent CTAs wrap the tile list), against float64 on the device, image by image, on the offsets the GPU produced"""
    cases = full_size_cases()
    if idx >= len(cases):
        pytest.skip("the plan has fewer DCN shapes")
    B, cin, cout, H, W = cases[idx]
    strict = prec == "strict"
    gen = np.random.Generator(np.random.PCG64(idx))
    x = torch.from_numpy(gen.standard_normal((B, cin, H, W)).astype(np.float32))
    d = dcn_module(gen, cin, cout, fp16=not strict)
    bn = FakeBN(cout, gen)
    P = engine.Plan("cuda", strict=strict)
    xa = P.act(B, H, W, cin)
    ya = P.dcn(xa, d, bn)
    P.finalize()
    xa.buf.copy_(to_rows_split(x) if strict else to_rows(x))
    P.run()
    torch.cuda.synchronize()
    om = P.keep[0]
    xv = xa.nchw_view().double()
    y = ya.nchw_view().double()
    w64 = d.weight.double().view(cout, cin * 9)
    err_om = err_y = 0.0
    max_om = max_y = 0.0
    where = ""
    for b in range(B):
        omb = om[b * H * W:(b + 1) * H * W]
        off = omb[:, :18].reshape(1, H, W, 18).permute(0, 3, 1, 2).contiguous()
        msk = omb[:, 18:27].reshape(1, H, W, 9).permute(0, 3, 1, 2).contiguous()
        o = F.conv2d(xv[b:b + 1], d.conv_offset_mask.weight.double(), d.conv_offset_mask.bias.double(), padding=1)
        o = torch.cat([o[:, :18], torch.sigmoid(o[:, 18:])], 1)
        got_o = torch.cat([off, msk], 1).double()
        e = (got_o - o).abs().max().item()
        err_om, max_om = max(err_om, e), max(max_om, o.abs().max().item())
        cols = dcn_ref.columns(xv[b:b + 1], off, msk).reshape(cin * 9, H * W)
        ref = F.relu(bn_eval64((w64 @ cols).view(1, cout, H, W), bn, d.bias))
        e = (y[b:b + 1] - ref).abs()
        if e.max().item() > err_y:
            err_y, where = e.max().item(), "image %d, %s" % (b, worst(y[b:b + 1], ref))
        max_y = max(max_y, ref.abs().max().item())
    assert err_om / max_om < 2e-5, (prec, cases[idx], "offset conv", err_om / max_om)
    tol = STRICT_TOL if strict else FAST_TOL
    assert err_y / max_y < tol, (prec, cases[idx], err_y / max_y, where)


# ----------------------------------------------------------------------------------------------------------- e
def _gcol64(w, dy):
    """dL/dcols [B, C, 9, H, W] = W^T dY, float64"""
    cout, cin = w.shape[:2]
    return torch.einsum("oct,bohw->bcthw", w.double().view(cout, cin, 9), dy.double())


@pytest.mark.parametrize("case", [(2, 64, 64, 10, 12), (2, 128, 256, 12, 20)])
def test_training_backward_on_edge_menu(case):
    """backward.dcn_backward vs float64 through the mask sigmoid: dX, the 18 offset gradients, the 9 mask pre-activation
    gradients (dL/dm * m (1 - m)), dW, dB. Tolerances as the random-offset test of the same operator (fp16 grad columns,
    fp16 atomics in dX, fp16 sampled columns in dW)."""
    from monoflex_b200 import backward
    B, C, Co, H, W = case
    gen = np.random.Generator(np.random.PCG64(sum(case)))
    x = h16(images(gen, B, C, H, W)).cuda()
    w = h16(torch.from_numpy((gen.standard_normal((Co, C, 3, 3)) / np.sqrt(9 * C)).astype(np.float32))).cuda()
    dy = h16(torch.from_numpy(gen.standard_normal((B, Co, H, W)).astype(np.float32))).cuda()
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=sum(case) + 1)
    offset, mask = offset.cuda(), mask.cuda()
    om = dcn_ref.to_offmask_rows(offset, mask)
    dx, dom, dw, db = backward.dcn_backward(rows16(x), om, rows16(dy), w, B, H, W)
    torch.cuda.synchronize()
    cols = dcn_ref.columns(x, offset, mask)
    dx64, doff64, dm64 = dcn_ref.backward(x, offset, mask, _gcol64(w, dy))
    m = mask.double()
    dpre64 = dm64 * m * (1 - m)
    dw64 = torch.einsum("bohw,bcthw->oct", dy.double(), cols).reshape(Co, C, 3, 3)
    db64 = dy.double().sum((0, 2, 3))
    dom = nchw(dom, B, H, W)
    for name, got, want, tol in (("dX", nchw(dx, B, H, W), dx64, 1e-2), ("dOffset", dom[:, :18], doff64, 1e-2),
                                 ("dMask pre-activation", dom[:, 18:27], dpre64, 1e-2), ("dW", dw, dw64, 3e-3),
                                 ("dB", db, db64, 1e-4)):
        assert rel(got, want) < tol, (name, case, rel(got, want), worst(got, want))
    assert (dom[:, 27:] == 0).all()


def test_tape_call_form_on_a_channel_slice():
    """the tape's call form: x is a channel slice (x_ld != C) of a wider buffer. Kernels: mf_dcn_sample_cols_nhwc_f16 and
    mf_dcn_col2im_nhwc_f16 with a given fp16 column gradient - the sampled columns must equal those of the compact layout bit
    for bit; with gcol given exactly, dOffset and dMask are fp32 sums over exact products (1e-5), dX carries the fp16 atomics
    (1e-2). Operator: backward.dcn_backward on the slice, dX accumulated into the same slice of a gradient buffer (whose
    other channels stay untouched), against float64 with the tolerances of test_training_backward_on_edge_menu."""
    from monoflex_b200 import backward
    B, C, H, W = 2, 128, 11, 13
    M = B * H * W
    gen = np.random.Generator(np.random.PCG64(21))
    x = h16(images(gen, B, C, H, W)).cuda()
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=22)
    offset, mask = offset.cuda(), mask.cuda()
    om = dcn_ref.to_offmask_rows(offset, mask)
    xo, lx = 32, C + 64
    xbuf = torch.full((M, lx), 1000.0, dtype=torch.half, device="cuda")
    xbuf[:, xo:xo + C] = rows16(x)
    xc = rows16(x)
    cols = torch.empty(M, 9 * C, dtype=torch.half, device="cuda")
    cols_c = torch.empty_like(cols)
    call("mf_dcn_sample_cols_nhwc_f16", xbuf.data_ptr() + 2 * xo, lx, om.data_ptr(), 32, cols.data_ptr(), B, H, W, C, stream())
    call("mf_dcn_sample_cols_nhwc_f16", xc.data_ptr(), C, om.data_ptr(), 32, cols_c.data_ptr(), B, H, W, C, stream())
    gcol = torch.from_numpy(gen.standard_normal((M, 9 * C)).astype(np.float32)).half().cuda()
    dx = torch.empty(M, C, dtype=torch.half, device="cuda")
    dom = torch.empty(M, 32, dtype=torch.float32, device="cuda")
    call("mf_dcn_col2im_nhwc_f16", xbuf.data_ptr() + 2 * xo, lx, om.data_ptr(), 32, gcol.data_ptr(), dx.data_ptr(), C,
         dom.data_ptr(), B, H, W, C, stream())
    torch.cuda.synchronize()
    assert torch.equal(cols, cols_c), worst(cols, cols_c)
    ref, absum = dcn_ref.columns(x, offset, mask, with_abs=True)
    ref = ref.permute(0, 3, 4, 2, 1).reshape(M, 9 * C)                 # rows [M, tap * C + c]
    absum = absum.permute(0, 3, 4, 2, 1).reshape(M, 9 * C)
    r16 = ref.half().double()
    err = (cols.double() - r16).abs()
    bound = torch.maximum(ulp16(r16), ulp16(cols)) + 8 * U * absum
    assert (err <= bound).all(), ("cols", worst(cols, ref, err - bound))
    g64 = gcol.double().view(B, H, W, 9, C).permute(0, 4, 3, 1, 2)
    dx64, doff64, dm64 = dcn_ref.backward(x, offset, mask, g64)
    m = mask.double()
    dom = nchw(dom, B, H, W)
    for name, got, want, tol in (("dX", nchw(dx, B, H, W), dx64, 1e-2), ("dOffset", dom[:, :18], doff64, 1e-5),
                                 ("dMask pre-activation", dom[:, 18:27], dm64 * m * (1 - m), 1e-5)):
        assert rel(got, want) < tol, (name, rel(got, want), worst(got, want))
    # the full operator on the slice
    Co = 64
    w = h16(torch.from_numpy((gen.standard_normal((Co, C, 3, 3)) / np.sqrt(9 * C)).astype(np.float32))).cuda()
    dy = h16(torch.from_numpy(gen.standard_normal((B, Co, H, W)).astype(np.float32))).cuda()
    gbuf = torch.zeros(M, lx, dtype=torch.half, device="cuda")
    _, dom, dw, db = backward.dcn_backward(engine.Act.on(xbuf, B, H, W, C, xo), om, rows16(dy), w, B, H, W,
                                           dx=engine.Act.on(gbuf, B, H, W, C, xo))
    torch.cuda.synchronize()
    assert (gbuf[:, :xo] == 0).all() and (gbuf[:, xo + C:] == 0).all(), "channels outside the dX slice were written"
    dx64, doff64, dm64 = dcn_ref.backward(x, offset, mask, _gcol64(w, dy))
    dw64 = torch.einsum("bohw,bcthw->oct", dy.double(), dcn_ref.columns(x, offset, mask)).reshape(Co, C, 3, 3)
    dom = nchw(dom, B, H, W)
    for name, got, want, tol in (("dX", nchw(gbuf[:, xo:xo + C], B, H, W), dx64, 1e-2), ("dOffset", dom[:, :18], doff64, 1e-2),
                                 ("dMask pre-activation", dom[:, 18:27], dm64 * m * (1 - m), 1e-2), ("dW", dw, dw64, 3e-3),
                                 ("dB", db, dy.double().sum((0, 2, 3)), 1e-4)):
        assert rel(got, want) < tol, ("operator", name, rel(got, want), worst(got, want))
    assert (dom[:, 27:] == 0).all()


def test_zero_offsets_half_mask_backward_known_answer():
    """the reference-init state on the fp16 training path: cols = fp16(0.5 x) bit for bit, and the offset gradients are the
    right differences of x (the reference's dmcn_get_coordinate_weight at integer coordinates), zero where the sample is
    past the border and at coordinate -1"""
    B, C, H, W = 2, 64, 9, 14
    M = B * H * W
    gen = np.random.Generator(np.random.PCG64(23))
    x = h16(images(gen, B, C, H, W)).cuda()
    om = torch.zeros(M, 32, dtype=torch.float32, device="cuda")
    om[:, 18:27] = 0.5
    xr = rows16(x)
    cols = torch.empty(M, 9 * C, dtype=torch.half, device="cuda")
    call("mf_dcn_sample_cols_nhwc_f16", xr.data_ptr(), C, om.data_ptr(), 32, cols.data_ptr(), B, H, W, C, stream())
    gcol = torch.from_numpy(gen.standard_normal((M, 9 * C)).astype(np.float32)).half().cuda()
    dx = torch.empty(M, C, dtype=torch.half, device="cuda")
    dom = torch.empty(M, 32, dtype=torch.float32, device="cuda")
    call("mf_dcn_col2im_nhwc_f16", xr.data_ptr(), C, om.data_ptr(), 32, gcol.data_ptr(), dx.data_ptr(), C, dom.data_ptr(), B,
         H, W, C, stream())
    torch.cuda.synchronize()
    want = (0.5 * F.unfold(x, 3, padding=1)).half().view(B, C, 9, H * W).permute(0, 3, 2, 1).reshape(M, 9 * C)
    assert torch.equal(cols.view(torch.int16), want.view(torch.int16)), worst(cols, want)
    # x zero-padded by one pixel on the top / left and two on the bottom / right: xp[r + 1, s + 1] = x[r, s]
    xp = F.pad(x.double(), (1, 2, 1, 2))
    g = gcol.double().view(B, H, W, 9, C).permute(0, 4, 3, 1, 2)            # [B, C, 9, H, W]
    ys, xs = torch.arange(H, device="cuda").view(H, 1), torch.arange(W, device="cuda").view(1, W)
    want_h, want_w = [], []
    for t in range(9):
        ky, kx = t // 3, t % 3
        r, s = ys - 1 + ky, xs - 1 + kx
        on = ((r >= 0) & (r <= H - 1) & (s >= 0) & (s <= W - 1)).double()    # coordinate -1, H or W: outside, no gradient
        here = xp[:, :, ky:ky + H, kx:kx + W]
        down = xp[:, :, ky + 1:ky + 1 + H, kx:kx + W]                       # row r + 1 (zero past the bottom border)
        right = xp[:, :, ky:ky + H, kx + 1:kx + 1 + W]
        want_h.append(0.5 * (g[:, :, t] * (down - here)).sum(1) * on)
        want_w.append(0.5 * (g[:, :, t] * (right - here)).sum(1) * on)
    want_off = torch.stack([torch.stack(want_h, 1), torch.stack(want_w, 1)], 2).reshape(B, 18, H, W)
    got_off = nchw(dom, B, H, W)[:, :18]
    assert rel(got_off, want_off) < 1e-5, ("right differences", rel(got_off, want_off), worst(got_off, want_off))
    assert (got_off[:, 0::2][:, 0:3, 0] == 0).all() and (got_off[:, 1::2][:, 0::3, :, 0] == 0).all()   # coordinate -1


# ----------------------------------------------------------------------------------------------------------- f
def test_ext_operator_exact_fp32_on_edge_menu():
    """_ext.dcn_v2_forward / dcn_v2_backward (exact fp32, reference NCHW layout): output and all five gradients within
    1e-5 of their magnitude of float64, at the kinks that the reference's gradcheck recipe cannot probe"""
    from monoflex_b200.model.backbone.DCNv2 import _ext
    B, C, Co, H, W = 2, 20, 7, 10, 12
    gen = np.random.Generator(np.random.PCG64(41))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()
    x = t(gen.standard_normal((B, C, H, W)))
    w = t(gen.standard_normal((Co, C, 3, 3)) * 0.3)
    bias = t(gen.standard_normal(Co))
    gy = t(gen.standard_normal((B, Co, H, W)))
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=42)
    offset, mask = offset.cuda(), mask.cuda()
    args = (3, 3, 1, 1, 1, 1, 1, 1, 1)
    y = _ext.dcn_v2_forward(x, w, bias, offset, mask, *args)
    gx, go, gm, gw, gb = _ext.dcn_v2_backward(x, w, bias, offset, mask, gy, *args)
    torch.cuda.synchronize()
    cols = dcn_ref.columns(x, offset, mask)
    y64 = torch.einsum("oct,bcthw->bohw", w.double().view(Co, C, 9), cols) + bias.double().view(1, -1, 1, 1)
    gx64, go64, gm64 = dcn_ref.backward(x, offset, mask, _gcol64(w, gy))
    gw64 = torch.einsum("bohw,bcthw->oct", gy.double(), cols).reshape(Co, C, 3, 3)
    gb64 = gy.double().sum((0, 2, 3))
    for name, got, want in (("y", y, y64), ("dX", gx, gx64), ("dOffset", go, go64), ("dMask", gm, gm64), ("dW", gw, gw64),
                            ("dB", gb, gb64)):
        assert rel(got, want) < 1e-5, (name, rel(got, want), worst(got, want))
