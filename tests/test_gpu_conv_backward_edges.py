"""The convolution backward at its tile, split and slice edges, element by element against float64 (-m gpu).

Operators: the general tensor-core weight gradient (csrc/mf_wgrad.cu), the stem's 16 -> 16 weight gradient
(csrc/mf_wgrad_narrow.cu), the rectangular 1x3 weight gradient of the edge-fusion Conv1d, the stride-1 data gradient
(the forward kernel on dgrad-packed weights, engine.Plan.conv_dgrad), the stride-2 data gradient (four parity
convolutions and mf_interleave2x2_nhwc_f16) and the up-sampling data gradient (upsample_bwd_dx_kernel). Every result is
held per element to the bounds of conv_backward_ref.py (2^-24 (P + S + 32) A for weight gradients, one fp16 rounding plus
2^-24 (k^2 Cout + 32) A for data gradients) and per tensor to a relative L2 threshold.

The cases place what the kernels have to get right at their edges:
  * general wgrad: Cin in {16, 32, 64, 192, 512} x Cout in {16, 32, 64, 192, 256}, k in {1, 3, 7}, stride 1 and 2
    (odd sizes), pad 0 or k/2, H or W = 1, images smaller than k, B = 3 (pixel blocks wrap across images), dummy
    slots in the last M tile (AW 16: up to 7, AW 32: 3, 1x1 at Cin / 64 odd: 1), Cout 192 as three 64-wide N tiles, and
    every split regime of the launcher (one split over several blocks, one block per split, an even spread, a remainder
    spread) - asserted from the launcher's formula with the device's SM count, so a case whose regime moves fails
    instead of silently testing something else; x as a channel slice of a wider NaN-bordered buffer, dY rows wider
    than Cout (NaN past Cout, never read); dW pre-filled with NaN.
  * narrow wgrad: k = 3 and 7, W in {1, 15, 16, 17, 33}, H in {1, 2, 5}, B in {1, 3}: ragged 16-pixel blocks, a
    half-empty last unit of two blocks, taps that read only padding (exactly 0); the 8 -> 16 widened stem image on an
    Act slice through backward.conv2d_wgrad.
  * rectangular wgrad: kh = 1, kw = 3 over one row of K + 2 pixels, K in {1, 2, 63, 64, 65, 832}.
  * stride-1 dgrad: the model's 3x3 stride-1 widths and its Root 1x1 widths (read from the built module), ragged M, dY
    with finite garbage in the padded Cout columns (the packer's zero weights cancel it), written and accumulated into
    a channel slice of a NaN-filled buffer with rows past M (neighbours bit-identical).
  * stride-2 dgrad: the level-entry pairs of the built module, Ho or Wo = 1, B = 3, written and through conv_backward
    into an Act slice; the odd-size refusal and add_rows' source check.
  * up-sampling dgrad: every factor of the built module's up-sampling layers, Hi or Wi = 1, C = 24 and 40 (no full
    64-channel group), written and accumulated.

Per-tensor relative L2 thresholds, at least 4x the worst measured on an NVIDIA H100 80GB HBM3 (700 W power limit):
  WGRAD_L2     2.5e-5 | 5.5e-6 (the B = 8 96x320 long reduction; 1.2e-7 narrow, 8.8e-8 stem, 1.6e-7 rectangular)
  DGRAD_L2     2e-3   | 4.6e-4 (stride 2, accumulated: two fp16 roundings; 2.2e-4 written, 2.9e-4 stride 1
                                accumulated); against the unrounded fp32 weights 5.1e-4 at worst (printed)
  UPSAMPLE_L2  1.5e-3 | 3.5e-4
Worst per-element err / bound measured there: general wgrad 0.033, narrow 0.045, stem 8 -> 16 0.018, rectangular
0.021; data gradients 0.92 (stride 1), 0.89 (stride 2), 0.98 (up-sampling): the fp16 rounding of the output is nearly
all of their bound, the accumulation error a small part. The file runs in about 15 s on that GPU.
"""
import functools
import math

import numpy as np
import pytest
import torch

import conv_backward_ref as R
from monoflex_b200 import _lib, backward, engine

pytestmark = pytest.mark.gpu

WGRAD_L2 = 2.5e-5
DGRAD_L2 = 2e-3
UPSAMPLE_L2 = 1.5e-3
NAN = float("nan")


# ------------------------------------------------------------------------------------------------ cases (CPU only)
# general wgrad: B, H, W, Cin, Cout, k, stride, pad, split regime on 132 SMs (H100 SXM)
WGRAD_CASES = [
    (3, 5, 7, 16, 32, 3, 1, 1, "one block per split"),         # AW 16: 9 slots in 2 tiles, 7 dummies; B = 3 wraps
    (2, 9, 13, 16, 64, 7, 2, 3, "one block per split"),        # AW 16 7x7: 49 slots, 7 dummies; odd sizes at stride 2
    (3, 1, 37, 16, 16, 3, 2, 1, "one block per split"),        # 16 -> 16 at stride 2 (general kernel), H = 1
    (2, 6, 5, 16, 16, 1, 1, 0, "one block per split"),         # 16 -> 16 1x1
    (2, 9, 8, 16, 16, 7, 1, 0, "one block per split"),         # 16 -> 16 7x7 without padding
    (3, 88, 128, 16, 16, 1, 1, 0, "even"),                     # 528 blocks over 264 splits
    (2, 5, 6, 16, 192, 3, 2, 1, "one block per split"),        # Cout 192: three 64-wide N tiles over 16-byte boxes
    (1, 7, 7, 16, 256, 7, 1, 3, "one block per split"),
    (3, 7, 11, 32, 32, 3, 2, 1, "one block per split"),        # AW 32: 9 slots in 3 tiles, 3 dummies
    (2, 3, 3, 32, 192, 7, 1, 3, "one block per split"),        # image smaller than the kernel
    (1, 16, 20, 32, 64, 1, 2, 0, "one block per split"),       # 1x1 at stride 2
    (2, 13, 17, 32, 256, 3, 1, 0, "one block per split"),      # 6 blocks over 6 splits
    (2, 6, 7, 32, 16, 3, 1, 1, "one block per split"),
    (3, 11, 13, 64, 16, 3, 2, 1, "one block per split"),
    (2, 1, 1, 64, 256, 3, 1, 1, "one block per split"),        # H = W = 1: every tap but the centre reads only padding
    (1, 5, 9, 64, 32, 7, 1, 3, "one block per split"),
    (3, 31, 41, 64, 64, 3, 1, 1, "remainder"),                 # 60 blocks over 53 splits, ragged last block
    (1, 3, 4, 64, 192, 3, 2, 1, "one block per split"),
    (2, 7, 9, 192, 64, 1, 1, 0, "one block per split"),        # 1x1 at Cin / 64 = 3: 1 dummy slot
    (3, 25, 25, 192, 192, 3, 2, 1, "remainder"),               # 8 blocks over 7 splits, odd sizes at stride 2
    (1, 1, 6, 192, 16, 7, 1, 3, "one block per split"),
    (2, 9, 11, 192, 32, 3, 1, 0, "one block per split"),
    (2, 4, 5, 192, 256, 1, 1, 0, "one block per split"),
    (3, 5, 7, 512, 256, 7, 1, 3, "one split"),                 # 392 tiles: one split over 2 blocks
    (2, 4, 3, 512, 32, 3, 1, 1, "one block per split"),
    (3, 9, 13, 512, 256, 3, 1, 1, "remainder"),                # 6 blocks over 4 splits
    (1, 2, 1, 512, 16, 1, 1, 0, "one block per split"),
    (2, 3, 5, 512, 64, 1, 2, 0, "one block per split"),
    (1, 3, 3, 512, 192, 3, 1, 1, "one block per split"),
    (8, 96, 320, 64, 64, 3, 1, 1, "remainder"),                # the long reduction: 3840 blocks over 53 splits
]
LONG = (8, 96, 320)

# narrow wgrad: k, W, H, B
NARROW_CASES = [(k, W, H, B) for k in (3, 7) for W in (1, 15, 16, 17, 33) for H, B in ((1, 3), (2, 1), (5, 3))]

RECT_KS = [1, 2, 63, 64, 65, 832]


@functools.lru_cache(maxsize=None)
def model_shapes():
    """(stride-1 3x3 (Cin, Cout) pairs, Root 1x1 (Cin, Cout) pairs, stride-2 (Cin, Cout) pairs, up-sampling factors) of
    the built DLA-34 backbone"""
    import torch.nn as nn
    from monoflex_b200.model.backbone import dla_dcn
    m = dla_dcn.DLASeg("dla34", False, 4, 5)
    convs = [c for c in m.base.modules() if isinstance(c, nn.Conv2d)]
    s1 = sorted({(c.in_channels, c.out_channels) for c in convs if c.kernel_size == (3, 3) and c.stride == (1, 1)})
    s2 = sorted({(c.in_channels, c.out_channels) for c in convs if c.kernel_size == (3, 3) and c.stride == (2, 2)})
    roots = sorted({(r.conv.in_channels, r.conv.out_channels) for r in m.modules() if isinstance(r, dla_dcn.Root)})
    ups = sorted({f for r in m.modules() if isinstance(r, dla_dcn.IDAUp) for f in r.up_f[1:]})
    return s1, roots, s2, ups


def dgrad1_cases():
    """B, H, W, Cin, Cout, k, pad, dY column padding (to the next width the weight gradient takes, every other case)"""
    s1, roots, _, _ = model_shapes()
    s1 = sorted(set(s1) | {(32, 32)})                    # and the level-1 width, whose only conv has stride 2
    geo = [(3, 5, 7), (1, 1, 9), (2, 7, 1), (3, 3, 5)]
    cases = [geo[i % len(geo)] + (cin, cout, 3, 1) for i, (cin, cout) in enumerate(s1)]
    cases += [geo[(i + 1) % len(geo)] + (cin, cout, 1, 0) for i, (cin, cout) in enumerate(roots)]
    return [c + ((min(c[4], 64) if i % 2 == 0 else 0),) for i, c in enumerate(cases)]


def dgrad2_cases():
    """B, H, W, Cin, Cout (H, W even)"""
    _, _, s2, _ = model_shapes()
    geo = [(3, 2, 14), (3, 10, 2), (3, 2, 2), (1, 6, 10), (3, 8, 6)]
    return [geo[i % len(geo)] + pair for i, pair in enumerate(s2)]


def upsample_cases():
    """B, Hi, Wi, C, f"""
    _, _, _, ups = model_shapes()
    return [g + (f,) for f in ups for g in ((3, 1, 7, 24), (2, 5, 1, 40), (1, 3, 4, 64))]


def f16(gen, shape, scale=1.0, mean=0.0):
    """CPU float tensor of fp16-representable values"""
    return torch.from_numpy((gen.standard_normal(shape) * scale + mean).astype(np.float32)).half().float()


def wgrad_inputs(B, H, W, Cin, Cout, kernel, stride, pad, seed):
    """x [B, Cin, H, W], dy [B, Cout, Ho, Wo] (CPU, fp16-representable); one dY channel all zero (its dW row is exactly 0)"""
    gen = np.random.Generator(np.random.PCG64(seed))
    Ho, Wo = R.out_hw(H, W, kernel, stride, pad)
    x = f16(gen, (B, Cin, H, W))
    dy = f16(gen, (B, Cout, Ho, Wo), 0.1, 0.02)
    dy[:, Cout // 2] = 0
    return x, dy


def dgrad_inputs(B, Ho, Wo, Cin, Cout, k, seed):
    """dy [B, Cout, Ho, Wo] fp16-representable, w [Cout, Cin, k, k] random fp32 (not rounded)"""
    gen = np.random.Generator(np.random.PCG64(seed))
    dy = f16(gen, (B, Cout, Ho, Wo))
    w = torch.from_numpy((gen.standard_normal((Cout, Cin, k, k)) / math.sqrt(Cout * k * k)).astype(np.float32))
    return dy, w


def upsample_inputs(B, Hi, Wi, C, f, seed):
    gen = np.random.Generator(np.random.PCG64(seed))
    x = f16(gen, (B, C, Hi, Wi))
    dy = f16(gen, (B, C, Hi * f, Wi * f))
    w = torch.from_numpy(gen.uniform(-0.5, 0.5, (C, 1, 2 * f, 2 * f)).astype(np.float32))
    return x, dy, w


# ------------------------------------------------------------------------------------------------ GPU helpers
def nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rows_buf(t4, ld, off, fill=NAN, extra_rows=0):
    """fp16 CUDA rows [B*H*W + extra_rows, ld] holding [B, C, H, W] at columns [off, off + C), `fill` elsewhere"""
    r = R.flat_pixels(t4)
    buf = torch.full((r.shape[0] + extra_rows, ld), fill, dtype=torch.half)
    buf[:r.shape[0], off:off + r.shape[1]] = r.half()
    return buf.cuda()


def nchw(rows, B, H, W):
    """[B*H*W, C] rows (a column slice is fine) -> [B, C, H, W] float64 CPU"""
    return R.from_flat(rows.double().cpu(), B, H, W)


def bits(t):
    return t.view(torch.int16).cpu()


def report(name, **kv):
    print(name + ": " + " ".join("%s=%s" % (k, ("%.3g" % v) if isinstance(v, float) else v) for k, v in kv.items()))


# ------------------------------------------------------------------------------------------------ general wgrad
@pytest.mark.parametrize("case", WGRAD_CASES, ids=["B%d-%dx%d-%d-%d-k%d-s%d-p%d" % c[:8] for c in WGRAD_CASES])
def test_wgrad_general_edges(case):
    B, H, W, Cin, Cout, k, s, pad, regime = case
    i = WGRAD_CASES.index(case)
    assert not R.goes_narrow(Cin, Cout, k, s, pad)
    plan = R.wgrad_plan(B, H, W, Cin, Cout, k, s, pad, nsm())
    assert plan["regime"] == regime, (plan["regime"], plan["nkb"], plan["splits"], plan["tiles"])
    x, dy = wgrad_inputs(B, H, W, Cin, Cout, k, s, pad, 100 + i)
    x_off = 8 if i % 2 == 0 else 0                     # x as a channel slice of a wider NaN-bordered buffer
    dy_pad = 16 if i % 3 == 0 else 0                   # dY rows wider than Cout, NaN past Cout
    xb = rows_buf(x, Cin + 2 * x_off, x_off)
    dyb = rows_buf(dy, Cout + dy_pad, 0)
    dw = torch.full((Cout, Cin, k, k), NAN, dtype=torch.float32, device="cuda")
    _lib.call("mf_conv2d_wgrad_nhwc_f16", xb.data_ptr() + 2 * x_off, xb.shape[1], B, H, W, Cin, dyb.data_ptr(), dyb.shape[1],
              Cout, k, s, pad, dw.data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    ref, A = R.wgrad_ref(x, dy, k, s, pad, per_image=(B, H, W) == LONG)
    got = dw.double().cpu()
    r = R.ratio((got - ref).abs(), R.wgrad_bound(A, plan["P"], plan["S"]))
    l2 = R.rel_l2(got, ref)
    report("wgrad B=%d %dx%d %d->%d k=%d s=%d p=%d" % case[:8], regime=regime, blocks=plan["nkb"], splits=plan["splits"],
           tiles=plan["tiles"], dummies=plan["dummies"], ragged=plan["ragged"], ratio=r, rel_l2=l2)
    assert r <= 1.0, r
    assert l2 <= WGRAD_L2, l2
    assert torch.equal(got[Cout // 2], torch.zeros_like(got[Cout // 2]))      # the all-zero dY channel


# ------------------------------------------------------------------------------------------------ narrow wgrad
def dead_taps(H, W, k):
    """(ky, kx) taps of a k x k "same" convolution that read only padding on an H x W image"""
    pad = k // 2
    live_y = {ky for ky in range(k) for oy in range(H) if 0 <= oy + ky - pad < H}
    live_x = {kx for kx in range(k) for ox in range(W) if 0 <= ox + kx - pad < W}
    return [(ky, kx) for ky in range(k) for kx in range(k) if ky not in live_y or kx not in live_x]


@pytest.mark.parametrize("k,W,H,B", NARROW_CASES, ids=["k%d-W%d-H%d-B%d" % c for c in NARROW_CASES])
def test_wgrad_narrow_edges(k, W, H, B):
    plan = R.narrow_plan(B, H, W, k, nsm())
    assert R.goes_narrow(16, 16, k, 1, k // 2)
    x, dy = wgrad_inputs(B, H, W, 16, 16, k, 1, k // 2, 1000 + 100 * k + 10 * W + H + B)
    xb = rows_buf(x, 32, 8)
    dyb = rows_buf(dy, 32, 8)
    dw = torch.full((16, 16, k, k), NAN, dtype=torch.float32, device="cuda")
    _lib.call("mf_conv2d_wgrad_nhwc_f16", xb.data_ptr() + 16, 32, B, H, W, 16, dyb.data_ptr() + 16, 32, 16, k, 1, k // 2,
              dw.data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    ref, A = R.wgrad_ref(x, dy, k, 1, k // 2)
    got = dw.double().cpu()
    r = R.ratio((got - ref).abs(), R.wgrad_bound(A, plan["P"], plan["S"]))
    l2 = R.rel_l2(got, ref)
    dead = dead_taps(H, W, k)
    report("narrow k=%d W=%d H=%d B=%d" % (k, W, H, B), blocks=plan["nblocks"], units=plan["nunits"],
           half_unit=plan["last_unit_half"], dead_taps=len(dead), ratio=r, rel_l2=l2)
    assert r <= 1.0, r
    assert l2 <= WGRAD_L2, l2
    for ky, kx in dead:
        assert A[:, :, ky, kx].abs().max().item() == 0 and got[:, :, ky, kx].abs().max().item() == 0, (ky, kx)
    if H == 2 and k == 7:
        assert {ky for ky in range(k) if all((ky, kx) in dead for kx in range(k))} == {0, 1, 5, 6}


@pytest.mark.parametrize("k", [3, 7])
def test_wgrad_stem_widened_on_act_slice(k):
    """backward.conv2d_wgrad on the 8-channel stem image, an Act slice of a NaN-bordered buffer: widened to 16 zero
    channels for the narrow kernel, dW [16, 8, k, k]"""
    B, H, W = 2, 5, 17
    x, dy = wgrad_inputs(B, H, W, 8, 16, k, 1, k // 2, 50 + k)
    xa = engine.Act.on(rows_buf(x, 32, 8), B, H, W, C=8, ch_off=8)
    dw = backward.conv2d_wgrad(xa, rows_buf(dy, 16, 0), B, H, W, k, 1, k // 2)
    torch.cuda.synchronize()
    assert tuple(dw.shape) == (16, 8, k, k)
    plan = R.narrow_plan(B, H, W, k, nsm())
    ref, A = R.wgrad_ref(x, dy, k, 1, k // 2)
    got = dw.double().cpu()
    r = R.ratio((got - ref).abs(), R.wgrad_bound(A, plan["P"], plan["S"]))
    report("stem 8->16 k=%d" % k, ratio=r, rel_l2=R.rel_l2(got, ref))
    assert r <= 1.0 and R.rel_l2(got, ref) <= WGRAD_L2, r


# ------------------------------------------------------------------------------------------------ rectangular wgrad
@pytest.mark.parametrize("K", RECT_KS)
def test_wgrad_rect_edge_fusion(K):
    """the edge-fusion Conv1d's weight gradient: kh = 1, kw = 3, no padding, over B rows of K + 2 border positions"""
    B, C = 2, 256
    x, dy = wgrad_inputs(B, 1, K + 2, C, C, (1, 3), 1, 0, 70 + K)
    xb = rows_buf(x, C + 16, 8)
    dyb = rows_buf(dy, C, 0)
    dw = torch.full((C, C, 1, 3), NAN, dtype=torch.float32, device="cuda")
    _lib.call("mf_conv2d_wgrad_rect_nhwc_f16", xb.data_ptr() + 16, C + 16, B, 1, K + 2, C, dyb.data_ptr(), C, C, 1, 3, 1, 0, 0,
              dw.data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    plan = R.wgrad_plan(B, 1, K + 2, C, C, (1, 3), 1, 0, nsm())
    ref, A = R.wgrad_ref(x, dy, (1, 3), 1, 0)
    got = dw.double().cpu()
    r = R.ratio((got - ref).abs(), R.wgrad_bound(A, plan["P"], plan["S"]))
    l2 = R.rel_l2(got, ref)
    report("rect K=%d" % K, regime=plan["regime"], blocks=plan["nkb"], splits=plan["splits"], ratio=r, rel_l2=l2)
    assert r <= 1.0 and l2 <= WGRAD_L2, (r, l2)


# ------------------------------------------------------------------------------------------------ stride-1 dgrad
def dgrad_check(name, got, ref, A, ref32, terms, before=None, roundings=1):
    r = R.ratio((got - (ref if before is None else before.double() + ref)).abs(),
                R.dgrad_bound(ref, A, terms, before, roundings))
    inc = got if before is None else got - before.double()
    l2 = R.rel_l2(inc, ref)
    report(name, ratio=r, rel_l2=l2, rel_l2_vs_fp32_w=R.rel_l2(inc, ref32))
    return r, l2


@pytest.mark.parametrize("case", dgrad1_cases(), ids=lambda c: "B%d-%dx%d-%d-%d-k%d-pad%d-dypad%d" % c)
def test_dgrad_stride1_edges(case):
    B, H, W, Cin, Cout, k, pad, cpad = case
    dy, w = dgrad_inputs(B, H, W, Cin, Cout, k, 200 + Cin + Cout + k)
    gen = np.random.Generator(np.random.PCG64(300 + Cin))
    M = B * H * W
    dyb = rows_buf(dy, Cout + cpad, 0, fill=0.0)
    if cpad:                                                  # finite garbage in the padded columns
        dyb[:, Cout:] = torch.from_numpy(gen.uniform(-1e3, 1e3, (M, cpad)).astype(np.float32)).half().cuda()
    wc = w.cuda()
    ref, A = R.dgrad_ref(dy, w.half(), (H, W), 1, pad)
    ref32, _ = R.dgrad_ref(dy, w, (H, W), 1, pad)
    terms = k * k * Cout
    # written
    dx = backward.conv2d_dgrad(dyb, wc, B, H, W, pad)
    torch.cuda.synchronize()
    assert tuple(dx.shape) == (M, Cin)
    r1, l1 = dgrad_check("dgrad s1 B=%d %dx%d %d->%d k=%d dy+%d written" % (B, H, W, Cin, Cout, k, cpad), nchw(dx, B, H, W),
                         ref, A, ref32, terms)
    # accumulated through conv_backward into a channel slice of a NaN buffer with rows past M
    before = f16(gen, (B, Cin, H, W), 0.5)
    buf = rows_buf(before, Cin + 16, 8, extra_rows=5)
    keep = buf.clone()
    x = f16(gen, (B, Cin, H, W))
    xa = engine.Act.on(rows_buf(x, Cin, 0), B, H, W)
    dw, db = backward.conv_backward(xa, wc, None, 1, pad, dyb, engine.Act.on(buf, B, H, W, C=Cin, ch_off=8))
    torch.cuda.synchronize()
    r2, l2 = dgrad_check("dgrad s1 B=%d %dx%d %d->%d k=%d dy+%d accumulated" % (B, H, W, Cin, Cout, k, cpad),
                         nchw(buf[:M, 8:8 + Cin], B, H, W), ref, A, ref32, terms, before)
    assert db is None and tuple(dw.shape) == (Cout, Cin, k, k)
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    assert l1 <= DGRAD_L2 and l2 <= DGRAD_L2, (l1, l2)
    b0, b1 = bits(buf), bits(keep)
    assert torch.equal(b0[:, :8], b1[:, :8]) and torch.equal(b0[:, 8 + Cin:], b1[:, 8 + Cin:]) and torch.equal(b0[M:], b1[M:])
    # the weight gradient of the same call (padded dY rows: dW has them as extra rows, cut off)
    wref, wA = R.wgrad_ref(x, dy, k, 1, pad)
    plan = R.wgrad_plan(B, H, W, Cin, Cout + cpad, k, 1, pad, nsm())
    assert R.ratio((dw.double().cpu() - wref).abs(), R.wgrad_bound(wA, plan["P"], plan["S"])) <= 1.0


# ------------------------------------------------------------------------------------------------ stride-2 dgrad
@pytest.mark.parametrize("case", dgrad2_cases(), ids=lambda c: "B%d-%dx%d-%d-%d" % c)
def test_dgrad_stride2_edges(case):
    B, H, W, Cin, Cout = case
    Ho, Wo = H // 2, W // 2
    dy, w = dgrad_inputs(B, Ho, Wo, Cin, Cout, 3, 400 + Cin + H)
    gen = np.random.Generator(np.random.PCG64(500 + Cin))
    M = B * H * W
    dyb = rows_buf(dy, Cout, 0)
    wc = w.cuda()
    ref, A = R.dgrad_ref(dy, w.half(), (H, W), 2, 1)
    ref32, _ = R.dgrad_ref(dy, w, (H, W), 2, 1)
    terms = 9 * Cout
    dx = backward.conv2d_dgrad_stride2(dyb, wc, B, Ho, Wo)
    torch.cuda.synchronize()
    assert tuple(dx.shape) == (M, Cin)
    r1, l1 = dgrad_check("dgrad s2 B=%d %dx%d %d->%d written" % case, nchw(dx, B, H, W), ref, A, ref32, terms)
    before = f16(gen, (B, Cin, H, W), 0.5)
    buf = rows_buf(before, Cin + 16, 8, extra_rows=5)
    keep = buf.clone()
    x = f16(gen, (B, Cin, H, W))
    dw, _ = backward.conv_backward(engine.Act.on(rows_buf(x, Cin, 0), B, H, W), wc, None, 2, 1, dyb,
                                   engine.Act.on(buf, B, H, W, C=Cin, ch_off=8))
    torch.cuda.synchronize()
    r2, l2 = dgrad_check("dgrad s2 B=%d %dx%d %d->%d accumulated" % case, nchw(buf[:M, 8:8 + Cin], B, H, W), ref, A, ref32,
                         terms, before, roundings=2)
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    assert l1 <= DGRAD_L2 and l2 <= DGRAD_L2, (l1, l2)
    b0, b1 = bits(buf), bits(keep)
    assert torch.equal(b0[:, :8], b1[:, :8]) and torch.equal(b0[:, 8 + Cin:], b1[:, 8 + Cin:]) and torch.equal(b0[M:], b1[M:])


@pytest.mark.parametrize("H,W", [(7, 8), (8, 7), (5, 5)])
def test_dgrad_stride2_refuses_odd_sizes(H, W):
    """the parity decomposition covers (H + 1) x (W + 1) pixels on an odd input: conv_backward refuses before it
    launches anything, and the destination is left as it was"""
    B, Cin, Cout = 2, 16, 32
    Ho, Wo = R.out_hw(H, W, 3, 2, 1)
    dy, w = dgrad_inputs(B, Ho, Wo, Cin, Cout, 3, 9)
    gen = np.random.Generator(np.random.PCG64(H * W))
    buf = rows_buf(f16(gen, (B, Cin, H, W)), Cin, 0)
    keep = buf.clone()
    xa = engine.Act.on(rows_buf(f16(gen, (B, Cin, H, W)), Cin, 0), B, H, W)
    with pytest.raises(NotImplementedError, match="odd"):
        backward.conv_backward(xa, w.cuda(), None, 2, 1, rows_buf(dy, Cout, 0), engine.Act.on(buf, B, H, W))
    torch.cuda.synchronize()
    assert torch.equal(bits(buf), bits(keep))


def test_add_rows_checks_its_source():
    """add_rows refuses a source with more rows than the destination (what the odd-size stride-2 data gradient
    produced) and one with fewer channels, without touching the destination; a matching source still adds"""
    gen = np.random.Generator(np.random.PCG64(11))
    B, H, W, C = 2, 3, 5, 24
    M = B * H * W
    dst = rows_buf(f16(gen, (B, C, H, W)), C, 0)
    keep = dst.clone()
    longer = rows_buf(f16(gen, (B, C, H + 1, W + 1)), C, 0)
    with pytest.raises(ValueError, match="rows"):
        backward.add_rows(dst, longer)
    with pytest.raises(ValueError, match="rows"):
        backward.add_rows(engine.Act.on(dst, B, H, W), engine.Act.on(longer, B, H + 1, W + 1))
    narrow = engine.Act.on(rows_buf(f16(gen, (B, C, H, W)), C, 0), B, H, W, C=C - 8)     # reads stay inside its buffer
    with pytest.raises(ValueError, match="rows"):
        backward.add_rows(dst, narrow)
    torch.cuda.synchronize()
    assert torch.equal(bits(dst), bits(keep))
    src = rows_buf(f16(gen, (B, C, H, W)), C, 0)
    backward.add_rows(dst, src)
    torch.cuda.synchronize()
    assert torch.equal(dst.cpu(), (keep.float() + src.float()).half().cpu())
    assert dst.shape[0] == M


# ------------------------------------------------------------------------------------------------ up-sampling dgrad
@pytest.mark.parametrize("case", upsample_cases(), ids=lambda c: "B%d-%dx%d-C%d-f%d" % c)
def test_upsample_dx_edges(case):
    B, Hi, Wi, C, f = case
    x, dy, w = upsample_inputs(B, Hi, Wi, C, f, 600 + C + f)
    gen = np.random.Generator(np.random.PCG64(700 + C))
    k = 2 * f
    M = B * Hi * Wi
    ref, A = R.upsample_dx_ref(dy, w, f)
    taps = w.view(C, k * k).t().contiguous().cuda()
    xr, dyr = rows_buf(x, C, 0), rows_buf(dy, C, 0)
    dx, _ = backward.upsample_backward(xr, taps, dyr, B, Hi, Wi, f)
    torch.cuda.synchronize()
    got = nchw(dx, B, Hi, Wi)
    r1 = R.ratio((got - ref).abs(), R.dgrad_bound(ref, A, k * k))
    l1 = R.rel_l2(got, ref)
    before = f16(gen, (B, C, Hi, Wi), 0.5)
    buf = rows_buf(before, C + 16, 8, extra_rows=3)
    keep = buf.clone()
    backward.upsample_backward(xr, taps, dyr, B, Hi, Wi, f, dx=engine.Act.on(buf, B, Hi, Wi, C=C, ch_off=8))
    torch.cuda.synchronize()
    acc = nchw(buf[:M, 8:8 + C], B, Hi, Wi)
    r2 = R.ratio((acc - before.double() - ref).abs(), R.dgrad_bound(ref, A, k * k, before, roundings=2))
    l2 = R.rel_l2(acc - before.double(), ref)
    report("upsample dx B=%d %dx%d C=%d f=%d" % case, ratio_written=r1, ratio_accumulated=r2, rel_l2=max(l1, l2))
    assert r1 <= 1.0 and r2 <= 1.0, (r1, r2)
    assert l1 <= UPSAMPLE_L2 and l2 <= UPSAMPLE_L2, (l1, l2)
    b0, b1 = bits(buf), bits(keep)
    assert torch.equal(b0[:, :8], b1[:, :8]) and torch.equal(b0[:, 8 + C:], b1[:, 8 + C:]) and torch.equal(b0[M:], b1[M:])
