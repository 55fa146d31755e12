"""GPU: the DCN offset/mask convolution (csrc/mf_offset_conv.cu) through its entry points, both precisions, against float64
conv2d on the inputs the kernel reads (strict: hi + lo pairs; fast and the train-mode forward: fp16 rows and fp16 weights),
with sigmoid on the mask channels 18-26. Channels 27-31 have zero weights: they hold sigmoid(0) = 0.5, as before.

Also the addressing the kernel rests on: wgmma A descriptors on SWIZZLE_128B rows whose start lies 1..7 rows past a
swizzle atom (mf_selftest_sw128_shift)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import rel_err
from monoflex_b200 import engine
from monoflex_b200._lib import call, stream

pytestmark = pytest.mark.gpu

FAST_TOL, STRICT_TOL = 2e-3, 3e-5


def test_sw128_shifted_descriptor_selftest():
    """D = A[s .. s + 63] B^T for s = 0..7 with the matrix base-offset field 0 (the form the kernel uses) and
    (start >> 7) & 7; the first must be exact for every shift. The second is reported, not required."""
    gen = np.random.Generator(np.random.PCG64(11))
    a = torch.from_numpy(gen.standard_normal((80, 64)).astype(np.float32)).half()
    b = torch.from_numpy(gen.standard_normal((32, 64)).astype(np.float32)).half()
    d = torch.full((2, 8, 64, 32), float("nan"), dtype=torch.float32, device="cuda")
    ac, bc = a.cuda(), b.cuda()
    call("mf_selftest_sw128_shift", ac.data_ptr(), bc.data_ptr(), d.data_ptr(), stream())
    torch.cuda.synchronize()
    d = d.cpu().double()
    errs = [[rel_err(d[v, s], a[s:s + 64].double() @ b.double().t()) for s in range(8)] for v in range(2)]
    print("sw128 shifted descriptor: max rel err per shift, base offset 0:", errs[0], "(start >> 7) & 7:", errs[1])
    assert max(errs[0]) < 1e-6, errs[0]


def weights(gen, cin):
    w = torch.from_numpy((gen.standard_normal((27, cin, 3, 3)) * 1.5 / np.sqrt(9 * cin)).astype(np.float32))
    bias = torch.from_numpy((gen.standard_normal(27) * 0.2).astype(np.float32))
    return w, bias


def reference(x64, w64, bias):
    o = F.conv2d(x64, w64, bias.double(), 1, 1)
    return torch.cat([o[:, :18], torch.sigmoid(o[:, 18:])], 1)


def run(B, cin, H, W, strict, seed=0, scales=None, slice_pad=0):
    """the offset conv on a [B H W, ld] buffer whose first `slice_pad` channels and the gap after the hi block are not the
    input (a channel slice of a wider tensor); image b scaled by scales[b]. Returns (GPU rows [M, 32], fp64 reference
    [B, 27, H, W])."""
    gen = np.random.Generator(np.random.PCG64(seed))
    x = torch.from_numpy(gen.standard_normal((B, cin, H, W)).astype(np.float32))
    if scales is not None:
        x = x * torch.tensor(scales, dtype=torch.float32).view(B, 1, 1, 1)
    w, bias = weights(gen, cin)
    M = B * H * W
    rows = x.permute(0, 2, 3, 1).reshape(M, cin)
    hi = rows.half()
    lo = (rows - hi.float()).half()
    gap = slice_pad
    ld = slice_pad + (2 * cin + gap if strict else cin) + slice_pad
    buf = torch.full((M, ld), 1e4, dtype=torch.half)                  # what is not the input is large
    buf[:, slice_pad:slice_pad + cin] = hi
    if strict:
        buf[:, slice_pad + cin + gap:slice_pad + 2 * cin + gap] = lo
    buf = buf.cuda()
    xp = buf.data_ptr() + 2 * slice_pad
    wc = w.cuda()
    n_pad, k_pad = 32, (3 if strict else 1) * 9 * cin
    wp = torch.empty(n_pad, k_pad, dtype=torch.half, device="cuda")
    if strict:
        call("mf_pack_conv_weight_split", wc.data_ptr(), 27, cin, 3, 3, n_pad, k_pad, wp.data_ptr(), stream())
    else:
        call("mf_pack_conv_weight", wc.data_ptr(), 27, cin, 3, 3, cin, n_pad, k_pad, wp.data_ptr(), stream())
    scale = torch.ones(32, dtype=torch.float32, device="cuda")
    shift = torch.zeros(32, dtype=torch.float32, device="cuda")
    shift[:27] = bias.cuda()
    outs = []
    for _ in range(2):
        om = torch.full((M, 32), float("nan"), dtype=torch.float32, device="cuda")
        if strict:
            call("mf_conv2d_nhwc_f16x2", xp, ld, cin + gap, B, H, W, cin, wp.data_ptr(), n_pad, k_pad, 3, 3, 1, 1, 27,
                 scale.data_ptr(), shift.data_ptr(), None, 0, 0, engine.ACT_OFFMASK, engine.OUT_F32_NHWC, om.data_ptr(), 32, 0,
                 1, 0, stream())
        else:
            call("mf_conv2d_nhwc_f16", xp, ld, B, H, W, cin, wp.data_ptr(), n_pad, k_pad, 3, 3, 1, 1, 27, scale.data_ptr(),
                 shift.data_ptr(), None, 0, engine.ACT_OFFMASK, engine.OUT_F32_NHWC, om.data_ptr(), 32, stream())
        torch.cuda.synchronize()
        outs.append(om.cpu())
    assert torch.equal(outs[0], outs[1]), "repeated launches differ"
    if strict:
        x64 = (hi.double() + lo.double()).reshape(B, H, W, cin).permute(0, 3, 1, 2)
        w64 = w.double()
    else:
        x64 = hi.double().reshape(B, H, W, cin).permute(0, 3, 1, 2)
        w64 = w.half().double()
    return outs[0], reference(x64, w64, bias)


def check(om, ref, tol):
    B, _, H, W = ref.shape
    got = om[:, :27].reshape(B, H, W, 27).permute(0, 3, 1, 2).double()
    for b in range(B):
        assert rel_err(got[b], ref[b]) < tol, (b, rel_err(got[b], ref[b]))
    assert torch.equal(om[:, 27:], torch.full_like(om[:, 27:], 0.5))


# the four (Cin, H, W) of the backbone at 384 x 1280, B = 8
LAYER_SHAPES = [(64, 96, 320), (128, 48, 160), (256, 24, 80), (512, 12, 40)]
# odd cases: B = 1 and 3, H not a multiple of the tile rows, W not a multiple of the segment
ODD_CASES = [(1, 64, 13, 40), (1, 512, 4, 6), (3, 64, 13, 72), (3, 512, 7, 130), (1, 512, 13, 72), (3, 128, 5, 130)]


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
@pytest.mark.parametrize("shape", LAYER_SHAPES)
def test_offset_conv_layer_shapes(shape, strict):
    cin, H, W = shape
    om, ref = run(8, cin, H, W, strict, seed=cin)
    check(om, ref, STRICT_TOL if strict else FAST_TOL)


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
@pytest.mark.parametrize("case", ODD_CASES)
def test_offset_conv_odd_shapes(case, strict):
    B, cin, H, W = case
    om, ref = run(B, cin, H, W, strict, seed=B + cin)
    check(om, ref, STRICT_TOL if strict else FAST_TOL)


@pytest.mark.parametrize("strict", [True, False], ids=["strict", "fast"])
@pytest.mark.parametrize("cin", [64, 512])
def test_offset_conv_image_borders_and_slices(cin, strict):
    """the middle image is 1000x larger and the input is a channel slice of a buffer filled with 1e4 elsewhere: a tap
    that reads across an image border or outside the slice shows up in the other images' error"""
    om, ref = run(3, cin, 9, 44, strict, seed=7, scales=[1.0, 1000.0, 1.0], slice_pad=32)
    check(om, ref, STRICT_TOL if strict else FAST_TOL)


def test_offset_conv_train_forward():
    """train mode: the offset conv of a DCN plan takes the fp16 path with weights re-packed from the live parameter"""
    gen = np.random.Generator(np.random.PCG64(3))
    B, cin, H, W = 2, 128, 11, 37

    class D(object):
        pass
    d = D()
    d.weight = torch.from_numpy((gen.standard_normal((64, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32)).cuda()
    d.bias = torch.zeros(64, device="cuda")
    w, bias = weights(gen, cin)
    d.conv_offset_mask = torch.nn.Conv2d(cin, 27, 3, 1, 1).cuda()
    with torch.no_grad():
        d.conv_offset_mask.weight.copy_(w)
        d.conv_offset_mask.bias.copy_(bias)
    bn = torch.nn.BatchNorm2d(64).cuda()
    P = engine.Plan("cuda", train=True)
    xa = P.act(B, H, W, cin)
    P.dcn(xa, d, bn)
    P.finalize()
    x = torch.from_numpy(gen.standard_normal((B, cin, H, W)).astype(np.float32))
    xa.buf.copy_(x.permute(0, 2, 3, 1).reshape(-1, cin).half().cuda())
    P.run()
    torch.cuda.synchronize()
    om = next(t for t in P.keep if t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == 32).cpu()
    ref = reference(x.half().double(), w.half().double(), bias)
    check(om, ref, FAST_TOL)


@pytest.mark.parametrize("bad", ["cin32", "stride2"])
def test_offset_conv_rejects_unsupported(bad):
    """an offset/mask conv the kernel does not cover is an error, not a silent fall-back"""
    cin, stride = (32, 1) if bad == "cin32" else (64, 2)
    B, H, W = 1, 8, 8
    x = torch.zeros(B * H * W, cin, dtype=torch.half, device="cuda")
    wp = torch.zeros(32, 9 * cin, dtype=torch.half, device="cuda")
    v = torch.zeros(32, dtype=torch.float32, device="cuda")
    Ho = (H + 2 - 3) // stride + 1
    om = torch.zeros(B * Ho * Ho, 32, dtype=torch.float32, device="cuda")
    with pytest.raises(RuntimeError, match="offset/mask conv"):
        call("mf_conv2d_nhwc_f16", x.data_ptr(), cin, B, H, W, cin, wp.data_ptr(), 32, (9 * cin + 63) // 64 * 64, 3, 3, stride,
             1, 27, v.data_ptr(), v.data_ptr(), None, 0, engine.ACT_OFFMASK, engine.OUT_F32_NHWC, om.data_ptr(), 32, stream())
