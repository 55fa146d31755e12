"""-m gpu: the wide-gather configuration of the fused DCN (64-column tiles: 16 gather warps, one consumer warpgroup that
finishes its own tiles) where the model's shapes do not take it: Cout < 64 (padded N), maps ragged against the 8 x 16
pixel tile, tile lists that wrap the persistent grid several times and end on a partial tile, and the direct-store output
forms. Checked against the float64 reference of tests/dcn_ref.py on its edge menu, at the tolerances of
tests/test_gpu_dcn_edges.py."""
import numpy as np
import pytest
import torch

import dcn_ref
from gpu_util import FakeBN, to_rows, to_rows_split
from monoflex_b200 import engine
from monoflex_b200._lib import call, stream

pytestmark = pytest.mark.gpu

FAST_TOL, STRICT_TOL = 1.5e-3, 3e-5

# (B, Cin, Cout, H, W)
CASES = [
    (2, 64, 48, 13, 41),       # padded N (48 of 64 columns), H and W not multiples of 8 and 16
    (3, 128, 64, 50, 100),     # 3 x 7 x 7 = 147 tiles per image, 441 in all: the grid wraps three times, partial last tile
    (1, 256, 40, 9, 7),        # fewer tiles than SMs, W < 16
    (4, 64, 33, 37, 45),       # the narrowest Cout of a 64-column tile, 4 x 5 x 3 tiles per image
]


def h16(t):
    return t.half().float()


def rel(got, want):
    got, want = got.double(), want.double()
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def nchw(rows, B, H, W):
    return rows.reshape(B, H, W, -1).permute(0, 3, 1, 2)


def setup(case, strict):
    B, cin, cout, H, W = case
    gen = np.random.Generator(np.random.PCG64(B * 1000 + cin + cout + H * W))
    x = torch.from_numpy(gen.standard_normal((B, cin, H, W)).astype(np.float32))
    wt = torch.from_numpy((gen.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin)).astype(np.float32))
    wt = wt if strict else h16(wt)
    bias = torch.from_numpy((gen.standard_normal(cout) * 0.1).astype(np.float32)).cuda()
    bn = FakeBN(cout, gen)
    offset, mask, _ = dcn_ref.edge_menu(B, H, W, seed=cin + cout + H)
    offset, mask = offset.cuda(), mask.cuda()
    om = dcn_ref.to_offmask_rows(offset, mask)
    P = engine.Plan("cuda", strict=strict)
    wp, n_pad, k_pad = P.pack_weight(wt.cuda(), split=strict)
    assert n_pad == 64, n_pad                                        # one 64-column tile: the wide-gather configuration
    scale, shift = P.affine(cout, n_pad, bn, bias)
    return x, wt, offset, mask, om, wp, n_pad, k_pad, scale, shift


def reference(xv, wt, offset, mask, scale, shift, act_relu):
    """float64: DCN columns on the given offsets and masks, contracted with W, scale / shift, optional ReLU; NCHW"""
    cout, cin = wt.shape[:2]
    B, _, H, W = xv.shape
    cols = dcn_ref.columns(xv, offset, mask)
    ref = torch.einsum("okt,bkthw->bohw", wt.cuda().double().view(cout, cin, 9), cols)
    ref = ref * scale[:cout].double().view(1, -1, 1, 1) + shift[:cout].double().view(1, -1, 1, 1)
    return ref.clamp_min(0.0) if act_relu else ref


@pytest.mark.parametrize("prec", ["fast", "strict"])
@pytest.mark.parametrize("case", CASES)
def test_wide_gather_against_float64(case, prec):
    """the fused DCN (ReLU epilogue, staged TMA-store output) against float64; the output channels past the tile's
    boxes stay untouched"""
    B, cin, cout, H, W = case
    M = B * H * W
    strict = prec == "strict"
    x, wt, offset, mask, om, wp, n_pad, k_pad, scale, shift = setup(case, strict)
    SENT = 1000.0
    ly = (cout + 7) // 8 * 8 + 64                                    # rows wider than the tile: the rest stays untouched
    if strict:
        xs = to_rows_split(x)
        y = torch.full((M, 2 * ly), SENT, dtype=torch.half, device="cuda")
        call("mf_dcn_nhwc_f16x2", xs.data_ptr(), 2 * cin, cin, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad,
             cout, scale.data_ptr(), shift.data_ptr(), engine.ACT_RELU, y.data_ptr(), 2 * ly, ly, stream())
        xv = xs[:, :cin].double() + xs[:, cin:].double()
        got = y[:, :cout].double() + y[:, ly:ly + cout].double()
        inside = torch.zeros(2 * ly, dtype=torch.bool, device="cuda")
        inside[:64] = inside[ly:ly + 64] = True                      # a 64-column tile stores all 64 columns of its box
    else:
        xr = to_rows(x)
        y = torch.full((M, ly), SENT, dtype=torch.half, device="cuda")
        call("mf_dcn_nhwc_f16", xr.data_ptr(), cin, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, cout,
             scale.data_ptr(), shift.data_ptr(), engine.ACT_RELU, engine.OUT_F16_NHWC, y.data_ptr(), ly, stream())
        xv = xr.double()
        got = y[:, :cout].double()
        inside = torch.zeros(ly, dtype=torch.bool, device="cuda")
        inside[:64] = True
    torch.cuda.synchronize()
    assert (y[:, ~inside] == SENT).all(), (prec, case, "channels past the tile were written")
    assert torch.isfinite(got).all(), (prec, case, "rows left unwritten")
    ref = reference(nchw(xv, B, H, W), wt, offset, mask, scale, shift, True)
    tol = STRICT_TOL if strict else FAST_TOL
    assert rel(nchw(got, B, H, W), ref) < tol, (prec, case, rel(nchw(got, B, H, W), ref))


@pytest.mark.parametrize("out", ["f16_unstaged", "f32_nhwc", "f32_nchw"])
@pytest.mark.parametrize("case", CASES[:2])
def test_wide_gather_direct_stores(case, out):
    """fast precision, the output forms without the TMA store: fp16 rows whose stride is not a multiple of 8, fp32 rows,
    fp32 NCHW planes (no activation, so negative values are checked too)"""
    B, cin, cout, H, W = case
    M = B * H * W
    x, wt, offset, mask, om, wp, n_pad, k_pad, scale, shift = setup(case, False)
    xr = to_rows(x)
    SENT = 1000.0
    if out == "f16_unstaged":
        ld = 68                                                       # 8-byte aligned rows: no TMA store
        y = torch.full((M, ld), SENT, dtype=torch.half, device="cuda")
        mode = engine.OUT_F16_NHWC
    elif out == "f32_nhwc":
        ld = 64
        y = torch.full((M, ld), SENT, dtype=torch.float32, device="cuda")
        mode = engine.OUT_F32_NHWC
    else:
        ld = cout
        y = torch.full((B, cout, H, W), SENT, dtype=torch.float32, device="cuda")
        mode = engine.OUT_F32_NCHW
    call("mf_dcn_nhwc_f16", xr.data_ptr(), cin, B, H, W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, cout,
         scale.data_ptr(), shift.data_ptr(), engine.ACT_NONE, mode, y.data_ptr(), ld, stream())
    torch.cuda.synchronize()
    if out == "f32_nchw":
        got = y.double()
    else:
        assert (y[:, 64:] == SENT).all(), (out, case, "channels past the tile were written")
        got = nchw(y[:, :cout].double(), B, H, W)
    assert torch.isfinite(got).all() and (got != SENT).all(), (out, case, "elements left unwritten")
    ref = reference(nchw(xr.double(), B, H, W), wt, offset, mask, scale, shift, False)
    assert rel(got, ref) < FAST_TOL, (out, case, rel(got, ref))
