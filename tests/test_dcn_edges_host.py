"""CPU: pin the float64 DCNv2 reference of tests/dcn_ref.py to the reference's own three C loops (im2col, col2im,
col2im_coord of src/cpu/dcn_v2_im2col_cpu.cpp, built into oracle/_ref by oracle/Makefile) on the edge menu: samples on the
pixel grid, on the image border, in the bands just inside it, far outside it, and 1e-8 off the grid."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcn_ref
from conftest import ROOT

LIB = os.path.join(ROOT, "oracle", "_ref", "libdcn_im2col_ref.so")
B, C, H, W = 2, 13, 10, 12          # C not a multiple of 8; H, W >= len(REGIMES): every regime on every border
U32 = 2.0 ** -24


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(LIB):
        pytest.skip("oracle/_ref not built")
    return ctypes.CDLL(LIB)


@pytest.fixture(scope="module")
def case():
    gen = np.random.Generator(np.random.PCG64(11))
    x = torch.from_numpy(gen.standard_normal((B, C, H, W)).astype(np.float32))
    offset, mask, regs = dcn_ref.edge_menu(B, H, W, seed=12)
    gcol = torch.from_numpy(gen.standard_normal((B, C, 9, H, W)).astype(np.float32))
    return x, offset, mask, gcol, regs


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


GEOM = (H, W, 3, 3, 1, 1, 1, 1, 1, 1, 1)     # height_col, width_col, kernel, pad, stride, dilation, deformable groups


def ref_im2col(lib, x, offset, mask):
    cols = torch.zeros(B, C * 9, H * W)
    lib.modulated_deformable_im2col_cpu(_p(x), _p(offset), _p(mask), B, C, H, W, *GEOM, _p(cols))
    return cols.view(B, C, 9, H, W)


def ref_backward(lib, x, offset, mask, gcol):
    """col2im and col2im_coord read the column gradient in the reference's [C*9, B, H*W] layout"""
    data_col = gcol.permute(1, 2, 0, 3, 4).contiguous()
    grad_im = torch.zeros(B, C, H, W)
    lib.modulated_deformable_col2im_cpu(_p(data_col), _p(offset), _p(mask), B, C, H, W, *GEOM, _p(grad_im))
    grad_off = torch.zeros(B, 18, H, W)
    grad_mask = torch.zeros(B, 9, H, W)
    lib.modulated_deformable_col2im_coord_cpu(_p(data_col), _p(x), _p(offset), _p(mask), B, C, H, W, *GEOM, _p(grad_off),
                                              _p(grad_mask))
    return grad_im, grad_off, grad_mask


def _worst(got, want):
    d = (got.double() - want.double()).abs()
    i = int(d.argmax())
    return d.max().item(), np.unravel_index(i, tuple(d.shape)), got.reshape(-1)[i].item(), want.reshape(-1)[i].item()


def test_edge_menu_covers_every_regime_on_every_border(case):
    _, offset, mask, _, (reg_h, reg_w) = case
    R = len(dcn_ref.REGIMES)
    for name, reg in (("h", reg_h), ("w", reg_w)):
        for tap in range(9):
            for side, sel in (("top", reg[:, tap, 0, :]), ("bottom", reg[:, tap, H - 1, :]), ("left", reg[:, tap, :, 0]),
                              ("right", reg[:, tap, :, W - 1])):
                assert set(np.unique(sel)) == set(range(R)), (name, tap, side)
    h, w = dcn_ref.coords(offset)
    for v in (-1.0, H - 1.0, float(H)):
        assert (h == v).any(), v
    for v in (-1.0, W - 1.0, float(W)):
        assert (w == v).any(), v
    assert ((h > -1) & (h < 0)).any() and ((h > H - 1) & (h < H)).any() and (h.abs() > 1e9).any()
    assert ((w > -1) & (w < 0)).any() and ((w > W - 1) & (w < W)).any() and (w.abs() > 1e9).any()
    for v in (0.0, 0.5, 1.0):
        assert (mask == v).any(), v
    assert ((mask > 0) & (mask < 1) & (mask != 0.5)).any()


def test_columns_match_reference_im2col(lib, case):
    x, offset, mask, _, _ = case
    want = ref_im2col(lib, x, offset, mask)
    got, absum = dcn_ref.columns(x, offset, mask, with_abs=True)
    # the loops blend in float32: three roundings in each corner weight, one per product and per sum
    err = (got - want.double()).abs()
    bound = 8 * U32 * absum + 1e-30
    assert (err <= bound).all(), ("columns", _worst(got, want))


def test_backward_matches_reference_col2im_and_col2im_coord(lib, case):
    x, offset, mask, gcol, _ = case
    want = ref_backward(lib, x, offset, mask, gcol)
    got = dcn_ref.backward(x, offset, mask, gcol)
    for name, g, r in zip(("dX", "dOffset", "dMask"), got, want):
        err, at, gv, rv = _worst(g, r)
        assert err <= 1e-6 * r.abs().max().item(), (name, err, at, gv, rv)
    # and the gradients are not trivially zero on the border regimes
    assert (want[1] != 0).float().mean() > 0.2


def test_tiny_offsets_take_the_one_sided_derivative(lib, case):
    """with the coordinate formed in float64 the same inputs give a different offset gradient wherever h_in + i + 1e-8
    rounds onto the grid in float32: the float32 step is what the reference computes"""
    x, offset, mask, gcol, _ = case
    want = ref_backward(lib, x, offset, mask, gcol)[1]
    exact = dcn_ref.backward(x, offset, mask, gcol, fp32=True)[1]
    wrong = dcn_ref.backward(x, offset, mask, gcol, fp32=False)[1]
    scale = want.abs().max().item()
    assert (exact - want.double()).abs().max().item() <= 1e-6 * scale
    assert (wrong - want.double()).abs().max().item() > 0.1 * scale
    h32, _ = dcn_ref.coords(offset, fp32=True)
    h64, _ = dcn_ref.coords(offset, fp32=False)
    assert ((h32 != h64) & (h32 == torch.round(h32))).any()


def test_zero_offset_half_mask_is_half_im2col(lib):
    """the reference's DCN.init_offset state: every sample on the grid, every mask 0.5 -> cols = 0.5 * im2col(x)"""
    gen = np.random.Generator(np.random.PCG64(13))
    x = torch.from_numpy(gen.standard_normal((B, C, H, W)).astype(np.float32))
    offset = torch.zeros(B, 18, H, W)
    mask = torch.full((B, 9, H, W), 0.5)
    unfold = F.unfold(x.double(), 3, padding=1).view(B, C, 9, H, W)
    assert torch.equal(dcn_ref.columns(x, offset, mask), 0.5 * unfold)
    assert torch.equal(ref_im2col(lib, x, offset, mask).double(), 0.5 * unfold)
