"""Host side of the convolution backward edge tests (no GPU): the float64 references and their absolute-value twins
against float64 autograd and explicit sums, the launch emulations against the launchers' formulas, the case lists
against the edges they are meant to place, and - on the GPU test's own shapes and inputs - the per-element bounds
rejecting "near-miss" results built on the CPU: the ragged last 64-pixel block left out of the reduction, one tap's dY
read one pixel late, one split's sum added twice, one dgrad tap not rotated, and the stride-2 interleave's parities
swapped. A kernel with one of those defects would fail the GPU test."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_backward_ref as R
import test_gpu_conv_backward_edges as G

NSM = 132          # H100 SXM, what the case list's split regimes are written for
MISS_MARGIN = 4    # a near miss must exceed its bound by at least this factor somewhere


def leaf(t):
    return t.clone().double().requires_grad_(True)


# ------------------------------------------------------------------------------------------------ references
@pytest.mark.parametrize("k,stride,pad", [(1, 1, 0), (3, 1, 1), (3, 2, 1), (7, 2, 3), ((1, 3), 1, 0)])
def test_conv_refs_match_autograd(k, stride, pad):
    gen = torch.Generator().manual_seed(3)
    kh, kw = R.pair(k)
    x = torch.randn(2, 5, 7, 9, generator=gen, dtype=torch.float64)
    w = torch.randn(6, 5, kh, kw, generator=gen, dtype=torch.float64)
    xl, wl = leaf(x), leaf(w)
    y = F.conv2d(xl, wl, stride=stride, padding=pad)
    dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    y.backward(dy)
    dw, A = R.wgrad_ref(x, dy, k, stride, pad)
    assert (dw - wl.grad).abs().max().item() < 1e-12
    assert torch.allclose(R.wgrad_ref(x, dy, k, stride, pad, per_image=True)[0], dw, rtol=0, atol=1e-12)
    # A = sum over pixels of |x| |dy| per weight, from the explicit im2col
    cols = F.unfold(x.abs(), (kh, kw), padding=R.pair(pad), stride=stride)           # [B, Cin kh kw, L]
    A2 = torch.einsum("bol,bcl->oc", dy.abs().flatten(2), cols).reshape(A.shape)
    assert torch.allclose(A, A2, rtol=1e-12, atol=0)
    if kh == kw:
        dx, Ax = R.dgrad_ref(dy, w, x.shape[2:], stride, pad)
        assert (dx - xl.grad).abs().max().item() < 1e-12
        assert torch.allclose(Ax, torch.nn.grad.conv2d_input(x.shape, w.abs(), dy.abs(), stride=stride, padding=pad))
        assert (Ax >= dx.abs() - 1e-12).all()


@pytest.mark.parametrize("f", [2, 4])
def test_upsample_ref_matches_autograd(f):
    gen = torch.Generator().manual_seed(f)
    C = 8
    x = leaf(torch.randn(2, C, 3, 4, generator=gen, dtype=torch.float64))
    w = torch.randn(C, 1, 2 * f, 2 * f, generator=gen, dtype=torch.float64)
    y = F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=C)
    dy = torch.randn(y.shape, generator=gen, dtype=torch.float64)
    y.backward(dy)
    dx, A = R.upsample_dx_ref(dy, w, f)
    assert (dx - x.grad).abs().max().item() < 1e-12
    assert (A >= dx.abs() - 1e-12).all() and A.min().item() > 0


# ------------------------------------------------------------------------------------------------ launch emulations
def test_wgrad_plan_partitions_the_blocks():
    for case in G.WGRAD_CASES:
        B, H, W, Cin, Cout, k, s, pad, _ = case
        p = R.wgrad_plan(B, H, W, Cin, Cout, k, s, pad, NSM)
        assert p["ranges"][0][0] == 0 and p["ranges"][-1][1] == p["nkb"]
        assert all(a[1] == b[0] for a, b in zip(p["ranges"], p["ranges"][1:]))
        assert all(hi > lo for lo, hi in p["ranges"]), case                      # no empty split
        assert max(hi - lo for lo, hi in p["ranges"]) * R.WG_BK == p["P"]
        assert p["splits"] <= p["nkb"] and (p["nkb"] - 1) * R.WG_BK < p["M"] <= p["nkb"] * R.WG_BK


def test_narrow_plan_and_dead_taps():
    p = R.narrow_plan(3, 5, 33, 3, NSM)
    assert (p["nblocks"], p["nunits"], p["last_unit_half"]) == (45, 23, True)
    assert sorted({ky for ky, _ in G.dead_taps(2, 40, 7)}) == [0, 1, 5, 6]
    assert G.dead_taps(1, 1, 3) == [(ky, kx) for ky in range(3) for kx in range(3) if (ky, kx) != (1, 1)]
    x, dy = G.wgrad_inputs(1, 2, 1, 16, 16, 7, 1, 3, 0)
    _, A = R.wgrad_ref(x, dy, 7, 1, 3)
    for ky, kx in G.dead_taps(2, 1, 7):
        assert A[:, :, ky, kx].abs().max().item() == 0


# ------------------------------------------------------------------------------------------------ case coverage
def test_case_lists_place_the_edges():
    cases = [c[:8] for c in G.WGRAD_CASES]
    plans = [R.wgrad_plan(*c, NSM) for c in cases]
    assert {(c[3], c[4]) for c in cases} >= {(i, o) for i in (16, 32, 64, 192, 512) for o in (16, 32, 64, 192, 256)}
    assert {c[5] for c in cases} == {1, 3, 7} and {c[6] for c in cases} == {1, 2}
    assert all(c[7] in (0, c[5] // 2) for c in cases)
    assert not any(R.goes_narrow(c[3], c[4], c[5], c[6], c[7]) for c in cases)
    assert [p["regime"] for p in plans] == [c[8] for c in G.WGRAD_CASES]
    assert {p["regime"] for p in plans} == {"one split", "one block per split", "even", "remainder"}
    assert any(p["regime"] == "one block per split" and p["nkb"] > 1 for p in plans)
    assert {(p["aw"], p["dummies"]) for p in plans} >= {(16, 7), (32, 3), (64, 1)}
    assert any(c[3] == 192 and c[5] == 1 for c in cases)                       # 1x1 with Cin / 64 odd
    assert any(c[1] == 1 for c in cases) and any(c[2] == 1 for c in cases)
    assert any(c[1] < c[5] and c[2] < c[5] for c in cases)
    assert any(c[6] == 2 and (c[1] % 2 or c[2] % 2) for c in cases)
    assert any(c[0] == 3 and p["nkb"] > 1 for c, p in zip(cases, plans))
    assert any(p["ragged"] and p["nkb"] > p["splits"] > 1 for p in plans)
    units = [R.narrow_plan(B, H, W, k, NSM) for k, W, H, B in G.NARROW_CASES if k == 3]
    assert {u["last_unit_half"] for u in units} == {True, False}
    assert set(G.upsample_cases()) and {c[4] for c in G.upsample_cases()} == set(G.model_shapes()[3])
    assert any(c[1] == 1 for c in G.dgrad1_cases()) and any(c[2] == 1 for c in G.dgrad1_cases())
    assert any(c[1] == 2 for c in G.dgrad2_cases()) and any(c[2] == 2 for c in G.dgrad2_cases())
    assert [c[3:] for c in G.dgrad2_cases()] == [(16, 32), (32, 64), (64, 128), (128, 256), (256, 512)]


# ------------------------------------------------------------------------------------------------ near misses
def wgrad_margin(miss, ref, A, plan):
    return R.ratio((miss - ref).abs(), R.wgrad_bound(A, plan["P"], plan["S"]))


NEAR_CASES = [c for c in G.WGRAD_CASES if c[:3] != G.LONG]     # the long case's single block is within its bound


@pytest.mark.parametrize("case", NEAR_CASES, ids=["B%d-%dx%d-%d-%d-k%d-s%d-p%d" % c[:8] for c in NEAR_CASES])
def test_wgrad_bound_rejects_near_misses(case):
    B, H, W, Cin, Cout, k, s, pad, _ = case
    i = G.WGRAD_CASES.index(case)
    x, dy = G.wgrad_inputs(B, H, W, Cin, Cout, k, s, pad, 100 + i)
    plan = R.wgrad_plan(B, H, W, Cin, Cout, k, s, pad, NSM)
    ref, A = R.wgrad_ref(x, dy, k, s, pad)
    assert wgrad_margin(ref, ref, A, plan) == 0
    margins = {}
    if plan["nkb"] > 1 and plan["ragged"]:
        margins["last block dropped"] = wgrad_margin(R.miss_last_block_dropped(x, dy, k, s, pad), ref, A, plan)
    centre = (k // 2) * k + k // 2
    margins["tap shifted"] = wgrad_margin(R.miss_tap_shifted(x, dy, k, s, pad, centre), ref, A, plan)
    margins["split twice"] = wgrad_margin(R.miss_split_twice(x, dy, k, s, pad, plan), ref, A, plan)
    print(case[:8], {n: "%.3g" % v for n, v in margins.items()})
    assert all(v >= MISS_MARGIN for v in margins.values()), margins


@pytest.mark.parametrize("case", G.NARROW_CASES[::3], ids=["k%d-W%d-H%d-B%d" % c for c in G.NARROW_CASES[::3]])
def test_narrow_bound_rejects_a_shifted_tap(case):
    k, W, H, B = case
    x, dy = G.wgrad_inputs(B, H, W, 16, 16, k, 1, k // 2, 1000 + 100 * k + 10 * W + H + B)
    plan = R.narrow_plan(B, H, W, k, NSM)
    ref, A = R.wgrad_ref(x, dy, k, 1, k // 2)
    if B * H * W == 1:
        pytest.skip("one pixel: no neighbour to shift to")
    m = wgrad_margin(R.miss_tap_shifted(x, dy, k, 1, k // 2, (k // 2) * k + k // 2), ref, A, plan)
    assert m >= MISS_MARGIN, m


@pytest.mark.parametrize("case", [c for c in G.dgrad1_cases() if c[5] == 3], ids=lambda c: "B%d-%dx%d-%d-%d-k%d-pad%d-dypad%d" % c)
def test_dgrad_bound_rejects_an_unrotated_tap(case):
    B, H, W, Cin, Cout, k, pad, _ = case
    dy, w = G.dgrad_inputs(B, H, W, Cin, Cout, k, 200 + Cin + Cout + k)
    w16 = w.half().double()
    ref, A = R.dgrad_ref(dy, w16, (H, W), 1, pad)
    tap = (0 if H > 1 else 1) * k + (0 if W > 1 else 1)         # a tap whose mirror image reads the image, not padding
    miss = R.miss_tap_unrotated(dy, w16, (H, W), 1, pad, tap)
    m = R.ratio((miss - ref).abs(), R.dgrad_bound(ref, A, k * k * Cout))
    assert m >= MISS_MARGIN, m


@pytest.mark.parametrize("case", G.dgrad2_cases(), ids=lambda c: "B%d-%dx%d-%d-%d" % c)
def test_dgrad_stride2_bound_rejects_swapped_parities(case):
    B, H, W, Cin, Cout = case
    dy, w = G.dgrad_inputs(B, H // 2, W // 2, Cin, Cout, 3, 400 + Cin + H)
    ref, A = R.dgrad_ref(dy, w.half().double(), (H, W), 2, 1)
    m = R.ratio((R.miss_parities_swapped(ref) - ref).abs(), R.dgrad_bound(ref, A, 9 * Cout))
    m_rot = R.ratio((R.miss_tap_unrotated(dy, w.half().double(), (H, W), 2, 1, tap=0) - ref).abs(),
                    R.dgrad_bound(ref, A, 9 * Cout))
    assert m >= MISS_MARGIN and m_rot >= MISS_MARGIN, (m, m_rot)


def test_ratio_semantics():
    z = torch.zeros(3, dtype=torch.float64)
    assert R.ratio(z, z) == 0.0
    assert R.ratio(torch.tensor([0.0, 1e-300], dtype=torch.float64), torch.tensor([1.0, 0.0])) == float("inf")     # nonzero where A = 0
    assert R.ratio(torch.tensor([float("nan"), 0.0]), torch.tensor([1.0, 1.0])) == float("inf")
    assert R.ratio(torch.tensor([0.5, 2.0]), torch.tensor([1.0, 4.0])) == 0.5
