"""The float64 per-record references of tests/tape_ref.py against torch autograd of the same layer, on small CPU tensors
away from the activation kinks: the layer-by-layer tape test (test_gpu_tape_layers.py) is only as good as they are."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcn_ref
import tape_ref


def _gen(seed):
    g = torch.Generator().manual_seed(seed)
    return lambda *shape, scale=1.0: torch.randn(*shape, generator=g, dtype=torch.float64) * scale


def _close(a, b, tol=1e-12):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1e-300)


@pytest.mark.parametrize("act", [tape_ref.ACT_NONE, tape_ref.ACT_RELU, tape_ref.ACT_LEAKY])
@pytest.mark.parametrize("stride,k,residual,abs_weight", [(1, 3, True, False), (2, 3, False, False), (1, 1, True, True),
                                                          (1, 7, False, False)])
def test_conv_bn_residual_act(act, stride, k, residual, abs_weight):
    r = _gen(10 * stride + k + act)
    B, Cin, Cout, H, W = 2, 5, 6, 9, 8
    x, w = r(B, Cin, H, W).requires_grad_(True), r(Cout, Cin, k, k, scale=0.3).requires_grad_(True)
    gamma, beta = r(Cout).requires_grad_(True), r(Cout, scale=0.1).requires_grad_(True)
    raw = F.conv2d(x, w, None, stride, k // 2)
    res = r(*raw.shape).requires_grad_(True) if residual else None
    raw.retain_grad()
    g_eff = gamma.abs() + 1e-5 if abs_weight else gamma
    z = F.batch_norm(raw, None, None, g_eff, beta, True, 0.0, 1e-5) + (res if residual else 0)
    y = {0: lambda v: v, 1: F.relu, 2: lambda v: F.leaky_relu(v, 0.01)}[act](z)
    dy = r(*y.shape)
    y.backward(dy)
    assert z.detach().abs().min().item() > 1e-6                          # away from the kink
    d_raw, d_res, dgamma, dbeta = tape_ref.bn_backward(raw.detach(), y.detach(), dy, gamma.detach(), 1e-5, act, abs_weight)
    _close(d_raw, raw.grad)
    _close(dgamma, gamma.grad)
    _close(dbeta, beta.grad)
    if residual:
        _close(d_res, res.grad)
    dx, dw = tape_ref.conv_backward(x.detach(), w.detach(), d_raw, stride, k // 2)
    _close(dx, x.grad)
    _close(dw, w.grad)


def test_bn_backward_1d():
    """BatchNorm1d over [B, C, L] (the edge-fusion tail), identity activation"""
    r = _gen(3)
    raw, gamma, beta = r(2, 4, 11).requires_grad_(True), r(4).requires_grad_(True), r(4).requires_grad_(True)
    y = F.batch_norm(raw, None, None, gamma, beta, True, 0.0, 1e-5)
    dy = r(*y.shape)
    y.backward(dy)
    d_raw, _, dgamma, dbeta = tape_ref.bn_backward(raw.detach(), y.detach(), dy, gamma.detach(), 1e-5, tape_ref.ACT_NONE)
    _close(d_raw, raw.grad)
    _close(dgamma, gamma.grad)
    _close(dbeta, beta.grad)


def test_act_mask_takes_the_sign_of_the_output():
    y = torch.tensor([-1.0, -0.0, 0.0, 2.0], dtype=torch.half)
    assert tape_ref.act_mask(y, tape_ref.ACT_RELU).tolist() == [0, 0, 0, 1]
    assert tape_ref.act_mask(y, tape_ref.ACT_LEAKY).tolist() == [0.01, 0.01, 0.01, 1]
    assert tape_ref.act_mask(y, tape_ref.ACT_NONE).tolist() == [1, 1, 1, 1]


def _dcn_forward(x, w, b, offset, pre):
    """out = b + W . columns, with a differentiable bilinear sampler that forms the coordinates exactly like dcn_ref"""
    B, C, H, W = x.shape
    h, wc = dcn_ref.coords(offset.detach())                       # float32-formed coordinates, float64
    h = h + (offset.view(B, 9, 2, H, W)[:, :, 0] - offset.view(B, 9, 2, H, W)[:, :, 0].detach())
    wc = wc + (offset.view(B, 9, 2, H, W)[:, :, 1] - offset.view(B, 9, 2, H, W)[:, :, 1].detach())
    m = torch.sigmoid(pre)
    inside = ((h > -1) & (wc > -1) & (h < H) & (wc < W)).detach()
    hl, wl = torch.floor(h.detach()), torch.floor(wc.detach())
    lh, lw = h - hl, wc - wl
    xf = x.reshape(B, C, H * W)
    cols = 0
    for dr, dc, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
        rr, cc = hl.long() + dr, wl.long() + dc
        ok = (inside & (rr >= 0) & (rr <= H - 1) & (cc >= 0) & (cc <= W - 1)).double()
        idx = (rr.clamp(0, H - 1) * W + cc.clamp(0, W - 1)).view(B, 1, -1).expand(B, C, -1)
        v = xf.gather(2, idx).view(B, C, 9, H, W)
        cols = cols + (m * wt * ok).unsqueeze(1) * v
    return torch.einsum("oct,bcthw->bohw", w.reshape(w.shape[0], C, 9), cols) + b.view(1, -1, 1, 1)


def test_dcn_backward():
    r = _gen(4)
    B, C, Co, H, W = 2, 3, 4, 6, 7
    x, w, b = r(B, C, H, W).requires_grad_(True), r(Co, C, 3, 3, scale=0.3).requires_grad_(True), r(Co).requires_grad_(True)
    # offsets away from integers (bilinear kinks), some of them far outside the image
    off = (torch.rand(B, 18, H, W, generator=torch.Generator().manual_seed(5), dtype=torch.float64) * 0.8 + 0.1) * \
        torch.where(r(B, 18, H, W) > 0, 1.0, -1.0).double() + r(B, 18, H, W).round()
    off = off.float().double().requires_grad_(True)
    pre = r(B, 9, H, W).requires_grad_(True)
    out = _dcn_forward(x, w, b, off, pre)
    dy = r(*out.shape)
    out.backward(dy)
    # the kernels keep the SIGMOID-ED mask in float32
    mask = torch.sigmoid(pre.detach())
    dx, d_off, d_pre, dw, db = tape_ref.dcn_backward(x.detach(), off.detach().float(), mask, w.detach(), dy)
    _close(dx, x.grad)
    _close(d_off, off.grad)
    _close(d_pre, pre.grad)
    _close(dw, w.grad)
    _close(db, b.grad)
    # and the same forward is the oracle's DCNv2
    from oracle import monoflex_oracle as mo
    ref = mo.dcn_v2_forward(x.detach().float(), w.detach().float(), b.detach().float(), off.detach().float(), mask.float())
    assert (ref.double() - out.detach()).abs().max().item() <= 1e-5 * out.abs().max().item()


def test_maxpool2_backward_first_maximum_on_ties():
    """ties everywhere (ReLU zeros, repeated values): the gradient goes where torch's max_pool2d sends it"""
    r = _gen(6)
    x = F.relu(r(2, 3, 8, 10)).round()                                # mostly exact zeros and small integers: many ties
    x.requires_grad_(True)
    dy = r(2, 3, 4, 5)
    F.max_pool2d(x, 2).backward(dy)
    win = x.detach().reshape(2, 3, 4, 2, 5, 2)
    n_tied = ((win == win.amax((3, 5), keepdim=True)).sum((3, 5)) > 1).sum().item()
    assert n_tied > 20
    assert torch.equal(tape_ref.maxpool2_backward(x.detach(), dy), x.grad)


@pytest.mark.parametrize("f", [2, 4])
def test_upsample_backward(f):
    r = _gen(7 + f)
    B, C, Hi, Wi = 2, 3, 4, 5
    x, w = r(B, C, Hi, Wi).requires_grad_(True), r(C, 1, 2 * f, 2 * f).requires_grad_(True)
    skip = r(B, C, Hi * f, Wi * f).requires_grad_(True)
    y = F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=C) + skip
    dy = r(*y.shape)
    y.backward(dy)
    dx, dw, dskip = tape_ref.upsample_backward(x.detach(), w.detach(), dy, f)
    _close(dx, x.grad)
    _close(dw, w.grad)
    assert torch.equal(dskip, skip.grad)
    assert np.isfinite(dw.numpy()).all()
