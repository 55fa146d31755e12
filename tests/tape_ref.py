"""Float64 backward of each kind of training-tape record (monoflex_b200/tape.py::backbone_backward), taken at the forward
point the kernels recorded: the caller passes the recorded fp16 tensors widened to float64, and the activation mask comes
from the sign of the recorded output, as the BN backward kernel takes it. Every function works on CPU and CUDA tensors
in NCHW (or [B, C, L]) layout and returns float64. Checked against torch autograd by tests/test_tape_ref_host.py.
"""
import torch
import torch.nn.functional as F

import dcn_ref

ACT_NONE, ACT_RELU, ACT_LEAKY = 0, 1, 2          # engine.ACT_*


def act_mask(y, act):
    """derivative of the activation from the sign of its output y: ReLU 0 / 1, leaky_relu(0.01) 0.01 / 1, identity 1"""
    pos = y.double() > 0
    if act == ACT_RELU:
        return pos.double()
    if act == ACT_LEAKY:
        return torch.full_like(y, 0.01, dtype=torch.float64).masked_fill(pos, 1.0)
    return torch.ones_like(y, dtype=torch.float64)


def bn_xhat(raw, eps):
    """(xhat, rstd) of training-mode BatchNorm: statistics over every dimension but 1, biased variance (float64)"""
    raw = raw.double()
    dims = [d for d in range(raw.dim()) if d != 1]
    mean = raw.mean(dims, keepdim=True)
    rstd = (((raw - mean) ** 2).mean(dims, keepdim=True) + eps).rsqrt()
    return (raw - mean) * rstd, rstd


def bn_backward(raw, y, dy, gamma, eps, act, abs_weight=False, count=None, rows=None):
    """y = act(BN_train(raw; gamma, beta) + residual), biased batch variance over every dimension but 1 ->
    (d_raw, d_residual, dgamma, dbeta). abs_weight: InPlaceABN's |gamma| + eps, dgamma carries sign(gamma).
    count: the element count dividing the sums in d_raw (a SyncBatchNorm's global count; raw's own by default); rows: a
    0/1 mask, broadcastable to raw, of the elements the sums take (all by default)."""
    dy, gamma = dy.double(), gamma.double()
    dims = [d for d in range(raw.dim()) if d != 1]
    shape = [1, -1] + [1] * (raw.dim() - 2)
    xhat, rstd = bn_xhat(raw, eps)
    g = dy * act_mask(y, act)
    gs = g if rows is None else g * rows.double()
    sg, sgx = gs.sum(dims, keepdim=True), (gs * xhat).sum(dims, keepdim=True)
    n = raw.numel() // raw.shape[1] if count is None else count
    g_eff = gamma.abs() + eps if abs_weight else gamma
    d_raw = g_eff.view(shape) * rstd * (g - sg / n - xhat * sgx / n)
    dgamma = sgx.flatten()
    if abs_weight:
        dgamma = dgamma * torch.sign(gamma)
    return d_raw, g, dgamma, sg.flatten()


def conv_backward(x, weight, d_out, stride, pad):
    """y = conv2d(x, weight, stride, pad) -> (dx, dW)"""
    x, w, d = x.double(), weight.double(), d_out.double()
    dx = torch.nn.grad.conv2d_input(x.shape, w, d, stride=stride, padding=pad)
    dw = torch.nn.grad.conv2d_weight(x, w.shape, d, stride=stride, padding=pad)
    return dx, dw


def dcn_backward(x, offset, mask, weight, d_out):
    """out = bias + W . dcn_ref.columns(x, offset, mask) (DCNv2, 3x3, stride 1, pad 1), mask = sigmoid(pre) ->
    (dx, d_offset [B, 18, H, W], d_pre [B, 9, H, W], dW, dbias)"""
    B, C, H, W = x.shape
    cout = weight.shape[0]
    w = weight.double().reshape(cout, C, 9)
    d = d_out.double()
    gcol = torch.einsum("oct,bohw->bcthw", w, d)
    dx, d_off, d_mask = dcn_ref.backward(x, offset, mask, gcol)
    m = mask.double()
    cols = dcn_ref.columns(x, offset, mask)
    dw = torch.einsum("bohw,bcthw->oct", d, cols).reshape(cout, C, 3, 3)
    return dx, d_off, d_mask * m * (1 - m), dw, d.sum((0, 2, 3))


def maxpool2_backward(x, dy):
    """MaxPool2d(2): each output gradient goes to the FIRST maximum of its window in scan order (0,0) (0,1) (1,0) (1,1)"""
    B, C, H, W = x.shape
    win = x.double().reshape(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)
    first = win == win.max(-1, keepdim=True).values
    first = first & (first.cumsum(-1) == 1)
    dx = first.double() * dy.double().unsqueeze(-1)
    return dx.reshape(B, C, H // 2, W // 2, 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H, W)


def upsample_backward(x, weight, dy, f):
    """y = depth-wise conv_transpose2d(x, weight [C, 1, 2f, 2f], stride f, pad f/2) + skip -> (dx, dW, dskip)"""
    C = x.shape[1]
    d = dy.double()
    dx = F.conv2d(d, weight.double(), None, stride=f, padding=f // 2, groups=C)
    # dW[c, 0, ky, kx] = sum over b, i, j of x[b, c, i, j] * dy[b, c, f i - f/2 + ky, f j - f/2 + kx]
    xs = x.double()
    k = weight.shape[2]
    dp = F.pad(d, (f // 2, f // 2, f // 2, f // 2))
    Hi, Wi = x.shape[2], x.shape[3]
    dw = torch.empty(C, 1, k, k, dtype=torch.float64, device=x.device)
    for ky in range(k):
        for kx in range(k):
            win = dp[:, :, ky:ky + f * (Hi - 1) + 1:f, kx:kx + f * (Wi - 1) + 1:f]
            dw[:, 0, ky, kx] = (xs * win).sum((0, 2, 3))
    return dx, dw, d
