"""Backward building blocks of the convolutional layers (training path of SURVEY §8 rows R2/R3/R6; the reference gets
them from cuDNN through autograd, engine/trainer.py:116-117). Both run on the hand-written tensor-core kernels:

  * conv2d_wgrad : dW from NHWC fp16 activations and output gradients - `mf_conv2d_wgrad_nhwc_f16` (csrc/mf_wgrad.cu:
                   wgmma GEMM whose MN-major operands come straight from im2col / tiled TMA boxes, split-K);
  * conv2d_dgrad : dX of a stride-1 convolution = the forward implicit-GEMM kernel (csrc/mf_igemm2.cu) run on dY with the
                   180-degree rotated, in/out-transposed weights and padding k-1-p (no new kernel); 3x3 stride-2 layers
                   use the four-parity decomposition (`conv2d_dgrad_stride2`).

These are operators with parity tests (tests/test_gpu_train.py); `tape.py` / `head_backward.py` chain them into the whole-
network backward that KeypointDetector's tape bridge (model/detector.py) runs under `losses.backward()`.
"""
import torch

from . import engine
from ._lib import call


def _rows(t, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.half and t.dim() == 2 and t.is_contiguous()):
        raise RuntimeError("%s must be a contiguous CUDA fp16 [pixels, channels] tensor (no CPU / PyTorch fallback)" % name)
    return t


def conv2d_wgrad(x_rows, dy_rows, B, H, W, k, stride=1, pad=0):
    """x_rows [B*H*W, Cin], dy_rows [B*Ho*Wo, Cout] (NHWC fp16 rows) -> dW [Cout, Cin, k, k] fp32."""
    x_rows, dy_rows = _rows(x_rows, "x_rows"), _rows(dy_rows, "dy_rows")
    cin, cout = x_rows.shape[1], dy_rows.shape[1]
    ho, wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    if x_rows.shape[0] != B * H * W or dy_rows.shape[0] != B * ho * wo:
        raise ValueError("conv2d_wgrad: row counts %d / %d do not match B=%d H=%d W=%d k=%d stride=%d pad=%d"
                         % (x_rows.shape[0], dy_rows.shape[0], B, H, W, k, stride, pad))
    dw = torch.empty(cout, cin, k, k, dtype=torch.float32, device=x_rows.device)
    call("mf_conv2d_wgrad_nhwc_f16", x_rows.data_ptr(), cin, B, H, W, cin, dy_rows.data_ptr(), cout, cout, k, stride, pad,
         dw.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return dw


def conv2d_dgrad(dy_rows, weight, B, Ho, Wo, pad=0):
    """dy_rows [B*Ho*Wo, Cout] fp16, weight [Cout, Cin, k, k] (stride-1 convolution with padding `pad`) ->
    dx_rows [B*H*W, Cin] fp16 with H = Ho + k - 1 - 2 pad."""
    dy_rows = _rows(dy_rows, "dy_rows")
    cout, cin, k, k2 = weight.shape
    if k != k2 or dy_rows.shape != (B * Ho * Wo, cout):
        raise ValueError("conv2d_dgrad: shapes do not match")
    if k - 1 - pad < 0:
        raise NotImplementedError("conv2d_dgrad: pad > k - 1")
    w_rot = weight.detach().float().flip(2, 3).transpose(0, 1).contiguous()          # [Cin, Cout, k, k]
    P = engine.Plan(str(dy_rows.device))
    dya = P.act(B, Ho, Wo, cout)
    dya.buf = dy_rows                                                                  # zero-copy: the plan reads dY in place
    dxa = P.conv(dya, w_rot, 1, k - 1 - pad, None, act=engine.ACT_NONE)
    P.finalize()
    P.run()
    return dxa.buf[:, :cin] if dxa.buf.shape[1] != cin else dxa.buf


class BatchNormTrain(object):
    """Training-mode nn.BatchNorm2d / InPlaceABN over NHWC fp16 rows on the mf_bn_train_* kernels. forward() keeps what
    backward() needs (raw input, activated output, batch statistics); running statistics are updated in place like torch."""

    def __init__(self, gamma, beta, running_mean=None, running_var=None, eps=1e-5, momentum=0.1, act=1, abs_gamma=False):
        self.gamma, self.beta, self.running_mean, self.running_var = gamma, beta, running_mean, running_var
        self.eps, self.momentum, self.act, self.abs_gamma = eps, momentum, act, abs_gamma
        self.saved = None

    def forward(self, x_rows, residual=None):
        from ._lib import load
        x_rows = _rows(x_rows, "x_rows")
        M, C = x_rows.shape
        dev = x_rows.device
        y = torch.empty_like(x_rows)
        stats = torch.empty(4, C, dtype=torch.float32, device=dev)            # mean, rstd, scale, shift
        ws = torch.empty(load().mf_bn_train_workspace(M, C) // 4, dtype=torch.float32, device=dev)
        call("mf_bn_train_forward", x_rows.data_ptr(), C, M, C, self.gamma.data_ptr(), self.beta.data_ptr(), self.eps,
             self.momentum, 1 if self.abs_gamma else 0,
             self.running_mean.data_ptr() if self.running_mean is not None else None,
             self.running_var.data_ptr() if self.running_var is not None else None,
             residual.data_ptr() if residual is not None else None, C, self.act, y.data_ptr(), C, stats[0].data_ptr(),
             stats[1].data_ptr(), stats[2].data_ptr(), stats[3].data_ptr(), ws.data_ptr(),
             torch.cuda.current_stream().cuda_stream)
        self.saved = (x_rows, y, stats, ws, residual is not None)
        return y

    def backward(self, dy_rows):
        """-> (dx_rows, dgamma, dbeta, dresidual_rows or None)"""
        x_rows, y, stats, ws, has_res = self.saved
        dy_rows = _rows(dy_rows, "dy_rows")
        M, C = x_rows.shape
        dx = torch.empty_like(x_rows)
        dres = torch.empty_like(x_rows) if has_res else None
        dg = torch.empty(2, C, dtype=torch.float32, device=x_rows.device)
        call("mf_bn_train_backward", x_rows.data_ptr(), C, dy_rows.data_ptr(), C, y.data_ptr(), C, M, C, stats[0].data_ptr(),
             stats[1].data_ptr(), stats[2].data_ptr(), self.act, dx.data_ptr(), C, dres.data_ptr() if has_res else None, C,
             dg[0].data_ptr(), dg[1].data_ptr(), ws.data_ptr(), torch.cuda.current_stream().cuda_stream)
        dgamma = dg[0] * torch.sign(self.gamma) if self.abs_gamma else dg[0]
        return dx, dgamma, dg[1], dres


def _st():
    return torch.cuda.current_stream().cuda_stream


def conv2d_dgrad_stride2(dy_rows, weight, B, Ho, Wo):
    """dX of a 3x3 / stride-2 / pad-1 convolution (the level-entry convs, dla_dcn.py:69-79 with stride 2): the transposed
    convolution splits by output parity (py, px) into four stride-1 convolutions of dY whose 3x3 kernels hold the 1, 2, 2
    or 4 taps of W that reach that parity (zeros elsewhere) - run on the forward tensor-core kernel - and a 2x2 interleave.
    dy_rows [B*Ho*Wo, Cout] fp16 -> dx_rows [B*(2Ho)*(2Wo), Cin] fp16."""
    dy_rows = _rows(dy_rows, "dy_rows")
    cout, cin, k, k2 = weight.shape
    if (k, k2) != (3, 3) or dy_rows.shape != (B * Ho * Wo, cout):
        raise NotImplementedError("conv2d_dgrad_stride2: only 3x3 / stride 2 / pad 1 is built")
    w = weight.detach().float()
    pad = 1
    P = engine.Plan(str(dy_rows.device))
    dya = P.act(B, Ho, Wo, cout)
    dya.buf = dy_rows
    parts = []
    for py in (0, 1):
        for px in (0, 1):
            ws = torch.zeros(cin, cout, 3, 3, dtype=torch.float32, device=w.device)
            for ky in range(3):
                if (py + pad - ky) % 2:
                    continue
                ta = (py + pad - ky) // 2 + 1               # dX[2i+py] += dY[i + a] * W[ky], a = (py + pad - ky) / 2
                for kx in range(3):
                    if (px + pad - kx) % 2:
                        continue
                    tb = (px + pad - kx) // 2 + 1
                    ws[:, :, ta, tb] = w[:, :, ky, kx].t()
            parts.append(P.conv(dya, ws, 1, 1, None, act=engine.ACT_NONE))
    P.finalize()
    P.run()
    dx = torch.empty(B * 2 * Ho * 2 * Wo, cin, dtype=torch.half, device=dy_rows.device)
    call("mf_interleave2x2_nhwc_f16", parts[0].ptr(), parts[1].ptr(), parts[2].ptr(), parts[3].ptr(), parts[0].ld, dx.data_ptr(),
         cin, B, Ho, Wo, cin, _st())
    return dx


def maxpool2_backward(x_rows, dy_rows, B, H, W):
    x_rows, dy_rows = _rows(x_rows, "x_rows"), _rows(dy_rows, "dy_rows")
    C = x_rows.shape[1]
    dx = torch.empty_like(x_rows)
    call("mf_maxpool2_bwd_nhwc_f16", x_rows.data_ptr(), dy_rows.data_ptr(), dx.data_ptr(), B, H, W, C, C, C, C, _st())
    return dx


def upsample_backward(x_rows, w_taps, dy_rows, B, Hi, Wi, f):
    """-> (dx_rows, dw_taps [k*k, C] fp32); the skip input's gradient is dy_rows itself."""
    from ._lib import load
    x_rows, dy_rows = _rows(x_rows, "x_rows"), _rows(dy_rows, "dy_rows")
    C = x_rows.shape[1]
    dx = torch.empty_like(x_rows)
    dw = torch.empty(4 * f * f, C, dtype=torch.float32, device=x_rows.device)
    ws = torch.empty(load().mf_upsample_bwd_workspace(B, Hi, Wi, C, f) // 4, dtype=torch.float32, device=x_rows.device)
    call("mf_upsample_bwd_nhwc_f16", x_rows.data_ptr(), w_taps.data_ptr(), dy_rows.data_ptr(), dx.data_ptr(), dw.data_ptr(), B, Hi,
         Wi, C, f, C, C, C, ws.data_ptr(), _st())
    return dx, dw


def sigmoid_clamp_backward(y, dy):
    dx = torch.empty_like(y)
    call("mf_sigmoid_clamp_bwd", y.data_ptr(), dy.data_ptr(), dx.data_ptr(), y.numel(), _st())
    return dx


def column_sum(rows):
    from ._lib import load
    rows = _rows(rows, "rows")
    M, C = rows.shape
    out = torch.empty(C, dtype=torch.float32, device=rows.device)
    ws = torch.empty(load().mf_column_sum_workspace(M, C) // 4, dtype=torch.float32, device=rows.device)
    call("mf_column_sum_nhwc_f16", rows.data_ptr(), C, M, C, out.data_ptr(), ws.data_ptr(), _st())
    return out


def dcn_backward(x_rows, offmask_rows, dy_rows, weight, B, H, W):
    """Backward of the fused DCNv2 layer (3x3, stride 1, pad 1) on NHWC fp16 rows.
    x_rows [M, C], offmask_rows [M, 32] fp32 (the forward's offset-conv output: 18 offsets, 9 sigmoid-ed masks),
    dy_rows [M, Cout], weight [Cout, C, 3, 3] ->
    (dx_rows [M, C] fp16, d_offmask_rows [M, 32] fp32 = gradient of the offset conv's pre-activation output,
     dW [Cout, C, 3, 3] fp32, dbias [Cout] fp32)."""
    x_rows, dy_rows = _rows(x_rows, "x_rows"), _rows(dy_rows, "dy_rows")
    M, C = x_rows.shape
    cout = weight.shape[0]
    if weight.shape != (cout, C, 3, 3) or dy_rows.shape != (M, cout) or offmask_rows.shape != (M, 32) or M != B * H * W:
        raise ValueError("dcn_backward: shapes do not match")
    dev = x_rows.device
    # grad columns: a 1x1 forward conv of dY with W^T, output channel n = tap * C + c
    wt = weight.detach().float().permute(2, 3, 1, 0).reshape(9 * C, cout, 1, 1).contiguous()
    P = engine.Plan(str(dev))
    dya = P.act(B, H, W, cout)
    dya.buf = dy_rows
    gcol = P.conv(dya, wt, 1, 0, None, act=engine.ACT_NONE)
    P.finalize()
    P.run()
    cols = torch.empty(M, 9 * C, dtype=torch.half, device=dev)
    call("mf_dcn_sample_cols_nhwc_f16", x_rows.data_ptr(), C, offmask_rows.data_ptr(), 32, cols.data_ptr(), B, H, W, C, _st())
    dw9 = conv2d_wgrad(cols, dy_rows, B, H, W, 1, 1, 0)                                   # [Cout, 9C, 1, 1]
    dw = dw9.view(cout, 3, 3, C).permute(0, 3, 1, 2).contiguous()
    dx = torch.empty_like(x_rows)
    dom = torch.empty(M, 32, dtype=torch.float32, device=dev)
    call("mf_dcn_col2im_nhwc_f16", x_rows.data_ptr(), C, offmask_rows.data_ptr(), 32, gcol.ptr(), dx.data_ptr(), C, dom.data_ptr(),
         B, H, W, C, _st())
    return dx, dom, dw, column_sum(dy_rows)
