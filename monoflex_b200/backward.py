"""Backward operators of the detector's layers over NHWC fp16 pixel rows, one function per layer type (training path of
SURVEY §8 rows R2/R3/R6; the reference gets them from cuDNN through autograd, engine/trainer.py:116-117). tape.py chains
them into the whole-network backward that KeypointDetector's tape bridge (model/detector.py) runs under `losses.backward()`.

Forward activations are contiguous [pixels, channels] fp16 rows or engine.Act, so a channel slice of a Root concatenation
works as it is; gradient rows likewise. The input gradient is returned as a new tensor when `dx` is None; given a
destination `dx` (the tape's shared gradient buffers), the operator ACCUMULATES into it (dx += dL/dx): the stride-1 data
gradient in place through the forward kernel's residual input (engine.Plan.conv_dgrad), the others through a temporary
and `mf_add_rows_f16`. Weight gradients are fp32.

  * conv2d_wgrad : dW on the tensor-core wgrad kernel (csrc/mf_wgrad.cu: wgmma GEMM whose MN-major operands come straight
                   from im2col / tiled TMA boxes, split-K);
  * conv2d_dgrad : dX of a stride-1 convolution = the forward implicit-GEMM kernel (csrc/mf_igemm2.cu) run on dY with the
                   rotated, in/out-transposed weights (Plan.conv_dgrad); 3x3 stride-2 layers use the four-parity
                   decomposition (`conv2d_dgrad_stride2`);
  * conv_backward: dW, dbias and dX of a convolution from the three above;
  * bn_backward, dcn_backward, maxpool2_backward, upsample_backward, sigmoid_clamp_backward, column_sum.
"""
import torch

from . import engine
from ._lib import call, load, stream


def _rows(t, name):
    """(device pointer, row stride) of fp16 pixel rows given as an engine.Act or a contiguous [pixels, channels] tensor"""
    act = isinstance(t, engine.Act)
    buf = t.buf if act else t
    if not (isinstance(buf, torch.Tensor) and buf.is_cuda and buf.dtype == torch.half and buf.dim() == 2 and
            (act or buf.is_contiguous())):
        raise RuntimeError("%s must be CUDA fp16 [pixels, channels] rows (no CPU / PyTorch fallback)" % name)
    return (t.ptr(), t.ld) if act else (t.data_ptr(), t.shape[1])


def _act(x, name, B, H, W):
    """x as an engine.Act (rows tensors are checked and wrapped)"""
    _rows(x, name)
    return x if isinstance(x, engine.Act) else engine.Act.on(x, B, H, W)


def _into(dx, t):
    """the input gradient held in the temporary `t`: returned as it is, or added into the destination dx"""
    if dx is None:
        return t
    add_rows(dx, t)
    return dx


def add_rows(dst, src):
    """dst += src (fp16 rows: Acts or tensors of the same pixel count; src has at least dst's channels)"""
    (d, d_ld), (s, s_ld) = _rows(dst, "dst"), _rows(src, "src")
    M, C = (dst.M, dst.C) if isinstance(dst, engine.Act) else dst.shape
    sM, sC = (src.M, src.C) if isinstance(src, engine.Act) else src.shape
    if sM != M or sC < C:
        raise ValueError("add_rows: source rows [%d, %d] do not cover destination rows [%d, %d]" % (sM, sC, M, C))
    call("mf_add_rows_f16", d, d_ld, s, s_ld, M, C, stream())


def run_plan(device, emit):
    """Build and run a one-off plan of forward kernels: emit(P) adds its ops and returns their outputs, which this returns
    once the plan has run."""
    P = engine.Plan(str(device))
    out = emit(P)
    P.finalize()
    P.run()
    return out


def conv2d_wgrad(x, dy_rows, B, H, W, k, stride=1, pad=0):
    """x [B*H*W, Cin] (rows or engine.Act), dy_rows [B*Ho*Wo, N] fp16 (N = Cout, or Cout zero-padded) -> dW [N, Cin, k, k]
    fp32. The stem's 8-channel packed image is widened to 16 zero channels, the narrowest box the kernel takes."""
    x = _act(x, "x", B, H, W)
    xp, x_ld = _rows(x, "x")
    dyp, n = _rows(dy_rows, "dy_rows")
    ho, wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    if x.M != B * H * W or dy_rows.shape[0] != B * ho * wo:
        raise ValueError("conv2d_wgrad: row counts %d / %d do not match B=%d H=%d W=%d k=%d stride=%d pad=%d"
                         % (x.M, dy_rows.shape[0], B, H, W, k, stride, pad))
    cin = x.C
    if cin == 8:
        x16 = torch.zeros(x.M, 16, dtype=torch.half, device=dy_rows.device)
        x16[:, :8] = x.buf.view(x.M, -1)[:, x.ch_off:x.ch_off + 8]
        xp, x_ld, cin = x16.data_ptr(), 16, 16
    elif not (cin in (16, 32) or cin % 64 == 0):
        raise NotImplementedError("conv2d_wgrad: %d input channels" % cin)
    dw = torch.empty(n, cin, k, k, dtype=torch.float32, device=dy_rows.device)
    call("mf_conv2d_wgrad_nhwc_f16", xp, x_ld, B, H, W, cin, dyp, n, n, k, stride, pad, dw.data_ptr(), stream())
    return dw[:, :x.C]


def conv2d_dgrad(dy_rows, weight, B, Ho, Wo, pad=0, dx=None):
    """dy_rows [B*Ho*Wo, Cout or zero-padded Cout] fp16, weight [Cout, Cin, k, k] fp32 of a stride-1 convolution with padding
    `pad` -> dx_rows [B*H*W, Cin] fp16 with H = Ho + k - 1 - 2 pad, or dx += that in place (dx: engine.Act)."""
    _rows(dy_rows, "dy_rows")
    cout, cin, k, k2 = weight.shape
    if k != k2 or dy_rows.shape[0] != B * Ho * Wo or dy_rows.shape[1] < cout:
        raise ValueError("conv2d_dgrad: shapes do not match")
    if k - 1 - pad < 0:
        raise NotImplementedError("conv2d_dgrad: pad > k - 1")
    out = run_plan(dy_rows.device, lambda P: P.conv_dgrad(engine.Act.on(dy_rows, B, Ho, Wo), weight, pad, dx))
    return dx if dx is not None else out.buf


def conv2d_dgrad_stride2(dy_rows, weight, B, Ho, Wo):
    """dX of a 3x3 / stride-2 / pad-1 convolution (the level-entry convs, dla_dcn.py:69-79 with stride 2): the transposed
    convolution splits by output parity (py, px) into four stride-1 convolutions of dY whose 3x3 kernels hold the 1, 2, 2
    or 4 taps of W that reach that parity (zeros elsewhere) - run on the forward tensor-core kernel - and a 2x2 interleave.
    dy_rows [B*Ho*Wo, Cout] fp16 -> dx_rows [B*(2Ho)*(2Wo), Cin] fp16."""
    _rows(dy_rows, "dy_rows")
    cout, cin, k, k2 = weight.shape
    if (k, k2) != (3, 3) or dy_rows.shape != (B * Ho * Wo, cout):
        raise NotImplementedError("conv2d_dgrad_stride2: only 3x3 / stride 2 / pad 1 is built")
    w = weight.detach().float()
    pad = 1
    taps = []
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
            taps.append(ws)
    dya = engine.Act.on(dy_rows, B, Ho, Wo)
    parts = run_plan(dy_rows.device, lambda P: [P.conv(dya, ws, 1, 1, None, act=engine.ACT_NONE) for ws in taps])
    dx = torch.empty(B * 2 * Ho * 2 * Wo, cin, dtype=torch.half, device=dy_rows.device)
    call("mf_interleave2x2_nhwc_f16", parts[0].ptr(), parts[1].ptr(), parts[2].ptr(), parts[3].ptr(), parts[0].ld, dx.data_ptr(),
         cin, B, Ho, Wo, cin, stream())
    return dx


def conv_backward(x, weight, bias, stride, pad, dy, dx=None):
    """y = conv(x, weight, stride, pad) (+ bias) with x an engine.Act and dy = dL/dy rows [B*Ho*Wo, Cout or zero-padded Cout]
    fp16 -> (dW, dbias or None); dx += dL/dx unless dx is None. The stride-2 data gradient is built for 3x3 / pad 1 on
    even H and W only."""
    cout, cin, k, _ = weight.shape
    if dx is not None and stride != 1:
        if (stride, k, pad) != (2, 3, 1):
            raise NotImplementedError("data gradient of a %dx%d stride-%d pad-%d convolution" % (k, k, stride, pad))
        if x.H % 2 or x.W % 2:
            # the four parities cover 2Ho x 2Wo = (H + 1) x (W + 1) pixels; nothing crops them back to H x W
            raise NotImplementedError("data gradient of a 3x3 stride-2 convolution on an odd %dx%d input" % (x.H, x.W))
    dw = conv2d_wgrad(x, dy, x.B, x.H, x.W, k, stride, pad)[:cout, :cin]
    db = column_sum(dy)[:cout] if bias is not None else None
    if dx is not None:
        ho, wo = (x.H + 2 * pad - k) // stride + 1, (x.W + 2 * pad - k) // stride + 1
        if stride == 1:
            conv2d_dgrad(dy, weight, x.B, ho, wo, pad, dx)
        else:
            add_rows(dx, conv2d_dgrad_stride2(dy, weight, x.B, ho, wo))
    return dw, db


def bn_backward(entries, dy, dx, act, abs_weight=False, dres=None):
    """Backward of a training-mode BatchNorm2d / InPlaceABN (abs_weight) / BatchNorm1d layer, y = act(bn(raw) + residual),
    from the Plan.bn_saved `entries` of its forward: (module, raw, y, stats, c0, cc) per <= 256-channel chunk, the chunks
    of one module consecutive. dy = dL/dy; dx = dL/draw and dres = dL/dresidual (or None) are written, dx may be dy itself.
    All three are rows in the channel numbering of `raw`. A torch.nn.SyncBatchNorm module exchanges its sums across ranks
    (engine.bn_backward_launch). Returns [(module, dgamma, dbeta)], whole-parameter fp32 gradients."""
    (dy_p, dy_ld), (dx_p, dx_ld) = _rows(dy, "dy"), _rows(dx, "dx")
    dres_p, dres_ld = _rows(dres, "dres") if dres is not None else (None, 0)
    dgs, first = {}, {}
    for mod, raw, y, stats, c0, cc in entries:
        if id(mod) not in dgs:
            dgs[id(mod)] = (mod, torch.empty(2, mod.weight.numel(), dtype=torch.float32, device=raw.buf.device))
            first[id(mod)] = c0
        off = c0 - first[id(mod)]
        ws = torch.empty(max(1, load().mf_bn_train_workspace(raw.M, cc) // 4), dtype=torch.float32, device=raw.buf.device)
        engine.bn_backward_launch(mod, raw.ptr() + 2 * c0, raw.ld, dy_p + 2 * c0, dy_ld, y.ptr() + 2 * c0, y.ld, raw.M, cc, stats,
                                  act, dx_p + 2 * c0, dx_ld, (dres_p + 2 * c0) if dres is not None else None, dres_ld,
                                  dgs[id(mod)][1][:, off:off + cc], ws, stream())
    return [(mod, dg[0] * torch.sign(mod.weight.detach()) if abs_weight else dg[0], dg[1]) for mod, dg in dgs.values()]


def maxpool2_backward(x, dy_rows, B, H, W, dx=None):
    """MaxPool2d(2) with input x [B*H*W, C] (rows or engine.Act) and dy_rows = dL/dy -> dx_rows, or dx += that."""
    x = _act(x, "x", B, H, W)
    (xp, x_ld), (dyp, dy_ld) = _rows(x, "x"), _rows(dy_rows, "dy_rows")
    t = torch.empty(x.M, x.C, dtype=torch.half, device=x.buf.device)
    call("mf_maxpool2_bwd_nhwc_f16", xp, dyp, t.data_ptr(), B, H, W, x.C, x_ld, dy_ld, x.C, stream())
    return _into(dx, t)


def upsample_backward(x, w_taps, dy_rows, B, Hi, Wi, f, dx=None, dskip=None):
    """y = depth-wise ConvTranspose2d(x; k = 2f, stride f) (+ skip) -> (dx_rows, dw_taps [k*k, C] fp32); a given dx is
    accumulated into (dx += dL/dx), and so is a given dskip (dskip += dy: the skip input's gradient is dy itself)."""
    x = _act(x, "x", B, Hi, Wi)
    (xp, x_ld), (dyp, dy_ld) = _rows(x, "x"), _rows(dy_rows, "dy_rows")
    if dskip is not None:
        add_rows(dskip, dy_rows)
    C, dev = x.C, x.buf.device
    t = torch.empty(x.M, C, dtype=torch.half, device=dev)
    dw = torch.empty(4 * f * f, C, dtype=torch.float32, device=dev)
    ws = torch.empty(max(1, load().mf_upsample_bwd_workspace(B, Hi, Wi, C, f) // 4), dtype=torch.float32, device=dev)
    call("mf_upsample_bwd_nhwc_f16", xp, w_taps.data_ptr(), dyp, t.data_ptr(), dw.data_ptr(), B, Hi, Wi, C, f, x_ld, dy_ld, C,
         ws.data_ptr(), stream())
    return _into(dx, t), dw


def sigmoid_clamp_backward(y, dy):
    dx = torch.empty_like(y)
    call("mf_sigmoid_clamp_bwd", y.data_ptr(), dy.data_ptr(), dx.data_ptr(), y.numel(), stream())
    return dx


def column_sum(rows):
    _rows(rows, "rows")
    M, C = rows.shape
    out = torch.empty(C, dtype=torch.float32, device=rows.device)
    ws = torch.empty(load().mf_column_sum_workspace(M, C) // 4, dtype=torch.float32, device=rows.device)
    call("mf_column_sum_nhwc_f16", rows.data_ptr(), C, M, C, out.data_ptr(), ws.data_ptr(), stream())
    return out


def dcn_backward(x, offmask_rows, dy_rows, weight, B, H, W, dx=None):
    """Backward of the fused DCNv2 layer (3x3, stride 1, pad 1) on NHWC fp16 rows.
    x [M, C] (rows or engine.Act), offmask_rows [M, 32] fp32 (the forward's offset-conv output: 18 offsets, 9 sigmoid-ed
    masks), dy_rows [M, Cout], weight [Cout, C, 3, 3] ->
    (dx_rows [M, C] fp16 or, given dx, dx += that; d_offmask_rows [M, 32] fp32 = gradient of the offset conv's
     pre-activation output; dW [Cout, C, 3, 3] fp32; dbias [Cout] fp32)."""
    x = _act(x, "x", B, H, W)
    xp, x_ld = _rows(x, "x")
    _rows(dy_rows, "dy_rows")
    M, C = x.M, x.C
    cout = weight.shape[0]
    if weight.shape != (cout, C, 3, 3) or dy_rows.shape != (M, cout) or offmask_rows.shape != (M, 32) or M != B * H * W:
        raise ValueError("dcn_backward: shapes do not match")
    dev = dy_rows.device
    # grad columns: a 1x1 forward conv of dY with W^T, output channel n = tap * C + c
    wt = weight.detach().float().permute(2, 3, 1, 0).reshape(9 * C, cout, 1, 1).contiguous()
    gcol = run_plan(dev, lambda P: P.conv(engine.Act.on(dy_rows, B, H, W), wt, 1, 0, None, act=engine.ACT_NONE))
    cols = torch.empty(M, 9 * C, dtype=torch.half, device=dev)
    call("mf_dcn_sample_cols_nhwc_f16", xp, x_ld, offmask_rows.data_ptr(), 32, cols.data_ptr(), B, H, W, C, stream())
    dw = conv2d_wgrad(cols, dy_rows, B, H, W, 1).view(cout, 3, 3, C).permute(0, 3, 1, 2).contiguous()
    db = column_sum(dy_rows)
    t = torch.empty(M, C, dtype=torch.half, device=dev)
    dom = torch.empty(M, 32, dtype=torch.float32, device=dev)
    call("mf_dcn_col2im_nhwc_f16", xp, x_ld, offmask_rows.data_ptr(), 32, gcol.ptr(), t.data_ptr(), C, dom.data_ptr(), B, H, W,
         C, stream())
    return _into(dx, t), dom, dw, db
