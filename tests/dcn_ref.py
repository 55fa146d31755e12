"""Float64 DCNv2 reference (3x3 kernel, stride 1, pad 1, dilation 1, one deformable group) shared by the DCN edge tests.

The sample coordinate is formed exactly as the reference's loops (dcn_v2_im2col_cpu.cpp:178, :232, :307) and every kernel
here form it: `h_in + i + offset_h` rounded ONCE to float32. Everything after that step is float64. The difference matters
at the kinks of the bilinear interpolation: an offset of 1e-8 added to an integer base rounds back onto the pixel grid in
float32, where the offset gradient is the one-sided (right) difference, while a float64 coordinate stays just below the
grid point and takes the left difference.

Layouts: x [B, C, H, W]; offset [B, 18, H, W] with channels (dy, dx) per tap; mask [B, 9, H, W]; columns and column
gradients [B, C, 9, H, W] (tap = 3 * ky + kx). Works on CPU and CUDA tensors alike.
"""
import numpy as np
import torch

# regimes of one coordinate component (edge_menu)
REGIMES = ("zero", "integer", "half", "exact -1", "exact H-1", "exact H", "band (-1,0)", "band (H-1,H)", "far", "tiny")
MASKS = ("0", "0.5", "1", "sigmoid")


def coords(offset, fp32=True):
    """sample coordinates (h, w) [B, 9, H, W] in float64. fp32=True: formed in float32 as the reference does; fp32=False:
    formed in float64 (wrong at the kinks; only used to show that the distinction matters)."""
    B, _, H, W = offset.shape
    dev = offset.device
    tap = torch.arange(9, device=dev)
    ky, kx = (tap // 3).view(1, 9, 1, 1), (tap % 3).view(1, 9, 1, 1)
    base_h = torch.arange(H, device=dev).view(1, 1, H, 1) - 1 + ky
    base_w = torch.arange(W, device=dev).view(1, 1, 1, W) - 1 + kx
    off = offset.view(B, 9, 2, H, W)
    if fp32:
        return (base_h.float() + off[:, :, 0].float()).double(), (base_w.float() + off[:, :, 1].float()).double()
    return base_h.double() + off[:, :, 0].double(), base_w.double() + off[:, :, 1].double()


def _sampling(x, offset, fp32=True):
    """per (b, tap, pixel): the four corners' float64 bilinear weights (0 where the corner or the sample is outside), their
    derivatives w.r.t. h and w, and the gathered corner values [B, C, 9, H, W]"""
    B, C, H, W = x.shape
    h, w = coords(offset, fp32)
    inside = (h > -1) & (w > -1) & (h < H) & (w < W)
    # far-outside samples never reach an index: clamp before any float -> int conversion
    h = torch.where(inside, h, torch.zeros_like(h))
    w = torch.where(inside, w, torch.zeros_like(w))
    hl, wl = torch.floor(h), torch.floor(w)
    lh, lw = h - hl, w - wl
    hh, hw = 1 - lh, 1 - lw
    hl, wl = hl.long(), wl.long()
    xf = x.double().reshape(B, C, H * W)
    corners = []
    for dr, dc, wt, dh, dw in ((0, 0, hh * hw, -hw, -hh), (0, 1, hh * lw, -lw, hh), (1, 0, lh * hw, hw, -lh), (1, 1, lh * lw, lw, lh)):
        r, c = hl + dr, wl + dc
        ok = (inside & (r >= 0) & (r <= H - 1) & (c >= 0) & (c <= W - 1)).double()
        idx = (r.clamp(0, H - 1) * W + c.clamp(0, W - 1)).view(B, 1, -1)
        v = xf.gather(2, idx.expand(B, C, -1)).view(B, C, 9, H, W)
        corners.append((idx, wt * ok, dh * ok, dw * ok, v))
    return corners


def columns(x, offset, mask, fp32=True, with_abs=False):
    """modulated im2col: cols[b, c, tap, y, x] = mask * bilinear(x[b, c], coordinate of (tap, y, x)). with_abs=True also
    returns sum over the four corners of |mask * weight * value| (the scale of the rounding error of any blend)."""
    m = mask.double().unsqueeze(1)
    cols, absum = 0, 0
    for _, wt, _, _, v in _sampling(x, offset, fp32):
        t = m * wt.unsqueeze(1) * v
        cols = cols + t
        absum = absum + t.abs()
    return (cols, absum) if with_abs else cols


def backward(x, offset, mask, gcol, fp32=True):
    """given gcol = dL/dcols [B, C, 9, H, W] -> (dX [B, C, H, W], dOffset [B, 18, H, W], dMask [B, 9, H, W]), float64
    (the reference's col2im and col2im_coord: dmcn_get_gradient_weight, dmcn_get_coordinate_weight)"""
    B, C, H, W = x.shape
    g = gcol.double()
    m = mask.double()
    dx = torch.zeros(B, C, H * W, dtype=torch.float64, device=x.device)
    d_h = d_w = d_m = 0
    for idx, wt, dh, dw, v in _sampling(x, offset, fp32):
        contrib = (g * (m * wt).unsqueeze(1)).reshape(B, C, -1)
        dx.scatter_add_(2, idx.expand(B, C, -1), contrib)
        gv = (g * v).sum(1)                              # [B, 9, H, W]: sum over channels of gcol * corner value
        d_h = d_h + dh * gv
        d_w = d_w + dw * gv
        d_m = d_m + wt * gv
    d_off = torch.stack([d_h * m, d_w * m], 2).reshape(B, 18, H, W)
    return dx.view(B, C, H, W), d_off, d_m


def edge_menu(B, H, W, seed):
    """offsets [B, 18, H, W] and masks [B, 9, H, W] (float32) where every tap of every pixel draws a regime (REGIMES) for
    each coordinate component and a mask (MASKS). Interior pixels draw at random; on the first and last row and column
    the regime cycles with the pixel position, so that every regime occurs at every tap on each of the four borders
    whenever that border is at least len(REGIMES) pixels long."""
    gen = np.random.Generator(np.random.PCG64(seed))
    R = len(REGIMES)
    b = np.arange(B).reshape(B, 1, 1, 1)
    tap = np.arange(9).reshape(1, 9, 1, 1)
    y = np.arange(H).reshape(1, 1, H, 1)
    x = np.arange(W).reshape(1, 1, 1, W)
    border = (y == 0) | (y == H - 1) | (x == 0) | (x == W - 1)
    shape = (B, 9, H, W)
    # along a row the h-regime steps by 1 per pixel, along a column by 3 (coprime with R): both cycle through all of them
    reg_h = np.where(border, (x + 3 * y + 7 * tap + 11 * b) % R, gen.integers(0, R, shape))
    reg_w = np.where(border, (y + 3 * x + 5 * tap + 13 * b + 1) % R, gen.integers(0, R, shape))

    def component(reg, base, n):
        sign = gen.choice([-1.0, 1.0], shape)
        u = gen.uniform(0.05, 0.95, shape)
        table = [
            np.zeros(shape),                                       # the reference's init (conv_offset_mask zeroed)
            sign * gen.choice([1.0, 2.0], shape),
            sign * 0.5,
            -1.0 - base,
            (n - 1.0) - base,
            float(n) - base,
            -u - base,
            (n - 1.0 + u) - base,
            sign * gen.choice([1e3, 3e9], shape),
            sign * 1e-8,
        ]
        out = np.zeros(shape)
        for k in range(R):
            out = np.where(reg == k, table[k], out)
        return out.astype(np.float32)

    off_h = component(reg_h, (y - 1 + tap // 3) * np.ones(shape), H)
    off_w = component(reg_w, (x - 1 + tap % 3) * np.ones(shape), W)
    offset = np.stack([off_h, off_w], 2).reshape(B, 18, H, W)
    mreg = gen.integers(0, len(MASKS), shape)
    sig = 1.0 / (1.0 + np.exp(-gen.standard_normal(shape)))
    mask = np.select([mreg == 0, mreg == 1, mreg == 2], [0.0, 0.5, 1.0], sig).astype(np.float32)
    return torch.from_numpy(np.ascontiguousarray(offset)), torch.from_numpy(mask), (reg_h, reg_w)


def to_offmask_rows(offset, mask):
    """[B, 18, H, W], [B, 9, H, W] -> the kernels' offset/mask rows [B*H*W, 32] fp32 (18 offsets, 9 masks, 5 zeros)"""
    B, _, H, W = offset.shape
    om = torch.zeros(B * H * W, 32, dtype=torch.float32, device=offset.device)
    om[:, :18] = offset.permute(0, 2, 3, 1).reshape(-1, 18)
    om[:, 18:27] = mask.permute(0, 2, 3, 1).reshape(-1, 9)
    return om
