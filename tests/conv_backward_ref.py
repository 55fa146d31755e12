"""Float64 references of the convolution backward operators, the per-element bounds the edge tests hold the kernels to,
the launchers' work splits those bounds depend on, and the "near-miss" results the bounds must reject.

Every reference runs in float64 on the CPU and comes with its absolute-value twin: the same operation on |x|, |dy| and
|w|, which gives A = sum |terms| for every output element. The bounds:

  weight gradient   |dW - ref| <= 2^-24 (P + S + 32) A
                    The operands are fp16-representable, so every product is exact in fp32; the error is the fp32
                    summation: P pixels summed inside one split (one CTA work item), S partial sums meeting through
                    atomics, 32 for the tensor core's own accumulation steps. A = 0 (a tap that reads only padding, a
                    zero dY channel) forces an exact 0.
  data gradient     |dx - ref| <= 2^-11 |ref| + 2^-24 (k^2 Cout + 32) A          (fp16 output, written)
                    |out - (before + ref)| <= 2^-11 |before + ref| + ...         (accumulated in one rounding)
                    The reference uses fp16(w), the operand the dgrad packer writes. Each fp16 rounding is also allowed
                    2^-25 absolute: half the spacing of fp16's subnormals.
"""
import math

import torch
import torch.nn.functional as F

U24 = 2.0 ** -24
U11 = 2.0 ** -11
SUB = 2.0 ** -25        # half the spacing of fp16 subnormals: the absolute error of one rounding below 2^-14
WG_BK = 64              # output pixels per k block of the general wgrad kernel (csrc/mf_wgrad.cu)


# ------------------------------------------------------------------------------------------------ references
def pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


def wgrad_ref(x, dy, kernel, stride, pad, per_image=False):
    """dW of y = conv2d(x, W, stride, pad): x [B, Cin, H, W], dy [B, Cout, Ho, Wo] -> (ref, A) [Cout, Cin, kh, kw]
    float64. per_image sums the images one by one (the long reductions: smaller temporaries)."""
    kh, kw = pair(kernel)
    x, dy = x.double(), dy.double()
    shape = (dy.shape[1], x.shape[1], kh, kw)

    def one(a, b):
        if not per_image:
            return torch.nn.grad.conv2d_weight(a, shape, b, stride=stride, padding=pad)
        return sum(torch.nn.grad.conv2d_weight(a[i:i + 1], shape, b[i:i + 1], stride=stride, padding=pad)
                   for i in range(a.shape[0]))

    return one(x, dy), one(x.abs(), dy.abs())


def dgrad_ref(dy, w, in_hw, stride, pad):
    """dX of y = conv2d(x, w, stride, pad): dy [B, Cout, Ho, Wo], w [Cout, Cin, k, k] (already the operand the kernel
    multiplies, e.g. fp16(w)) -> (ref, A) [B, Cin, H, W] float64"""
    dy, w = dy.double(), w.double()
    shape = (dy.shape[0], w.shape[1]) + tuple(in_hw)
    return (torch.nn.grad.conv2d_input(shape, w, dy, stride=stride, padding=pad),
            torch.nn.grad.conv2d_input(shape, w.abs(), dy.abs(), stride=stride, padding=pad))


def upsample_dx_ref(dy, w, f):
    """dX of the depth-wise ConvTranspose2d(k = 2f, stride f, pad f/2): dy [B, C, f Hi, f Wi], w [C, 1, 2f, 2f] -> (ref, A)
    [B, C, Hi, Wi] float64"""
    dy, w = dy.double(), w.double()
    C = dy.shape[1]
    return (F.conv2d(dy, w, None, stride=f, padding=f // 2, groups=C),
            F.conv2d(dy.abs(), w.abs(), None, stride=f, padding=f // 2, groups=C))


# ------------------------------------------------------------------------------------------------ launcher work splits
def out_hw(H, W, kernel, stride, pad):
    (kh, kw), (ph, pw) = pair(kernel), pair(pad)
    return (H + 2 * ph - kh) // stride + 1, (W + 2 * pw - kw) // stride + 1


def goes_narrow(Cin, Cout, kernel, stride, pad):
    """mf_conv2d_wgrad_rect_nhwc_f16 hands the full-resolution 16 -> 16 stem layers to mf_wgrad_narrow.cu"""
    (kh, kw), (ph, pw) = pair(kernel), pair(pad)
    return Cin == 16 and Cout == 16 and stride == 1 and kh == kw and kh in (3, 7) and ph == pw == kh // 2


def wgrad_plan(B, H, W, Cin, Cout, kernel, stride, pad, nsm):
    """the general kernel's launch (mf_conv2d_wgrad_rect_nhwc_f16): slots, tiles, k blocks, splits and their ranges.
    Returns a dict with P = the most pixels one split sums, S = splits, regime and dummy slots of the last M tile."""
    kh, kw = pair(kernel)
    Ho, Wo = out_hw(H, W, kernel, stride, pad)
    aw = min(Cin, 64)
    spt = 128 // aw
    nslots = kh * kw * (Cin // aw)
    ntm = -(-nslots // spt)
    bn = Cout if Cout < 64 else (128 if Cout % 128 == 0 else 64)
    ntn = Cout // bn
    M = B * Ho * Wo
    nkb = -(-M // WG_BK)
    tiles = ntm * ntn
    splits = max(1, min(-(-2 * nsm // tiles), nkb))
    base, extra = nkb // splits, nkb % splits
    ranges = []
    for sp in range(splits):                         # decode() in the kernel
        lo = sp * base + min(sp, extra)
        ranges.append((lo, lo + base + (1 if sp < extra else 0)))
    if splits == 1 and nkb > 1:
        regime = "one split"
    elif splits == nkb:
        regime = "one block per split"
    elif extra:
        regime = "remainder"
    else:
        regime = "even"
    return dict(M=M, Ho=Ho, Wo=Wo, aw=aw, spt=spt, nslots=nslots, ntm=ntm, ntn=ntn, bn=bn, nkb=nkb, tiles=tiles,
                splits=splits, ranges=ranges, P=(base + (1 if extra else 0)) * WG_BK, S=splits, regime=regime,
                dummies=ntm * spt - nslots, ragged=M % WG_BK)


def narrow_plan(B, H, W, k, nsm):
    """mf_wgrad_narrow.cu's launch: 16-pixel blocks of image rows, G blocks per unit, 4 CTAs per SM striding over units.
    P = the most pixels one warp sums into one output, S = the partial sums that meet through atomics."""
    G = 2 if k == 3 else 1
    bw = -(-W // 16)
    nblocks = B * H * bw
    nunits = -(-nblocks // G)
    grid = 4 * nsm
    return dict(G=G, nblocks=nblocks, nunits=nunits, grid=grid, P=-(-nunits // grid) * 16, S=min(grid, nunits) * G,
                last_unit_half=nblocks % G != 0, ragged=W % 16)


# ------------------------------------------------------------------------------------------------ bounds
def wgrad_bound(A, P, S):
    return U24 * (P + S + 32) * A


def dgrad_bound(ref, A, terms, before=None, roundings=1):
    """fp16 result of a sum of `terms` fp32 products (ref = its exact value, A = sum |products|), added into `before`
    when given. roundings = 2: the result was rounded to fp16 once on its own and once more after the addition (the
    temporary + mf_add_rows_f16 form)."""
    acc = U24 * (terms + 32) * A
    if before is None:
        return U11 * ref.abs() + SUB + acc
    tot = (before.double() + ref).abs()
    if roundings == 1:
        return U11 * tot + SUB + acc
    first = U11 * ref.abs() + SUB + acc
    return U11 * (tot + first) + SUB + first


def ratio(err, bound):
    """worst err / bound; an element whose bound is 0 must be exactly 0 (inf otherwise); NaN anywhere -> inf"""
    err, bound = err.double(), bound.double()
    if torch.isnan(err).any():
        return math.inf
    zero = bound == 0
    if (err[zero] != 0).any():
        return math.inf
    if zero.all():
        return 0.0
    return (err[~zero] / bound[~zero]).max().item()


def rel_l2(got, ref):
    ref = ref.double()
    n = ref.norm().item()
    return (got.double() - ref).norm().item() / n if n > 0 else (0.0 if got.double().norm().item() == 0 else math.inf)


# ------------------------------------------------------------------------------------------------ near misses
def flat_pixels(t):
    """[B, C, H, W] -> [B*H*W, C] in the kernels' NHWC row order"""
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def from_flat(rows, B, H, W):
    return rows.reshape(B, H, W, -1).permute(0, 3, 1, 2)


def dy_rows_kept(dy, lo, hi):
    """dy with every output pixel outside the flat NHWC range [lo, hi) zeroed"""
    B, C, Ho, Wo = dy.shape
    r = flat_pixels(dy.double()).clone()
    keep = torch.zeros(r.shape[0], 1, dtype=torch.float64)
    keep[lo:hi] = 1
    return from_flat(r * keep, B, Ho, Wo)


def miss_last_block_dropped(x, dy, kernel, stride, pad):
    """dW without the last (ragged) 64-pixel block of the reduction"""
    M = dy.shape[0] * dy.shape[2] * dy.shape[3]
    return wgrad_ref(x, dy_rows_kept(dy, 0, (M - 1) // WG_BK * WG_BK), kernel, stride, pad)[0]


def miss_tap_shifted(x, dy, kernel, stride, pad, tap):
    """dW with one tap's dY read one output pixel late (flat NHWC order)"""
    kh, kw = pair(kernel)
    B, C, Ho, Wo = dy.shape
    r = flat_pixels(dy.double())
    shifted = torch.cat([r[1:], torch.zeros(1, C, dtype=torch.float64)])
    out = wgrad_ref(x, dy, kernel, stride, pad)[0].clone()
    wrong = wgrad_ref(x, from_flat(shifted, B, Ho, Wo), kernel, stride, pad)[0]
    ky, kx = divmod(tap, kw)
    out[:, :, ky, kx] = wrong[:, :, ky, kx]
    return out


def miss_split_twice(x, dy, kernel, stride, pad, plan, split=None):
    """dW with one split's partial sum added twice (the middle split by default)"""
    sp = plan["splits"] // 2 if split is None else split
    lo, hi = plan["ranges"][sp]
    extra = wgrad_ref(x, dy_rows_kept(dy, lo * WG_BK, hi * WG_BK), kernel, stride, pad)[0]
    return wgrad_ref(x, dy, kernel, stride, pad)[0] + extra


def miss_tap_unrotated(dy, w, in_hw, stride, pad, tap=0):
    """dX as if the dgrad packer had written packed tap `tap` unrotated (w[tap] where w[taps - 1 - tap] belongs)"""
    k = w.shape[2]
    wf = w.double().reshape(w.shape[0], w.shape[1], k * k).clone()
    wf[:, :, k * k - 1 - tap] = w.double().reshape(w.shape[0], w.shape[1], k * k)[:, :, tap]
    return dgrad_ref(dy, wf.reshape(w.shape), in_hw, stride, pad)[0]


def miss_parities_swapped(dx):
    """a stride-2 data gradient [B, C, H, W] (H, W even) interleaved with parities (0, 1) and (1, 0) swapped"""
    out = dx.clone()
    out[:, :, 0::2, 1::2] = dx[:, :, 1::2, 0::2]
    out[:, :, 1::2, 0::2] = dx[:, :, 0::2, 1::2]
    return out
