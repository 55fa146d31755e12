"""TEST INFRASTRUCTURE ONLY (oracle) — CPU fp32 restatement of MonoFlex's per-image hot path.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may
import this file; the product (`monoflex_b200/`) never does.

It is a *functional* restatement over a reference-keyed `state_dict` (no nn.Module tree): each function
cites the reference lines it follows. Parity status: PINNED for every stage against the unmodified
reference executed in the build container (`oracle/make_golden.py` -> `tests/golden/`,
`tests/test_oracle_golden.py`), except the third-party InPlaceABN op whose definition is not in the
reference tree ("parity unpinned" at that op only, see DESIGN.md).

Everything is torch-CPU fp32 (the reference itself is torch; ATen conv/pool/grid_sample are the same
library arithmetic the reference calls). DCNv2 is restated explicitly (vectorised gather) and checked
bit-for-bit against the reference's own C loops (`oracle/_ref/libdcn_im2col_ref.so`).
"""
import math

import torch
import torch.nn.functional as F

BN_EPS = 1e-5
PI = math.pi

# runs/monoflex.yaml:27-28 -> flattened channel map (model/layers/utils.py:22-37)
REG_KEYS = ['2d_dim', '3d_offset', 'corner_offset', 'corner_uncertainty', '3d_dim', 'ori_cls', 'ori_offset',
            'depth', 'depth_uncertainty']
REG_CH = [4, 2, 20, 3, 3, 8, 8, 1, 1]
REG_BRANCHES = [[(0, 4)], [(1, 2)], [(2, 20)], [(3, 3)], [(4, 3)], [(5, 8), (6, 8)], [(7, 1)], [(8, 1)]]
DIM_MEAN = ((3.8840, 1.5261, 1.6286), (0.8423, 1.7607, 0.6602), (1.7635, 1.7372, 0.5968))  # config/defaults.py:206-208


def key2channel(key):
    i = REG_KEYS.index(key)
    s = sum(REG_CH[:i])
    return slice(s, s + REG_CH[i])


# ------------------------------------------------------------------------------------------------ layers
_TRAIN = [False]     # train-mode switch of every normalisation layer (batch statistics), see training_mode()


class training_mode(object):
    """with training_mode(): ... -> BatchNorm / InPlaceABN / BatchNorm1d use batch statistics like module.train()
    (running statistics are not updated: they do not enter the forward value or the gradients)."""

    def __enter__(self):
        self.prev = _TRAIN[0]
        _TRAIN[0] = True

    def __exit__(self, *a):
        _TRAIN[0] = self.prev


def bn_eval(sd, p, x, abs_weight=False):
    """nn.BatchNorm2d (dla_dcn.py:76 etc.): (x-mean)/sqrt(var+eps)*w+b, running statistics in eval mode, batch statistics
    under training_mode(). IABN uses |w|+eps."""
    w = sd[p + '.weight']
    if abs_weight:
        w = w.abs() + BN_EPS
    if _TRAIN[0]:
        return F.batch_norm(x, None, None, w, sd[p + '.bias'], True, 0.0, BN_EPS)
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], w, sd[p + '.bias'], False, 0.0, BN_EPS)


def conv_bn(sd, conv, bn, x, stride=1, pad=1, relu=True, residual=None):
    y = F.conv2d(x, sd[conv + '.weight'], None, stride, pad)
    y = bn_eval(sd, bn, y)
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


def basic_block(sd, p, x, stride, residual=None):
    """BasicBlock.forward dla_dcn.py:84-98."""
    if residual is None:
        residual = x
    out = conv_bn(sd, p + '.conv1', p + '.bn1', x, stride, 1, True)
    return conv_bn(sd, p + '.conv2', p + '.bn2', out, 1, 1, True, residual)


def root(sd, p, xs):
    """Root.forward dla_dcn.py:195-203 (residual=False in dla34)."""
    return conv_bn(sd, p + '.conv', p + '.bn', torch.cat(xs, 1), 1, 0, True)


def tree(sd, p, levels, x, cin, cout, stride, level_root, children=None):
    """Tree.forward dla_dcn.py:246-259. The `residual` argument of nested trees is overwritten at :249,
    so the outer `project` of a 2-level tree never reaches the output; it is skipped here."""
    children = [] if children is None else children
    bottom = F.max_pool2d(x, stride, stride) if stride > 1 else x
    if level_root:
        children.append(bottom)
    if levels == 1:
        residual = conv_bn(sd, p + '.project.0', p + '.project.1', bottom, 1, 0, False) if cin != cout else bottom
        x1 = basic_block(sd, p + '.tree1', x, stride, residual)
        x2 = basic_block(sd, p + '.tree2', x1, 1)
        return root(sd, p + '.root', [x2, x1] + children)
    x1 = tree(sd, p + '.tree1', levels - 1, x, cin, cout, stride, False)
    children.append(x1)
    return tree(sd, p + '.tree2', levels - 1, x1, cout, cout, 1, False, children)


def dla34_base(sd, x, p='backbone.base'):
    """DLA.forward dla_dcn.py:324-331 with dla34 config :347-349."""
    ch = [16, 32, 64, 128, 256, 512]
    lv = [1, 1, 1, 2, 2, 1]
    x = conv_bn(sd, p + '.base_layer.0', p + '.base_layer.1', x, 1, 3)
    y = []
    x = conv_bn(sd, p + '.level0.0', p + '.level0.1', x, 1, 1)
    y.append(x)
    x = conv_bn(sd, p + '.level1.0', p + '.level1.1', x, 2, 1)
    y.append(x)
    for i in range(2, 6):
        x = tree(sd, '%s.level%d' % (p, i), lv[i], x, ch[i - 1], ch[i], 2, i > 2)
        y.append(x)
    return y


# ------------------------------------------------------------------------------------------------ DCNv2
def dcn_columns(x, offset, mask, k=3, pad=1, dil=1):
    """modulated_deformable_im2col (src/cpu/dcn_v2_im2col_cpu.cpp:27-56,127-196), stride 1, dg=1.
    Returns columns [B, C, k*k, H*W] (reference layout [B, C*k*k, H*W] viewed)."""
    B, C, H, W = x.shape
    dev = x.device
    ys = torch.arange(H, dtype=torch.float32, device=dev).view(1, 1, H, 1)
    xs = torch.arange(W, dtype=torch.float32, device=dev).view(1, 1, 1, W)
    ki = torch.arange(k * k, device=dev) // k
    kj = torch.arange(k * k, device=dev) % k
    off = offset.view(B, k * k, 2, H, W)
    h_im = (ys - pad) + (ki.view(1, -1, 1, 1) * dil).float() + off[:, :, 0]   # h_in + i*dil + offset_h  (:176)
    w_im = (xs - pad) + (kj.view(1, -1, 1, 1) * dil).float() + off[:, :, 1]
    inside = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)            # :180
    h_low, w_low = torch.floor(h_im), torch.floor(w_im)
    lh, lw = h_im - h_low, w_im - w_low
    hh, hw = 1 - lh, 1 - lw
    h_low, w_low = h_low.long(), w_low.long()
    h_high, w_high = h_low + 1, w_low + 1
    xf = x.reshape(B, C, H * W)

    def corner(hi, wi, ok):
        ok = ok & inside
        idx = (hi.clamp(0, H - 1) * W + wi.clamp(0, W - 1)).view(B, 1, -1).expand(B, C, -1)
        v = xf.gather(2, idx).view(B, C, k * k, H, W)
        return v * ok.unsqueeze(1).float()

    v1 = corner(h_low, w_low, (h_low >= 0) & (w_low >= 0))                    # :37-48
    v2 = corner(h_low, w_high, (h_low >= 0) & (w_high <= W - 1))
    v3 = corner(h_high, w_low, (h_high <= H - 1) & (w_low >= 0))
    v4 = corner(h_high, w_high, (h_high <= H - 1) & (w_high <= W - 1))
    w1, w2, w3, w4 = (hh * hw).unsqueeze(1), (hh * lw).unsqueeze(1), (lh * hw).unsqueeze(1), (lh * lw).unsqueeze(1)
    val = w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4                              # :52-54
    return (val * mask.view(B, 1, k * k, H, W)).reshape(B, C, k * k, H * W)   # :189


def dcn_v2_forward(x, weight, bias, offset, mask):
    """dcn_v2_cpu_forward (src/cpu/dcn_v2_cpu.cpp:17-107): out = bias + W[Cout, C*9] . columns."""
    B, C, H, W = x.shape
    cols = dcn_columns(x, offset, mask).reshape(B, C * 9, H * W)
    out = torch.matmul(weight.reshape(weight.shape[0], -1), cols) + bias.view(1, -1, 1)
    return out.view(B, -1, H, W)


def dcn(sd, p, x):
    """DCN.forward dcn_v2.py:118-128: conv_offset_mask -> chunk/cat -> sigmoid(mask) -> dcn_v2_conv."""
    om = F.conv2d(x, sd[p + '.conv_offset_mask.weight'], sd[p + '.conv_offset_mask.bias'], 1, 1)
    o1, o2, m = torch.chunk(om, 3, dim=1)
    return dcn_v2_forward(x, sd[p + '.weight'], sd[p + '.bias'], torch.cat((o1, o2), 1), torch.sigmoid(m))


def deform_conv(sd, p, x):
    """DeformConv.forward dla_dcn.py:393-396: DCN -> BN -> ReLU."""
    return F.relu(bn_eval(sd, p + '.actf.0', dcn(sd, p + '.conv', x)))


def up(sd, p, x, f):
    """depthwise ConvTranspose2d(o,o,2f,stride f,pad f//2,groups=o) dla_dcn.py:409-411."""
    w = sd[p + '.weight']
    return F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=w.shape[0])


def ida_up(sd, p, layers, startp, endp, up_f):
    """IDAUp.forward dla_dcn.py:419-425."""
    for i in range(startp + 1, endp):
        j = i - startp
        layers[i] = up(sd, '%s.up_%d' % (p, j), deform_conv(sd, '%s.proj_%d' % (p, j), layers[i]), up_f[j])
        layers[i] = deform_conv(sd, '%s.node_%d' % (p, j), layers[i] + layers[i - 1])


def backbone(sd, x, p='backbone', taps=None):
    """DLASeg.forward dla_dcn.py:48-58 (+ DLAUp.forward :446-452)."""
    layers = dla34_base(sd, x, p + '.base')
    if taps is not None:
        for i, l in enumerate(layers):
            taps['level%d' % i] = l
    layers = list(layers)
    out = [layers[-1]]
    up_fs = [[1, 2], [1, 2, 2], [1, 2, 2, 2]]
    for i in range(3):
        ida_up(sd, '%s.dla_up.ida_%d' % (p, i), layers, 6 - i - 2, 6, up_fs[i])
        out.insert(0, layers[-1])
    if taps is not None:
        for i, l in enumerate(out):
            taps['dla_up%d' % i] = l
    y = [out[0].clone(), out[1], out[2]]
    ida_up(sd, p + '.ida_up', y, 0, 3, [1, 2, 4])
    return y[-1]


# ------------------------------------------------------------------------------------------------ head
def iabn(sd, p, x):
    """InPlaceABN(activation='leaky_relu', slope 0.01): third-party, as recalled (SURVEY H4)."""
    return F.leaky_relu(bn_eval(sd, p, x, abs_weight=True), 0.01)


def predictor(sd, features, edge_indices, edge_lens, p='heads.predictor', out_w=None, out_h=None, taps=None, stored=None):
    """_predictor.forward detector_predictor.py:121-165.
    edge_indices int64 [B,K,2] (x,y); edge_lens int [B]. Runs in the dtype of `features` (float64 with a float64 `sd`).
    stored: optional function applied to every intermediate an implementation keeps in memory between its stages (the
    hidden activations of the nine branches, the gathered edge features, the edge Conv1d + BN output), e.g. an fp16 round
    trip to model a reduced-precision implementation; identity by default."""
    st = (lambda t: t) if stored is None else stored
    b, c, h, w = features.shape
    out_w = w if out_w is None else out_w
    out_h = h if out_h is None else out_h
    feature_cls = st(iabn(sd, p + '.class_head.1', F.conv2d(features, sd[p + '.class_head.0.weight'], None, 1, 1)))
    output_cls = F.conv2d(feature_cls, sd[p + '.class_head.2.weight'], sd[p + '.class_head.2.bias'])
    regs = []
    for i, branch in enumerate(REG_BRANCHES):
        rf = st(iabn(sd, '%s.reg_features.%d.1' % (p, i),
                     F.conv2d(features, sd['%s.reg_features.%d.0.weight' % (p, i)], None, 1, 1)))
        for j, (ki, ch) in enumerate(branch):
            o = F.conv2d(rf, sd['%s.reg_heads.%d.%d.weight' % (p, i, j)], sd['%s.reg_heads.%d.%d.bias' % (p, i, j)])
            if REG_KEYS[ki] == '3d_offset':                                      # edge fusion :137-158
                g = edge_indices.view(b, -1, 1, 2).to(features.dtype).clone()
                g[..., 0] = g[..., 0] / (out_w - 1) * 2 - 1
                g[..., 1] = g[..., 1] / (out_h - 1) * 2 - 1
                ef = st(F.grid_sample(torch.cat((feature_cls, rf), 1), g, align_corners=True).squeeze(-1))
                if taps is not None:
                    taps['edge_features'] = ef

                def trunc(q, e):
                    e = F.conv1d(F.pad(e, (1, 1), mode='replicate'), sd[q + '.0.weight'], sd[q + '.0.bias'])
                    if _TRAIN[0]:
                        e = F.batch_norm(e, None, None, sd[q + '.1.weight'], sd[q + '.1.bias'], True, 0.0, BN_EPS)
                    else:
                        e = F.batch_norm(e, sd[q + '.1.running_mean'], sd[q + '.1.running_var'], sd[q + '.1.weight'],
                                         sd[q + '.1.bias'], False, 0.0, BN_EPS)
                    return F.conv1d(st(e), sd[q + '.3.weight'], sd[q + '.3.bias'])

                e_cls = trunc(p + '.trunc_heatmap_conv', ef[:, :256])
                e_off = trunc(p + '.trunc_offset_conv', ef[:, 256:])
                if taps is not None:
                    taps['e_cls'], taps['e_off'] = e_cls, e_off
                for k in range(b):
                    n = int(edge_lens[k])
                    ek = edge_indices[k, :n]
                    output_cls[k, :, ek[:, 1], ek[:, 0]] += e_cls[k, :, :n]
                    o[k, :, ek[:, 1], ek[:, 0]] += e_off[k, :, :n]
            regs.append(o)
    if taps is not None:
        taps['cls_logits'] = output_cls.clone()
    cls = torch.sigmoid(output_cls).clamp(min=1e-4, max=1 - 1e-4)               # sigmoid_hm layers/utils.py:39-43
    return {'cls': cls, 'reg': torch.cat(regs, 1)}


# ------------------------------------------------------------------------------------------------ decode
def nms_hm(heat):
    """layers/utils.py:45-58."""
    hmax = F.max_pool2d(heat, 3, 1, 1)
    return heat * (hmax == heat).float()


def select_topk(heat, K=50):
    """layers/utils.py:61-100 with torch-1.4 floor division (SURVEY H5). Tie rule of this oracle and of the
    CUDA kernel: (score desc, flat index asc) at both stages — torch.topk leaves ties unspecified."""
    B, C, H, W = heat.shape
    flat = heat.reshape(B, C, H * W)
    # stable sort on -score gives (score desc, index asc)
    order = torch.sort(-flat, dim=2, stable=True).indices[:, :, :K]
    sc_all = flat.gather(2, order)                                              # [B,C,K]
    sc_all2 = sc_all.reshape(B, C * K)
    order2 = torch.sort(-sc_all2, dim=1, stable=True).indices[:, :K]
    scores = sc_all2.gather(1, order2)
    clses = (order2 // K).float()
    inds = order.reshape(B, C * K).gather(1, order2)
    ys = (inds // W).float()
    xs = (inds % W).float()
    return scores, inds, clses, ys, xs


def gather_pois(reg, inds):
    """select_point_of_interest layers/utils.py:120-145 -> [B,K,C]."""
    B, C, H, W = reg.shape
    return reg.reshape(B, C, H * W).gather(2, inds.view(B, 1, -1).expand(B, C, -1)).permute(0, 2, 1).contiguous()


def calib_from_P(P):
    """Calibration intrinsics, kitti_utils.py:211-218. Returns python floats (float64) like the reference."""
    f_u, f_v, c_u, c_v = float(P[0][0]), float(P[1][1]), float(P[0][2]), float(P[1][2])
    return dict(f_u=f_u, f_v=f_v, c_u=c_u, c_v=c_v, b_x=float(P[0][3]) / (-f_u), b_y=float(P[1][3]) / (-f_v))


def decode_image(scores, clses, xs, ys, pois, calib, pad_size, img_size, det_threshold=0.2, down_ratio=4):
    """PostProcessor.forward detector_infer.py:103-232 for ONE image (the reference is batch-1 only, SURVEY H8),
    OUTPUT_DEPTH='soft', UNCERTAINTY_AS_CONFIDENCE=True. All inputs [K] / [K,50]; calib = calib_from_P(...);
    pad_size [2] (x,y) ; img_size (W,H). Returns result[N,14]."""
    valid = scores >= det_threshold
    if int(valid.sum()) == 0:
        return scores.new_zeros(0, 14)
    scores, clses, xs, ys, pois = scores[valid], clses[valid], xs[valid], ys[valid], pois[valid]
    pts = torch.stack([xs, ys], 1)
    pad = pad_size.view(1, 2).float()
    ltrb = F.relu(pois[:, key2channel('2d_dim')])
    off3d = pois[:, key2channel('3d_offset')]
    # decode_box2d_fcos anno_encoder.py:69-86
    box = torch.cat([pts - ltrb[:, :2], pts + ltrb[:, 2:]], 1) * down_ratio - pad.repeat(1, 2)
    box[:, 0::2] = box[:, 0::2].clamp(min=0, max=float(img_size[0]) - 1)
    box[:, 1::2] = box[:, 1::2].clamp(min=0, max=float(img_size[1]) - 1)
    # decode_dimension :221-243 ('exp', mean, no std)
    dim_mean = torch.tensor(DIM_MEAN)[clses.long()]
    dims = pois[:, key2channel('3d_dim')].exp() * dim_mean                      # (l,h,w)
    # decode_depth :124-140 inv_sigmoid, range [0.1,100]
    d_direct = (1 / torch.sigmoid(pois[:, key2channel('depth')].squeeze(-1)) - 1).clamp(0.1, 100)
    s_direct = pois[:, key2channel('depth_uncertainty')].exp()
    kp = pois[:, key2channel('corner_offset')].view(-1, 10, 2)
    h3d = dims[:, 1]
    f_u = calib['f_u']
    # decode_depth_from_keypoints_batch :187-219
    center_h = kp[:, -2, 1] - kp[:, -1, 1]
    c02_h = kp[:, [0, 2], 1] - kp[:, [4, 6], 1]
    c13_h = kp[:, [1, 3], 1] - kp[:, [5, 7], 1]
    d_c = f_u * h3d / (F.relu(center_h) * down_ratio + 1e-3)
    d_02 = (f_u * h3d.unsqueeze(-1) / (F.relu(c02_h) * down_ratio + 1e-3)).mean(1)
    d_13 = (f_u * h3d.unsqueeze(-1) / (F.relu(c13_h) * down_ratio + 1e-3)).mean(1)
    d_kp = torch.stack([d_c, d_02, d_13], 1).clamp(0.1, 100)
    s_kp = pois[:, key2channel('corner_uncertainty')].exp()
    depths = torch.cat([d_direct.unsqueeze(1), d_kp], 1)
    sig = torch.cat([s_direct, s_kp], 1)
    wts = 1 / sig                                                               # detector_infer.py:176-198
    wts = wts / wts.sum(1, keepdim=True)
    depth = (depths * wts).sum(1)
    err = (wts * sig).sum(1)
    # decode_location_flatten :142-155 + project_image_to_rect kitti_utils.py:350-369
    uv = (pts + off3d) * down_ratio - pad
    x3 = ((uv[:, 0] - calib['c_u']) * depth) / calib['f_u'] + calib['b_x']
    y3 = ((uv[:, 1] - calib['c_v']) * depth) / calib['f_v'] + calib['b_y']
    loc = torch.stack([x3, y3, depth], 1)
    # decode_axes_orientation :245-295 (multi-bin)
    ori = torch.cat([pois[:, key2channel('ori_cls')], pois[:, key2channel('ori_offset')]], 1)
    bin_cls = torch.softmax(ori[:, :8].view(-1, 4, 2), 2)[..., 1]
    bi = bin_cls.argmax(1)
    offs = ori[:, 8:].view(-1, 4, 2)[torch.arange(ori.shape[0]), bi]
    centers = torch.tensor([0, PI / 2, PI, -PI / 2])
    alpha = torch.atan2(offs[:, 0], offs[:, 1]) + centers[bi]
    ray = torch.atan2(loc[:, 0], loc[:, 2])
    roty = alpha + ray
    roty = torch.where(roty > PI, roty - 2 * PI, roty)
    roty = torch.where(roty < -PI, roty + 2 * PI, roty)
    alpha = torch.where(alpha > PI, alpha - 2 * PI, alpha)
    alpha = torch.where(alpha < -PI, alpha + 2 * PI, alpha)
    loc[:, 1] = loc[:, 1] + dims[:, 1] / 2                                      # detector_infer.py:215
    dims_hwl = dims.roll(shifts=-1, dims=1)
    scores = scores * (1 - err.clamp(0.01, 1))                                  # :225-227
    return torch.cat([clses.view(-1, 1), alpha.view(-1, 1), box, dims_hwl, loc, roty.view(-1, 1),
                      scores.view(-1, 1)], 1)


def post_process(pred, calibs_P, pad_sizes, img_sizes, det_threshold=0.2, K=50):
    """Batch wrapper: loops the batch-1 reference semantics per image. Returns list of result[N_i,14] plus the
    top-k tensors (scores, inds, clses, ys, xs)."""
    heat = nms_hm(pred['cls'])
    scores, inds, clses, ys, xs = select_topk(heat, K)
    pois = gather_pois(pred['reg'], inds)
    results = []
    for b in range(heat.shape[0]):
        results.append(decode_image(scores[b], clses[b], xs[b], ys[b], pois[b], calib_from_P(calibs_P[b]),
                                    pad_sizes[b], img_sizes[b], det_threshold))
    return results, (scores, inds, clses, ys, xs)


def detector_eval(sd, images, edge_indices, edge_lens, calibs_P, pad_sizes, img_sizes, det_threshold=0.2, taps=None):
    """KeypointDetector.forward eval branch model/detector.py:26-37."""
    feats = backbone(sd, images, taps=taps)
    if taps is not None:
        taps['features'] = feats
    pred = predictor(sd, feats, edge_indices, edge_lens, taps=taps)
    if taps is not None:
        taps['cls'], taps['reg'] = pred['cls'], pred['reg']
    return post_process(pred, calibs_P, pad_sizes, img_sizes, det_threshold)


# ------------------------------------------------------------------------------------------------ loss
def focal_loss(pred, target, alpha=2, beta=4):
    """FocalLoss.forward layers/focal_loss.py:35-55 -> (loss_sum, num_pos)."""
    pos = target.eq(1).float()
    neg = (target.lt(1) & target.ge(0)).float()
    pl = (torch.log(pred) * torch.pow(1 - pred, alpha) * pos).sum()
    nl = (torch.log(1 - pred) * torch.pow(pred, alpha) * torch.pow(1 - target, beta) * neg).sum()
    return -nl - pl, pos.sum()


# ------------------------------------------------------------------------------------------------ 11-term loss (row R12)
LOSS_NAMES = ['hm_loss', 'bbox_loss', 'depth_loss', 'offset_loss', 'orien_loss', 'dims_loss', 'corner_loss',
              'keypoint_loss', 'keypoint_depth_loss', 'trunc_offset_loss', 'weighted_avg_depth_loss']   # runs/monoflex.yaml:45
LOSS_WEIGHTS = dict(zip(LOSS_NAMES, [1, 1, 1, 0.5, 1, 1, 0.2, 1.0, 0.2, 0.1, 0.2]))                   # runs/monoflex.yaml:47
UNC_RANGE = (-10.0, 10.0)                                                                              # config/defaults.py:162


def encode_box3d(rotys, dims, locs):
    """Anno_Encoder.encode_box3d anno_encoder.py:88-122: 8 corners [N,8,3] of boxes (l,h,w) rotated by ry about y."""
    N = rotys.shape[0]
    l, h, w = dims[:, 0:1] * 0.5, dims[:, 1:2] * 0.5, dims[:, 2:3] * 0.5
    sx = torch.tensor([-1., -1, 1, 1, -1, -1, 1, 1])          # index row [4,5,0,1,6,7,2,3] of the +/- half-extent table
    sy = torch.tensor([1., 1, 1, 1, -1, -1, -1, -1])          # [0..7]
    sz = torch.tensor([-1., 1, 1, -1, -1, 1, 1, -1])          # [4,0,1,5,6,2,3,7]
    X, Y, Z = l * sx, h * sy, w * sz
    c, s = rotys.cos().view(N, 1), rotys.sin().view(N, 1)
    bx = c * X + s * Z + locs[:, 0:1]
    by = Y + locs[:, 1:2]
    bz = -s * X + c * Z + locs[:, 2:3]
    return torch.stack([bx, by, bz], 2)


def giou_loss(pred, target):
    """IOULoss('giou').forward layers/iou_loss.py:12-49 -> (1 - giou, iou)."""
    pl, pt, pr, pb = pred.unbind(1)
    tl, tt, tr, tb = target.unbind(1)
    t_area, p_area = (tl + tr) * (tt + tb), (pl + pr) * (pt + pb)
    w_i = torch.min(pl, tl) + torch.min(pr, tr)
    gw = torch.max(pl, tl) + torch.max(pr, tr)
    h_i = torch.min(pb, tb) + torch.min(pt, tt)
    gh = torch.max(pb, tb) + torch.max(pt, tt)
    ac = gw * gh + 1e-7
    inter = w_i * h_i
    union = t_area + p_area - inter
    ious = (inter + 1.0) / (union + 1.0)
    return 1 - (ious - (ac - union) / ac), ious


def multibin_loss(vec, gt, num_bin=4):
    """Real_MultiBin_loss detector_loss.py:495-517."""
    cls_losses, reg_losses, reg_cnt = 0, 0, 0
    for i in range(num_bin):
        cls_losses = cls_losses + F.cross_entropy(vec[:, 2 * i:2 * i + 2], gt[:, i].long(), reduction='none').mean()
        m = gt[:, i] == 1
        if m.sum() > 0:
            s = num_bin * 2 + i * 2
            po = F.normalize(vec[m, s:s + 2])
            reg = (po[:, 0] - torch.sin(gt[m, num_bin + i])).abs() + (po[:, 1] - torch.cos(gt[m, num_bin + i])).abs()
            reg_losses = reg_losses + reg.sum()
            reg_cnt = reg_cnt + m.sum()
    return cls_losses / num_bin + reg_losses / reg_cnt


def loss_computation(pred_cls, pred_reg, fields, calibs_P, down_ratio=4):
    """Loss_Computation.__call__ detector_loss.py:267-493 with prepare_targets :88-114 and prepare_predictions :116-265 for
    the runs/monoflex.yaml configuration (L1 regression, giou, L1 depth with uncertainty, multi-bin, soft_combine corner
    depth, 'log' truncation offset loss, MODIFY_INVALID_KEYPOINT_DEPTH). `fields`: list (per image) of dicts of tensors
    named like the ParamsList fields; `pred_cls` is the sigmoid-ed, clamped heat map. Returns (loss_dict, log_dict) of
    tensors; every entry of loss_dict is differentiable w.r.t. pred_cls / pred_reg. The shapely '3D_IoU' logging metric
    (:333) is not restated (SURVEY §8c iii)."""
    B, C, H, W = pred_reg.shape
    st = lambda k: torch.stack([torch.as_tensor(f[k]) for f in fields])
    hm = st('hm').float()
    reg_mask = st('reg_mask').view(-1).bool()
    M = st('reg_mask').shape[1]
    batch_idxs = torch.arange(B).view(-1, 1).expand(B, M).reshape(-1)[reg_mask]
    centers = st('target_centers')
    pts = centers.view(-1, 2)[reg_mask]                                   # int
    box = st('bboxes').view(-1, 4)[reg_mask].float()
    t_h, t_w = box[:, 3] - box[:, 1], box[:, 2] - box[:, 0]
    t_reg2d = torch.cat((pts - box[:, :2], box[:, 2:] - pts), 1)
    m2d = (t_h > 0) & (t_w > 0)
    t_reg2d = t_reg2d[m2d]
    t_cls = st('cls_ids').view(-1)[reg_mask].long()
    t_depth = st('locations')[..., -1].reshape(-1)[reg_mask].float()
    t_roty = st('rotys').view(-1)[reg_mask].float()
    t_off = st('offset_3D').view(-1, 2)[reg_mask].float()
    t_dims = st('dimensions').view(-1, 3)[reg_mask].float()
    t_ori = st('orientations').view(-1, 8)[reg_mask].float()
    pads = st('pad_size').float()
    calibs = [calib_from_P(P) for P in calibs_P]

    def unproject(points, offsets, depths):                               # decode_location_flatten anno_encoder.py:142-155
        uv = (points + offsets) * down_ratio - pads[batch_idxs]
        cu = torch.tensor([calibs[int(b)]['c_u'] for b in batch_idxs]); cv = torch.tensor([calibs[int(b)]['c_v'] for b in batch_idxs])
        fu = torch.tensor([calibs[int(b)]['f_u'] for b in batch_idxs]); fv = torch.tensor([calibs[int(b)]['f_v'] for b in batch_idxs])
        bx = torch.tensor([calibs[int(b)]['b_x'] for b in batch_idxs]); by = torch.tensor([calibs[int(b)]['b_y'] for b in batch_idxs])
        x = ((uv[:, 0] - cu) * depths) / fu + bx
        y = ((uv[:, 1] - cv) * depths) / fv + by
        return torch.stack([x, y, depths], 1)

    t_loc = unproject(pts, t_off, t_depth)
    t_corners = encode_box3d(t_roty, t_dims, t_loc)
    trunc = st('trunc_mask').view(-1)[reg_mask].bool()

    # predictions at the object centres (select_point_of_interest layers/utils.py:120-145)
    idx = (centers[..., 1].long() * W + centers[..., 0].long())           # [B, M]
    pois = pred_reg.view(B, C, H * W).permute(0, 2, 1).gather(1, idx.unsqueeze(-1).expand(B, M, C)).reshape(-1, C)[reg_mask]
    p_reg2d = F.relu(pois[m2d][:, key2channel('2d_dim')])
    p_off = pois[:, key2channel('3d_offset')]
    p_dims = pois[:, key2channel('3d_dim')].exp() * torch.tensor(DIM_MEAN)[t_cls]
    p_ori = torch.cat((pois[:, key2channel('ori_cls')], pois[:, key2channel('ori_offset')]), 1)
    p_depth = (1 / torch.sigmoid(pois[:, key2channel('depth')].squeeze(-1)) - 1).clamp(0.1, 100)
    p_dunc = pois[:, key2channel('depth_uncertainty')].squeeze(-1).clamp(*UNC_RANGE)
    kpt = st('keypoints').view(B * M, -1, 3)[reg_mask].float()
    t_kp, t_kpm = kpt[..., :2], kpt[..., 2]
    t_kdm = st('keypoints_depth_mask').view(-1, 3)[reg_mask].bool()
    p_kp = pois[:, key2channel('corner_offset')].reshape(-1, 10, 2)
    # decode_depth_from_keypoints_batch anno_encoder.py:174-206 -- NB calib = calibs[idx] with idx the RANK of the image
    # among the images that have objects (enumerate over unique batch indices), not the image index itself
    ranks = {int(g): r for r, g in enumerate(torch.unique(batch_idxs, sorted=True).tolist())}
    fu_kp = torch.tensor([calibs[0 if B == 1 else ranks[int(b)]]['f_u'] for b in batch_idxs])
    h3d = p_dims[:, 1]
    ch = p_kp[:, -2, 1] - p_kp[:, -1, 1]
    c02 = p_kp[:, [0, 2], 1] - p_kp[:, [4, 6], 1]
    c13 = p_kp[:, [1, 3], 1] - p_kp[:, [5, 7], 1]
    d_c = fu_kp * h3d / (F.relu(ch) * down_ratio + 1e-3)
    d_02 = (fu_kp.unsqueeze(-1) * h3d.unsqueeze(-1) / (F.relu(c02) * down_ratio + 1e-3)).mean(1)
    d_13 = (fu_kp.unsqueeze(-1) * h3d.unsqueeze(-1) / (F.relu(c13) * down_ratio + 1e-3)).mean(1)
    p_kd = torch.stack([d_c, d_02, d_13], 1).clamp(0.1, 100)
    p_kunc = pois[:, key2channel('corner_uncertainty')].clamp(*UNC_RANGE)
    # soft_combine :241-248
    unc = torch.cat((p_dunc.unsqueeze(-1), p_kunc), 1).exp()
    depths = torch.cat((p_depth.unsqueeze(-1), p_kd), 1)
    wts = 1 / unc
    wts = wts / wts.sum(1, keepdim=True)
    soft = (depths * wts).sum(1)
    p_loc = unproject(pts, p_off, soft)
    bin_cls = torch.softmax(p_ori[:, :8].view(-1, 4, 2), 2)[..., 1]        # decode_axes_orientation :245-295
    bi = bin_cls.argmax(1)
    offs = p_ori[:, 8:].view(-1, 4, 2)[torch.arange(p_ori.shape[0]), bi]
    alpha = torch.atan2(offs[:, 0], offs[:, 1]) + torch.tensor([0, PI / 2, PI, -PI / 2])[bi]
    roty = alpha + torch.atan2(p_loc[:, 0], p_loc[:, 2])
    roty = torch.where(roty > PI, roty - 2 * PI, roty)
    roty = torch.where(roty < -PI, roty + 2 * PI, roty)
    p_corners = encode_box3d(roty, p_dims, p_loc)

    w = LOSS_WEIGHTS
    out, log = {}, {}
    hl, npos = focal_loss(pred_cls, hm)
    out['hm_loss'] = w['hm_loss'] * hl / torch.clamp(npos, 1)
    l2d, iou = giou_loss(p_reg2d, t_reg2d)
    out['bbox_loss'] = w['bbox_loss'] * l2d.mean()
    log['2D_IoU'] = iou.mean().detach()
    depth_mae = (p_depth - t_depth).abs() / t_depth
    dl = w['depth_loss'] * (p_depth - t_depth).abs()
    log['depth_loss'] = dl.detach().mean()
    out['depth_loss'] = (dl * torch.exp(-p_dunc) + p_dunc * w['depth_loss']).mean()
    ol = (p_off - t_off).abs().sum(1)
    out['trunc_offset_loss'] = w['trunc_offset_loss'] * torch.log(1 + ol[trunc]).sum() / torch.clamp(trunc.sum(), min=1)
    out['offset_loss'] = w['offset_loss'] * ol[~trunc].mean()
    out['orien_loss'] = w['orien_loss'] * multibin_loss(p_ori, t_ori)
    out['dims_loss'] = w['dims_loss'] * (p_dims - t_dims).abs().sum(1).mean()
    out['corner_loss'] = w['corner_loss'] * (p_corners - t_corners).abs().sum(2).mean()
    kl = w['keypoint_loss'] * (p_kp - t_kp).abs().sum(2) * t_kpm
    out['keypoint_loss'] = kl.sum() / torch.clamp(t_kpm.sum(), min=1)
    t_kd = t_depth.unsqueeze(-1).repeat(1, 3)
    vl = w['keypoint_depth_loss'] * (p_kd[t_kdm] - t_kd[t_kdm]).abs()
    il = w['keypoint_depth_loss'] * (p_kd[~t_kdm].detach() - t_kd[~t_kdm]).abs()
    log['keypoint_depth_loss'] = vl.detach().mean()
    vl = vl * torch.exp(-p_kunc[t_kdm]) + w['keypoint_depth_loss'] * p_kunc[t_kdm]
    il = il * torch.exp(-p_kunc[~t_kdm])
    out['keypoint_depth_loss'] = vl.sum() / torch.clamp(t_kdm.sum(), 1) + il.sum() / torch.clamp((~t_kdm).sum(), 1)
    kmae = (p_kd - t_depth.unsqueeze(-1)).abs() / t_depth.unsqueeze(-1)
    cmae = torch.cat((depth_mae.unsqueeze(1), kmae), 1)
    out['weighted_avg_depth_loss'] = w['weighted_avg_depth_loss'] * (soft - t_depth).abs().mean()
    log.update(depth_MAE=depth_mae.mean(), center_MAE=kmae[:, 0].mean(), **{'02_MAE': kmae[:, 1].mean(), '13_MAE': kmae[:, 2].mean()})
    log['lower_MAE'] = cmae.min(1)[0].mean()
    log['hard_MAE'] = cmae[torch.arange(cmae.shape[0]), unc.argmin(1)].mean()
    log['soft_MAE'] = ((soft - t_depth).abs() / t_depth).mean()
    log['mean_MAE'] = ((depths.mean(1) - t_depth).abs() / t_depth).mean()
    return out, {k: v.detach() for k, v in log.items()}


def detector_train_losses(sd, images, fields, edge_indices, edge_lens, calibs_P):
    """KeypointDetector.forward training branch (model/detector.py:32-34 -> Detect_Head.forward detector_head.py:17-21):
    train-mode backbone + predictor, then Loss_Computation. Returns (loss_dict, log_dict); differentiable w.r.t. every
    tensor of `sd` that requires grad."""
    with training_mode():
        feats = backbone(sd, images)
        pred = predictor(sd, feats, edge_indices, edge_lens)
    return loss_computation(pred['cls'], pred['reg'], fields, calibs_P)
