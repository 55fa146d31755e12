"""Deterministic synthetic KITTI-shaped workload (SURVEY.md §8d): weights, images, edge indices, calibration.

Everything is drawn from a numpy PCG64 stream so that the build container, the GPU box, the tests and
bench.py all see bit-identical tensors without any dataset or checkpoint (there is no network).
Shapes follow the reference: data/datasets/kitti.py:126-179 (edge indices), :218-228 (padding),
config/defaults.py (sizes), runs/monoflex.yaml (heads).
"""
import math

import numpy as np
import torch

# typical KITTI P2 (SURVEY §8d)
KITTI_P2 = ((721.5377, 0.0, 609.5593, 44.85728),
            (0.0, 721.5377, 172.854, 0.2163791),
            (0.0, 0.0, 1.0, 0.002745884))
PAD_SIZE = (19, 4)                       # 1242x375 image centred in 1280x384 (kitti.py:222-223)

REG_BRANCH_CH = [[4], [2], [20], [3], [3], [8, 8], [1], [1]]   # runs/monoflex.yaml:28
NUM_CLASSES = 3
HEAD_CONV = 256


def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))


def dla34_param_shapes():
    """(key, shape, kind) for every tensor of KeypointDetector.state_dict() in reference order-independent form.
    kind in {conv, bn_w, bn_b, bn_m, bn_v, bn_n, bias, up, offw, offb, dcnw, dcnb, conv1d}."""
    out = []

    def conv(p, co, ci, k):
        out.append((p + '.weight', (co, ci, k, k), 'conv'))

    def bn(p, c):
        out.extend([(p + '.weight', (c,), 'bn_w'), (p + '.bias', (c,), 'bn_b'), (p + '.running_mean', (c,), 'bn_m'),
                    (p + '.running_var', (c,), 'bn_v'), (p + '.num_batches_tracked', (), 'bn_n')])

    def block(p, ci, co):
        conv(p + '.conv1', co, ci, 3); bn(p + '.bn1', co); conv(p + '.conv2', co, co, 3); bn(p + '.bn2', co)

    def tree(p, levels, ci, co, level_root, root_dim=0):
        if root_dim == 0:
            root_dim = 2 * co
        if level_root:
            root_dim += ci
        if levels == 1:
            block(p + '.tree1', ci, co); block(p + '.tree2', co, co)
            conv(p + '.root.conv', co, root_dim, 1); bn(p + '.root.bn', co)
        else:
            tree(p + '.tree1', levels - 1, ci, co, False, 0)
            tree(p + '.tree2', levels - 1, co, co, False, root_dim + co)
        if ci != co:
            conv(p + '.project.0', co, ci, 1); bn(p + '.project.1', co)

    b = 'backbone.base'
    conv(b + '.base_layer.0', 16, 3, 7); bn(b + '.base_layer.1', 16)
    conv(b + '.level0.0', 16, 16, 3); bn(b + '.level0.1', 16)
    conv(b + '.level1.0', 32, 16, 3); bn(b + '.level1.1', 32)
    ch, lv = [16, 32, 64, 128, 256, 512], [1, 1, 1, 2, 2, 1]
    for i in range(2, 6):
        tree('%s.level%d' % (b, i), lv[i], ch[i - 1], ch[i], i > 2)

    def dcn(p, ci, co):
        out.append((p + '.conv.weight', (co, ci, 3, 3), 'dcnw'))
        out.append((p + '.conv.bias', (co,), 'dcnb'))
        out.append((p + '.conv.conv_offset_mask.weight', (27, ci, 3, 3), 'offw'))
        out.append((p + '.conv.conv_offset_mask.bias', (27,), 'offb'))
        bn(p + '.actf.0', co)

    def ida(p, o, chans, up_f):
        for i in range(1, len(chans)):
            dcn('%s.proj_%d' % (p, i), chans[i], o)
            out.append(('%s.up_%d.weight' % (p, i), (o, 1, 2 * up_f[i], 2 * up_f[i]), 'up'))
            dcn('%s.node_%d' % (p, i), o, o)

    ida('backbone.dla_up.ida_0', 256, [256, 512], [1, 2])
    ida('backbone.dla_up.ida_1', 128, [128, 256, 256], [1, 2, 2])
    ida('backbone.dla_up.ida_2', 64, [64, 128, 128, 128], [1, 2, 2, 2])
    ida('backbone.ida_up', 64, [64, 128, 256], [1, 2, 4])

    h = 'heads.predictor'
    conv(h + '.class_head.0', HEAD_CONV, 64, 3)
    for s, k in (('weight', 'bn_w'), ('bias', 'bn_b'), ('running_mean', 'bn_m'), ('running_var', 'bn_v')):
        out.append(('%s.class_head.1.%s' % (h, s), (HEAD_CONV,), k))
    out.append((h + '.class_head.2.weight', (NUM_CLASSES, HEAD_CONV, 1, 1), 'conv'))
    out.append((h + '.class_head.2.bias', (NUM_CLASSES,), 'clsbias'))
    for i, br in enumerate(REG_BRANCH_CH):
        conv('%s.reg_features.%d.0' % (h, i), HEAD_CONV, 64, 3)
        for s, k in (('weight', 'bn_w'), ('bias', 'bn_b'), ('running_mean', 'bn_m'), ('running_var', 'bn_v')):
            out.append(('%s.reg_features.%d.1.%s' % (h, i, s), (HEAD_CONV,), k))
        for j, c in enumerate(br):
            out.append(('%s.reg_heads.%d.%d.weight' % (h, i, j), (c, HEAD_CONV, 1, 1), 'conv'))
            out.append(('%s.reg_heads.%d.%d.bias' % (h, i, j), (c,), 'bias'))
    for name, co in (('trunc_heatmap_conv', NUM_CLASSES), ('trunc_offset_conv', 2)):
        q = '%s.%s' % (h, name)
        out.append((q + '.0.weight', (HEAD_CONV, HEAD_CONV, 3), 'conv1d'))
        out.append((q + '.0.bias', (HEAD_CONV,), 'bias'))
        bn(q + '.1', HEAD_CONV)
        out.append((q + '.3.weight', (co, HEAD_CONV, 1), 'conv1d'))
        out.append((q + '.3.bias', (co,), 'bias'))
    return out


_CALIB = None


def _calibration():
    global _CALIB
    if _CALIB is None:
        import os
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'synthetic_calib.npz')
        with np.load(path) as z:
            _CALIB = {k: z[k] for k in z.files}
    return _CALIB


def make_state_dict(seed=0, calibrated=True):
    """Random-init weights of the reference architecture (same keys/shapes as the reference state_dict).
    He-normal convs, BN/IABN stats randomised (gamma>0 so |gamma| == gamma, SURVEY H4), non-zero
    conv_offset_mask (SURVEY Appendix B.7), bilinear up-sampling kernels (fill_up_weights dla_dcn.py:372)."""
    g = _rng(seed)
    sd = {}
    for key, shape, kind in dla34_param_shapes():
        if kind in ('conv', 'dcnw', 'conv1d'):
            fan_in = int(np.prod(shape[1:]))
            # residual branches sum two unit-variance signals: keep the variance stationary (gain 1 not 2)
            gain = 1.0 if key.endswith('conv2.weight') else 2.0
            if '.reg_heads.' in key or key.endswith('class_head.2.weight') or key.endswith('.3.weight'):
                gain = 0.125   # keep logits / regression outputs O(1): no sigmoid saturation ties
            v = g.standard_normal(shape) * math.sqrt(gain / fan_in)
        elif kind == 'offw':
            # offsets of ~1 px for unit-variance inputs whatever Cin (real DCN offsets are a few pixels)
            v = g.standard_normal(shape) / math.sqrt(int(np.prod(shape[1:])))
        elif kind == 'offb':
            v = g.standard_normal(shape) * 0.1
        elif kind == 'bn_w':
            v = g.uniform(0.5, 1.5, shape)
        elif kind == 'bn_b':
            v = g.standard_normal(shape) * 0.1
        elif kind == 'bn_m':
            v = g.standard_normal(shape) * 0.1
        elif kind == 'bn_v':
            v = g.uniform(0.5, 1.5, shape)
        elif kind == 'bn_n':
            sd[key] = torch.tensor(0, dtype=torch.long)
            continue
        elif kind in ('bias', 'dcnb'):
            v = g.standard_normal(shape) * 0.05
        elif kind == 'clsbias':
            v = np.full(shape, -math.log(1 / 0.01 - 1))
        elif kind == 'up':
            k = shape[2]
            f = math.ceil(k / 2)
            c = (2 * f - 1 - f % 2) / (2.0 * f)
            w1 = np.array([1 - abs(i / f - c) for i in range(k)])
            v = np.broadcast_to(np.outer(w1, w1), shape) * g.uniform(0.9, 1.1, (shape[0], 1, 1, 1))
        else:
            raise KeyError(kind)
        sd[key] = _t(v)
    if calibrated:
        # per-DCN factor bringing the rms offset to ~1.5 px (oracle/calibrate_bn.py), as in a trained net
        for k, v in _calibration().items():
            sd[k] = sd[k] * float(v)
    return sd


def make_images(batch, height=384, width=1280, seed=1):
    """randn images ~ normalised KITTI (config/defaults.py:34-36)."""
    return _t(_rng(seed).standard_normal((batch, 3, height, width)))


def edge_indices(out_w=320, out_h=96, pad=PAD_SIZE, down_ratio=4):
    """Border pixel list of the un-padded image on the stride-4 map, (x,y) int64 [K_max,2] zero padded, and
    edge_len = count-1 (data/datasets/kitti.py:126-179, 279-285)."""
    img_w, img_h = out_w * down_ratio - 2 * pad[0], out_h * down_ratio - 2 * pad[1] - 1
    x_min, y_min = math.ceil(pad[0] / down_ratio), math.ceil(pad[1] / down_ratio)
    x_max, y_max = (pad[0] + img_w - 1) // down_ratio, (pad[1] + img_h - 1) // down_ratio
    pts = [(x_min, y) for y in range(y_min, y_max)]
    pts += [(x, y_max) for x in range(x_min, x_max)]
    pts += [(x_max, y) for y in range(y_max, y_min, -1)]
    pts += [(x, y_min) for x in range(x_max, x_min - 1, -1)]
    k_max = (out_w + out_h) * 2
    idx = torch.zeros(k_max, 2, dtype=torch.long)
    idx[:len(pts)] = torch.tensor(pts, dtype=torch.long)
    return idx, len(pts) - 1, (img_w, img_h)


def make_targets(batch, out_w=320, out_h=96):
    """Per-image inference-time target fields the hot path reads (detector_infer.py:53-58,
    detector_predictor.py:138-139): calib P, pad_size, size, edge_indices, edge_len."""
    idx, n, img_size = edge_indices(out_w, out_h)
    return dict(edge_indices=idx.unsqueeze(0).repeat(batch, 1, 1), edge_len=torch.full((batch,), n, dtype=torch.long),
                calib_P=[KITTI_P2 for _ in range(batch)],
                pad_size=torch.tensor([PAD_SIZE] * batch, dtype=torch.float32).view(batch, 2),
                size=[(out_w * 4, out_h * 4)] * batch)   # ParamsList.size = PADDED image (kitti.py:271,289)


def make_head_logits(batch, out_w=320, out_h=96, seed=2):
    """Decode-only workload (SURVEY §8d): heat-map logits ~N(-3,1.5) -> >>50 distinct local maxima per class;
    regression map ~N(0,0.5)."""
    g = _rng(seed)
    cls = _t(g.standard_normal((batch, NUM_CLASSES, out_h, out_w)) * 1.5 - 3.0)
    reg = _t(g.standard_normal((batch, 50, out_h, out_w)) * 0.5)
    return cls, reg


def make_param_lists(tg):
    """The per-image ParamsList objects engine/inference.py hands to model(images, targets)."""
    from .structures import Calibration, ParamsList
    out = []
    for b in range(len(tg['calib_P'])):
        t = ParamsList(tg['size'][b], is_train=False)
        t.add_field('calib', Calibration(tg['calib_P'][b]))
        t.add_field('pad_size', tg['pad_size'][b])
        t.add_field('edge_indices', tg['edge_indices'][b])
        t.add_field('edge_len', tg['edge_len'][b])
        out.append(t)
    return out


# ------------------------------------------------------------------------------------------- training targets (row R12)
DIM_MEAN = ((3.8840, 1.5261, 1.6286), (0.8423, 1.7607, 0.6602), (1.7635, 1.7372, 0.5968))   # config/defaults.py:206-208
MAX_OBJECTS = 40                                                                             # config/defaults.py DATASETS.MAX_OBJECTS
ALPHA_CENTERS = (0.0, math.pi / 2, math.pi, -math.pi / 2)                                    # kitti.py:75


def _project(P, pts):
    """rect-camera points [n,3] -> pixel (u, v) with the 3x4 projection matrix (kitti_utils.py project_rect_to_image)."""
    h = np.concatenate([pts, np.ones((pts.shape[0], 1))], axis=1) @ np.asarray(P, dtype=np.float64).T
    return h[:, :2] / h[:, 2:3]


def _gaussian(hm, cx, cy, rx, ry):
    """umich gaussian splat with independent radii (data/datasets/kitti_utils.py draw_umich_gaussian[_2D] semantics:
    sigma = (2r+1)/6 per axis, element-wise max with what is already there)."""
    H, W = hm.shape
    sx, sy = (2 * rx + 1) / 6.0, (2 * ry + 1) / 6.0
    x0, x1, y0, y1 = max(0, cx - rx), min(W - 1, cx + rx), max(0, cy - ry), min(H - 1, cy + ry)
    ys, xs = np.mgrid[y0:y1 + 1, x0:x1 + 1]
    g = np.exp(-((xs - cx) ** 2) / (2 * sx * sx) - ((ys - cy) ** 2) / (2 * sy * sy)).astype(np.float32)
    hm[y0:y1 + 1, x0:x1 + 1] = np.maximum(hm[y0:y1 + 1, x0:x1 + 1], g)
    hm[cy, cx] = 1.0


def make_train_targets(batch, seed=5, out_w=320, out_h=96, max_objs=MAX_OBJECTS, empty_image=1):
    """Synthetic per-image TRAINING target fields with the shapes, dtypes and encodings of KITTIDataset.__getitem__
    (data/datasets/kitti.py:296-521): objects are sampled in 3D (class-mean dimensions, depth 4-60 m, random yaw),
    projected with KITTI_P2, and encoded exactly like the reference encodes labels (projected centre, truncated centres
    moved to the image border, 10 keypoints relative to the integer centre with visibility, multi-bin orientation, ...).
    Image `empty_image` (if < batch) gets no object: the reference indexes calibrations by RANK among non-empty images in
    decode_depth_from_keypoints_batch (anno_encoder.py:186), which only shows with an empty image in the batch.
    Returns a list of dicts of numpy arrays (one per image)."""
    g = _rng(seed)
    img_w, img_h = out_w * 4 - 2 * PAD_SIZE[0], out_h * 4 - 2 * PAD_SIZE[1]
    pad = np.asarray(PAD_SIZE, dtype=np.float64)
    x_min, y_min = math.ceil(PAD_SIZE[0] / 4), math.ceil(PAD_SIZE[1] / 4)
    x_max, y_max = (PAD_SIZE[0] + img_w - 1) // 4, (PAD_SIZE[1] + img_h - 1) // 4
    P = np.asarray(KITTI_P2, dtype=np.float64)
    out = []
    for b in range(batch):
        f = dict(hm=np.zeros((NUM_CLASSES, out_h, out_w), np.float32), cls_ids=np.zeros(max_objs, np.int32),
                 target_centers=np.zeros((max_objs, 2), np.int32), bboxes=np.zeros((max_objs, 4), np.float32),
                 keypoints=np.zeros((max_objs, 10, 3), np.float32), keypoints_depth_mask=np.zeros((max_objs, 3), np.float32),
                 dimensions=np.zeros((max_objs, 3), np.float32), locations=np.zeros((max_objs, 3), np.float32),
                 rotys=np.zeros(max_objs, np.float32), alphas=np.zeros(max_objs, np.float32),
                 offset_3D=np.zeros((max_objs, 2), np.float32), orientations=np.zeros((max_objs, 8), np.float32),
                 reg_mask=np.zeros(max_objs, np.uint8), trunc_mask=np.zeros(max_objs, np.uint8),
                 reg_weight=np.zeros(max_objs, np.float32), pad_size=np.asarray(PAD_SIZE, np.float32),
                 ori_img=np.zeros((1,), np.float32))
        n_obj = 0 if b == empty_image else int(g.integers(3, 14))
        i = 0
        for _ in range(n_obj * 3):
            if i >= n_obj:
                break
            cls = int(g.choice(3, p=[0.7, 0.15, 0.15]))
            l, h, w = (np.asarray(DIM_MEAN[cls]) * g.uniform(0.85, 1.15, 3))
            z = float(g.uniform(4.0, 60.0))
            x = float(g.uniform(-0.98, 0.98)) * z                     # beyond ~0.84 z the centre leaves the image: truncated
            yb = 1.65 + float(g.normal(0, 0.15))                      # bottom-face height in camera coordinates (y down)
            ry = float(g.uniform(-math.pi, math.pi))
            loc = np.array([x, yb - h / 2, z])                        # kitti.py:352-353: centre of the box
            c, s = math.cos(ry), math.sin(ry)
            xc = np.array([l, l, -l, -l, l, l, -l, -l]) / 2
            yc = np.array([0, 0, 0, 0, -h, -h, -h, -h])
            zc = np.array([w, -w, -w, w, w, -w, -w, w]) / 2
            corners = np.stack([c * xc + s * zc + x, yc + yb, -s * xc + c * zc + z], axis=1)   # object3d generate_corners3d
            if corners[:, 2].min() <= 0.5:
                continue
            c2 = _project(P, corners)
            box = np.array([c2[:, 0].min(), c2[:, 1].min(), c2[:, 0].max(), c2[:, 1].max()])
            box = np.array([max(box[0], 0), max(box[1], 0), min(box[2], img_w - 1), min(box[3], img_h - 1)])
            if box[2] - box[0] < 4 or box[3] - box[1] < 4:
                continue
            pc = _project(P, loc[None])[0]
            inside = (0 <= pc[0] <= img_w - 1) and (0 <= pc[1] <= img_h - 1)
            tpc = pc.copy()
            if not inside:                                            # kitti.py:372-381 / approx_proj_center 'intersect'
                c2d = (box[:2] + box[2:]) / 2
                d = pc - c2d
                ts = [1.0]
                for k, lim in ((0, img_w - 1), (1, img_h - 1)):
                    if d[k] > 0:
                        ts.append((lim - c2d[k]) / d[k])
                    elif d[k] < 0:
                        ts.append((0 - c2d[k]) / d[k])
                tpc = c2d + d * max(0.0, min(ts))
            kp3 = np.concatenate([corners, corners[:4].mean(0, keepdims=True), corners[4:].mean(0, keepdims=True)], 0)
            kp2 = _project(P, kp3)
            vis = (kp2[:, 0] >= 0) & (kp2[:, 0] <= img_w - 1) & (kp2[:, 1] >= 0) & (kp2[:, 1] <= img_h - 1) & (kp3[:, 2] > 0)
            vis = np.append(np.tile(vis[:4] | vis[4:8], 2), np.tile(vis[8] | vis[9], 2))        # kitti.py:397-399
            dvalid = np.stack((vis[[8, 9]].all(), vis[[0, 2, 4, 6]].all(), vis[[1, 3, 5, 7]].all())).astype(np.float32)
            kp2 = (kp2 + pad) / 4
            tpc, pcf = (tpc + pad) / 4, (pc + pad) / 4
            boxf = (box + np.tile(pad, 2)) / 4
            tc = np.round(tpc).astype(np.int64)
            tc[0], tc[1] = min(max(tc[0], x_min), x_max), min(max(tc[1], y_min), y_max)
            pred_2d = boxf[0] <= tc[0] <= boxf[2] and boxf[1] <= tc[1] <= boxf[3] and g.uniform() > 0.08   # + some 'wrong annotations'
            bw, bh = boxf[2] - boxf[0], boxf[3] - boxf[1]
            if not inside:                                            # kitti.py:428-433 (edge heat map: 1-D gaussian)
                rx = max(0, int(min(tc[0] - boxf[0], boxf[2] - tc[0]) * 0.5))
                ryy = max(0, int(min(tc[1] - boxf[1], boxf[3] - tc[1]) * 0.5))
                if min(rx, ryy) > 0:
                    rx = 0
                _gaussian(f["hm"][cls], int(tc[0]), int(tc[1]), rx, ryy)
            else:
                r = max(0, int(0.3 * min(bw, bh)))
                _gaussian(f["hm"][cls], int(tc[0]), int(tc[1]), r, r)
            alpha = ry - math.atan2(x, z)
            alpha = (alpha + math.pi) % (2 * math.pi) - math.pi
            f["cls_ids"][i] = cls
            f["target_centers"][i] = tc
            f["offset_3D"][i] = pcf - tc
            if pred_2d:
                f["bboxes"][i] = boxf
            f["keypoints"][i] = np.concatenate([kp2 - tc[None].astype(np.float64), vis[:, None].astype(np.float64)], 1)
            f["keypoints_depth_mask"][i] = dvalid
            f["dimensions"][i] = (l, h, w)
            f["locations"][i] = loc
            f["rotys"][i], f["alphas"][i] = ry, alpha
            enc = np.zeros(8)                                          # kitti.py:181-200 encode_alpha_multibin(num_bin=4)
            offs = alpha - np.asarray(ALPHA_CENTERS)
            offs[offs > math.pi] -= 2 * math.pi
            offs[offs < -math.pi] += 2 * math.pi
            for k in range(4):
                if abs(offs[k]) < math.pi / 4 + math.pi / 12:
                    enc[k], enc[4 + k] = 1, offs[k]
            f["orientations"][i] = enc
            f["reg_mask"][i], f["reg_weight"][i], f["trunc_mask"][i] = 1, 1, int(not inside)
            i += 1
        out.append(f)
    return out


def make_train_param_lists(fields, out_w=320, out_h=96):
    """ParamsList objects (is_train=True) as the reference's collate hands them to model(images, targets)
    (data/collate_batch.py); field names of kitti.py:496-521. The edge indices are those of an (out_w x 4) x (out_h x 4)
    padded image, the geometry make_train_targets was given."""
    from .structures import Calibration, ParamsList
    idx, n, img_size = edge_indices(out_w, out_h)
    res = []
    for f in fields:
        t = ParamsList((out_w * 4, out_h * 4), is_train=True)
        for k, v in f.items():
            t.add_field("2d_bboxes" if k == "bboxes" else k, torch.from_numpy(np.ascontiguousarray(v)))
        t.add_field("calib", Calibration(KITTI_P2))
        t.add_field("edge_indices", idx)
        t.add_field("edge_len", torch.tensor(n, dtype=torch.long))
        res.append(t)
    return res


def make_train_predictions(batch, fields, seed=6, out_w=320, out_h=96):
    """Predictor outputs for loss tests: `cls` = a valid heat map in (1e-4, 1-1e-4) (sigmoid_hm already applied,
    detector_predictor.py:163), `reg` ~ N(0, 0.5) with the regression vector at every object centre nudged towards the
    label so that all loss branches (valid / invalid key-point depths, every orientation bin) see sane magnitudes."""
    g = _rng(seed)
    logits = g.standard_normal((batch, NUM_CLASSES, out_h, out_w)) * 1.5 - 3.0
    cls = np.clip(1.0 / (1.0 + np.exp(-logits)), 1e-4, 1 - 1e-4).astype(np.float32)
    reg = (g.standard_normal((batch, 50, out_h, out_w)) * 0.5).astype(np.float32)
    for b, f in enumerate(fields):
        for i in np.nonzero(f["reg_mask"])[0]:
            x, y = f["target_centers"][i]
            kp = f["keypoints"][i, :, :2].reshape(-1)
            reg[b, 6:26, y, x] = kp + g.standard_normal(20).astype(np.float32) * 0.3
            reg[b, 4:6, y, x] = f["offset_3D"][i] + g.standard_normal(2).astype(np.float32) * 0.1
            bx = f["bboxes"][i]
            if bx[2] > bx[0]:
                reg[b, 0:4, y, x] = np.array([x - bx[0], y - bx[1], bx[2] - x, bx[3] - y]) * g.uniform(0.7, 1.3, 4)
            reg[b, 29:32, y, x] = g.standard_normal(3).astype(np.float32) * 0.1
            z = f["locations"][i, 2] * float(np.exp(g.normal(0, 0.1)))
            reg[b, 48, y, x] = -math.log(z)                              # 1/sigmoid(v) - 1 = exp(-v) = z
    return torch.from_numpy(cls), torch.from_numpy(reg)


def natural_image(w, h, seed):
    """uint8 [h, w, 3] RGB with smooth gradients, a few soft shapes and sensor-like noise: compressed as a PNG it behaves
    like a photograph rather than like zeros (the PNG decode's tests and tools/bench_png.py)"""
    g = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.empty((h, w, 3))
    for c in range(3):
        img[..., c] = 90 + 60 * np.sin(x / (37 + 11 * c) + g.uniform(0, 6)) * np.cos(y / (23 + 5 * c)) + 0.1 * y
    for _ in range(6):
        cx, cy, r = g.uniform(0, w), g.uniform(0, h), g.uniform(5, 80)
        img += (g.uniform(-60, 60, 3) * np.exp(-((x - cx) ** 2 + (y - cy) ** 2) / (2 * r * r))[..., None])
    img += g.normal(0, 4, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def dla34_imagenet_weights(seed=0, num_classes=1000):
    """A seeded stand-in for the ImageNet DLA-34 file (dla34-ba72cf86.pth) with its keys, in its order, and its shapes:
    the DLA-34 base's parameters and BN statistics (no num_batches_tracked, which the file predates) and the classifier
    `fc` (Conv2d(512, num_classes, 1)) last. Conv weights at He scale, BN affine and statistics near identity."""
    from .model.backbone.dla_dcn import dla34
    g = _rng(seed)
    base = dla34(pretrained=False)
    base.fc = torch.nn.Conv2d(base.channels[-1], num_classes, kernel_size=1, bias=True)
    out = {}
    for k, v in base.state_dict().items():
        if k.endswith("num_batches_tracked"):
            continue
        shape = tuple(v.shape)
        if k.endswith("running_var"):
            a = g.uniform(0.5, 1.5, shape)
        elif k.endswith("running_mean") or k.endswith("bias"):
            a = g.normal(0.0, 0.05, shape)
        elif len(shape) == 1:                                          # BN weight
            a = g.uniform(0.8, 1.2, shape)
        else:
            a = g.standard_normal(shape) * math.sqrt(2.0 / (shape[1] * shape[2] * shape[3]))
        out[k] = _t(a)
    return out
