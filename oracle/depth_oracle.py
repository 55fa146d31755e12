"""TEST INFRASTRUCTURE ONLY (oracle) — CPU fp32 restatement of every OUTPUT_DEPTH estimator of the PostProcessor
(model/head/detector_infer.py:148-278), oracle included, for ONE image at a time like the reference.

`decode_image(..., output_depth='soft')` restates the same decode as `monoflex_oracle.decode_image`, with the depth and its
error chosen by `output_depth`; tests/test_decode_depth.py checks that the soft result is bit-identical to it and pins
every method against the unmodified reference (oracle/make_golden_depth.py -> tests/golden/decode_depth.npz). The
shared pieces (channel map, class-mean dimensions, NMS / top-k / POI gather, calibration) come from monoflex_oracle."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.monoflex_oracle import DIM_MEAN, PI, calib_from_P, gather_pois, key2channel, nms_hm, select_topk

DEPTH_MODES = ('soft', 'hard', 'mean', 'oracle', 'direct', 'keypoints_avg', 'keypoints_center', 'keypoints_02',
               'keypoints_13')


def oracle_depths(box, clses, depths, sig, gt):
    """get_oracle_depths detector_infer.py:239-278 against ONE image's ground truth gt [G,7] = (valid, class, x1, y1, x2,
    y2, z). Starts from the mean of the four estimators; a detection whose nearest GT centre (same class; other classes
    count as 9999) overlaps it with 2D IoU >= 0.5 takes the estimator closest to the GT depth. The IoU is box_iou of
    engine/visualize_infer.py:23-27 in fp32: a zero-area union gives NaN, which is not < 0.5, so the match stands. Without
    valid GT the mean is kept (the reference raises there)."""
    depth, err = depths.mean(1), sig.mean(1)
    gt = gt[gt[:, 0] != 0]
    if gt.shape[0] == 0:
        return depth, err
    gt_center = (gt[:, 2:4] + gt[:, 4:6]) / 2
    for i in range(box.shape[0]):
        center = (box[i, :2] + box[i, 2:]) / 2
        dis = ((center.view(1, 2) - gt_center) ** 2).sum(1)
        dis[gt[:, 1] != clses[i]] = 9999
        g = gt[int(torch.argmin(dis))]
        b = box[i].numpy()
        t = g[2:6].numpy()
        inter = max(min(b[2], t[2]) - max(b[0], t[0]), 0) * max(min(b[3], t[3]) - max(b[1], t[1]), 0)
        union = (b[2] - b[0]) * (b[3] - b[1]) + (t[2] - t[0]) * (t[3] - t[1]) - inter
        with np.errstate(invalid='ignore', divide='ignore'):
            iou = np.float32(inter) / np.float32(union)
        if iou < 0.5:
            continue
        e = int(torch.argmin((depths[i] - g[6]).abs()))
        depth[i], err[i] = depths[i, e], sig[i, e]
    return depth, err


def decode_image(scores, clses, xs, ys, pois, calib, pad_size, img_size, det_threshold=0.2, down_ratio=4,
                 output_depth='soft', gt=None):
    """PostProcessor.forward detector_infer.py:103-232 for ONE image (the reference is batch-1 only, SURVEY H8),
    UNCERTAINTY_AS_CONFIDENCE=True. All inputs [K] / [K,50]; calib = calib_from_P(...); pad_size [2] (x,y) ;
    img_size (W,H); output_depth one of DEPTH_MODES; gt [G,7] (see oracle_depths) for 'oracle'. Returns result[N,14]."""
    if output_depth not in DEPTH_MODES:
        raise ValueError("output_depth %r is not one of %s" % (output_depth, DEPTH_MODES))
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
    if output_depth == 'soft':
        wts = 1 / sig                                                           # detector_infer.py:176-198
        wts = wts / wts.sum(1, keepdim=True)
        depth = (depths * wts).sum(1)
        err = (wts * sig).sum(1)
    elif output_depth == 'hard':                                                # :187-191
        best = (1 / sig).argmax(1)
        depth, err = depths[torch.arange(depths.shape[0]), best], sig.min(1).values
    elif output_depth == 'mean':                                                # :200-204
        depth, err = depths.mean(1), sig.mean(1)
    elif output_depth == 'oracle':                                              # :207-209
        depth, err = oracle_depths(box, clses, depths, sig, gt)
    elif output_depth == 'direct':                                              # :150-153
        depth, err = depths[:, 0], sig[:, 0]
    elif output_depth == 'keypoints_avg':                                       # :156-158
        depth, err = depths[:, 1:].mean(1), sig[:, 1:].mean(1)
    else:                                                                       # :160-170
        i = ('keypoints_center', 'keypoints_02', 'keypoints_13').index(output_depth) + 1
        depth, err = depths[:, i], sig[:, i]
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


def post_process(pred, calibs_P, pad_sizes, img_sizes, det_threshold=0.2, K=50, output_depth='soft', gts=None):
    """Batch wrapper: loops the batch-1 reference semantics per image (image b matched against its own ground truth
    gts[b] for the oracle depth). Returns list of result[N_i,14] plus the top-k tensors (scores, inds, clses, ys, xs)."""
    heat = nms_hm(pred['cls'])
    scores, inds, clses, ys, xs = select_topk(heat, K)
    pois = gather_pois(pred['reg'], inds)
    results = []
    for b in range(heat.shape[0]):
        results.append(decode_image(scores[b], clses[b], xs[b], ys[b], pois[b], calib_from_P(calibs_P[b]),
                                    pad_sizes[b], img_sizes[b], det_threshold, output_depth=output_depth,
                                    gt=None if gts is None else gts[b]))
    return results, (scores, inds, clses, ys, xs)
