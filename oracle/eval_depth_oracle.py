"""TEST INFRASTRUCTURE ONLY (oracle) — numpy float32 restatement of PostProcessor.evaluate_3D_depths
(model/head/detector_infer.py:280-359, the --eval_depth diagnostic), step by step in float32 like the reference's torch
ops, extended image by image for B > 1.

The reference is batch-1 only: it gathers every slot at its centre, keeps the reg_mask ones, decodes the dimensions
(anno_encoder.py:221-243), the direct depth (:124-140, inv_sigmoid) and the three key-point depths of
decode_depth_from_keypoints_batch (:187-219, with calibs[0]), and measures every estimator against locations[..., 2].
Here every image uses its own f_u and contributes its valid slots in slot order, and a valid slot whose centre lies
outside the map (or whose class lies outside dim_mean) gives NaN in every key, as the kernel does. Pinned against the
unmodified reference by tests/golden/eval_depths.npz (oracle/make_golden_eval_depths.py)."""
import numpy as np

KEYS = ('direct', 'direct_sigma', 'keypoint_center', 'keypoint_02', 'keypoint_13', 'keypoint_center_sigma',
        'keypoint_02_sigma', 'keypoint_13_sigma', 'sigma_min', 'sigma_weighted', 'mean', 'min', 'target')
f32 = np.float32


def image_errors(reg, f_u, dim_mean, centers, reg_mask, cls_ids, locations, down_ratio=4, depth_range=(0.1, 100.0)):
    """ONE image: reg [50, H, W], f_u scalar, dim_mean [C, 3], centers [M, 2] (x, y), reg_mask / cls_ids [M],
    locations [M, 3] -> {key: float32 [n_valid]} in slot order."""
    reg = np.asarray(reg, f32)
    R, H, W = reg.shape
    valid = np.asarray(reg_mask) != 0
    pts = np.asarray(centers, f32)[valid]
    cls_f = np.asarray(cls_ids, f32)[valid]
    z = np.asarray(locations, f32).reshape(-1, 3)[valid, 2]
    idx_f = pts[:, 1] * f32(W) + pts[:, 0]                               # index[:, :, 1] * w + index[:, :, 0]
    inside = (pts[:, 0] >= 0) & (pts[:, 0] < W) & (pts[:, 1] >= 0) & (pts[:, 1] < H) & (idx_f < f32(H * W)) \
        & (cls_f > -1) & (cls_f < len(dim_mean))
    idx = np.where(inside, idx_f, 0).astype(np.int64)                     # .long() truncates
    q = reg.reshape(R, H * W)[:, idx].T                                   # [n, 50]
    cls = np.where(inside, cls_f, 0).astype(np.int64)
    dims = np.exp(q[:, 29:32]) * np.asarray(dim_mean, f32)[cls]          # (l, h, w)
    h = dims[:, 1]
    lo, hi = f32(depth_range[0]), f32(depth_range[1])
    direct = np.clip(f32(1) / (f32(1) / (f32(1) + np.exp(-q[:, 48]))) - f32(1), lo, hi)
    kp_y = q[:, 6:26].reshape(-1, 10, 2)[:, :, 1]
    fu, dr, eps = f32(f_u), f32(down_ratio), f32(1e-3)

    def kp_depth(top, bottom):
        return fu * h / (np.maximum(kp_y[:, top] - kp_y[:, bottom], f32(0)) * dr + eps)
    center = np.clip(kp_depth(8, 9), lo, hi)
    c02 = np.clip((kp_depth(0, 4) + kp_depth(2, 6)) / f32(2), lo, hi)
    c13 = np.clip((kp_depth(1, 5) + kp_depth(3, 7)) / f32(2), lo, hi)
    depths = np.stack([direct, center, c02, c13], 1).astype(f32)
    sig = np.exp(np.concatenate([q[:, 49:50], q[:, 26:29]], 1)).astype(f32)
    min_unc = depths[np.arange(len(depths)), np.argmin(sig, 1)]           # first index on ties, like torch.argmin
    w = f32(1) / sig
    w = w / w.sum(1, keepdims=True)
    weighted = (depths * w).sum(1)
    err = np.abs(depths - z[:, None])
    out = {'direct': err[:, 0], 'direct_sigma': sig[:, 0], 'keypoint_center': err[:, 1], 'keypoint_02': err[:, 2],
           'keypoint_13': err[:, 3], 'keypoint_center_sigma': sig[:, 1], 'keypoint_02_sigma': sig[:, 2],
           'keypoint_13_sigma': sig[:, 3], 'sigma_min': np.abs(min_unc - z), 'sigma_weighted': np.abs(weighted - z),
           'mean': np.abs(depths.mean(1) - z), 'min': err.min(1), 'target': z}
    return {k: np.where(inside, v, f32(np.nan)).astype(f32) for k, v in out.items()}


def eval_depths(reg, f_u, dim_mean, centers, reg_mask, cls_ids, locations):
    """B images: reg [B, 50, H, W], f_u [B], the label fields [B, M, ...] -> ({key: float32 [N]} in (image, slot)
    order, valid objects per image)"""
    per = [image_errors(reg[b], f_u[b], dim_mean, centers[b], reg_mask[b], cls_ids[b], locations[b])
           for b in range(len(reg))]
    return ({k: np.concatenate([p[k] for p in per]) for k in KEYS},
            [int((np.asarray(reg_mask[b]) != 0).sum()) for b in range(len(reg))])
