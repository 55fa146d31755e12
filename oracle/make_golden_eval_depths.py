"""TEST TOOLING — tests/golden/eval_depths.npz: the UNMODIFIED reference PostProcessor.evaluate_3D_depths
(model/head/detector_infer.py:280-359, via oracle/ref_shims.py) at batch 1, on seeded 16 x 48 regression maps with
MAX_OBJECTS = 40 slots. Build container only:

    python -m oracle.make_golden_eval_depths

Every image mixes:
  * valid centres on every border of the map (the four corners and one point on each edge) and inside it;
  * all three classes;
  * invalid slots (reg_mask 0) between the valid ones, holding other classes, depths and centres, all inside the map:
    the reference gathers every slot before it applies reg_mask;
  * key-point heights <= 0 (relu makes the depth f_u * h / 1e-3, which clamps at 100);
  * direct depths beyond both ends of DEPTH_RANGE;
  * exact ties between the four uncertainties (argmin takes the first).
Images 0 and 2 use synthetic.py's KITTI P2, images 1 and 3 a second P2. The channels evaluate_3D_depths does not read are
zero. The script also asserts that the reference raises on an image without valid objects (torch.cat of no tensors)."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shims as rs            # noqa: E402
from monoflex_b200 import synthetic as syn    # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
H, W, M = 16, 48, 40
P2_OTHER = ((707.0493, 0.0, 604.0814, 45.75831), (0.0, 707.0493, 180.5066, -0.3454157), (0.0, 0.0, 1.0, 0.004981016))
KEYS = ('direct', 'direct_sigma', 'keypoint_center', 'keypoint_02', 'keypoint_13', 'keypoint_center_sigma',
        'keypoint_02_sigma', 'keypoint_13_sigma', 'sigma_min', 'sigma_weighted', 'mean', 'min', 'target')
BORDER = ((0, 0), (W - 1, 0), (0, H - 1), (W - 1, H - 1), (17, 0), (23, H - 1), (0, 7), (W - 1, 9))


def make_image(seed):
    """-> (reg [50, H, W] float32, centers [M, 2] int32, reg_mask [M] uint8, cls_ids [M] int32, locations [M, 3] f32)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    reg = np.zeros((50, H, W), np.float32)
    reg[6:26] = rng.normal(0, 4, (20, H, W))                 # key points: random heights, many of them <= 0
    reg[26:29] = rng.normal(0, 0.5, (3, H, W))               # key-point uncertainties (log)
    reg[29:32] = rng.normal(0, 0.2, (3, H, W))               # dimension offsets
    reg[48] = -np.log(rng.uniform(3, 70, (H, W)))            # direct depth 1 / sigmoid(x) - 1 = exp(-x)
    reg[49] = rng.normal(0, 0.5, (H, W))
    pix = [(x, y) for x in range(1, W - 1) for y in range(1, H - 1)]
    inner = [pix[i] for i in rng.permutation(len(pix))[:M]]
    n_valid = 16
    valid_slots = np.sort(rng.permutation(M)[:n_valid])
    centers = np.array(inner, np.int32)
    reg_mask = np.zeros(M, np.uint8)
    reg_mask[valid_slots] = 1
    for j, s in enumerate(valid_slots[:len(BORDER)]):
        centers[s] = BORDER[j]
    cls_ids = rng.integers(0, 3, M).astype(np.int32)
    cls_ids[valid_slots[:3]] = (0, 1, 2)
    locations = rng.uniform(-10, 10, (M, 3)).astype(np.float32)
    locations[:, 2] = rng.uniform(2, 80, M)
    for j, s in enumerate(valid_slots):
        x, y = centers[s]
        kind = j % 8
        if kind in (0, 1, 5):                                # plausible key points: heights that give depths 4..70
            hgt = rng.uniform(3, 60, 5).astype(np.float32)
            for top, bottom, hh in ((8, 9, hgt[0]), (0, 4, hgt[1]), (2, 6, hgt[2]), (1, 5, hgt[3]), (3, 7, hgt[4])):
                reg[6 + 2 * top + 1, y, x] = hh / 2
                reg[6 + 2 * bottom + 1, y, x] = -hh / 2
        if kind == 2:                                        # key-point heights <= 0: exactly zero and negative
            reg[6 + 2 * 8 + 1, y, x] = reg[6 + 2 * 9 + 1, y, x] = 1.5
            reg[6 + 2 * 0 + 1, y, x], reg[6 + 2 * 4 + 1, y, x] = -2.0, 3.0
            reg[6 + 2 * 1 + 1, y, x], reg[6 + 2 * 5 + 1, y, x] = -0.25, 0.25
        if kind == 3:                                        # direct depth below / above DEPTH_RANGE
            reg[48, y, x] = 6.0 if j % 16 == 3 else -6.5
        if kind == 4:                                        # all four uncertainties tied
            reg[49, y, x] = reg[26:29, y, x] = np.float32(rng.normal(0, 0.5))
        if kind == 6:                                        # a tie between the last two (argmin keeps index 2)
            reg[26:29, y, x] = (1.5, -0.75, -0.75)
            reg[49, y, x] = 0.25
        if kind == 7:                                        # the direct depth ties the smallest key-point uncertainty
            reg[49, y, x] = reg[27, y, x] = np.float32(-1.0)
            reg[26, y, x], reg[28, y, x] = 0.5, 0.0
    return reg, centers, reg_mask, cls_ids, locations


def ref_calib(P):
    from data.datasets.kitti_utils import Calibration
    c = Calibration.__new__(Calibration)
    P = np.array(P)
    c.P = P
    c.c_u, c.c_v, c.f_u, c.f_v = P[0, 2], P[1, 2], P[0, 0], P[1, 1]
    c.b_x, c.b_y = P[0, 3] / (-c.f_u), P[1, 3] / (-c.f_v)
    return c


def ref_targets(P, centers, reg_mask, cls_ids, locations):
    """the dict of the reference's prepare_targets(test=False) for one image: the fields evaluate_3D_depths reads"""
    return dict(calib=[ref_calib(P)], target_centers=torch.from_numpy(centers)[None],
                reg_mask=torch.from_numpy(reg_mask)[None], cls_ids=torch.from_numpy(cls_ids)[None],
                locations=torch.from_numpy(locations)[None])


def main():
    torch.set_num_threads(8)
    cfg = rs.reference_cfg(width=W * 4, height=H * 4)
    from model.head.detector_infer import make_post_processor
    pp = make_post_processor(cfg)
    out = {'n_images': np.int64(4), 'P2_0': np.array(syn.KITTI_P2, np.float64), 'P2_1': np.array(P2_OTHER, np.float64)}
    for b in range(4):
        reg, centers, reg_mask, cls_ids, locations = make_image(100 + b)
        P = syn.KITTI_P2 if b % 2 == 0 else P2_OTHER
        with torch.no_grad():
            errs = pp.evaluate_3D_depths(ref_targets(P, centers, reg_mask, cls_ids, locations),
                                         torch.from_numpy(reg)[None].clone())
        assert list(errs) == list(KEYS), list(errs)
        for k in KEYS:
            out['%s_b%d' % (k, b)] = errs[k].numpy().astype(np.float32)
        out['reg_b%d' % b], out['centers_b%d' % b], out['reg_mask_b%d' % b] = reg, centers, reg_mask
        out['cls_ids_b%d' % b], out['locations_b%d' % b] = cls_ids, locations
        d = np.stack([errs[k].numpy() for k in ('direct', 'keypoint_center', 'keypoint_02', 'keypoint_13')], 1)
        print("image %d: %d objects, depth errors %.3f..%.3f" % (b, len(errs['target']), d.min(), d.max()))
    reg, centers, reg_mask, cls_ids, locations = make_image(200)
    try:
        with torch.no_grad():
            pp.evaluate_3D_depths(ref_targets(syn.KITTI_P2, centers, np.zeros_like(reg_mask), cls_ids, locations),
                                  torch.from_numpy(reg)[None])
    except (RuntimeError, ValueError) as e:            # torch.cat([]): ValueError in recent torch, RuntimeError before
        print("an image without valid objects raises in the reference: %s" % str(e).splitlines()[0])
    else:
        raise AssertionError("the reference was expected to raise on an image without valid objects")
    np.savez_compressed(os.path.join(OUT, "eval_depths.npz"), **out)
    print("eval_depths.npz", os.path.getsize(os.path.join(OUT, "eval_depths.npz")))


if __name__ == "__main__":
    main()
