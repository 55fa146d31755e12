"""Every OUTPUT_DEPTH estimator of the PostProcessor (detector_infer.py:148-278), oracle included.

CPU: the depth oracle (oracle/depth_oracle.py) against the unmodified reference's results (oracle/make_golden_depth.py ->
tests/golden/decode_depth.npz) and the configuration errors of the product module. GPU (-m gpu): the decode kernel per
method against the same fixture, and the product path the way engine/inference.py's inference_all_depths drives it."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from oracle import depth_oracle as do
from oracle import monoflex_oracle as mo
from oracle.make_golden_depth import METHODS, depth_inputs

THRS = (0.0, 0.2)


def load():
    with np.load(os.path.join(GOLDEN, "decode_depth.npz")) as z:
        return {k: torch.from_numpy(z[k]) for k in z.files}


def gt_table(g):
    """[2, 40, 7] (valid, class, x1, y1, x2, y2, z) from the fixture's label fields"""
    return torch.stack([torch.cat([g['gt_reg_mask_b%d' % b].float().view(-1, 1), g['gt_cls_ids_b%d' % b].float().view(-1, 1),
                                   g['gt_bboxes_b%d' % b], g['gt_locations_b%d' % b][:, 2:]], 1) for b in range(2)])


def assert_columns(got, ref, tol):
    """each of the 14 result columns relative to its largest reference magnitude; the class column exactly"""
    assert got.shape == ref.shape
    if ref.shape[0] == 0:
        return
    assert torch.equal(got[:, 0], ref[:, 0])
    for c in range(1, 14):
        d = (got[:, c].double() - ref[:, c].double()).abs()
        if c in (1, 12):
            d = torch.minimum(d, (d - 2 * np.pi).abs())
        assert d.max().item() <= tol * max(ref[:, c].abs().max().item(), 1e-6), (c, d.max().item())


def assert_close(got, ref, tol):
    assert got.shape == ref.shape
    if ref.numel():
        assert (got.double() - ref.double()).abs().max().item() <= tol * max(ref.abs().max().item(), 1.0)


def post_processor():
    from monoflex_b200.model.head.detector_infer import make_post_processor
    return make_post_processor(default_cfg(width=320, height=96))


# ------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("method", METHODS)
def test_oracle_matches_reference_for_every_method(method):
    g = load()
    heat, reg, tg = depth_inputs()
    for thr in THRS:
        res, _ = do.post_process({'cls': heat, 'reg': reg}, tg['calib_P'], tg['pad_size'], tg['size'], thr,
                                 output_depth=method, gts=gt_table(g))
        for b in range(2):
            assert_columns(res[b], g['result_%s_b%d_thr%s' % (method, b, thr)], 1e-6)


def test_fixture_exercises_every_oracle_branch():
    """the fixture's ground truth makes the oracle reject some matches and pick each of the four estimators"""
    g = load()
    picked = set()
    for b in range(2):
        for thr in THRS:
            tag = '_b%d_thr%s' % (b, thr)
            z = {m: g['result_%s%s' % (m, tag)][:, 11] for m in ('oracle', 'mean', 'direct', 'keypoints_center',
                                                                 'keypoints_02', 'keypoints_13')}
            assert (z['oracle'] == z['mean']).any() and (z['oracle'] != z['mean']).any()
            for i, m in enumerate(('direct', 'keypoints_center', 'keypoints_02', 'keypoints_13')):
                if ((z['oracle'] == z[m]) & (z['oracle'] != z['mean'])).any():
                    picked.add(i)
    assert picked == {0, 1, 2, 3}


def test_soft_matches_the_monoflex_oracle_decode_bit_for_bit():
    heat, reg, tg = depth_inputs()
    scores, inds, clses, ys, xs = mo.select_topk(mo.nms_hm(heat), 50)
    pois = mo.gather_pois(reg, inds)
    for b in range(2):
        args = (scores[b], clses[b], xs[b], ys[b], pois[b], mo.calib_from_P(tg['calib_P'][b]), tg['pad_size'][b],
                tg['size'][b], 0.0)
        assert torch.equal(do.decode_image(*args, output_depth='soft'), mo.decode_image(*args))


@pytest.mark.parametrize("name", ["keypoints_mean", "median", "SOFT", None])
def test_invalid_depth_names_raise_value_error(name):
    from monoflex_b200.model.layers.utils import decode_detections
    pp = post_processor()
    pp.output_depth = name
    with pytest.raises(ValueError):
        pp.check_config()
    with pytest.raises(ValueError):
        decode_detections(torch.zeros(1, 3, 8, 8), torch.zeros(1, 50, 8, 8), None, None, None, None, 5, 0.0,
                          depth_mode=name)
    heat, reg, tg = depth_inputs()
    with pytest.raises(ValueError):
        do.post_process({'cls': heat, 'reg': reg}, tg['calib_P'], tg['pad_size'], tg['size'], 0.0, output_depth=name)


def test_oracle_without_labels_raises_runtime_error():
    pp = post_processor()
    pp.output_depth = 'oracle'
    targets = syn.make_param_lists(syn.make_targets(1, 80, 24))          # what a TEST_SPLIT='test' loader hands over
    with pytest.raises(RuntimeError, match="reg_mask, cls_ids, gt_bboxes, locations"):
        pp.prepare_targets(targets, True, torch.device("cpu"))
    pp.output_depth = 'soft'
    assert len(pp.prepare_targets(targets, True, torch.device("cpu"))) == 3


def test_oracle_table_from_label_fields():
    g = load()
    pp = post_processor()
    pp.output_depth = 'oracle'
    tg = syn.make_targets(2, 80, 24)
    targets = syn.make_param_lists(tg)
    for b, t in enumerate(targets):
        t.add_field('reg_mask', g['gt_reg_mask_b%d' % b])
        t.add_field('cls_ids', g['gt_cls_ids_b%d' % b])
        t.add_field('gt_bboxes', g['gt_bboxes_b%d' % b])
        t.add_field('locations', g['gt_locations_b%d' % b])
    meta = pp.prepare_targets(targets, True, torch.device("cpu"))
    assert torch.equal(meta[3], gt_table(g))


# ------------------------------------------------------------------------------------------------------------- GPU
def kernel_inputs():
    heat, reg, tg = depth_inputs()
    calib = torch.tensor([[c for c in mo.calib_from_P(P).values()] for P in tg['calib_P']], dtype=torch.float32).cuda()
    size = torch.tensor(tg['size'], dtype=torch.float32).cuda()
    return heat.cuda(), reg.cuda(), calib, tg['pad_size'].cuda(), size, torch.tensor(mo.DIM_MEAN).cuda(), tg


@pytest.mark.gpu
@pytest.mark.parametrize("method", METHODS)
def test_kernel_matches_reference_for_every_method(method):
    from test_gpu_ops import assert_decode_columns
    from monoflex_b200.model.layers.utils import decode_detections
    g = load()
    heat, reg, calib, pad, size, dim_mean, _ = kernel_inputs()
    gt = gt_table(g).cuda() if method == 'oracle' else None
    for thr in THRS:
        ws = decode_detections(heat, reg, calib, pad, size, dim_mean, 50, thr, depth_mode=method, gt=gt)
        torch.cuda.synchronize()
        for b in range(2):
            tag = '%s_b%d_thr%s' % (method, b, thr)
            ref = g['result_' + tag]
            n = int(ws.count[b])
            assert n == ref.shape[0]
            assert_decode_columns(ws.result[b, :n].cpu(), ref)
            assert_close(ws.depth_err[b, :n].cpu(), g['depth_err_' + tag], 1e-5)
            assert_close(ws.proj[b, :n].cpu(), g['proj_' + tag], 1e-5)
        if method == 'soft':
            result = ws.result.clone()
            plain = decode_detections(heat, reg, calib, pad, size, dim_mean, 50, thr)
            assert torch.equal(plain.result, result)


@pytest.mark.gpu
def test_kernel_oracle_matches_each_image_against_its_own_ground_truth():
    """B = 2 with the two images' ground truth swapped: each image follows the table it is given"""
    from test_gpu_ops import assert_decode_columns
    from monoflex_b200.model.layers.utils import decode_detections
    g = load()
    heat, reg, calib, pad, size, dim_mean, tg = kernel_inputs()
    swapped = gt_table(g).flip(0).contiguous()
    ws = decode_detections(heat, reg, calib, pad, size, dim_mean, 50, 0.0, depth_mode='oracle', gt=swapped.cuda())
    torch.cuda.synchronize()
    res, _ = do.post_process({'cls': heat.cpu(), 'reg': reg.cpu()}, tg['calib_P'], tg['pad_size'], tg['size'], 0.0,
                             output_depth='oracle', gts=swapped)
    differs = False
    for b in range(2):
        got = ws.result[b, :int(ws.count[b])].cpu()
        assert_decode_columns(got, res[b])
        differs |= not torch.equal(got[:, 11], g['result_oracle_b%d_thr0.0' % b][:, 11])
    assert differs
    # no valid ground truth at all: the mean of the four estimators
    empty = torch.zeros(2, 40, 7, device="cuda")
    ws = decode_detections(heat, reg, calib, pad, size, dim_mean, 50, 0.0, depth_mode='oracle', gt=empty)
    torch.cuda.synchronize()
    for b in range(2):
        assert_decode_columns(ws.result[b, :int(ws.count[b])].cpu(), g['result_mean_b%d_thr0.0' % b])


VIS_KEYS = ('heat_map', 'keypoints', 'proj_center')          # engine/visualize_infer.py:93-100


@pytest.mark.gpu
def test_inference_all_depths_on_the_product_path():
    """engine/inference.py:130-197: set post_processor.output_depth to each method and run model(images, targets)"""
    from test_gpu_ops import assert_decode_columns
    from monoflex_b200.model.detector import KeypointDetector
    H, W = 128, 256
    m = KeypointDetector(default_cfg(width=W, height=H))
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval()
    post = m.heads.post_processor
    post.det_threshold = 0.0
    x = syn.make_images(1, H, W).cuda()
    tg = syn.make_targets(1, W // 4, H // 4)
    with torch.no_grad():
        base, _, _ = m(x, [t.to("cuda") for t in syn.make_param_lists(tg)])
    base = base.cpu()
    # ground truth: exact copies of five detections' boxes (IoU 1) at depths 10, 17, ..., the other slots invalid
    gt = torch.zeros(1, 40, 7)
    for k in range(5):
        gt[0, 3 * k] = torch.tensor([1.0, base[k, 0], *base[k, 2:6].tolist(), 10.0 + 7 * k])
    targets = syn.make_param_lists(tg)
    targets[0].add_field('reg_mask', (gt[0, :, 0] != 0).to(torch.uint8))
    targets[0].add_field('cls_ids', gt[0, :, 1].long())
    targets[0].add_field('gt_bboxes', gt[0, :, 2:6].clone())
    locs = torch.zeros(40, 3)
    locs[:, 2] = gt[0, :, 6]
    targets[0].add_field('locations', locs)
    targets = [t.to("cuda") for t in targets]
    first = {}
    with torch.no_grad():
        for method in METHODS + ('soft',):
            post.output_depth = method
            result, eval_utils, vis = m(x, targets)
            plan = m.heads.predictor.last_plan
            res_o, _ = do.post_process({'cls': plan.cls.cpu(), 'reg': plan.reg.cpu()}, tg['calib_P'], tg['pad_size'],
                                       tg['size'], 0.0, output_depth=method, gts=gt)
            assert_decode_columns(result.cpu(), res_o[0])
            if method in first:
                assert torch.equal(result.cpu(), first[method])
            first[method] = result.cpu()
            n = result.shape[0]
            for k in VIS_KEYS:
                assert vis[k].shape[0] in (1, n)
            assert vis['proj_center'].shape == (n, 2) and eval_utils['estimated_depth_error'].shape == (n,)
            assert vis['depth_uncertainty'].shape == (1, H // 4, W // 4)
            assert ('min_uncertainty' in vis) == (method in ('soft', 'hard', 'mean', 'oracle'))
        post.output_depth = 'oracle'
        ref, eu, _ = m(x, targets)
        got, counts = m.forward_async(x, targets).result()
    assert counts == eu['counts'] and torch.equal(got, ref.cpu())
    assert not torch.equal(first['oracle'][:, 11], first['mean'][:, 11])     # some detections took a GT-matched estimator
