"""TEST.EVAL_DEPTH (--eval_depth) on the GPU: mf_eval_depth_errors against the unmodified reference's evaluate_3D_depths
(tests/golden/eval_depths.npz) and against the numpy oracle at B = 1, 2 and 8, NaN rows for centres outside the map,
and the PostProcessor / KeypointDetector paths: graph replay, eager, forward_async and forward_depths give the same
dict, and with EVAL_DEPTH off nothing changes."""
import os

import numpy as np
import pytest
import torch

from monoflex_b200 import _lib
from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.inference import EVAL_DEPTH_METHODS
from monoflex_b200.model.layers.utils import EVAL_DEPTH_KEYS, depth_error_dict, eval_depth_errors
from monoflex_b200.structures import Calibration
from oracle.eval_depth_oracle import eval_depths
from oracle.make_golden_eval_depths import P2_OTHER, make_image
from oracle.monoflex_oracle import DIM_MEAN, calib_from_P

pytestmark = pytest.mark.gpu
DIM = torch.tensor(DIM_MEAN, dtype=torch.float32)


def assert_keys_close(got, ref, tol=1e-5):
    """row count, row order and `target` exact; every other key within tol * max(|key|, |target|) of the reference"""
    got = {k: v.cpu().numpy() if torch.is_tensor(v) else v for k, v in got.items()}
    assert list(got) == list(EVAL_DEPTH_KEYS)
    assert np.array_equal(got['target'], ref['target'])
    scale = max(np.abs(ref['target']).max(initial=0.0), 1e-6)
    for k in EVAL_DEPTH_KEYS:
        assert got[k].shape == ref[k].shape and got[k].dtype == np.float32, k
        d = np.abs(got[k].astype(np.float64) - ref[k].astype(np.float64))
        assert d.max(initial=0.0) <= tol * max(np.abs(ref[k]).max(initial=0.0), scale), (k, d.max())


def table_of(centers, reg_mask, cls_ids, locations):
    """[B, M, 5] (reg_mask, cls_id, x, y, z) from [B, M, ...] numpy label fields"""
    t = np.concatenate([reg_mask[..., None], cls_ids[..., None], centers, locations[..., 2:]], -1)
    return torch.from_numpy(t.astype(np.float32)).cuda().contiguous()


def run_kernel(reg, P2s, centers, reg_mask, cls_ids, locations):
    calib = torch.tensor([list(calib_from_P(p).values()) for p in P2s], dtype=torch.float32).cuda()
    out, counts = eval_depth_errors(torch.from_numpy(reg).cuda(), calib, DIM.cuda(),
                                    table_of(centers, reg_mask, cls_ids, locations))
    counts = counts.tolist()
    return depth_error_dict(out, counts), counts


def test_fixture_at_batch_1(golden_dir):
    from monoflex_b200.model.head.detector_infer import make_post_processor
    g = np.load(os.path.join(golden_dir, "eval_depths.npz"))
    post = make_post_processor(default_cfg(width=192, height=64)).cuda()
    for b in range(int(g['n_images'])):
        f = {k: g['%s_b%d' % (k, b)][None] for k in ('reg', 'centers', 'reg_mask', 'cls_ids', 'locations')}
        ref = {k: g['%s_b%d' % (k, b)] for k in EVAL_DEPTH_KEYS}
        P = g['P2_%d' % (b % 2)]
        got, counts = run_kernel(f['reg'], [P], f['centers'], f['reg_mask'], f['cls_ids'], f['locations'])
        assert counts == [len(ref['target'])]
        assert_keys_close(got, ref)
        # the reference's signature: the dict of prepare_targets(test=False), calibrations as objects
        targets = {'calib': [Calibration(P)], 'target_centers': torch.from_numpy(f['centers']),
                   'reg_mask': torch.from_numpy(f['reg_mask']), 'cls_ids': torch.from_numpy(f['cls_ids']),
                   'locations': torch.from_numpy(f['locations'])}
        via_post = post.evaluate_3D_depths(targets, torch.from_numpy(f['reg']).cuda())
        assert list(via_post) == list(EVAL_DEPTH_KEYS)
        for k in EVAL_DEPTH_KEYS:
            assert via_post[k].is_cuda and via_post[k].dim() == 1 and torch.equal(via_post[k], got[k]), k


def batch(B, empty=None):
    """B seeded images, a different P2 each; image `empty` has no valid object"""
    imgs = [make_image(300 + b) for b in range(B)]
    reg, centers, reg_mask, cls_ids, locations = (np.stack(x) for x in zip(*imgs))
    if empty is not None:
        reg_mask[empty] = 0
    P2s = [np.array(syn.KITTI_P2 if b % 2 == 0 else P2_OTHER) * np.array([[1 + 0.03 * b], [1 + 0.03 * b], [1]])
           for b in range(B)]
    return reg, P2s, centers, reg_mask, cls_ids, locations


@pytest.mark.parametrize("B", [1, 2, 8])
def test_oracle_at_several_batch_sizes(B):
    empty = None if B == 1 else B // 2
    reg, P2s, centers, reg_mask, cls_ids, locations = batch(B, empty)
    got, counts = run_kernel(reg, P2s, centers, reg_mask, cls_ids, locations)
    ref, ref_counts = eval_depths(reg, [np.float32(P[0, 0]) for P in P2s], np.asarray(DIM_MEAN, np.float32), centers,
                                  reg_mask, cls_ids, locations)
    assert counts == ref_counts
    assert_keys_close(got, ref)
    if empty is not None:
        assert counts[empty] == 0
        # every other image's rows equal its own batch-1 run, bit for bit
        start = 0
        for b in range(B):
            one, n = run_kernel(reg[b:b + 1], P2s[b:b + 1], centers[b:b + 1], reg_mask[b:b + 1], cls_ids[b:b + 1],
                                locations[b:b + 1])
            assert n == [counts[b]]
            for k in EVAL_DEPTH_KEYS:
                assert torch.equal(got[k][start:start + counts[b]], one[k]), (b, k)
            start += counts[b]
        # a batch whose only image has no valid object: every key empty
        none, n = run_kernel(reg[empty:empty + 1], P2s[:1], centers[:1], reg_mask[empty:empty + 1], cls_ids[:1],
                             locations[:1])
        assert n == [0] and all(v.shape == (0,) for v in none.values())


def test_out_of_map_centre_gives_nan_and_changes_no_other_row():
    reg, P2s, centers, reg_mask, cls_ids, locations = batch(2)
    H, W = reg.shape[2:]
    base, counts = run_kernel(reg, P2s, centers, reg_mask, cls_ids, locations)
    moved = centers.copy()
    cls2 = cls_ids.copy()
    slots = [(0, s) for s in np.nonzero(reg_mask[0])[0][[1, 4, 7, 10]]] + [(1, s) for s in np.nonzero(reg_mask[1])[0][[2, 5]]]
    outside = [(W, 0), (-1, 3), (5, H), (2, -1), (W - 1, H)]
    for (b, s), c in zip(slots, outside):
        moved[b, s] = c
    cls2[slots[-1]] = 3                                        # a class outside dim_mean
    got, n = run_kernel(reg, P2s, moved, reg_mask, cls2, locations)
    assert n == counts
    rows = [int(reg_mask[:b].sum() + reg_mask[b, :s].sum()) for b, s in slots]
    keep = np.setdiff1d(np.arange(sum(counts)), rows)
    for k in EVAL_DEPTH_KEYS:
        assert torch.isnan(got[k][rows]).all(), k
        assert torch.equal(got[k][keep], base[k][keep]), k


# ------------------------------------------------------------------------------------------------------------- model
H, W = 128, 256


def make_model(precision, eval_depth=True):
    from monoflex_b200.model.detector import KeypointDetector
    cfg = default_cfg(width=W, height=H)
    cfg.TEST.EVAL_DEPTH = eval_depth
    m = KeypointDetector(cfg)
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval().set_precision(precision)
    m.heads.post_processor.det_threshold = 0.0
    return m


def labelled_targets(B, n_valid, seed):
    """inference param lists with the label fields evaluate_3D_depths reads; image b has n_valid[b] valid slots"""
    rng = np.random.Generator(np.random.PCG64(seed))
    tg = syn.make_targets(B, W // 4, H // 4)
    tg['calib_P'] = [np.array(syn.KITTI_P2) * np.array([[1 + 0.05 * b], [1 + 0.05 * b], [1]]) for b in range(B)]
    targets = syn.make_param_lists(tg)
    for b, t in enumerate(targets):
        mask = np.zeros(40, np.uint8)
        mask[rng.permutation(40)[:n_valid[b]]] = 1
        t.add_field('reg_mask', torch.from_numpy(mask))
        t.add_field('cls_ids', torch.from_numpy(rng.integers(0, 3, 40).astype(np.int32)))
        t.add_field('target_centers', torch.from_numpy(np.stack([rng.integers(0, W // 4, 40),
                                                                 rng.integers(0, H // 4, 40)], 1).astype(np.int32)))
        t.add_field('locations', torch.from_numpy(rng.uniform(2, 60, (40, 3)).astype(np.float32)))
        xy = rng.uniform(0, (W - 40, H - 40), (40, 2))                     # for forward_depths' oracle estimator
        t.add_field('gt_bboxes', torch.from_numpy(np.concatenate([xy, xy + 30], 1).astype(np.float32)))
    return [t.to("cuda") for t in targets]


def assert_same_dict(a, b):
    assert list(a) == list(b) == list(EVAL_DEPTH_KEYS)
    for k in EVAL_DEPTH_KEYS:
        assert a[k].is_cuda and a[k].dtype == torch.float32 and a[k].dim() == 1
        assert torch.equal(a[k], b[k]), k


def expected(m, x, targets):
    """the kernel on the eager forward's own regression map, through evaluate_3D_depths' reference signature"""
    pred = m.heads.predictor(m.backbone(x), targets)
    f = {k: torch.stack([t.get_field(k) for t in targets]) for k in ('target_centers', 'reg_mask', 'cls_ids', 'locations')}
    f['calib'] = [t.get_field('calib') for t in targets]
    return m.heads.post_processor.evaluate_3D_depths(f, pred['reg'])


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_graph_replays_with_changing_objects_equal_the_eager_forward(precision):
    m = make_model(precision)
    B = 2
    x = syn.make_images(B, H, W).cuda()
    first, second = labelled_targets(B, (12, 5), 1), labelled_targets(B, (0, 17), 2)
    with torch.no_grad():
        m.use_cuda_graph = False
        eager = [m(x, t) for t in (first, second)]
        ref = [expected(m, x, t) for t in (first, second)]
        m.use_cuda_graph = True
        for _ in range(2):                                 # capture + replay, then two replays
            graph = [m(x, t) for t in (first, second)]
            for (r, eu, _), (r0, eu0, _), want, n in zip(graph, eager, ref, ((12, 5), (0, 17))):
                assert torch.equal(r, r0)
                assert eu['depth_error_counts'] == eu0['depth_error_counts'] == list(n)
                assert_same_dict(eu['depth_errors'], eu0['depth_errors'])
                assert_same_dict(eu['depth_errors'], want)
                assert not torch.isnan(eu['depth_errors']['mean']).any()


def test_every_path_gives_the_same_dict():
    m = make_model("strict")
    B = 2
    x = syn.make_images(B, H, W).cuda()
    targets = labelled_targets(B, (9, 14), 3)
    with torch.no_grad():
        _, eu, _ = m(x, targets)
        handle = m.forward_async(x, targets)
        assert handle.eval_utils['depth_errors'] is None
        rows, counts = handle.result()
        assert counts == eu['counts']
        assert_same_dict(handle.eval_utils['depth_errors'], eu['depth_errors'])
        assert handle.eval_utils['depth_error_counts'] == eu['depth_error_counts'] == [9, 14]
        for graph in (True, False):
            m.use_cuda_graph = graph
            got = m.forward_depths(x, targets, EVAL_DEPTH_METHODS)
            shared = got[EVAL_DEPTH_METHODS[0]][1]['depth_errors']
            for method in EVAL_DEPTH_METHODS:
                assert got[method][1]['depth_errors'] is shared       # computed once per call
                assert got[method][1]['depth_error_counts'] == [9, 14]
            assert_same_dict(shared, eu['depth_errors'])
        m.use_cuda_graph = False
        _, eu_eager, _ = m(x, targets)
        assert_same_dict(eu_eager['depth_errors'], eu['depth_errors'])


def recorded_calls(monkeypatch):
    """names of the C entry points called, in order"""
    names = []
    call = _lib.call

    def recording(name, *args):
        names.append(name)
        return call(name, *args)
    import monoflex_b200.model.layers.utils as lu
    monkeypatch.setattr(lu, "call", recording)
    return names


@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_eval_depth_off_changes_nothing(precision, monkeypatch):
    B = 2
    x = syn.make_images(B, H, W).cuda()
    targets = labelled_targets(B, (9, 14), 4)
    names = recorded_calls(monkeypatch)
    out, launches = {}, {}
    for on in (False, True):
        m = make_model(precision, eval_depth=on)
        with torch.no_grad():
            del names[:]
            r, eu, _ = m(x, targets)                          # capture: eager warm-up, then the captured body
            launches[on] = list(names)
            out[on] = (r, eu, m(x, targets))
    assert launches[False] == ["mf_decode_detections"] * 2
    assert launches[True] == ["mf_decode_detections", "mf_eval_depth_errors"] * 2
    (r0, eu0, again0), (r1, eu1, again1) = out[False], out[True]
    assert torch.equal(r0, r1) and torch.equal(again0[0], again1[0]) and torch.equal(r0, again0[0])
    assert eu0['depth_errors'] is None and 'depth_error_counts' not in eu0
    assert set(eu1) - set(eu0) == {'depth_error_counts'}
    for k in ('uncertainty_conf', 'estimated_depth_error', 'vis_scores', 'padded_result'):
        assert torch.equal(eu0[k], eu1[k]), k
