"""TEST.EVAL_DEPTH (--eval_depth) without a GPU: the numpy oracle (oracle/eval_depth_oracle.py) against the unmodified
reference's evaluate_3D_depths (tests/golden/eval_depths.npz), the C ABI's argument checks, and the configurations the
PostProcessor refuses before any launch."""
import os

import numpy as np
import pytest
import torch

from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.model.head.detector_infer import EVAL_DEPTH_FIELDS, make_post_processor
from oracle.eval_depth_oracle import KEYS, eval_depths
from oracle.monoflex_oracle import DIM_MEAN


def load_fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "eval_depths.npz"))


def assert_keys_close(got, ref, tol=1e-5):
    """row count, row order and `target` exact; every other key within tol * max(|key|, |target|) of the reference"""
    assert list(got) == list(KEYS)
    assert np.array_equal(got['target'], ref['target'])
    scale = max(np.abs(ref['target']).max(initial=0.0), 1e-6)
    for k in KEYS:
        assert got[k].shape == ref[k].shape, k
        d = np.abs(got[k].astype(np.float64) - ref[k].astype(np.float64))
        assert d.max(initial=0.0) <= tol * max(np.abs(ref[k]).max(initial=0.0), scale), (k, d.max())


def test_oracle_reproduces_the_reference_key_by_key(golden_dir):
    g = load_fixture(golden_dir)
    for b in range(int(g['n_images'])):
        P = g['P2_%d' % (b % 2)]
        got, counts = eval_depths(g['reg_b%d' % b][None], [np.float32(P[0, 0])], np.asarray(DIM_MEAN, np.float32),
                                  g['centers_b%d' % b][None], g['reg_mask_b%d' % b][None], g['cls_ids_b%d' % b][None],
                                  g['locations_b%d' % b][None])
        ref = {k: g['%s_b%d' % (k, b)] for k in KEYS}
        assert counts == [len(ref['target'])] == [int(g['reg_mask_b%d' % b].sum())]
        assert_keys_close(got, ref)


def test_fixture_covers_the_edge_cases(golden_dir):
    """every border, every class, clamped depths at both ends of DEPTH_RANGE, and uncertainty ties"""
    g = load_fixture(golden_dir)
    H, W = g['reg_b0'].shape[1:]
    for b in range(int(g['n_images'])):
        valid = g['reg_mask_b%d' % b] != 0
        c = g['centers_b%d' % b][valid]
        assert {0, W - 1} <= set(c[:, 0].tolist()) and {0, H - 1} <= set(c[:, 1].tolist())
        assert set(g['cls_ids_b%d' % b][valid].tolist()) == {0, 1, 2}
        assert (~valid[:valid.nonzero()[0][-1]]).any()                           # invalid slots between valid ones
        for k in ('keypoint_center', 'keypoint_02', 'keypoint_13'):                  # heights <= 0 clamp at 100
            assert np.isclose(depths(g, k, b), 100, atol=1e-4).any(), (b, k)
        sig = np.stack([g['%s_b%d' % (k, b)] for k in ('direct_sigma', 'keypoint_center_sigma', 'keypoint_02_sigma',
                                                        'keypoint_13_sigma')], 1)
        assert (sig[:, :, None] == sig[:, None, :]).sum((1, 2)).max() > 4                     # exact ties
    direct = np.concatenate([depths(g, 'direct', b) for b in range(int(g['n_images']))])
    assert np.isclose(direct, 0.1, atol=1e-6).any() and np.isclose(direct, 100, atol=1e-4).any()


def depths(g, key, b):
    """the two depths z -+ error that agree with the fixture's error of `key`; one of them is the estimator's depth"""
    err, z = g['%s_b%d' % (key, b)], g['target_b%d' % b]
    return np.stack([z - err, z + err], 1)


def test_c_abi_refuses_malformed_arguments_before_any_launch():
    from monoflex_b200 import _lib
    lib = _lib.load()
    P = 16                                     # never dereferenced: the arguments are refused first
    ok = dict(reg=P, calib=P, dim_mean=P, gt=P, B=1, M=40, C=3, H=16, W=48, R=50, out=P, counts=P)
    cases = [(dict(R=49), "R=49"), (dict(B=0), "B=0"), (dict(M=0), "M=0"), (dict(H=0), "H=0"), (dict(C=0), "C=0"),
             (dict(reg=None), "null pointer"), (dict(gt=None), "null pointer"), (dict(out=None), "null pointer"),
             (dict(counts=None), "null pointer"), (dict(calib=None), "null pointer"), (dict(dim_mean=None), "null")]
    for change, message in cases:
        a = dict(ok, **change)
        rc = lib.mf_eval_depth_errors(a['reg'], a['calib'], a['dim_mean'], a['gt'], a['B'], a['M'], a['C'], a['H'],
                                      a['W'], a['R'], a['out'], a['counts'], None)
        assert rc == -1, change
        assert message in lib.mf_last_error().decode(), (change, lib.mf_last_error().decode())


def post_processor(**test):
    cfg = default_cfg(width=256, height=128, device="cpu")
    for k, v in test.items():
        setattr(cfg.TEST, k, v)
    return make_post_processor(cfg)


def test_eval_dis_ious_still_raises_not_implemented():
    post = post_processor(EVAL_DIS_IOUS=True)
    with pytest.raises(NotImplementedError, match="eval_iou"):
        post.check_config()
    with pytest.raises(NotImplementedError):
        post.forward({'cls': torch.zeros(1, 3, 32, 64), 'reg': torch.zeros(1, 50, 32, 64)}, [])
    assert post_processor(EVAL_DEPTH=True).check_config() == ('soft',)


def test_test_split_without_labels_raises_runtime_error_naming_the_fields():
    post = post_processor(EVAL_DEPTH=True)
    targets = syn.make_param_lists(syn.make_targets(2, 64, 32))          # what a TEST_SPLIT='test' loader attaches
    with pytest.raises(RuntimeError, match=", ".join(EVAL_DEPTH_FIELDS)):
        post.prepare_targets(targets, True, torch.device("cpu"))
    for t in targets:
        t.add_field('reg_mask', torch.ones(40, dtype=torch.uint8))
    with pytest.raises(RuntimeError, match="target_centers, cls_ids, locations"):
        post.prepare_targets(targets, True, torch.device("cpu"))
    assert len(post_processor().prepare_targets(targets, True, torch.device("cpu"))) == 3   # EVAL_DEPTH off: untouched


def test_depth_table_from_label_fields():
    post = post_processor(EVAL_DEPTH=True)
    targets = syn.make_train_param_lists(syn.make_train_targets(2))         # image 1 has no object
    meta = post.prepare_targets(targets, False, torch.device("cpu"))
    table = meta[-1]
    assert len(meta) == 4 and table.shape == (2, 40, 5) and table.dtype == torch.float32
    for b, t in enumerate(targets):
        assert torch.equal(table[b, :, 0], t.get_field('reg_mask').float())
        assert torch.equal(table[b, :, 1], t.get_field('cls_ids').float())
        assert torch.equal(table[b, :, 2:4], t.get_field('target_centers').float())
        assert torch.equal(table[b, :, 4], t.get_field('locations')[:, 2])
    assert table[0, :, 0].sum() > 0 and table[1, :, 0].sum() == 0
