"""Every depth estimator from one decode (mf_decode_detections_depths, PostProcessor / KeypointDetector.forward_depths)
and the one-pass inference_all_depths (monoflex_b200/inference.py).

CPU: the C ABI refuses bad mode lists before any CUDA call. GPU (-m gpu): each mode's block of the multi-mode decode
equals the single-mode decode bit for bit; forward_depths equals the eight passes of engine/inference.py's
inference_all_depths with one backbone + predictor run; the drop-in writes the same files, computes the same ret_dicts
and logs the same lines as the eight-pass loop."""
import ctypes
import logging
import os
import types

import numpy as np
import pytest
import torch

from monoflex_b200 import evaluation as E
from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.inference import EVAL_DEPTH_METHODS, inference_all_depths
from monoflex_b200.model.layers.utils import DEPTH_MODES
from oracle.make_golden_depth import depth_inputs

SUBSETS = (DEPTH_MODES, EVAL_DEPTH_METHODS, ('oracle',), tuple(reversed(DEPTH_MODES)))
SHARED = ('scores', 'inds', 'clses', 'ys', 'xs', 'pois', 'proj', 'count')
PER_MODE = ('result', 'depth_err', 'min_unc')


# ------------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("modes,n,message", [((0, 0), 2, "listed twice"), ((2, 9), 2, "9 is not one of"),
                                             ((-1,), 1, "-1 is not one of"), ((1, 3), 2, "oracle depth needs"),
                                             ((0,), 0, "0 depth modes"), (tuple(range(9)) + (0,), 10, "10 depth modes")])
def test_c_abi_refuses_bad_mode_lists_before_any_launch(modes, n, message):
    from monoflex_b200 import _lib
    lib = _lib.load()
    P = 16                                     # never dereferenced: the list is refused first
    arr = (ctypes.c_int * len(modes))(*modes)
    assert lib.mf_decode_detections_depths(P, P, P, P, P, P, 1, 3, 24, 80, 50, 50, 0.0, 0, arr, n, None, 0,
                                           *([P] * 14), None) == -1
    assert message in lib.mf_last_error().decode()


@pytest.mark.parametrize("modes", [('soft', 'soft'), ('mean', 'median'), (), ('soft', None)])
def test_python_refuses_bad_mode_lists(modes):
    from monoflex_b200.model.layers.utils import decode_detections
    with pytest.raises(ValueError):
        decode_detections(torch.zeros(1, 3, 8, 8), torch.zeros(1, 50, 8, 8), None, None, None, None, 5, 0.0,
                          depth_mode=modes)


# ------------------------------------------------------------------------------------------------------------- kernel
def kernel_inputs(B):
    """depth_inputs' maps (key-point estimators spread over the depth range) tiled to B images with per-image noise"""
    from oracle import monoflex_oracle as mo
    heat, reg, tg = depth_inputs()
    g = torch.Generator().manual_seed(B)
    heat = heat.repeat((B + 1) // 2, 1, 1, 1)[:B]
    reg = reg.repeat((B + 1) // 2, 1, 1, 1)[:B] + 0.05 * torch.randn(B, *reg.shape[1:], generator=g)
    P = [syn.KITTI_P2] * B
    calib = torch.tensor([list(mo.calib_from_P(p).values()) for p in P], dtype=torch.float32)
    size = torch.tensor([tg['size'][0]] * B, dtype=torch.float32)
    pad = tg['pad_size'][:1].repeat(B, 1)
    return [t.cuda() for t in (heat.contiguous(), reg.contiguous(), calib, pad, size, torch.tensor(mo.DIM_MEAN))]


def oracle_gt(ws, B, empty):
    """[B, 40, 7]: copies of some detections' boxes at depths 8, 13, ... (a match for the oracle); image `empty` (the last
    one of a batch of several) has no valid object"""
    gt = torch.zeros(B, 40, 7)
    res = ws.result.cpu()
    for b in range(B):
        if b == empty:
            continue
        for k in range(0, 30, 3):
            gt[b, k] = torch.tensor([1.0, res[b, k, 0], *res[b, k, 2:6].tolist(), 8.0 + 5 * k])
    return gt.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3, 8])
@pytest.mark.parametrize("thr", [0.0, 0.2])
def test_each_mode_block_equals_the_single_mode_decode(B, thr):
    from monoflex_b200.model.layers.utils import decode_detections
    args = kernel_inputs(B)
    gt = oracle_gt(decode_detections(*args, 50, thr), B, empty=B - 1 if B > 1 else None)
    single = {}
    for mode in DEPTH_MODES:
        ws = decode_detections(*args, 50, thr, depth_mode=mode, gt=gt)
        single[mode] = {k: getattr(ws, k).clone() for k in SHARED + PER_MODE}
    assert not torch.equal(single['oracle']['result'], single['mean']['result'])       # some detections matched
    for subset in SUBSETS:
        ws = decode_detections(*args, 50, thr, depth_mode=subset, gt=gt if 'oracle' in subset else None)
        assert ws.result.shape == (len(subset), B, 50, 14) and ws.min_unc.shape == (len(subset), B, 50)
        for m, mode in enumerate(subset):
            for k in PER_MODE:
                assert torch.equal(getattr(ws, k)[m], single[mode][k]), (subset, mode, k)
            for k in SHARED:
                assert torch.equal(getattr(ws, k), single[mode][k]), (subset, mode, k)


@pytest.mark.gpu
def test_gpu_decode_refuses_bad_mode_lists():
    from monoflex_b200.model.layers.utils import decode_detections
    args = kernel_inputs(1)
    with pytest.raises(ValueError, match="distinct"):
        decode_detections(*args, 50, 0.2, depth_mode=('hard', 'soft', 'hard'))
    with pytest.raises(ValueError, match="oracle"):
        decode_detections(*args, 50, 0.2, depth_mode=('soft', 'oracle'))
    with pytest.raises(ValueError, match="not one of"):
        decode_detections(*args, 50, 0.2, depth_mode=('soft', 'keypoints_mean'))


# ------------------------------------------------------------------------------------------------------------- model
H, W = 128, 256


def make_model(precision):
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg(width=W, height=H))
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval().set_precision(precision)
    m.heads.post_processor.det_threshold = 0.0
    return m


def labelled_targets(tg, gt):
    """param lists with the label fields the oracle reads, from gt [B, 40, 7] (valid, class, x1, y1, x2, y2, z)"""
    targets = syn.make_param_lists(tg)
    for b, t in enumerate(targets):
        t.add_field('reg_mask', (gt[b, :, 0] != 0).to(torch.uint8))
        t.add_field('cls_ids', gt[b, :, 1].long())
        t.add_field('gt_bboxes', gt[b, :, 2:6].clone())
        locs = torch.zeros(40, 3)
        locs[:, 2] = gt[b, :, 6]
        t.add_field('locations', locs)
    return [t.to("cuda") for t in targets]


def assert_same_output(got, ref):
    (r, eu, vis), (r0, eu0, vis0) = got, ref
    assert torch.equal(r, r0)
    assert set(eu) == set(eu0) and list(vis) == list(vis0)
    for k in ('uncertainty_conf', 'estimated_depth_error', 'vis_scores', 'batch_idxs', 'padded_result'):
        assert torch.equal(eu[k], eu0[k]), k
    assert eu['counts'] == eu0['counts']
    for a, b in zip(eu['topk'], eu0['topk']):
        assert torch.equal(a, b)
    for k in vis0:
        assert torch.equal(vis[k], vis0[k]), k


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["strict", "fast"])
@pytest.mark.parametrize("graph", [True, False])
def test_forward_depths_equals_the_eight_pass_loop(precision, graph, monkeypatch):
    from monoflex_b200 import engine
    B = 2
    m = make_model(precision)
    m.use_cuda_graph = graph
    post = m.heads.post_processor
    x = syn.make_images(B, H, W).cuda()
    tg = syn.make_targets(B, W // 4, H // 4)
    with torch.no_grad():
        base, eu, _ = m(x, [t.to("cuda") for t in syn.make_param_lists(tg)])
    base, n0 = base.cpu(), eu['counts'][0]
    gt = torch.zeros(B, 40, 7)
    for k in range(5):                # image 0: exact copies of five detections' boxes; image 1: no valid object
        gt[0, 3 * k] = torch.tensor([1.0, base[k, 0], *base[k, 2:6].tolist(), 10.0 + 7 * k])
    assert n0 > 5
    targets = labelled_targets(tg, gt)
    runs = {'plan': 0, 'replay': 0}
    plan_run, replay = engine.Plan.run, torch.cuda.CUDAGraph.replay

    def counted(name, fn):
        def wrapper(self, *a, **k):
            runs[name] += 1
            return fn(self, *a, **k)
        return wrapper
    monkeypatch.setattr(engine.Plan, "run", counted('plan', plan_run))
    monkeypatch.setattr(torch.cuda.CUDAGraph, "replay", counted('replay', replay))
    with torch.no_grad():
        loop = {}
        for method in EVAL_DEPTH_METHODS:
            post.output_depth = method
            r, eu, vis = m(x, targets)
            loop[method] = (r, dict(eu, padded_result=eu['padded_result'].clone()), vis)   # the workspace is re-used
        post.output_depth = 'soft'
        m(x, targets)
        runs.update(plan=0, replay=0)
        m(x, targets)
        per_forward = dict(runs)      # eager: the backbone's and the predictor's plans; graph: one replay
        for call in range(3):         # the first graph call captures, the others replay; alternating with forward
            runs.update(plan=0, replay=0)
            got = m.forward_depths(x, targets, EVAL_DEPTH_METHODS)
            if graph:
                assert runs['replay'] == 1 and (runs['plan'] == 0 or call == 0)      # the first call captures
            else:
                assert runs == per_forward and runs['plan'] >= 2
            assert list(got) == list(EVAL_DEPTH_METHODS)
            for method in EVAL_DEPTH_METHODS:
                assert_same_output(got[method], loop[method])
            assert torch.equal(m(x, targets)[0], loop['soft'][0])
        sub = m.forward_depths(x, targets, ['keypoints_13', 'direct'])
    assert torch.equal(sub['direct'][0], loop['direct'][0]) and torch.equal(sub['keypoints_13'][0], loop['keypoints_13'][0])
    assert not torch.equal(got['oracle'][0][:, 11], got['mean'][0][:, 11])


@pytest.mark.gpu
def test_forward_depths_needs_labels_for_the_oracle_only():
    m = make_model("strict")
    x = syn.make_images(1, H, W).cuda()
    targets = [t.to("cuda") for t in syn.make_param_lists(syn.make_targets(1, W // 4, H // 4))]
    with torch.no_grad():
        with pytest.raises(RuntimeError, match="reg_mask, cls_ids, gt_bboxes, locations"):
            m.forward_depths(x, targets, EVAL_DEPTH_METHODS)
        out = m.forward_depths(x, targets, ('soft', 'hard'))
        with pytest.raises(ValueError):
            m.forward_depths(x, targets, ('soft', 'soft'))
    assert set(out) == {'soft', 'hard'}


# ------------------------------------------------------------------------------------------------------------- drop-in
class Loader(object):
    """the reference's test-loader batches: {"images": [B,3,H,W], "targets": [ParamsList], "img_ids": [str]}"""

    def __init__(self, dataset, images, targets, ids, batch_size):
        self.dataset, self.images, self.targets, self.ids, self.bs = dataset, images, targets, ids, batch_size

    def __iter__(self):
        for i in range(0, len(self.ids), self.bs):
            yield {"images": self.images[i:i + self.bs], "targets": self.targets[i:i + self.bs],
                   "img_ids": self.ids[i:i + self.bs]}


def kitti_set(root, m, n_img=5, H=384, W=1280):
    """A KITTI-layout directory (label_2, calib, ImageSets split in a shuffled order) and a loader over it. The labels are
    the make_golden_targets generator's objects plus copies of a few of the model's own detections, so that AP is not
    zero; the loader's targets carry them as the oracle's label fields."""
    from oracle import make_golden_targets as mg
    from monoflex_b200 import targets as T
    g = np.random.default_rng(7)
    for d in ("label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    ids = ["%06d" % i for i in g.permutation(40)[:n_img]]
    images = syn.make_images(n_img, H, W, seed=3)
    targets = []
    for b, img_id in enumerate(ids):
        P2 = mg.make_P2(g, W, H)
        with open(os.path.join(root, "calib", img_id + ".txt"), "w") as f:
            f.write(mg.calib_text(P2))
        tg = syn.make_targets(1, W // 4, H // 4)
        tg['calib_P'] = [T.read_kitti_calib(os.path.join(root, "calib", img_id + ".txt"))]
        with torch.no_grad():
            m.heads.post_processor.output_depth = 'direct'
            det = m(images[b:b + 1].cuda(), [t.to("cuda") for t in syn.make_param_lists(tg)])[0].double().cpu()
        lines = mg.image_labels(g, P2, W, H, b)[:6]
        for p in det[:20:2].tolist():
            lines.append("%s 0.00 0 %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                E.ID_TYPE_CONVERSION[int(p[0])], *p[1:13]))
        with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
            f.write("".join(l + "\n" for l in lines))
        rows = T.read_kitti_label(lines)
        gt = torch.zeros(40, 7)
        gt[:len(rows), 0] = 1
        gt[:len(rows), 1] = torch.from_numpy(rows[:, 0])
        gt[:len(rows), 2:6] = torch.from_numpy(rows[:, 3:7])
        gt[:len(rows), 6] = torch.from_numpy(rows[:, 12])
        targets += labelled_targets(tg, gt[None])
    split = os.path.join(root, "ImageSets", "val.txt")
    with open(split, "w") as f:
        f.write("".join(i + "\n" for i in ids))
    dataset = types.SimpleNamespace(label_dir=os.path.join(root, "label_2"), imageset_txt=split,
                                    classes=["Car", "Pedestrian", "Cyclist"])
    return dataset, images, [t.to("cpu") for t in targets], ids


def eight_passes(model, loader, output_folder):
    """engine/inference.py:130-197 on the product path: per method set output_depth, run the whole loader, write the
    files, evaluate_python the folder; then the summary lines"""
    log = logging.getLogger("monoflex.inference")
    rets = []
    for method in EVAL_DEPTH_METHODS:
        log.info("evaluation with depth method: %s" % method)
        folder = os.path.join(output_folder, "eval_all_depths", method)
        os.makedirs(folder, exist_ok=True)
        for name in os.listdir(folder):
            os.remove(os.path.join(folder, name))
        model.heads.post_processor.output_depth = method
        with torch.no_grad():
            for batch in loader:
                out, eu, _ = model(batch["images"].cuda(), [t.to("cuda") for t in batch["targets"]])
                for img_id, r in zip(batch["img_ids"], out.cpu().split(eu['counts'])):
                    E.write_kitti_detections(r, os.path.join(folder, img_id + ".txt"))
        ds = loader.dataset
        rets.append(E.evaluate_python(ds.label_dir, folder, ds.imageset_txt, ds.classes, "R40")[1])
    log.info("Car AP@0.70, 0.70:")
    moderate = []
    for method, r in zip(EVAL_DEPTH_METHODS, rets):
        log.info("bev/3d AP, method %s:" % method)
        v = [r["Car_%s_0.70/%s" % (kind, level)] for level in ("easy", "moderate", "hard") for kind in ("bev", "3d")]
        log.info("%.4f/%.4f, %.4f/%.4f, %.4f/%.4f" % tuple(v))
        moderate.append(r["Car_3d_0.70/moderate"])
    log.info("Cls Car, Thresh 0.7, Sort: " + " > ".join(EVAL_DEPTH_METHODS[i] for i in np.argsort(-np.array(moderate))))
    return rets


@pytest.mark.gpu
@pytest.mark.parametrize("batch_size", [1, 3])
def test_inference_all_depths_drop_in(tmp_path, caplog, monkeypatch, batch_size):
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg(width=1280, height=384))
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval()
    m.heads.post_processor.det_threshold = 0.0
    dataset, images, targets, ids = kitti_set(str(tmp_path / "kitti"), m)
    loader = Loader(dataset, images, targets, ids, batch_size)
    rets = []
    official = E.get_official_eval_result

    def recorded(*a, **k):
        out = official(*a, **k)
        rets.append(out[1])
        return out
    monkeypatch.setattr(E, "get_official_eval_result", recorded)
    a, b = tmp_path / "loop", tmp_path / "one_pass"
    stale = b / "eval_all_depths" / "soft"
    stale.mkdir(parents=True)
    (stale / "999999.txt").write_text("Car 0 0 0 0 0 10 10 1 1 1 0 0 5 0 0.9\n")      # removed before the pass
    with caplog.at_level(logging.INFO, logger="monoflex.inference"):
        eight_passes(m, loader, str(a))
        loop_log = [r.getMessage() for r in caplog.records if r.name == "monoflex.inference"]
        loop_rets, rets[:] = list(rets), []
        caplog.clear()
        assert inference_all_depths(m, loader, "kitti_val", output_folder=str(b), metrics=["R11"]) == (None, None, None)
        one_log = [r.getMessage() for r in caplog.records if r.name == "monoflex.inference"]
    assert one_log == loop_log and len(one_log) == 8 + 1 + 16 + 1
    assert len(rets) == len(loop_rets) == 8
    for r, r0 in zip(rets, loop_rets):
        assert list(r) == list(r0)
        assert np.array_equal(list(r.values()), list(r0.values()), equal_nan=True)
    assert max(np.nan_to_num(list(rets[EVAL_DEPTH_METHODS.index('direct')].values()))) > 0     # detections matched
    for method in EVAL_DEPTH_METHODS:
        fa, fb = a / "eval_all_depths" / method, b / "eval_all_depths" / method
        assert sorted(os.listdir(fa)) == sorted(os.listdir(fb)) == sorted(i + ".txt" for i in ids)
        for name in os.listdir(fa):
            assert (fa / name).read_bytes() == (fb / name).read_bytes(), (method, name)


def test_drop_in_refuses_other_models_and_the_visualiser(tmp_path):
    loader = types.SimpleNamespace(dataset=None)
    with pytest.raises(TypeError, match="KeypointDetector"):
        inference_all_depths(torch.nn.Linear(2, 2), loader, "kitti_val", output_folder=str(tmp_path))
    with pytest.raises(NotImplementedError):
        inference_all_depths(None, loader, "kitti_val", output_folder=str(tmp_path), vis=True)
