"""-m gpu: the training loader (monoflex_b200/loader.py KittiTrainLoader) on a generated KITTI-layout directory with
mixed image sizes and right images of other sizes than the left ones, with DATASETS.USE_RIGHT_IMAGE off and on, B = 1
and 3, world 1 and rank 1 of world 2, over two epochs and more. Every batch equals, bit for bit, the host path on the
same (index, flip) rows: GpuInputPipeline.images on the PIL-decoded arrays and GpuTargetEncoder.encode on the host-parsed
labels and calibration. Yielding a batch does not synchronise with the device; a truncated file and an object the
reference cannot encode in one flip state raise at construction; the reference's do_train body and the Trainer, eager
and captured, run on its batches."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from monoflex_b200 import loader as L
from monoflex_b200 import synthetic as syn
from monoflex_b200 import targets as T
from monoflex_b200.config import default_cfg
from monoflex_b200.data import GpuInputPipeline
from monoflex_b200.png import read_png
from monoflex_b200.structures import Calibration
from png_util import png_bytes

pytestmark = pytest.mark.gpu
SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370), (1234, 376), (1242, 374)]
RIGHT_SIZES = SIZES[3:] + SIZES[:3]
IDS = ["000004", "000001", "000010", "000003", "000007", "000002", "000008"]
ENC_FIELDS = ("edge_indices", "edge_len", "alphas", "gt_bboxes", "reg_weight", "occlusions", "truncations", "obj6", "P2",
              "status")


def train_cfg(right, B, world=1):
    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT = "train"
    cfg.DATASETS.USE_RIGHT_IMAGE = right
    cfg.SOLVER.IMS_PER_BATCH = B * world
    return cfg


def make_kitti(root):
    """labels that every view encodes in both flip states (the reference's oracle drops the others)"""
    from oracle import make_golden_targets as mg
    from oracle import make_golden_targets_right as mgr
    g = np.random.default_rng(23)
    for d in ("image_2", "image_3", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    for k, img_id in enumerate(IDS):
        for cam, (w, h), seed in (("image_2", SIZES[k], 200 + k), ("image_3", RIGHT_SIZES[k], 300 + k)):
            Image.fromarray(syn.natural_image(w, h, seed)).save(os.path.join(root, cam, img_id + ".png"),
                                                                compress_level=(1, 6, 9)[k % 3])
        calib = os.path.join(root, "calib", img_id + ".txt")
        with open(calib, "w") as f:
            f.write(mg.calib_text(mg.make_P2(g, *SIZES[k])))
        P2, P3 = T.read_kitti_calib(calib), T.read_kitti_calib(calib, use_right_cam=True)
        views = [(P2, SIZES[k], f, False) for f in (0, 1)] + [(P3, RIGHT_SIZES[k], f, True) for f in (0, 1)]
        lines = mgr.keep_encodable(mg.image_labels(g, P2, SIZES[k][0], SIZES[k][1], (0, 1, 2, 3, 4, 6, 7)[k]), views)
        with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
            f.write("".join(l + "\n" for l in lines))
    with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
        f.write("".join(i + "\n" for i in IDS))


@pytest.fixture(scope="module")
def kitti(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("kitti"))
    make_kitti(root)
    arrays = {(cam, i): np.asarray(Image.open(os.path.join(root, cam, i + ".png")).convert("RGB"))
              for cam in ("image_2", "image_3") for i in IDS}
    return root, arrays


def host_batch(cfg, root, arrays, rows):
    """the host path on (index, flip) rows: PIL arrays in pinned memory, files parsed on the host"""
    F = len(IDS)
    views = [T.dataset_view(i, F, cfg) for i in rows[:, 0]]
    flips = rows[:, 1].astype(bool)
    arrs = [arrays[("image_3" if r else "image_2", IDS[f])] for f, r in views]
    images, _ = GpuInputPipeline(cfg).images([torch.from_numpy(a.copy()).pin_memory() for a in arrs], flips=flips)
    labels = T.pack_labels([T.read_kitti_label(os.path.join(root, "label_2", IDS[f] + ".txt")) for f, _ in views], 40)
    P = np.stack([T.read_kitti_calib(os.path.join(root, "calib", IDS[f] + ".txt"), use_right_cam=r) for f, r in views])
    sizes = np.array([(a.shape[1], a.shape[0]) for a in arrs])
    right = np.array([r for _, r in views], dtype=np.int32) if cfg.DATASETS.USE_RIGHT_IMAGE else None
    enc = T.GpuTargetEncoder(cfg).encode(labels, P, sizes, flips.astype(np.int32), right=right)
    return images, enc, tuple(IDS[f] for f, _ in views)


def same_field(a, b):
    if isinstance(a, Calibration):
        return np.array_equal(np.asarray(a.P), np.asarray(b.P))
    return a.dtype == b.dtype and torch.equal(a.cpu(), b.cpu())


@pytest.mark.parametrize("right", [False, True])
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("rank,world", [(0, 1), (1, 2)])
def test_batches_equal_the_host_path(kitti, right, B, rank, world):
    root, arrays = kitti
    cfg = train_cfg(right, B, world)
    loader = L.KittiTrainLoader(cfg, root, rank=rank, world=world, seed=1000 + B)
    assert len(loader.dataset) == T.dataset_len(len(IDS), cfg) and loader.seed == 1000 + B
    assert not hasattr(loader, "__len__")
    n_batches = -(-3 * len(loader.dataset) // (world * B))           # three epochs of this rank's rows
    seen_flips = set()
    for k, (batch, rows) in enumerate(zip(loader, loader.sampler)):
        if k == n_batches:
            break
        images, enc, ids = host_batch(cfg, root, arrays, rows)
        seen_flips |= set(rows[:, 1].tolist())
        assert batch["img_ids"] == ids
        assert batch["images"].tensors.shape == (B, 3, 384, 1280)
        assert torch.equal(batch["images"].tensors, images)
        got = batch["encoded"]
        for a, b in zip(got.prepared, enc.prepared):
            assert torch.equal(a, b)
        for name in ENC_FIELDS:
            assert torch.equal(getattr(got, name), getattr(enc, name)), name
        assert int(got.status.item()) == 0
        want = enc.param_lists()
        assert len(batch["targets"]) == B
        for tg, tr, P in zip(batch["targets"], want, got.P2.cpu().numpy()):
            assert sorted(tg.fields()) == sorted(tr.fields())
            for name in tr.fields():
                assert same_field(tg.get_field(name), tr.get_field(name)), name
            assert not tg.has_field("ori_img")
            assert np.array(tg.get_field("calib").P).tobytes() == P.tobytes()   # the host flip, bit for bit the kernel's
    assert seen_flips == {0, 1}


def test_no_host_synchronisation_per_batch(kitti):
    root, _ = kitti
    cfg = train_cfg(True, 3)
    loader = L.KittiTrainLoader(cfg, root)
    n = -(-2 * len(loader.dataset) // 3)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        batches = [b for _, b in zip(range(n), loader)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert len(batches) == n
    assert all(int(b["encoded"].status.item()) == 0 for b in batches)


def test_truncated_png_raises_at_construction(tmp_path):
    root = str(tmp_path / "kitti")
    make_kitti(root)
    path = os.path.join(root, "image_3", IDS[5] + ".png")
    f = read_png(path)
    with open(path, "wb") as out:
        out.write(png_bytes(f.w, f.h, f.data[:len(f.data) // 2]))       # a cut stream in well-formed chunks
    L.KittiTrainLoader(train_cfg(False, 1), root)                         # image_3 is not read without USE_RIGHT_IMAGE
    with pytest.raises(ValueError, match="image_3/%s.png: PNG image data not decoded: truncated" % IDS[5]):
        L.KittiTrainLoader(train_cfg(True, 1), root)


def test_object_refused_in_one_flip_state_raises_at_construction(tmp_path):
    """an object across the right border whose heat-map radii are both non-zero only in the flipped view (the image
    pads by 19 px on both sides, the feature map rounds the border point differently after the flip)"""
    from oracle import make_golden_targets as mg
    from oracle import target_oracle_right as tor
    root = str(tmp_path / "kitti")
    make_kitti(root)
    k, (w, h) = 0, SIZES[0]
    P2 = mg.make_P2(np.random.default_rng(5), w, h)
    with open(os.path.join(root, "calib", IDS[k] + ".txt"), "w") as f:
        f.write(mg.calib_text(P2))
    line = "Car 0.42 1 -10.00 %.2f 179.50 %.2f 349.58 1.49 1.41 3.35 6.36 1.56 7.09 0.00" % (w - 1 - 179.48, w - 1 + 7.0)
    P2 = T.read_kitti_calib(os.path.join(root, "calib", IDS[k] + ".txt"))
    rows = T.read_kitti_label([line])
    assert [tor.encode_image(rows, P2, (w, h), f, False)[1] for f in (0, 1)] == [0, 1]
    with open(os.path.join(root, "label_2", IDS[k] + ".txt"), "w") as f:
        f.write(line + "\n")
    with pytest.raises(RuntimeError, match="frame %s, image_2, flipped: an object the reference cannot encode" % IDS[k]):
        L.KittiTrainLoader(train_cfg(False, 2), root)


def test_reference_training_loop_runs_on_the_batches(kitti):
    """engine/trainer.py:103-126: images and targets moved to the device, model(images, targets), the sum of the losses,
    zero_grad, backward, optimizer.step - with torch.optim.AdamW over the reference's parameter groups"""
    from monoflex_b200 import solver
    from monoflex_b200.model.detector import KeypointDetector
    root, _ = kitti
    cfg = train_cfg(True, 2)
    model = KeypointDetector(cfg).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    optimizer = torch.optim.AdamW(solver.get_model_params(model, cfg), lr=cfg.SOLVER.BASE_LR,
                                  weight_decay=cfg.SOLVER.WEIGHT_DECAY, betas=(0.9, 0.99))
    device = torch.device("cuda")
    w0 = model.backbone.base.level3.tree1.tree1.conv1.weight.detach().clone()
    totals = []
    for data, iteration in zip(L.KittiTrainLoader(cfg, root), range(0, 3)):
        images = data["images"].to(device)
        targets = [target.to(device) for target in data["targets"]]
        loss_dict, log_loss_dict = model(images, targets)
        losses = sum(loss for loss in loss_dict.values())
        optimizer.zero_grad()
        losses.backward()
        optimizer.step()
        totals.append(losses.item())
    assert len(totals) == 3 and np.isfinite(totals).all()
    assert not torch.equal(model.backbone.base.level3.tree1.tree1.conv1.weight.detach(), w0)


def test_captured_trainer_fed_encoded_matches_eager_fed_targets(kitti):
    """the tolerances of test_gpu_targets_right.py::test_captured_trainer_fed_right_targets_matches_eager"""
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.train import Trainer
    root, _ = kitti
    cfg = train_cfg(True, 2)
    models = []
    for _ in range(2):
        m = KeypointDetector(cfg).cuda()
        m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        models.append(m)
    ta = Trainer(models[0], cfg, loss_scale=128.0)
    tb = Trainer(models[1], cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    logs_a, logs_b = [], []
    for batch, _ in zip(L.KittiTrainLoader(cfg, root, seed=3), range(4)):
        x = batch["images"].tensors
        logs_a.append(ta.step(x, list(batch["targets"]))[1])
        logs_b.append(tb.step(x, batch["encoded"], sync_log=False)[1])
    assert tb._graph is not None
    logs_b = [l.resolve() for l in logs_b]
    for k, v in logs_a[0].items():
        assert abs(v - logs_b[0][k]) <= 1e-5 * max(abs(v), 1e-3), (k, v, logs_b[0][k])
    for i, (la, lb) in enumerate(zip(logs_a, logs_b)):
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(ta_tot) and np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
    assert logs_b[2] != logs_b[3]
