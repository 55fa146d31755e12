"""-m gpu: the evaluation loader (monoflex_b200/loader.py) on generated KITTI-layout directories of PNGs with image
content, val- and test-style splits, mixed image sizes, B = 1 and 3, one and several decode windows. Its images equal
GpuInputPipeline.images on the PIL-decoded arrays bit for bit, its targets equal GpuTargetEncoder's for the same files,
and the reference's evaluation loop writes byte-identical result files from it and from the PIL host path."""
import os

import numpy as np
import pytest
import torch
from PIL import Image

from monoflex_b200 import evaluation as E
from monoflex_b200 import loader as L
from monoflex_b200 import synthetic as syn
from monoflex_b200 import targets as T
from monoflex_b200.config import default_cfg
from monoflex_b200.data import GpuInputPipeline
from monoflex_b200.structures import Calibration
from monoflex_b200.png import read_png
from monoflex_b200.synthetic import natural_image
from png_util import png_bytes

pytestmark = pytest.mark.gpu
SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1242, 375)]
IDS = ["000007", "000003", "000011", "000000", "000005", "000002", "000009"]


def make_kitti(root, labelled):
    from oracle import make_golden_targets as mg
    g = np.random.default_rng(11)
    for d in ("image_2", "calib", "ImageSets") + (("label_2",) if labelled else ()):
        os.makedirs(os.path.join(root, d))
    for k, img_id in enumerate(IDS):
        w, h = SIZES[k % len(SIZES)]
        Image.fromarray(natural_image(w, h, 100 + k)).save(os.path.join(root, "image_2", img_id + ".png"),
                                                           compress_level=(1, 6, 9)[k % 3])
        P2 = mg.make_P2(g, w, h)
        with open(os.path.join(root, "calib", img_id + ".txt"), "w") as f:
            f.write(mg.calib_text(P2))
        if labelled:
            lines = mg.keep_encodable(mg.image_labels(g, P2, w, h, k), P2, (w, h), False)
            with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
                f.write("".join(l + "\n" for l in lines))
    split = "val" if labelled else "test"
    with open(os.path.join(root, "ImageSets", split + ".txt"), "w") as f:
        f.write("".join(i + "\n" for i in IDS))
    return split


def host_batches(cfg, root, split, B):
    """the PIL host path: decode, pinned memory, GpuInputPipeline.images, GpuTargetEncoder"""
    pipe, enc = GpuInputPipeline(cfg), T.GpuTargetEncoder(cfg)
    for i in range(0, len(IDS), B):
        ids = IDS[i:i + B]
        arrs = [np.asarray(Image.open(os.path.join(root, "image_2", j + ".png")).convert("RGB")) for j in ids]
        images, _ = pipe.images([torch.from_numpy(a.copy()).pin_memory() for a in arrs])
        sizes = np.array([(a.shape[1], a.shape[0]) for a in arrs])
        P2 = np.stack([T.read_kitti_calib(os.path.join(root, "calib", j + ".txt")) for j in ids])
        if split == "test":
            targets = enc.encode_inference(P2, sizes)
        else:
            labels = T.pack_labels([T.read_kitti_label(os.path.join(root, "label_2", j + ".txt")) for j in ids], 40)
            targets = enc.encode(labels, P2, sizes, flips=None).param_lists()
        yield dict(images=images.clone(), targets=targets, img_ids=ids)


def same_field(a, b):
    if isinstance(a, Calibration):
        return np.array_equal(np.asarray(a.P), np.asarray(b.P))
    if torch.is_tensor(a):
        return a.dtype == b.dtype and torch.equal(a.cpu(), b.cpu())
    return np.array_equal(np.asarray(a), np.asarray(b))


def eval_loop(model, batches, folder):
    """engine/inference.py's compute_on_dataset: model, result rows, generate_kitti_3d_detection per image"""
    os.makedirs(folder)
    with torch.no_grad():
        for batch in batches:
            images = batch["images"].tensors if hasattr(batch["images"], "tensors") else batch["images"]
            out, eu, _ = model(images.cuda(), [t.to("cuda") for t in batch["targets"]])
            for img_id, r in zip(batch["img_ids"], out.cpu().split(eu["counts"])):
                E.write_kitti_detections(r, os.path.join(folder, img_id + ".txt"))


@pytest.fixture(scope="module")
def model():
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg())
    m.load_state_dict(syn.make_state_dict(0))
    m = m.cuda().eval()
    m.heads.post_processor.det_threshold = 0.0
    return m


@pytest.mark.parametrize("labelled", [True, False])
@pytest.mark.parametrize("B,window", [(1, 64), (3, 64), (3, 2), (1, 3)])
def test_loader_matches_the_host_path(tmp_path, monkeypatch, model, labelled, B, window):
    monkeypatch.setattr(L, "DECODE_WINDOW", window)
    root = str(tmp_path / "kitti")
    split = make_kitti(root, labelled)
    cfg = default_cfg()
    cfg.TEST.IMS_PER_BATCH = B
    cfg.DATASETS.TEST_SPLIT = split
    loader = L.KittiEvalLoader(cfg, root)
    got = list(loader)
    ref = list(host_batches(cfg, root, split, B))
    assert len(got) == len(ref) == len(loader)
    for g, r in zip(got, ref):
        assert list(g["img_ids"]) == list(r["img_ids"])
        assert g["images"].tensors.shape == (len(r["img_ids"]), 3, 384, 1280)
        assert torch.equal(g["images"].tensors, r["images"])
        assert len(g["targets"]) == len(r["targets"])
        for tg, tr in zip(g["targets"], r["targets"]):
            assert sorted(tg.fields()) == sorted(tr.fields())
            for name in tr.fields():
                assert same_field(tg.get_field(name), tr.get_field(name)), name
            assert not tg.has_field("ori_img")
    if B == 3 and window == 2:
        eval_loop(model, got, str(tmp_path / "gpu"))
        eval_loop(model, ref, str(tmp_path / "host"))
        names = sorted(os.listdir(str(tmp_path / "host")))
        assert names == sorted(i + ".txt" for i in IDS) == sorted(os.listdir(str(tmp_path / "gpu")))
        for n in names:
            a = open(os.path.join(str(tmp_path / "gpu"), n), "rb").read()
            b = open(os.path.join(str(tmp_path / "host"), n), "rb").read()
            assert a == b, n
        assert any(len(open(os.path.join(str(tmp_path / "host"), n)).read()) > 1 for n in names)


def test_malformed_file_raises_before_its_window_is_yielded(tmp_path, monkeypatch):
    monkeypatch.setattr(L, "DECODE_WINDOW", 3)
    root = str(tmp_path / "kitti")
    split = make_kitti(root, False)
    path = os.path.join(root, "image_2", IDS[4] + ".png")
    f = read_png(path)
    with open(path, "wb") as out:
        out.write(png_bytes(f.w, f.h, f.data[:len(f.data) // 2]))       # a cut stream in well-formed chunks
    cfg = default_cfg()
    cfg.DATASETS.TEST_SPLIT = split
    seen = []
    with pytest.raises(ValueError, match="%s.png: PNG image data not decoded: truncated" % IDS[4]):
        for batch in L.KittiEvalLoader(cfg, root):
            seen += list(batch["img_ids"])
    assert seen == IDS[:3]
