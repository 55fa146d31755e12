"""The reference's inference() as a drop-in (monoflex_b200/inference.py: inference) and the evaluation loader's kept passes
(monoflex_b200/loader.py: KittiEvalLoader).

CPU: the refusals that need no model, the row order the metric scores and the memory rule. GPU (-m gpu), on a generated
KITTI-layout directory of PNGs whose labels hold copies of the model's own detections (so that AP is not zero): the
drop-in writes the same files, returns the same ret_dicts and text and logs the same lines as compute_on_dataset +
evaluate_python, over a streamed, a kept and a host loader, at B = 1 and 3, with one and two metrics; the files do not
depend on the batch size; the kept passes equal the first bit for bit without reading a file or synchronising per
batch; a folder with a file the call did not write is scored as text; an evaluation between captured training steps
leaves the training state bit-identical and the captured step training on."""
import logging
import os
import re
import time
import types

import numpy as np
import pytest
import torch
from PIL import Image

from monoflex_b200 import evaluation as E
from monoflex_b200 import loader as L
from monoflex_b200 import synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.inference import detect_pass, inference, scored_rows

SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1242, 375)]
IDS = ["000017", "000003", "000011", "000000", "000025", "000002", "000009", "000031", "000006", "000014"]
TIMING = re.compile(r"^(Total run time|Model inference time): \S+ \(\S+ s / img per device, on (\d+) devices\)$")


# ------------------------------------------------------------------------------------------------------------- CPU
def test_drop_in_refuses_other_models_and_the_visualiser(tmp_path):
    loader = types.SimpleNamespace(dataset=None)
    with pytest.raises(TypeError, match="KeypointDetector"):
        inference(torch.nn.Linear(2, 2), loader, "kitti_val", output_folder=str(tmp_path))
    with pytest.raises(NotImplementedError):
        inference(None, loader, "kitti_val", output_folder=str(tmp_path), vis=True)
    assert os.listdir(str(tmp_path)) == []


def test_scored_rows_follow_the_result_files():
    """sorted ids, the last of a repeated id, ids that name no result file left out"""
    ids = ["000007", "000002", "abc", "000007", "000004"]
    counts = [2, 1, 3, 0, 2]
    pick, dt_counts = scored_rows(ids, counts, [0, 10, 20, 30, 40])
    assert dt_counts == [1, 2, 0]
    assert pick.dtype == torch.int64 and pick.tolist() == [10, 40, 41]
    pick, dt_counts = scored_rows([], [], [])
    assert pick.tolist() == [] and dt_counts == []


def test_store_budget_is_the_windows_images_plus_two_transient_buffers(monkeypatch):
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (12345, 1 << 40))
    sizes = [(64, 32), (48, 40), (80, 24)] * 3
    store, need, free = L.store_budget(sizes, 4)
    windows = [L.window_bytes(sizes[i:i + 4]) for i in (0, 4, 8)]
    assert store == sum(b for b, _ in windows) and need == store + 2 * max(f for _, f in windows) and free == 12345
    assert L.store_budget([], 4) == (0, 0, 12345)


# ------------------------------------------------------------------------------------------------------------- GPU
def make_model():
    """synthetic weights whose 2D boxes are widened by 24 px a side (the 2d_dim head's bias), so that the copies of its
    detections in the labels are tall enough for the metric's moderate and easy difficulties"""
    from monoflex_b200.model.detector import KeypointDetector
    m = KeypointDetector(default_cfg())
    sd = syn.make_state_dict(0)
    sd["heads.predictor.reg_heads.0.0.bias"] += 6.0
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.heads.post_processor.det_threshold = 0.0
    return m


def eval_cfg(B, split="val"):
    cfg = default_cfg()
    cfg.TEST.IMS_PER_BATCH = B
    cfg.DATASETS.TEST_SPLIT = split
    return cfg


def make_kitti(root, model):
    """PNG images of KITTI's sizes, calibrations and labels: the generator's objects plus copies of some of the model's
    detections on the image, each kept only if the target encoder takes it"""
    from oracle import make_golden_targets as mg
    g = np.random.default_rng(19)
    for d in ("image_2", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    P = {}
    for k, img_id in enumerate(IDS):
        w, h = SIZES[k % len(SIZES)]
        Image.fromarray(syn.natural_image(w, h, 400 + k)).save(os.path.join(root, "image_2", img_id + ".png"),
                                                               compress_level=6)
        P[img_id] = mg.make_P2(g, w, h)
        with open(os.path.join(root, "calib", img_id + ".txt"), "w") as f:
            f.write(mg.calib_text(P[img_id]))
        open(os.path.join(root, "label_2", img_id + ".txt"), "w").close()
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as f:
        f.write("".join(i + "\n" for i in IDS))
    with torch.no_grad():
        for batch in L.KittiEvalLoader(eval_cfg(1), root):
            img_id = batch["img_ids"][0]
            k = IDS.index(img_id)
            w, h = SIZES[k % len(SIZES)]
            det = model(batch["images"], list(batch["targets"]))[0].double().cpu()
            lines = mg.image_labels(g, P[img_id], w, h, k % 8)[:6]
            for p in det[:24:2].tolist():
                lines.append("%s 0.00 0 %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                    E.ID_TYPE_CONVERSION[int(p[0])], *p[1:13]))
            lines = mg.keep_encodable(lines, P[img_id], (w, h), False)
            with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
                f.write("".join(l + "\n" for l in lines))


@pytest.fixture(scope="module")
def model():
    return make_model()


@pytest.fixture(scope="module")
def kitti(tmp_path_factory, model):
    root = str(tmp_path_factory.mktemp("kitti"))
    make_kitti(root, model)
    return root


class HostLoader(object):
    """a host DataLoader's batches: the images and targets in host memory"""

    def __init__(self, dataset, batches):
        self.dataset, self.batches = dataset, batches

    def __iter__(self):
        return iter(self.batches)


def host_loader(loader, drop_last_image=False):
    out = []
    for b in loader:
        out.append(dict(images=b["images"].tensors.cpu(), targets=[t.to("cpu") for t in b["targets"]],
                        img_ids=b["img_ids"]))
    if drop_last_image:
        last = out.pop()
        if len(last["img_ids"]) > 1:
            out.append(dict(images=last["images"][:-1], targets=last["targets"][:-1], img_ids=last["img_ids"][:-1]))
    return HostLoader(loader.dataset, out)


def reference_inference(model, data_loader, dataset_name, output_folder, metrics):
    """engine/inference.py:17-128 on the product path: compute_on_dataset (model, output.cpu(), one file per image) and
    evaluate_python per metric, with the same log lines"""
    logger = logging.getLogger("monoflex.inference")
    dataset = data_loader.dataset
    logger.info("Start evaluation on {} dataset({} images).".format(dataset_name, len(dataset)))
    folder = os.path.join(output_folder, "data")
    os.makedirs(folder, exist_ok=True)
    t0 = time.time()
    model.eval()
    with torch.no_grad():
        for batch in data_loader:
            images = batch["images"].to("cuda")
            targets = [t.to("cuda") for t in batch["targets"]]
            output, eval_utils, _ = model(images, targets)
            output = output.to("cpu")
            for img_id, r in zip(batch["img_ids"], output.split(eval_utils["counts"])):
                E.write_kitti_detections(r, os.path.join(folder, img_id + ".txt"))
    total = time.time() - t0
    logger.info("Total run time: {} ({} s / img per device, on {} devices)".format(total, total / len(dataset), 1))
    logger.info("Model inference time: {} ({} s / img per device, on {} devices)".format(total, total / len(dataset), 1))
    logger.info('Finishing generating predictions, start evaluating ...')
    ret_dicts = []
    for metric in metrics:
        result, ret_dict = E.evaluate_python(dataset.label_dir, folder, dataset.imageset_txt, dataset.classes, metric)
        logger.info('metric = {}'.format(metric))
        logger.info('\n' + result)
        ret_dicts.append(ret_dict)
    return ret_dicts, result, {}


def messages(caplog):
    out = []
    for r in caplog.records:
        if r.name == "monoflex.inference":
            m = r.getMessage()
            t = TIMING.match(m)
            out.append("%s: <time> on %s devices" % (t.group(1), t.group(2)) if t else m)
    return out


def files(folder):
    return {n: open(os.path.join(folder, n), "rb").read() for n in sorted(os.listdir(folder))}


def assert_same_rets(got, ref):
    assert len(got) == len(ref)
    for r, r0 in zip(got, ref):
        assert list(r) == list(r0)
        assert np.array_equal(np.array(list(r.values()), np.float64), np.array(list(r0.values()), np.float64),
                              equal_nan=True)


@pytest.mark.gpu
@pytest.mark.parametrize("source", ["streamed", "kept", "host"])
@pytest.mark.parametrize("metrics", [["R40"], ["R40", "R11"]])
@pytest.mark.parametrize("B", [1, 3])
def test_drop_in_equals_the_reference_loop(tmp_path, caplog, model, kitti, source, metrics, B):
    ref_loader = L.KittiEvalLoader(eval_cfg(B), kitti)
    loader = L.KittiEvalLoader(eval_cfg(B), kitti)
    if source == "kept":
        list(loader)
        assert loader.kept
    elif source == "host":
        loader = host_loader(loader)
    with caplog.at_level(logging.INFO, logger="monoflex.inference"):
        ref = reference_inference(model, ref_loader, "kitti_val", str(tmp_path / "ref"), metrics)
        ref_log = messages(caplog)
        caplog.clear()
        got = inference(model, loader, "kitti_val", output_folder=str(tmp_path / "drop_in"), metrics=metrics)
        got_log = messages(caplog)
    assert got_log == ref_log and len(got_log) == 4 + 2 * len(metrics)
    assert_same_rets(got[0], ref[0])
    assert got[1] == ref[1] and got[2] == {}
    assert max(np.nan_to_num(list(got[0][0].values()))) > 0                    # detections matched the labels
    a, b = files(str(tmp_path / "ref" / "data")), files(str(tmp_path / "drop_in" / "data"))
    assert list(a) == list(b) == sorted(i + ".txt" for i in IDS)
    for name in a:
        assert a[name] == b[name], name
    assert any(len(v) > 1 for v in b.values())
    if source != "host":
        assert loader.kept                                                     # KITTI-sized images fit


@pytest.mark.gpu
def test_files_do_not_depend_on_the_batch_size(tmp_path, model, kitti):
    """no eval kernel reduces across the images of a batch"""
    out = {}
    for B in (1, 3, 8):
        folder = tmp_path / ("B%d" % B)
        inference(model, L.KittiEvalLoader(eval_cfg(B), kitti), "kitti_val", output_folder=str(folder))
        out[B] = files(str(folder / "data"))
    assert len(out[1]) == len(IDS)
    assert out[3] == out[1] and out[8] == out[1]


def batch_tensors(batch):
    t = [batch["images"].tensors]
    for tg in batch["targets"]:
        for name in sorted(tg.fields()):
            v = tg.get_field(name)
            t.append(v if torch.is_tensor(v) else torch.tensor(v.P, dtype=torch.float64))
    return batch["img_ids"], [x.clone() for x in t]


def assert_same_pass(got, ref):
    assert len(got) == len(ref)
    for (ids, ts), (ids0, ts0) in zip(got, ref):
        assert ids == ids0 and len(ts) == len(ts0)
        for x, x0 in zip(ts, ts0):
            assert x.dtype == x0.dtype and x.device == x0.device and torch.equal(x, x0)


def refuse(*a, **k):
    raise AssertionError("a kept pass read or decoded a file")


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 3])
def test_kept_passes_equal_the_first_without_reading_files(monkeypatch, kitti, B):
    from monoflex_b200 import png
    from monoflex_b200 import targets as T
    loader = L.KittiEvalLoader(eval_cfg(B), kitti)
    first = [batch_tensors(b) for b in loader]
    assert loader.kept and loader.store_bytes > 0
    with monkeypatch.context() as mp:
        for mod, name in ((png, "read_png"), (png, "decode_png"), (L, "read_png"), (L, "decode_windows"),
                          (L, "read_ihdr"), (T, "read_kitti_label"), (T, "read_kitti_calib")):
            mp.setattr(mod, name, refuse)
        for _ in range(2):
            assert_same_pass([batch_tensors(b) for b in loader], first)


@pytest.mark.gpu
def test_too_little_memory_keeps_nothing_and_streams_every_pass(monkeypatch, kitti):
    ref = [batch_tensors(b) for b in L.KittiEvalLoader(eval_cfg(3), kitti)]
    loader = L.KittiEvalLoader(eval_cfg(3), kitti)
    total = torch.cuda.mem_get_info()[1]
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda device=None: (1 << 20, total))
    decoded = []
    windows = L.decode_windows

    def counted(paths, device="cuda"):
        decoded.append(len(paths))
        return windows(paths, device)
    monkeypatch.setattr(L, "decode_windows", counted)
    for _ in range(3):
        assert_same_pass([batch_tensors(b) for b in loader], ref)
        assert not loader.kept
    assert decoded == [1, 1, 1]


@pytest.mark.gpu
def test_a_window_that_does_not_fit_drops_what_was_kept(monkeypatch, kitti):
    """memory enough for the whole store at the start, then not for the windows left: nothing is kept"""
    monkeypatch.setattr(L, "DECODE_WINDOW", 4)
    ref = [batch_tensors(b) for b in L.KittiEvalLoader(eval_cfg(2), kitti)]
    loader = L.KittiEvalLoader(eval_cfg(2), kitti)
    calls = []
    real = torch.cuda.mem_get_info

    def shrinking(device=None):
        calls.append(1)
        return (1 << 50, 1 << 50) if len(calls) == 1 else (0, real()[1])
    monkeypatch.setattr(torch.cuda, "mem_get_info", shrinking)
    assert_same_pass([batch_tensors(b) for b in loader], ref)
    assert not loader.kept and len(calls) >= 2


@pytest.mark.gpu
def test_store_bytes_equal_the_training_loaders(tmp_path):
    from test_gpu_train_loader import make_kitti as make_train_kitti, train_cfg
    root = str(tmp_path / "kitti")
    make_train_kitti(root)
    train = L.KittiTrainLoader(train_cfg(False, 1), root)
    ev = L.KittiEvalLoader(eval_cfg(1, "train"), root)
    list(ev)
    assert ev.store_bytes == train.store_bytes > 0
    assert ev.kept


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 5])
def test_kept_pass_does_not_synchronise_per_batch(tmp_path, model, kitti, B):
    loader = L.KittiEvalLoader(eval_cfg(B), kitti)
    inference(model, loader, "kitti_val", output_folder=str(tmp_path / "first"))    # decodes, keeps, captures
    assert loader.kept
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        rows = detect_pass(model, loader)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    result, counts = rows.read()
    assert rows.img_ids == IDS and len(counts) == len(IDS)
    os.makedirs(str(tmp_path / "second"))
    for img_id, r, n in zip(rows.img_ids, result, counts):
        E.write_kitti_detections(r[:n], str(tmp_path / "second" / (img_id + ".txt")))
    assert files(str(tmp_path / "second")) == files(str(tmp_path / "first" / "data"))


@pytest.mark.gpu
def test_a_file_the_call_did_not_write_is_scored_as_text(tmp_path, model, kitti):
    """the loader leaves out the split's last image and the folder holds a stale 999999.txt: evaluate_python pairs the
    sorted files with the split by position, so the reference scores the stale file in the last image's place"""
    loader = host_loader(L.KittiEvalLoader(eval_cfg(3), kitti), drop_last_image=True)
    stale = "Car 0 0 -1.5 500.0 150.0 600.0 250.0 1.5 1.6 3.9 1.0 1.6 20.0 -1.5 0.8\n"
    for name in ("ref", "drop_in"):
        os.makedirs(str(tmp_path / name / "data"))
        (tmp_path / name / "data" / "999999.txt").write_text(stale)
    ref = reference_inference(model, loader, "kitti_val", str(tmp_path / "ref"), ["R40", "R11"])
    got = inference(model, loader, "kitti_val", output_folder=str(tmp_path / "drop_in"), metrics=["R40", "R11"])
    assert_same_rets(got[0], ref[0])
    assert got[1] == ref[1]
    assert files(str(tmp_path / "ref" / "data")) == files(str(tmp_path / "drop_in" / "data"))


@pytest.mark.gpu
def test_drop_in_refuses_the_iou_diagnostic(tmp_path, kitti):
    from monoflex_b200.model.detector import KeypointDetector
    cfg = default_cfg()
    cfg.TEST.EVAL_DIS_IOUS = True
    m = KeypointDetector(cfg).cuda()
    with pytest.raises(NotImplementedError, match="EVAL_DIS_IOUS"):
        inference(m, L.KittiEvalLoader(eval_cfg(1), kitti), "kitti_val", output_folder=str(tmp_path))


def training_state(trainer):
    opt, g = trainer.optimizer, trainer._graph
    state = {"params": [p.detach().clone() for p in trainer.model.parameters()],
             "buffers": [b.detach().clone() for b in trainer.model.buffers()],
             "graph_inputs": [g["x"].clone()] + [t.clone() for t in g["prep"]]}
    for name in ("exp_avg", "exp_avg_sq"):
        state[name] = [getattr(opt, name).detach().clone()]
    state["steps"] = (opt.step_count, opt._step_t)
    return state


def assert_same_state(a, b):
    assert a["steps"] == b["steps"]
    for name in ("params", "buffers", "graph_inputs", "exp_avg", "exp_avg_sq"):
        assert len(a[name]) == len(b[name])
        for x, y in zip(a[name], b[name]):
            assert torch.equal(x, y), name


@pytest.mark.gpu
def test_evaluation_between_captured_steps_leaves_training_unchanged(tmp_path, kitti):
    """do_train's evaluation: k steps of a captured Trainer, the drop-in, model.train(), k more steps. The evaluation
    leaves the parameters, the optimiser state, the BN buffers and the captured step's inputs bit-identical, and the
    captured step goes on training after it; its files equal those of a fresh eval-mode model loaded from the state_dict
    of step k. Two training runs differ in the last bits (the scatter atomics of the DCN backward) and the synthetic
    network amplifies that from step to step, so the run with the evaluation is compared with one without it by the
    tolerances of test_gpu_train.py's captured-against-eager test."""
    from test_gpu_train_loader import make_kitti as make_train_kitti, train_cfg
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.train import Trainer
    root = str(tmp_path / "train")
    make_train_kitti(root)
    cfg = train_cfg(False, 2)
    k = 3
    batches = [b for b, _ in zip(L.KittiTrainLoader(cfg, root, seed=5), range(2 * k))]
    trainers = []
    for _ in range(2):
        m = KeypointDetector(cfg).cuda()
        m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        trainers.append(Trainer(m, cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2))
    ta, tb = trainers
    p0 = ta.optimizer.arena.params.clone()
    loader = L.KittiEvalLoader(eval_cfg(2), kitti)
    logs = {id(ta): [], id(tb): []}
    for i, batch in enumerate(batches):
        if i == k:
            assert ta._graph is not None
            torch.cuda.synchronize()
            before = training_state(ta)
            snapshot = {n: v.detach().clone() for n, v in ta.model.state_dict().items()}
            ta.model.heads.post_processor.det_threshold = 0.0
            inference(ta.model, loader, "kitti_val", output_folder=str(tmp_path / "between"))
            ta.model.train()
            assert_same_state(training_state(ta), before)
        for t in trainers:
            logs[id(t)].append(t.step(batch["images"].tensors, batch["encoded"], sync_log=False)[1])
    torch.cuda.synchronize()
    for i, (la, lb) in enumerate(zip(logs[id(ta)], logs[id(tb)])):
        la, lb = la.resolve(), lb.resolve()
        tot_a, tot_b = (sum(l[n] for n in l if n.endswith("_loss")) for l in (la, lb))
        assert np.isfinite(tot_a) and abs(tot_a - tot_b) <= (0.03 if i <= 2 else 0.25) * abs(tot_b), (i, tot_a, tot_b)
    da, db = ta.optimizer.arena.params - p0, tb.optimizer.arena.params - p0
    cos = float((da * db).sum() / (da.norm() * db.norm()))
    assert float(da.norm()) > 0 and cos > 0.5, cos
    assert ta.optimizer.skipped_steps() == 0 and ta.optimizer.step_count == tb.optimizer.step_count == 2 * k
    fresh = KeypointDetector(cfg).cuda()
    fresh.load_state_dict(snapshot)
    fresh.eval()
    fresh.heads.post_processor.det_threshold = 0.0
    inference(fresh, L.KittiEvalLoader(eval_cfg(2), kitti), "kitti_val", output_folder=str(tmp_path / "fresh"))
    between, again = files(str(tmp_path / "between" / "data")), files(str(tmp_path / "fresh" / "data"))
    assert list(between) == sorted(i + ".txt" for i in IDS) and between == again
