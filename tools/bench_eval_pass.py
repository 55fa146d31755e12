"""The reference's per-epoch evaluation (engine/inference.py:inference, called by do_eval) against the drop-in
monoflex_b200.inference.inference, on a generated KITTI-layout directory.

Data: --images synthetic 1242x375 PNGs (synthetic.natural_image, PIL compress level 6) with calibrations and labels from
the target generator, in a temporary directory removed at the end. --distinct frames are generated, the others are
copies of them (image, calibration and labels) under their own ids, so every file is still read, decoded and parsed. Model: 384x1280, synthetic weights, strict precision, detection
threshold 0.

  reference    KittiEvalLoader at B = 1 (a fresh one per round, so every image is decoded), model(images, targets),
               output.cpu() and one file per image, then evaluation.evaluate_python on the folder (labels parsed as text)
  first_pass   the drop-in over a fresh KittiEvalLoader at B: streamed decode, the split's labels parsed once
  kept_pass    the drop-in again over the same loader: the kept images and targets, the kept ground truth
  phases       one more kept pass at B = 8 split into the drop-in's steps, run one after the other: the model loop
               (detect_pass), the end-of-pass read, the result files, the metric

Each case is timed between device synchronisations, in alternating rounds; medians are reported. The decoded split's
device bytes (`store_bytes`) and the card's name and power limit are read in the same run. Prints one JSON line.

    python tools/bench_eval_pass.py [--images 3769] [--distinct 32] [--rounds 2] [--kept 2]"""
import argparse
import json
import logging
import os
import shutil
import statistics
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def make_kitti(root, n_img, n_distinct):
    """image_2, calib, label_2 and ImageSets/val.txt of n_img frames; returns the split name"""
    import numpy as np
    from PIL import Image
    from monoflex_b200 import synthetic as syn
    from oracle import make_golden_targets as mg
    g = np.random.default_rng(0)
    for d in ("image_2", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    ids = ["%06d" % i for i in range(n_img)]
    w, h = 1242, 375
    for k, img_id in enumerate(ids):
        kinds = (("image_2", ".png"), ("calib", ".txt"), ("label_2", ".txt"))
        files = [os.path.join(root, d, img_id + ext) for d, ext in kinds]
        if k >= n_distinct:                   # a copy of frame k % n_distinct: image, calibration and labels
            for (d, ext), f in zip(kinds, files):
                shutil.copyfile(os.path.join(root, d, ids[k % n_distinct] + ext), f)
            continue
        Image.fromarray(syn.natural_image(w, h, k)).save(files[0], compress_level=6)
        P2 = mg.make_P2(g, w, h)
        with open(files[1], "w") as f:
            f.write(mg.calib_text(P2))
        lines = mg.keep_encodable(mg.image_labels(g, P2, w, h, k % 8), P2, (w, h), False)
        with open(files[2], "w") as f:
            f.write("".join(l + "\n" for l in lines))
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))
    return "val"


def reference_loop(model, loader, folder):
    import torch
    from monoflex_b200 import evaluation as E
    predict = os.path.join(folder, "data")
    os.makedirs(predict, exist_ok=True)
    model.eval()
    with torch.no_grad():
        for batch in loader:
            output, eval_utils, _ = model(batch["images"].to("cuda"), [t.to("cuda") for t in batch["targets"]])
            output = output.to("cpu")
            for img_id, r in zip(batch["img_ids"], output.split(eval_utils["counts"])):
                E.write_kitti_detections(r, os.path.join(predict, img_id + ".txt"))
    ds = loader.dataset
    return E.evaluate_python(ds.label_dir, predict, ds.imageset_txt, ds.classes, "R40")[1]


def timed(fn, *args):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kept", type=int, default=2, help="kept passes per round at B = 8 (one at B = 1)")
    a = ap.parse_args()
    import numpy as np
    import torch
    from bench_decode import card
    from monoflex_b200 import loader as L
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.config import default_cfg
    from monoflex_b200 import evaluation as E
    from monoflex_b200.inference import write_result_files as write_files
    from monoflex_b200.inference import detect_pass, inference, scored_rows, split_ground_truth
    from monoflex_b200.model.detector import KeypointDetector
    logging.getLogger("monoflex.inference").setLevel(logging.WARNING)
    tmp = tempfile.mkdtemp(prefix="bench_eval_pass_")
    try:
        root = os.path.join(tmp, "kitti")
        t0 = time.perf_counter()
        split = make_kitti(root, a.images, min(a.distinct, a.images))
        gen_s = time.perf_counter() - t0
        print("generated %d images in %.1f s" % (a.images, gen_s), flush=True)
        assert torch.cuda.is_available(), "bench_eval_pass needs a GPU"
        model = KeypointDetector(default_cfg())
        model.load_state_dict(syn.make_state_dict(0))
        model = model.cuda().eval().set_precision("strict")
        model.heads.post_processor.det_threshold = 0.0

        def cfg(B):
            c = default_cfg()
            c.TEST.IMS_PER_BATCH, c.DATASETS.TEST_SPLIT = B, split
            return c

        def out(name):
            path = os.path.join(tmp, "out", name)
            shutil.rmtree(path, ignore_errors=True)
            return path
        name, power = card()
        res = {"gpu": name, "power_limit": power, "images": a.images, "distinct_pngs": min(a.distinct, a.images),
               "H": 384, "W": 1280, "precision": "strict", "rounds": a.rounds}
        # warm-up: every batch shape's graph captured, the library loaded
        with torch.no_grad():
            for B in (1, 8):
                warm = L.KittiEvalLoader(cfg(B), root)
                warm.dataset.ids = warm.dataset.ids[:B + 1]
                for batch in warm:
                    model(batch["images"], list(batch["targets"]))

        def drop_in(loader, folder):
            return inference(model, loader, "kitti_val", output_folder=folder)
        times = {k: [] for k in ("reference_B1", "first_B1", "kept_B1", "first_B8", "kept_B8")}
        store = None
        for r in range(a.rounds):
            t, ret_ref = timed(reference_loop, model, L.KittiEvalLoader(cfg(1), root), out("reference"))
            times["reference_B1"].append(t)
            print("reference loop B=1: %.2f s" % t, flush=True)
            for B, kept in ((1, 1), (8, a.kept)):
                loader = L.KittiEvalLoader(cfg(B), root)
                t, ret = timed(drop_in, loader, out("first"))
                times["first_B%d" % B].append(t)
                print("first pass B=%d: %.2f s" % (B, t), flush=True)
                assert loader.kept, "the split did not fit in device memory"
                store = loader.store_bytes
                for _ in range(kept):
                    t, ret_k = timed(drop_in, loader, out("kept"))
                    times["kept_B%d" % B].append(t)
                    print("kept pass B=%d: %.2f s" % (B, t), flush=True)
                assert list(ret_k[0][0]) == list(ret[0][0]) == list(ret_ref)
                assert np.array_equal(list(ret_k[0][0].values()), list(ret_ref.values()), equal_nan=True)
                del loader
        # where a kept pass at B = 8 spends its time: the same steps as the drop-in, one after the other
        loader = L.KittiEvalLoader(cfg(8), root)
        drop_in(loader, out("first"))
        phases = {}
        t, rows = timed(detect_pass, model, loader)
        phases["model_loop_s"] = t
        t, (result, counts) = timed(rows.read)
        phases["read_s"] = t
        folder = out("phases")
        os.makedirs(folder)
        t, _ = timed(write_files, folder, rows.img_ids, result, counts)
        phases["write_files_s"] = t

        def metric():
            pick, dt_counts = scored_rows(rows.img_ids, counts, np.arange(rows.n) * result.shape[1])
            dt = E.KittiAnnos.from_results(rows.rows().index_select(0, pick.to(rows.device)), dt_counts)
            return E.get_official_eval_result(split_ground_truth(loader.dataset), dt, loader.dataset.classes)
        t, _ = timed(metric)
        phases["metric_s"] = t
        res["kept_B8_phases"] = {k: round(v, 3) for k, v in phases.items()}
        print("kept pass B=8 by phase: %s" % res["kept_B8_phases"], flush=True)
        del loader
        res["store_bytes"] = store
        res["generate_s"] = round(gen_s, 1)
        for k, v in times.items():
            m = statistics.median(v)
            res[k] = {"median_s": round(m, 3), "img_per_s": round(a.images / m, 1), "runs_s": [round(x, 3) for x in v]}
        res["speedup_kept_B8_vs_reference"] = round(res["reference_B1"]["median_s"] / res["kept_B8"]["median_s"], 2)
        print("on %s, power limit %s" % (name, power))
        print(json.dumps(res))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
