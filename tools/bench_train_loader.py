"""The training loader (monoflex_b200/loader.py KittiTrainLoader) on the GPU: its one-time build and the captured training
step it feeds.

Workload: a KITTI-layout training split of --frames frames (default 512) generated under --out: --distinct synthetic
1242x375 images (synthetic.natural_image, PIL compress_level 6) per camera, hard-linked up to --frames in image_2 and
image_3 (other sizes for image_3), with labels and calibration from oracle/make_golden_targets.py's builders. No KITTI
files are used.

  build     KittiTrainLoader(cfg) with DATASETS.USE_RIGHT_IMAGE on (2 x --frames views), for each of --windows as
            loader.TRAIN_DECODE_WINDOW: wall time per phase (labels and calibration, IHDRs, decode, validation), per view,
            and the store's bytes; plus the host half of the decode alone (read_png + PngBatch on one thread) per view
  memory    torch.cuda.max_memory_allocated() after --steps captured steps at B = 8 (strict model, synthetic weights),
            fed by the loader (the store resident) and fed by prebuilt batches without a store
  rate      images/s of a captured Trainer (Trainer.step(images, encoded, sync_log=False), log read after the timed
            steps) at B = 8: fed by the loader, against the same loop fed by --prebuilt batches taken from the loader
            beforehand and kept on the device (images and encoded targets). --rounds rounds of --steps steps per arm,
            alternating, after a warm-up; medians and all rounds are reported

The card's name and power limit are read in the same run. Prints one JSON line.

    python tools/bench_train_loader.py --out /tmp/train_loader [--frames 512] [--distinct 32] [--windows 256,512]
                                       [--steps 60] [--rounds 3] [--prebuilt 16]"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def make_split(root, frames, distinct):
    import numpy as np
    from PIL import Image
    from monoflex_b200 import synthetic as syn
    from monoflex_b200 import targets as T
    from oracle import make_golden_targets as mg
    for d in ("image_2", "image_3", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    g = np.random.default_rng(7)
    ids = ["%06d" % i for i in range(frames)]
    sizes = {"image_2": (1242, 375), "image_3": (1238, 374)}
    for i, img_id in enumerate(ids):
        for cam, (w, h) in sizes.items():
            path = os.path.join(root, cam, img_id + ".png")
            if i < distinct:
                Image.fromarray(syn.natural_image(w, h, i + (0 if cam == "image_2" else 10000))).save(path, compress_level=6)
            else:
                os.link(os.path.join(root, cam, ids[i % distinct] + ".png"), path)
        calib = os.path.join(root, "calib", img_id + ".txt")
        with open(calib, "w") as f:
            f.write(mg.calib_text(mg.make_P2(g, *sizes["image_2"])))
        P2 = T.read_kitti_calib(calib)
        lines = [mg.random_object(g, P2, 1242, 375, "inside") for _ in range(int(g.integers(2, 12)))]
        with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
            f.write("".join(l + "\n" for l in lines))
    with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))


def train_cfg(B):
    from monoflex_b200.config import default_cfg
    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT = "train"
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    cfg.SOLVER.IMS_PER_BATCH = B
    return cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--windows", default="256,512")
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--prebuilt", type=int, default=16)
    args = ap.parse_args()
    import numpy as np
    import torch
    assert torch.cuda.is_available(), "bench_train_loader.py measures on a GPU"
    from monoflex_b200 import loader as L
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    from monoflex_b200.png import PngBatch, read_png
    from monoflex_b200.train import Trainer
    root = os.path.join(args.out, "kitti")
    if not os.path.exists(os.path.join(root, "ImageSets", "train.txt")):
        make_split(root, args.frames, args.distinct)
    B = 8
    cfg = train_cfg(B)
    res = {"card": card(), "frames": args.frames, "views": 2 * args.frames, "B": B}

    # host half of the decode alone, one thread
    ds = L.KittiTrainSplit(cfg, root, "train")
    files = [os.path.join(d, i + ".png") for d in (ds.image_dir, ds.image_right_dir) for i in ds.ids]
    t0 = time.perf_counter()
    for k in range(0, len(files), 256):
        PngBatch([read_png(p) for p in files[k:k + 256]])
    res["host_staging_ms_per_view"] = 1e3 * (time.perf_counter() - t0) / len(files)

    builds, loader = {}, None
    for win in [int(w) for w in args.windows.split(",")]:
        L.TRAIN_DECODE_WINDOW = win
        loader = None
        torch.cuda.empty_cache()
        t0 = time.perf_counter()
        loader = L.KittiTrainLoader(cfg, root, seed=0)
        total = time.perf_counter() - t0
        builds[win] = dict(total_s=total, per_view_ms=1e3 * total / len(loader.dataset),
                           phases_ms_per_view={k: 1e3 * v / len(loader.dataset) for k, v in loader.build_seconds.items()},
                           store_bytes=loader.store_bytes)
    res["build"] = builds

    def trainer():
        m = KeypointDetector(cfg).cuda()
        m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
        return Trainer(m, cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)

    it = iter(loader)
    prebuilt = []
    for _ in range(args.prebuilt):
        b = next(it)
        prebuilt.append((b["images"].tensors.clone(), b["encoded"]))
    torch.cuda.synchronize()

    def run(tr, feed, steps):
        log = None
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(steps):
            x, enc = feed(k)
            log = tr.step(x, enc, sync_log=False)[1]
        log.resolve()
        torch.cuda.synchronize()
        return steps * B / (time.perf_counter() - t0)

    from_loader = lambda k: (lambda b: (b["images"].tensors, b["encoded"]))(next(it))
    from_prebuilt = lambda k: prebuilt[k % len(prebuilt)]
    ta, tb = trainer(), trainer()
    run(ta, from_loader, 10)
    run(tb, from_prebuilt, 10)
    rates = {"loader": [], "prebuilt": []}
    for _ in range(args.rounds):
        rates["loader"].append(run(ta, from_loader, args.steps))
        rates["prebuilt"].append(run(tb, from_prebuilt, args.steps))
    res["img_per_s"] = {k: dict(median=float(np.median(v)), rounds=v) for k, v in rates.items()}

    # peak memory of a captured run with the store and without it
    del ta, tb
    gc.collect()                               # a Trainer and its model hold reference cycles
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t = trainer()
    run(t, from_loader, args.steps)
    with_store = torch.cuda.max_memory_allocated()
    pre = [(x.clone(), e) for x, e in prebuilt[:4]]
    del t, it, prebuilt, loader
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t = trainer()
    run(t, lambda k: pre[k % len(pre)], args.steps)
    res["max_memory_allocated"] = dict(with_store=with_store, without_store=torch.cuda.max_memory_allocated(),
                                       note="without_store keeps 4 prebuilt batches on the device")
    print(json.dumps(res, default=lambda o: o.item()))


if __name__ == "__main__":
    main()
