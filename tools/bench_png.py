"""The PNG decode (csrc/mf_png.cu) and the evaluation loader (monoflex_b200/loader.py) on the GPU, against PIL.

Workload: --distinct synthetic 1242x375 RGB images with natural-looking content (gradients, soft shapes, sensor noise;
synthetic.natural_image), saved by PIL at its default compress_level 6, and hard links to them up to --files files
(default 3,769, the size of KITTI val) in a temporary KITTI-layout test split (image_2, calib, ImageSets/test.txt). No
KITTI files are used.

  kernels   mf_png_inflate + mf_png_unfilter over decode windows of --kernel-windows files, staged on the device once;
            CUDA events around --reps back-to-back launches after one warm-up launch; time per image
  staging   the host half of a window's decode (read_png of every file + PngBatch: read, CRCs, IDAT join, pinned
            staging), per image, one thread
  pil       np.asarray(Image.open(f).convert('RGB')) of the distinct files, one host thread, per image
  loop      images/s of KittiEvalLoader + the strict model (synthetic weights) + the result rows copied to the host, at
            B = 1 and B = 8 over every file, for each of --windows as loader.DECODE_WINDOW; against the same loop fed
            from the distinct images PIL-decoded ahead into pinned memory and cycled (GpuInputPipeline.images +
            encode_inference), whose decode is not timed. One warm-up pass over the first 64 files each, then
            --rounds passes, the arms alternating; all passes are reported

The card's name and power limit are read in the same run. Prints one JSON line; files go to a temporary directory.

    python tools/bench_png.py [--files 3769] [--distinct 32] [--windows 256,1024] [--kernel-windows 8,64,256,1024]
                              [--reps 5] [--rounds 2]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def make_split(root, n_files, n_distinct):
    import numpy as np
    from PIL import Image
    from monoflex_b200 import synthetic as syn
    for d in ("image_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    P2 = np.array(syn.KITTI_P2, dtype=np.float64).reshape(3, 4)
    calib = "".join("%s: %s\n" % (k, " ".join("%.12e" % v for v in P2.ravel())) for k in ("P0", "P1", "P2", "P3"))
    ids = ["%06d" % i for i in range(n_files)]
    for i, img_id in enumerate(ids):
        path = os.path.join(root, "image_2", img_id + ".png")
        if i < n_distinct:
            Image.fromarray(syn.natural_image(1242, 375, i)).save(path, compress_level=6)
        else:
            os.link(os.path.join(root, "image_2", ids[i % n_distinct] + ".png"), path)
        with open(os.path.join(root, "calib", img_id + ".txt"), "w") as f:
            f.write(calib)
    with open(os.path.join(root, "ImageSets", "test.txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))
    return [os.path.join(root, "image_2", i + ".png") for i in ids]


def kernel_times(files, windows, reps):
    import torch
    from monoflex_b200 import png as P
    out = {}
    pngs = [P.read_png(f) for f in files]
    for n in windows:
        batch = P.PngBatch([pngs[i % len(pngs)] for i in range(n)])
        dev = batch.upload()
        filtered = torch.empty(batch.filt_total, dtype=torch.uint8, device="cuda")
        images = torch.empty(batch.out_total, dtype=torch.uint8, device="cuda")
        status = torch.empty(n, dtype=torch.int32, device="cuda")
        batch.launch(dev, filtered, images, status)
        torch.cuda.synchronize()
        assert int(status.abs().sum()) == 0
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            batch.launch(dev, filtered, images, status)
        t1.record()
        torch.cuda.synchronize()
        out[n] = {"ms_per_image": t0.elapsed_time(t1) / (reps * n), "ms_per_window": t0.elapsed_time(t1) / reps,
                  "mean_png_bytes": sum(len(p.data) for p in batch.pngs) / n}
    return out


def staging_time(files):
    from monoflex_b200 import png as P
    t0 = time.perf_counter()
    P.PngBatch([P.read_png(f) for f in files])
    return (time.perf_counter() - t0) * 1e3 / len(files)


def pil_time(files):
    import numpy as np
    from PIL import Image
    t0 = time.perf_counter()
    for f in files:
        np.asarray(Image.open(f).convert("RGB"))
    return (time.perf_counter() - t0) * 1e3 / len(files)


def run_loader(model, loader):
    for batch in loader:
        model(batch["images"], batch["targets"])[0].cpu()


def run_pinned(model, pipe, enc, pinned, P2, B, n_files):
    import numpy as np
    from monoflex_b200.structures import to_image_list
    for i in range(0, n_files, B):
        imgs = [pinned[j % len(pinned)] for j in range(i, min(i + B, n_files))]
        sizes = np.array([(t.shape[1], t.shape[0]) for t in imgs])
        images, _ = pipe.images(imgs)
        targets = enc.encode_inference(np.repeat(P2[None], len(imgs), 0), sizes)
        model(to_image_list(images), targets)[0].cpu()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--files", type=int, default=3769)
    ap.add_argument("--distinct", type=int, default=32)
    ap.add_argument("--windows", default="256,1024", help="loader.DECODE_WINDOW values for the loop")
    ap.add_argument("--kernel-windows", default="8,64,256,1024")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch
    from PIL import Image
    from monoflex_b200 import loader as L
    from monoflex_b200 import synthetic as syn
    from monoflex_b200 import targets as T
    from monoflex_b200.config import default_cfg
    from monoflex_b200.data import GpuInputPipeline
    from monoflex_b200.model.detector import KeypointDetector
    assert torch.cuda.is_available(), "bench_png needs a GPU"
    windows = [int(w) for w in args.windows.split(",")]
    result = {"card": card(), "files": args.files}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "testing")
        files = make_split(root, args.files, args.distinct)
        result["kernels"] = kernel_times(files[:args.distinct], [int(w) for w in args.kernel_windows.split(",")],
                                         args.reps)
        result["staging_ms_per_image"] = staging_time(files[:args.distinct])
        result["pil_ms_per_image"] = pil_time(files[:args.distinct])
        cfg = default_cfg()
        model = KeypointDetector(cfg)
        model.load_state_dict(syn.make_state_dict(0))
        model = model.cuda().eval()
        pipe, enc = GpuInputPipeline(cfg), T.GpuTargetEncoder(cfg)
        pinned = [torch.from_numpy(np.asarray(Image.open(f).convert("RGB")).copy()).pin_memory()
                  for f in files[:args.distinct]]
        P2 = T.read_kitti_calib(os.path.join(root, "calib", "000000.txt"))
        loop = result["loop_img_per_s"] = {}
        with torch.no_grad():
            for B in (1, 8):
                cfg.TEST.IMS_PER_BATCH = B
                run_pinned(model, pipe, enc, pinned, P2, B, 64)
                arms = [("pinned_memory", lambda: run_pinned(model, pipe, enc, pinned, P2, B, args.files))]
                for w in windows:
                    L.DECODE_WINDOW = w
                    loader = L.KittiEvalLoader(cfg, root, "test")
                    arms.append(("png_loader_window_%d" % w, lambda loader=loader: run_loader(model, loader)))
                rates = {name: [] for name, _ in arms}
                for _ in range(args.rounds):
                    for name, fn in arms:
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        fn()
                        torch.cuda.synchronize()
                        rates[name].append(round(args.files / (time.perf_counter() - t0), 1))
                loop["B%d" % B] = rates
    print(json.dumps(result))


if __name__ == "__main__":
    main()
