"""Training throughput of the reference's do_train loop three ways, in one process, the arms alternated:

  reference  the reference-shaped do_train body: eager `model(images, targets)`, FusedAdamW, `scheduler.step(i)`, and per
             step MetricLogger.update on the host log and TensorBoard writes of every meter (engine/trainer.py)
  drop_in    monoflex_b200.train.do_train: the captured Trainer step, logs read two steps late, the same TensorBoard
             writes
  floor      Trainer(use_cuda_graph=True) fed the same loader, nothing logged

on a synthetic KITTI directory of KITTI-sized PNGs, B = 8 at 384x1280, with no evaluation or checkpoint inside the timed
window (EVAL_INTERVAL and SAVE_CHECKPOINT_INTERVAL past the run). Each arm starts from the same synthetic weights; its
first --warmup steps (graph capture included) are not timed. One checkpoint save (model, optimiser, scheduler through
torch.save) is timed too. Prints one JSON line with img/s per arm and repeat, the card's name and power limit.

    python tools/bench_do_train.py --steps 60 --warmup 6 --repeats 3 --frames 48
"""
import argparse
import io
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from monoflex_b200 import loader as L          # noqa: E402
from monoflex_b200 import solver               # noqa: E402
from monoflex_b200 import synthetic as syn     # noqa: E402
from monoflex_b200 import train as TR          # noqa: E402
from monoflex_b200.config import default_cfg   # noqa: E402
from monoflex_b200.model.detector import KeypointDetector   # noqa: E402

SIZES = [(1242, 375), (1224, 370), (1238, 374), (1241, 376), (1226, 370)]


def make_kitti(root, frames):
    from oracle import make_golden_targets as mg
    from oracle import make_golden_targets_right as mgr
    g = np.random.default_rng(7)
    for d in ("image_2", "label_2", "calib", "ImageSets"):
        os.makedirs(os.path.join(root, d))
    ids = ["%06d" % i for i in range(frames)]
    for k, img_id in enumerate(ids):
        w, h = SIZES[k % len(SIZES)]
        Image.fromarray(syn.natural_image(w, h, 500 + k)).save(os.path.join(root, "image_2", img_id + ".png"),
                                                               compress_level=6)
        P2 = mg.make_P2(g, w, h)
        with open(os.path.join(root, "calib", img_id + ".txt"), "w") as f:
            f.write(mg.calib_text(P2))
        views = [(P2, (w, h), f, False) for f in (0, 1)]
        lines = mgr.keep_encodable(mg.image_labels(g, P2, w, h, k % 8), views)
        with open(os.path.join(root, "label_2", img_id + ".txt"), "w") as f:
            f.write("".join(l + "\n" for l in lines))
    with open(os.path.join(root, "ImageSets", "train.txt"), "w") as f:
        f.write("".join(i + "\n" for i in ids))


def make_cfg(out, max_iter):
    cfg = default_cfg()
    cfg.DATASETS.TRAIN_SPLIT, cfg.DATASETS.USE_RIGHT_IMAGE = "train", False
    cfg.DATASETS.TEST = ("kitti_val",)
    cfg.SOLVER.IMS_PER_BATCH, cfg.SOLVER.MAX_ITERATION = 8, max_iter
    cfg.SOLVER.EVAL_INTERVAL = cfg.SOLVER.SAVE_CHECKPOINT_INTERVAL = 10 ** 9
    cfg.OUTPUT_DIR, cfg.START_TIME = out, "bench"
    return cfg


def make_model(cfg):
    m = KeypointDetector(cfg).cuda()
    m.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    return m.train()


class Timed(object):
    """the loader's batches; synchronises once when batch `warmup` is drawn and records the time"""

    def __init__(self, loader, warmup):
        self.loader, self.warmup, self.t0 = loader, warmup, None
        self.dataset = loader.dataset

    def __iter__(self):
        for i, batch in enumerate(self.loader):
            if i == self.warmup:
                torch.cuda.synchronize()
                self.t0 = time.perf_counter()
            yield batch


def arm_reference(cfg, loader, steps, warmup):
    from torch.utils.tensorboard import SummaryWriter
    model = make_model(cfg)
    opt = solver.build_optimizer(model, cfg)
    sched, _ = solver.build_scheduler(opt, cfg.SOLVER)
    meters = TR.MetricLogger()
    writer = SummaryWriter(os.path.join(cfg.OUTPUT_DIR, "writer", "reference"))
    src = Timed(loader, warmup)
    for i, data in zip(range(steps + warmup), src):
        loss_dict, log_loss_dict = model(data["images"].tensors, list(data["targets"]))   # host floats: one D2H read
        losses = sum(loss for loss in loss_dict.values())
        meters.update(loss=sum(v for k, v in log_loss_dict.items() if k.find("loss") >= 0), **log_loss_dict)
        opt.zero_grad()
        losses.backward()
        if i == 0:
            opt.mark_unused({n for n, _ in model.named_parameters()} - set(model.last_grad_names), model)
        opt.step()
        sched.step(i)
        meters.update(time=0.0, data=0.0)
        writer.add_scalars("train_metric/depth_errors", {k: m.value for k, m in meters.meters.items() if "MAE" in k}, i + 1)
        writer.add_scalar("stat/lr", opt.param_groups[0]["lr"], i + 1)
        for name, m in meters.meters.items():
            if "MAE" not in name:
                writer.add_scalar(("stat/{}" if name in ("time", "data") else "train_metric/{}").format(name), m.value,
                                  i + 1)
    torch.cuda.synchronize()
    dt = time.perf_counter() - src.t0
    writer.close()
    return dt, (model, opt, sched)


class _NoCheckpoints(object):
    """the run's only save is model_final after its last step; it is timed on its own below"""

    def save(self, name, **kwargs):
        if name != "model_final":
            raise RuntimeError("a checkpoint inside the timed window: %s" % name)


def arm_drop_in(cfg, loader, steps, warmup):
    model = make_model(cfg)
    opt = solver.build_optimizer(model, cfg)
    sched, _ = solver.build_scheduler(opt, cfg.SOLVER)
    src = Timed(loader, warmup)
    cfg.SOLVER.MAX_ITERATION = steps + warmup
    TR.do_train(cfg, False, model, src, None, opt, sched, None, _NoCheckpoints(), torch.device("cuda"),
                {"iteration": 0, "iter_per_epoch": 1})
    torch.cuda.synchronize()
    return time.perf_counter() - src.t0, (model, opt, sched)


def arm_floor(cfg, loader, steps, warmup):
    model = make_model(cfg)
    tr = TR.Trainer(model, cfg, use_cuda_graph=True)
    src = Timed(loader, warmup)
    for _, data in zip(range(steps + warmup), src):
        tr.step(data["images"].tensors, data["encoded"], sync_log=False)
    torch.cuda.synchronize()
    return time.perf_counter() - src.t0, (model, tr.optimizer, tr.scheduler)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else ""
    except Exception as e:                      # noqa: BLE001 - the numbers stand without it
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=6)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--frames", type=int, default=48)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_do_train needs a GPU")
    arms = {"reference": arm_reference, "drop_in": arm_drop_in, "floor": arm_floor}
    res = {k: [] for k in arms}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "kitti")
        make_kitti(root, a.frames)
        cfg0 = make_cfg(os.path.join(tmp, "out"), a.steps + a.warmup)
        loader = L.KittiTrainLoader(cfg0, root, seed=3)
        save_s = None
        for r in range(a.repeats):
            for name in (list(arms) if r % 2 == 0 else list(arms)[::-1]):
                cfg = make_cfg(os.path.join(tmp, "out"), a.steps + a.warmup)
                dt, state = arms[name](cfg, loader, a.steps, a.warmup)
                res[name].append(8 * a.steps / dt)
                if save_s is None:
                    model, opt, sched = state
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    buf = io.BytesIO()
                    torch.save({"model": model.state_dict(), "optimizer": opt.state_dict(),
                                "scheduler": sched.state_dict(), "iteration": 1, "iter_per_epoch": 1}, buf)
                    save_s = time.perf_counter() - t
                del state
                torch.cuda.empty_cache()
    out = {"workload": "do_train B=8 384x1280 frames=%d steps=%d warmup=%d" % (a.frames, a.steps, a.warmup),
           "img_per_s": {k: [round(v, 1) for v in vs] for k, vs in res.items()},
           "checkpoint_save_s": round(save_s, 3), "card": card()}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
