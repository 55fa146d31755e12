"""inference_all_depths (--eval_all_depths) on the GPU: the reference's eight passes over the split against one
forward_depths pass, and the decode kernels alone with one estimator and with eight.

Workload: 384x1280 images, synthetic weights (synthetic.make_state_dict), strict precision, at B = 1 (the reference's
test loader, data/build.py:142-144) and B = 8, over --images images held in pinned host memory. Each batch goes up with a
non-blocking copy, its targets (calibration, padding, edge list and the oracle's label fields) with ParamsList.to.

  eight_pass  for each of the eight methods: set post_processor.output_depth, run model(images, targets) over every
              batch and copy the rows to the host (engine/inference.py:130-197 without the text files and the metric;
              each method's first batch captures its own graph, as on the product path)
  one_pass    model.forward_depths(images, targets, EVAL_DEPTH_METHODS) over every batch, the eight row sets copied to
              the host at once

The two alternate --rounds times in the same run, each window between device synchronisations; the medians are
reported. The decode kernels are timed in a CUDA graph of --reps back-to-back decodes of one predictor output (96x320
maps, K = 50, threshold 0.2) with CUDA events. The card's name and power limit are read in the same run. Prints one JSON
line and writes nothing.

    python tools/bench_all_depths.py [--images 320] [--rounds 3] [--reps 20] [--iters 50]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def workload(n_img, H, W):
    """pinned images [n_img, 3, H, W] (16 distinct synthetic images, repeated) and per-image targets with labels"""
    import torch
    from monoflex_b200 import synthetic as syn
    distinct = syn.make_images(16, H, W)
    images = torch.empty(n_img, 3, H, W).pin_memory()
    for i in range(0, n_img, 16):
        images[i:i + 16] = distinct[:n_img - i]
    g = torch.Generator().manual_seed(0)
    targets = syn.make_param_lists(syn.make_targets(n_img, W // 4, H // 4))
    for t in targets:
        n = 12
        xy = torch.rand(n, 2, generator=g) * torch.tensor([W - 200.0, H - 100.0])
        box = torch.cat([xy, xy + 20 + torch.rand(n, 2, generator=g) * torch.tensor([180.0, 80.0])], 1)
        t.add_field('reg_mask', torch.cat([torch.ones(n), torch.zeros(40 - n)]).to(torch.uint8))
        t.add_field('cls_ids', torch.randint(0, 3, (40,), generator=g))
        t.add_field('gt_bboxes', torch.cat([box, torch.zeros(40 - n, 4)]))
        t.add_field('locations', torch.rand(40, 3, generator=g) * 60)
    return images, targets


def batches(images, targets, B):
    import torch
    for i in range(0, images.shape[0], B):
        yield images[i:i + B].to("cuda", non_blocking=True), [t.to(torch.device("cuda")) for t in targets[i:i + B]]


def eight_pass(model, images, targets, B, methods):
    post = model.heads.post_processor
    for method in methods:
        post.output_depth = method
        for x, tg in batches(images, targets, B):
            model(x, tg)[0].cpu()


def one_pass(model, images, targets, B, methods):
    import torch
    for x, tg in batches(images, targets, B):
        out = model.forward_depths(x, tg, methods)
        torch.stack([out[m][0] for m in methods]).cpu()


def timed(fn, *args):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn(*args)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def time_decodes(B, modes, reps, iters):
    """us per decode of one B x 3 x 96 x 320 predictor output, `modes` a mode name or a tuple of them"""
    import torch
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.layers.utils import decode_detections, sigmoid_hm
    from oracle import monoflex_oracle as mo
    cl, rgm = syn.make_head_logits(B, 320, 96)
    heat, reg = sigmoid_hm(cl.cuda()), rgm.cuda()
    tg = syn.make_targets(B, 320, 96)
    calib = torch.tensor([list(mo.calib_from_P(P).values()) for P in tg["calib_P"]], dtype=torch.float32).cuda()
    pad, size = tg["pad_size"].cuda(), torch.tensor(tg["size"], dtype=torch.float32).cuda()
    gt = torch.zeros(B, 40, 7, device="cuda")
    args = (heat, reg, calib, pad, size, torch.tensor(mo.DIM_MEAN).cuda(), 50, 0.2)
    ws = decode_detections(*args, depth_mode=modes, gt=gt)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(reps):
            decode_detections(*args, ws=ws, depth_mode=modes, gt=gt)
    for _ in range(5):
        graph.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        graph.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / (iters * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=320)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import torch
    from bench_decode import card
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.config import default_cfg
    from monoflex_b200.inference import EVAL_DEPTH_METHODS
    from monoflex_b200.model.detector import KeypointDetector
    assert torch.cuda.is_available(), "bench_all_depths needs a GPU"
    H, W = 384, 1280
    model = KeypointDetector(default_cfg(width=W, height=H))
    model.load_state_dict(syn.make_state_dict(0))
    model = model.cuda().eval().set_precision("strict")
    images, targets = workload(a.images, H, W)
    name, power = card()
    res = {"gpu": name, "power_limit": power, "H": H, "W": W, "images": a.images, "precision": "strict",
           "methods": len(EVAL_DEPTH_METHODS), "rounds": a.rounds}
    with torch.no_grad():
        for B in (1, 8):
            warm_images, warm_targets = images[:2 * B], targets[:2 * B]
            eight_pass(model, warm_images, warm_targets, B, EVAL_DEPTH_METHODS)
            one_pass(model, warm_images, warm_targets, B, EVAL_DEPTH_METHODS)
            t8, t1 = [], []
            for _ in range(a.rounds):
                t8.append(timed(eight_pass, model, images, targets, B, EVAL_DEPTH_METHODS))
                t1.append(timed(one_pass, model, images, targets, B, EVAL_DEPTH_METHODS))
            m8, m1 = statistics.median(t8), statistics.median(t1)
            res["B%d" % B] = {"eight_pass_s": round(m8, 3), "one_pass_s": round(m1, 3), "speedup": round(m8 / m1, 2),
                              "eight_pass_img_per_s": round(a.images / m8, 1),
                              "one_pass_img_per_s": round(a.images / m1, 1),
                              "eight_pass_rounds_s": [round(t, 3) for t in t8],
                              "one_pass_rounds_s": [round(t, 3) for t in t1]}
            print("B=%d: eight passes %.3f s, one pass %.3f s over %d images (x%.2f)" % (B, m8, m1, a.images, m8 / m1))
        for B in (1, 8):
            one = time_decodes(B, 'soft', a.reps, a.iters)
            eight = time_decodes(B, EVAL_DEPTH_METHODS, a.reps, a.iters)
            res["decode_B%d_us" % B] = {"one_mode": round(one, 2), "eight_modes": round(eight, 2)}
            print("decode B=%d: one mode %.2f us, eight modes %.2f us" % (B, one, eight))
    print("on %s, power limit %s" % (name, power))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
