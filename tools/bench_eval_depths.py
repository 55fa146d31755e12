"""TEST.EVAL_DEPTH (--eval_depth) on the GPU: what the depth-error kernel adds to the graph-replayed eval forward.

Workload: 384x1280 images, synthetic weights (synthetic.make_state_dict), strict and fast precision, B = 1 (the
reference's test loader) and B = 8, 40 object slots per image of which 15 are valid, at seeded centres on the 96x320 map.

  forward     model(images, targets) with the graph replayed and the rows read back (the eval loop's call), timed over
              --iters calls between device synchronisations, without and with EVAL_DEPTH, alternating, --rounds rounds;
              the medians are reported
  kernel      mf_eval_depth_errors alone on one predictor output, --reps back-to-back launches between CUDA events

The card's name and power limit are read in the same run. Prints one JSON line and writes nothing.

    python tools/bench_eval_depths.py [--rounds 3] [--iters 50] [--reps 2000]"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

H, W, SLOTS, VALID = 384, 1280, 40, 15


def labelled_targets(B):
    import torch
    from monoflex_b200 import synthetic as syn
    g = torch.Generator().manual_seed(B)
    targets = syn.make_param_lists(syn.make_targets(B, W // 4, H // 4))
    for t in targets:
        t.add_field('reg_mask', torch.cat([torch.ones(VALID), torch.zeros(SLOTS - VALID)])[torch.randperm(SLOTS, generator=g)]
                    .to(torch.uint8))
        t.add_field('cls_ids', torch.randint(0, 3, (SLOTS,), generator=g))
        t.add_field('target_centers', torch.stack([torch.randint(0, W // 4, (SLOTS,), generator=g),
                                                   torch.randint(0, H // 4, (SLOTS,), generator=g)], 1).int())
        t.add_field('locations', torch.rand(SLOTS, 3, generator=g) * 60)
    return [t.to(torch.device("cuda")) for t in targets]


def time_forward(model, x, targets, iters):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(iters):
        model(x, targets)                  # finish() reads the counts: one host synchronisation per call
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / iters * 1e3


def time_kernel(model, x, targets, reps):
    import torch
    from monoflex_b200.model.layers.utils import eval_depth_errors
    post = model.heads.post_processor
    pred = model.heads.predictor(model.backbone(x), targets)
    reg = pred['reg'].float().contiguous()
    calib, table = post.prepare_targets(targets, False, x.device)[0], post.depth_table(targets, x.device)
    out, counts = eval_depth_errors(reg, calib, post.dim_mean, table)
    for _ in range(20):
        eval_depth_errors(reg, calib, post.dim_mean, table, out, counts)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        eval_depth_errors(reg, calib, post.dim_mean, table, out, counts)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / reps * 1e3


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--reps", type=int, default=2000)
    a = ap.parse_args()
    import torch
    from bench_decode import card
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.detector import KeypointDetector
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval_depths needs a GPU")
    name, power = card()
    sd = syn.make_state_dict(0)
    res = {"gpu": name, "power_limit": power, "H": H, "W": W, "slots": SLOTS, "valid": VALID, "rounds": a.rounds,
           "iters": a.iters, "runs": []}
    for precision in ("strict", "fast"):
        models = {}
        for on in (False, True):
            cfg = default_cfg(width=W, height=H)
            cfg.TEST.EVAL_DEPTH = on
            m = KeypointDetector(cfg)
            m.load_state_dict(sd)
            models[on] = m.cuda().eval().set_precision(precision)
        for B in (1, 8):
            x = syn.make_images(B, H, W).cuda()
            targets = labelled_targets(B)
            times = {False: [], True: []}
            with torch.no_grad():
                for on in (False, True):
                    for _ in range(3):
                        models[on](x, targets)                # capture, then warm replays
                for _ in range(a.rounds):
                    for on in (False, True):
                        times[on].append(time_forward(models[on], x, targets, a.iters))
                kernel_us = time_kernel(models[True], x, targets, a.reps)
            off, on = statistics.median(times[False]), statistics.median(times[True])
            res["runs"].append({"precision": precision, "B": B, "forward_ms": off, "forward_eval_depth_ms": on,
                                "added_ms": on - off, "kernel_us": kernel_us, "rounds_ms": {"off": times[False],
                                                                                           "on": times[True]}})
            print("%s B=%d: forward %.3f ms, with EVAL_DEPTH %.3f ms (%+.3f ms); kernel %.2f us"
                  % (precision, B, off, on, on - off, kernel_us), file=sys.stderr)
        del models
    print("on %s, power limit %s" % (name, power), file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
