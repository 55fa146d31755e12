"""Cost and behaviour of the dynamic loss scale (monoflex_b200/loss_scale.py). Prints one JSON line with the card's name and
power limit, read in the same run.

    python tools/bench_loss_scale.py [--iters 50] [--rounds 5] [--runs 3] [--steps 20] [--settle 100]

1. The captured Trainer (B = 8, 384x1280, one CUDA graph per step): static loss scale 128 against DynamicLossScale
   (init_scale 128, growth_interval 2000: no growth and, checked, no skipped step inside the timed window, so both variants
   run the same work plus the dynamic one's seeding multiply by the device scale, its unscale launch and its update
   launch). Runs alternate static / dynamic; every run builds its model and trainer afresh.
2. Unscale-and-accumulate into p.grad at the detector's 280 gradient sizes: one mf_unscale_accumulate launch against
   torch._foreach_add_(grads, srcs, alpha=1/S), CUDA events, interleaved round by round: device time (--iters calls
   replayed from one CUDA graph, as in the captured step) and eager time (the same calls from Python, host work included).
3. On the synthetic data, captured B = 8 from GradScaler's default 2^16: the scale after each of the first --settle steps and
   the number of skipped steps among them."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_grad_clip import card, new_model  # noqa: E402
from monoflex_b200 import synthetic as syn  # noqa: E402
from monoflex_b200.config import default_cfg  # noqa: E402
from monoflex_b200.loss_scale import DynamicLossScale  # noqa: E402


def batches(B, n_in=3):
    dev = torch.device("cuda")
    imgs = [syn.make_images(B, 384, 1280, seed=100 + i).to(dev) for i in range(n_in)]
    tgs = [[t.to(dev) for t in syn.make_train_param_lists(syn.make_train_targets(B, seed=5 + i, empty_image=B))]
           for i in range(n_in)]
    return imgs, tgs


def bench_trainer(runs, steps, B=8):
    from monoflex_b200.train import Trainer
    imgs, tgs = batches(B)
    n_in = len(imgs)
    res = {"batch": B, "steps": steps, "static_img_s": [], "dynamic_img_s": []}
    for r in range(2 * runs):
        dyn = r % 2 == 1
        scale = DynamicLossScale(init_scale=128.0) if dyn else 128.0
        tr = Trainer(new_model(), default_cfg(), loss_scale=scale, use_cuda_graph=True, graph_warmup=2)
        for i in range(4):
            tr.step(imgs[i % n_in], tgs[i % n_in], sync_log=False)
        torch.cuda.synchronize()
        assert tr._graph is not None
        skipped0 = tr.optimizer.skipped_steps()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            tr.step(imgs[i % n_in], tgs[i % n_in], sync_log=False)
        e1.record()
        e1.synchronize()
        res["dynamic_img_s" if dyn else "static_img_s"].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
        assert tr.optimizer.skipped_steps() == skipped0, "a timed step was skipped"
        if dyn:
            assert tr.scaler.get_scale() == 128.0
        del tr
        torch.cuda.empty_cache()
    for k in ("static_img_s", "dynamic_img_s"):
        v = sorted(res[k])
        res[k + "_median"] = v[len(v) // 2]
    return res


def bench_unscale(iters, rounds):
    model = new_model()
    gen = torch.Generator(device="cuda").manual_seed(0)
    dsts = [torch.zeros(p.shape, device="cuda") for p in model.parameters()]
    srcs = [torch.randn(p.shape, generator=gen, device="cuda") for p in model.parameters()]
    s = DynamicLossScale(init_scale=128.0)
    inv = s.scale.double().reciprocal().float().item()
    variants = {"unscale_accumulate": lambda: s.unscale_accumulate(dsts, srcs),
                "foreach_add": lambda: torch._foreach_add_(dsts, srcs, alpha=inv)}
    for fn in variants.values():
        for _ in range(5):
            fn()
    # device time: `iters` calls captured in one CUDA graph per variant (what the captured training step replays);
    # eager: the same calls launched from Python, host overhead included
    graphs = {}
    torch.cuda.synchronize()
    for k, fn in variants.items():
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(iters):
                fn()
        graphs[k] = g
    runs = {"graph": {k: (lambda g=g: g.replay()) for k, g in graphs.items()},
            "eager": {k: (lambda fn=fn: [fn() for _ in range(iters)]) for k, fn in variants.items()}}
    for k in graphs:
        graphs[k].replay()
    times = {mode: {k: [] for k in variants} for mode in runs}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for mode, fns in runs.items():
            for k, fn in fns.items():
                torch.cuda.synchronize()
                e0.record()
                fn()
                e1.record()
                e1.synchronize()
                times[mode][k].append(e0.elapsed_time(e1) / iters)
    n = sum(d.numel() for d in dsts)
    med = {mode: {k: sorted(v)[len(v) // 2] for k, v in t.items()} for mode, t in times.items()}
    return {"tensors": len(dsts), "elements": n, "bytes_per_call": 12 * n, "iters": iters, "rounds": rounds,
            "ms_per_call_median": med, "ms_per_call_all": times,
            "device_GB_s_median": {k: 12 * n / (v * 1e-3) / 1e9 for k, v in med["graph"].items()}}


def settle(steps, B=8):
    from monoflex_b200.train import Trainer
    imgs, tgs = batches(B)
    tr = Trainer(new_model(), default_cfg(), loss_scale="dynamic", use_cuda_graph=True, graph_warmup=2)
    scales, skips = [], []
    for i in range(steps):
        k0 = tr.optimizer.skipped_steps()
        tr.step(imgs[i % len(imgs)], tgs[i % len(tgs)], sync_log=False)
        skips.append(tr.optimizer.skipped_steps() - k0)
        scales.append(tr.scaler.get_scale())
    return {"batch": B, "steps": steps, "init_scale": 2.0 ** 16, "skipped": sum(skips),
            "skipped_at": [i for i, k in enumerate(skips) if k], "final_scale": scales[-1],
            "min_scale": min(scales), "scales": scales}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--settle", type=int, default=100)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_loss_scale.py needs a GPU"
    name, power = card()
    out = {"card": name, "power_limit": power, "unscale": bench_unscale(args.iters, args.rounds),
           "captured_trainer": bench_trainer(args.runs, args.steps), "settle": settle(args.settle)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
