"""Cost of SOLVER.GRAD_NORM_CLIP on the device. Prints one JSON line with the card's name and power limit.

    python tools/bench_grad_clip.py [--iters 50] [--rounds 5] [--runs 3] [--steps 20]

1. The optimiser step at the detector's arena size (20,952,538 parameters), CUDA events, variants interleaved round by round:
     plain       FusedAdamW.step()                                   (scan + prepare + update)
     fused_clip  FusedAdamW.step(max_grad_norm=c), clipping active   (sum-of-squares scan + prepare + update + write-back)
     torch_clip  torch.nn.utils.clip_grad_norm_ over the 280 arena views, then FusedAdamW.step()
   Clipping changes the gradient in place (after one clipped step its norm is c and the next would not clip), so every
   iteration first restores the gradient arena from a copy; `restore` times that copy alone and `net_ms` subtracts it.
2. The captured Trainer (B = 8, 384x1280, one CUDA graph per step) without and with GRAD_NORM_CLIP, alternating runs.
   c is 1/50 of the gradient norm of the first (eager) step: this synthetic network's norm falls about 5-10x over the first
   steps, and the cost of clipping only has to be measured on steps that clip (checked on the last timed step of each run).
   Every run builds its model and trainer afresh."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from monoflex_b200 import solver  # noqa: E402
from monoflex_b200 import synthetic as syn  # noqa: E402
from monoflex_b200.config import default_cfg  # noqa: E402
from monoflex_b200.model.detector import KeypointDetector  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def new_model():
    m = KeypointDetector(default_cfg())
    m.load_state_dict(syn.make_state_dict(0))
    return m.cuda()


def bench_optimizer(iters, rounds):
    cfg = default_cfg()
    model = new_model()
    opt = solver.build_optimizer(model, cfg)
    n = sum(p.numel() for p in opt.arena.tensors)
    torch.manual_seed(0)
    opt.arena.grads.normal_(std=1e-3)
    for p, o in zip(opt.arena.tensors, opt.arena.offsets):            # padding stays zero, as backward leaves it
        opt.arena.grads[o + p.numel():o + -(-p.numel() // opt.arena.chunk) * opt.arena.chunk].zero_()
    g0 = opt.arena.grads.clone()
    c = 0.5 * float(g0.double().norm())
    views = [p for p in opt.arena.tensors]

    def restore():
        opt.arena.grads.copy_(g0)

    variants = {
        "restore": restore,
        "plain": lambda: (restore(), opt.step()),
        "fused_clip": lambda: (restore(), opt.step(max_grad_norm=c)),
        "torch_clip": lambda: (restore(), torch.nn.utils.clip_grad_norm_(views, c), opt.step()),
    }
    for fn in variants.values():                                       # warm every path (torch's foreach kernels included)
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    # clipping was active: the fused step's norm is above c and the arena it leaves has norm c
    variants["fused_clip"]()
    torch.cuda.synchronize()
    active = float(opt.last_grad_norm) > c and abs(float(opt.arena.grads.double().norm()) - c) <= 1e-5 * c
    times = {k: [] for k in variants}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, fn in variants.items():
            torch.cuda.synchronize()
            e0.record()
            for _ in range(iters):
                fn()
            e1.record()
            e1.synchronize()
            times[k].append(e0.elapsed_time(e1) / iters)
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out = {"params": n, "arena_elems": opt.arena.numel, "tensors": len(views), "iters": iters, "rounds": rounds,
           "clip": c, "clip_active": bool(active), "ms_per_call_median": med,
           "ms_per_call_all": times, "net_ms": {k: med[k] - med["restore"] for k in med if k != "restore"}}
    del opt, model
    torch.cuda.empty_cache()
    return out


def bench_trainer(runs, steps, B=8):
    from monoflex_b200.train import Trainer
    dev = torch.device("cuda")
    n_in = 3
    imgs = [syn.make_images(B, 384, 1280, seed=100 + i).to(dev) for i in range(n_in)]
    tgs = [[t.to(dev) for t in syn.make_train_param_lists(syn.make_train_targets(B, seed=5 + i, empty_image=B))]
           for i in range(n_in)]
    probe = Trainer(new_model(), default_cfg(), use_cuda_graph=False)
    probe.step(imgs[0], tgs[0])
    c = 0.02 * float(probe.optimizer.arena.grads.double().norm())
    del probe
    torch.cuda.empty_cache()
    res = {"batch": B, "steps": steps, "clip": c, "off_img_s": [], "on_img_s": [], "on_last_grad_norm": []}
    for r in range(2 * runs):
        on = r % 2 == 1
        cfg = default_cfg()
        if on:
            cfg.SOLVER.GRAD_NORM_CLIP = c
        tr = Trainer(new_model(), cfg, use_cuda_graph=True, graph_warmup=2)
        for i in range(4):
            tr.step(imgs[i % n_in], tgs[i % n_in], sync_log=False)
        torch.cuda.synchronize()
        assert tr._graph is not None
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            tr.step(imgs[i % n_in], tgs[i % n_in], sync_log=False)
        e1.record()
        e1.synchronize()
        res["on_img_s" if on else "off_img_s"].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
        if on:
            res["on_last_grad_norm"].append(float(tr.optimizer.last_grad_norm))
            assert res["on_last_grad_norm"][-1] > c, "the timed steps did not clip"
        assert tr.optimizer.skipped_steps() == 0
        del tr
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_grad_clip.py needs a GPU"
    name, power = card()
    out = {"card": name, "power_limit": power, "optimizer_step": bench_optimizer(args.iters, args.rounds),
           "captured_trainer": bench_trainer(args.runs, args.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
