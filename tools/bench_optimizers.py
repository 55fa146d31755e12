"""Cost of the reference's SOLVER.OPTIMIZER choices on the device. Prints one JSON line with the card's name and power limit.

    python tools/bench_optimizers.py [--iters 50] [--rounds 5] [--runs 2] [--steps 20]

1. One optimiser step at the detector's arena size (20,952,538 parameters), CUDA events, variants interleaved round by round,
   for each OPTIMIZER:
     fused        the arena optimiser's step()                       (finite scan + prepare + one update pass)
     fused_clip   step(max_grad_norm=c), clipping active             (sum-of-squares scan + prepare + update + write-back)
     torch        what the reference runs on the same tensors: torch.optim.AdamW / torch.optim.Adam over the one-group-
                  per-tensor params (torch's default multi-tensor path on CUDA); for 'adam_onecycle' fastai's OptimWrapper
                  step: every grouped tensor multiplied by 1 - wd * lr, then torch.optim.Adam over the two groups
   Every iteration first restores the gradient arena from a copy (clipping rewrites it); `restore` times that copy alone and
   `net_ms` subtracts it.
2. The captured Trainer (B = 8, 384x1280, one CUDA graph per step) for each OPTIMIZER, runs alternating between them;
   every run builds its model and trainer afresh."""
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

OPTIMIZERS = ("adamw", "adam", "adam_onecycle")


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


def _torch_step(name, model, cfg, opt):
    """the reference's optimiser on the same parameters (p.grad are arena views)"""
    sc = cfg.SOLVER
    if name == "adamw":
        ref = torch.optim.AdamW(solver.get_model_params(model, cfg), lr=sc.BASE_LR, weight_decay=sc.WEIGHT_DECAY,
                                betas=(0.9, 0.99))
        return ref.step
    if name == "adam":
        ref = torch.optim.Adam(solver.get_model_params(model, cfg), lr=sc.BASE_LR, weight_decay=sc.WEIGHT_DECAY,
                               betas=(0.9, 0.99))
        return ref.step
    groups = [g["params"] for g in opt.param_groups]
    ref = torch.optim.Adam([{"params": g, "lr": sc.BASE_LR} for g in groups], betas=(0.9, 0.99))

    def wrapper_step():                         # fastai OptimWrapper.step with true_wd and bn_wd
        with torch.no_grad():
            for g in groups:
                for p in g:
                    p.data.mul_(1 - sc.WEIGHT_DECAY * sc.BASE_LR)
        ref.step()
    return wrapper_step


def bench_optimizer(name, iters, rounds):
    cfg = default_cfg()
    cfg.SOLVER.OPTIMIZER = name
    model = new_model()
    opt = solver.build_optimizer(model, cfg)
    arena = opt.arena
    n = sum(p.numel() for p in model.parameters())
    torch.manual_seed(0)
    arena.grads.normal_(std=1e-3)
    for p, o in zip(arena.tensors, arena.offsets):                      # padding stays zero, as backward leaves it
        arena.grads[o + p.numel():o + -(-p.numel() // arena.chunk) * arena.chunk].zero_()
    g0 = arena.grads.clone()
    c = 0.5 * float(g0.double().norm())
    torch_step = _torch_step(name, model, cfg, opt)

    def restore():
        arena.grads.copy_(g0)

    variants = {
        "restore": restore,
        "fused": lambda: (restore(), opt.step()),
        "fused_clip": lambda: (restore(), opt.step(max_grad_norm=c)),
        "torch": lambda: (restore(), torch_step()),
        "torch_clip": lambda: (restore(), torch.nn.utils.clip_grad_norm_(model.parameters(), c), torch_step()),
    }
    for fn in variants.values():                                       # warm every path (torch's foreach kernels included)
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    variants["fused_clip"]()
    torch.cuda.synchronize()
    active = float(opt.last_grad_norm) > c
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
    out = {"params": n, "arena_elems": arena.numel, "tensors": len(arena.tensors), "iters": iters, "rounds": rounds,
           "clip_active": bool(active), "ms_per_call_median": med, "ms_per_call_all": times,
           "net_ms": {k: med[k] - med["restore"] for k in med if k != "restore"}}
    del opt, model, torch_step
    torch.cuda.empty_cache()
    return out


def bench_trainer(runs, steps, B=8):
    from monoflex_b200.train import Trainer
    dev = torch.device("cuda")
    n_in = 3
    imgs = [syn.make_images(B, 384, 1280, seed=100 + i).to(dev) for i in range(n_in)]
    tgs = [[t.to(dev) for t in syn.make_train_param_lists(syn.make_train_targets(B, seed=5 + i, empty_image=B))]
           for i in range(n_in)]
    res = {"batch": B, "steps": steps, "img_s": {k: [] for k in OPTIMIZERS}}
    for _ in range(runs):
        for name in OPTIMIZERS:
            cfg = default_cfg()
            cfg.SOLVER.OPTIMIZER = name
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
            res["img_s"][name].append(B * steps / (e0.elapsed_time(e1) * 1e-3))
            assert tr.optimizer.skipped_steps() == 0
            del tr
            torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_optimizers.py needs a GPU"
    name, power = card()
    out = {"card": name, "power_limit": power,
           "optimizer_step": {k: bench_optimizer(k, args.iters, args.rounds) for k in OPTIMIZERS},
           "captured_trainer": bench_trainer(args.runs, args.steps)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
