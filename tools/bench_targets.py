"""Times GpuTargetEncoder.encode (csrc/mf_targets.cu + the heat-map kernel) on a batch of 8 seeded KITTI-like label sets
with CUDA events over a warmed loop, and, beside it, the per-image host time of oracle/target_oracle.py (the CPU port of the
reference's target encoding, not the reference itself) on this machine's CPU. With --right it times instead a batch that
mixes right-camera items (DATASETS.USE_RIGHT_IMAGE) and flips against the all-left batch of the same frames. Prints one JSON
line with the card's name and power limit.

    python tools/bench_targets.py [--iters 200] [--oracle-images 64]
    python tools/bench_targets.py --right [--iters 200] [--rounds 5]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from monoflex_b200 import targets as tg  # noqa: E402
from monoflex_b200.config import default_cfg  # noqa: E402
from oracle import target_oracle as to  # noqa: E402
from test_gpu_targets import random_batch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_encode(enc, inp, iters, right=None):
    """ms per encode call of a batch: eager (Python and launches included) and replayed from a CUDA graph (the kernels)"""
    out = tuple(t.clone() for t in enc.encode(*inp, right=right).prepared)
    for _ in range(20):
        enc.encode(*inp, out=out, right=right)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        enc.encode(*inp, out=out, right=right)
    t1.record()
    t1.synchronize()
    gpu_ms = t0.elapsed_time(t1) / iters
    # the same loop replayed from a CUDA graph: the kernels alone, without the Python and launch overhead
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enc.encode(*inp, out=out, right=right)
    g.replay()
    torch.cuda.synchronize()
    t0.record()
    for _ in range(iters):
        g.replay()
    t1.record()
    t1.synchronize()
    return gpu_ms, t0.elapsed_time(t1) / iters


def device_inputs(labels, P2, sizes, flips):
    dev = torch.device("cuda")
    return (torch.from_numpy(labels).to(dev), torch.from_numpy(P2).to(dev), torch.from_numpy(sizes).to(dev, torch.int32),
            torch.from_numpy(flips).to(dev, torch.int32))


def bench_right(args):
    """A mixed batch of 8 (four right-camera items, four flipped; every combination twice) against the same inputs
    encoded as left items (right flags off), timed alternately in rounds; the best round of each is reported."""
    from test_gpu_targets_right import random_batch as random_views
    cfg = default_cfg()
    cfg.DATASETS.USE_RIGHT_IMAGE = True
    enc = tg.GpuTargetEncoder(cfg)
    labels, P, sizes, _, right = random_views(7, B=8, right=[1, 0] * 4)
    inp = device_inputs(labels, P, sizes, np.array([1, 1, 0, 0] * 2))
    batches = {"left": (inp, torch.zeros(8, dtype=torch.int32, device="cuda"), int(labels[..., 0].sum())),
               "mixed": (inp, torch.from_numpy(right).cuda().to(torch.int32), int(labels[..., 0].sum()))}
    best = {k: [float("inf"), float("inf")] for k in batches}
    for _ in range(args.rounds):
        for name, (inp, rt, _) in batches.items():
            ms = time_encode(enc, inp, args.iters, right=rt)
            best[name] = [min(a, b) for a, b in zip(best[name], ms)]
    name, power = card()
    res = {"card": name, "power_limit": power, "batch": 8, "rounds": args.rounds}
    for k, (_, _, n) in batches.items():
        res.update({k + "_objects": n, k + "_encode_ms_per_batch": round(best[k][0], 4),
                    k + "_encode_graph_replay_ms_per_batch": round(best[k][1], 4)})
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--oracle-images", type=int, default=64)
    ap.add_argument("--right", action="store_true", help="time a batch mixing right-camera and flipped items against the "
                    "all-left batch (DATASETS.USE_RIGHT_IMAGE)")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds of --right")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_targets needs a GPU")
    if args.right:
        return bench_right(args)
    enc = tg.GpuTargetEncoder(default_cfg())
    labels, P2, sizes, flips = random_batch(7, B=8)
    gpu_ms, graph_ms = time_encode(enc, device_inputs(labels, P2, sizes, flips), args.iters)

    n, c0 = 0, time.perf_counter()
    while n < args.oracle_images:
        lab, p2, sz, fl = random_batch(1000 + n, B=8)
        for b in range(8):
            to.encode_image(lab[b, lab[b, :, 0] != 0, 1:15], p2[b], sz[b], bool(fl[b]))
        n += 8
    oracle_ms = (time.perf_counter() - c0) * 1e3 / n
    name, power = card()
    print(json.dumps({"card": name, "power_limit": power, "batch": 8, "objects": int(labels[..., 0].sum()),
                      "encode_ms_per_batch": round(gpu_ms, 4), "encode_graph_replay_ms_per_batch": round(graph_ms, 4),
                      "oracle_port_cpu_ms_per_image": round(oracle_ms, 3)}))


if __name__ == "__main__":
    main()
