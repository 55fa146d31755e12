"""Times GpuTargetEncoder.encode (csrc/mf_targets.cu + the heat-map kernel) on a batch of 8 seeded KITTI-like label sets
with CUDA events over a warmed loop, and, beside it, the per-image host time of oracle/target_oracle.py (the CPU port of the
reference's target encoding, not the reference itself) on this machine's CPU. Prints one JSON line with the card's name and
power limit.

    python tools/bench_targets.py [--iters 200] [--oracle-images 64]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--oracle-images", type=int, default=64)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_targets needs a GPU")
    enc = tg.GpuTargetEncoder(default_cfg())
    labels, P2, sizes, flips = random_batch(7, B=8)
    dev = torch.device("cuda")
    inp = (torch.from_numpy(labels).to(dev), torch.from_numpy(P2).to(dev), torch.from_numpy(sizes).to(dev, torch.int32),
           torch.from_numpy(flips).to(dev, torch.int32))
    out = tuple(t.clone() for t in enc.encode(*inp).prepared)
    for _ in range(20):
        enc.encode(*inp, out=out)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(args.iters):
        enc.encode(*inp, out=out)
    t1.record()
    t1.synchronize()
    gpu_ms = t0.elapsed_time(t1) / args.iters
    # the same loop replayed from a CUDA graph: the kernels alone, without the Python and launch overhead
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        enc.encode(*inp, out=out)
    g.replay()
    torch.cuda.synchronize()
    t0.record()
    for _ in range(args.iters):
        g.replay()
    t1.record()
    t1.synchronize()
    graph_ms = t0.elapsed_time(t1) / args.iters

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
