"""Time the two decode kernels (csrc/mf_decode.cu: nms_topk_stage1 + topk_decode_stage2) at B = 8, 96x320, C = 3, K = 50
inside a CUDA graph, on two heat maps:

  synthetic  sigmoid_hm of synthetic.make_head_logits (N(-3, 1.5) logits): every slab takes stage 1's fast path
  clamped    oracle/decode_edge_cases.py's clamp_s5: logits <= -9.3 (heat exactly 1e-4) with 0 to 200 objects per
             plane, the background a trained focal-loss head is expected to produce: every slab takes the radix fallback

The graph holds REPS back-to-back decodes of the same map (L2-warm); CUDA events around the replays give the time per
decode. Prints the card's name and power limit with the numbers, and one JSON line.

    python tools/bench_decode.py [--reps 20] [--iters 50]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], check=True,
                             capture_output=True, text=True).stdout.strip().splitlines()[0]
        return [s.strip() for s in out.split(",")]
    except (OSError, subprocess.CalledProcessError):
        import torch
        return [torch.cuda.get_device_name(0), "unknown"]


def time_decode(heat, reg, calib, pad, size, dim_mean, reps, iters):
    import torch
    from monoflex_b200.model.layers.utils import DecodeWorkspace, decode_detections
    B, C = heat.shape[:2]
    ws = DecodeWorkspace(B, C, 50, 50, heat.device)
    run = lambda: decode_detections(heat, reg, calib, pad, size, dim_mean, 50, 0.2, False, ws)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(3):
            run()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            run()
    for _ in range(5):
        g.replay()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        g.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e3 / (iters * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    import torch
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.layers.utils import sigmoid_hm
    from oracle import decode_edge_cases as de
    from oracle import monoflex_oracle as mo
    assert torch.cuda.is_available(), "bench_decode needs a GPU"
    B, H, W = 8, 96, 320
    cl, rgm = syn.make_head_logits(B, W, H)
    clamped = de.build("clamp_s5")
    assert tuple(clamped["maps"].shape) == (B, 3, H, W)
    tg = syn.make_targets(B, W, H)
    calib = torch.tensor([list(mo.calib_from_P(P).values()) for P in tg["calib_P"]], dtype=torch.float32).cuda()
    pad, size = tg["pad_size"].cuda(), torch.tensor(tg["size"], dtype=torch.float32).cuda()
    dim_mean, reg = torch.tensor(mo.DIM_MEAN).cuda(), rgm.cuda()
    name, power = card()
    res = {"gpu": name, "power_limit": power, "B": B, "H": H, "W": W, "reps": a.reps, "iters": a.iters}
    for key, logits in (("synthetic", cl), ("clamped", clamped["maps"])):
        heat = sigmoid_hm(logits.clone().cuda())
        paths = sorted(set(de.stage1_paths(heat.cpu(), 50, de.slab_count(B, 3, H, W, 50, *limits(torch))).reshape(-1)))
        us = time_decode(heat, reg, calib, pad, size, dim_mean, a.reps, a.iters)
        res[key + "_us"] = round(us, 2)
        res[key + "_paths"] = paths
        print("%-9s stage-1 paths %-16s %7.2f us per decode" % (key, "/".join(paths), us))
    print("on %s, power limit %s" % (name, power))
    print(json.dumps(res))


def limits(torch):
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


if __name__ == "__main__":
    main()
