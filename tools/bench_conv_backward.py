"""Timing of the conv backward building blocks (wgrad on MN-major wgmma operands, dgrad via the forward kernel) at the
detector's 3x3 layer shapes, B = 8. One JSON line per shape (CUDA events, median of 7 after 3 warm-ups)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200._lib import call                                       # noqa: E402

SHAPES = [(8, 96, 320, 64, 64, 3, 1, 1), (8, 48, 160, 128, 128, 3, 1, 1), (8, 24, 80, 256, 256, 3, 1, 1),
          (8, 12, 40, 512, 512, 3, 1, 1), (8, 96, 320, 64, 128, 3, 2, 1), (8, 96, 320, 64, 256, 3, 1, 1)]


def timed(fn, n=7, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


def main():
    st = torch.cuda.current_stream().cuda_stream
    for (B, H, W, Cin, Cout, k, s, pad) in SHAPES:
        Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
        x = (torch.randn(B * H * W, Cin, device="cuda") * 0.5).half()
        dy = (torch.randn(B * Ho * Wo, Cout, device="cuda") * 0.1).half()
        dw = torch.empty(Cout, Cin, k, k, device="cuda")
        ms = timed(lambda: call("mf_conv2d_wgrad_nhwc_f16", x.data_ptr(), Cin, B, H, W, Cin, dy.data_ptr(), Cout, Cout, k, s, pad,
                                dw.data_ptr(), st))
        fl = 2.0 * B * Ho * Wo * Cout * Cin * k * k
        print(json.dumps({"op": "wgrad", "shape": [B, H, W, Cin, Cout, k, s, pad], "ms": ms, "TFLOPs": fl / ms / 1e9}), flush=True)


if __name__ == "__main__":
    main()
