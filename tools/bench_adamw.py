"""Microbenchmark of the optimiser row (R13): one fused AdamW launch over the detector's 20.95 M-parameter arena.
Algorithmic bytes = 28 B/parameter (read p, g, m, v; write p, m, v); 4 arenas x 84 MB = 336 MB > 50 MB L2.
Prints one JSON line (HBM roofline against MEASURED_PEAKS.json)."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200 import solver                                      # noqa: E402
from monoflex_b200.config import default_cfg                          # noqa: E402
from monoflex_b200.model.detector import KeypointDetector             # noqa: E402


def main():
    cfg = default_cfg()
    model = KeypointDetector(cfg).cuda()
    opt = solver.build_optimizer(model, cfg)
    opt.arena.grads.normal_(std=1e-3)
    for _ in range(5):
        opt.step()
    torch.cuda.synchronize()
    iters = 50
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # python-side per-step overhead (280 version bumps) is outside the device time: time the kernel through the C ABI too
    from monoflex_b200 import _lib
    table = opt._lr_table()
    b1, b2 = opt.defaults["betas"]
    st = torch.cuda.current_stream().cuda_stream
    e0.record()
    for i in range(iters):
        _lib.call("mf_adamw_step", opt.arena.params.data_ptr(), opt.arena.grads.data_ptr(), opt.exp_avg.data_ptr(),
                  opt.exp_avg_sq.data_ptr(), table.data_ptr(), opt.arena.n_chunks, b1, b2, 1e-8, 1e-5, 6 + i, 1.0, 1.0, st)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    n = sum(p.numel() for p in opt.arena.tensors)
    peak = 3350.0                   # H100 SXM HBM3 data sheet, unless MEASURED_PEAKS.json has a measurement
    try:
        pk = json.load(open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")))
        peak = float(pk.get("hbm_gbs", peak))
    except Exception:
        pass
    gbs = 28.0 * n / (ms * 1e-3) / 1e9
    import time
    t0 = time.perf_counter()
    for _ in range(20):
        opt.step()
    torch.cuda.synchronize()
    host_ms = (time.perf_counter() - t0) / 20 * 1e3
    print(json.dumps({"kernel": "adamw_arena_kernel", "params": n, "arena_elems": opt.arena.numel, "tensors": len(opt.arena.tensors),
                      "ms_per_launch": ms, "algorithmic_bytes": 28 * n, "achieved_GBps": gbs, "peak_GBps": peak,
                      "frac": gbs / peak, "optimizer_step_wall_ms": host_ms}))


if __name__ == "__main__":
    main()
