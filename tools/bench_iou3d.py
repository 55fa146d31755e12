"""Times the CUDA get_iou_3d (csrc/mf_iou3d.cu) at N = 320 (one batch of 8's worth of objects) and N = 10^6 seeded
encode_box3d pairs, and mf_loss_forward (focal sum + the fused loss kernel, '3D_IoU' included) at B = 8, with CUDA events over
warmed loops. Prints one JSON line with the card's name and power limit.

    python tools/bench_iou3d.py [--iters 200] [--lib PATH] [--dump out.npy] [--loss-only]

--lib times mf_loss_forward of another build of libmonoflex_b200.so (same C ABI) and --dump writes its 48-float output
buffer, so two builds can be compared on the same seeded batch; --loss-only skips the get_iou_3d timings (a build without
mf_iou3d_corners)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from monoflex_b200 import _lib  # noqa: E402
from monoflex_b200 import synthetic as syn  # noqa: E402
from monoflex_b200.config import default_cfg  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, iters):
    for _ in range(10):
        fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(iters):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / iters


def bench_op(iters):
    from monoflex_b200.model.layers.iou_loss import get_iou_3d
    from test_gpu_iou3d import random_pairs
    res = {}
    for n in (320, 10 ** 6):
        a, b = (t.cuda() for t in random_pairs(n, seed=7))
        out = torch.empty(n, dtype=torch.float32, device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        raw = lambda: _lib.call("mf_iou3d_corners", a.data_ptr(), b.data_ptr(), n, out.data_ptr(), st)
        res["iou3d_kernel_ms_N%d" % n] = round(timed(raw, iters if n < 10 ** 5 else max(iters // 10, 10)), 5)
        res["get_iou_3d_call_ms_N%d" % n] = round(timed(lambda: get_iou_3d(a, b), iters if n < 10 ** 5 else max(iters // 10, 10)), 5)
    return res


def bench_loss(iters, lib_path, dump):
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    lib = ctypes.CDLL(lib_path)
    lib.mf_loss_forward.argtypes = _lib.SIGNATURES["mf_loss_forward"]
    lib.mf_loss_forward.restype = ctypes.c_int
    B = 8
    fields = syn.make_train_targets(B, seed=5)
    cls, reg = syn.make_train_predictions(B, fields, seed=6)
    lc = Loss_Computation(default_cfg())
    hm, obj, img = lc.prepare_targets([t.to("cuda") for t in syn.make_train_param_lists(fields)], torch.device("cuda"))
    cls, reg = cls.cuda().contiguous(), reg.cuda().contiguous()
    out = torch.zeros(48, dtype=torch.float32, device="cuda")
    ws = torch.zeros(96, dtype=torch.float32, device="cuda")        # ws96
    st = torch.cuda.current_stream().cuda_stream
    _, C, H, W = reg.shape

    def run():
        rc = lib.mf_loss_forward(cls.data_ptr(), hm.data_ptr(), reg.data_ptr(), obj.data_ptr(), img.data_ptr(),
                                 ctypes.addressof(lc._w11), ctypes.addressof(lc._dm9), B, cls.shape[1], lc.max_objs, H, W, C,
                                 out.data_ptr(), ws.data_ptr(), st)
        assert rc == 0
    ms = timed(run, iters)
    run()
    torch.cuda.synchronize()
    if dump:
        np.save(dump, out.cpu().numpy())
    return {"loss_forward_ms_B8": round(ms, 5), "objects": int(out[32].item())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--lib", default=_lib.LIB_PATH)
    ap.add_argument("--dump", default=None)
    ap.add_argument("--loss-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_iou3d needs a GPU")
    name, power = card()
    res = {"card": name, "power_limit": power, "lib": os.path.relpath(args.lib, ROOT)}
    if not args.loss_only:
        res.update(bench_op(args.iters))
    res.update(bench_loss(args.iters, args.lib, args.dump))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
