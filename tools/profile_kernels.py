"""ncu driver: replays selected launches of the B=8 inference plan (MF_PRECISION = strict | fast) between cudaProfilerStart/Stop.
   ncu --set full --clock-control none --import-source on --profile-from-start off -o gpurun_out/prof python tools/profile_kernels.py
Selected: the head 3x3 implicit GEMM (N=2304), one 64->64 DCN (+ its offset conv) at 96x320, a level-3 3x3 conv,
the stem 7x7, an up-sample+add, and the two decode kernels."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200 import synthetic as syn                      # noqa: E402
from monoflex_b200.config import default_cfg                    # noqa: E402
from monoflex_b200.model.detector import KeypointDetector       # noqa: E402

H, W, B = 384, 1280, int(os.environ.get("B", "8"))
model = KeypointDetector(default_cfg(width=W, height=H))
model.load_state_dict(syn.make_state_dict(0))
model = model.cuda().eval()
tg = syn.make_targets(B, W // 4, H // 4)
targets = [t.to("cuda") for t in syn.make_param_lists(tg)]
x = syn.make_images(B, H, W).cuda()
with torch.no_grad():
    for _ in range(2):
        model(x, targets)
torch.cuda.synchronize()
bp, hp = model.backbone.last_plan, model.heads.predictor.last_plan
st = torch.cuda.current_stream().cuda_stream


def pick(plan, name, pred):
    for fn, args, n in plan.launches:
        if n == name and pred(args):
            return fn, args, n
    raise KeyError(name)


if model.precision == "strict":
    # strict precision: pair kernels (argument lists of engine.py's x2 emitters)
    sel_spec = [
        ("head", hp, "mf_head_conv_f16x2", lambda a: True),
        ("head2_reduce", hp, "mf_head2_reduce", lambda a: True),
        ("dcn64", bp, "mf_dcn_nhwc_f16x2", lambda a: a[6] == 64 and a[4] == 96),
        ("dcn128", bp, "mf_dcn_nhwc_f16x2", lambda a: a[6] == 128 and a[4] == 48),
        ("offconv64", bp, "mf_conv2d_nhwc_f16x2", lambda a: a[14] == 27 and a[6] == 64 and a[4] == 96),
        ("conv128", bp, "mf_conv2d_nhwc_f16x2", lambda a: a[14] == 128 and a[6] == 128 and a[10] == 3),
        ("conv64", bp, "mf_conv2d_nhwc_f16x2", lambda a: a[14] == 64 and a[6] == 64 and a[10] == 3),
        ("conv512", bp, "mf_conv2d_nhwc_f16x2", lambda a: a[14] == 512 and a[6] == 512 and a[10] == 3),
        ("stem", bp, "mf_conv2d_rows_f16x2", lambda a: a[4] == 8),
        ("level0", bp, "mf_conv2d_rows_f16x2", lambda a: a[4] == 16),
        ("upadd", bp, "mf_upsample_add_nhwc_f16", lambda a: a[12] == 160),
    ]
else:
    sel_spec = [
        ("head", hp, "mf_head_fused", lambda a: True),
        ("dcn64", bp, "mf_dcn_nhwc_f16", lambda a: a[5] == 64 and a[3] == 96),
        ("dcn128", bp, "mf_dcn_nhwc_f16", lambda a: a[5] == 128 and a[3] == 48),
        ("offconv64", bp, "mf_conv2d_nhwc_f16", lambda a: a[13] == 27 and a[5] == 64 and a[3] == 96),
        ("conv128", bp, "mf_conv2d_nhwc_f16", lambda a: a[13] == 128 and a[5] == 128 and a[9] == 3),
        ("conv64", bp, "mf_conv2d_nhwc_f16", lambda a: a[13] == 64 and a[5] == 64 and a[9] == 3),
        ("stem", bp, "mf_conv2d_rows_f16", lambda a: a[4] == 8),
        ("level0", bp, "mf_conv2d_rows_f16", lambda a: a[4] == 16 and a[5] == 1),
        ("upadd", bp, "mf_upsample_add_nhwc_f16", lambda a: a[12] == 160),
    ]
only = os.environ.get("ONLY")
sel = [(n, pick(pl, k, pred)) for n, pl, k, pred in sel_spec if not only or n in only.split(",")]
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for name, (fn, args, n) in sel:
    flush.zero_()                      # L2 flush before each profiled launch (outside the profiler range)
    torch.cuda.synchronize()
    torch.cuda.profiler.start()
    assert fn(*args, st) == 0, name
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
if not only or "decode" in only:
    pred = {'cls': hp.cls, 'reg': hp.reg}
    torch.cuda.profiler.start()
    with torch.no_grad():
        model.heads.post_processor(pred, targets)
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
print("profiled", [s[0] for s in sel])
