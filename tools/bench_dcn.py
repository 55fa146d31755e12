"""Timing of Plan.dcn alone (the offset conv + the fused DCN launch) at the seven DCN layer shapes of a 384 x 1280 input,
B = 8, fast and strict precision. Prints one JSON line per (shape, precision): the plan's time (CUDA events around
Plan.run, median of 20 after 3 warm-ups), the two launches separately (Plan.run_timed, median of 5), the number of
layers of that shape in the backbone and the fused DCN's algorithmic TFLOP/s (2 x pixels x Cout x 9 Cin); then one line
with the layer-weighted totals and the share of the 64-column-tile (Cout <= 64) layers.

Offsets come from a random offset conv scaled so the rms offset is about 1.5 px, as in the calibrated synthetic weights.
Each line also gives the offset conv's L2 -> SM bytes, computed from the shape (offset_conv_traffic)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from monoflex_b200 import engine                                    # noqa: E402

B = 8


class _Mod(object):
    pass


def layer_shapes():
    """(Cin, Cout, H, W) -> number of DCN layers of that shape in the backbone plan of a 384 x 1280 input"""
    from monoflex_b200.config import default_cfg
    from monoflex_b200.model.backbone.dla_dcn import build_backbone
    counts = {}
    orig = engine.Plan.dcn

    def record(self, x, dcn_mod, bn, out=None):
        s = (x.C, dcn_mod.weight.shape[0], x.H, x.W)
        counts[s] = counts.get(s, 0) + 1
        return orig(self, x, dcn_mod, bn, out)

    net = build_backbone(default_cfg(width=1280, height=384)).cuda().eval()
    engine.Plan.dcn = record
    try:
        net.build_plan(1, 384, 1280, "cuda")
    finally:
        engine.Plan.dcn = orig
    del net
    torch.cuda.empty_cache()
    return counts


def dcn_module(gen, cin, cout):
    d = _Mod()
    t = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()
    d.weight = t(gen.standard_normal((cout, cin, 3, 3)) / np.sqrt(9 * cin))
    d.bias = t(gen.standard_normal(cout) * 0.1)
    d.conv_offset_mask = _Mod()
    d.conv_offset_mask.weight = t(gen.standard_normal((27, cin, 3, 3)) * 1.5 / np.sqrt(9 * cin))
    d.conv_offset_mask.bias = t(gen.standard_normal(27) * 0.2)
    return d


class _BN(object):
    def __init__(self, c, gen):
        self.weight = torch.from_numpy(gen.uniform(0.5, 1.5, c).astype(np.float32)).cuda()
        self.bias = torch.from_numpy((gen.standard_normal(c) * 0.1).astype(np.float32)).cuda()
        self.running_mean = torch.from_numpy((gen.standard_normal(c) * 0.1).astype(np.float32)).cuda()
        self.running_var = torch.from_numpy(gen.uniform(0.5, 1.5, c).astype(np.float32)).cuda()
        self.eps = 1e-5


def offset_conv_traffic(B, cin, H, W, pair, nsm=132):
    """L2 -> SM bytes of one offset/mask conv (csrc/mf_offset_conv.cu): the tile launch_offset_conv picks (the same search and
    cost estimate, restated), its input boxes per (tile, chunk, hi | lo) and the weight boxes (once per CTA when resident,
    per tile and chunk otherwise). Returns (bytes, (R, S, resident))."""
    nch, nhl, w_stage, smem_max = cin // 64, 2 if pair else 1, 3 * (64 if pair else 32) * 128, 232448
    best = None
    for nseg in range(1, W + 1):
        S = (W + nseg - 1) // nseg
        if nseg > 1 and S < 8:
            break
        if S + 2 > 256 or (W + S - 1) // S != nseg:
            continue
        P = S + 2
        for R in range(1, min(H, 254) + 1):
            nblk = (R * P - 2 + 127) // 128 * 2
            if nblk > 8:
                break
            a_half = ((nblk * 64 + 2 * P + 2) * 128 + 1023) & ~1023
            res = 3 * nch <= 24 and 3 * nch * w_stage + 2 * nhl * a_half + 2048 <= smem_max
            nas = min(4, (smem_max - 2048 - (3 * nch if res else 3) * w_stage) // (nhl * a_half))
            if nas < 2:
                continue
            ntiles = B * ((H + R - 1) // R) * nseg
            mma = nch * nblk * 36.0 * (26.2 if pair else 8.7)
            load = nch * (nhl * (R + 2.0) * P * 128 + (0.0 if res else 3.0 * w_stage)) / 30.0
            cost = -(-ntiles // nsm) * (max(mma, load) + 300.0)
            if best is None or cost < best[0]:
                a = ntiles * nch * nhl * (R + 2) * P * 128
                w = (min(ntiles, nsm) if res else ntiles) * nch * 3 * w_stage
                best = (cost, a + w, (R, S, res))
    return best[1], best[2]


def time_plan(P, n=20, warm=3):
    for _ in range(warm):
        P.run()
    torch.cuda.synchronize()
    ts = []
    for _ in range(n):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        P.run()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    per = [P.run_timed() for _ in range(5)]
    split = {}
    for i, (name, _, _) in enumerate(per[0]):
        split[name] = sorted(r[i][2] for r in per)[len(per) // 2]
    return sorted(ts)[len(ts) // 2], split


def main():
    counts = layer_shapes()
    shapes = sorted(counts, key=lambda s: (s[2], -s[0], -s[1]))
    total = {"fast": 0.0, "strict": 0.0}
    narrow = {"fast": 0.0, "strict": 0.0}
    for i, (cin, cout, H, W) in enumerate(shapes):
        for prec in ("fast", "strict"):
            gen = np.random.Generator(np.random.PCG64(i))
            d, bn = dcn_module(gen, cin, cout), _BN(cout, gen)
            P = engine.Plan("cuda", strict=prec == "strict")
            xa = P.act(B, H, W, cin)
            P.dcn(xa, d, bn)
            P.finalize()
            x = torch.from_numpy(gen.standard_normal((B * H * W, cin)).astype(np.float32)).cuda()
            if prec == "strict":
                hi = x.half()
                xa.buf.copy_(torch.cat([hi, (x - hi.float()).half()], 1))
            else:
                xa.buf.copy_(x.half())
            ms, split = time_plan(P)
            dcn_ms = sum(v for k, v in split.items() if k.startswith("mf_dcn"))
            off_ms = sum(v for k, v in split.items() if not k.startswith("mf_dcn"))
            n = counts[(cin, cout, H, W)]
            total[prec] += n * ms
            if cout <= 64:
                narrow[prec] += n * ms
            l2_bytes, tile = offset_conv_traffic(B, cin, H, W, prec == "strict")
            print(json.dumps({"shape": [B, cin, cout, H, W], "precision": prec, "layers": n, "plan_ms": ms,
                              "offset_conv_ms": off_ms, "offset_conv_l2_MB": l2_bytes / 1e6, "offset_conv_tile": tile,
                              "dcn_ms": dcn_ms,
                              "dcn_TFLOPs": 2.0 * B * H * W * cout * 9 * cin / dcn_ms / 1e9}), flush=True)
            del P, xa, x
            torch.cuda.empty_cache()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0), "layer_weighted_plan_ms": total,
                      "share_of_cout_le_64_layers": {k: narrow[k] / total[k] for k in total}}), flush=True)


if __name__ == "__main__":
    main()
