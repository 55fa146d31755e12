"""The predictor head kernel by kernel, in both precisions (-m gpu, except the float64-oracle check).

Every case drives the real Base_Predictor module on synthetic weights, so the plan builder's dispatch is exercised along with
the kernels, and compares it with the CPU oracle (oracle/monoflex_oracle.py::predictor, pinned to the reference by
tests/test_oracle_golden.py). The three paths, each asserted through the launch names of its plan:
  head2   strict, H*W % 4 == 0: the pair GEMM with the 1x1 heads in its epilogue (csrc/mf_igemm2.cu HEAD2) + mf_head2_reduce
  split   strict, H*W % 4 != 0: the N = 2304 split conv, then one split 1x1 conv per head
  fused   fast: the fused head (csrc/mf_head.cu)
and in each the edge fusion: mf_edge_mask, the gather, the Conv1d + BN through the conv kernels, the indexed add.

What makes the comparison sharp:
  - each regression head's channels relative to that head's own largest value; the heat map on its own, as logits;
  - at the border pixels of each image, the error relative to the edge-fusion term itself (the oracle's e_cls / e_off);
  - the gathered edge rows against the oracle's grid_sample; the hidden-row mask bit for bit;
  - per-image edge lists of different lengths, one of them along the last row and column of the map.
Strict precision runs the oracle in float64 on the values the pair rows hold, held to STRICT_TOL. At the product map size the
largest error (1.6e-5, at the border pixels) is the float32 grid arithmetic of the edge gather, which the reference's float32
grid_sample shares: its float32 oracle is as far from the float64 one there. Fast precision runs the oracle on fp16 features and
weights, rounding to fp16 where the kernels store (hidden activations, gathered rows, edge Conv1d output). Its floor is set by
single rounding flips: a hidden activation whose fp32 value lies next to an fp16 rounding boundary may round either way, which
moves one output by ~1e-4 of its head's range. Measured on an H100 80GB HBM3 (700 W power limit): at most 2.2e-4 on the outputs
(FAST_TOL = 5e-4) and 5.0e-4 on the gathered rows, which are fp16 themselves (FAST_ROW_TOL = 2^-10). In strict precision a lost
lo half of the hidden or gathered rows measures 1.6e-4 to 4.5e-4 on the same metrics: fast precision has no lo half to lose, and
its bound could not resolve one."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import rel_err, to_rows, to_rows_split
from test_gpu_ops import STRICT_TOL
from monoflex_b200 import engine, synthetic as syn
from monoflex_b200.config import default_cfg
from monoflex_b200.model.detector import KeypointDetector
from oracle import monoflex_oracle as mo

FAST_TOL = 5e-4          # fast precision against the fp16-rounded oracle
FAST_ROW_TOL = 2 ** -10  # fast gathered edge rows (fp16): one rounding step at the top of their range

CASES = [
    # B, H, W, edge-list pad per image, strict path, fast path
    (2, 96, 320, [(19, 4), (0, 0)], "head2", "fused"),        # product map size, two different edge lists
    (3, 12, 20, [(0, 0), (8, 2), (19, 4)], "head2", "fused"),  # H*W = 240: m-tiles span images, the last is ragged (720 = 5*128 + 80)
    (2, 10, 30, [(12, 6), (0, 0)], "head2", "fused"),         # H*W = 300, ragged; image 1's border is the last row and column
    (1, 9, 23, [(0, 0)], "split", "fused"),                   # H*W = 207 is odd: strict falls back to the split convs
]
CASE_IDS = ["%dx%dx%d" % c[:3] for c in CASES]

PATH_LAUNCHES = {
    "head2": {"mf_edge_mask", "mf_head_conv_f16x2", "mf_head2_reduce", "mf_edge_gather_split", "mf_conv2d_nhwc_f16x2",
              "mf_edge_head_add_split", "mf_sigmoid_clamp"},
    "split": {"mf_conv2d_nhwc_f16x2", "mf_edge_gather_split", "mf_edge_head_add_split", "mf_sigmoid_clamp"},
    "fused": {"mf_edge_mask", "mf_head_fused", "mf_edge_gather", "mf_conv2d_nhwc_f16", "mf_edge_head_add", "mf_sigmoid_clamp"},
}
PREFIX = "heads.predictor."


def r16(t):
    return t.half().to(t.dtype)


def oracle_state_dict(precision):
    """the predictor's parameters in float64; fast precision: the conv weights the kernels pack to fp16, rounded (all but the
    edge fusion's last Conv1d, which mf_edge_head_add reads in fp32)"""
    sd = {}
    for k, v in syn.make_state_dict(0).items():
        if k.startswith(PREFIX) and v.is_floating_point():
            if precision == "fast" and v.dim() >= 3 and not k.endswith(".3.weight"):
                v = r16(v)
            sd[k] = v.double()
    return sd


def features(B, H, W, seed=0):
    gen = np.random.Generator(np.random.PCG64(seed))
    return torch.from_numpy(gen.standard_normal((B, 64, H, W)).astype(np.float32))


def edge_lists(W, H, pads):
    """per-image border lists [B,K,2] and lengths [B] (K = 2 (W + H) whatever the pad, so one plan serves every list)"""
    lists = [syn.edge_indices(W, H, pad) for pad in pads]
    return torch.stack([l[0] for l in lists]), torch.tensor([l[1] for l in lists], dtype=torch.long)


def targets_of(W, H, idx, lens, pads):
    B = idx.shape[0]
    tg = dict(edge_indices=idx, edge_len=lens, calib_P=[syn.KITTI_P2] * B,
              pad_size=torch.tensor(pads, dtype=torch.float32).view(B, 2), size=[(4 * W, 4 * H)] * B)
    return [t.to("cuda") for t in syn.make_param_lists(tg)]


def predictor_module(H, W):
    m = KeypointDetector(default_cfg(width=4 * W, height=4 * H))
    m.load_state_dict(syn.make_state_dict(0))
    return m.heads.predictor.cuda().eval()


def feature_rows(precision, x):
    """the predictor's input as a plan activation: hi/lo pair rows (strict) or fp16 rows (fast)"""
    B, C, H, W = x.shape
    P = engine.Plan("cuda", strict=precision == "strict")
    act = P.act(B, H, W, C)
    P.finalize()
    act.buf.copy_(to_rows_split(x) if precision == "strict" else to_rows(x))
    return act


def run_gpu(pred, act, targets):
    with torch.no_grad():
        out = pred(act, targets)
        plan = pred.last_plan
        rows = lambda a: a.nchw_view().float().cpu()[:, :, 0]           # [B,256,1,K+2] -> [B,256,K+2]
        g = dict(plan=plan, cls=out['cls'].cpu(), reg=out['reg'].cpu(), ea=rows(plan.ea), eb=rows(plan.eb),
                 mask=None if plan.hid_mask is None else plan.hid_mask.cpu())
    torch.cuda.synchronize()
    return g


def run_oracle(precision, x, idx, lens):
    torch.set_num_threads(min(32, os.cpu_count() or 1))
    taps = {}
    with torch.no_grad():
        out = mo.predictor(oracle_state_dict(precision), x.double(), idx, lens, taps=taps,
                           stored=r16 if precision == "fast" else None)
    return dict(logits=taps['cls_logits'], reg=out['reg'], ef=taps['edge_features'], e_cls=taps['e_cls'], e_off=taps['e_off'])


def mask_reference(idx, B, H, W):
    """the bilinear corners of every listed position, with edge_mask_kernel's float32 grid arithmetic (output map = W x H)"""
    e = idx.numpy().astype(np.float32)
    one, two = np.float32(1), np.float32(2)
    gx, gy = e[..., 0] / np.float32(W - 1) * two - one, e[..., 1] / np.float32(H - 1) * two - one
    ix, iy = ((gx + one) / two) * np.float32(W - 1), ((gy + one) / two) * np.float32(H - 1)
    x0, y0 = np.floor(ix).astype(np.int64), np.floor(iy).astype(np.int64)
    b = np.broadcast_to(np.arange(B)[:, None], x0.shape)
    mask = np.zeros((B, H, W), np.uint8)
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = y0 + dy, x0 + dx
            ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
            mask[b[ok], yy[ok], xx[ok]] = 1
    return mask


def head_errors(g, o, idx, lens):
    """every metric of the module docstring -> {name: error}"""
    e = {}
    p = g['cls'].double()
    assert (o['logits'].abs() < 9).all()                 # no heat-map value reaches the clamp: the logits are recoverable
    logits = torch.log(p) - torch.log1p(-p)
    e['cls'] = rel_err(logits, o['logits'])
    for key in mo.REG_KEYS:
        sl = mo.key2channel(key)
        e[key] = rel_err(g['reg'][:, sl], o['reg'][:, sl])
    off = mo.key2channel('3d_offset')
    e['edge_cls'] = e['edge_off'] = 0.0
    for b in range(idx.shape[0]):
        n = int(lens[b])
        xs, ys = idx[b, :n, 0], idx[b, :n, 1]
        for name, got, ref, term in (('edge_cls', logits[b], o['logits'][b], o['e_cls'][b, :, :n]),
                                     ('edge_off', g['reg'][b, off].double(), o['reg'][b, off], o['e_off'][b, :, :n])):
            err = (got[:, ys, xs] - ref[:, ys, xs]).abs().max().item() / term.abs().max().item()
            e[name] = max(e[name], err)
    rows = F.pad(o['ef'], (1, 1), mode='replicate')     # the Conv1d's replicate padding is part of the gathered rows
    for name, got, ref in (('ea', g['ea'], rows[:, :256]), ('eb', g['eb'], rows[:, 256:])):
        e[name] = rel_err(got, ref)
    return e


def check(precision, path, x, pred, act, idx, lens, pads, label):
    B, _, H, W = x.shape
    g = run_gpu(pred, act, targets_of(W, H, idx, lens, pads))
    names = {name for _, _, name in g['plan'].launches}
    assert names == PATH_LAUNCHES[path], names
    if path == "split":
        assert g['mask'] is None
    else:
        assert np.array_equal(g['mask'].view(B, H, W).numpy(), mask_reference(idx, B, H, W))
    xq = act.nchw_view().cpu() if precision == "strict" else x       # strict: the values the pair rows hold
    e = head_errors(g, run_oracle(precision, xq, idx, lens), idx, lens)
    print(precision, path, label, {k: "%.2e" % v for k, v in e.items()})
    tol = STRICT_TOL if precision == "strict" else FAST_TOL
    bad = {k: v for k, v in e.items() if v >= (FAST_ROW_TOL if precision == "fast" and k in ('ea', 'eb') else tol)}
    assert not bad, bad
    return g


def test_oracle_float64_matches_float32():
    """the predictor oracle runs in float64 (grid included) and agrees with its float32 run"""
    B, H, W, pads = 2, 10, 30, [(12, 6), (0, 0)]
    x = features(B, H, W, seed=3)
    idx, lens = edge_lists(W, H, pads)
    sd32 = {k: v for k, v in syn.make_state_dict(0).items() if k.startswith(PREFIX) and v.is_floating_point()}
    out = {}
    for dt in (torch.float32, torch.float64):
        taps = {}
        with torch.no_grad():
            r = mo.predictor({k: v.to(dt) for k, v in sd32.items()}, x.to(dt), idx, lens, taps=taps)
        assert r['cls'].dtype == r['reg'].dtype == taps['edge_features'].dtype == dt
        out[dt] = dict(logits=taps['cls_logits'], reg=r['reg'], ef=taps['edge_features'], e_cls=taps['e_cls'],
                       e_off=taps['e_off'])
    e = {k: rel_err(out[torch.float32][k], out[torch.float64][k]) for k in out[torch.float64]}
    print(e)
    assert max(e.values()) < 3e-6, e


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["strict", "fast"])
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_predictor_vs_oracle(case, precision):
    B, H, W, pads, strict_path, fast_path = case
    x = features(B, H, W)
    if precision == "fast":
        x = r16(x)
    pred = predictor_module(H, W)
    idx, lens = edge_lists(W, H, pads)
    assert len(set(lens.tolist())) == len(pads)                       # every image has its own edge_len
    check(precision, strict_path if precision == "strict" else fast_path, x, pred, feature_rows(precision, x), idx, lens, pads,
          "%dx%dx%d" % (B, H, W))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["strict", "fast"])
def test_plan_reuse_with_new_edge_lists(precision):
    """one plan, two batches of edge lists: the second run matches the oracle for the second lists (no stale hidden row,
    the mask is rebuilt before the head kernel reads it)"""
    B, H, W = 3, 12, 20
    x = features(B, H, W, seed=1)
    if precision == "fast":
        x = r16(x)
    pred = predictor_module(H, W)
    act = feature_rows(precision, x)
    path = "head2" if precision == "strict" else "fused"
    plans = []
    for pads in ([(0, 0), (8, 2), (19, 4)], [(19, 4), (0, 0), (8, 2)]):
        idx, lens = edge_lists(W, H, pads)
        plans.append(check(precision, path, x, pred, act, idx, lens, pads, "reuse %s" % (pads,))['plan'])
    assert plans[0] is plans[1]
