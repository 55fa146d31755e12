"""-m gpu: the decode kernels (csrc/mf_decode.cu) on the edge cases of oracle/decode_edge_cases.py — clamped plateaus that
send stage 1 to its radix-select fallback at every slab count, saturated ties across slabs, halo rows and classes, fewer
maxima than K, the candidate-count boundaries, degenerate geometry, thresholds, the fused sigmoid's clamp edges and signed
maps — against the CPU oracle (pinned to the unmodified reference by tests/test_decode_edges_host.py) and the reference's
own detections (tests/golden/decode_edges.npz).

Integer outputs and scores are compared with torch.equal, the result rows column by column (assert_decode_columns), and
stage 1's per-slab top-K in the workspace entry by entry, so a selection error that stage 2 would hide still fails."""
import math
import os
import types

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import decode_edge_cases as de
from oracle import monoflex_oracle as mo
from test_gpu_ops import assert_decode_columns

pytestmark = pytest.mark.gpu

OUTPUTS = ("scores", "inds", "clses", "ys", "xs", "pois", "result", "count", "depth_err", "proj", "min_unc")


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "decode_edges.npz")) as z:
        return {k: z[k] for k in z.files}


def limits():
    p = torch.cuda.get_device_properties(0)
    return p.multi_processor_count, p.shared_memory_per_block_optin


def decode(case, maps, apply_sigmoid, ws=None):
    from monoflex_b200.model.layers.utils import decode_detections
    return decode_detections(maps, case["reg"].cuda(), case["calib"].cuda(), case["pad"].cuda(), case["size"].cuda(),
                             torch.tensor(mo.DIM_MEAN).cuda(), case["K"], case["thresh"], apply_sigmoid, ws)


def heat_on_gpu(case):
    """the heat map the kernel selects from: the case's map, or sigmoid_hm of its logits computed on the GPU"""
    from monoflex_b200.model.layers.utils import sigmoid_hm
    return sigmoid_hm(case["maps"].clone().cuda()) if case["apply_sigmoid"] else case["maps"].cuda()


def bits(t):
    t = t.detach().contiguous().cpu()
    return t.view(torch.int32) if t.dtype == torch.float32 else t


def assert_same_outputs(a, b, n_ws):
    for k in OUTPUTS:
        assert torch.equal(bits(getattr(a, k)), bits(getattr(b, k))), k
    assert torch.equal(bits(a.ws_score[:n_ws]), bits(b.ws_score[:n_ws]))
    assert torch.equal(a.ws_idx[:n_ws].cpu(), b.ws_idx[:n_ws].cpu())


def slabs_of(case):
    B, C, H, W = case["maps"].shape
    S = de.slab_count(B, C, H, W, case["K"], *limits())
    assert S > 0
    return S, B * C * S * case["K"]


@pytest.mark.parametrize("name", de.CASES)
def test_decode_matches_oracle(name):
    case = de.build(name)
    heat = heat_on_gpu(case)
    ws = decode(case, heat, False)
    torch.cuda.synchronize()
    heat = heat.cpu()
    B, C, H, W = heat.shape
    K, thr = case["K"], case["thresh"]
    res, (sc, inds, cls_, ys, xs) = mo.post_process({"cls": heat, "reg": case["reg"]}, case["calib_P"], case["pad"],
                                                    case["size"].tolist(), thr, K)
    assert torch.equal(ws.inds.cpu(), inds)
    assert torch.equal(ws.clses.cpu(), cls_)
    assert torch.equal(ws.ys.cpu(), ys) and torch.equal(ws.xs.cpu(), xs)
    assert torch.equal(ws.scores.cpu(), sc)
    assert torch.equal(ws.pois.cpu(), mo.gather_pois(case["reg"], inds))
    for b in range(B):
        n = int(ws.count[b])
        assert n == res[b].shape[0]
        assert_decode_columns(ws.result[b, :n].cpu(), res[b])
    # stage 1 alone: each slab's top-K of its own pixel range
    S, n_ws = slabs_of(case)
    s_sc, s_ix = de.slab_topk(heat, K, S)
    assert torch.equal(ws.ws_idx[:n_ws].cpu().view(B, C, S, K), s_ix)
    assert torch.equal(ws.ws_score[:n_ws].cpu().view(B, C, S, K), s_sc)
    if case["apply_sigmoid"]:
        # the fused sigmoid: bit-identical in every output to sigmoid_hm followed by the unfused decode
        fused = decode(case, case["maps"].cuda(), True)
        assert_same_outputs(fused, ws, n_ws)


@pytest.mark.parametrize("name", de.GOLDEN_CASES)
def test_decode_matches_reference(name, gold):
    """the detections at or above the threshold are the reference's, as a set keyed by (class, flat index); each matched
    row agrees column by column"""
    case = de.build(name)
    assert str(gold[name + "/checksum"]) == de.checksum(case)
    ws = decode(case, heat_on_gpu(case), False)
    thr = torch.tensor(case["thresh"], dtype=torch.float32)
    for b in range(case["maps"].shape[0]):
        n = int(ws.count[b])
        mine = {(int(c), int(i)): r for r, (c, i) in enumerate(zip(ws.clses[b, :n].tolist(), ws.inds[b, :n].tolist()))}
        g_sc, g_inds, g_cls = (torch.from_numpy(gold["%s/%s" % (name, k)][b]) for k in ("scores", "inds", "clses"))
        keep = g_sc >= thr
        ref = {(int(c), int(i)): r for r, (c, i) in enumerate(zip(g_cls[keep].tolist(), g_inds[keep].tolist()))}
        assert set(mine) == set(ref)
        order = sorted(ref)
        g_res = torch.from_numpy(gold["%s/result_b%d" % (name, b)])
        assert torch.equal(ws.scores[b, [mine[k] for k in order]].cpu(), g_sc[keep][[ref[k] for k in order]])
        assert_decode_columns(ws.result[b, [mine[k] for k in order]].cpu(), g_res[[ref[k] for k in order]])


def test_score_equal_to_threshold_is_counted():
    case = de.build("thr_equal")
    ws = decode(case, heat_on_gpu(case), False)
    t = torch.tensor(0.7, dtype=torch.float32)
    assert float(t) < 0.7                       # float32(0.7) is below the double 0.7, so only a float32 >= counts it
    for b in range(2):
        n = int(ws.count[b])
        assert (ws.scores[b, :n].cpu() == t).sum() == 1 and (ws.scores[b, n:].cpu() < t).all()


def test_sigmoid_clamp_constants():
    from monoflex_b200.model.layers.utils import sigmoid_hm
    x = torch.tensor([-1e4, -100.0, -9.3, 9.3, 100.0, 1e4, 0.0])
    y = sigmoid_hm(x.clone().cuda()).cpu()
    lo, hi = torch.tensor(1e-4, dtype=torch.float32), torch.tensor(1 - 1e-4, dtype=torch.float32)
    assert torch.equal(y, torch.stack([lo, lo, lo, hi, hi, hi, torch.tensor(0.5)]))
    assert float(hi) == float(np.float32(1) - np.float32(1e-4))


def test_nms_hm_and_select_topk_on_signed_maps():
    from monoflex_b200.model.layers import utils as lu
    for name in ("signed_small", "signed_large"):
        case = de.build(name)
        h, K = case["maps"], case["K"]
        assert torch.equal(bits(lu.nms_hm(h.cuda())), bits(mo.nms_hm(h)))     # -0 where the reference has -0
        for got, ref in zip(lu.select_topk(h.cuda(), K=K), mo.select_topk(mo.nms_hm(h), K)):
            assert torch.equal(got.cpu(), ref)
    # nothing positive: the zeros (non-maxima) by index first, then the negative maximum
    h = -torch.arange(1, 26, dtype=torch.float32).view(1, 1, 5, 5)
    sc, inds, cls_, ys, xs = lu.select_topk(h.cuda(), K=25)
    assert inds.cpu().tolist() == [list(range(1, 25)) + [0]]
    assert sc.cpu().tolist() == [[0.0] * 24 + [-1.0]]


def test_reused_workspace_matches_fresh_workspaces():
    """every case through one set of buffers (left dirty by the previous case) equals a fresh, garbage-filled workspace"""
    from monoflex_b200.model.layers.utils import DecodeWorkspace
    dims = {n: (c["maps"].shape[0], c["maps"].shape[1], c["K"]) for n, c in ((n, de.build(n)) for n in de.CASES)}
    top = lambda f: max(f(*d) for d in dims.values())
    sizes = dict(ws_score=top(lambda B, C, K: B * C * K * 8), ws_idx=top(lambda B, C, K: B * C * K * 8),
                 scores=top(lambda B, C, K: B * K), inds=top(lambda B, C, K: B * K), clses=top(lambda B, C, K: B * K),
                 ys=top(lambda B, C, K: B * K), xs=top(lambda B, C, K: B * K), pois=top(lambda B, C, K: B * K * 50),
                 result=top(lambda B, C, K: B * K * 14), count=top(lambda B, C, K: B),
                 depth_err=top(lambda B, C, K: B * K), proj=top(lambda B, C, K: B * K * 2),
                 min_unc=top(lambda B, C, K: B * K))
    fresh0 = DecodeWorkspace(1, 1, 1, 50, "cuda")
    pool = {k: torch.full((n,), 7, dtype=getattr(fresh0, k).dtype, device="cuda") for k, n in sizes.items()}
    shapes = dict(ws_score=lambda B, C, K: (B * C * K * 8,), ws_idx=lambda B, C, K: (B * C * K * 8,),
                  pois=lambda B, C, K: (B, K, 50), result=lambda B, C, K: (B, K, 14), count=lambda B, C, K: (B,),
                  proj=lambda B, C, K: (B, K, 2))
    for name in de.CASES:
        case = de.build(name)
        B, C, K = dims[name]
        shared = types.SimpleNamespace(B=B, C=C, K=K, R=50)
        for k in sizes:
            shape = shapes.get(k, lambda B, C, K: (B, K))(B, C, K)
            setattr(shared, k, pool[k][:math.prod(shape)].view(shape))
        fresh = DecodeWorkspace(B, C, K, 50, "cuda")
        for k in sizes:
            getattr(fresh, k).fill_(-3)
        heat = heat_on_gpu(case)
        a = decode(case, heat, False, fresh)
        b = decode(case, heat, False, shared)
        assert b is shared
        assert_same_outputs(a, b, slabs_of(case)[1])


def test_rejects_unsupported_shapes():
    from monoflex_b200.model.layers import utils as lu

    def run(B, C, H, W, K):
        heat = torch.rand(B, C, H, W, device="cuda")
        lu.decode_detections(heat, torch.zeros(B, 50, H, W, device="cuda"), *lu._dummy_decode_inputs(heat), K=K,
                             thresh=0.2)
        torch.cuda.synchronize()

    with pytest.raises(RuntimeError, match="K=65"):
        run(1, 3, 24, 80, 65)
    with pytest.raises(RuntimeError, match=r"K=51 .*H\*W=50"):
        run(1, 3, 5, 10, 51)
    with pytest.raises(RuntimeError, match=r"K=17 .*H\*W=16"):
        lu.select_topk(torch.rand(1, 1, 4, 4, device="cuda"), K=17)
    with pytest.raises(RuntimeError, match="K=0"):
        run(1, 1, 4, 4, 0)
    with pytest.raises(RuntimeError, match="H\\*W=32769"):
        run(1, 1, 3, 10923, 50)
    run(1, 1, 5, 10, 50)                        # K = H*W is fine
