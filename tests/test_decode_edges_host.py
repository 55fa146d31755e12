"""CPU: the decode edge cases (oracle/decode_edge_cases.py) and the oracle's nms_hm / select_topk / post_process on them,
pinned to the UNMODIFIED reference (tests/golden/decode_edges.npz, oracle/make_golden_decode_edges.py). Every case
reaches the stage-1 path it is built for, and on an H100 (132 SMs, 227 KB of opt-in shared memory) the cases cover every
slab count S = 1 .. 8 and both paths. The GPU test (tests/test_gpu_decode_edges.py) then uses the oracle as its
reference."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import decode_edge_cases as de
from oracle import monoflex_oracle as mo
from test_gpu_ops import assert_decode_columns


@pytest.fixture(scope="module")
def gold():
    with np.load(os.path.join(GOLDEN, "decode_edges.npz")) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def summary():
    """name -> (S, set of stage-1 paths, checksum) on an H100, every case built once"""
    out = {}
    for name in de.CASES:
        case = de.build(name)
        B, C, H, W = case["maps"].shape
        out[name] = (de.slab_count(B, C, H, W, case["K"]), set(de.paths_of(case).reshape(-1).tolist()), de.checksum(case))
    return out


def test_slab_rule_matches_the_h100_splits():
    """mf_decode_detections' choice of S with 132 SMs, C = 3, K = 50"""
    got = {B: de.slab_count(B, 3, 96, 320, 50) for B in (1, 5, 6, 8, 11, 14, 16)}
    assert got == {1: 8, 5: 8, 6: 6, 8: 5, 11: 4, 14: 3, 16: 2}
    assert de.slab_count(6, 3, 112, 256, 50) == 7
    assert de.slab_count(2, 3, 24, 40, 50) == 1 and de.slab_count(2, 3, 32, 33, 50) == 2     # S = 1 needs H*W <= 1024
    assert de.slab_count(8, 3, 96, 320, 50, nsm=148) == 6
    assert de.slab_count(1, 3, 96, 320, 64) == 8 and de.slab_count(1, 3, 96, 320, 100) == 6   # C*S*K <= 2048
    assert de.slab_count(1, 1, 1, 32768 * 8, 50) == 0                                         # no split fits
    for HW, S in ((30720, 5), (1000, 7), (28672, 7)):
        r = de.slab_ranges(HW, S)
        assert r[0][0] == 0 and r[-1][1] == HW and all(a[1] == b[0] for a, b in zip(r, r[1:]))


def test_stage1_path_rule():
    heat = torch.zeros(1, 1, 64, 64)
    heat.view(-1)[:2049] = 0.5                      # a 2049-pixel plateau: every pixel a maximum
    assert de.stage1_paths(heat, 50, 1).tolist() == [[["radix"]]]
    heat.view(-1)[2048] = 0.0
    heat.view(-1)[2047] = 0.0
    assert de.stage1_paths(heat, 50, 1).tolist() == [[["fast"]]]
    heat = -torch.rand(1, 1, 8, 8) - 0.1            # negative maxima are not fast-path candidates
    assert de.stage1_paths(heat, 5, 1).tolist() == [[["radix"]]]


@pytest.mark.parametrize("name", de.CASES)
def test_builder_reaches_its_path_and_is_deterministic(name, summary, gold):
    case = de.build(name)                           # asserts the declared path
    S, paths, digest = summary[name]
    assert de.checksum(case) == digest, "the builder is not deterministic"
    assert S > 0
    assert paths == ({"fast", "radix"} if case["path"] == "mixed" else {case["path"]})
    if name in de.GOLDEN_CASES:
        assert str(gold[name + "/checksum"]) == digest, "the builder drifted from tests/golden/decode_edges.npz"


def test_cases_cover_every_slab_count_and_both_paths(summary):
    assert {s for s, _, _ in summary.values()} == set(range(1, 9))
    assert set().union(*(p for _, p, _ in summary.values())) == {"fast", "radix"}
    for S in range(1, 9):                           # the clamped background at every S, the radix path from S = 2 on
        s, paths, _ = summary["clamp_s%d" % S]
        assert s == S and (S == 1 or "radix" in paths)


def test_counts_case_puts_the_boundaries_in_single_slabs():
    case = de.build("counts")
    B, C, H, W = case["maps"].shape
    S = de.slab_count(B, C, H, W, case["K"])
    pos = (mo.nms_hm(case["maps"]) > 0).reshape(C, H * W)
    n = [[int(pos[c, lo:hi].sum()) for lo, hi in de.slab_ranges(H * W, S)] for c in range(C)]
    K = case["K"]
    assert {K - 1, K, 2048, 2049} <= set(sum(n, []))
    paths = de.paths_of(case)[0]
    for c in range(C):
        for s in range(S):
            assert paths[c, s] == ("fast" if K <= n[c][s] <= 2048 else "radix")


def test_golden_cases_have_at_most_k_detections():
    for name in de.GOLDEN_CASES:
        case = de.build(name)
        assert int(de.n_above(case).max()) <= case["K"]


def keyed(scores, inds, clses, thresh):
    """(class, flat index) -> rank of every top-k entry at or above the threshold"""
    keep = scores >= torch.tensor(thresh, dtype=torch.float32)
    return {(int(c), int(i)): r for r, (c, i) in enumerate(zip(clses[keep].tolist(), inds[keep].tolist()))}


@pytest.mark.parametrize("name", de.GOLDEN_CASES)
def test_oracle_matches_the_reference(name, gold):
    case = de.build(name)
    heat, reg, K, thr = case["maps"], case["reg"], case["K"], case["thresh"]
    res, (sc, inds, cls_, ys, xs) = mo.post_process({"cls": heat, "reg": reg}, case["calib_P"], case["pad"],
                                                    case["size"].tolist(), thr, K)
    g_sc, g_inds, g_cls = (torch.from_numpy(gold["%s/%s" % (name, k)]) for k in ("scores", "inds", "clses"))
    for b in range(heat.shape[0]):
        mine, ref = keyed(sc[b], inds[b], cls_[b], thr), keyed(g_sc[b], g_inds[b], g_cls[b], thr)
        assert set(mine) == set(ref)
        g_res = torch.from_numpy(gold["%s/result_b%d" % (name, b)])
        assert res[b].shape == g_res.shape and g_res.shape[0] == len(ref)
        order = sorted(ref)
        assert torch.equal(sc[b, [mine[k] for k in order]], g_sc[b, [ref[k] for k in order]])
        assert_decode_columns(res[b][[mine[k] for k in order]], g_res[[ref[k] for k in order]])
    # outside the ties the two agree entry by entry: the oracle's tie rule is one of the orders torch.topk may return
    assert torch.equal(sc, g_sc)
