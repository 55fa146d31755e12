"""TEST TOOLING — heat maps that drive the decode kernels (csrc/mf_decode.cu) onto each of their stage-1 paths, slab splits
and tie rules.

Stage 1 splits every (image, class) plane into S slabs (`slab_count`, a copy of mf_decode_detections' rule) and selects each
slab's top-K in one of two ways: rank by counting when the slab holds between k_eff = min(K, slab size) and S1_CAND
strictly positive local maxima ('fast'), otherwise an MSB-first radix select plus a 256-key bitonic sort ('radix').
The synthetic N(-3, 1.5) logits of synthetic.make_head_logits only ever take the fast path. The families here:

  clamp_s1 .. clamp_s8  logits <= -9.3 (heat exactly float32(1e-4) after sigmoid_hm) with M in {0, 1, K-1, K, K+1, 200}
                        Gaussian objects of assorted heights per plane, at the shapes whose slab count is S = 1 .. 8 on
                        132 SMs; a clamped background makes every pixel a maximum, so each slab of more than 2048 pixels
                        takes the radix path (S = 1, 24x40, the fast one)
  clamp_b2              the clamped background at 96x320, B = 2, as a heat map (the reference fixture's case)
  ties_*                object cores of 2x2 or more at exactly float32(1 - 1e-4): one pixel saturated in two or three
                        classes, tied maxima on the last pixel of a slab and the first of the next, tied and larger maxima
                        across the one-row halo of a slab boundary
  few_*                 fewer positive maxima than K: one blob per plane on a strictly monotone background, constant planes
                        (zero and positive); the radix path then fills with zero scores by index
  counts                exactly K-1, K, 2048 and 2049 positive maxima in one slab
  geom_*                H = 1, W = 1, H*W = K, H*W = 32768 with maxima at flat index 0 and 32767, C = 1 / 2 / 3, K = 1 / 50 / 64
  thr_*                 a selected score exactly float32(thresh) (thresh 0.7 rounds down in float32), a threshold above
                        every score, a threshold of 0
  sigmoid_edges         logits on both sides of both clamp edges, including values whose sigmoid rounds onto the bound
  signed_*              signed maps with negative maxima, -0 and all-negative planes, as the public nms_hm / select_topk
                        accept them

Every case declares the stage-1 path it is built to reach ('fast', 'radix' or 'mixed' = both occur) and `build` checks
it on the heat map (sigmoid_hm on the CPU for logit cases). Deterministic: numpy PCG64 seeds only."""
import hashlib

import numpy as np
import torch

from monoflex_b200 import synthetic as syn
from oracle import monoflex_oracle as mo

S1_THREADS, S1_CAND, S2_KEYS, MAX_SLABS = 1024, 2048, 2048, 8
H100_SMS, H100_SMEM_OPTIN = 132, 227 * 1024
LO, HI = np.float32(1e-4), np.float32(1 - 1e-4)          # sigmoid_hm's clamp bounds (layers/utils.py:39-43)
R = 50


# -------------------------------------------------------------------------------------- mf_decode_detections' rules
def _cdiv(a, b):
    return -(-a // b)


def slab_count(B, C, H, W, K, nsm=H100_SMS, smem_max=H100_SMEM_OPTIN):
    """mf_decode_detections' slab rule: the S <= 8 minimising waves x (items per thread + 6) among the splits whose slab (score
    keys + staged pixels with the one-row halo) fits the opt-in shared memory and whose C*S*K candidates fit stage 2.
    0 = no split fits."""
    HW = H * W
    S, best = 0, 1 << 30
    for s in range(1, MAX_SLABS + 1):
        if C * s * K > S2_KEYS:
            break
        items = _cdiv(_cdiv(HW, s), S1_THREADS)
        if items * S1_THREADS * 4 + (_cdiv(HW, s) + 2 * W + 2) * 4 > smem_max:
            continue
        cost = _cdiv(B * C * s, nsm) * (items + 6)
        if cost < best:
            best, S = cost, s
    return S


def slab_ranges(HW, S):
    """[(lo, hi)] pixel range of each slab of a plane"""
    chunk = _cdiv(HW, S)
    return [(s * chunk, min(HW, s * chunk + chunk)) for s in range(S)]


def sigmoid_hm(logits):
    return torch.sigmoid(logits).clamp(min=1e-4, max=1 - 1e-4)


def heat_of(case):
    return sigmoid_hm(case["maps"]) if case["apply_sigmoid"] else case["maps"]


def stage1_paths(heat, K, S):
    """[B, C, S] array of 'fast' / 'radix': the path each (image, class, slab) takes, from its count of strictly positive
    maxima after the 3x3 NMS"""
    B, C, H, W = heat.shape
    pos = (mo.nms_hm(heat) > 0).reshape(B, C, H * W)
    out = np.empty((B, C, S), object)
    for s, (lo, hi) in enumerate(slab_ranges(H * W, S)):
        n = pos[:, :, lo:hi].sum(2).numpy()
        out[:, :, s] = np.where((n >= min(K, hi - lo)) & (n <= S1_CAND), "fast", "radix")
    return out


def paths_of(case, nsm=H100_SMS, smem_max=H100_SMEM_OPTIN):
    B, C, H, W = case["maps"].shape
    return stage1_paths(heat_of(case), case["K"], slab_count(B, C, H, W, case["K"], nsm, smem_max))


def reached(paths):
    kinds = set(paths.reshape(-1).tolist())
    return "mixed" if len(kinds) == 2 else kinds.pop()


def slab_topk(heat, K, S):
    """the top-K of every slab's pixel range of the NMS-ed map under (score desc, index asc), padded with 0 / -1 when the
    slab is narrower than K -> (scores [B, C, S, K] float32, idx [B, C, S, K] int32): what stage 1 leaves in ws_score /
    ws_idx"""
    B, C, H, W = heat.shape
    flat = mo.nms_hm(heat).reshape(B, C, H * W)
    sc = torch.zeros(B, C, S, K)
    ix = torch.full((B, C, S, K), -1, dtype=torch.int32)
    for s, (lo, hi) in enumerate(slab_ranges(H * W, S)):
        n = min(K, max(hi - lo, 0))
        if n == 0:
            continue
        order = torch.sort(-flat[:, :, lo:hi], dim=2, stable=True).indices[:, :, :n]
        sc[:, :, s, :n] = flat[:, :, lo:hi].gather(2, order)
        ix[:, :, s, :n] = (order + lo).int()
    return sc, ix


# ------------------------------------------------------------------------------------------------ map builders
def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _clamped(rng, shape):
    """logits in [-20, -9.3]: sigmoid_hm maps every one to exactly float32(1e-4)"""
    return rng.uniform(-20.0, -9.3, shape)


def _objects(rng, plane, m, saturate=0.3, high=None):
    """m Gaussian bumps on one logit plane [H, W] (in place, max with what is there), peak logits from -2 to 14: a share
    `saturate` of them above 9.3, whose cores clamp to 1 - 1e-4. With `high` = n, only the first n peak above 2 (up to
    10.5, narrow) and the rest stay in [-2, 2]."""
    H, W = plane.shape
    yy, xx = np.mgrid[0:H, 0:W]
    for i in range(m):
        cy, cx = rng.integers(H), rng.integers(W)
        if high is not None:
            peak, sig = (rng.uniform(3.0, 10.5), rng.uniform(0.7, 1.5)) if i < high else (rng.uniform(-2.0, 2.0), 2.0)
        else:
            peak = rng.uniform(9.5, 14.0) if rng.uniform() < saturate else rng.uniform(-2.0, 9.0)
            sig = rng.uniform(0.7, 3.0)
        bump = peak - 4.0 * ((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * sig * sig)
        np.maximum(plane, bump, out=plane)


def _heat_bg(rng, shape, top=0.5):
    """sigmoid_hm of N(-3, 1.5) logits (make_head_logits' distribution), capped at `top`"""
    return np.minimum(sigmoid_hm(torch.from_numpy(rng.standard_normal(shape) * 1.5 - 3.0).float()).numpy(), top)


def _case(name, maps, K, thresh, path, apply_sigmoid=False, seed=0, family=None):
    maps = torch.from_numpy(np.ascontiguousarray(maps, np.float32))
    B, C, H, W = maps.shape
    rng = _rng(1000 + seed)
    reg = torch.from_numpy(rng.standard_normal((B, R, H, W), dtype=np.float32) * np.float32(0.5))
    tg = syn.make_targets(B, W, H)
    calib = torch.tensor([list(mo.calib_from_P(P).values()) for P in tg["calib_P"]], dtype=torch.float32)
    return dict(name=name, family=family or name.split("_")[0], maps=maps, reg=reg, calib_P=tg["calib_P"], calib=calib,
                pad=tg["pad_size"].clone(), size=torch.tensor(tg["size"], dtype=torch.float32), K=K, thresh=thresh,
                apply_sigmoid=apply_sigmoid, path=path)


# (B, H, W) -> S on 132 SMs with C = 3, K = 50 (see slab_count)
CLAMP_SHAPES = {1: (2, 24, 40), 2: (16, 96, 320), 3: (14, 96, 320), 4: (11, 96, 320), 5: (8, 96, 320), 6: (6, 96, 320),
                7: (6, 112, 256), 8: (5, 96, 320)}


def _clamp(S):
    B, H, W = CLAMP_SHAPES[S]
    K = 50
    rng = _rng(100 + S)
    lg = _clamped(rng, (B, 3, H, W))
    ms = (0, 1, K - 1, K, K + 1, 200)
    for p in range(B * 3):                        # every M on some plane, in a different order for every S
        _objects(rng, lg[p // 3, p % 3], ms[(p + S) % len(ms)])
    # a 960-pixel slab holds fewer than S1_CAND pixels, so at S = 1 even the all-maxima plateau takes the fast path; in the
    # slabs of 6 to 8 a plane with 200 objects leaves fewer than S1_CAND plateau pixels, and those take it too
    path = "fast" if S == 1 else "radix" if S <= 5 else "mixed"
    return _case("clamp_s%d" % S, lg, K, 0.2, path, apply_sigmoid=True, seed=S, family="clamp")


def _clamp_b2():
    """96x320, B = 2 as a heat map: at most three objects per plane peak above heat 0.88 (some saturated), so the threshold
    0.9 keeps at most K scores at or above it per image"""
    rng = _rng(120)
    lg = _clamped(rng, (2, 3, 96, 320))
    for p, m in enumerate((0, 1, 49, 50, 51, 200)):
        _objects(rng, lg[p // 3, p % 3], m, high=3)
    return _case("clamp_b2", sigmoid_hm(torch.from_numpy(lg).float()).numpy(), 50, 0.9, "mixed", seed=20, family="clamp")


def _ties(name, B, H, W, clamped, seed, thresh):
    """2x2 and 3x2 cores at exactly 1 - 1e-4, placed on slab boundaries, in the halo rows and in several classes at once"""
    rng = _rng(seed)
    C, K = 3, 50
    if clamped:
        heat = np.full((B, C, H, W), LO, np.float32)
    else:
        heat = _heat_bg(rng, (B, C, H, W))
    flat = heat.reshape(B, C, H * W)
    S = slab_count(B, C, H, W, K)
    bounds = [lo for lo, _ in slab_ranges(H * W, S)][1:]
    for b in range(B):
        # the same saturated 2x2 core in classes (0, 1, 2) and (0, 2)
        for classes, (y, x) in (((0, 1, 2), (5, 7)), ((0, 2), (H // 2, W // 3))):
            for c in classes:
                heat[b, c, y:y + 2, x:x + 2] = HI
        for j, lo in enumerate(bounds):
            c = (b + j) % C
            y, x = divmod(lo, W)
            # tied maxima on the last pixel of slab j and the first of slab j + 1 (same row or across a row end)
            flat[b, c, lo - 1] = HI
            flat[b, c, lo] = HI
            # a 3x2 saturated core straddling the boundary row: tied maxima on both sides of the one-row halo
            x2 = (x + W // 2) % (W - 2)
            c2 = (c + 1) % C
            heat[b, c2, max(y - 1, 0):y + 1, x2:x2 + 3] = HI
            # a larger value in the halo row above the slab's first row suppresses the pixel below it, and vice versa
            x3 = (x2 + 7) % (W - 1)
            heat[b, c, y, x3] = np.float32(0.95)
            heat[b, c, max(y - 1, 0), x3] = np.float32(0.96)
            heat[b, c, min(y + 1, H - 1), x3] = np.float32(0.97) if y + 1 < H else heat[b, c, y, x3]
    return _case(name, heat, K, thresh, "radix" if clamped and H * W > 2 * S1_CAND else "fast", seed=seed, family="ties")


def _few(name, B, C, H, W, seed, constant=False):
    """one smooth blob per plane on a strictly monotone background (increasing with the flat index, so its only maximum
    is the last pixel), or constant planes: fewer than K positive maxima per slab"""
    rng = _rng(seed)
    idx = np.arange(H * W, dtype=np.float64).reshape(H, W)
    heat = np.empty((B, C, H, W), np.float32)
    yy, xx = np.mgrid[0:H, 0:W]
    for b in range(B):
        for c in range(C):
            p = b * C + c
            if constant and p % 3 == 0:
                heat[b, c] = 0.0
                continue
            if constant and p % 3 == 1:
                heat[b, c] = LO
                continue
            bg = 1e-3 + 1e-7 * idx if p % 2 == 0 else 1e-3 + 1e-7 * (idx[::-1, ::-1])
            cy, cx = rng.integers(2, H - 2), rng.integers(2, W - 2)
            blob = rng.uniform(0.3, 0.95) * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * 2.0 ** 2))
            heat[b, c] = np.maximum(bg, blob)
    return _case(name, heat, 50, 0.2, "radix", seed=seed, family="few")


def _counts():
    """96x320, B = 1, C = 3 (S = 8, 3840-pixel slabs) on a zero background: isolated distinct peaks for K - 1 and K maxima,
    equal-valued runs of flat indices (a plateau: every pixel a maximum) for 2048 and 2049; other slabs empty"""
    H, W, K = 96, 320, 50
    rng = _rng(130)
    heat = np.zeros((1, 3, H, W), np.float32)
    flat = heat.reshape(3, H * W)
    sl = slab_ranges(H * W, slab_count(1, 3, H, W, K))
    plan = {0: ((0, K - 1), (1, K), (2, 2048), (3, 2049)), 1: ((4, 2049), (6, K)), 2: ((5, 2048), (7, K - 1))}
    for c, slabs in plan.items():
        for s, n in slabs:
            lo, hi = sl[s]
            if n <= K:
                # peaks two rows apart in every other column: no two in one 3x3 window
                ys, xs = np.divmod(np.arange(n) * 2, W)
                pix = lo + W + (ys * 2) * W + xs
                flat[c, pix] = rng.uniform(0.05, 0.95, n).astype(np.float32)
            else:
                start = lo + (hi - lo - n) // 2
                flat[c, start:start + n] = np.float32(0.5)
    return _case("counts", heat, K, 0.2, "mixed", seed=30, family="counts")


def _geom(name, B, C, H, W, K, seed, path, peaks=()):
    rng = _rng(seed)
    heat = _heat_bg(rng, (B, C, H, W), top=0.9)
    for b, c, i, v in peaks:
        heat.reshape(B, C, H * W)[b, c, i] = v
    return _case(name, heat, K, 0.2, path, seed=seed, family="geom")


def _thr(name, thresh, seed):
    """24x80, B = 2: the map of make_head_logits; one local maximum per image set to exactly float32(0.7)"""
    rng = _rng(seed)
    heat = _heat_bg(rng, (2, 3, 24, 80), top=0.69)
    heat[0, 1, 10, 30] = np.float32(0.7)
    heat[1, 2, 3, 79] = np.float32(0.7)
    heat[1, 0, 20, 5] = np.float32(0.8)
    return _case(name, heat, 50, thresh, "fast", seed=seed, family="thr")


def _sigmoid_edges():
    """logits straddling both clamp edges (+-9.2103..., where sigmoid crosses 1e-4 / 1 - 1e-4) on a clamped background;
    the objects' peaks land on both sides of the upper edge"""
    rng = _rng(140)
    B, C, H, W = 1, 3, 96, 320
    lg = _clamped(rng, (B, C, H, W))
    edge = np.float32(9.2103404)
    near = np.float32(edge + np.arange(-40, 41, dtype=np.float32) * np.float32(2e-6))
    flat = lg.reshape(B * C, H * W)
    for p in range(B * C):
        pix = rng.choice(H * W, size=2 * near.size, replace=False)
        flat[p, pix[:near.size]] = -near                       # lower edge: at, above and below -9.2103
        flat[p, pix[near.size:]] = near                        # upper edge
        flat[p, rng.choice(H * W, size=8, replace=False)] = rng.uniform(-9.3, 9.3, 8)
    return _case("sigmoid_edges", lg, 50, 0.2, "radix", apply_sigmoid=True, seed=40, family="sigmoid")


def _signed(name, B, C, H, W, seed, path):
    """signed maps: N(0, 1) with a -0 plane region, an all-negative plane and a plane with a few positive pixels"""
    rng = _rng(seed)
    heat = rng.standard_normal((B, C, H, W)).astype(np.float32)
    heat[0, 0, :3] = np.float32(-0.0)
    heat[0, 0, 3, :5] = np.float32(0.0)
    heat[0, C - 1] = -np.abs(heat[0, C - 1])
    if B > 1:
        heat[1, 0] = -np.abs(heat[1, 0])
        heat[1, 0].reshape(-1)[rng.choice(H * W, size=7, replace=False)] = rng.uniform(0.1, 2.0, 7)
    return _case(name, heat, 50, 0.0, path, seed=seed, family="signed")


_BUILDERS = {"clamp_s%d" % s: (lambda s=s: _clamp(s)) for s in range(1, 9)}
_BUILDERS.update({
    "clamp_b2": _clamp_b2,
    "ties_fast": lambda: _ties("ties_fast", 2, 96, 320, False, 150, 0.2),      # S = 8
    "ties_clamped": lambda: _ties("ties_clamped", 3, 96, 320, True, 151, 0.2),  # S = 8, radix
    "ties_b2": lambda: _ties("ties_b2", 2, 32, 64, True, 152, 0.5),             # S = 2, 1024-pixel slabs: fast
    "few_blob": lambda: _few("few_blob", 2, 3, 32, 64, 160),
    "few_constant": lambda: _few("few_constant", 2, 3, 96, 320, 161, constant=True),
    "counts": _counts,
    "geom_h1": lambda: _geom("geom_h1", 2, 3, 1, 300, 50, 170, "fast"),
    "geom_w1": lambda: _geom("geom_w1", 2, 2, 300, 1, 50, 171, "fast"),
    "geom_hw_eq_k": lambda: _geom("geom_hw_eq_k", 3, 1, 8, 8, 64, 172, "radix"),
    "geom_k1": lambda: _geom("geom_k1", 2, 3, 24, 80, 1, 173, "fast"),
    "geom_32768": lambda: _geom("geom_32768", 2, 2, 128, 256, 64, 174, "fast",
                                peaks=((0, 0, 0, 0.99), (0, 1, 32767, 0.99), (1, 0, 32767, 0.95), (1, 1, 0, 0.97),
                                       (1, 1, 32767, 0.97))),
    "thr_equal": lambda: _thr("thr_equal", 0.7, 180),
    "thr_above": lambda: _thr("thr_above", 0.9, 181),
    "thr_zero": lambda: _thr("thr_zero", 0.0, 182),
    "sigmoid_edges": _sigmoid_edges,
    "signed_small": lambda: _signed("signed_small", 2, 3, 24, 80, 190, "mixed"),
    "signed_large": lambda: _signed("signed_large", 2, 2, 96, 320, 191, "mixed"),
})
CASES = tuple(_BUILDERS)
GOLDEN_CASES = ("clamp_b2", "ties_b2", "few_blob")      # recorded from the reference


def build(name):
    """-> dict(name, family, maps [B, C, H, W] (logits when apply_sigmoid), reg [B, 50, H, W], calib_P, calib [B, 6] (f_u,
    f_v, c_u, c_v, b_x, b_y), pad [B, 2], size [B, 2], K, thresh, apply_sigmoid, path); checks the declared path"""
    case = _BUILDERS[name]()
    got = reached(paths_of(case))
    assert got == case["path"], "%s reaches %s, built for %s" % (name, got, case["path"])
    return case


def checksum(case):
    """sha256 over every input of a case in a fixed order"""
    h = hashlib.sha256()
    for k in ("maps", "reg", "calib", "pad", "size"):
        h.update(k.encode())
        h.update(np.ascontiguousarray(case[k].numpy()).tobytes())
    h.update(np.asarray(case["calib_P"], np.float64).tobytes())
    h.update(repr((case["K"], float(case["thresh"]), bool(case["apply_sigmoid"]))).encode())
    return h.hexdigest()


def n_above(case, heat=None):
    """per image, the number of local maxima at or above the threshold over all classes"""
    heat = heat_of(case) if heat is None else heat
    return above_threshold(mo.nms_hm(heat).reshape(heat.shape[0], -1), case["thresh"])


def above_threshold(scores, thresh):
    """per image, the number of scores at or above the threshold in float32 (the comparison of the kernel and of the
    reference's `scores >= det_threshold` on a float32 tensor)"""
    return (scores >= torch.tensor(thresh, dtype=torch.float32)).sum(-1)
