"""TEST TOOLING — loss inputs that put chosen objects on the branches of the fused training loss (csrc/mf_loss.cu).

The present loss tests feed predictions that are nudged towards their labels (synthetic.make_train_predictions), so the
clamps, relus, ties, wraps and degenerate normalisers of the loss are never reached. `build(case)` starts from the same
synthetic labels, gives every labelled centre a sane regression vector and then overwrites chosen objects' vectors and
labels so that each of them sits on one branch:

  kinks        B=4: direct depth and uncertainties clamped (and exactly on the uncertainty bound), key-point heights
               negative / tiny / in range, an invalid key-point-depth group on an in-range depth, 2D distances below
               zero, equal to the fp32 label distances (min/max ties), disjoint and enclosing 2D boxes, tied bin logits,
               a zero and a 1e-20 bin offset (F.normalize eps), roty wrapping past +pi and -pi, a truncated object far
               off its offset, key points and 3D offset exactly on their labels (abs at 0), two objects on one centre
               pixel, objects at the map corners;
  calib        B=5: a different P and pad_size per image, images 0 and 2 empty (key-point depths take f_u by rank);
  full         B=7: image 0 has all 40 slots (three share a centre), image 6 one object in slot 39 (slot index > 256,
               the strided loop of the one-CTA forward), images 1-5 empty;
  full_b1      image 0 of `full` alone (the batch-size-1 calibration branch);
  all_trunc    every object truncated: offset_loss is the mean of an empty set (NaN), nothing else is;
  no_valid_kd  no valid key-point-depth group: the logged keypoint_depth_loss is NaN, the loss is finite;
  no_object, no_box2d   kernel-only deviations (the reference crashes / raises NameError), no fixture.

Every comparison the loss branches on that is not a deliberate exact tie is kept at least MARGIN (relative) from its
boundary, so that float32 and float64 evaluations take the same branch; `check_margins` asserts this in float64 and the
builder calls it on every case. Deterministic: fixed seeds, no dependence on anything but numpy / torch arithmetic."""
import hashlib
import math

import numpy as np
import torch

from monoflex_b200 import synthetic as syn

CASES = ("kinks", "calib", "full", "full_b1", "all_trunc", "no_valid_kd")   # recorded from the reference
KERNEL_ONLY = ("no_object", "no_box2d")
MARGIN = 1e-3
OUT_W, OUT_H, M = 320, 96, syn.MAX_OBJECTS
PER_OBJECT = ("cls_ids", "target_centers", "bboxes", "keypoints", "keypoints_depth_mask", "dimensions", "locations",
              "rotys", "alphas", "offset_3D", "orientations", "reg_mask", "trunc_mask", "reg_weight")
CENTERS = (0.0, math.pi / 2, math.pi, -math.pi / 2)


def f32(x):
    return np.float32(x)


# ------------------------------------------------------------------------------------------------ labels
def _clear(f, i):
    for k in PER_OBJECT:
        f[k][i] = 0


def _copy(dst, j, src, i):
    for k in PER_OBJECT:
        dst[k][j] = src[k][i]


def _objects(f):
    return [int(i) for i in np.nonzero(f["reg_mask"])[0]]


def _pool(n, seed):
    """n labelled objects (image, slot) drawn from synthetic images without empty ones"""
    fs = syn.make_train_targets(max(4, n // 3), seed=seed, empty_image=-1)
    return [(f, i) for f in fs for i in _objects(f)][:n]


def _free_pixel(f, x, y, used):
    while (x, y) in used:
        x = x + 1 if x + 1 < f["hm"].shape[2] - 1 else 1
    return x, y


# ------------------------------------------------------------------------------------------------ predictions
def _sane(rng, f, i):
    """regression vector near the object's label (the make_train_predictions recipe), float64"""
    p = rng.standard_normal(50) * 0.5
    x, y = f["target_centers"][i]
    p[6:26] = f["keypoints"][i, :, :2].reshape(-1) + rng.standard_normal(20) * 0.3
    p[4:6] = f["offset_3D"][i] + rng.standard_normal(2) * 0.1
    bx = f["bboxes"][i]
    if bx[2] > bx[0] and bx[3] > bx[1]:
        p[0:4] = (np.array([x - bx[0], y - bx[1], bx[2] - x, bx[3] - y]) + 0.5) * rng.uniform(0.7, 1.3, 4)   # > 0
    p[29:32] = rng.standard_normal(3) * 0.1
    p[48] = -math.log(float(f["locations"][i, 2]) * math.exp(rng.normal(0, 0.1)))
    return p


def _set_heights(p, h):
    """key-point y offsets with heights ky(8)-ky(9), ky(0)-ky(4), ky(2)-ky(6), ky(1)-ky(5), ky(3)-ky(7) = h[0..4]"""
    for (a, b), v in zip(((8, 9), (0, 4), (2, 6), (1, 5), (3, 7)), h):
        p[7 + 2 * b] = p[7 + 2 * a] - v


def _heights_for_depth(f, i, p, fu, z):
    """key-point height (feature-map pixels) at which the key-point depth of object i equals z"""
    cls = int(f["cls_ids"][i])
    fh = fu * math.exp(float(f32(p[30]))) * syn.DIM_MEAN[cls][1]
    return (fh / z - 1e-3) / 4.0


# recipes: fn(p, f, i, ctx) edits the vector / labels of one object and returns the set of deliberate exact ties it
# builds (names of check_margins' comparisons)
def r_depth_low(p, f, i, ctx):
    p[48] = 6.0                                   # exp(-6) = 0.0025 -> clamp at 0.1
    return set()


def r_depth_high(p, f, i, ctx):
    p[48] = -6.0                                  # exp(6) = 403 -> clamp at 100
    return set()


def r_dunc(v):
    def r(p, f, i, ctx):
        p[49] = v
        return {"clamp_u0_lo"} if v == -10.0 else set()
    r.__name__ = "r_dunc_%g" % v
    return r


def r_kunc_clamped(p, f, i, ctx):
    p[26], p[27] = 12.0, -12.0
    return set()


def r_unc_tie(p, f, i, ctx):
    p[49], p[26], p[27], p[28] = 12.0, 10.0, 11.0, 10.5      # all four clamp to exactly 10: exp ties, first arg-min
    return {"clamp_u1_hi", "argmin_unc"}


def r_heights_negative(p, f, i, ctx):
    _set_heights(p, [-0.6, -0.8, -0.5, -0.7, -0.9])        # relu = 0: depth = f*h/1e-3, clamped at 100
    return set()


def r_heights_tiny(p, f, i, ctx):
    _set_heights(p, [0.01] * 5)                            # depth ~ 2.6e4 in (100, 1e5): clamped at 100
    return set()


def r_heights_inside(p, f, i, ctx):
    z = float(f["locations"][i, 2])
    _set_heights(p, [_heights_for_depth(f, i, p, ctx["fu_kp"], z * s) for s in (0.8, 1.15, 1.2, 0.85, 0.9)])
    return set()


def r_invalid_kd(p, f, i, ctx):
    z = float(f["locations"][i, 2])
    _set_heights(p, [_heights_for_depth(f, i, p, ctx["fu_kp"], z * s) for s in (0.9, 1.1, 1.1, 0.95, 0.95)])
    f["keypoints_depth_mask"][i] = (1, 0, 1)               # group 02 in range but invalid: detached
    return set()


def _box_about_centre(f, i):
    x, y = f["target_centers"][i]
    if not (f["bboxes"][i, 2] > f["bboxes"][i, 0] and f["bboxes"][i, 3] > f["bboxes"][i, 1]):
        f["bboxes"][i] = (x - 3.25, y - 2.5, x + 4.5, y + 3.75)
    b = f["bboxes"][i]
    return [f32(np.float32(x) - b[0]), f32(np.float32(y) - b[1]), f32(b[2] - np.float32(x)), f32(b[3] - np.float32(y))]


def r_box_relu(p, f, i, ctx):
    t = _box_about_centre(f, i)
    p[0:4] = [-0.7, t[1] * 0.8, t[2] * 1.2, t[3] * 0.9]
    return set()


def r_box_tie(p, f, i, ctx):
    p[0:4] = _box_about_centre(f, i)                       # exactly the fp32 label distances: every min / max ties
    return {"minmax_2d0", "minmax_2d1", "minmax_2d2", "minmax_2d3"}


def r_box_disjoint(p, f, i, ctx):
    x, y = f["target_centers"][i]
    f["bboxes"][i] = (x + 1.5, y - 2.0, x + 6.0, y + 3.0)  # label box right of the centre; predicted box left of it
    p[0:4] = [2.0, 1.5, 1.0, 2.5]
    return set()


def r_box_encloses(p, f, i, ctx):
    t = _box_about_centre(f, i)
    p[0:4] = [v * 1.5 + 0.5 for v in t]
    return set()


def _ori_on(f, i):
    return [k for k in range(4) if f["orientations"][i, k] == 1]


def _win(p, k):
    """bin k wins the arg-max clearly"""
    p[32:40:2], p[33:40:2] = 1.0, -1.0
    p[32 + 2 * k], p[33 + 2 * k] = -1.5, 2.0


def r_bin_tie(p, f, i, ctx):
    p[32:40:2], p[33:40:2] = 0.25, 0.75                    # four equal bins: the first wins
    for k in range(4):
        a = -1.2 + 0.7 * k
        p[40 + 2 * k], p[41 + 2 * k] = math.sin(a) * 1.3, math.cos(a) * 1.3
    return {"argmax_bin"}


def _eps(v):
    def r(p, f, i, ctx):
        k = _ori_on(f, i)[0]
        f["orientations"][i, 4 + k] = 0.3
        _win(p, (k + 1) % 4)                               # atan2 never sees the zero vector
        p[40 + 2 * k], p[41 + 2 * k] = v, 0.0
        return set()
    r.__name__ = "r_ori_eps_%g" % v
    return r


def _ray(p, f, i, ctx):
    return ctx["geometry"](p)["ray"]


def r_wrap_pos(p, f, i, ctx):
    _win(p, 2)
    a = 0.3 - _ray(p, f, i, ctx)                           # roty = a + pi + ray = pi + 0.3
    p[44], p[45] = math.sin(a) * 0.9, math.cos(a) * 0.9
    return set()


def r_wrap_neg(p, f, i, ctx):
    _win(p, 3)
    a = -math.pi / 2 - 0.35 - _ray(p, f, i, ctx)           # roty = a - pi/2 + ray = -pi - 0.35
    p[46], p[47] = math.sin(a) * 1.1, math.cos(a) * 1.1
    return set()


def r_trunc_log(p, f, i, ctx):
    f["trunc_mask"][i] = 1
    p[4], p[5] = f["offset_3D"][i, 0] + 3.0, f["offset_3D"][i, 1] - 2.5
    return set()


def r_abs_zero(p, f, i, ctx):
    p[6:26] = f["keypoints"][i, :, :2].reshape(-1)         # exactly the fp32 labels
    p[4:6] = f["offset_3D"][i]
    return {"abs_off0", "abs_off1"} | {"abs_kp%d" % k for k in range(20)}


def r_plain(p, f, i, ctx):
    return set()


# gradients the float64 reference has exactly 0 by a branch (not by cancellation), per recipe: (losses or None for all
# eleven, regression channels) at the object's centre. The kernel has to produce exact zeros there too.
KY = [7 + 2 * k for k in range(10)]                       # key-point y offsets: every key-point height uses them
KD_LOSSES = ["keypoint_depth_loss", "weighted_avg_depth_loss"]
ZEROS = {
    "depth_low": [(None, [48])], "depth_high": [(None, [48])],                     # clamped direct depth
    "dunc_12": [(None, [49])], "dunc_-12": [(None, [49])],                          # clamped uncertainty
    "kunc_clamped": [(None, [26, 27])], "unc_tie": [(None, [49, 27, 28])],
    "heights_negative": [(KD_LOSSES, KY + [30]), (["corner_loss"], KY)],            # relu 0 / depth clamped at 100
    "heights_tiny": [(KD_LOSSES, KY + [30]), (["corner_loss"], KY)],
    "invalid_kd": [(["keypoint_depth_loss"], [7, 11, 15, 19])],                     # detached group 02
    "box_relu": [(["bbox_loss"], [0])],
}
# ... and gradients that must NOT vanish: a value exactly on a clamp bound (torch passes the gradient on [lo, hi])
NONZERO = {"unc_tie": [(["keypoint_depth_loss"], [26])], "dunc_-10": [(["depth_loss"], [49])]}

KINKS = [r_depth_low, r_depth_high, r_dunc(12.0), r_dunc(-12.0), r_dunc(9.5), r_dunc(-9.5), r_dunc(-10.0), r_kunc_clamped,
         r_unc_tie, r_heights_negative, r_heights_tiny, r_heights_inside, r_invalid_kd, r_box_relu, r_box_tie,
         r_box_disjoint, r_box_encloses, r_bin_tie, _eps(0.0), _eps(1e-20), r_wrap_pos, r_wrap_neg, r_trunc_log,
         r_abs_zero]


# ------------------------------------------------------------------------------------------------ float64 branch points
def geometry(p, f, i, cal, pad, fu_kp):
    """float64 evaluation of one object's loss branch points: {'pairs': [(name, a, b, floor)], 'ray': ...}. A pair is a
    comparison the loss branches on (relu / clamp / abs / min / max arguments, arg-max / arg-min runners-up, roty vs +-pi);
    floor is the magnitude below which its operands count as 0 (corners are in metres)."""
    p = np.asarray(p, np.float64)
    pairs = []

    def add(name, a, b, floor=1e-6):
        pairs.append((name, float(a), float(b), floor))

    cx, cy = (float(v) for v in f["target_centers"][i])
    box = f["bboxes"][i].astype(np.float64)
    td = float(f["locations"][i, 2])
    if box[3] - box[1] > 0 and box[2] - box[0] > 0:
        t = [f32(f32(cx) - f32(box[0])), f32(f32(cy) - f32(box[1])), f32(f32(box[2]) - f32(cx)), f32(f32(box[3]) - f32(cy))]
        for k in range(4):
            add("relu_2d%d" % k, p[k], 0.0)
            add("minmax_2d%d" % k, max(p[k], 0.0), t[k])
    cls = int(f["cls_ids"][i])
    dims = np.exp(p[29:32]) * np.asarray(syn.DIM_MEAN[cls], np.float32).astype(np.float64)
    for k in range(3):
        add("abs_dim%d" % k, dims[k], f["dimensions"][i, k])
    raw = math.exp(-p[48])
    add("clamp_d_lo", raw, 0.1)
    add("clamp_d_hi", raw, 100.0)
    pd = min(max(raw, 0.1), 100.0)
    add("abs_depth", pd, td)
    u = [p[49], p[26], p[27], p[28]]
    for k in range(4):
        add("clamp_u%d_lo" % k, u[k], -10.0)
        add("clamp_u%d_hi" % k, u[k], 10.0)
    u = [min(max(v, -10.0), 10.0) for v in u]
    add("abs_off0", p[4], f["offset_3D"][i, 0])
    add("abs_off1", p[5], f["offset_3D"][i, 1])
    for k in range(4):
        if f["orientations"][i, k] == 1:
            x0, x1 = p[40 + 2 * k], p[41 + 2 * k]
            nrm = math.hypot(x0, x1)
            add("eps_norm%d" % k, nrm, 1e-12, 0.0)
            den = max(nrm, 1e-12)
            ang = float(f["orientations"][i, 4 + k])
            add("abs_sin%d" % k, x0 / den, math.sin(ang))
            add("abs_cos%d" % k, x1 / den, math.cos(ang))
    kp = f["keypoints"][i]
    for k in range(10):
        if kp[k, 2] != 0:
            add("abs_kp%d" % (2 * k), p[6 + 2 * k], kp[k, 0])
            add("abs_kp%d" % (2 * k + 1), p[7 + 2 * k], kp[k, 1])
    ky = lambda k: p[7 + 2 * k]
    fh = fu_kp * dims[1]
    hs = []
    for name, (a, b) in zip(("c", "02a", "02b", "13a", "13b"), ((8, 9), (0, 4), (2, 6), (1, 5), (3, 7))):
        add("relu_h%s" % name, ky(a) - ky(b), 0.0)          # fp32 subtraction of fp32 inputs keeps the exact sign
        hs.append(fh / (max(ky(a) - ky(b), 0.0) * 4.0 + 1e-3))
    kd = [hs[0], 0.5 * (hs[1] + hs[2]), 0.5 * (hs[3] + hs[4])]
    for g in range(3):
        add("clamp_kd%d_lo" % g, kd[g], 0.1)
        add("clamp_kd%d_hi" % g, kd[g], 100.0)
        kd[g] = min(max(kd[g], 0.1), 100.0)
        add("abs_kd%d" % g, kd[g], td)
    unc = sorted(math.exp(v) for v in u)
    add("argmin_unc", unc[0], unc[1])
    w = [math.exp(-v) for v in u]
    soft = (pd * w[0] + kd[0] * w[1] + kd[1] * w[2] + kd[2] * w[3]) / sum(w)
    add("abs_soft", soft, td)
    fu, fv, c_u, c_v, b_x, b_y = cal
    uu, vv = (cx + p[4]) * 4 - float(pad[0]), (cy + p[5]) * 4 - float(pad[1])
    lx, ly = (uu - c_u) * soft / fu + b_x, (vv - c_v) * soft / fv + b_y
    pr = [1.0 / (1.0 + math.exp(p[32 + 2 * k] - p[33 + 2 * k])) for k in range(4)]
    best = int(np.argmax(pr))
    s = sorted(pr, reverse=True)
    add("argmax_bin", s[0], s[1])
    ray = math.atan2(lx, soft)
    roty = math.atan2(p[40 + 2 * best], p[41 + 2 * best]) + CENTERS[best] + ray
    add("wrap_hi", roty, math.pi)
    add("wrap_lo", roty, -math.pi)
    roty = roty - 2 * math.pi if roty > math.pi else (roty + 2 * math.pi if roty < -math.pi else roty)
    tu, tv = (cx + float(f["offset_3D"][i, 0])) * 4 - float(pad[0]), (cy + float(f["offset_3D"][i, 1])) * 4 - float(pad[1])
    tl = np.array([(tu - c_u) * td / fu + b_x, (tv - c_v) * td / fv + b_y, td])
    pc = _corners(roty, dims, np.array([lx, ly, soft]))
    tc = _corners(float(f["rotys"][i]), f["dimensions"][i].astype(np.float64), tl)
    for k in range(8):
        for j in range(3):
            add("abs_corner%d%s" % (k, "xyz"[j]), pc[k, j], tc[k, j], 1.0)
    return {"pairs": pairs, "ray": ray}


def _corners(ry, dims, loc):
    sx = np.array([-1., -1, 1, 1, -1, -1, 1, 1])
    sy = np.array([1., 1, 1, 1, -1, -1, -1, -1])
    sz = np.array([-1., 1, 1, -1, -1, 1, 1, -1])
    X, Y, Z = dims[0] * 0.5 * sx, dims[1] * 0.5 * sy, dims[2] * 0.5 * sz
    c, s = math.cos(ry), math.sin(ry)
    return np.stack([c * X + s * Z + loc[0], Y + loc[1], -s * X + c * Z + loc[2]], 1)


def margin_violations(pairs, ties):
    """the comparisons of one object that are closer than MARGIN to their boundary without being a declared exact tie,
    and the declared ties that are not exact"""
    bad = []
    for name, a, b, floor in pairs:
        if name in ties:
            if a != b:
                bad.append((name, a, b, "declared tie is not exact"))
        elif abs(a - b) < MARGIN * max(abs(a), abs(b), floor):
            bad.append((name, a, b, "within %g of the boundary" % MARGIN))
    return bad


# ------------------------------------------------------------------------------------------------ cases
def _calib_rows(calibs_P):
    from oracle.monoflex_oracle import calib_from_P
    rows = []
    for P in calibs_P:
        c = calib_from_P(P)
        rows.append(tuple(float(f32(c[k])) for k in ("f_u", "f_v", "c_u", "c_v", "b_x", "b_y")))
    return rows


def _ranks(fields):
    owners = [b for b, f in enumerate(fields) if f["reg_mask"].any()]
    return {b: (0 if len(fields) == 1 else owners.index(b)) for b in owners}


def _contexts(fields, calibs_P):
    rows, ranks = _calib_rows(calibs_P), _ranks(fields)
    return {b: dict(cal=rows[b], pad=fields[b]["pad_size"], fu_kp=rows[r][0]) for b, r in ranks.items()}


def _geometry_of(fields, ctxs, b, i, p):
    c = ctxs[b]
    return geometry(np.asarray(p, np.float32), fields[b], i, c["cal"], c["pad"], c["fu_kp"])


def _assemble(name, fields, calibs_P, recipes, seed, shared=()):
    """recipes: {(b, i): recipe}; shared: ((b, i, j), ...) object j of image b sits on object i's centre (set here).
    Every labelled pixel gets a sane vector, then its recipes; a pixel whose comparisons come closer than MARGIN to a
    boundary (that is not a declared tie) is redrawn."""
    rng = np.random.default_rng(seed)
    B = len(fields)
    for b, i, j in shared:
        fields[b]["target_centers"][j] = fields[b]["target_centers"][i]
    H, W = fields[0]["hm"].shape[1:]
    cls, reg = syn.make_train_predictions(B, fields, seed=seed + 1, out_w=W, out_h=H)
    reg = reg.numpy().copy()
    ctxs = _contexts(fields, calibs_P)
    table, ties_of = [], {}
    pixels = {}
    for b, f in enumerate(fields):
        for i in _objects(f):
            x, y = (int(v) for v in f["target_centers"][i])
            pixels.setdefault((b, x, y), []).append(i)
    for (b, x, y), objs in sorted(pixels.items()):
        ctx = dict(ctxs[b])
        for attempt in range(200):
            p = _sane(rng, fields[b], objs[0])
            ties = {}
            for i in objs:
                r = recipes.get((b, i), r_plain)
                ctx["geometry"] = lambda q, i=i: _geometry_of(fields, ctxs, b, i, q)
                ties[i] = r(p, fields[b], i, ctx)
                p = p.astype(np.float32).astype(np.float64)
            bad = [v for i in objs for v in margin_violations(_geometry_of(fields, ctxs, b, i, p)["pairs"], ties[i])]
            if not bad:
                break
        else:
            raise AssertionError("%s: no vector for image %d pixel (%d, %d) keeps its margins: %s" % (name, b, x, y, bad[:3]))
        reg[b, :, y, x] = p.astype(np.float32)
        for i in objs:
            ties_of[(b, i)] = ties[i]
            r = recipes.get((b, i), r_plain)
            branch = r.__name__[2:]
            if len(objs) > 1:
                branch += "+shared_centre"
            table.append((b, i, branch))
    case = dict(name=name, fields=fields, calibs_P=[tuple(tuple(float(v) for v in row) for row in P) for P in calibs_P],
                cls=cls, reg=torch.from_numpy(reg), table=sorted(table), ties=ties_of)
    check_margins(case)
    return case


def check_margins(case):
    """assert, in float64, that every object of `case` keeps its comparisons MARGIN away from their boundaries except
    its declared exact ties"""
    fields, reg = case["fields"], case["reg"].numpy()
    ctxs = _contexts(fields, case["calibs_P"])
    for b, f in enumerate(fields):
        for i in _objects(f):
            x, y = (int(v) for v in f["target_centers"][i])
            bad = margin_violations(_geometry_of(fields, ctxs, b, i, reg[b, :, y, x])["pairs"], case["ties"].get((b, i), set()))
            assert not bad, "%s image %d object %d: %s" % (case["name"], b, i, bad)


def _kinks():
    fields = syn.make_train_targets(4, seed=5)
    spare = _pool(40, seed=31)
    # room for every recipe: top up images 0, 2 and 3 with objects from other synthetic images (distinct centres)
    for b in (0, 2, 3):
        f = fields[b]
        used = {tuple(int(v) for v in f["target_centers"][i]) for i in _objects(f)}
        want = 13
        for j in range(M):
            if len(_objects(f)) >= want or not spare:
                break
            if f["reg_mask"][j]:
                continue
            src, i = spare.pop(0)
            _copy(f, j, src, i)
            x, y = _free_pixel(f, int(f["target_centers"][j, 0]), int(f["target_centers"][j, 1]), used)
            f["target_centers"][j] = (x, y)
            used.add((x, y))
    objs = [(b, i) for b in (0, 2, 3) for i in _objects(fields[b])]
    recipes = {}
    for r, key in zip(KINKS, objs):
        recipes[key] = r
    rest = objs[len(KINKS):]
    assert len(rest) >= 4, "kinks: not enough objects for the centre cases"
    # two objects with different labels on one centre pixel of image 3, and the two map corners of image 2
    (b0, a), (b1, c) = [o for o in rest if o[0] == 3][:2]
    corners = [o for o in rest if o[0] == 2][:2]
    for (b, i), xy in zip(corners, ((0, 0), (OUT_W - 1, OUT_H - 1))):
        fields[b]["target_centers"][i] = xy
        fields[b]["bboxes"][i] = 0                          # no 2D box: the FCOS distances would leave the map
        recipes[(b, i)] = r_corner
    calibs = [syn.KITTI_P2] * 4
    return _assemble("kinks", fields, calibs, recipes, seed=101, shared=((3, a, c),))


def r_corner(p, f, i, ctx):
    return set()


def _calib():
    fields = syn.make_train_targets(5, seed=7, empty_image=0)
    _empty(fields[2])
    calibs = []
    for b in range(5):
        P = np.array(syn.KITTI_P2, np.float64)
        P[0, 0] *= 1.0 + 0.07 * b
        P[1, 1] *= 0.97 + 0.05 * b
        P[0, 2] += 9.0 * b - 11.0
        P[1, 2] -= 4.0 * b - 5.0
        P[0, 3] = -0.54 * P[0, 0] * (b % 3) + 44.85728       # b_x: left, right and a third camera
        P[1, 3] += 0.1 * b
        calibs.append(P.tolist())
        fields[b]["pad_size"] = np.asarray((19 - 3 * b, 4 + 2 * b), np.float32)
    return _assemble("calib", fields, calibs, {}, seed=202)


def _empty(f):
    for i in range(M):
        _clear(f, i)


def _full(batch=7):
    fields = syn.make_train_targets(batch, seed=11, empty_image=-1)
    for f in fields[1:]:
        _empty(f)
    f0 = fields[0]
    used = {tuple(int(v) for v in f0["target_centers"][i]) for i in _objects(f0)}
    spare = _pool(60, seed=41)
    for j in range(M):
        if f0["reg_mask"][j]:
            continue
        src, i = spare.pop(0)
        _copy(f0, j, src, i)
        x, y = _free_pixel(f0, int(f0["target_centers"][j, 0]), int(f0["target_centers"][j, 1]), used)
        f0["target_centers"][j] = (x, y)
        used.add((x, y))
    src, i = spare.pop(0)
    _copy(fields[batch - 1], M - 1, src, i)                 # last slot of the last image
    return fields, ((0, 5, 17), (0, 5, 33))             # three objects on slot 5's centre


def _full_case():
    fields, shared = _full()
    return _assemble("full", fields, [syn.KITTI_P2] * len(fields), {}, seed=303, shared=shared)


def _full_b1():
    fields, shared = _full()
    return _assemble("full_b1", fields[:1], [syn.KITTI_P2], {}, seed=404, shared=shared)


def _all_trunc():
    fields = syn.make_train_targets(3, seed=13)
    for f in fields:
        f["trunc_mask"][:] = f["reg_mask"]
    return _assemble("all_trunc", fields, [syn.KITTI_P2] * 3, {}, seed=505)


def _no_valid_kd():
    fields = syn.make_train_targets(3, seed=17)
    for f in fields:
        f["keypoints_depth_mask"][:] = 0
    return _assemble("no_valid_kd", fields, [syn.KITTI_P2] * 3, {}, seed=606)


def _no_object():
    fields = syn.make_train_targets(2, seed=19)
    for f in fields:
        _empty(f)
    cls, reg = syn.make_train_predictions(2, fields, seed=20)
    return dict(name="no_object", fields=fields, calibs_P=[syn.KITTI_P2] * 2, cls=cls, reg=reg, table=[], ties={})


def _no_box2d():
    fields = syn.make_train_targets(3, seed=23)
    for f in fields:
        f["bboxes"][:] = 0
    return _assemble("no_box2d", fields, [syn.KITTI_P2] * 3, {}, seed=707)


def wide_batch(batch):
    """`batch` images on 48x160 maps (GPU test of the batch limit): every third image but the last empty, so the rank an
    image's key-point depths take f_u from trails its index; a different P per image"""
    fields = syn.make_train_targets(batch, seed=29, out_w=160, out_h=48, empty_image=-1)
    for b in range(0, batch - 1, 3):
        _empty(fields[b])
    calibs = []
    for b in range(batch):
        P = np.array(syn.KITTI_P2, np.float64)
        P[0, 0] *= 1.0 + 0.004 * b
        P[0, 2] += 0.5 * b
        calibs.append(P.tolist())
    return _assemble("batch%d" % batch, fields, calibs, {}, seed=808)


_BUILDERS = dict(kinks=_kinks, calib=_calib, full=_full_case, full_b1=_full_b1, all_trunc=_all_trunc,
                 no_valid_kd=_no_valid_kd, no_object=_no_object, no_box2d=_no_box2d)


def build(name):
    """-> dict(fields, calibs_P, cls, reg, table, ties): `fields` per-image dicts of numpy arrays named like the ParamsList
    fields ('bboxes' for '2d_bboxes'), `calibs_P` one 3x4 P per image, `cls` / `reg` float32 CPU tensors, `table` a sorted
    list of (image, slot, branch) for every labelled object, `ties` {(image, slot): names of its deliberate exact ties}"""
    return _BUILDERS[name]()


def checksum(case):
    """sha256 over every input of a case (labels, calibrations, predictions) in a fixed order"""
    h = hashlib.sha256()
    for f in case["fields"]:
        for k in sorted(f):
            a = np.ascontiguousarray(f[k])
            h.update(k.encode())
            h.update(str(a.dtype).encode())
            h.update(a.tobytes())
    h.update(np.asarray(case["calibs_P"], np.float64).tobytes())
    h.update(case["cls"].numpy().tobytes())
    h.update(case["reg"].numpy().tobytes())
    return h.hexdigest()


def centers_of(case):
    """(image, x, y) of every labelled object in the order the loss enumerates them (image-major, slot order)"""
    return [(b, int(f["target_centers"][i, 0]), int(f["target_centers"][i, 1])) for b, f in enumerate(case["fields"])
            for i in _objects(f)]


def grads_at_centres(grad, case):
    """[N_obj, 50] rows of a [B, 50, H, W] gradient at the labelled centres (shared pixels repeat their sum)"""
    g = grad.detach().cpu().double().numpy() if torch.is_tensor(grad) else np.asarray(grad, np.float64)
    return np.stack([g[b, :, y, x] for b, x, y in centers_of(case)])
