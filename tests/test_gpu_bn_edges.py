"""The BatchNorm backward, the SyncBatchNorm halves and the backward's other fixed-order reductions at their edges, against
float64 (-m gpu; the host-side checks of the references and of the grid emulations run without one).

mf_bn_train_backward runs after every backbone conv and every head InPlaceABN; the SyncBatchNorm halves
(mf_bn_sync_forward_stats / _apply, mf_bn_sync_backward_stats / _apply) are what a multi-GPU run with USE_SYNC_BN uses.
Each is held per channel to float64 at the row-count edges of the CTA split the forward edge test uses (1 row, fewer rows
than one CTA's row lanes, one CTA's 4 x RL row group + 1, exactly the 132 x 8-CTA cap and one row past it), C in
{8, 16, 64, 256}, mean/std up to 300, a constant channel, negative gammas, rows wider than C with NaN neighbours (never
read, never written), every activation with and without a residual, dx written over dy (the tape's call form), and the
256-channel chunks of a 512- and a 320-channel module through backward.bn_backward (|gamma| + eps included). The
SyncBatchNorm exchange is simulated on one GPU: the rows are split unevenly between 2 or 3 ranks (one of a single row, one
of fewer rows than a CTA's row lanes), their double sums added, and every rank normalised with the global count.

The float64 backward (bn_backward_ref) takes the activation mask from the sign of the stored fp16 output, as the kernel
does, so the kink never enters; it is held to torch autograd of F.batch_norm(training=True) on the host.

Bounds, about 3x the worst measured on an NVIDIA H100 80GB HBM3 (700 W) over every case (given beside):
  BN backward dx, dres       per channel (channel_err), one fp16 rounding of the output      FAST_CONV_TOL 1e-3 | 4.8e-4
  BN dgamma                  per channel, against sum|g xhat|                               DGAMMA_TOL 3e-5 | 1.1e-5
                             (at mean/std = 300: xhat carries the fp32 rounding of the mean, ~2e-5 std; 1.1e-6 at 30)
  BN dbeta                   per channel, against sum|g|                                     DBETA_TOL 1e-6 | 2.9e-7
  SyncBN statistics          mean, rstd, scale, shift (the fused forward's bound)             STATS_TOL 1e-5 | 4.4e-7
  SyncBN running statistics                                                                RUNNING_TOL 1.2e-6 | 1.4e-7
  SyncBN y, dx               per channel                                                  FAST_CONV_TOL 1e-3 | 4.8e-4
  SyncBN dres                bit for bit equal to the fused backward's on the same y
  column sum                 per channel, against sum|x|                                    COLSUM_TOL 1.5e-7 | 4.6e-8
  up-sample dw               per (tap, channel), against sum|x dy|                             UPW_TOL 3e-7 | 9.9e-8
  edge head add d_t          per element, against sum_o |g_o w_oc| (at least 2^-14)         EDGE_T_TOL 1e-3 | 4.9e-4
  edge head add dw, dbias    per element, against the sum of the magnitudes of their terms  EDGE_W_TOL 2e-7 | 5.9e-8
  max-pool backward, ties    bit for bit, torch's first-maximum rule
On the constant channel dgamma is exactly 0 and the SyncBatchNorm mean is exactly its value and rstd exactly 1/sqrt(eps)
in fp32; at M = 1, dx and dgamma are exactly 0. The edge head add backward writes d_t = 0 exactly past edge_len and leaves
the dw / dbias rows of the heads past n_out untouched.

The SyncBatchNorm statistics pass used to sum x and x^2 in fp32 (no pivot), so the variance lost ~2^-24 (mean/std)^2 of
itself and a constant channel kept a variance of rounding noise. Measured on the same H100 with that form, worst
stats_err: 2.4e-3, 3.5e-3, 4.8e-3 and 2.7e-4 at mean/std = 1 (M = 1025, 513, 540673 with dx 5.0e-3, and 33: the
constant channel's rstd), 1.7e-6 at mean/std = 10, 9.0e-6 at 30, 1.5e-3 at 300 (running statistics 7.3e-5, y 1.3e-3,
dx 1.8e-3): those five of the thirteen cases failed. The pass now pivots on each rank's first row and un-pivots the sums in double before the exchange
(csrc/mf_bn_train.cu, bn_reduce_kernel): 4.4e-7 at worst, 1.3e-7 at mean/std = 300.

Each bound is shown to be sharp by a swapped reference failing it by at least SWAP_MARGIN: the local row count instead of
the global one in the SyncBatchNorm backward, dgamma without the sign(gamma) factor of |gamma| + eps, the other 256-channel
chunk's parameters, the last CTA's rows dropped from the sums (emulated on the reference side), and every border position
taken by the edge head add, edge_len ignored. Smallest margins measured (error / bound): local count 169x (SyncBatchNorm
dx), no sign(gamma) 6300x (dgamma), neighbouring chunk's gamma 1900x, last CTA dropped 577x (BN dbeta, the gradients
have a mean of 0.5) and 4300x (column sum), edge_len ignored 8.8e5x (edge head add dw, dbias). The file runs in about 40 s
on the GPU.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import tape_ref
from test_gpu_train_forward_layers import (FAST_CONV_TOL, RUNNING_TOL, STATS_TOL, SWAP_MARGIN, activate, bn_case_list,
                                           bn_kernel_inputs, bn_train_ref, channel_err, run_bn_kernel, running_err,
                                           stats_err)
from monoflex_b200 import _lib, backward, engine

DGAMMA_TOL = 3e-5       # dgamma per channel, relative to sum|g xhat|
DBETA_TOL = 1e-6        # dbeta per channel, relative to sum|g|
COLSUM_TOL = 1.5e-7     # column sum per channel, relative to sum|x|
UPW_TOL = 3e-7          # up-sample dw per (tap, channel), relative to sum|x dy|
EDGE_T_TOL = 1e-3       # edge head add d_t per element, relative to sum_o |g_o w_oc|: one fp16 rounding (4.9e-4)
EDGE_W_TOL = 2e-7       # edge head add dw, dbias per element, relative to the sum of the magnitudes of their terms
EPS = 1e-5

BN_CASES = bn_case_list()


# ------------------------------------------------------------------------------------------------ float64 references
def bn_backward_ref(x, dy, y, gamma, eps, act, abs_gamma, count=None, rows=None):
    """float64 backward of y = act(BN_train(x; gamma, beta) [+ residual]) over rows [M, C] (x, dy, y widened to float64;
    the mask is act'(.) from the sign of the stored output y, as bn_act_grad takes it; beta and the residual reach the
    backward only through y). The statistics are those of x. `count` divides the sums in dx (the global element count;
    M by default), `rows` (bool [M]) selects the rows the sums take (all by default). tape_ref.bn_backward on rows, plus
    the sizes of the terms of the sums -> dict of dx, dres = g, dgamma (times sign(gamma) when abs_gamma, as
    backward.bn_backward returns it), dbeta, dgamma_size = sum|g xhat|, dbeta_size = sum|g|."""
    x = x.double()
    mask = None if rows is None else rows.view(-1, 1).to(x.device)
    dx, g, dgamma, dbeta = tape_ref.bn_backward(x, y, dy, gamma.to(x.device), eps, act, abs_gamma, count, mask)
    xhat, _ = tape_ref.bn_xhat(x, eps)
    return dict(dx=dx, dres=g, dgamma=dgamma, dbeta=dbeta, dgamma_size=(g * xhat).abs().sum(0), dbeta_size=g.abs().sum(0))


def nc(rows):
    """[M, C] rows -> [1, C, M, 1] float64, the layout channel_err takes"""
    return rows.double().t().reshape(1, rows.shape[1], rows.shape[0], 1)


def rows_err(got, ref):
    """channel_err of [M, C] rows, the constant channel 0 on its own (its dx is ~1/sqrt(eps) larger than the others', and
    channel_err's 0.05-of-the-largest floor would loosen every other channel by that)"""
    return max(channel_err(nc(got[:, 1:]), nc(ref[:, 1:])), channel_err(nc(got[:, :1]), nc(ref[:, :1])))


def sum_err(got, ref, size):
    """worst per channel |got - ref| / size; a channel whose terms are all 0 must be exactly 0"""
    return ((got.double().to(ref.device) - ref).abs() / size.clamp_min(1e-300)).max().item()


def bn_grid(M, C):
    """(CTAs, rows per CTA) of bn_grid in csrc/mf_bn_train.cu"""
    RL = 256 // (C // 8)
    group = 4 * RL
    ncta = min(max(-(-M // group), 1), 132 * 8)
    rpc = -(-M // ncta)
    rpc = -(-rpc // group) * group
    return -(-M // rpc), rpc


def colsum_grid(M):
    """(CTAs, rows per CTA) of colsum_grid in csrc/mf_bwd_misc.cu"""
    n = min(max(-(-M // 64), 1), 132 * 8)
    rpc = -(-M // n)
    return -(-M // rpc), rpc


def upsample_slabs(npix):
    """(slabs, pixels per slab) of upsample_slabs in csrc/mf_bwd_misc.cu"""
    ns = min(max(-(-npix // 256), 1), 512)
    per = -(-npix // ns)
    return -(-npix // per), per


def last_cta_dropped(M, rpc):
    """bool [M]: every row but those of the last CTA's slab"""
    keep = torch.ones(M, dtype=torch.bool)
    keep[(-(-M // rpc) - 1) * rpc:] = False
    return keep


# ------------------------------------------------------------------------------------------------ launches
def slice_ptr(t, row=0):
    """pointer to column 8 of row `row` of [M, C + 16] rows"""
    return t.data_ptr() + 2 * (row * t.shape[1] + 8)


def nan_rows(v):
    """fp16 rows [M, C + 16]: the float array v [M, C] at column 8, NaN around it"""
    M, C = v.shape
    t = torch.full((M, C + 16), float("nan"), dtype=torch.half)
    t[:, 8:8 + C] = torch.from_numpy(np.asarray(v, dtype=np.float32)).half()
    return t


def workspace(M, C, dev="cuda"):
    return torch.empty(max(1, _lib.load().mf_bn_train_workspace(M, C) // 4), dtype=torch.float32, device=dev)


def run_bn_backward(x, dy, y, stats, M, C, act, dx, dres):
    """mf_bn_train_backward on the column-8 slices -> [2, C] (dgamma, dbeta)"""
    ld = C + 16
    dg = torch.empty(2, C, dtype=torch.float32, device=x.device)
    _lib.call("mf_bn_train_backward", slice_ptr(x), ld, slice_ptr(dy), ld, slice_ptr(y), ld, M, C, stats[0].data_ptr(),
              stats[1].data_ptr(), stats[2].data_ptr(), act, slice_ptr(dx), ld, None if dres is None else slice_ptr(dres), ld,
              dg[0].data_ptr(), dg[1].data_ptr(), workspace(M, C).data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    return dg


def case_flags(i):
    """(act, residual, abs_gamma, dx written over dy) of case i: every combination turns up over the case list"""
    return i % 3, i % 2 == 0, int(i % 4 == 1), i % 5 in (1, 3)


# ------------------------------------------------------------------------------------------------ BN backward, per kernel
@pytest.mark.gpu
@pytest.mark.parametrize("M,C,ratio", BN_CASES, ids=["M%d-C%d-r%d" % c for c in BN_CASES])
def test_bn_train_backward_edges(M, C, ratio):
    """mf_bn_train_backward on the forward kernel's own y and statistics, against float64 per channel"""
    i = BN_CASES.index((M, C, ratio))
    act, with_res, abs_gamma, alias = case_flags(i)
    x, res, gamma, beta, rm, rv = [t.cuda() for t in bn_kernel_inputs(M, C, ratio, 2000 + i)]
    gen = np.random.Generator(np.random.PCG64(3000 + i))
    dy = nan_rows(gen.standard_normal((M, C)) + 0.5).cuda()           # a gradient with a mean: every row's term counts
    y, stats = run_bn_kernel(x, res if with_res else None, gamma, beta, rm, rv, M, C, act, abs_gamma)
    dy0 = dy.clone()
    dx = dy if alias else torch.full_like(dy, float("nan"))
    dres = torch.full_like(dy, float("nan")) if with_res else None
    dg = run_bn_backward(x, dy, y, stats, M, C, act, dx, dres)
    s = slice(8, 8 + C)
    r = bn_backward_ref(x[:, s], dy0[:, s], y[:, s], gamma, EPS, act, abs_gamma)
    sign = torch.sign(gamma.double()) if abs_gamma else 1.0            # what backward.bn_backward applies
    e = dict(dx=rows_err(dx[:, s], r["dx"]), dgamma=sum_err(dg[0] * sign, r["dgamma"], r["dgamma_size"]),
             dbeta=sum_err(dg[1], r["dbeta"], r["dbeta_size"]))
    if with_res:
        e["dres"] = rows_err(dres[:, s], r["dres"])
    _, rpc = bn_grid(M, C)
    drop = last_cta_dropped(M, rpc)
    swap = {}
    ncta = -(-M // rpc)
    if ncta > 4 and M - (ncta - 1) * rpc >= rpc // 2:                  # a last CTA of at least half a slab
        rd = bn_backward_ref(x[:, s], dy0[:, s], y[:, s], gamma, EPS, act, abs_gamma, rows=drop)
        swap["last CTA dropped"] = sum_err(dg[1], rd["dbeta"], r["dbeta_size"]) / DBETA_TOL
    print("M=%d C=%d mean/std=%d act=%d res=%d abs=%d alias=%d: %s%s" % (
        M, C, ratio, act, with_res, abs_gamma, alias, {k: "%.2e" % v for k, v in e.items()},
        " swap margins %s" % {k: "%.0f" % v for k, v in swap.items()} if swap else ""))
    assert e["dx"] <= FAST_CONV_TOL and e.get("dres", 0) <= FAST_CONV_TOL, e
    assert e["dgamma"] <= DGAMMA_TOL and e["dbeta"] <= DBETA_TOL, e
    assert all(v >= SWAP_MARGIN for v in swap.values()), swap
    # nothing outside the slice is written
    for t in (dx, dres):
        if t is not None:
            assert t[:, :8].isnan().all() and t[:, 8 + C:].isnan().all()
    # the constant channel: xhat = 0 exactly, so dgamma = 0 exactly
    assert dg[0, 0].item() == 0.0
    if M == 1:
        assert torch.equal(dx[:, s].double(), torch.zeros(1, C, dtype=torch.float64, device=dx.device))
        assert torch.equal(dg[0], torch.zeros_like(dg[0]))


# ------------------------------------------------------------------------------------------------ BN backward, per module
MODULE_CASES = [(512, engine.ACT_RELU, True, False, True), (320, engine.ACT_LEAKY, False, True, False),
                (512, engine.ACT_NONE, False, True, True), (320, engine.ACT_RELU, True, False, False),
                (64, engine.ACT_LEAKY, True, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("C,act,with_res,abs_gamma,alias", MODULE_CASES,
                         ids=["C%d-act%d-res%d-abs%d-alias%d" % c for c in MODULE_CASES])
def test_bn_backward_operator_chunks(C, act, with_res, abs_gamma, alias):
    """backward.bn_backward (the tape's operator) over a module of C channels run as 256-channel chunks: each chunk's
    dgamma / dbeta lands at its own offset, dx may be dy itself, |gamma| + eps carries sign(gamma) into dgamma"""
    B, H, W = 2, 24, 40
    M = B * H * W
    gen = np.random.Generator(np.random.PCG64(C + 10 * act + 100 * with_res + 1000 * abs_gamma))
    t = lambda a: torch.from_numpy(np.asarray(a, dtype=np.float32))
    x = t(gen.standard_normal((M, C)) * gen.uniform(0.2, 3.0, C) + gen.uniform(-2, 2, C)).half().cuda()
    res = t(gen.standard_normal((M, C))).half().cuda() if with_res else None
    dy = t(gen.standard_normal((M, C)) + 0.3).half().cuda()
    mod = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        mod.weight.copy_(t(gen.uniform(0.5, 1.5, C) * np.where(np.arange(C) % 3 == 1, -1, 1)))
        mod.bias.copy_(t(gen.standard_normal(C) * 0.1))
    P = engine.Plan("cuda", train=True)
    ya = P.act(B, H, W, C)
    P.bn_train(engine.Act.on(x, B, H, W), ya, [(mod, 0, C)], act, engine.Act.on(res, B, H, W) if with_res else None,
               abs_weight=abs_gamma)
    P.finalize()
    P.run()
    y = ya.buf
    dy0 = dy.clone()
    dx = dy if alias else torch.empty_like(dy)
    dres = torch.empty_like(dy) if with_res else None
    [(m2, dgamma, dbeta)] = backward.bn_backward(P.bn_saved, dy, dx, act, abs_weight=abs_gamma, dres=dres)
    torch.cuda.synchronize()
    assert m2 is mod and len(P.bn_saved) == (C + 255) // 256
    gamma = mod.weight.detach()
    r = bn_backward_ref(x, dy0, y, gamma, EPS, act, abs_gamma)
    e = dict(dx=channel_err(nc(dx), nc(r["dx"])), dgamma=sum_err(dgamma, r["dgamma"], r["dgamma_size"]),
             dbeta=sum_err(dbeta, r["dbeta"], r["dbeta_size"]))
    if with_res:
        e["dres"] = channel_err(nc(dres), nc(r["dres"]))
    swap = {}
    if C > 256:
        # the parameters of the neighbouring chunk: chunk k reads gamma[256 (1 - k):...]
        perm = torch.cat([torch.arange(256, C), torch.arange(0, C - 256)]) if C == 512 else None
        if perm is None:                                   # 320 = 256 + 64: the first 64 channels of each chunk swapped
            perm = torch.arange(C)
            perm[:64], perm[256:320] = torch.arange(256, 320), torch.arange(0, 64)
        rs = bn_backward_ref(x, dy0, y, gamma[perm.cuda()], EPS, act, abs_gamma)
        swap["neighbouring chunk's gamma"] = max(channel_err(nc(dx), nc(rs["dx"])) / FAST_CONV_TOL,
                                                 sum_err(dgamma, rs["dgamma"], rs["dgamma_size"]) / DGAMMA_TOL)
    if abs_gamma:
        rs = bn_backward_ref(x, dy0, y, gamma.abs(), EPS, act, abs_gamma)           # sign(gamma) = 1: no sign factor
        swap["dgamma without sign(gamma)"] = sum_err(dgamma, rs["dgamma"], rs["dgamma_size"]) / DGAMMA_TOL
    print("C=%d act=%d res=%d abs=%d alias=%d: %s swap margins %s" % (
        C, act, with_res, abs_gamma, alias, {k: "%.2e" % v for k, v in e.items()}, {k: "%.0f" % v for k, v in swap.items()}))
    assert e["dx"] <= FAST_CONV_TOL and e.get("dres", 0) <= FAST_CONV_TOL, e
    assert e["dgamma"] <= DGAMMA_TOL and e["dbeta"] <= DBETA_TOL, e
    assert all(v >= SWAP_MARGIN for v in swap.values()), swap


# ------------------------------------------------------------------------------------------------ SyncBatchNorm halves
def sync_case_list():
    cases = []
    for C in (8, 16, 64, 256):
        RL = 256 // (C // 8)
        cases += [(4 * RL + 1, C, 1), (1056 * 4 * RL + 1, C, 1)]
    return cases + [(245760, 64, r) for r in (0, 1, 10, 30, 300)]


SYNC_CASES = sync_case_list()


def rank_split(M, C, i):
    """uneven row ranges of 3 ranks (one row, fewer rows than a CTA's row lanes, the rest) or of 2 ranks (3/8, 5/8)"""
    RL = 256 // (C // 8)
    if i % 2 == 0:
        cut = [0, 1, RL, M]
    else:
        cut = [0, M * 3 // 8, M]
    return [(lo, hi) for lo, hi in zip(cut[:-1], cut[1:])]


@pytest.mark.gpu
@pytest.mark.parametrize("M,C,ratio", SYNC_CASES, ids=["M%d-C%d-r%d" % c for c in SYNC_CASES])
def test_sync_batchnorm_halves_edges(M, C, ratio):
    """the four SyncBatchNorm halves on simulated ranks against float64 with the fused path's bounds; dres bit for bit
    equal to the fused backward's on the same y"""
    i = SYNC_CASES.index((M, C, ratio))
    act, with_res, abs_gamma, _ = case_flags(i)
    x, res, gamma, beta, rm0, rv0 = [t.cuda() for t in bn_kernel_inputs(M, C, ratio, 4000 + i)]
    gen = np.random.Generator(np.random.PCG64(5000 + i))
    dy = nan_rows(gen.standard_normal((M, C)) + 0.5).cuda()
    ranks = rank_split(M, C, i)
    ld = C + 16
    st = _lib.stream()
    # forward: local sums -> the all-reduce -> every rank normalises with the global statistics
    sums = []
    for lo, hi in ranks:
        sm = torch.full((2 * C,), float("nan"), dtype=torch.float64, device="cuda")
        _lib.call("mf_bn_sync_forward_stats", slice_ptr(x, lo), ld, hi - lo, C, workspace(hi - lo, C).data_ptr(),
                  sm.data_ptr(), st)
        sums.append(sm)
    total = torch.stack(sums).sum(0)
    y = torch.full_like(x, float("nan"))
    stats = [torch.empty(4, C, dtype=torch.float32, device="cuda") for _ in ranks]
    running = [(rm0.clone(), rv0.clone()) for _ in ranks]
    for (lo, hi), s4, (rm, rv) in zip(ranks, stats, running):
        _lib.call("mf_bn_sync_forward_apply", slice_ptr(x, lo), ld, hi - lo, C, total.data_ptr(), float(M), gamma.data_ptr(),
                  beta.data_ptr(), EPS, 0.1, abs_gamma, rm.data_ptr(), rv.data_ptr(),
                  slice_ptr(res, lo) if with_res else None, ld, act, slice_ptr(y, lo), ld, s4[0].data_ptr(), s4[1].data_ptr(),
                  s4[2].data_ptr(), s4[3].data_ptr(), st)
    torch.cuda.synchronize()
    s = slice(8, 8 + C)
    raw = nc(x[:, s])
    r64 = nc(res[:, s]) if with_res else None
    rf = bn_train_ref(raw, gamma, beta, EPS, 0.1, abs_gamma, rm0, rv0, act, r64)
    e = dict(stats=max(stats_err(s4, rf) for s4 in stats), running=max(running_err(rm, rv, rf) for rm, rv in running),
             y=channel_err(nc(y[:, s]), rf["y"]))
    # backward: local sums (and local dgamma / dbeta) -> the all-reduce -> every rank applies with the global count
    bsums, dgs = [], []
    for (lo, hi), s4 in zip(ranks, stats):
        sm = torch.full((2 * C,), float("nan"), dtype=torch.float64, device="cuda")
        dg = torch.empty(2, C, dtype=torch.float32, device="cuda")
        _lib.call("mf_bn_sync_backward_stats", slice_ptr(x, lo), ld, slice_ptr(dy, lo), ld, slice_ptr(y, lo), ld, hi - lo, C,
                  s4[0].data_ptr(), s4[1].data_ptr(), act, workspace(hi - lo, C).data_ptr(), sm.data_ptr(), dg[0].data_ptr(),
                  dg[1].data_ptr(), st)
        bsums.append(sm)
        dgs.append(dg)
    btot = torch.stack(bsums).sum(0)
    dx = torch.full_like(x, float("nan"))
    dres = torch.full_like(x, float("nan")) if with_res else None
    for (lo, hi), s4 in zip(ranks, stats):
        _lib.call("mf_bn_sync_backward_apply", slice_ptr(x, lo), ld, slice_ptr(dy, lo), ld, slice_ptr(y, lo), ld, hi - lo, C,
                  s4[0].data_ptr(), s4[1].data_ptr(), s4[2].data_ptr(), btot.data_ptr(), float(M), act, slice_ptr(dx, lo), ld,
                  slice_ptr(dres, lo) if with_res else None, ld, workspace(hi - lo, C).data_ptr(), st)
    torch.cuda.synchronize()
    dg = torch.stack(dgs).sum(0)
    r = bn_backward_ref(x[:, s], dy[:, s], y[:, s], gamma, EPS, act, abs_gamma)
    sign = torch.sign(gamma.double()) if abs_gamma else 1.0
    e.update(dx=rows_err(dx[:, s], r["dx"]), dgamma=sum_err(dg[0] * sign, r["dgamma"], r["dgamma_size"]),
             dbeta=sum_err(dg[1], r["dbeta"], r["dbeta_size"]))
    # swapped reference: each rank divides the global sums by its own row count
    local = torch.cat([bn_backward_ref(x[:, s], dy[:, s], y[:, s], gamma, EPS, act, abs_gamma, count=hi - lo)["dx"][lo:hi]
                       for lo, hi in ranks])
    swap = rows_err(dx[:, s], local) / FAST_CONV_TOL
    print("M=%d C=%d mean/std=%d ranks=%s act=%d res=%d abs=%d: %s swap margin (local count) %.0f" % (
        M, C, ratio, [hi - lo for lo, hi in ranks], act, with_res, abs_gamma, {k: "%.2e" % v for k, v in e.items()}, swap))
    assert e["stats"] <= STATS_TOL and e["running"] <= RUNNING_TOL and e["y"] <= FAST_CONV_TOL, e
    assert e["dx"] <= FAST_CONV_TOL and e["dgamma"] <= DGAMMA_TOL and e["dbeta"] <= DBETA_TOL, e
    assert swap >= SWAP_MARGIN
    for t in (y, dx, dres):
        if t is not None:
            assert t[:, :8].isnan().all() and t[:, 8 + C:].isnan().all()
    # the constant channel: var = 0 exactly, so the mean is its value and rstd = 1/sqrt(eps) in fp32; dgamma = 0
    rstd0 = np.float32(1.0 / math.sqrt(float(np.float32(EPS))))
    for s4 in stats:
        assert s4[1, 0].item() == rstd0 and s4[0, 0].item() == float(x[0, 8])
    assert dg[0, 0].item() == 0.0
    # dres = g: the fused backward on the same y writes the same fp16 values
    if with_res:
        dx_f, dres_f = torch.full_like(x, float("nan")), torch.full_like(x, float("nan"))
        run_bn_backward(x, dy, y, stats[0], M, C, act, dx_f, dres_f)
        assert torch.equal(dres[:, s], dres_f[:, s])


# ------------------------------------------------------------------------------------------------ column sum
COLSUM_CASES = [(M, C) for C in (8, 24, 2048) for M in (1, 7, 1056 * 64 + 1)] + [(245760, 8), (245760, 24), (245760, 256)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,C", COLSUM_CASES, ids=["M%d-C%d" % c for c in COLSUM_CASES])
def test_column_sum_edges(M, C):
    """mf_column_sum_nhwc_f16 (conv-bias gradients) per channel against float64: past the 1056-CTA cap with a ragged last
    CTA, C down to 8 and up to 2048, rows wider than C with NaN neighbours"""
    gen = np.random.Generator(np.random.PCG64(M + C))
    x = nan_rows(gen.standard_normal((M, C)) + gen.uniform(-1, 1, C)).cuda()
    out = torch.empty(C, dtype=torch.float32, device="cuda")
    ws = torch.empty(_lib.load().mf_column_sum_workspace(M, C) // 4, dtype=torch.float32, device="cuda")
    _lib.call("mf_column_sum_nhwc_f16", slice_ptr(x), C + 16, M, C, out.data_ptr(), ws.data_ptr(), _lib.stream())
    torch.cuda.synchronize()
    v = x[:, 8:8 + C].double()
    size = v.abs().sum(0)
    err = sum_err(out, v.sum(0), size)
    ncta, rpc = colsum_grid(M)
    swap = None
    if ncta > 1:
        keep = last_cta_dropped(M, rpc).cuda()
        swap = sum_err(out, v[keep].sum(0), size) / COLSUM_TOL
    print("M=%d C=%d CTAs=%d rows/CTA=%d last=%d: %.2e%s" % (M, C, ncta, rpc, M - (ncta - 1) * rpc, err,
                                                            "" if swap is None else " swap margin (last CTA) %.0f" % swap))
    assert err <= COLSUM_TOL
    assert swap is None or swap >= SWAP_MARGIN


# ------------------------------------------------------------------------------------------------ up-sample dw
# one slab; a ragged last slab (1001 pixels: 4 slabs of 251, the last 248); past the 512-slab cap (131241 pixels: 511
# slabs of 257, the last 171); C = 24 and 40 leave a CTA's last warps without channels
UPW_CASES = [(2, 5, 7, 64, 2), (1, 13, 77, 24, 4), (2, 3, 5, 40, 8), (1, 13, 77, 40, 8), (3, 97, 451, 24, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,Hi,Wi,C,f", UPW_CASES, ids=["B%d-%dx%d-C%d-f%d" % c for c in UPW_CASES])
def test_upsample_backward_dw_edges(B, Hi, Wi, C, f):
    """mf_upsample_bwd_nhwc_f16's dw per (tap, channel) against float64 (tape_ref.upsample_backward): f = 2, 4, 8, a ragged
    last slab, C / 8 not a multiple of 8 (a CTA's last warps own no channels)"""
    gen = np.random.Generator(np.random.PCG64(B * Hi * Wi * C + f))
    k = 2 * f
    x = torch.from_numpy(gen.standard_normal((B, C, Hi, Wi)).astype(np.float32)).half().cuda()
    dy = torch.from_numpy((gen.standard_normal((B, C, Hi * f, Wi * f)) + 0.5).astype(np.float32)).half().cuda()
    w = torch.from_numpy(gen.uniform(0.05, 0.5, (C, 1, k, k)).astype(np.float32)).cuda()
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous()
    _, dw = backward.upsample_backward(rows(x), w.view(C, k * k).t().contiguous(), rows(dy), B, Hi, Wi, f)
    torch.cuda.synchronize()
    _, dw_ref, _ = tape_ref.upsample_backward(x.double(), w.double(), dy.double(), f)
    _, size, _ = tape_ref.upsample_backward(x.double().abs(), w.double(), dy.double().abs(), f)
    got = dw.t().reshape(C, 1, k, k)
    err = ((got.double() - dw_ref).abs() / size.clamp_min(1e-300)).max().item()
    ns, per = upsample_slabs(B * Hi * Wi)
    print("B=%d %dx%d C=%d f=%d slabs=%d pixels/slab=%d last=%d: %.2e" % (B, Hi, Wi, C, f, ns, per,
                                                                         B * Hi * Wi - (ns - 1) * per, err))
    assert err <= UPW_TOL


# ------------------------------------------------------------------------------------------------ edge head add backward
# (B, K, n_out): B K = 111 and 505 leave the last CTA of 64 positions partly empty, 1664 (the product's 2 x 832) fills it
EDGE_CASES = [(3, 37, 1), (3, 37, 2), (5, 101, 3), (5, 101, 4), (2, 832, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("B,K,n_out", EDGE_CASES, ids=["B%d-K%d-n%d" % c for c in EDGE_CASES])
def test_edge_head_add_backward_edges(B, K, n_out):
    """mf_edge_head_add_bwd per element against float64: n_out 1 to 4 (the kernel is built for 4), edge_len 0, K and in
    between, repeated border positions, B K not a multiple of 64. d_t is written for every position (0 at e >= edge_len);
    dw / dbias only for the n_out heads."""
    H, W, ctot, ch0 = 12, 40, 9, 3
    gen = np.random.Generator(np.random.PCG64(B * K + n_out))
    t = torch.from_numpy(gen.standard_normal((B, K, 256)).astype(np.float32)).half().cuda()
    w = torch.from_numpy((gen.standard_normal((n_out, 256)) * 0.1).astype(np.float32)).cuda()
    d_out = torch.from_numpy((gen.standard_normal((B, ctot, H, W)) + 0.3).astype(np.float32)).cuda()
    idx = torch.stack([torch.from_numpy(gen.integers(0, W, (B, K))), torch.from_numpy(gen.integers(0, H, (B, K)))], 2)
    elen = torch.tensor([[0, K, K // 2 + 1, K - 1, 1][b % 5] for b in range(B)], dtype=torch.long)
    idx, elen = idx.cuda(), elen.cuda()
    d_t = torch.full((B, K, 256), float("nan"), dtype=torch.half, device="cuda")
    dw = torch.full((4, 256), float("nan"), dtype=torch.float32, device="cuda")
    db = torch.full((4,), float("nan"), dtype=torch.float32, device="cuda")
    _lib.call("mf_edge_head_add_bwd", t.data_ptr(), w.data_ptr(), n_out, idx.data_ptr(), elen.data_ptr(), d_out.data_ptr(), ctot,
              ch0, d_t.data_ptr(), dw.data_ptr(), db.data_ptr(), B, K, H, W, _lib.stream())
    torch.cuda.synchronize()

    def ref(lens):
        """float64 (d_t, dw, dbias) and the sizes of their terms, the positions e < lens[b] taking part"""
        live = (torch.arange(K, device="cuda").view(1, K) < lens.view(B, 1)).double()           # [B, K]
        bi = torch.arange(B, device="cuda").view(B, 1)
        g = d_out.double()[:, ch0:ch0 + n_out].permute(0, 2, 3, 1)[bi, idx[..., 1], idx[..., 0]]     # [B, K, n_out]
        g = g * live.unsqueeze(2)
        td, wd = t.double(), w.double()
        return (g @ wd, torch.einsum("bko,bkc->oc", g, td), g.sum((0, 1)),
                g.abs() @ wd.abs(), torch.einsum("bko,bkc->oc", g.abs(), td.abs()), g.abs().sum((0, 1)))

    r_t, r_w, r_b, s_t, s_w, s_b = ref(elen)
    # below fp16's smallest normal 2^-14 the stored d_t has a fixed spacing of 2^-24, so its size is floored there
    e = dict(d_t=((d_t.double() - r_t).abs() / s_t.clamp_min(2.0 ** -14)).max().item(),
             dw=sum_err(dw[:n_out], r_w, s_w), dbias=sum_err(db[:n_out], r_b, s_b))
    # swapped reference: every position counts, edge_len ignored
    _, q_w, q_b, _, _, _ = ref(torch.full_like(elen, K))
    swap = min(sum_err(dw[:n_out], q_w, s_w) / EDGE_W_TOL, sum_err(db[:n_out], q_b, s_b) / EDGE_W_TOL)
    print("B=%d K=%d n_out=%d edge_len=%s: %s swap margin (edge_len ignored) %.0f" % (
        B, K, n_out, elen.tolist(), {k: "%.2e" % v for k, v in e.items()}, swap))
    assert e["d_t"] <= EDGE_T_TOL and e["dw"] <= EDGE_W_TOL and e["dbias"] <= EDGE_W_TOL, e
    assert swap >= SWAP_MARGIN
    # past edge_len, d_t is exactly 0; the unused heads' dw / dbias rows are not written
    dead = torch.arange(K, device="cuda").view(1, K) >= elen.view(B, 1)
    assert int(dead.sum()) > 0 and torch.equal(d_t[dead].double(), torch.zeros(int(dead.sum()), 256, dtype=torch.float64,
                                                                                  device="cuda"))
    assert dw[n_out:].isnan().all() and db[n_out:].isnan().all()


# ------------------------------------------------------------------------------------------------ max-pool ties
@pytest.mark.gpu
def test_maxpool2_backward_ties():
    """mf_maxpool2_bwd_nhwc_f16 on tied windows, bit for bit against torch's max_pool2d backward (the first maximum in
    scan order takes the gradient) and tape_ref.maxpool2_backward: all-zero windows (as after a ReLU), +0 / -0 ties, and
    the maximum tied at every pair of scan positions"""
    B, C, H, W = 2, 24, 12, 16
    gen = np.random.Generator(np.random.PCG64(77))
    v = gen.standard_normal((B, C, H, W)).astype(np.float32)
    win = v.reshape(B, C, H // 2, 2, W // 2, 2)
    Ho, Wo = H // 2, W // 2
    pos = [(0, 0), (0, 1), (1, 0), (1, 1)]
    for oy in range(Ho):
        for ox in range(Wo):
            kind = (oy * Wo + ox) % 9
            w = win[:, :, oy, :, ox, :]
            if kind == 0:
                w[...] = 0.0                                            # all-zero window
            elif kind == 1:
                w[...] = np.where((np.arange(4) % 2 == 0).reshape(2, 2), 0.0, -0.0)   # +0 / -0
            elif kind == 2:
                w[...] = np.where((np.arange(4) % 2 == 0).reshape(2, 2), -0.0, 0.0)
            else:
                a, b = [(p, q) for p in range(4) for q in range(p + 1, 4)][kind - 3]   # tie at scan positions a < b
                m = np.abs(w).max((-2, -1)) + 1.0
                w[..., pos[a][0], pos[a][1]] = m
                w[..., pos[b][0], pos[b][1]] = m
    x = torch.from_numpy(v).half().float().requires_grad_(True)
    dy = torch.from_numpy(gen.standard_normal((B, C, Ho, Wo)).astype(np.float32)).half().float()
    F.max_pool2d(x, 2).backward(dy)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1]).contiguous().half().cuda()
    dx = backward.maxpool2_backward(rows(x.detach()), rows(dy), B, H, W)
    torch.cuda.synchronize()
    got = dx.float().cpu().view(B, H, W, C).permute(0, 3, 1, 2)
    ref = tape_ref.maxpool2_backward(x.detach(), dy)
    assert torch.equal(ref.float(), x.grad)
    assert torch.equal(got, x.grad)


# ------------------------------------------------------------------------------------------------ host side
def test_bn_backward_ref_matches_torch():
    """bn_backward_ref against torch float64 autograd of F.batch_norm(training=True) + residual + activation, with
    gamma and with |gamma| + eps, on rows; `count` and `rows` change only what they name"""
    gen = torch.Generator().manual_seed(5)
    B, C, H, W = 3, 16, 5, 7
    x = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64) * 2 + 1
    res = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64)
    dy = torch.randn(B, C, H, W, generator=gen, dtype=torch.float64)
    g = torch.randn(C, generator=gen, dtype=torch.float64)
    b = torch.randn(C, generator=gen, dtype=torch.float64)
    rows = lambda t: t.permute(0, 2, 3, 1).reshape(-1, C)
    for abs_gamma in (0, 1):
        for act in (engine.ACT_NONE, engine.ACT_RELU, engine.ACT_LEAKY):
            leaves = [t.clone().requires_grad_(True) for t in (x, g, b, res)]
            gw = leaves[1].abs() + EPS if abs_gamma else leaves[1]
            z = F.batch_norm(leaves[0], None, None, gw, leaves[2], True, 0.1, EPS) + leaves[3]
            assert z.detach().abs().min().item() > 1e-6                  # away from the kink
            y = activate(z, act)
            y.backward(dy)
            r = bn_backward_ref(rows(x), rows(dy), rows(y.detach()), g, EPS, act, abs_gamma)
            assert (r["dx"] - rows(leaves[0].grad)).abs().max().item() < 1e-12
            assert (r["dres"] - rows(leaves[3].grad)).abs().max().item() < 1e-12
            assert (r["dgamma"] - leaves[1].grad).abs().max().item() < 1e-12
            assert (r["dbeta"] - leaves[2].grad).abs().max().item() < 1e-12
    M = B * H * W
    r = bn_backward_ref(rows(x), rows(dy), rows(x), g, EPS, engine.ACT_NONE, 0)
    assert torch.allclose(bn_backward_ref(rows(x), rows(dy), rows(x), g, EPS, engine.ACT_NONE, 0, count=M)["dx"], r["dx"],
                          rtol=0, atol=1e-14)
    keep = torch.arange(M) % 4 != 3
    rd = bn_backward_ref(rows(x), rows(dy), rows(x), g, EPS, engine.ACT_NONE, 0, rows=keep)
    assert torch.allclose(rd["dbeta"], rows(dy)[keep].sum(0), rtol=0, atol=1e-12)
    assert torch.equal(rd["dgamma_size"], r["dgamma_size"])


def test_bn_backward_ref_sizes_and_edges():
    """one row: xhat = 0, so dx and dgamma are exactly 0; a constant channel: dgamma exactly 0; the sizes are the sums
    of the magnitudes of the terms"""
    x = torch.tensor([[0.25, -1.0, 3.0]], dtype=torch.float64)
    dy = torch.tensor([[2.0, -1.5, 0.5]], dtype=torch.float64)
    r = bn_backward_ref(x, dy, x, torch.tensor([1.0, -2.0, 0.5]), EPS, engine.ACT_NONE, 1)
    assert torch.equal(r["dx"], torch.zeros_like(x)) and torch.equal(r["dgamma"], torch.zeros(3, dtype=torch.float64))
    assert torch.equal(r["dbeta"], dy[0]) and torch.equal(r["dbeta_size"], dy[0].abs())
    x = torch.tensor([[0.3, 1.0], [0.3, 2.0], [0.3, 4.0]], dtype=torch.float64)
    dy = torch.tensor([[1.0, -1.0], [2.0, 0.5], [-0.5, 1.0]], dtype=torch.float64)
    r = bn_backward_ref(x, dy, x, torch.tensor([1.0, 1.0]), EPS, engine.ACT_NONE, 0)
    assert r["dgamma"][0].item() == 0.0 and r["dgamma_size"][0].item() == 0.0
    xhat = (x[:, 1] - x[:, 1].mean()) / torch.sqrt(x[:, 1].var(unbiased=False) + EPS)
    assert abs(r["dgamma_size"][1].item() - (dy[:, 1] * xhat).abs().sum().item()) < 1e-12


@pytest.mark.parametrize("C", [8, 16, 24, 64, 256, 2048])
def test_grid_emulations_match_the_kernels(C):
    """bn_grid / colsum_grid / upsample_slabs here against the CTA counts the library's workspace sizes imply, at the row
    counts the tests use (the swapped references drop the emulated last CTA's rows)"""
    lib = _lib.load()
    for M in (1, 7, 31, 127, 129, 4097, 33793, 245760, 1056 * 64 + 1, 1081345):
        ncta, rpc = bn_grid(M, C)
        assert lib.mf_bn_train_workspace(M, C) == 4 * (ncta * 2 * C + 2 * C), (M, C)
        assert (ncta - 1) * rpc < M <= ncta * rpc and ncta <= 1056
        ncta, rpc = colsum_grid(M)
        assert lib.mf_column_sum_workspace(M, C) == 4 * ncta * C, (M, C)
        assert (ncta - 1) * rpc < M <= ncta * rpc and ncta <= 1056
    for (B, Hi, Wi, _, f) in UPW_CASES:
        ns, per = upsample_slabs(B * Hi * Wi)
        assert lib.mf_upsample_bwd_workspace(B, Hi, Wi, C, f) == 4 * ns * 4 * f * f * C
