"""-m gpu: training-side kernels (SURVEY §8 rows R11 backward, R13) against torch-CPU fp32 references of the same op."""
import os

import numpy as np
import pytest
import torch

from monoflex_b200 import solver
from monoflex_b200.config import default_cfg
from oracle import monoflex_oracle as mo

pytestmark = pytest.mark.gpu


def _tensors(gen, shapes):
    return [torch.from_numpy(gen.standard_normal(s).astype(np.float32) * 0.1) for s in shapes]


def test_fused_adamw_matches_torch_adamw():
    """One launch over the arena == torch.optim.AdamW with the reference's groups (solver/__init__.py:10-37), 5 steps,
    ragged tensor sizes (1, chunk-1, chunk, chunk+1, ...), lr decay in between. Tolerance: fp32 re-association only."""
    gen = np.random.Generator(np.random.PCG64(3))
    shapes = [(1,), (511,), (512,), (513,), (16, 3, 7, 7), (27, 64, 3, 3), (27,), (256, 64, 3, 3), (3, 256, 1, 1), (3,)]
    names = ["w%d" % i if i % 2 == 0 else "b%d.bias" % i for i in range(len(shapes))]
    init = _tensors(gen, shapes)
    ref_p = [torch.nn.Parameter(t.clone()) for t in init]
    lrs = [3e-4 * (2.0 if "bias" in n else 1.0) for n in names]
    ref = torch.optim.AdamW([{"params": [p], "lr": lr} for p, lr in zip(ref_p, lrs)], lr=3e-4, weight_decay=1e-5,
                            betas=(0.9, 0.99))
    our_p = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    ours = solver.FusedAdamW([{"params": [p], "lr": lr} for p, lr in zip(our_p, lrs)], lr=3e-4, weight_decay=1e-5,
                             betas=(0.9, 0.99))
    for it in range(5):
        grads = _tensors(gen, shapes)
        for p, q, g in zip(ref_p, our_p, grads):
            p.grad = g.clone()
            q.grad.copy_(g.cuda())                                    # .grad is a view of the gradient arena
        if it == 3:                                                    # scheduler-style lr change (LambdaLR rewrites group lr)
            for opt in (ref, ours):
                for g in opt.param_groups:
                    g["lr"] *= 0.1
        ref.step()
        ours.step()
        for p, q in zip(ref_p, our_p):
            d = (q.detach().cpu() - p.detach()).abs().max().item()
            assert d <= 2e-7 + 1e-6 * p.detach().abs().max().item(), (it, tuple(p.shape), d)
    for p, q in zip(ref_p, our_p):
        st = ref.state[p]
        assert torch.allclose(ours.state[q]["exp_avg"].cpu(), st["exp_avg"], rtol=1e-5, atol=1e-8)
        assert torch.allclose(ours.state[q]["exp_avg_sq"].cpu(), st["exp_avg_sq"], rtol=1e-5, atol=1e-10)
        assert float(ours.state[q]["step"]) == float(st["step"]) == 5.0
    # padding between tensors is never touched
    a = ours.arena
    used = torch.zeros(a.numel, dtype=torch.bool)
    for o, p in zip(a.offsets, a.tensors):
        used[o:o + p.numel()] = True
    assert a.params.cpu()[~used].abs().sum() == 0 and ours.exp_avg_sq.cpu()[~used].abs().sum() == 0


def test_fused_adamw_grad_scale_is_ddp_mean():
    """grad_scale = 1/world on a SUM-reduced arena == AdamW on the mean gradient (DDP semantics)."""
    gen = np.random.Generator(np.random.PCG64(4))
    shapes = [(64, 64, 3, 3), (64,)]
    init, g0, g1 = _tensors(gen, shapes), _tensors(gen, shapes), _tensors(gen, shapes)
    ref_p = [torch.nn.Parameter(t.clone()) for t in init]
    ref = torch.optim.AdamW(ref_p, lr=3e-4, weight_decay=1e-5, betas=(0.9, 0.99))
    our_p = [torch.nn.Parameter(t.clone().cuda()) for t in init]
    ours = solver.FusedAdamW(our_p, lr=3e-4, weight_decay=1e-5, betas=(0.9, 0.99))
    for p, q, a, b in zip(ref_p, our_p, g0, g1):
        p.grad = (a + b) / 2
        q.grad.copy_((a + b).cuda())
    ref.step()
    ours.step(grad_scale=0.5)
    for p, q in zip(ref_p, our_p):
        assert torch.allclose(q.detach().cpu(), p.detach(), rtol=1e-6, atol=2e-7)


def test_detector_optimizer_layout_and_version_bump():
    """build_optimizer on the real detector: the reference's group census (SURVEY R13: 280 tensors, 112 'bias' names at
    2x lr, 20.95 M parameters), one launch updates all of them and invalidates the cached kernel plans."""
    from monoflex_b200 import engine
    from monoflex_b200.model.detector import KeypointDetector
    cfg = default_cfg()
    model = KeypointDetector(cfg).cuda()
    opt = solver.build_optimizer(model, cfg)
    n_par = sum(p.numel() for p in model.parameters() if p.requires_grad)
    n_bias = sum(1 for g in opt.param_groups if g["lr"] == pytest.approx(6e-4))
    names = [k for k, v in model.named_parameters() if v.requires_grad]
    assert len(opt.param_groups) == len(names) and n_bias == sum("bias" in k for k in names)
    assert opt.arena.numel >= n_par and opt.arena.numel - n_par < len(names) * opt.arena.chunk
    before = opt.arena.params.clone()
    fp0 = engine.fingerprint(model)
    opt.arena.grads.normal_()
    opt.step()
    torch.cuda.synchronize()
    assert engine.fingerprint(model) != fp0
    delta = (opt.arena.params - before).abs()
    # first AdamW step moves every weight by ~lr (m/sqrt(v) = +-1): between 0.5 lr and 2.1 lr where the gradient is non-zero
    used = opt.arena.chunk_table([1.0] * len(names)).cuda().repeat_interleave(opt.arena.chunk) > 0
    assert delta[used].max().item() < 2.1 * 6e-4 and delta.max().item() > 0.5 * 3e-4


def test_focal_loss_backward_matches_autograd():
    from monoflex_b200._lib import call, stream
    gen = np.random.Generator(np.random.PCG64(12))
    pred = torch.from_numpy(gen.uniform(1e-4, 1 - 1e-4, (2, 3, 24, 80)).astype(np.float32)).requires_grad_(True)
    tgt = torch.from_numpy((gen.uniform(0, 1, (2, 3, 24, 80)) ** 8).astype(np.float32))
    tgt.view(-1)[::97] = 1.0
    tgt.view(-1)[5::193] = -1.0                                        # ignored pixels
    loss, npos = mo.focal_loss(pred, tgt)
    (loss / torch.clamp(npos, 1)).backward()                           # detector_loss.py:276 with hm_loss weight 1
    p, t = pred.detach().cuda(), tgt.cuda()
    scale = (1.0 / torch.clamp(npos, 1)).reshape(1).cuda()
    grad = torch.empty_like(p)
    call("mf_focal_loss_backward", p.data_ptr(), t.data_ptr(), p.numel(), scale.data_ptr(), grad.data_ptr(), stream())
    ref = pred.grad
    assert (grad.cpu() - ref).abs().max().item() <= 1e-5 * ref.abs().max().item()
    assert grad.cpu()[tgt == -1].abs().sum() == 0


# ------------------------------------------------------------------------------------------------ row R12: the 11-term loss
def _loss_case(batch, seed=5):
    from monoflex_b200 import synthetic as syn
    fields = syn.make_train_targets(batch, seed=seed)
    cls, reg = syn.make_train_predictions(batch, fields, seed=seed + 1)
    return syn, fields, cls, reg


def _run_cuda_loss(syn, fields, cls, reg):
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    lc = Loss_Computation(default_cfg())
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    c, r = cls.clone().cuda().requires_grad_(True), reg.clone().cuda().requires_grad_(True)
    loss_dict, log = lc({"cls": c, "reg": r}, targets)
    return loss_dict, log, c, r


@pytest.mark.parametrize("batch", [1, 4, 8])
def test_loss_forward_matches_oracle(batch):
    """11 losses + logged metrics of the fused kernel vs the CPU oracle (itself pinned against the unmodified reference,
    tests/test_oracle_golden.py). batch 4 / 8 contain an image without objects (calibration-rank quirk), truncated
    objects, objects without 2D box and invisible key points; batch 1 takes the reference's batch_size == 1 branch."""
    syn, fields, cls, reg = _loss_case(batch)
    if batch == 1:
        fields = syn.make_train_targets(1, empty_image=-1)
        cls, reg = syn.make_train_predictions(1, fields)
    loss_dict, log, _, _ = _run_cuda_loss(syn, fields, cls, reg)
    ref, ref_log = mo.loss_computation(cls, reg, fields, [syn.KITTI_P2] * batch)
    assert list(loss_dict) == mo.LOSS_NAMES
    for k in mo.LOSS_NAMES:
        a, b = loss_dict[k].item(), ref[k].item()
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (k, a, b)
    for k, v in ref_log.items():
        assert abs(log[k] - v.item()) <= 1e-5 * max(1.0, abs(v.item())), (k, log[k], v.item())


def test_loss_matches_reference_golden():
    """straight against the fixture recorded from the unmodified reference (oracle/make_golden_loss.py)."""
    import os
    from conftest import GOLDEN
    gold = np.load(os.path.join(GOLDEN, "loss_4x96x320.npz"))
    syn, fields, cls, reg = _loss_case(4)
    loss_dict, log, c, r = _run_cuda_loss(syn, fields, cls, reg)
    for k in mo.LOSS_NAMES:
        assert abs(loss_dict[k].item() - gold["loss_" + k]) <= 1e-5 * max(1.0, abs(gold["loss_" + k])), k
    total = sum(loss_dict.values())                                   # engine/trainer.py:110
    assert abs(total.item() - gold["total"]) <= 1e-5 * abs(gold["total"])
    total.backward()
    centers = np.stack([f["target_centers"] for f in fields])
    mask = np.stack([f["reg_mask"] for f in fields]).astype(bool)
    g = r.grad.cpu().numpy()
    rows = np.stack([g[b, :, centers[b, i, 1], centers[b, i, 0]] for b in range(4) for i in range(mask.shape[1]) if mask[b, i]])
    ref = gold["grad_reg_at_centers"]
    assert np.abs(rows - ref).max() <= 2e-5 * np.abs(ref).max()
    assert abs(np.abs(g).sum() - gold["grad_reg_abs_sum"]) <= 1e-4 * gold["grad_reg_abs_sum"]   # nothing outside the centres
    gc = c.grad.cpu().numpy().reshape(-1)
    assert np.abs(gc[::97] - gold["grad_cls_sample"]).max() <= 1e-5 * np.abs(gold["grad_cls_sample"]).max()


def test_loss_backward_matches_oracle_autograd_weighted():
    """dual-number backward with NON-uniform upstream gradients per loss term vs torch autograd through the oracle."""
    syn, fields, cls, reg = _loss_case(8, seed=9)
    wts = torch.tensor([0.3, 1.7, 0.9, 2.0, 0.5, 1.1, 3.0, 0.7, 1.3, 4.0, 0.2])
    loss_dict, _, c, r = _run_cuda_loss(syn, fields, cls, reg)
    sum(w * loss_dict[k] for w, k in zip(wts.cuda(), mo.LOSS_NAMES)).backward()
    cr, rr = cls.clone().requires_grad_(True), reg.clone().requires_grad_(True)
    ref, _ = mo.loss_computation(cr, rr, fields, [syn.KITTI_P2] * 8)
    sum(w * ref[k] for w, k in zip(wts, mo.LOSS_NAMES)).backward()
    gr, gc = r.grad.cpu(), c.grad.cpu()
    assert (gr - rr.grad).abs().max().item() <= 2e-5 * rr.grad.abs().max().item()
    assert (gc - cr.grad).abs().max().item() <= 1e-5 * cr.grad.abs().max().item()
    at_centre = torch.zeros_like(gr, dtype=torch.bool)                 # the gradient lives at the object centres only
    for b, f in enumerate(fields):
        for i in np.nonzero(f["reg_mask"])[0]:
            at_centre[b, :, f["target_centers"][i, 1], f["target_centers"][i, 0]] = True
    assert gr[~at_centre].abs().sum().item() == 0 and rr.grad[~at_centre].abs().sum().item() == 0


def test_loss_config_guard():
    from monoflex_b200.model.head.detector_loss import Loss_Computation
    cfg = default_cfg()
    cfg.MODEL.HEAD.CORNER_LOSS_DEPTH = 'direct'
    with pytest.raises(NotImplementedError):
        Loss_Computation(cfg)


def test_fused_gradient_exchange_multi_gpu():
    """world >= 2 only (skipped on a 1-GPU box): reduce-scatter + AdamW + all-gather in ONE peer-memory kernel is bit-identical
    to NCCL all-reduce + the single-GPU kernel, for the plain NVLink and the NVLS multicast variants (tools/p2p_adamw_check.py)."""
    import os
    import subprocess
    import sys
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", os.path.join(root, "tools", "p2p_adamw_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert '"ok": true' in r.stdout


def test_sync_batchnorm_two_ranks_match_two_image_batch():
    """world >= 2 only (skipped on a 1-GPU box): after the reference's `SyncBatchNorm.convert_sync_batchnorm(model)` the train-mode
    backbone on one image per rank reproduces the two-image single-process forward (global batch statistics), its running
    statistics and - summed over ranks - its parameter gradients (tools/syncbn_check.py)."""
    import os
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(root, "tools", "syncbn_check.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, cwd=root)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert '"ok": true' in r.stdout


# ------------------------------------------------------------------------------------------------ conv backward building blocks
@pytest.mark.parametrize("case", [
    # B, H, W, Cin, Cout, k, stride, pad
    (2, 12, 20, 64, 64, 3, 1, 1),        # two taps share an M tile; 9 taps -> a dummy half tile
    (2, 14, 18, 128, 128, 3, 2, 1),      # stride 2, N = 128, ragged last pixel block
    (1, 9, 23, 64, 256, 1, 1, 0),        # 1x1, two N tiles
    (2, 10, 12, 192, 64, 3, 1, 1),       # odd number of 64-channel slots
    (8, 96, 320, 64, 64, 3, 1, 1),       # full-size level-2 layer: long split-K reduction
    (2, 20, 36, 16, 16, 3, 1, 1),        # level0: the narrow warp-MMA kernel (mf_wgrad_narrow.cu), two 16-pixel blocks + ragged third
    (2, 11, 37, 16, 16, 7, 1, 3),        # 7x7 stem on 16-channel padded rows: one tap row per warp, ragged width
    (3, 5, 16, 16, 16, 3, 1, 1),         # exactly one block per row, images / rows wrap
    (2, 20, 36, 16, 32, 3, 2, 1),        # level1 entry: stride 2, N = 32
    (1, 18, 26, 32, 64, 3, 2, 1),        # level2 entry: 64-byte A boxes, 128-byte B boxes
    (2, 12, 14, 32, 32, 3, 1, 1),        # level1 second conv
    (1, 10, 22, 32, 64, 1, 1, 0),        # project 1x1 after max-pool
])
def test_conv_wgrad_tensor_core(case):
    """dW of a convolution from NHWC fp16 activations / output gradients (MN-major wgmma operands, split-K) vs
    torch.nn.grad.conv2d_weight on the same fp16-representable operands in fp32 (CPU)."""
    from monoflex_b200._lib import call, stream
    B, H, W, Cin, Cout, k, s, pad = case
    gen = np.random.Generator(np.random.PCG64(sum(case)))
    Ho, Wo = (H + 2 * pad - k) // s + 1, (W + 2 * pad - k) // s + 1
    x = torch.from_numpy(gen.standard_normal((B, Cin, H, W)).astype(np.float32)).half()
    dy = torch.from_numpy((gen.standard_normal((B, Cout, Ho, Wo)) * 0.1).astype(np.float32)).half()
    xr = x.permute(0, 2, 3, 1).reshape(-1, Cin).contiguous().cuda()
    dyr = dy.permute(0, 2, 3, 1).reshape(-1, Cout).contiguous().cuda()
    dw = torch.full((Cout, Cin, k, k), float("nan"), dtype=torch.float32, device="cuda")
    call("mf_conv2d_wgrad_nhwc_f16", xr.data_ptr(), Cin, B, H, W, Cin, dyr.data_ptr(), Cout, Cout, k, s, pad, dw.data_ptr(),
         stream())
    if B * H * W > 100000:       # CPU reference of the big case in chunks of images (conv2d_weight is slow but exact enough)
        ref = sum(torch.nn.grad.conv2d_weight(x[b:b + 1].float(), (Cout, Cin, k, k), dy[b:b + 1].float(), stride=s, padding=pad)
                  for b in range(B))
    else:
        ref = torch.nn.grad.conv2d_weight(x.float(), (Cout, Cin, k, k), dy.float(), stride=s, padding=pad)
    err = (dw.cpu() - ref).abs().max().item() / ref.abs().max().item()
    assert err < 1e-4, err


@pytest.mark.parametrize("case", [(2, 12, 20, 64, 64, 3, 1), (1, 9, 23, 64, 128, 1, 0), (2, 10, 12, 128, 64, 3, 1)])
def test_conv_dgrad_via_forward_kernel(case):
    """dX of a stride-1 conv = the forward tensor-core kernel on dY with rotated/transposed weights, vs
    torch.nn.grad.conv2d_input on the same fp16-representable operands: written to a new buffer, and - the training tape's
    call form, through backward.conv_backward - accumulated into a destination that already holds random values."""
    from monoflex_b200 import backward, engine
    B, H, W, Cin, Cout, k, pad = case
    gen = np.random.Generator(np.random.PCG64(sum(case) + 1))
    Ho, Wo = H + 2 * pad - k + 1, W + 2 * pad - k + 1
    w = torch.from_numpy((gen.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cout * k * k)).astype(np.float32)).half().float()
    dy = torch.from_numpy(gen.standard_normal((B, Cout, Ho, Wo)).astype(np.float32)).half()
    dyr = dy.permute(0, 2, 3, 1).reshape(-1, Cout).contiguous().cuda()
    dx = backward.conv2d_dgrad(dyr, w.cuda(), B, Ho, Wo, pad)
    torch.cuda.synchronize()
    assert dx.shape == (B * H * W, Cin)
    ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w, dy.float(), stride=1, padding=pad)
    got = dx.float().cpu().view(B, H, W, Cin).permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() / ref.abs().max().item() < 1e-3      # fp16 output rounding
    # accumulation: out == before + dgrad
    before = torch.from_numpy((gen.standard_normal((B * H * W, Cin)) * 0.25).astype(np.float32)).half().cuda()
    out = before.clone()
    x = torch.from_numpy(gen.standard_normal((B, Cin, H, W)).astype(np.float32)).half()
    xr = x.permute(0, 2, 3, 1).reshape(-1, Cin).contiguous().cuda()
    dw, db = backward.conv_backward(engine.Act.on(xr, B, H, W), w.cuda(), None, 1, pad, dyr, engine.Act.on(out, B, H, W))
    torch.cuda.synchronize()
    assert db is None
    got = (out.float() - before.float()).cpu().view(B, H, W, Cin).permute(0, 3, 1, 2)
    assert (got - ref).abs().max().item() / ref.abs().max().item() < 1e-3
    ref_w = torch.nn.grad.conv2d_weight(x.float(), (Cout, Cin, k, k), dy.float(), stride=1, padding=pad)
    assert (dw.cpu() - ref_w).abs().max().item() / ref_w.abs().max().item() < 1e-4


def test_backward_python_wrappers_reject_cpu():
    from monoflex_b200 import backward
    with pytest.raises(RuntimeError):
        backward.conv2d_wgrad(torch.zeros(64, 64, dtype=torch.half), torch.zeros(64, 64, dtype=torch.half).cuda(), 1, 8, 8, 1)


@pytest.mark.parametrize("case", [(2, 12, 20, 64, 1, True), (1, 9, 23, 16, 1, False), (3, 7, 11, 512, 0, False),
                                  (2, 16, 24, 256, 2, False), (8, 96, 320, 64, 1, True), (2, 6, 10, 320, 1, True)])
def test_batchnorm_train_plan_and_backward_operator(case):
    """train-mode BN (+ residual + activation) over NHWC fp16 rows vs torch (CPU fp32) batch_norm(training=True) and its
    autograd, on the same fp16-representable inputs: output, running statistics, dx, dgamma, dbeta, dresidual. The forward
    is a one-op train-mode plan (Plan.bn_train), the backward the training tape's operator (backward.bn_backward); 512 and
    320 channels run as 256-channel chunks (the last one ragged)."""
    from monoflex_b200 import backward, engine
    import torch.nn.functional as F
    B, H, W, C, act, use_res = case
    gen = np.random.Generator(np.random.PCG64(sum(case[:4])))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    x = t(gen.standard_normal((B, C, H, W)) * 1.7 + 0.3).half().float()
    res = t(gen.standard_normal((B, C, H, W))).half().float() if use_res else None
    dy = t(gen.standard_normal((B, C, H, W))).half().float()
    gamma, beta = t(gen.uniform(0.5, 1.5, C)), t(gen.standard_normal(C) * 0.1)
    rm, rv = t(gen.standard_normal(C) * 0.1), t(gen.uniform(0.5, 1.5, C))
    rows = lambda v: engine.Act.on(v.permute(0, 2, 3, 1).reshape(-1, C).contiguous().half().cuda(), B, H, W)
    bn = torch.nn.BatchNorm2d(C).cuda()
    with torch.no_grad():
        for p, v in ((bn.weight, gamma), (bn.bias, beta), (bn.running_mean, rm), (bn.running_var, rv)):
            p.copy_(v)
    P = engine.Plan("cuda", train=True)
    ya = P.act(B, H, W, C)
    P.bn_train(rows(x), ya, [(bn, 0, C)], act, rows(res) if use_res else None)
    P.finalize()
    P.run()
    y = ya.buf
    dx, dres = torch.empty_like(y), (torch.empty_like(y) if use_res else None)
    [(mod, dgamma, dbeta)] = backward.bn_backward(P.bn_saved, rows(dy), dx, act, dres=dres)
    torch.cuda.synchronize()
    assert mod is bn and len(P.bn_saved) == (C + 255) // 256
    # reference
    xr = x.clone().requires_grad_(True)
    gr, br = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    rr = res.clone().requires_grad_(True) if use_res else None
    rm_ref, rv_ref = rm.clone(), rv.clone()
    z = F.batch_norm(xr, rm_ref, rv_ref, gr, br, True, 0.1, 1e-5)
    if use_res:
        z = z + rr
    z = {0: lambda v: v, 1: F.relu, 2: lambda v: F.leaky_relu(v, 0.01)}[act](z)
    back = lambda v: v.float().cpu().view(B, H, W, C).permute(0, 3, 1, 2)
    yq = back(y)
    assert (yq - z.detach()).abs().max().item() <= 2e-3 * z.detach().abs().max().item()          # fp16 output rounding
    assert torch.allclose(bn.running_mean.cpu(), rm_ref, rtol=1e-4, atol=1e-5)
    assert torch.allclose(bn.running_var.cpu(), rv_ref, rtol=1e-4, atol=1e-5)
    # backward through the SAME activation mask the kernel saw (sign of the fp16 output): use autograd on the fp32 reference;
    # elements within fp16 rounding of the ReLU kink may differ, so compare in the 1e-2-of-max norm on dx and tightly on sums
    z.backward(dy)
    # the kernel takes the activation mask from the sign of its fp16 output; reference pre-activations within fp16 rounding of
    # the kink can land on the other side, so those elements are excluded from the element-wise comparisons
    zd = z.detach()
    safe = (zd.abs() > 2e-3 * zd.abs().max()) if act != 0 else torch.ones_like(zd, dtype=torch.bool)
    assert safe.float().mean().item() > 0.3
    assert ((back(dx) - xr.grad).abs() * safe).max().item() <= 1e-2 * xr.grad.abs().max().item()
    assert (dgamma.cpu() - gr.grad).abs().max().item() <= 2e-3 * gr.grad.abs().max().item()
    assert (dbeta.cpu() - br.grad).abs().max().item() <= 2e-3 * br.grad.abs().max().item()
    if use_res:
        assert ((back(dres) - rr.grad).abs() * safe).max().item() <= 1e-2 * rr.grad.abs().max().item()


def _rows_of(t4):
    B, C, H, W = t4.shape
    return t4.permute(0, 2, 3, 1).reshape(-1, C).contiguous().half().cuda()


def _nchw_of(rows, B, H, W):
    return rows.float().cpu().view(B, H, W, -1).permute(0, 3, 1, 2)


@pytest.mark.parametrize("case", [(4096, 64, 1, True), (3000, 16, 1, False), (2048, 256, 2, False)])
def test_sync_batchnorm_halves_equal_fused_kernels(case):
    """SyncBatchNorm kernels (mf_bn_sync_*) with the exchange SIMULATED on one GPU: the rows of a tensor are split between two
    "ranks", each computes its local sums, the sums are added (what the NCCL all-reduce does) and each half is normalised /
    back-propagated with the global count - the result must equal the single-call mf_bn_train_forward / _backward on the whole
    tensor (same arithmetic, different partial-sum grouping), including running statistics, dgamma and dbeta (summed over ranks)."""
    from monoflex_b200._lib import call, load, stream
    M, C, act, with_res = case
    gen = np.random.Generator(np.random.PCG64(M + C))
    dev = "cuda"
    x = torch.from_numpy((gen.standard_normal((M, C)) * 1.5 + 0.3).astype(np.float32)).half().to(dev)
    dy = torch.from_numpy((gen.standard_normal((M, C)) * 0.2).astype(np.float32)).half().to(dev)
    res = torch.from_numpy(gen.standard_normal((M, C)).astype(np.float32)).half().to(dev) if with_res else None
    gamma = torch.from_numpy(gen.uniform(0.5, 1.5, C).astype(np.float32)).to(dev)
    beta = torch.from_numpy((gen.standard_normal(C) * 0.1).astype(np.float32)).to(dev)
    st = stream()

    def ws_for(m):
        return torch.empty(load().mf_bn_train_workspace(m, C) // 4, dtype=torch.float32, device=dev)

    # ---- fused reference on the whole tensor
    rm, rv = torch.zeros(C, device=dev), torch.ones(C, device=dev)
    y = torch.empty_like(x)
    stats = torch.empty(4, C, dtype=torch.float32, device=dev)
    ws = ws_for(M)
    call("mf_bn_train_forward", x.data_ptr(), C, M, C, gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.1, 0, rm.data_ptr(), rv.data_ptr(),
         res.data_ptr() if with_res else None, C, act, y.data_ptr(), C, stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(),
         stats[3].data_ptr(), ws.data_ptr(), st)
    dx, dres = torch.empty_like(x), (torch.empty_like(x) if with_res else None)
    dg = torch.empty(2, C, dtype=torch.float32, device=dev)
    call("mf_bn_train_backward", x.data_ptr(), C, dy.data_ptr(), C, y.data_ptr(), C, M, C, stats[0].data_ptr(), stats[1].data_ptr(),
         stats[2].data_ptr(), act, dx.data_ptr(), C, dres.data_ptr() if with_res else None, C, dg[0].data_ptr(), dg[1].data_ptr(),
         ws.data_ptr(), st)
    # ---- two simulated ranks
    split = (M * 3 // 8) // 8 * 8
    parts = [(0, split), (split, M)]
    sums = [torch.zeros(2 * C, dtype=torch.float64, device=dev) for _ in parts]
    for (lo, hi), sm in zip(parts, sums):
        call("mf_bn_sync_forward_stats", x[lo:hi].data_ptr(), C, hi - lo, C, ws_for(hi - lo).data_ptr(), sm.data_ptr(), st)
    total = sums[0] + sums[1]                                             # the all-reduce
    y2 = torch.empty_like(x)
    st2 = [torch.empty(4, C, dtype=torch.float32, device=dev) for _ in parts]
    rms = [(torch.zeros(C, device=dev), torch.ones(C, device=dev)) for _ in parts]
    for (lo, hi), s4, (rm2, rv2) in zip(parts, st2, rms):
        call("mf_bn_sync_forward_apply", x[lo:hi].data_ptr(), C, hi - lo, C, total.data_ptr(), float(M), gamma.data_ptr(), beta.data_ptr(),
             1e-5, 0.1, 0, rm2.data_ptr(), rv2.data_ptr(), res[lo:hi].data_ptr() if with_res else None, C, act, y2[lo:hi].data_ptr(), C,
             s4[0].data_ptr(), s4[1].data_ptr(), s4[2].data_ptr(), s4[3].data_ptr(), st)
    torch.cuda.synchronize()
    assert torch.equal(y2, y) or (y2.float() - y.float()).abs().max().item() <= 2e-3 * y.float().abs().max().item()
    for s4, (rm2, rv2) in zip(st2, rms):
        assert (s4 - stats).abs().max().item() <= 1e-5 * stats.abs().max().item()
        assert (rm2 - rm).abs().max().item() <= 1e-6 and (rv2 - rv).abs().max().item() <= 1e-6
    bs = [torch.zeros(2 * C, dtype=torch.float64, device=dev) for _ in parts]
    dgs = [torch.empty(2, C, dtype=torch.float32, device=dev) for _ in parts]
    for (lo, hi), sm, d2 in zip(parts, bs, dgs):
        call("mf_bn_sync_backward_stats", x[lo:hi].data_ptr(), C, dy[lo:hi].data_ptr(), C, y[lo:hi].data_ptr(), C, hi - lo, C,
             stats[0].data_ptr(), stats[1].data_ptr(), act, ws_for(hi - lo).data_ptr(), sm.data_ptr(), d2[0].data_ptr(), d2[1].data_ptr(), st)
    btot = bs[0] + bs[1]
    dx2, dres2 = torch.empty_like(x), (torch.empty_like(x) if with_res else None)
    for (lo, hi) in parts:
        call("mf_bn_sync_backward_apply", x[lo:hi].data_ptr(), C, dy[lo:hi].data_ptr(), C, y[lo:hi].data_ptr(), C, hi - lo, C,
             stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), btot.data_ptr(), float(M), act, dx2[lo:hi].data_ptr(), C,
             dres2[lo:hi].data_ptr() if with_res else None, C, ws_for(hi - lo).data_ptr(), st)
    torch.cuda.synchronize()
    assert (dx2.float() - dx.float()).abs().max().item() <= 2e-3 * dx.float().abs().max().item()
    if with_res:
        assert torch.equal(dres2, dres)
    assert ((dgs[0] + dgs[1]) - dg).abs().max().item() <= 1e-4 * dg.abs().max().item()


def test_conv_dgrad_stride2_parity_decomposition():
    from monoflex_b200 import backward
    gen = np.random.Generator(np.random.PCG64(91))
    for (B, H, W, Cin, Cout) in ((2, 12, 20, 64, 128), (1, 16, 24, 128, 64)):
        Ho, Wo = H // 2, W // 2
        w = torch.from_numpy((gen.standard_normal((Cout, Cin, 3, 3)) / np.sqrt(Cout * 9)).astype(np.float32)).half().float()
        dy = torch.from_numpy(gen.standard_normal((B, Cout, Ho, Wo)).astype(np.float32)).half().float()
        dx = backward.conv2d_dgrad_stride2(_rows_of(dy), w.cuda(), B, Ho, Wo)
        torch.cuda.synchronize()
        ref = torch.nn.grad.conv2d_input((B, Cin, H, W), w, dy, stride=2, padding=1)
        assert (_nchw_of(dx, B, H, W) - ref).abs().max().item() <= 1e-3 * ref.abs().max().item()


def test_maxpool_upsample_sigmoid_colsum_backward():
    """backward twins of the HBM-bound layers vs torch autograd (CPU fp32) on fp16-representable inputs."""
    from monoflex_b200 import backward
    import torch.nn.functional as F
    gen = np.random.Generator(np.random.PCG64(92))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).half().float()
    # MaxPool2d(2): distinct values (ties carry torch's first-index rule; continuous data has none)
    B, C, H, W = 2, 64, 10, 12
    x = t(gen.standard_normal((B, C, H, W))).requires_grad_(True)
    dy = t(gen.standard_normal((B, C, H // 2, W // 2)))
    F.max_pool2d(x, 2).backward(dy)
    dx = backward.maxpool2_backward(_rows_of(x.detach()), _rows_of(dy), B, H, W)
    assert torch.equal(_nchw_of(dx, B, H, W), x.grad)
    # depth-wise ConvTranspose2d(k = 2f, s = f, p = f/2), f = 2 and 4
    for f in (2, 4):
        B, C, Hi, Wi = 2, 64, 6, 7
        k = 2 * f
        x = t(gen.standard_normal((B, C, Hi, Wi))).requires_grad_(True)
        w = torch.from_numpy(gen.uniform(0.05, 0.5, (C, 1, k, k)).astype(np.float32)).requires_grad_(True)
        dy = t(gen.standard_normal((B, C, Hi * f, Wi * f)))
        F.conv_transpose2d(x, w, None, stride=f, padding=f // 2, groups=C).backward(dy)
        w_taps = w.detach().view(C, k * k).t().contiguous().cuda()
        dx, dw = backward.upsample_backward(_rows_of(x.detach()), w_taps, _rows_of(dy), B, Hi, Wi, f)
        assert (_nchw_of(dx, B, Hi, Wi) - x.grad).abs().max().item() <= 2e-3 * x.grad.abs().max().item()
        dw_ref = w.grad.view(C, k * k).t()
        assert (dw.cpu() - dw_ref).abs().max().item() <= 1e-4 * dw_ref.abs().max().item()
    # sigmoid_hm
    z = t(gen.standard_normal((2, 3, 8, 10)) * 6).requires_grad_(True)
    g = t(gen.standard_normal((2, 3, 8, 10)))
    y = torch.clamp(torch.sigmoid(z), 1e-4, 1 - 1e-4)
    y.backward(g)
    got = backward.sigmoid_clamp_backward(y.detach().cuda(), g.cuda())
    assert (got.cpu() - z.grad).abs().max().item() <= 1e-6
    # column sum (conv-bias gradient)
    m = t(gen.standard_normal((5000, 24)))
    cs = backward.column_sum(m.half().cuda())
    assert (cs.cpu() - m.sum(0)).abs().max().item() <= 1e-4 * m.sum(0).abs().max().item() + 1e-3


def test_edge_gather_backward_is_the_transpose():
    """<edge_gather(feat), d_e> == <feat, edge_gather_bwd(d_e)> (adjoint identity) with the real 832-entry border list."""
    from monoflex_b200._lib import call, stream
    from monoflex_b200 import synthetic as syn
    gen = np.random.Generator(np.random.PCG64(93))
    B, H, W, K = 2, 96, 320, 832
    idx, n, _ = syn.edge_indices()
    edge = idx.unsqueeze(0).repeat(B, 1, 1).cuda()
    feat = torch.from_numpy((gen.standard_normal((B * H * W, 512)) * 0.5).astype(np.float32)).half().cuda()
    ea = torch.zeros(B, K + 2, 256, dtype=torch.half, device="cuda")
    eb = torch.zeros_like(ea)
    call("mf_edge_gather", feat.data_ptr(), 512, 0, 0, 256, edge.data_ptr(), ea.data_ptr(), eb.data_ptr(), B, H, W, K, 320, 96,
         stream())
    da = torch.from_numpy(gen.standard_normal((B, K + 2, 256)).astype(np.float32)).half().cuda()
    db = torch.from_numpy(gen.standard_normal((B, K + 2, 256)).astype(np.float32)).half().cuda()
    dfeat = torch.zeros_like(feat)
    call("mf_edge_gather_bwd", da.data_ptr(), db.data_ptr(), 0, 256, edge.data_ptr(), dfeat.data_ptr(), 512, B, H, W, K, 320, 96,
         stream())
    lhs = (ea.double() * da.double()).sum() + (eb.double() * db.double()).sum()
    rhs = (feat.double() * dfeat.double()).sum()
    assert abs(lhs.item() - rhs.item()) <= 2e-3 * abs(lhs.item())
    touched = (dfeat != 0).any(1).sum().item()
    assert 0 < touched <= 4 * B * K


@pytest.mark.parametrize("case", [(2, 64, 64, 10, 12), (1, 128, 64, 8, 9), (1, 512, 256, 6, 10)])
def test_dcn_backward_tensor_core_path(case):
    """fp16 NHWC DCN backward (two existing tensor-core GEMMs + the sampling / col2im kernels) vs torch autograd through
    the CPU oracle's dcn_v2_forward with mask = sigmoid(pre): dX, d offsets, d mask pre-activation, dW, dB."""
    from monoflex_b200 import backward
    B, C, Co, H, W = case
    gen = np.random.Generator(np.random.PCG64(sum(case)))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    x = t(gen.standard_normal((B, C, H, W))).half().float()
    w = t(gen.standard_normal((Co, C, 3, 3)) / np.sqrt(9 * C)).half().float()
    bias = t(gen.standard_normal(Co) * 0.1)
    off = t(gen.standard_normal((B, 18, H, W)) * 1.5)
    pre = t(gen.standard_normal((B, 9, H, W)))
    dy = t(gen.standard_normal((B, Co, H, W))).half().float()
    leaves = [v.clone().requires_grad_(True) for v in (x, w, bias, off, pre)]
    mo.dcn_v2_forward(leaves[0], leaves[1], leaves[2], leaves[3], torch.sigmoid(leaves[4])).backward(dy)
    om = torch.zeros(B * H * W, 32)
    om[:, :18] = off.permute(0, 2, 3, 1).reshape(-1, 18)
    om[:, 18:27] = torch.sigmoid(pre).permute(0, 2, 3, 1).reshape(-1, 9)
    dx, dom, dw, db = backward.dcn_backward(_rows_of(x), om.cuda(), _rows_of(dy), w.cuda(), B, H, W)
    torch.cuda.synchronize()
    rel = lambda a, b: (a - b).abs().max().item() / b.abs().max().item()
    assert rel(_nchw_of(dx, B, H, W), leaves[0].grad) < 1e-2               # fp16 grad columns + half2 atomics
    assert rel(dw.cpu(), leaves[1].grad) < 3e-3                            # fp16 sampled columns
    assert rel(db.cpu(), leaves[2].grad) < 1e-4
    dom = dom.cpu().view(B, H, W, 32).permute(0, 3, 1, 2)
    assert rel(dom[:, :18], leaves[3].grad) < 1e-2
    assert rel(dom[:, 18:27], leaves[4].grad) < 1e-2
    assert dom[:, 27:].abs().sum().item() == 0


def test_edge_fusion_conv1d_and_head_backward():
    """Backward of the edge-fusion tail (detector_predictor.py:149-158): the Conv1d(256, 256, 3) weight gradient through the
    rectangular (1 x 3) wgrad, and edge_head_add (1x1 Conv1d + indexed add) vs torch autograd on CPU."""
    from monoflex_b200._lib import call, stream
    from monoflex_b200 import synthetic as syn
    import torch.nn.functional as F
    gen = np.random.Generator(np.random.PCG64(94))
    t32 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32))
    B, K, H, W = 2, 832, 96, 320
    # ---- Conv1d(256 -> 256, k = 3) on the replicate-padded [B, K + 2, 256] rows == 1 x 3 convolution, pad 0
    xin = t32(gen.standard_normal((B, 256, K + 2))).half().float()
    dy = t32(gen.standard_normal((B, 256, K)) * 0.1).half().float()
    ref = torch.nn.grad.conv1d_weight(xin, (256, 256, 3), dy)
    xr = xin.permute(0, 2, 1).reshape(-1, 256).contiguous().half().cuda()
    dyr = dy.permute(0, 2, 1).reshape(-1, 256).contiguous().half().cuda()
    dw = torch.empty(256, 256, 1, 3, dtype=torch.float32, device="cuda")
    call("mf_conv2d_wgrad_rect_nhwc_f16", xr.data_ptr(), 256, B, 1, K + 2, 256, dyr.data_ptr(), 256, 256, 1, 3, 1, 0, 0,
         dw.data_ptr(), stream())
    assert (dw.cpu().view(256, 256, 3) - ref).abs().max().item() <= 1e-4 * ref.abs().max().item()
    # ---- edge_head_add backward
    idx, n, _ = syn.edge_indices()
    edge = idx.unsqueeze(0).repeat(B, 1, 1)
    elen = torch.tensor([n, n - 37], dtype=torch.long)
    n_out, ctot, ch0 = 2, 50, 4
    tt = t32(gen.standard_normal((B, K, 256))).half().float().requires_grad_(True)
    w = t32(gen.standard_normal((n_out, 256)) * 0.1).requires_grad_(True)
    bias = t32(gen.standard_normal(n_out)).requires_grad_(True)
    d_out = t32(gen.standard_normal((B, ctot, H, W)))
    out = torch.zeros(B, ctot, H, W)
    for b in range(B):                                           # the reference's python loop, detector_predictor.py:155-158
        L = int(elen[b])
        val = F.conv1d(tt[b].t().unsqueeze(0), w.unsqueeze(-1), bias)[0]           # [n_out, K]
        ex, ey = edge[b, :L, 0], edge[b, :L, 1]
        out[b, ch0:ch0 + n_out, ey, ex] = out[b, ch0:ch0 + n_out, ey, ex] + val[:, :L]
    out.backward(d_out)
    d_t = torch.empty(B, K, 256, dtype=torch.half, device="cuda")
    gw = torch.empty(n_out, 256, device="cuda")
    gb = torch.empty(n_out, device="cuda")
    th, wc, ec, lc, dc = tt.detach().half().cuda(), w.detach().cuda(), edge.cuda(), elen.cuda(), d_out.cuda()
    call("mf_edge_head_add_bwd", th.data_ptr(), wc.data_ptr(), n_out, ec.data_ptr(), lc.data_ptr(), dc.data_ptr(), ctot, ch0,
         d_t.data_ptr(), gw.data_ptr(), gb.data_ptr(), B, K, H, W, stream())
    assert (d_t.float().cpu() - tt.grad).abs().max().item() <= 2e-3 * tt.grad.abs().max().item()
    assert (gw.cpu() - w.grad).abs().max().item() <= 1e-4 * w.grad.abs().max().item()
    assert (gb.cpu() - bias.grad).abs().max().item() <= 1e-4 * bias.grad.abs().max().item()


def test_train_mode_forward_losses_vs_reference_golden():
    """Train-mode FORWARD of the whole detector on the CUDA kernels (batch-statistics BN / IABN / BN1d, unfused head, 11-term
    loss) against the losses of the UNMODIFIED reference in train() mode (tests/golden/train_step_2x384x1280.npz). fp16
    operands end to end, so the comparison is at the few-percent level per loss term; the exact-arithmetic check of every
    operator is in the tests above."""
    import os
    from conftest import GOLDEN
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    gold = np.load(os.path.join(GOLDEN, "train_step_2x384x1280.npz"))
    model = KeypointDetector(default_cfg()).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    rm_before = model.backbone.base.level2.tree1.bn1.running_mean.clone()
    loss_dict, log = model.train_forward_losses(images, targets)
    torch.cuda.synchronize()
    assert list(loss_dict) == mo.LOSS_NAMES
    for k in mo.LOSS_NAMES:
        ref = float(gold["loss_" + k])
        got = loss_dict[k].item()
        assert np.isfinite(got) and abs(got - ref) <= 5e-2 * max(abs(ref), 0.05), (k, got, ref)
    assert not torch.equal(model.backbone.base.level2.tree1.bn1.running_mean, rm_before)      # running statistics moved
    # the reference call `loss_dict, log_loss_dict = model(images, targets)` (engine/trainer.py:109) is the same path and its
    # losses carry the backward tape (model/detector.py::_TapeBridge)
    l2, log2 = model(images, targets)
    assert list(l2) == mo.LOSS_NAMES and all(v.requires_grad for v in l2.values()) and isinstance(log2, dict)
    with pytest.raises(ValueError):
        model(images)                                                                         # model/detector.py:27-28


def test_tape_predictor_backward_vs_reference_gradients():
    """First complete slice of the training tape: loss -> sigmoid_hm -> edge fusion -> 1x1 heads -> InPlaceABN -> 3x3 convs,
    composed from the backward operators (monoflex_b200/tape.py::predictor_backward), against the UNMODIFIED reference's
    autograd in train mode (golden: gradient norm of every predictor parameter, norm and a strided sample of the feature-map
    gradient). Forward activations are fp16 here and fp32 there, so the comparison is at the 10 % level on norms; the
    operators themselves are checked tightly above."""
    import os
    from conftest import GOLDEN
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.tape import predictor_backward
    from monoflex_b200.model.detector import KeypointDetector
    gold = np.load(os.path.join(GOLDEN, "train_step_2x384x1280.npz"))
    model = KeypointDetector(default_cfg()).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    feats = model.backbone.train_forward(images)
    pred_mod = model.heads.predictor
    pred = pred_mod.train_forward(feats, targets)
    c = pred["cls"].detach().clone().requires_grad_(True)
    r = pred["reg"].detach().clone().requires_grad_(True)
    loss_dict, _ = model.heads.loss_evaluator({"cls": c, "reg": r}, targets)
    S = 256.0                                                   # loss scale: gradients travel in fp16
    (S * sum(loss_dict.values())).backward()
    grads, d_feat = predictor_backward(pred_mod, pred_mod.last_plan, c.grad, r.grad)
    torch.cuda.synchronize()
    ref = dict(zip([str(n) for n in gold["grad_names"]], gold["grad_norms"]))
    checked = 0
    for name, g in grads.items():
        want = ref["heads.predictor." + name]
        got = float(g.double().norm()) / S
        if want < 1e-6:                                          # conv biases in front of a train-mode BN: analytically zero
            assert got < 1e-3, (name, got, want)
            continue
        assert abs(got - want) <= 0.12 * want, (name, got, want)
        checked += 1
    assert checked >= 50 and len(grads) == len(list(pred_mod.parameters()))
    fn = float(d_feat.double().norm()) / S
    assert abs(fn - float(gold["grad_features_norm"])) <= 0.12 * float(gold["grad_features_norm"])
    B, H, W = 2, 96, 320
    got = (d_feat.float().cpu().view(B, H, W, 64).permute(0, 3, 1, 2).reshape(-1)[::997] / S).numpy()
    want = gold["grad_features_sample"]
    cos = float((got * want).sum() / (np.linalg.norm(got) * np.linalg.norm(want)))
    assert cos > 0.98, cos


def test_full_backward_tape_with_stem_vs_reference_gradients():
    """Whole-network backward: predictor + backbone replays (tape.py) composed from the backward operators, against the
    UNMODIFIED reference's autograd in train mode (gradient norm of every parameter, the stem's 7x7 weight included). fp16
    activations and gradients over ~60 layers vs fp32 there: norms are compared at the 25 % level, most are within a few
    per cent."""
    import os
    from conftest import GOLDEN
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.tape import backbone_backward, predictor_backward
    from monoflex_b200.model.detector import KeypointDetector
    gold = np.load(os.path.join(GOLDEN, "train_step_2x384x1280.npz"))
    model = KeypointDetector(default_cfg()).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    model.train()
    fields = syn.make_train_targets(2, empty_image=0)
    images = syn.make_images(2, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    feats = model.backbone.train_forward(images)
    pred_mod = model.heads.predictor
    pred = pred_mod.train_forward(feats, targets)
    c = pred["cls"].detach().clone().requires_grad_(True)
    r = pred["reg"].detach().clone().requires_grad_(True)
    loss_dict, _ = model.heads.loss_evaluator({"cls": c, "reg": r}, targets)
    S = float(os.environ.get("MF_TAPE_LOSS_SCALE", "64"))     # gradients travel in fp16 rows
    (S * sum(loss_dict.values())).backward()
    _, d_feat = predictor_backward(pred_mod, pred_mod.last_plan, c.grad, r.grad)
    grads = backbone_backward(model.backbone, model.backbone.last_plan, d_feat)
    torch.cuda.synchronize()
    ref = dict(zip([str(n) for n in gold["grad_names"]], gold["grad_norms"]))
    # every backbone parameter the reference's autograd gives a gradient
    missing = sorted(n for n, v in ref.items() if n.startswith("backbone.") and v > 0 and n[len("backbone."):] not in grads)
    devs = []
    for name, g in grads.items():
        want = ref["backbone." + name]
        got = float(g.double().norm()) / S
        assert np.isfinite(got), name
        if want < 1e-5:                                          # conv biases in front of a train-mode BN: analytically zero
            continue
        devs.append((abs(got - want) / want, name, got, want))
    if os.environ.get("MF_TAPE_DUMP"):
        with open(os.environ["MF_TAPE_DUMP"], "w") as fh:
            for d, name, got, want in devs:
                fh.write("%-60s got %.6g want %.6g dev %+.3f\n" % (name, got, want, (got - want) / want))
    devs.sort(reverse=True)
    print("worst:", devs[:5], "median dev:", devs[len(devs) // 2][0], "n:", len(devs), "missing:", missing)
    assert not missing, missing
    assert "base.base_layer.0.weight" in [name for _, name, _, _ in devs]
    assert len(devs) >= 150
    # the worst deviations sit on the two earliest full-resolution BN layers, where the fp16 rounding of ~60 layers of
    # gradient flow and of the forward activations has accumulated the most. The median moves with the summation ORDER of the
    # batch statistics (partial-sum grid of the statistics kernels; the BN operators themselves pass
    # test_batchnorm_train_forward_backward unchanged): this synthetic network amplifies last-bit
    # differences of the forward, which is what the fp16-forward emulation yardstick of
    # test_reference_training_loop_unchanged quantifies.
    assert devs[0][0] < 0.40, devs[:5]
    assert devs[len(devs) // 10][0] < 0.25
    assert devs[len(devs) // 2][0] < 0.10


def _train_setup(B=2):
    import os
    from conftest import GOLDEN
    from monoflex_b200 import synthetic as syn
    from monoflex_b200.model.detector import KeypointDetector
    gold = np.load(os.path.join(GOLDEN, "train_step_2x384x1280.npz"))
    cfg = default_cfg()
    model = KeypointDetector(cfg).cuda()
    model.load_state_dict(syn.make_state_dict(seed=0), strict=False)
    fields = syn.make_train_targets(B, empty_image=0)
    images = syn.make_images(B, 384, 1280, seed=1).cuda()
    targets = [t.to("cuda") for t in syn.make_train_param_lists(fields)]
    return gold, cfg, model, images, targets


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float((a @ b) / (a.norm() * b.norm()).clamp_min(1e-300))


def test_reference_training_loop_unchanged():
    """engine/trainer.py:103-126 verbatim with the reference's own optimiser class: `loss_dict, log = model(images, targets);
    losses = sum(...); optimizer.zero_grad(); losses.backward(); optimizer.step()` with torch.optim.AdamW over the reference's
    one-group-per-tensor params (solver/__init__.py:10-37). Checks against the unmodified reference's train-mode golden: the
    total loss, WHICH parameters receive gradients (autograd leaves the unused `project` convs at None), and - element-wise,
    not just by norm - the three gradients stored in full (stem 7x7 weight, a level-2 BN gamma, the class-head bias)."""
    from monoflex_b200 import solver
    gold, cfg, model, images, targets = _train_setup()
    model.train()
    optimizer = torch.optim.AdamW(solver.get_model_params(model, cfg), lr=cfg.SOLVER.BASE_LR, weight_decay=cfg.SOLVER.WEIGHT_DECAY,
                                  betas=(0.9, 0.99))
    w0 = model.backbone.base.level3.tree1.tree1.conv1.weight.detach().clone()
    loss_dict, log_loss_dict = model(images, targets)
    losses = sum(loss for loss in loss_dict.values())
    assert set(loss_dict) == {k[5:] for k in gold.files if k.startswith("loss_")}
    assert abs(losses.item() - float(gold["total"])) <= 0.05 * float(gold["total"])
    optimizer.zero_grad()
    losses.backward()
    ref = dict(zip([str(n) for n in gold["grad_names"]], gold["grad_norms"]))
    params = dict(model.named_parameters())
    unused = {n for n, p in params.items() if p.grad is None}
    for n, v in ref.items():
        if v > 0:
            assert params[n].grad is not None, n                          # every gradient the reference's autograd produces
    # exactly the parameters outside the reference's forward graph stay at None (the outer `project` of the 2-level trees,
    # dla_dcn.py:249; the golden stores norm 0 for them), like autograd leaves them
    assert unused == {n for n in params if ".project." in n and n.count("tree") == 0 and ("level3" in n or "level4" in n)}, sorted(unused)
    # Element-wise gradient check, along the whole depth of the network (17 tensors stored in full by oracle/make_golden_train.py).
    # Yardstick: tests/golden/grad_cos_f16_forward_emulation.json = cosine between the reference's gradients and an EXACT fp32
    # backward (torch autograd) evaluated on the oracle forward with only the kernels' fp16 rounding points emulated
    # (tools/grad_emulation_cpu.py). On this synthetic network (random weights + batch-statistics BN: the chaotic regime) that
    # alone moves the gradients to cos 0.87-0.98 in the backbone - the derivative is ill-conditioned in the point it is taken
    # at, whatever computes it. The tape has to stay within 0.08 of that yardstick (a different realisation of the forward
    # rounding plus its own fp16 gradient rounding), and the head, whose forward is two layers deep, has to be right outright.
    import json
    from conftest import GOLDEN
    yard = json.load(open(os.path.join(GOLDEN, "grad_cos_f16_forward_emulation.json")))["cos"]
    report = []
    for name, want_np in ((k[5:], gold[k]) for k in gold.files if k.startswith("grad_") and k[5:] in yard):
        got, want = params[name].grad.detach().cpu(), torch.from_numpy(want_np)
        c = _cos(got, want)
        ratio = float(got.double().norm() / want.double().norm())
        report.append((name, c, yard[name], ratio))
        print("%-58s cos %.5f (fp16-forward yardstick %.5f) |g|/|ref| %.4f" % (name, c, yard[name], ratio))
    for name, c, y, ratio in report:
        if name.endswith("node_1.conv.bias"):
            continue          # a bias in front of a batch-statistics BN: the true gradient is 0, both sides hold rounding noise
        assert c > y - 0.08, (name, c, y)
        assert 0.8 < ratio < 1.2, (name, ratio)
        if name.startswith("heads."):
            assert c > 0.985, (name, c)
    optimizer.step()
    assert not torch.equal(model.backbone.base.level3.tree1.tree1.conv1.weight.detach(), w0)
    with torch.no_grad():
        l2, _ = model(images, targets)
    total2 = sum(v.item() for v in l2.values())
    assert np.isfinite(total2) and total2 < 1.01 * losses.item()


def test_captured_train_step_matches_eager_and_late_log_reads():
    """The whole optimisation step replayed from ONE CUDA graph (Trainer(use_cuda_graph=True): forward, loss, backward, finite
    guard, AdamW with the device-side step counter) against the eager loop on a twin model: per-step logged losses agree,
    the parameter updates point the same way. The captured trainer's logs are read LATE (DeferredLog.snapshot: after the
    following replays have overwritten the device buffer) - what bench.py's end-to-end loop does."""
    from monoflex_b200.train import Trainer
    _, cfg, model_a, images, targets = _train_setup()
    _, _, model_b, _, _ = _train_setup()
    ta = Trainer(model_a, cfg, loss_scale=128.0)
    tb = Trainer(model_b, cfg, loss_scale=128.0, use_cuda_graph=True, graph_warmup=2)
    p0 = ta.optimizer.arena.params.clone()
    assert torch.equal(p0, tb.optimizer.arena.params)
    logs_a, logs_b = [], []
    for _ in range(4):
        logs_a.append(ta.step(images, targets)[1])
        logs_b.append(tb.step(images, targets, sync_log=False)[1])
    assert tb._graph is not None                                   # steps 2 and 3 were graph replays
    logs_b = [l.resolve() for l in logs_b]
    for i, (la, lb) in enumerate(zip(logs_a, logs_b)):
        ta_tot, tb_tot = sum(la[k] for k in la if k.endswith("_loss")), sum(lb[k] for k in lb if k.endswith("_loss"))
        # the scatter atomics of the DCN backward make two runs differ in the last bits and this synthetic network amplifies
        # that from step to step (two EAGER runs drift the same way): tight on the first replay, loose after it
        tol = 0.03 if i <= 2 else 0.25
        assert np.isfinite(tb_tot) and abs(ta_tot - tb_tot) <= tol * abs(ta_tot), (i, ta_tot, tb_tot)
    assert logs_b[0] != logs_b[3]                                  # four different evaluations, not one buffer read four times
    da, db = ta.optimizer.arena.params - p0, tb.optimizer.arena.params - p0
    assert float(da.norm()) > 0 and _cos(da, db) > 0.5, _cos(da, db)
    assert tb.optimizer.skipped_steps() == 0 and tb.optimizer.step_count == ta.optimizer.step_count == 4


def test_end_to_end_train_steps():
    """Trainer (monoflex_b200/train.py) = the same loop around the arena optimiser: forward -> loss -> whole-network backward ->
    gradient arena -> finite guard + one-launch AdamW, two steps on one batch: first-step loss equals the reference's
    train-mode total, every parameter of the forward graph receives a gradient (the stem's 7x7 weight gradient checked
    against the reference), parameters move, the loss of the updated model is finite and lower; a poisoned gradient skips
    the update instead of reaching the parameters."""
    import time
    from monoflex_b200.train import Trainer
    gold, cfg, model, images, targets = _train_setup()
    tr = Trainer(model, cfg, loss_scale=128.0)
    w0 = model.backbone.base.level3.tree1.tree1.conv1.weight.detach().clone()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    loss1, _ = tr.step(images, targets)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    total1 = sum(v.item() for v in loss1.values())
    assert abs(total1 - float(gold["total"])) <= 0.05 * float(gold["total"])
    ref = dict(zip([str(n) for n in gold["grad_names"]], gold["grad_norms"]))
    used = {n for n, v in ref.items() if v > 0}
    got_names = set(model.last_grad_names)
    assert used <= got_names, sorted(used - got_names)[:5]
    # beyond those only parameters whose reference gradient is exactly zero on this batch (the truncation-offset branch: no
    # truncated object in the synthetic labels) - never the convs outside the forward graph
    assert all(ref[n] == 0 and ".project." not in n for n in got_names - used), sorted(got_names - used)
    stem = model.backbone.base.base_layer[0].weight.grad
    got = float(stem.double().norm())
    assert abs(got - ref["backbone.base.base_layer.0.weight"]) <= 0.10 * ref["backbone.base.base_layer.0.weight"], got
    assert not torch.equal(model.backbone.base.level3.tree1.tree1.conv1.weight.detach(), w0)
    unused = model.backbone.base.level3.project[0].weight          # outside the forward graph: never decayed, never moved
    u0 = unused.detach().clone()
    loss2, _ = tr.step(images, targets)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    total2 = sum(v.item() for v in loss2.values())
    print("train step wall s:", t1 - t0, t2 - t1, "loss:", total1, "->", total2)
    assert np.isfinite(total2) and total2 < 1.01 * total1          # one AdamW step at lr 3e-4 must not blow the loss up
    assert torch.equal(unused.detach(), u0)
    assert tr.optimizer.skipped_steps() == 0
    # finite guard: a non-finite gradient must not touch parameters or moments
    snap = tr.optimizer.arena.params.clone()
    model.loss_scale = 1e30                                          # overflows the fp16 gradient flow
    tr.step(images, targets)
    assert tr.optimizer.skipped_steps() == 1 and torch.equal(tr.optimizer.arena.params, snap)
    assert bool(torch.isfinite(tr.optimizer.exp_avg).all())
