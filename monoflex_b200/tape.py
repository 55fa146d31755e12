"""Whole-network backward from what the train-mode forward plans kept, every layer's backward one operator of backward.py:

  * predictor_backward: the predictor (detector_predictor.py:121-165) from the activations its plan kept (`plan.ctx`,
    model/head/detector_predictor.py): loss gradients -> sigmoid_hm -> edge-fusion tail -> 1x1 heads -> InPlaceABN -> the
    nine 3x3 convs -> gradient of the backbone's feature map;
  * backbone_backward: the backbone (DLA-34 base + DLAUp/IDAUp with DCNv2, model/backbone/dla_dcn.py) from the tape its
    plan recorded (engine.Plan.tape), one record per emitted layer, replayed in reverse emission order.

Both return {parameter name: fp32 gradient} for every parameter the forward used. Gradients flow in fp16 NHWC rows, so the
caller multiplies the loss gradients by a loss scale (>= 128) and divides the results by it, like any fp16 training step.

Backbone bookkeeping: every activation buffer of the plan gets a zero-initialised fp16 gradient buffer of the same shape
(channel slices of a Root concatenation share their parent's, exactly like the forward shares storage) and every backward
operator accumulates into it. That makes the result independent of which consumer of a multiply-used activation runs first.
"""
import torch

from . import backward, engine
from ._lib import call, stream


def _collector(module):
    """({parameter name: fp32 gradient}, put(param, value)) for the parameters of `module`; put(None, ...) does nothing"""
    names = {id(p): n for n, p in module.named_parameters()}
    grads = {}

    def put(param, value):
        if param is not None:
            grads[names[id(param)]] = value.reshape(param.shape).float()
    return grads, put


def _put_bn(put, results):
    for mod, dgamma, dbeta in results:
        put(mod.weight, dgamma)
        put(mod.bias, dbeta)


@torch.no_grad()
def predictor_backward(pred, plan, grad_cls, grad_reg):
    """pred: the `_predictor` module in train mode, plan: its last train-mode plan (pred.last_plan), grad_cls [B,3,H,W] /
    grad_reg [B,50,H,W] fp32: (scaled) loss gradients w.r.t. the predictor outputs.
    Returns (grads, d_features: [B*H*W, 64] fp16 rows)."""
    ctx = plan.ctx
    x, hid = ctx["x"], ctx["hid"]
    B, H, W, hc = x.B, x.H, x.W, pred.head_conv
    M, dev = B * H * W, grad_reg.device
    HW = H * W
    grads, put = _collector(pred)
    branches = [pred.class_head] + list(pred.reg_features)
    head_lists = [[pred.class_head[2]]] + [list(h) for h in pred.reg_heads]
    nb = len(branches)
    # ---- sigmoid_hm
    g_logits = backward.sigmoid_clamp_backward(plan.cls, grad_cls.contiguous())
    d_hid = torch.zeros(M, nb * hc, dtype=torch.half, device=dev)          # gradient of the activated hidden map [M, 2304]
    # ---- 1x1 heads: weight / bias gradients and d_hid = dY W
    dys = []
    for i, heads in enumerate(head_lists):
        n_i = sum(h.weight.shape[0] for h in heads)
        src = g_logits if i == 0 else grad_reg[:, ctx["ch0s"][i - 1]:ctx["ch0s"][i - 1] + n_i].contiguous()
        dy = torch.zeros(M, 32, dtype=torch.half, device=dev)
        call("mf_nchw_f32_to_nhwc_f16", src.data_ptr(), dy.data_ptr(), B, n_i, HW, 32, stream())
        dys.append(dy)
        dw = backward.conv2d_wgrad(engine.Act.on(hid.buf, B, H, W, hc, hid.ch_off + i * hc), dy, B, H, W, 1)
        db = backward.column_sum(dy)
        r = 0
        for h in heads:
            n = h.weight.shape[0]
            put(h.weight, dw[r:r + n])
            put(h.bias, db[r:r + n])
            r += n

    def heads_dgrad(P):
        for i, heads in enumerate(head_lists):
            wcat = torch.cat([h.weight.detach().float().reshape(h.weight.shape[0], hc) for h in heads], 0)      # [n_i, 256]
            wd = torch.zeros(hc, 32, 1, 1, dtype=torch.float32, device=dev)
            wd[:, :wcat.shape[0], 0, 0] = wcat.t()
            P.conv(engine.Act.on(dys[i], B, H, W), wd, 1, 0, None, act=engine.ACT_NONE, out=engine.Act.on(d_hid, B, H, W, hc, i * hc))
    backward.run_plan(dev, heads_dgrad)
    # ---- edge-fusion tail
    if pred.enable_edge_fusion:
        K = ctx["K_edge"]
        d_e = []
        for seq, g_map, ctot, ch0, src in ((pred.trunc_heatmap_conv, g_logits, pred.num_classes, 0, ctx["ea"]),
                                          (pred.trunc_offset_conv, grad_reg.contiguous(), pred.num_reg, ctx["off_ch0"], ctx["eb"])):
            entries = ctx["bn"][id(seq[1])]
            t_y = entries[0][2]
            n_out = seq[3].weight.shape[0]
            w2 = seq[3].weight.detach().float().reshape(n_out, hc).contiguous()
            d_t = torch.empty(B * K, hc, dtype=torch.half, device=dev)
            dw2 = torch.empty(n_out, hc, dtype=torch.float32, device=dev)
            db2 = torch.empty(n_out, dtype=torch.float32, device=dev)
            call("mf_edge_head_add_bwd", t_y.ptr(), w2.data_ptr(), n_out, plan.edge_idx.data_ptr(), plan.edge_len.data_ptr(),
                 g_map.data_ptr(), ctot, ch0, d_t.data_ptr(), dw2.data_ptr(), db2.data_ptr(), B, K, H, W, stream())
            put(seq[3].weight, dw2)
            put(seq[3].bias, db2)
            d_raw = torch.empty(B * K, hc, dtype=torch.half, device=dev)
            _put_bn(put, backward.bn_backward(entries, d_t, d_raw, engine.ACT_NONE))
            dw1 = torch.empty(hc, hc, 1, 3, dtype=torch.float32, device=dev)
            call("mf_conv2d_wgrad_rect_nhwc_f16", src.ptr(), src.ld, B, 1, K + 2, hc, d_raw.data_ptr(), hc, hc, 1, 3, 1, 0, 0,
                 dw1.data_ptr(), stream())
            put(seq[0].weight, dw1)
            put(seq[0].bias, backward.column_sum(d_raw))
            # Conv1d data gradient: correlation of d_raw with the flipped, transposed taps, 2 columns of zero padding
            w5 = torch.zeros(hc, hc, 5, 3, dtype=torch.float32, device=dev)
            w5[:, :, 2, :] = seq[0].weight.detach().float().flip(2).transpose(0, 1)
            d_e.append(backward.run_plan(dev, lambda P: P.conv(engine.Act.on(d_raw, B, 1, K), w5, 1, 2, None, act=engine.ACT_NONE)))
        cols = (0, (pred.offset_index[0] + 1) * hc)
        call("mf_edge_gather_bwd", d_e[0].ptr(), d_e[1].ptr(), cols[0], cols[1], plan.edge_idx.data_ptr(), d_hid.data_ptr(), nb * hc,
             B, H, W, K, pred.output_width, pred.output_height, stream())
    # ---- InPlaceABN (leaky 0.01) per branch, in place on the gradient buffer: d_hid -> d_hid_raw
    entries = [e for b in branches for e in ctx["bn"][id(b[1])]]
    _put_bn(put, backward.bn_backward(entries, d_hid, d_hid, engine.ACT_LEAKY, abs_weight=True))
    # ---- the nine 3x3 convolutions: one wgrad with Cout = 2304, one dgrad with Cin = 2304
    dw_all = backward.conv2d_wgrad(x, d_hid, B, H, W, 3, 1, 1)
    for i, b in enumerate(branches):
        put(b[0].weight, dw_all[i * hc:(i + 1) * hc])
    w_all = torch.cat([b[0].weight.detach() for b in branches], 0)
    return grads, backward.conv2d_dgrad(d_hid, w_all, B, H, W, 1)


@torch.no_grad()
def backbone_backward(backbone, plan, d_feat_rows, observe=None):
    """backbone: DLASeg in train mode, plan: its last train-mode plan (backbone.last_plan), d_feat_rows [B*H/4*W/4, 64] fp16:
    (scaled) gradient of the loss w.r.t. the backbone's output feature map. Returns grads.
    observe: optional observe(rec, grad, done), called before (done=False) and after (done=True) each tape record is
    replayed, with `grad` the accessor below (activation -> engine.Act over its gradient buffer). It exists for the
    layer-by-layer test (tests/test_gpu_tape_layers.py), which checks every record on the inputs it actually saw."""
    grads, put = _collector(backbone)
    bufs = {}

    def grad(a):
        """engine.Act over the gradient buffer of activation `a`"""
        g = bufs.get(a.buf.data_ptr())
        if g is None:
            g = bufs[a.buf.data_ptr()] = torch.zeros_like(a.buf)
        return engine.Act.on(g, a.B, a.H, a.W, a.C, a.ch_off)

    backward.add_rows(grad(plan.output), d_feat_rows.contiguous())
    for rec in reversed(plan.tape):
        if observe is not None:
            observe(rec, grad, False)
        kind, x, y = rec["kind"], rec["x"], rec["y"]
        if kind == "conv_bn":
            raw, residual = rec["raw"], rec["residual"]
            d_raw = torch.empty(raw.M, raw.C, dtype=torch.half, device=raw.buf.device)
            d_res = torch.empty_like(d_raw) if residual is not None else None
            _put_bn(put, backward.bn_backward(rec["bn"], grad(y), d_raw, rec["act"], rec["abs_weight"], d_res))
            if residual is not None:
                backward.add_rows(grad(residual), d_res)
            dw, db = backward.conv_backward(x, rec["weight"], rec["bias"], rec["stride"], rec["pad"], d_raw,
                                            None if x is plan.input else grad(x))
            put(rec["weight"], dw)
            put(rec["bias"], db)
        elif kind == "dcn":
            raw, mod = rec["raw"], rec["mod"]
            d_raw = torch.empty(raw.M, raw.C, dtype=torch.half, device=raw.buf.device)
            _put_bn(put, backward.bn_backward(rec["bn"], grad(y), d_raw, engine.ACT_RELU))
            _, dom, dw, db = backward.dcn_backward(x, rec["om"], d_raw, mod.weight, x.B, x.H, x.W, grad(x))
            put(mod.weight, dw)
            put(mod.bias, db)
            # offset / mask convolution (3x3, bias, 27 -> padded 32 output channels): its pre-activation gradient is `dom`
            om = mod.conv_offset_mask
            dw, db = backward.conv_backward(x, om.weight, om.bias, 1, 1, dom.half(), grad(x))
            put(om.weight, dw)
            put(om.bias, db)
        elif kind == "maxpool2":
            backward.maxpool2_backward(x, grad(y), x.B, x.H, x.W, grad(x))
        elif kind == "upsample_add":
            skip = rec["skip"]
            _, dw = backward.upsample_backward(x, rec["wt"], grad(y), x.B, x.H, x.W, rec["f"], grad(x),
                                              grad(skip) if skip is not None else None)
            put(rec["weight"], dw.t().contiguous())
        else:
            raise NotImplementedError("tape record %r" % kind)
        if observe is not None:
            observe(rec, grad, True)
    return grads
