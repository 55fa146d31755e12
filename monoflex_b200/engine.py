"""Inference plan builder: turns the (reference-keyed) parameters of the detector into a static list of C-ABI kernel
launches over pre-allocated NHWC fp16 buffers.

Data layout in HBM (DESIGN.md §3): every activation is a row-major [B*H*W, ld] fp16 matrix ("pixel rows"); a logical
tensor may be a channel slice of a wider buffer, which is how the Root concatenations (dla_dcn.py:195-203) are written
in place by their producers instead of being copied by torch.cat. Weights are repacked once per plan into
[n_pad, k_pad] fp16 (k = tap*Cin + c) and eval-mode BatchNorm / InPlaceABN / conv biases are folded into a per-channel
fp32 (scale, shift) pair applied in the GEMM epilogue.
"""
import math

import torch

from . import _lib

import os

ACT_NONE, ACT_RELU, ACT_LEAKY, ACT_OFFMASK = 0, 1, 2, 3
OUT_F16_NHWC, OUT_F32_NHWC, OUT_F32_NCHW = 0, 1, 2
BN_EPS = 1e-5

PRECISIONS = ("strict", "fast")


def default_precision():
    """Inference arithmetic (DESIGN.md §4 "Precision modes"): 'strict' (default) = every activation / weight an fp16 hi/lo
    pair, three tensor-core products per K step, fp32-grade results (<= 1e-3 of the reference end to end, the parity
    contract); 'fast' = one fp16 product (2-4e-3 end to end). `MF_PRECISION` overrides the default; a model can be switched
    with `KeypointDetector.set_precision()`."""
    p = os.environ.get("MF_PRECISION", "strict")
    if p not in PRECISIONS:
        raise ValueError("MF_PRECISION must be one of %s" % (PRECISIONS,))
    return p


class Act(object):
    """Logical NHWC fp16 activation [B,H,W,C]; storage is assigned at Plan.finalize()."""

    def __init__(self, B, H, W, C):
        self.B, self.H, self.W, self.C = B, H, W, C
        self.buf = None      # torch.half tensor [B*H*W, ld]
        self.owner = None    # concat group this activation is a slice of
        self.ch_off = 0
        self.npar = 0        # > 0: planar stem layout with `npar` column parities (16-byte pixels)
        self.split = False   # strict precision: rows are [hi channels | lo channels], lo block `lo` elements after hi

    @classmethod
    def on(cls, buf, B, H, W, C=None, ch_off=0):
        """activation over caller-owned rows `buf` [B*H*W, ld] fp16: channels [ch_off, ch_off + C), C defaults to the rest"""
        a = cls(B, H, W, buf.shape[1] - ch_off if C is None else C)
        a.buf, a.ch_off = buf, ch_off
        return a

    @property
    def M(self):
        return self.B * self.H * self.W

    @property
    def ld(self):
        return self.buf.shape[1]

    def ptr(self):
        return self.buf.data_ptr() + 2 * self.ch_off

    @property
    def lo(self):
        """element offset of the lo block of a split activation (0 for plain fp16 activations)"""
        return self.buf.shape[1] // 2 if self.split else 0

    def nchw_view(self):
        """torch view [B,C,H,W] of this activation (zero-copy, channels-last strides, for NHWC rows; a reshaped copy for
        the planar stem layout [B][H][C/8 x npar][W/npar][8])."""
        if self.npar:
            P, Wg = self.C // 8, self.W // self.npar
            if self.split:          # pair planes: hi planes then lo planes
                v = self.buf.view(self.B, self.H, 2, P, self.npar, Wg, 8).float().sum(2).permute(0, 2, 5, 1, 4, 3)
            else:
                v = self.buf.view(self.B, self.H, P, self.npar, Wg, 8).permute(0, 2, 5, 1, 4, 3)
            return v.reshape(self.B, self.C, self.H, self.W)
        if self.split:
            # hi + lo as a fresh fp32 NCHW tensor (one small kernel); `_mf_act` lets the predictor find the pair rows again
            out = torch.empty(self.B, self.C, self.H, self.W, dtype=torch.float32, device=self.buf.device)
            _lib.call("mf_split_to_nchw_f32", self.ptr(), self.ld, self.lo, out.data_ptr(), self.B, self.C, self.H * self.W,
                      _lib.stream())
            out._mf_act = self
            return out
        return self.buf.view(self.B, self.H, self.W, -1)[..., self.ch_off:self.ch_off + self.C].permute(0, 3, 1, 2)


_CONST_VECS = {}


def _const_vec(value, n, device):
    """read-only fp32 vector of `n` copies of `value` (never written by any kernel: scale / shift of identity epilogues)"""
    key = (float(value), str(device))
    v = _CONST_VECS.get(key)
    if v is None or v.numel() < n:
        v = torch.full((max(n, 4096),), float(value), dtype=torch.float32, device=device)
        _CONST_VECS[key] = v
    return v[:n]


class Plan(object):
    def __init__(self, device, train=False, strict=False):
        """strict=True: strict-precision inference plan (hi/lo fp16 pairs, csrc/mf_split.cu + the split paths of
        csrc/mf_igemm2.cu). train=True: every conv/DCN followed by a normalisation layer is emitted as a raw convolution + the training-mode
        BatchNorm kernels (batch statistics, running-stat update, fused residual + activation; csrc/mf_bn_train.cu) instead
        of folding eval statistics into the GEMM epilogue. `bn_saved` lists (module, raw, y, stats) per layer for a backward
        tape. Forward only so far (DESIGN.md, "Training tape")."""
        self.device = device
        self.train = train
        self.strict = strict
        if strict and train:
            raise NotImplementedError("strict precision is an inference mode; training plans run the fp16 kernels")
        self.bn_saved = []
        self.tape = []       # train mode: one record per emitted layer, consumed in reverse by monoflex_b200/tape.py
        self.acts = []
        self.groups = []     # (total_C, [acts]) concat groups
        self.ops = []        # (name, fn_name, argbuilder) resolved at finalize
        self.keep = []       # tensors that must outlive the plan (packed weights, scale/shift, ...)
        self.launches = []   # (fn, args) after finalize
        self.n_launch = 0
        self.pack_descs = [] # train mode: (src fp32 tensor, dst ptr, cout, cin, taps, cin_pad, n_pad, k_pad) re-packed on every run

    # ---- symbolic construction
    def act(self, B, H, W, C, split=None):
        a = Act(B, H, W, C)
        a.split = self.strict if split is None else split
        self.acts.append(a)
        return a

    def concat(self, parts):
        """Return an Act that is the channel concatenation of `parts`, placing every part as a slice of one buffer."""
        B, H, W = parts[0].B, parts[0].H, parts[0].W
        total = sum(p.C for p in parts)
        cat = self.act(B, H, W, total, split=parts[0].split)
        off = 0
        for p in parts:
            assert p.owner is None and (p.B, p.H, p.W) == (B, H, W), "activation already placed in another concat"
            assert p.split == cat.split
            p.owner, p.ch_off = cat, off
            off += p.C
        return cat

    def add(self, fn_name, argbuilder):
        self.ops.append((fn_name, argbuilder))

    def add_py(self, fn):
        """a host callable executed in launch order by run() (device-side torch ops only: no host sync, graph-capturable).
        Train-mode plans use it to refresh what an inference plan bakes in at build time - derived copies of parameters
        that the optimiser changes every step."""
        self.ops.append(("__py__", fn))

    def finalize(self):
        for a in self.acts:
            if a.owner is None and a.buf is None:          # a.buf already set = caller-owned storage bound before finalize
                if a.npar:
                    a.buf = torch.empty((2 if a.split else 1) * a.M * a.C // 8, 8, dtype=torch.half, device=self.device)
                else:
                    a.buf = torch.empty(a.M, (2 if a.split else 1) * a.C, dtype=torch.half, device=self.device)
        for a in self.acts:
            if a.owner is not None:
                root, off = a, 0
                while root.owner is not None:
                    off += root.ch_off
                    root = root.owner
                a.buf, a.ch_off = root.buf, off
                a.owner = None
        lib = _lib.load()
        if self.pack_descs:
            # ONE batched re-pack of every weight from its live parameter at the start of each run (weights only change between
            # runs); descriptor table on the device, see mf_pack_conv_weights_batched
            rows = [[src.data_ptr(), dst, cout | (cin << 32), taps | (cin_pad << 32), n_pad | (k_pad << 32)]
                    for (src, dst, cout, cin, taps, cin_pad, n_pad, k_pad) in self.pack_descs]
            table = torch.tensor(rows, dtype=torch.int64).to(self.device)
            self.keep.append(table)
            n_desc = len(rows)
            self.launches.append((lib.mf_pack_conv_weights_batched, (table.data_ptr(), n_desc), "mf_pack_conv_weights_batched"))
        for fn_name, argbuilder in self.ops:
            if fn_name == "__py__":
                self.launches.append((argbuilder, None, fn_name))
            else:
                self.launches.append((getattr(lib, fn_name), tuple(argbuilder()), fn_name))
        self.n_launch = len(self.launches)

    def run(self):
        st = torch.cuda.current_stream().cuda_stream
        for fn, args, name in self.launches:
            if args is None:
                fn()
            elif fn(*args, st) != 0:
                raise RuntimeError("%s failed: %s" % (name, _lib.load().mf_last_error().decode()))

    def run_timed(self):
        """Diagnostics: one pass with a CUDA event pair around every launch -> [(kernel, ms)] (adds launch gaps; used by
        bench.py for the per-kernel roofline numbers, never for throughput)."""
        st = torch.cuda.current_stream()
        evs = []
        for fn, args, name in self.launches:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            if args is None:
                fn()
                args = ()
            elif fn(*args, st.cuda_stream) != 0:
                raise RuntimeError("%s failed: %s" % (name, _lib.load().mf_last_error().decode()))
            b.record(st)
            evs.append((name, args, a, b))
        torch.cuda.synchronize()
        return [(name, args, a.elapsed_time(b)) for name, args, a, b in evs]

    # ---- parameter preparation
    def pack_weight(self, w, cin_pad=None, split=False):
        """OIHW (or OIW for Conv1d) fp32 parameter -> packed fp16 [n_pad, k_pad] device tensor. split=True: hi/lo pair
        weights in the tripled virtual K order of a split-input GEMM (mf_pack_conv_weight_split)."""
        if isinstance(w, (list, tuple)):
            # train mode: several parameters stacked along the output-channel axis (the nine head branches), each re-packed
            # from its LIVE storage on every run
            assert self.train and not split and cin_pad is None
            parts = [t.detach() for t in w]
            cout = sum(t.shape[0] for t in parts)
            _, cin, kh, kw = parts[0].shape
            bn = _lib.load().mf_conv_block_n(cout)
            assert all(t.shape[0] % bn == 0 and t.dtype == torch.float32 and t.is_contiguous() for t in parts)
            k_pad = (kh * kw * cin + 63) // 64 * 64
            out = torch.empty(cout, k_pad, dtype=torch.half, device=self.device)
            self.keep.append(out)
            row = 0
            for t in parts:
                self.keep.append(t)
                self.pack_descs.append((t, out.data_ptr() + 2 * row * k_pad, t.shape[0], cin, kh * kw, cin, t.shape[0], k_pad))
                row += t.shape[0]
            return out, cout, k_pad
        live = self.train and w.dtype == torch.float32 and w.is_contiguous()
        w = w.detach().float().contiguous()
        if w.dim() == 3:
            w = w.unsqueeze(2)   # Conv1d: [O, I, 1, k]
        cout, cin, kh, kw = w.shape
        cin_pad = cin if cin_pad is None else cin_pad
        bn = _lib.load().mf_conv_block_n(cout)
        n_pad = (cout + bn - 1) // bn * bn
        if split:
            assert cin_pad == cin
            k_pad = (3 * kh * kw * cin + 63) // 64 * 64
            out = torch.empty(n_pad, k_pad, dtype=torch.half, device=self.device)
            _lib.call("mf_pack_conv_weight_split", w.data_ptr(), cout, cin, kh, kw, n_pad, k_pad, out.data_ptr(), _lib.stream())
            self.keep.append(out)
            return out, n_pad, k_pad
        k_pad = (kh * kw * cin_pad + 63) // 64 * 64
        out = torch.empty(n_pad, k_pad, dtype=torch.half, device=self.device)
        if live:
            # train mode: `w` aliases the parameter's storage (the optimiser updates it in place), so the repack is a plan op
            # executed on every run instead of once at build time - the plan itself stays valid across optimiser steps
            self.keep.append(w)
            self.pack_descs.append((w, out.data_ptr(), cout, cin, kh * kw, cin_pad, n_pad, k_pad))
        else:
            assert not self.train or not w.requires_grad
            _lib.call("mf_pack_conv_weight", w.data_ptr(), cout, cin, kh, kw, cin_pad, n_pad, k_pad, out.data_ptr(),
                      _lib.stream())
        self.keep.append(out)
        return out, n_pad, k_pad

    def affine(self, cout, n_pad, bn=None, conv_bias=None, abs_weight=False):
        """Fold eval-mode BatchNorm (dla_dcn.py:76 etc.) / InPlaceABN (|w|+eps) and the conv bias into (scale, shift)."""
        if bn is None and conv_bias is None:
            # identity epilogue (raw train-mode convs, every data-gradient conv of the backward tape): shared read-only
            # constants instead of two fill kernels per plan - a captured training step replayed ~265 of them
            return _const_vec(1.0, n_pad, self.device), _const_vec(0.0, n_pad, self.device)
        scale = torch.ones(n_pad, dtype=torch.float32, device=self.device)
        shift = torch.zeros(n_pad, dtype=torch.float32, device=self.device)
        if self.train:
            # train-mode plans never fold normalisation layers; a conv bias is re-read from the live parameter on every run
            assert bn is None
            if conv_bias is not None:
                b = conv_bias.detach()
                self.add_py(lambda: shift[:cout].copy_(b))
            self.keep.extend([scale, shift])
            return scale, shift
        if bn is not None:
            w = bn.weight.detach().float()
            if abs_weight:
                w = w.abs() + BN_EPS
            s = w / torch.sqrt(bn.running_var.detach().float() + bn.eps)
            scale[:cout] = s
            shift[:cout] = bn.bias.detach().float() - bn.running_mean.detach().float() * s
        if conv_bias is not None:
            shift[:cout] += conv_bias.detach().float() * scale[:cout]
        self.keep.extend([scale, shift])
        return scale, shift

    # ---- op emitters
    def bn_train(self, raw, y, slices, act, residual=None, abs_weight=False):
        """Emit mf_bn_train_forward for `slices` = [(module, first channel, channels)] of raw -> y (<= 256 channels per
        launch: statistics are per channel, so column slices of one [M, ld] buffer are independent)."""
        lib = _lib.load()
        for mod, c_first, c_num in slices:
            for off in range(0, c_num, 256):
                cc = min(256, c_num - off)
                c0 = c_first + off
                stats = torch.empty(4, cc, dtype=torch.float32, device=self.device)
                ws = torch.empty(max(1, lib.mf_bn_train_workspace(raw.M, cc) // 4), dtype=torch.float32, device=self.device)
                self.keep.extend([stats, ws])
                self.bn_saved.append((mod, raw, y, stats, c0, cc))
                momentum = getattr(mod, "momentum", 0.1)
                eps = getattr(mod, "eps", BN_EPS)
                group, world = sync_bn_group(mod)
                if world > 1:
                    # torch.nn.SyncBatchNorm (the reference's convert_sync_batchnorm, tools/plain_train_net.py:131-132): local sums
                    # -> all-reduce of 2C doubles -> normalise with the statistics of the GLOBAL batch (csrc/mf_bn_train.cu)
                    import torch.distributed as dist
                    sums = torch.zeros(2 * cc, dtype=torch.float64, device=self.device)
                    self.keep.append(sums)
                    count = float(raw.M) * world
                    self.add("mf_bn_sync_forward_stats", lambda c0=c0, cc=cc, ws=ws, sums=sums: (
                        raw.ptr() + 2 * c0, raw.ld, raw.M, cc, ws.data_ptr(), sums.data_ptr()))
                    self.add_py(lambda sums=sums, group=group: dist.all_reduce(sums, group=group))
                    self.add("mf_bn_sync_forward_apply", lambda mod=mod, off=off, c0=c0, cc=cc, stats=stats, sums=sums, momentum=momentum, eps=eps, count=count: (
                        raw.ptr() + 2 * c0, raw.ld, raw.M, cc, sums.data_ptr(), count, mod.weight.data_ptr() + 4 * off,
                        mod.bias.data_ptr() + 4 * off, eps, momentum, 1 if abs_weight else 0, mod.running_mean.data_ptr() + 4 * off,
                        mod.running_var.data_ptr() + 4 * off, (residual.ptr() + 2 * c0) if residual is not None else None,
                        residual.ld if residual is not None else 0, act, y.ptr() + 2 * c0, y.ld, stats[0].data_ptr(),
                        stats[1].data_ptr(), stats[2].data_ptr(), stats[3].data_ptr()))
                    continue
                self.add("mf_bn_train_forward", lambda mod=mod, off=off, c0=c0, cc=cc, stats=stats, ws=ws, momentum=momentum, eps=eps: (
                    raw.ptr() + 2 * c0, raw.ld, raw.M, cc, mod.weight.data_ptr() + 4 * off, mod.bias.data_ptr() + 4 * off, eps,
                    momentum, 1 if abs_weight else 0, mod.running_mean.data_ptr() + 4 * off, mod.running_var.data_ptr() + 4 * off,
                    (residual.ptr() + 2 * c0) if residual is not None else None, residual.ld if residual is not None else 0, act,
                    y.ptr() + 2 * c0, y.ld, stats[0].data_ptr(), stats[1].data_ptr(), stats[2].data_ptr(), stats[3].data_ptr(),
                    ws.data_ptr()))

    def conv(self, x, weight, stride, pad, bn=None, bias=None, act=ACT_RELU, residual=None, out=None, abs_weight=False,
             cin_pad=None):
        if isinstance(weight, (list, tuple)):       # train mode: parameters stacked along Cout, see pack_weight
            cout, (_, _, kh, kw) = sum(t.shape[0] for t in weight), weight[0].shape
        else:
            cout, _, kh, kw = weight.shape if weight.dim() == 4 else (weight.shape[0], weight.shape[1], 1, weight.shape[2])
        if self.train and bn is not None:
            # training mode: raw convolution (+ bias), then batch-statistics normalisation + residual + activation
            assert not isinstance(pad, tuple), "non-square padding is not built"
            raw = self.conv(x, weight, stride, pad, None, bias, ACT_NONE, None, None, False, cin_pad)
            y = out if out is not None else self.act(raw.B, raw.H, raw.W, cout)
            slices = bn if isinstance(bn, list) else [(bn, 0, cout)]
            first = len(self.bn_saved)
            self.bn_train(raw, y, slices, act, residual, abs_weight)
            self.tape.append(dict(kind="conv_bn", x=x, weight=weight, bias=bias, stride=stride, pad=pad, raw=raw, y=y, act=act,
                                  residual=residual, abs_weight=abs_weight, bn=self.bn_saved[first:]))
            return y
        wp, n_pad, k_pad = self.pack_weight(weight, cin_pad, split=x.split)
        scale, shift = self.affine(cout, n_pad, bn, bias, abs_weight)
        Ho = (x.H + 2 * pad[0] - kh) // stride + 1 if isinstance(pad, tuple) else (x.H + 2 * pad - kh) // stride + 1
        Wo = (x.W + 2 * pad[1] - kw) // stride + 1 if isinstance(pad, tuple) else (x.W + 2 * pad - kw) // stride + 1
        assert not isinstance(pad, tuple), "non-square padding is not built"
        y = out if out is not None else self.act(x.B, Ho, Wo, cout)
        assert (y.H, y.W, y.C) == (Ho, Wo, cout)
        cin = x.C
        if x.split or y.split:
            assert residual is None or residual.split == y.split
            self.add("mf_conv2d_nhwc_f16x2", lambda: (
                x.ptr(), x.ld, x.lo, x.B, x.H, x.W, cin, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout,
                scale.data_ptr(), shift.data_ptr(), residual.ptr() if residual is not None else None,
                residual.ld if residual is not None else 0, residual.lo if residual is not None else 0, act, OUT_F16_NHWC,
                y.ptr(), y.ld, y.lo, 1 if x.split else 0, 1 if y.split else 0))
            return y
        self.add("mf_conv2d_nhwc_f16", lambda: (
            x.ptr(), x.ld, x.B, x.H, x.W, cin, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout,
            scale.data_ptr(), shift.data_ptr(), residual.ptr() if residual is not None else None,
            residual.ld if residual is not None else 0, act, OUT_F16_NHWC, y.ptr(), y.ld))
        return y

    def conv_dgrad(self, dy, weight, pad, out=None):
        """dL/dx of the stride-1 convolution y = conv(x, weight, padding=pad) given dy = dL/dy rows (its channel count may be
        the zero-padded Cout): the forward kernel on dY with the 180-degree rotated, in/out-transposed taps, packed straight
        from the live OIHW parameter by ONE kernel (mf_pack_conv_weight_dgrad). out=None: written to a new activation;
        otherwise accumulated in place, out += dL/dx, through the kernel's residual input. Returns the output activation."""
        cout, cin, kh, kw = weight.shape
        res = out
        if out is None:
            out = self.act(dy.B, dy.H + kh - 1 - 2 * pad, dy.W + kw - 1 - 2 * pad, cin)
        assert kh == kw and kh - 1 - pad >= 0 and dy.C >= cout and (out.H, out.W) == (dy.H + kh - 1 - 2 * pad, dy.W + kw - 1 - 2 * pad)
        w = weight.detach()
        assert w.dtype == torch.float32 and w.is_contiguous()
        bn_ = _lib.load().mf_conv_block_n(cin)
        n_pad = (cin + bn_ - 1) // bn_ * bn_
        k_pad = (kh * kw * dy.C + 63) // 64 * 64
        wp = torch.empty(n_pad, k_pad, dtype=torch.half, device=self.device)
        _lib.call("mf_pack_conv_weight_dgrad", w.data_ptr(), cout, cin, kh, kw, dy.C, n_pad, k_pad, wp.data_ptr(), _lib.stream())
        self.keep.extend([w, wp])
        scale, shift = self.affine(cin, n_pad)
        cpad, p2 = dy.C, kh - 1 - pad
        self.add("mf_conv2d_nhwc_f16", lambda: (
            dy.ptr(), dy.ld, dy.B, dy.H, dy.W, cpad, wp.data_ptr(), n_pad, k_pad, kh, kw, 1, p2, cin,
            scale.data_ptr(), shift.data_ptr(), res.ptr() if res is not None else None, res.ld if res is not None else 0,
            ACT_NONE, OUT_F16_NHWC, out.ptr(), out.ld))
        return out

    def conv_to_f32(self, x, weight, bias, out_tensor, out_mode, act, y_ld, stride=1, pad=0, bn=None):
        """conv whose result leaves the NHWC fp16 world: fp32 NHWC rows (offset/mask) or fp32 NCHW maps (heads)."""
        cout, _, kh, kw = weight.shape
        wp, n_pad, k_pad = self.pack_weight(weight, split=x.split)
        scale, shift = self.affine(cout, n_pad, bn, bias)
        cin = x.C
        if x.split:
            self.add("mf_conv2d_nhwc_f16x2", lambda: (
                x.ptr(), x.ld, x.lo, x.B, x.H, x.W, cin, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout,
                scale.data_ptr(), shift.data_ptr(), None, 0, 0, act, out_mode, out_tensor.data_ptr(), y_ld, 0, 1, 0))
            return
        self.add("mf_conv2d_nhwc_f16", lambda: (
            x.ptr(), x.ld, x.B, x.H, x.W, cin, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout,
            scale.data_ptr(), shift.data_ptr(), None, 0, act, out_mode, out_tensor.data_ptr(), y_ld))

    def dcn(self, x, dcn_mod, bn, out=None):
        """DeformConv (dla_dcn.py:384-396): conv_offset_mask -> fused gather+contract -> BN -> ReLU."""
        om = torch.empty(x.M, 32, dtype=torch.float32, device=self.device)
        self.keep.append(om)
        self.conv_to_f32(x, dcn_mod.conv_offset_mask.weight, dcn_mod.conv_offset_mask.bias, om, OUT_F32_NHWC,
                         ACT_OFFMASK, 32, stride=1, pad=1)
        cout = dcn_mod.weight.shape[0]
        wp, n_pad, k_pad = self.pack_weight(dcn_mod.weight, split=x.split)
        cin = x.C
        if x.split:
            scale, shift = self.affine(cout, n_pad, bn, dcn_mod.bias)
            y = out if out is not None else self.act(x.B, x.H, x.W, cout)
            assert y.split
            self.add("mf_dcn_nhwc_f16x2", lambda: (
                x.ptr(), x.ld, x.lo, x.B, x.H, x.W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, cout, scale.data_ptr(),
                shift.data_ptr(), ACT_RELU, y.ptr(), y.ld, y.lo))
            return y
        if self.train:
            scale, shift = self.affine(cout, n_pad, None, dcn_mod.bias)
            raw = self.act(x.B, x.H, x.W, cout)
            self.add("mf_dcn_nhwc_f16", lambda: (
                x.ptr(), x.ld, x.B, x.H, x.W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, cout, scale.data_ptr(),
                shift.data_ptr(), ACT_NONE, OUT_F16_NHWC, raw.ptr(), raw.ld))
            y = out if out is not None else self.act(x.B, x.H, x.W, cout)
            first = len(self.bn_saved)
            self.bn_train(raw, y, [(bn, 0, cout)], ACT_RELU)
            self.tape.append(dict(kind="dcn", x=x, mod=dcn_mod, om=om, raw=raw, y=y, bn=self.bn_saved[first:]))
            return y
        scale, shift = self.affine(cout, n_pad, bn, dcn_mod.bias)
        y = out if out is not None else self.act(x.B, x.H, x.W, cout)
        self.add("mf_dcn_nhwc_f16", lambda: (
            x.ptr(), x.ld, x.B, x.H, x.W, cin, om.data_ptr(), 32, wp.data_ptr(), n_pad, k_pad, cout, scale.data_ptr(),
            shift.data_ptr(), ACT_RELU, OUT_F16_NHWC, y.ptr(), y.ld))
        return y

    def planar_act(self, B, H, W, C, npar, split=False):
        a = self.act(B, H, W, C, split=split)
        a.npar = npar
        return a

    def conv_rows_strict(self, x, weight, stride, pad, bn, out_planar, out_npar=1, image=False):
        """Strict-precision stem convolution on 16-byte-pixel planes (mf_conv2d_rows_f16x2). The two products that read the
        same A rows are stacked along N (2 x cout weight rows, one MMA per A operand) and the kernel adds the two column
        halves in fp32. image=True: x is the image pair plane [hi3 | lo3 | 0 0] (8 channels, mf_pack_image_pair8), K runs
        over the kh x kw taps (two per MMA) and the weight rows are [W_hi | W_hi | 0 0] (A_hi W_hi + A_lo W_hi) over
        [W_lo | 0 ...] (A_hi W_lo); else x is a planar pair activation (planes hi0 hi1 lo0 lo1), K holds two tap sets
        along ky (hi planes, then lo planes) and the weight rows are [W_hi ; W_hi] over [W_lo ; 0]. Output: pair, planar or
        NHWC rows."""
        cout, cin_w, kh, kw = weight.shape
        w = weight.detach().float()
        w_hi = w.half().float()
        w_lo = (w - w_hi).half().float()
        if image:
            assert x.C == 8 and cin_w == 3 and not x.split
            taps = kh * kw                           # K = taps in (ky, kx) order, padded to an even count (two per MMA)
            wa = torch.zeros(cout, 8, 1, (taps + 1) // 2 * 2, dtype=torch.float32, device=w.device)
            wb = torch.zeros_like(wa)
            wa[:, 0:3, 0, :taps], wa[:, 3:6, 0, :taps] = w_hi.reshape(cout, 3, taps), w_hi.reshape(cout, 3, taps)
            wb[:, 0:3, 0, :taps] = w_lo.reshape(cout, 3, taps)
            wv, cin, in_mode, in_npar = torch.cat([wa, wb], 0), 8, 1, 1
        else:
            assert x.C == 16 and x.split and ((x.npar == 1 and stride == 1) or (x.npar == 2 and stride == 2))
            wv = torch.cat([torch.cat([w_hi, w_hi], 2), torch.cat([w_lo, torch.zeros_like(w_lo)], 2)], 0)
            cin, in_mode, in_npar = 16, 2, x.npar
        wp, n_pad, k_pad = self.pack_weight(wv.contiguous(), cin_pad=cin)
        scale, shift = self.affine(cout, n_pad, bn)
        Ho, Wo = (x.H + 2 * pad - kh) // stride + 1, (x.W + 2 * pad - kw) // stride + 1
        y = self.planar_act(x.B, Ho, Wo, cout, out_npar, split=True) if out_planar else self.act(x.B, Ho, Wo, cout, split=True)
        self.add("mf_conv2d_rows_f16x2", lambda: (
            x.ptr(), x.B, x.H, x.W, cin, in_npar, in_mode, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout,
            scale.data_ptr(), shift.data_ptr(), ACT_RELU, 1 if out_planar else 0, out_npar, y.ptr(),
            y.ld if not out_planar else 8, y.lo if not out_planar else 0))
        return y

    def conv_rows(self, x, weight, stride, pad, bn, out_planar, out_npar=1):
        """Stem convolution on 16-byte-pixel planes (csrc/mf_rows.cu): x is the packed image (8 ch) or a planar
        16-channel activation; output planar (next stem layer) or NHWC rows."""
        cout, cin_w, kh, kw = weight.shape
        cin = x.C
        in_npar = x.npar if x.npar else 1
        w = weight.detach().float()
        if cin == 8:
            # K = taps in (ky, kx) order, padded to an even count (two per MMA), 3 -> 8 channels
            taps = kh * kw
            w = torch.nn.functional.pad(w.reshape(cout, cin_w, 1, taps), (0, (taps + 1) // 2 * 2 - taps, 0, 0, 0, 8 - cin_w))
        wp, n_pad, k_pad = self.pack_weight(w.contiguous(), cin_pad=cin)
        scale, shift = self.affine(cout, n_pad, bn)
        Ho, Wo = (x.H + 2 * pad - kh) // stride + 1, (x.W + 2 * pad - kw) // stride + 1
        y = self.planar_act(x.B, Ho, Wo, cout, out_npar) if out_planar else self.act(x.B, Ho, Wo, cout)
        self.add("mf_conv2d_rows_f16", lambda: (
            x.ptr(), x.B, x.H, x.W, cin, in_npar, wp.data_ptr(), n_pad, k_pad, kh, kw, stride, pad, cout, scale.data_ptr(),
            shift.data_ptr(), ACT_RELU, 1 if out_planar else 0, out_npar, y.ptr(), y.ld if not out_planar else 8))
        return y

    def maxpool2(self, x, out=None):
        y = out if out is not None else self.act(x.B, x.H // 2, x.W // 2, x.C)
        assert y.split == x.split
        self.add("mf_maxpool2_nhwc_f16", lambda: (x.ptr(), x.ld, x.lo, y.ptr(), y.ld, y.lo, x.B, x.H, x.W, x.C))
        if self.train:
            self.tape.append(dict(kind="maxpool2", x=x, y=y))
        return y

    def upsample_add(self, x, up_weight, skip, f):
        """depthwise ConvTranspose2d (dla_dcn.py:409-411) fused with `+ layers[i-1]` (:425)."""
        C, k = up_weight.shape[0], up_weight.shape[2]
        assert k == 2 * f and C == x.C
        wt = up_weight.detach().float().reshape(C, k * k).t().contiguous()   # [k*k, C]
        self.keep.append(wt)
        if self.train:                         # trainable depth-wise kernel: refresh the tap-major copy on every run
            uw = up_weight.detach()
            self.add_py(lambda: wt.copy_(uw.reshape(C, k * k).t()))
        y = self.act(x.B, x.H * f, x.W * f, C)
        assert y.split == x.split and (skip is None or skip.split == x.split)
        self.add("mf_upsample_add_nhwc_f16", lambda: (
            x.ptr(), x.ld, x.lo, wt.data_ptr(), skip.ptr() if skip is not None else None, skip.ld if skip is not None else 0,
            skip.lo if skip is not None else 0, y.ptr(), y.ld, y.lo, x.B, x.H, x.W, C, f))
        if self.train:
            self.tape.append(dict(kind="upsample_add", x=x, weight=up_weight, wt=wt, skip=skip, f=f, y=y))
        return y


def sync_bn_group(mod):
    """(process group, world size) when `mod` is a torch.nn.SyncBatchNorm in an initialised multi-rank job, else (None, 1)"""
    import torch.distributed as dist
    if isinstance(mod, torch.nn.SyncBatchNorm) and dist.is_available() and dist.is_initialized():
        group = getattr(mod, "process_group", None)
        return group, dist.get_world_size(group)
    return None, 1


def bn_backward_launch(mod, x_ptr, x_ld, dy_ptr, dy_ld, y_ptr, y_ld, M, cc, stats, act, dx_ptr, dx_ld, dres_ptr, dres_ld, dg, ws,
                       stream):
    """mf_bn_train_backward, or its SyncBatchNorm form (local sums -> all-reduce -> apply with the global count) when `mod` is a
    converted SyncBatchNorm. dg: fp32 [2, cc] (dgamma, dbeta - LOCAL sums in both cases: DDP averages parameter gradients)."""
    group, world = sync_bn_group(mod)
    if world > 1:
        import torch.distributed as dist
        sums = torch.empty(2 * cc, dtype=torch.float64, device=dg.device)
        _lib.call("mf_bn_sync_backward_stats", x_ptr, x_ld, dy_ptr, dy_ld, y_ptr, y_ld, M, cc, stats[0].data_ptr(), stats[1].data_ptr(),
                  act, ws.data_ptr(), sums.data_ptr(), dg[0].data_ptr(), dg[1].data_ptr(), stream)
        dist.all_reduce(sums, group=group)
        _lib.call("mf_bn_sync_backward_apply", x_ptr, x_ld, dy_ptr, dy_ld, y_ptr, y_ld, M, cc, stats[0].data_ptr(), stats[1].data_ptr(),
                  stats[2].data_ptr(), sums.data_ptr(), float(M) * world, act, dx_ptr, dx_ld, dres_ptr, dres_ld, ws.data_ptr(), stream)
        return
    _lib.call("mf_bn_train_backward", x_ptr, x_ld, dy_ptr, dy_ld, y_ptr, y_ld, M, cc, stats[0].data_ptr(), stats[1].data_ptr(),
              stats[2].data_ptr(), act, dx_ptr, dx_ld, dres_ptr, dres_ld, dg[0].data_ptr(), dg[1].data_ptr(), ws.data_ptr(), stream)


def fingerprint(module, versions=True):
    """versions=False: addresses only - the key of train-mode plans, which read every parameter from its live storage on
    each run and therefore survive optimiser steps.
    Change detector for cached plans: (storage address, version) of every parameter and buffer + training flag. The
    address catches a ParamArena re-binding `p.data` (no version bump); versions catch optimiser steps, load_state_dict and
    the running-statistics updates of the train-mode BatchNorm kernels (`bump_buffers`)."""
    sig = tuple((t.data_ptr(), t._version if versions else 0) for t in module.parameters()) + \
        tuple((t.data_ptr(), t._version if versions else 0) for t in module.buffers())
    return (hash(sig), module.training, next(module.parameters()).device)


def bump_buffers(module):
    """the bn_train kernels update running_mean / running_var behind torch's back: bump their versions so that an eval plan
    or CUDA graph with folded statistics is rebuilt after training steps"""
    for t in module.buffers():
        torch.autograd.graph.increment_version(t)
