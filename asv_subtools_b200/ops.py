"""Thin Python wrappers over the C ABI for torch CUDA tensors (device memory + streams are the
only things torch is used for).  Frame matrices are channel-contiguous ``(B, T, C)``."""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import BN, RELU, SIGMOID, SWISH, TANH, TdnnArgs, check, int_array, lib  # noqa: F401
from .native import ShardExtractor, host_lengths


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _req(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise TypeError("{} must be a contiguous CUDA tensor of dtype {}".format(name, dtype))
    return t


class SplitPlanes:
    """fp32 tensor stored as two bf16 planes hi = bf16(x), lo = bf16(x - hi); last dim padded to `ld`."""

    def __init__(self, hi, lo, channels):
        self.hi, self.lo, self.channels = hi, lo, channels

    @property
    def ld(self):
        """Row pitch in elements (a channel slice keeps the pitch of the tensor it was cut from)."""
        return self.hi.stride(-2) if self.hi.dim() >= 2 else self.hi.shape[-1]

    def float(self):
        return (self.hi.float() + self.lo.float())[..., :self.channels]

    def slice(self, c0, c1):
        """Channel slice [c0, c1) as a view (c0 must keep 16-byte alignment: c0 % 8 == 0)."""
        if c0 % 8:
            raise ValueError("channel slices must start at a multiple of 8")
        return SplitPlanes(self.hi[..., c0:c1], self.lo[..., c0:c1], c1 - c0)

    @staticmethod
    def empty(shape, device):
        return SplitPlanes(torch.empty(shape, dtype=torch.bfloat16, device=device),
                           torch.empty(shape, dtype=torch.bfloat16, device=device), shape[-1])


def split_f32(x, ld=None):
    """(rows..., C) fp32 -> SplitPlanes with row pitch ld (default round_up(C, 8))."""
    x = _req(x, torch.float32, "x")
    c = x.shape[-1]
    ld = ld or (c + 7) // 8 * 8
    rows = x.numel() // c
    hi = torch.empty(x.shape[:-1] + (ld,), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    check(lib.xvb_split_f32(_ptr(x), rows, c, c, _ptr(hi), _ptr(lo), ld, _stream()), "xvb_split_f32")
    return SplitPlanes(hi, lo, c)


def split_frames(x, ld=None, pad_front=0, pad_back=0, lengths=None):
    """(B, T, C) fp32 -> SplitPlanes (B, pad_front + T + pad_back, ld) with zero frames around every utterance
    (xvb_split_frames).  lengths: int32 CUDA (B,) tensor of a masked batch (xvb_split_frames_lengths): the frames
    t >= lengths[b] are written as zeros and never read."""
    x = _req(x, torch.float32, "x")
    b, t, c = x.shape
    ld = ld or (c + 7) // 8 * 8
    hi = torch.empty(b, pad_front + t + pad_back, ld, dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    args = (_ptr(x), b, t, c, _ptr(hi), _ptr(lo), ld, pad_front, pad_back)
    if lengths is None:
        check(lib.xvb_split_frames(*args, _stream()), "xvb_split_frames")
    else:
        check(lib.xvb_split_frames_lengths(*args, _ptr(_req(lengths, torch.int32, "lengths")), _stream()),
              "xvb_split_frames_lengths")
    return SplitPlanes(hi, lo, c)


def context_span(context):
    """left/right/total context as TdnnAffine.__init__ (components.py:50-53)."""
    left = context[0] if context[0] < 0 else 0
    right = context[-1] if context[-1] > 0 else 0
    return left, right, right - left + 1


def pack_tdnn_weight(weight, context):
    """Reference weight (Cout, Cin, tot_context) fp32 CUDA -> packed K-major SplitPlanes."""
    weight = _req(weight, torch.float32, "weight")
    cout, cin, tot = weight.shape
    left, _, tot_expected = context_span(context)
    if tot != tot_expected:
        raise ValueError("weight kernel size {} does not match context {}".format(tot, context))
    n = lib.xvb_packed_weight_elems(cout, cin, len(context))
    hi = torch.empty(n, dtype=torch.bfloat16, device=weight.device)
    lo = torch.empty_like(hi)
    check(lib.xvb_pack_tdnn_weight(_ptr(weight), cout, cin, tot, left, int_array(context), len(context), _ptr(hi),
                                   _ptr(lo), _stream()), "xvb_pack_tdnn_weight")
    return SplitPlanes(hi.view(cout, -1), lo.view(cout, -1), cin)


def tdnn_affine(x, w, cout, context, bias=None, bn_scale=None, bn_shift=None, relu=False, out_planes=True,
                out_f32=False):
    """x: SplitPlanes (B, T, ld).  Returns (SplitPlanes | None, fp32 tensor | None)."""
    b, t, ldx = x.hi.shape
    flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0)
    dev = x.hi.device
    y = None
    yf = None
    if out_planes:
        y = SplitPlanes(torch.empty(b, t, cout, dtype=torch.bfloat16, device=dev),
                        torch.empty(b, t, cout, dtype=torch.bfloat16, device=dev), cout)
    if out_f32:
        yf = torch.empty(b, t, cout, dtype=torch.float32, device=dev)
    check(lib.xvb_tdnn_affine(_ptr(x.hi), _ptr(x.lo), ldx, _ptr(w.hi), _ptr(w.lo), _ptr(bias), _ptr(bn_scale),
                              _ptr(bn_shift), flags, int_array(context), len(context),
                              _ptr(y.hi) if y else None, _ptr(y.lo) if y else None, cout, _ptr(yf), cout,
                              b, t, x.channels, cout, _stream()), "xvb_tdnn_affine")
    return y, yf


def fused_pool_layer(x, w, cout, context, bias=None, bn_scale=None, bn_shift=None, relu=True, eps=1e-10, mode=0, planes=False):
    """TDNN layer whose epilogue pools over time (no (B,T,C) output) + the Chan merge: -> (B, 2*cout) fp32
    [, the same as SplitPlanes (B,1,2*cout) for a following segment-level GEMM]."""
    b, t = x.hi.shape[0], x.hi.shape[1]
    tb = C.c_int()
    nblk = lib.xvb_pool_partial_blocks(b, t, C.byref(tb))
    partial = torch.empty(nblk, b, 2 * cout, dtype=torch.float32, device=x.hi.device)
    tdnn_affine_ex(x, w, cout, context, bias=bias, bn_scale=bn_scale, bn_shift=bn_shift, relu=relu, pool_partial=partial)
    out = torch.empty(b, 2 * cout, dtype=torch.float32, device=x.hi.device)
    op = SplitPlanes.empty((b, 1, 2 * cout), x.hi.device) if planes else None
    check(lib.xvb_pool_finalize(_ptr(partial), nblk, tb.value, b, t, cout, eps, mode, _ptr(out),
                                op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, 2 * cout if op else 0,
                                _stream()), "xvb_pool_finalize")
    return (out, op) if planes else out


def tdnn_grouped_fits(cin, cout, groups):
    """True when the layer kernel's grouped mode takes a (cin -> cout, groups) 1x1 conv (xvb_tdnn_grouped_fits)."""
    return bool(lib.xvb_tdnn_grouped_fits(int(cin), int(cout), int(groups)))


def tdnn_affine_ex(x, w, cout, context, x2=None, bias=None, bn_scale=None, bn_shift=None, utt_bias=None, row_bias=None,
                   relu=False, tanh=False, sigmoid=False, y=None, y_f32=None, pool_partial=None, swish=False, groups=1,
                   x_batch_stride=0, lengths=None):
    """Full form of the wgmma layer (xvb_tdnn_affine_ex).  x / x2: SplitPlanes (B,T,*) (views
    allowed); y: SplitPlanes to write (view allowed) and/or y_f32: fp32 (B,T,>=cout) tensor.  swish: x * sigmoid(x)
    after the bias (and ReLU), before the BatchNorm (XVB_SWISH).  groups > 1: grouped 1x1 conv, w the compact packing
    of the (cout, Cin/groups, 1) weight.  x_batch_stride > 0: x is an im2col view (xvb_tdnn_args_t.x_batch_stride):
    frame t of utterance b is the x.channels-long window at element b * x_batch_stride + t * x.ld of the planes.
    lengths: int32 CUDA (B,) tensor of a masked batch (xvb_tdnn_args_t.lengths): frames t >= lengths[b] store zeros."""
    b, t = x.hi.shape[0], x.hi.shape[1]
    a = TdnnArgs()
    a.x_hi, a.x_lo, a.ldx = x.hi.data_ptr(), x.lo.data_ptr(), x.ld
    if x2 is not None:
        a.x2_hi, a.x2_lo, a.ldx2 = x2.hi.data_ptr(), x2.lo.data_ptr(), x2.ld
    a.w_hi, a.w_lo = w.hi.data_ptr(), w.lo.data_ptr()
    keep = []
    for name, v in (("bias", bias), ("bn_scale", bn_scale), ("bn_shift", bn_shift), ("row_bias", row_bias)):
        if v is not None:
            setattr(a, name, _req(v, torch.float32, name).data_ptr())
    if utt_bias is not None:
        a.utt_bias, a.ld_utt_bias = _req(utt_bias, torch.float32, "utt_bias").data_ptr(), utt_bias.shape[-1]
    a.flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0) | (TANH if tanh else 0) | \
        (SIGMOID if sigmoid else 0) | (SWISH if swish else 0)
    ctx = int_array(context)
    keep.append(ctx)
    a.context_host, a.ntaps = ctx, len(context)
    if y is not None:
        a.y_hi, a.y_lo, a.ldy = y.hi.data_ptr(), y.lo.data_ptr(), y.ld
    if y_f32 is not None:
        if y_f32.dtype != torch.float32 or not y_f32.is_cuda:
            raise TypeError("y_f32 must be a CUDA float32 tensor")
        a.y_f32, a.ldyf = y_f32.data_ptr(), y_f32.stride(-2)
    if pool_partial is not None:
        a.pool_partial = pool_partial.data_ptr()
    a.B, a.T, a.Cin, a.Cout = b, t, x.channels, cout
    a.groups = groups
    a.x_batch_stride = x_batch_stride
    if lengths is not None:
        a.lengths = _req(lengths, torch.int32, "lengths").data_ptr()
    check(lib.xvb_tdnn_affine_ex(C.byref(a), _stream()), "xvb_tdnn_affine_ex")


def to_device(a, device):
    """An array (ndarray or tensor) as a contiguous fp32 tensor on `device`; None stays None."""
    return None if a is None else torch.as_tensor(a).detach().float().to(device).contiguous()


def block_diagonal(w, groups):
    """(Cout, Cin/G, k) grouped weight -> (Cout, Cin, k) with group g's block at rows g*Cout/G, columns g*Cin/G (conv1d's rule)."""
    co, ci = w.shape[0] // groups, w.shape[1]
    dense = w.new_zeros(w.shape[0], ci * groups, w.shape[2])
    for g in range(groups):
        dense[g * co:(g + 1) * co, g * ci:(g + 1) * ci] = w[g * co:(g + 1) * co]
    return dense


class PackedAffine:
    """One affine layer packed on `device` for the wgmma layer kernel (tdnn_affine_ex): weight w (Cout, Cin, tot) over
    `context`, or (Cout, Cin) at one tap, with its bias, its folded eval BatchNorm (scale, shift) and ReLU / swish as the
    epilogue.  A weight whose kernel axis holds only the listed taps of a dilated context is spread over the span, the
    gaps as zero taps.  groups > 1: a grouped 1x1 conv with its weight as stored, (Cout, Cin/groups, 1), packed compactly
    for the grouped mode, or as its block-diagonal expansion when the shape does not fit that mode (tdnn_grouped_fits).
    row_scale: a per-output factor folded into weight and bias.  pad_to: output rows zero-padded to a multiple of it, the
    padded outputs exact zeros; the first cout_real rows are the layer's own."""

    def __init__(self, w, device, context=(0,), bias=None, scale=None, shift=None, relu=False, swish=False, groups=1,
                 pad_to=1, row_scale=None):
        w = to_device(w, device)
        w = w.reshape(w.shape[0], w.shape[1], -1)
        self.context = list(context)
        left, _, tot = context_span(self.context)
        if w.shape[2] != tot:
            full = w.new_zeros(w.shape[0], w.shape[1], tot)
            full[:, :, [c - left for c in self.context]] = w
            w = full
        self.groups = 1
        if groups > 1:
            if tdnn_grouped_fits(w.shape[1] * groups, w.shape[0], groups):
                self.groups = groups
            else:
                w = block_diagonal(w, groups)
        bias, scale, shift = (to_device(v, device) for v in (bias, scale, shift))
        if row_scale is not None:
            row_scale = to_device(row_scale, device)
            w = w * row_scale.view(-1, 1, 1)
            bias = bias * row_scale if bias is not None else None
        self.cout_real = w.shape[0]
        pad = (-w.shape[0]) % pad_to
        if pad:
            w = torch.cat([w, w.new_zeros(pad, w.shape[1], w.shape[2])], 0)
            bias, scale, shift = (torch.cat([v, v.new_zeros(pad)]) if v is not None else None for v in (bias, scale, shift))
        self.cout = w.shape[0]
        self.w = pack_tdnn_weight(w.contiguous(), self.context)
        self.bias, self.scale, self.shift = bias, scale, shift
        self.relu, self.swish = relu, swish

    def run(self, x, **kw):
        tdnn_affine_ex(x, self.w, self.cout, self.context, bias=self.bias, bn_scale=self.scale, bn_shift=self.shift,
                       relu=self.relu, swish=self.swish, groups=self.groups, **kw)

    def planes(self, b, t, device):
        """(buffer to write, view of the real channels for the next layer)."""
        y = SplitPlanes.empty((b, t, self.cout), device)
        return y, (y if self.cout == self.cout_real else y.slice(0, self.cout_real))


def plane_mean(x, planes=True, lengths=None, rows_per_length=1):
    """Mean over T of SplitPlanes (B,T,C) -> (fp32 (B,C), SplitPlanes (B,1,C) | None).  lengths: int32 CUDA (B,) tensor
    of a masked batch: utterance b averages its first lengths[b] * rows_per_length rows (xvb_plane_mean_lengths)."""
    b, t, c = x.hi.shape[0], x.hi.shape[1], x.channels
    out = torch.empty(b, c, dtype=torch.float32, device=x.hi.device)
    op = SplitPlanes.empty((b, 1, c), x.hi.device) if planes else None
    tail = (_ptr(out), op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, c, _stream())
    if lengths is None:
        check(lib.xvb_plane_mean(x.hi.data_ptr(), x.lo.data_ptr(), x.ld, b, t, c, *tail), "xvb_plane_mean")
    else:
        check(lib.xvb_plane_mean_lengths(x.hi.data_ptr(), x.lo.data_ptr(), x.ld, b, t, c,
                                         _ptr(_req(lengths, torch.int32, "lengths")), int(rows_per_length), *tail),
              "xvb_plane_mean_lengths")
    return out, op


def res2net_block(x, w_hi, w_lo, bias, scale, shift, dilation, nscale, y, width=128):
    """One-kernel Res2Net block: x, y SplitPlanes (B,T,nscale*width), width 64 or 128; stacked packed weights/params."""
    b, t = x.hi.shape[0], x.hi.shape[1]
    check(lib.xvb_res2net_block_ex(x.hi.data_ptr(), x.lo.data_ptr(), x.ld, _ptr(w_hi), _ptr(w_lo), _ptr(bias), _ptr(scale),
                                   _ptr(shift), int(dilation), int(nscale), y.hi.data_ptr(), y.lo.data_ptr(), y.ld, b, t,
                                   int(width), _stream()), "xvb_res2net_block_ex")


def copy_planes(src, dst):
    """dst[...] = src[...] for two SplitPlanes views of equal shape (B,T,c), c % 8 == 0."""
    rows = src.hi.shape[0] * src.hi.shape[1]
    for s, d in ((src.hi, dst.hi), (src.lo, dst.lo)):
        check(lib.xvb_copy_rows(s.data_ptr(), s.stride(-2) * 2, d.data_ptr(), d.stride(-2) * 2, rows, src.channels * 2,
                                _stream()), "xvb_copy_rows")


def se_apply(z, xin, gate, out, nxt=None):
    """out = z * gate[b] + xin ; nxt = xin + out   (all SplitPlanes (B,T,C), views allowed)."""
    b, t, c = z.hi.shape[0], z.hi.shape[1], z.channels
    gate = _req(gate, torch.float32, "gate")
    check(lib.xvb_se_apply(z.hi.data_ptr(), z.lo.data_ptr(), z.ld, xin.hi.data_ptr(), xin.lo.data_ptr(), xin.ld,
                           _ptr(gate), out.hi.data_ptr(), out.lo.data_ptr(), out.ld,
                           nxt.hi.data_ptr() if nxt else None, nxt.lo.data_ptr() if nxt else None,
                           nxt.ld if nxt else 0, b, t, c, _stream()), "xvb_se_apply")


def seg_gate_apply(z, gate, seg_len, out, xin=None):
    """out = z * gate[b, t // seg_len] [+ xin] (xvb_seg_gate_apply): z, out, xin SplitPlanes (B, T, C) views; gate
    (B, ceil(T / seg_len), C) fp32."""
    b, t, c = z.hi.shape[0], z.hi.shape[1], z.channels
    gate = _req(gate, torch.float32, "gate")
    ih, il = _planes_ptrs(xin)
    check(lib.xvb_seg_gate_apply(z.hi.data_ptr(), z.lo.data_ptr(), z.ld, ih, il, xin.ld if xin is not None else 0, _ptr(gate),
                                 int(seg_len), out.hi.data_ptr(), out.lo.data_ptr(), out.ld, b, t, c, _stream()),
          "xvb_seg_gate_apply")


def bn_relu_planes(x, scale, shift, y):
    """y = relu(x * scale + shift) (xvb_bn_relu_planes): x, y SplitPlanes (B, T, C) views (any pitch), scale / shift (C,)."""
    rows = x.hi.numel() // x.hi.shape[-1]
    check(lib.xvb_bn_relu_planes(x.hi.data_ptr(), x.lo.data_ptr(), x.ld, rows, x.channels,
                                 _ptr(_req(scale, torch.float32, "scale")), _ptr(_req(shift, torch.float32, "shift")),
                                 y.hi.data_ptr(), y.lo.data_ptr(), y.ld, _stream()), "xvb_bn_relu_planes")


def cam_gate(h, w1, b1, w2, b2, seg_len=100, out=None):
    """CAMLayer's per-segment mask (xvb_cam_gate): h SplitPlanes (B, T, C); w1 (R, C), b1 (R,), w2 (G, R), b2 (G,) fp32
    -> gate (B, ceil(T / seg_len), G) fp32 (written into `out` when given)."""
    b, t, c = h.hi.shape[0], h.hi.shape[1], h.channels
    w1, w2 = _req(w1, torch.float32, "w1"), _req(w2, torch.float32, "w2")
    r, g = w1.shape[0], w2.shape[0]
    nseg = (t + seg_len - 1) // seg_len
    if out is None:
        out = torch.empty(b, nseg, g, dtype=torch.float32, device=h.hi.device)
    elif _req(out, torch.float32, "out").shape != (b, nseg, g):
        raise ValueError("out must be ({}, {}, {})".format(b, nseg, g))
    check(lib.xvb_cam_gate(h.hi.data_ptr(), h.lo.data_ptr(), h.ld, b, t, c, int(seg_len), _ptr(w1),
                           _ptr(_req(b1, torch.float32, "b1")), r, _ptr(w2), _ptr(_req(b2, torch.float32, "b2")), g, _ptr(out),
                           _stream()), "xvb_cam_gate")
    return out


def _planes_ptrs(p):
    return (p.hi.data_ptr(), p.lo.data_ptr()) if p is not None else (None, None)


def pack_conv2d_weight(weight, taps=None):
    """Reference Conv2d weight (Cout, Cin, k, k) fp32 CUDA -> packed K-major SplitPlanes (tap = kf*k + kt).  taps: the
    strictly increasing tap list of conv2d(taps=...), packed in that order (None: all k*k taps)."""
    weight = _req(weight, torch.float32, "weight")
    cout, cin, kf, kt = weight.shape
    if kf != kt:
        raise ValueError("square kernels only, got {}x{}".format(kf, kt))
    if taps is None:
        return pack_tdnn_weight(weight.reshape(cout, cin, kf * kt).contiguous(), list(range(kf * kt)))
    taps = [int(j) for j in taps]
    if not taps or any(j < 0 or j >= kf * kt for j in taps) or any(b <= a for a, b in zip(taps, taps[1:])):
        raise ValueError("taps must be a strictly increasing list in [0, {}), got {}".format(kf * kt, taps))
    # xvb_pack_tdnn_weight takes at most XVB_MAX_TAPS (16) taps per call; the packed rows are tap-major, so packing
    # the list in pieces and concatenating the pieces along K gives the same layout
    sel = weight.reshape(cout, cin, kf * kt)[:, :, taps]
    pieces = [pack_tdnn_weight(sel[:, :, i:i + _lib.MAX_TAPS].contiguous(), list(range(min(_lib.MAX_TAPS, len(taps) - i))))
              for i in range(0, len(taps), _lib.MAX_TAPS)]
    if len(pieces) == 1:
        return pieces[0]
    return SplitPlanes(torch.cat([p.hi for p in pieces], 1).contiguous(), torch.cat([p.lo for p in pieces], 1).contiguous(), cin)


def conv2d(x, w, cout, ksize, stride=1, scale=None, shift=None, res=None, relu=False, y=None, y_f32=None,
           scale2=None, shift2=None, y2=None, taps=None, valid=False, stride_t=0, lengths=None):
    """One 2-D convolution (xvb_conv2d): x SplitPlanes (B, T, F, Cin); w from pack_conv2d_weight; res / y / y2
    SplitPlanes (B, T', F', cout), y_f32 fp32 of the same shape, with T' = ceil(T / stride), F' = ceil(F / stride).
    stride_t: the time axis's own stride (0: `stride`; CAM++'s FCM head uses stride=2, stride_t=1).
    taps: only these taps (kf*ksize + kt, strictly increasing, ksize 1, 3 or 5) are computed, with w packed by
    pack_conv2d_weight(weight, taps) (xvb_conv2d_taps).  valid: no padding, T' = (T - k) // stride + 1 and F' likewise
    (xvb_conv2d_valid; dense taps only).  lengths: int32 CUDA (B,) tensor of a masked batch, the input length of each
    utterance (xvb_conv2d_args_t.lengths): the outputs past each utterance's own output length store zeros."""
    b, t, f, cin = x.hi.shape
    a = _lib.Conv2dArgs()
    a.x_hi, a.x_lo = _planes_ptrs(x)
    a.w_hi, a.w_lo = w.hi.data_ptr(), w.lo.data_ptr()
    a.B, a.T, a.F, a.Cin, a.Cout, a.ksize, a.stride, a.stride_t = b, t, f, cin, cout, ksize, stride, stride_t
    for name, v in (("scale", scale), ("shift", shift), ("scale2", scale2), ("shift2", shift2)):
        if v is not None:
            setattr(a, name, _req(v, torch.float32, name).data_ptr())
    a.res_hi, a.res_lo = _planes_ptrs(res)
    a.relu = 1 if relu else 0
    a.y_hi, a.y_lo = _planes_ptrs(y)
    a.y2_hi, a.y2_lo = _planes_ptrs(y2)
    if y_f32 is not None:
        a.y_f32 = _req(y_f32, torch.float32, "y_f32").data_ptr()
    if lengths is not None:
        a.lengths = _req(lengths, torch.int32, "lengths").data_ptr()
    if valid:
        if taps is not None:
            raise ValueError("conv2d(valid=True) takes the dense window only")
        check(lib.xvb_conv2d_valid(C.byref(a), _stream()), "xvb_conv2d_valid")
    elif taps is None:
        check(lib.xvb_conv2d(C.byref(a), _stream()), "xvb_conv2d")
    else:
        check(lib.xvb_conv2d_taps(C.byref(a), int_array(taps), len(taps), _stream()), "xvb_conv2d_taps")


def conv2d_head(feats, weight, scale, shift, y, scale2=None, shift2=None, y2=None, lengths=None):
    """Head conv (xvb_conv2d_head_k): feats (B, T, F) fp32, weight (Cout, 1, k, k) fp32 with k = 3 or 5 -> y =
    relu(bn(conv)) SplitPlanes (B, T, F, Cout) [, y2 = relu(y * scale2 + shift2)].  lengths: int32 CUDA (B,) tensor of a
    masked batch (k = 3, xvb_conv2d_head_lengths): the frames t >= lengths[b] read as zeros and store zeros."""
    feats = _req(feats, torch.float32, "feats")
    weight = _req(weight, torch.float32, "weight")
    b, t, f = feats.shape
    k = weight.shape[-1]
    y2h, y2l = _planes_ptrs(y2)
    args = (_ptr(scale), _ptr(shift), y.hi.data_ptr(), y.lo.data_ptr(), _ptr(scale2), _ptr(shift2), y2h, y2l, _stream())
    if lengths is not None:
        if k != 3:
            raise ValueError("conv2d_head(lengths=...) takes the 3x3 head only, got k={}".format(k))
        check(lib.xvb_conv2d_head_lengths(_ptr(feats), b, t, f, _ptr(_req(lengths, torch.int32, "lengths")), _ptr(weight),
                                          weight.shape[0], *args), "xvb_conv2d_head_lengths")
    elif k == 3:
        check(lib.xvb_conv2d_head(_ptr(feats), b, t, f, _ptr(weight), weight.shape[0], *args), "xvb_conv2d_head")
    else:
        check(lib.xvb_conv2d_head_k(_ptr(feats), b, t, f, _ptr(weight), weight.shape[0], k, *args), "xvb_conv2d_head_k")


def se_residual(z, gate, identity, relu=False, y=None, y_f32=None, scale2=None, shift2=None, y2=None, lengths=None):
    """y = [relu](z * gate[b] + identity) over SplitPlanes (B, ..., C) (xvb_se_residual); gate (B, C) fp32.  lengths:
    int32 CUDA (B,) tensor of a masked batch of (B, T, F, C) planes (xvb_se_residual_lengths): the positions of frames
    t >= lengths[b] store zeros."""
    b, c = z.hi.shape[0], z.hi.shape[-1]
    gate = _req(gate, torch.float32, "gate")
    yh, yl = _planes_ptrs(y)
    y2h, y2l = _planes_ptrs(y2)
    if lengths is not None:
        _, t, f, _ = z.hi.shape
        check(lib.xvb_se_residual_lengths(z.hi.data_ptr(), z.lo.data_ptr(), _ptr(gate), identity.hi.data_ptr(),
                                          identity.lo.data_ptr(), b, t, f, c, _ptr(_req(lengths, torch.int32, "lengths")),
                                          1 if relu else 0, yh, yl, _ptr(y_f32), _ptr(scale2), _ptr(shift2), y2h, y2l,
                                          _stream()), "xvb_se_residual_lengths")
        return
    check(lib.xvb_se_residual(z.hi.data_ptr(), z.lo.data_ptr(), _ptr(gate), identity.hi.data_ptr(), identity.lo.data_ptr(), b,
                              z.hi.numel() // (b * c), c, 1 if relu else 0, yh, yl, _ptr(y_f32), _ptr(scale2), _ptr(shift2),
                              y2h, y2l, _stream()), "xvb_se_residual")


def subsample_head(feats, weight, bias, y, stride_f=None):
    """Conv2dSubsampling4's first conv + ReLU (xvb_subsample_head): feats (B, T, F) fp32, weight (C, 1, 3, 3) fp32 as
    stored, bias (C,) -> y SplitPlanes (B, (T - 1) // 2, (F - 1) // 2, C).  stride_f = 1 or 2: the feature stride of
    xvb_subsample_head_stride (1: SVConv2dSubsampling2's stride (2, 1), y (B, (T - 1) // 2, F - 2, C))."""
    feats = _req(feats, torch.float32, "feats")
    b, t, f = feats.shape
    args = (_ptr(feats), b, t, f, _ptr(_req(weight, torch.float32, "weight")), _ptr(_req(bias, torch.float32, "bias")),
            weight.shape[0])
    if stride_f is None:
        check(lib.xvb_subsample_head(*args, y.hi.data_ptr(), y.lo.data_ptr(), _stream()), "xvb_subsample_head")
    else:
        check(lib.xvb_subsample_head_stride(*args, int(stride_f), y.hi.data_ptr(), y.lo.data_ptr(), _stream()),
              "xvb_subsample_head_stride")


def _rows(t, name):
    """(rows, pitch) of a fp32 CUDA tensor whose last dim is contiguous and whose leading dims collapse."""
    if t.dtype != torch.float32 or not t.is_cuda or t.stride(-1) != 1:
        raise TypeError("{} must be a CUDA float32 tensor with contiguous rows".format(name))
    ld = t.stride(-2) if t.dim() >= 2 else t.shape[-1]
    # the kernels address row r at r * ld: a view such as buf[:, :T] of a longer buffer does not collapse that way
    want = ld
    for i in range(t.dim() - 2, -1, -1):
        if t.shape[i] > 1 and t.stride(i) != want:
            raise ValueError("{}: leading dimensions {} do not collapse into rows of pitch {} (strides {})".format(
                name, tuple(t.shape[:-1]), ld, t.stride()))
        want *= t.shape[i]
    return t.numel() // t.shape[-1], ld


def layer_norm(x, gamma=None, beta=None, eps=1e-5, delta=None, delta_scale=1.0, table=None, x_out=None, second=None,
               act=_lib.ACT_NONE, y=None, y_f32=None, channels=None):
    """Residual update + LayerNorm (xvb_layer_norm) over fp32 rows (..., C): v = x [+ table[row % len(table)]]
    [+ delta_scale * delta]; n1 = LN(v) [* gamma + beta]; x_out (may be x) receives v, or n1 when `second` = (gamma2,
    beta2) (either may be None: no affine) asks for y = act(LN(n1)); otherwise y = act(n1).  y: SplitPlanes and/or
    y_f32: fp32 rows."""
    rows, ldx = _rows(x, "x")
    c = channels or x.shape[-1]
    a = _lib.LayerNormArgs()
    a.rows, a.C, a.eps, a.x, a.ldx = rows, c, eps, x.data_ptr(), ldx
    if delta is not None:
        a.delta, a.ld_delta = delta.data_ptr(), _rows(delta, "delta")[1]
        a.delta_scale = delta_scale
    if table is not None:
        if _req(table, torch.float32, "table").dim() != 2 or table.shape[1] != c:
            raise ValueError("table must be (rows, {}), got {}".format(c, tuple(table.shape)))
        a.table, a.table_rows = table.data_ptr(), table.shape[0]
    if x_out is not None:
        a.x_out, a.ld_x_out = x_out.data_ptr(), _rows(x_out, "x_out")[1]
    if gamma is not None:
        a.gamma, a.beta = _req(gamma, torch.float32, "gamma").data_ptr(), _req(beta, torch.float32, "beta").data_ptr()
    if second is not None:
        a.second = 1
        if second[0] is not None:
            a.gamma2, a.beta2 = _req(second[0], torch.float32, "gamma2").data_ptr(), _req(second[1], torch.float32, "beta2").data_ptr()
    a.act = act
    if y is not None:
        a.y_hi, a.y_lo, a.ldy = y.hi.data_ptr(), y.lo.data_ptr(), y.ld
    if y_f32 is not None:
        a.y_f32, a.ldyf = y_f32.data_ptr(), _rows(y_f32, "y_f32")[1]
    check(lib.xvb_layer_norm(C.byref(a), _stream()), "xvb_layer_norm")


def rope_attention(qkv, heads, dk, y, rope=None, rope_v=False, score_mult=1.0):
    """Self-attention over the fused projection (xvb_rope_attention): qkv (B, T, >= 3 * heads * dk) fp32 rows, rope (T, dk)
    fp32 [sin | cos] or None -> y SplitPlanes (B, T, heads * dk)."""
    _, ldq = _rows(qkv, "qkv")
    b, t = qkv.shape[0], qkv.shape[1]
    if rope is not None and (_req(rope, torch.float32, "rope").dim() != 2 or rope.shape[0] < t or rope.shape[1] != dk):
        raise ValueError("rope must be (>= {}, {}), got {}".format(t, dk, tuple(rope.shape)))
    check(lib.xvb_rope_attention(qkv.data_ptr(), ldq, b, t, heads, dk,
                                 _ptr(_req(rope, torch.float32, "rope")) if rope is not None else None, 1 if rope_v else 0,
                                 float(score_mult), y.hi.data_ptr(), y.lo.data_ptr(), y.ld, _stream()), "xvb_rope_attention")


def conv_module(x, dw_weight, dw_bias, norm_a, norm_b, y, batch_norm=False, eps=1e-5, act=_lib.ACT_SWISH):
    """ConvolutionModule middle (xvb_conv_module): x (B, T, >= 2C) fp32 rows (pointwise_conv1's output), dw_weight (C, K)
    fp32, dw_bias (C,) -> GLU, depthwise conv, LayerNorm(gamma=norm_a, beta=norm_b) or y * norm_a + norm_b (folded eval
    BatchNorm), act -> y SplitPlanes (B, T, C)."""
    _, ldx = _rows(x, "x")
    b, t = x.shape[0], x.shape[1]
    c, k = dw_weight.shape
    check(lib.xvb_conv_module(x.data_ptr(), ldx, b, t, c, _ptr(_req(dw_weight, torch.float32, "dw_weight")),
                              _ptr(_req(dw_bias, torch.float32, "dw_bias")), k, _ptr(_req(norm_a, torch.float32, "norm_a")),
                              _ptr(_req(norm_b, torch.float32, "norm_b")), 1 if batch_norm else 0, eps, act, y.hi.data_ptr(),
                              y.lo.data_ptr(), y.ld, _stream()), "xvb_conv_module")


def stats_pool_ex(x, eps, mode, planes=False, lengths=None):
    """mode 0: StatisticsPooling; mode 1: ECAPA global context (unbiased var + eps).  lengths: int32 CUDA (B,) tensor of
    a masked batch (utterance b pools its first lengths[b] frames; xvb_stats_pool_lengths)."""
    x = _req(x, torch.float32, "x")
    b, t, c = x.shape
    out = torch.empty(b, 2 * c, dtype=torch.float32, device=x.device)
    op = SplitPlanes.empty((b, 1, 2 * c), x.device) if planes else None
    tail = (_ptr(out), op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, 2 * c, _stream())
    if lengths is None:
        check(lib.xvb_stats_pool_ex(_ptr(x), c, b, t, c, eps, mode, *tail), "xvb_stats_pool_ex")
    else:
        check(lib.xvb_stats_pool_lengths(_ptr(x), c, b, t, c, eps, mode, _ptr(_req(lengths, torch.int32, "lengths")), *tail),
              "xvb_stats_pool_lengths")
    return (out, op) if planes else out


def attn_stats_pool(logits, x, floor=1e-5, planes=False):
    """softmax over T of logits (B,T,C) -> weighted mean/std of x (B,T,C): (B,2C)."""
    logits = _req(logits, torch.float32, "logits")
    x = _req(x, torch.float32, "x")
    b, t, c = x.shape
    out = torch.empty(b, 2 * c, dtype=torch.float32, device=x.device)
    op = SplitPlanes.empty((b, 1, 2 * c), x.device) if planes else None
    check(lib.xvb_attn_stats_pool(_ptr(logits), c, _ptr(x), c, b, t, c, floor, _ptr(out),
                                  op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, 2 * c, _stream()),
          "xvb_attn_stats_pool")
    return (out, op) if planes else out


def lde_pool(x, mu, neg_beta, planes=False):
    """LDE pooling (xvb_lde_pool): x (B,T,C) fp32 (row stride may exceed C), mu (C,K) fp32, neg_beta (K,) fp32
    -> (B, C*K) fp32 [, SplitPlanes (B,1,round_up(C*K,8))]."""
    if x.dtype != torch.float32 or not x.is_cuda or x.dim() != 3 or x.stride(-1) != 1 or x.stride(0) != x.shape[1] * x.stride(1):
        raise TypeError("x must be a (B,T,C) CUDA float32 tensor with contiguous rows")
    mu = _req(mu, torch.float32, "mu")
    neg_beta = _req(neg_beta, torch.float32, "neg_beta")
    b, t, c = x.shape
    k = mu.shape[1]
    out = torch.empty(b, c * k, dtype=torch.float32, device=x.device)
    w = torch.empty(b * t, k, dtype=torch.float32, device=x.device)
    op = None
    if planes:
        op = SplitPlanes.empty((b, 1, (c * k + 7) // 8 * 8), x.device)
        if op.ld != c * k:
            op.hi.zero_()
            op.lo.zero_()
            op.channels = c * k
    check(lib.xvb_lde_pool(_ptr(x), x.stride(-2), b, t, c, _ptr(mu), k, _ptr(neg_beta), _ptr(w), _ptr(out),
                           op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, op.ld if op else 0, _stream()),
          "xvb_lde_pool")
    return (out, op) if planes else out


def small_affine(x, w, bias=None, bn_scale=None, bn_shift=None, relu=False, sigmoid=False, tanh=False, planes=False):
    """Segment-level fp32 affine on CUDA cores (xvb_small_affine): x (B, K) fp32, w (N, K) fp32 -> (B, N) fp32
    [, the same as SplitPlanes (B, 1, N)]."""
    x = _req(x, torch.float32, "x")
    w = _req(w, torch.float32, "w")
    b, k = x.shape
    n = w.shape[0]
    y = torch.empty(b, n, dtype=torch.float32, device=x.device)
    op = SplitPlanes.empty((b, 1, (n + 7) // 8 * 8), x.device) if planes else None
    flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0) | (TANH if tanh else 0) | (SIGMOID if sigmoid else 0)
    check(lib.xvb_small_affine(_ptr(x), k, _ptr(w), b, k, n, _ptr(bias), _ptr(bn_scale), _ptr(bn_shift), flags, _ptr(y), n,
                               op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, op.ld if op else 0, _stream()),
          "xvb_small_affine")
    return (y, op) if planes else y


def attn_head_stats_pool(logits, x, out_channels, gdiv, floor=1e-10, unweighted_var=False, planes=False, prior_logit=None,
                         prior_x=None, softplus2log=False, lengths=None):
    """Attention pooling with a head map (xvb_attn_head_stats_pool): logits (B,T,G) fp32 (any row pitch >= G), x (B,T,C)
    fp32; output channel o pools x[..., o % C] with softmax_T(logits[..., o // gdiv]).  -> (B, 2*out_channels).
    prior_logit / prior_x (C,) + softplus2log: the xi-vector form (a prior element in the softmax, logits = 2 log softplus).
    lengths: int32 CUDA (B,) tensor of a masked batch (xvb_attn_head_stats_pool_lengths): utterance b pools its first
    lengths[b] frames."""
    for name, v in (("logits", logits), ("x", x)):       # channel-slice views of wider buffers are fine: rows stay contiguous
        if v.dtype != torch.float32 or not v.is_cuda or v.dim() != 3 or v.stride(-1) != 1 or v.stride(0) != v.shape[1] * v.stride(1):
            raise TypeError("{} must be a (B,T,*) CUDA float32 tensor with contiguous rows".format(name))
    b, t, c = x.shape
    g = logits.shape[-1]
    out = torch.empty(b, 2 * out_channels, dtype=torch.float32, device=x.device)
    op = SplitPlanes.empty((b, 1, 2 * out_channels), x.device) if planes else None
    head = (_ptr(logits), logits.stride(-2), g, _ptr(x), x.stride(-2), b, t, c, out_channels, int(gdiv), floor,
            1 if unweighted_var else 0, _ptr(prior_logit), _ptr(prior_x), 1 if softplus2log else 0)
    tail = (_ptr(out), op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None, 2 * out_channels, _stream())
    if lengths is None:
        check(lib.xvb_attn_head_stats_pool_prior(*head, *tail), "xvb_attn_head_stats_pool")
    else:
        check(lib.xvb_attn_head_stats_pool_lengths(*head, _ptr(_req(lengths, torch.int32, "lengths")), *tail),
              "xvb_attn_head_stats_pool_lengths")
    return (out, op) if planes else out


def attn_head_stats_pool_mq(logits, x, out_channels, gdiv, head_width, rep, floor=1e-5, planes=False):
    """Multi-query multi-head attention pooling (xvb_attn_head_stats_pool_mq): output channel o pools
    x[..., (o // (rep*head_width))*head_width + o % head_width] with softmax_T(logits[..., o // gdiv]), weighted
    variance clamped at `floor`.  -> (B, 2*out_channels) [mean | std] (, SplitPlanes)."""
    for name, v in (("logits", logits), ("x", x)):
        if v.dtype != torch.float32 or not v.is_cuda or v.dim() != 3 or v.stride(-1) != 1 or v.stride(0) != v.shape[1] * v.stride(1):
            raise TypeError("{} must be a (B,T,*) CUDA float32 tensor with contiguous rows".format(name))
    b, t, c = x.shape
    out = torch.empty(b, 2 * out_channels, dtype=torch.float32, device=x.device)
    op = SplitPlanes.empty((b, 1, 2 * out_channels), x.device) if planes else None
    check(lib.xvb_attn_head_stats_pool_mq(_ptr(logits), logits.stride(-2), logits.shape[-1], _ptr(x), x.stride(-2), b, t, c,
                                          out_channels, int(gdiv), int(head_width), int(rep), floor, 0, _ptr(out),
                                          op.hi.data_ptr() if op else None, op.lo.data_ptr() if op else None,
                                          2 * out_channels, _stream()), "xvb_attn_head_stats_pool_mq")
    return (out, op) if planes else out


def tdnn_affine_simt(x, weight, context, bias=None, bn_scale=None, bn_shift=None, relu=False):
    """fp32 CUDA-core cross-check: x (B,T,Cin) fp32, weight (Cout,Cin,tot) as in the reference."""
    x = _req(x, torch.float32, "x")
    weight = _req(weight, torch.float32, "weight")
    b, t, cin = x.shape
    cout, _, tot = weight.shape
    left, _, _ = context_span(context)
    flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0)
    y = torch.empty(b, t, cout, dtype=torch.float32, device=x.device)
    check(lib.xvb_tdnn_affine_simt(_ptr(x), cin, _ptr(weight), tot, left, _ptr(bias), _ptr(bn_scale), _ptr(bn_shift),
                                   flags, int_array(context), len(context), _ptr(y), cout, b, t, cin, cout, _stream()),
          "xvb_tdnn_affine_simt")
    return y


def stats_pool(x, eps=1e-10, planes=False):
    """x (B,T,C) fp32 -> (B,2C) fp32 [, SplitPlanes]  (pooling.py:58-67)."""
    x = _req(x, torch.float32, "x")
    b, t, c = x.shape
    out = torch.empty(b, 2 * c, dtype=torch.float32, device=x.device)
    hi = lo = None
    if planes:
        hi = torch.empty(b, 2 * c, dtype=torch.bfloat16, device=x.device)
        lo = torch.empty_like(hi)
    check(lib.xvb_stats_pool(_ptr(x), c, b, t, c, eps, _ptr(out), _ptr(hi), _ptr(lo), 2 * c, _stream()),
          "xvb_stats_pool")
    return (out, SplitPlanes(hi, lo, 2 * c)) if planes else out


# ------------------------------------------------------------------ scoring
def center_length_norm(x, mean=None):
    x = _req(x, torch.float32, "x")
    y = torch.empty_like(x)
    check(lib.xvb_center_length_norm(_ptr(x), _ptr(mean), _ptr(y), x.shape[0], x.shape[1], _stream()),
          "xvb_center_length_norm")
    return y


def column_mean(x):
    x = _req(x, torch.float32, "x")
    m = torch.empty(x.shape[1], dtype=torch.float32, device=x.device)
    check(lib.xvb_column_mean(_ptr(x), x.shape[0], x.shape[1], _ptr(m), _stream()), "xvb_column_mean")
    return m


def cosine_trials(enroll, test, trial_e, trial_t):
    enroll = _req(enroll, torch.float32, "enroll")
    test = _req(test, torch.float32, "test")
    trial_e = _req(trial_e, torch.int32, "trial_e")
    trial_t = _req(trial_t, torch.int32, "trial_t")
    s = torch.empty(trial_e.shape[0], dtype=torch.float32, device=enroll.device)
    check(lib.xvb_cosine_trials(_ptr(enroll), _ptr(test), enroll.shape[1], _ptr(trial_e), _ptr(trial_t),
                                trial_e.shape[0], _ptr(s), _stream()), "xvb_cosine_trials")
    return s


def speaker_mean(x, spk2rows):
    """x (N,D) fp32 CUDA; spk2rows: list of row-index lists (spk2utt order) -> ((S,D) means, num_utts)."""
    x = _req(x, torch.float32, "x")
    counts = np.array([len(r) for r in spk2rows], dtype=np.int32)
    offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(x.device)
    members = torch.from_numpy(np.concatenate([np.asarray(r, dtype=np.int32) for r in spk2rows])).to(x.device)
    out = torch.empty(len(spk2rows), x.shape[1], dtype=torch.float32, device=x.device)
    check(lib.xvb_speaker_mean(_ptr(x), x.shape[1], _ptr(offsets), _ptr(members), len(spk2rows), _ptr(out), _stream()),
          "xvb_speaker_mean")
    return out, counts


def topn_mean_std(S, top_n=0, ddof=1):
    """Per row of a cohort score matrix: mean / std of the top_n largest entries (0 = all); ddof = 1 is pandas'
    .std() (score/ScoreNormalization.py), ddof = 0 np.std (subtools2/egrecho/score/asnorm.py)."""
    S = _req(S, torch.float32, "S")
    m = torch.empty(S.shape[0], dtype=torch.float32, device=S.device)
    sd = torch.empty_like(m)
    check(lib.xvb_topn_mean_std_ddof(_ptr(S), S.shape[1], S.shape[0], S.shape[1], int(top_n), int(ddof), _ptr(m), _ptr(sd),
                                     _stream()), "xvb_topn_mean_std")
    return m, sd


def snorm_trials(scores, trial_e, trial_t, mean_e, std_e, mean_t, std_t):
    scores = _req(scores, torch.float32, "scores")
    out = torch.empty_like(scores)
    check(lib.xvb_snorm_trials(_ptr(scores), _ptr(_req(trial_e, torch.int32, "trial_e")),
                               _ptr(_req(trial_t, torch.int32, "trial_t")), scores.shape[0], _ptr(mean_e), _ptr(std_e),
                               _ptr(mean_t), _ptr(std_t), _ptr(out), _stream()), "xvb_snorm_trials")
    return out


def bilinear_trials(enroll, test, trial_e, trial_t, row_term=None, col_term=None):
    enroll = _req(enroll, torch.float32, "enroll")
    test = _req(test, torch.float32, "test")
    trial_e = _req(trial_e, torch.int32, "trial_e")
    trial_t = _req(trial_t, torch.int32, "trial_t")
    s = torch.empty(trial_e.shape[0], dtype=torch.float32, device=enroll.device)
    check(lib.xvb_bilinear_trials(_ptr(enroll), _ptr(test), enroll.shape[1], _ptr(trial_e), _ptr(trial_t),
                                  trial_e.shape[0], _ptr(row_term), _ptr(col_term), _ptr(s), _stream()),
          "xvb_bilinear_trials")
    return s


def project(x, m):
    """x (rows, D) . m^T with m (Dout, D) -> (rows, Dout)."""
    x = _req(x, torch.float32, "x")
    m = _req(m, torch.float32, "m")
    y = torch.empty(x.shape[0], m.shape[0], dtype=torch.float32, device=x.device)
    check(lib.xvb_project(_ptr(x), x.shape[0], x.shape[1], _ptr(m), m.shape[0], _ptr(y), _stream()), "xvb_project")
    return y


def cosine_matrix(enroll, test):
    enroll = _req(enroll, torch.float32, "enroll")
    test = _req(test, torch.float32, "test")
    s = torch.empty(enroll.shape[0], test.shape[0], dtype=torch.float32, device=enroll.device)
    check(lib.xvb_cosine_matrix(_ptr(enroll), enroll.shape[0], _ptr(test), test.shape[0], enroll.shape[1], _ptr(s),
                                test.shape[0], _stream()), "xvb_cosine_matrix")
    return s


def plda_terms(x, gamma, c):
    x = _req(x, torch.float32, "x")
    term = torch.empty(x.shape[0], dtype=torch.float32, device=x.device)
    check(lib.xvb_plda_terms(_ptr(x), x.shape[0], x.shape[1], _ptr(_req(gamma, torch.float32, "gamma")),
                             _ptr(_req(c, torch.float32, "c")), _ptr(term), _stream()), "xvb_plda_terms")
    return term


def plda_matrix(enroll, test, l2, row, col):
    enroll = _req(enroll, torch.float32, "enroll")
    test = _req(test, torch.float32, "test")
    s = torch.empty(enroll.shape[0], test.shape[0], dtype=torch.float32, device=enroll.device)
    check(lib.xvb_plda_matrix(_ptr(enroll), enroll.shape[0], _ptr(test), test.shape[0], enroll.shape[1],
                              _ptr(_req(l2, torch.float32, "l2")), _ptr(row), _ptr(col), _ptr(s), test.shape[0],
                              _stream()), "xvb_plda_matrix")
    return s


def topn_indices(S, top_n):
    """(rows, top_n) int32: cohort indices of every row's top_n scores, best first."""
    S = _req(S, torch.float32, "S")
    top_n = min(int(top_n), S.shape[1])   # groupby().head(top_n): a cohort smaller than top_n is used whole
    idx = torch.empty(S.shape[0], top_n, dtype=torch.int32, device=S.device)
    check(lib.xvb_topn_indices(_ptr(S), S.shape[1], S.shape[0], S.shape[1], int(top_n), _ptr(idx), _stream()), "xvb_topn_indices")
    return idx


def snorm_cross_trials(scores, trial_e, trial_t, enroll_cohort, test_cohort, top_enroll, top_test):
    scores = _req(scores, torch.float32, "scores")
    out = torch.empty_like(scores)
    check(lib.xvb_snorm_cross_trials(_ptr(scores), _ptr(_req(trial_e, torch.int32, "trial_e")), _ptr(_req(trial_t, torch.int32, "trial_t")),
                                     scores.shape[0], _ptr(_req(enroll_cohort, torch.float32, "enroll_cohort")), enroll_cohort.shape[1],
                                     _ptr(_req(test_cohort, torch.float32, "test_cohort")), test_cohort.shape[1],
                                     _ptr(_req(top_enroll, torch.int32, "top_enroll")), _ptr(_req(top_test, torch.int32, "top_test")),
                                     top_enroll.shape[1], _ptr(out), _stream()), "xvb_snorm_cross_trials")
    return out


def matmul_nt(a, b, row_bias=None, col_bias=None):
    """a (M,K) . b (N,K)^T + row_bias[i] + col_bias[j] -> (M,N) fp32 on the wgmma layer (N % 4 == 0)."""
    a = _req(a, torch.float32, "a")
    b = a if b is a else _req(b, torch.float32, "b")
    out = torch.empty(a.shape[0], b.shape[0], dtype=torch.float32, device=a.device)
    check(lib.xvb_matmul_nt(_ptr(a), a.shape[0], _ptr(b), b.shape[0], a.shape[1], _ptr(row_bias), _ptr(col_bias), _ptr(out),
                            b.shape[0], _stream()), "xvb_matmul_nt")
    return out


def center_rows_transposed(x, spk, means, sqrt_weight=None):
    """-> (D, N): column i = sqrt_weight[spk[i]] * (x[i] - means[spk[i]])."""
    x = _req(x, torch.float32, "x")
    spk = _req(spk, torch.int32, "spk")
    means = _req(means, torch.float32, "means")
    out = torch.empty(x.shape[1], x.shape[0], dtype=torch.float32, device=x.device)
    check(lib.xvb_center_rows_transposed(_ptr(x), _ptr(spk), _ptr(means), _ptr(sqrt_weight), x.shape[0], x.shape[1], _ptr(out),
                                         x.shape[0], _stream()), "xvb_center_rows_transposed")
    return out


def plda_em_rows(u, n, weight, psi):
    """-> (what_T, resid_T), both (D, S); see include/xvb200.h."""
    u = _req(u, torch.float32, "u")
    s, d = u.shape
    what = torch.empty(d, s, dtype=torch.float32, device=u.device)
    resid = torch.empty(d, s, dtype=torch.float32, device=u.device)
    check(lib.xvb_plda_em_rows(_ptr(u), _ptr(_req(n, torch.float32, "n")), _ptr(weight), _ptr(_req(psi, torch.float32, "psi")),
                               s, d, _ptr(what), _ptr(resid), s, _stream()), "xvb_plda_em_rows")
    return what, resid


def plda_normalize_rows(u, psi, num_examples=None, simple=False):
    """In place: u[r] *= sqrt(D / sum_d u_d^2 / (psi_d + 1/n_r))  (simple: sqrt(D) / ||u[r]||)."""
    u = _req(u, torch.float32, "u")
    check(lib.xvb_plda_normalize_rows(_ptr(u), _ptr(_req(psi, torch.float32, "psi")), _ptr(num_examples), u.shape[0], u.shape[1],
                                      int(bool(simple)), _stream()), "xvb_plda_normalize_rows")
    return u


def plda_llr_operands(u, psi, num_examples, side):
    """-> ((rows, 2D) operand, (rows,) term) of the Kaldi-style PLDA LLR; side 0 = enroll, 1 = test."""
    u = _req(u, torch.float32, "u")
    a = torch.empty(u.shape[0], 2 * u.shape[1], dtype=torch.float32, device=u.device)
    term = torch.empty(u.shape[0], dtype=torch.float32, device=u.device)
    check(lib.xvb_plda_llr_operands(_ptr(u), _ptr(_req(psi, torch.float32, "psi")), _ptr(num_examples), u.shape[0], u.shape[1],
                                    int(side), _ptr(a), _ptr(term), _stream()), "xvb_plda_llr_operands")
    return a, term


def trial_histogram(enroll, enroll_spk, test, test_spk, lo, hi, nbins=2048, row_term=None, col_term=None,
                    symmetric=False, unit_first=0, unit_stride=1, out=None):
    """(2, nbins) int64 histogram [nontarget | target] of enroll.test^T (+ terms) -- scores are never
    stored.  `out` is accumulated into when given."""
    enroll = _req(enroll, torch.float32, "enroll")
    test = enroll if test is enroll else _req(test, torch.float32, "test")
    enroll_spk = _req(enroll_spk, torch.int32, "enroll_spk")
    test_spk = enroll_spk if test_spk is enroll_spk else _req(test_spk, torch.int32, "test_spk")
    if enroll_spk.shape[0] != enroll.shape[0] or test_spk.shape[0] != test.shape[0] or enroll.shape[1] != test.shape[1]:
        raise ValueError("trial_histogram: shape mismatch")
    if out is None:
        out = torch.zeros(2, nbins, dtype=torch.int64, device=enroll.device)
    elif out.dtype != torch.int64 or tuple(out.shape) != (2, nbins) or not out.is_contiguous() or out.device != enroll.device:
        raise ValueError("trial_histogram: out must be a contiguous (2, nbins) int64 tensor on the embeddings' device")
    check(lib.xvb_trial_histogram(_ptr(enroll), enroll.shape[0], _ptr(enroll_spk), _ptr(test), test.shape[0],
                                  _ptr(test_spk), enroll.shape[1], _ptr(row_term), _ptr(col_term), int(bool(symmetric)),
                                  int(unit_first), int(unit_stride), float(lo), float(hi), int(nbins), _ptr(out),
                                  _stream()), "xvb_trial_histogram")
    return out


# Test columns scored per GEMM call.  tools/bench_retrieval.py (H100 80GB HBM3, 700 W, N = 10^6, D = 256): 16 384,
# 65 536 and 262 144 columns ran within 2.6 % of each other at M = 1 000; at M = 10 000, 16 384 was the fastest.
RETRIEVE_SLAB_COLS = 16384
RETRIEVE_SLAB_BYTES = 1 << 30   # the default slab is narrowed so that M x slab_cols fp32 scores stay within 1 GiB


def retrieve_topk(enroll, test, k, row_bias=None, col_bias=None, slab_cols=None):
    """(scores (M, k) fp32, indices (M, k) int64): the k best test rows of every enroll row under
    enroll . test^T + row_bias[i] + col_bias[j], best first, equal scores by lower test index.  A row with fewer
    than k test rows has (-inf, -1) in its empty slots.  The (M, N) score matrix is never stored: the test set is
    scored `slab_cols` rows at a time (a multiple of 4) and merged into running lists."""
    a = _req(enroll, torch.float32, "enroll")
    b = _req(test, torch.float32, "test")
    if a.dim() != 2 or b.dim() != 2 or a.shape[1] != b.shape[1]:
        raise ValueError("retrieve_topk: enroll (M, D) and test (N, D) must share D")
    for t, n, name in ((row_bias, a.shape[0], "row_bias"), (col_bias, b.shape[0], "col_bias")):
        if t is not None and (_req(t, torch.float32, name).numel() != n):
            raise ValueError("retrieve_topk: {} must hold {} values".format(name, n))
    m, n = a.shape[0], b.shape[0]
    if slab_cols is None:
        fit = max(4, RETRIEVE_SLAB_BYTES // (4 * m) // 4 * 4)
        slab_cols = min(RETRIEVE_SLAB_COLS, fit, (n + 3) // 4 * 4)
    nbytes = lib.xvb_retrieve_topk_slab_bytes(m, int(slab_cols))
    check(0 if nbytes > 0 else nbytes, "xvb_retrieve_topk_slab_bytes")
    slab = torch.empty(nbytes // 4, dtype=torch.float32, device=a.device)
    scores = torch.empty(m, int(k), dtype=torch.float32, device=a.device)
    idx = torch.empty(m, int(k), dtype=torch.int64, device=a.device)
    check(lib.xvb_retrieve_topk(_ptr(a), m, _ptr(b), n, a.shape[1], _ptr(row_bias), _ptr(col_bias), int(k), _ptr(slab),
                                int(slab_cols), _ptr(scores), _ptr(idx), _stream()), "xvb_retrieve_topk")
    return scores, idx


# ------------------------------------------------------------------ whole-model extractor
class Extractor(ShardExtractor):
    """Owner of a native xvb_extractor_t (packed weights + workspace on the current device), built layer by layer with
    add_frame_layer / add_segment_layer / finalize or loaded from an XVBM0001 file; save() writes that file."""

    TAKES_LENGTHS = True

    PREFIX = "extractor"
    batch = 256

    def __init__(self, feat_dim):
        self._lib, self._check = lib, check
        self._h = C.c_void_p()
        check(lib.xvb_extractor_create(C.byref(self._h), int(feat_dim)), "xvb_extractor_create")
        self.feat_dim = int(feat_dim)

    @staticmethod
    def _np(a):
        if a is None:
            return None, None
        a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
        return a, a.ctypes.data_as(C.c_void_p)

    def add_frame_layer(self, weight, bias, context, bn_scale=None, bn_shift=None, relu=True):
        w, wp = self._np(weight)
        b, bp = self._np(bias)
        s, sp = self._np(bn_scale)
        t, tp = self._np(bn_shift)
        flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0)
        check(lib.xvb_extractor_add_frame_layer(self._h, w.shape[0], int_array(context), len(context), wp, bp, sp, tp,
                                                flags), "xvb_extractor_add_frame_layer")

    def add_segment_layer(self, weight, bias, bn_scale=None, bn_shift=None, relu=False):
        w, wp = self._np(weight)
        b, bp = self._np(bias)
        s, sp = self._np(bn_scale)
        t, tp = self._np(bn_shift)
        flags = (RELU if relu else 0) | (BN if bn_scale is not None else 0)
        check(lib.xvb_extractor_add_segment_layer(self._h, w.shape[0], wp, bp, sp, tp, flags),
              "xvb_extractor_add_segment_layer")

    def finalize(self, pooling_eps=1e-10):
        check(lib.xvb_extractor_finalize(self._h, pooling_eps), "xvb_extractor_finalize")
        self.embed_dim = lib.xvb_extractor_embed_dim(self._h)

    @classmethod
    def load(cls, path):
        """An extractor straight from an .xvbm file (no Python-side layer objects)."""
        self = cls.__new__(cls)
        self._lib, self._check = lib, check
        self._h = C.c_void_p()
        check(lib.xvb_extractor_load(C.byref(self._h), str(path).encode()), "xvb_extractor_load")
        self.feat_dim = lib.xvb_extractor_feat_dim(str(path).encode())
        self.embed_dim = lib.xvb_extractor_embed_dim(self._h)
        return self

    def extract(self, feats, lengths=None):
        """feats (B,T,F) fp32 CUDA -> (B,D) fp32 CUDA, asynchronous on the current stream.  lengths (B,) host ints
        (sequence, ndarray or CPU tensor), 1 <= lengths[b] <= T: a batch of utterances of different lengths, row b being
        feats[b, :lengths[b]] extracted alone (xvb_extractor_extract_lengths); the frames past them are never read."""
        feats = _req(feats, torch.float32, "feats")
        b, t, f = feats.shape
        if f != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, f))
        emb = torch.empty(b, self.embed_dim, dtype=torch.float32, device=feats.device)
        if lengths is None:
            check(lib.xvb_extractor_extract(self._h, _ptr(feats), b, t, _ptr(emb), _stream()), "xvb_extractor_extract")
            return emb
        lens = host_lengths(lengths, b)
        check(lib.xvb_extractor_extract_lengths(self._h, _ptr(feats), lens.ctypes.data_as(C.c_void_p), b, t, _ptr(emb),
                                                _stream()), "xvb_extractor_extract_lengths")
        return emb

    def submit_host(self, feats_ptr, b, t, emb_ptr, slot):
        """Pipelined host path: queue batch `slot` (0/1); pair with wait(slot)."""
        check(lib.xvb_extractor_submit_host(self._h, C.c_void_p(feats_ptr), b, t, C.c_void_p(emb_ptr), slot, _stream()),
              "xvb_extractor_submit_host")

    def wait(self, slot):
        check(lib.xvb_extractor_wait(self._h, slot), "xvb_extractor_wait")

    def extract_host_into(self, feats_ptr, b, t, emb_ptr):
        check(lib.xvb_extractor_extract_host(self._h, C.c_void_p(feats_ptr), b, t, C.c_void_p(emb_ptr), _stream()),
              "xvb_extractor_extract_host")

    def set_fused_pooling(self, enable):
        """Default on: tdnn5's epilogue pools over time itself; off: fp32 tensor + standalone pooling kernel."""
        check(lib.xvb_extractor_set_fused_pooling(self._h, 1 if enable else 0), "xvb_extractor_set_fused_pooling")

    def set_profiling(self, enable):
        check(lib.xvb_extractor_set_profiling(self._h, 1 if enable else 0), "xvb_extractor_set_profiling")

    def kernel_times_ms(self, max_n=64):
        """Durations (ms) between consecutive profiling events of the last extract call, launch order (needs
        set_profiling).  After extract_shard(): every batch contributes its kernels plus the gap to the next batch."""
        buf = (C.c_float * max_n)()
        n = lib.xvb_extractor_kernel_times(self._h, buf, max_n)
        if n < 0:
            check(n, "xvb_extractor_kernel_times")
        return [float(buf[i]) for i in range(n)]

    def debug_f32(self, which, shape):
        """View of an internal fp32 buffer of the last call (which=-1: pooled stats, 0: last frame layer)."""
        ptr = lib.xvb_extractor_debug_f32(self._h, which)
        if not ptr:
            raise _lib.XvbError("no debug buffer")

        class _DevPtr:  # zero-copy view through the CUDA array interface
            __cuda_array_interface__ = {"shape": tuple(shape), "typestr": "<f4", "data": (int(ptr), False),
                                        "version": 2}

        torch.cuda.synchronize()
        return torch.as_tensor(_DevPtr(), device="cuda").clone()
