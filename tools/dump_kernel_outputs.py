#!/usr/bin/env python
"""Seeded outputs of the 2-D conv entry points (xvb_conv2d, xvb_conv2d_taps), xvb_se_apply, the Conformer's head conv
(xvb_subsample_head[_stride]) and attention (xvb_rope_attention, softmax and softmax_plus), xvb_attn_stats_pool and the
layer kernel
(xvb_tdnn_affine_ex, every existing epilogue flag, the split-K segment path and the fused pooling; the five frame layers of bench.py at
256 x 200, with the im2col first layer and tdnn5's fused pooling; an ECAPA-sized and a Conformer-sized layer) written to
one .npz, so that two builds of the library can be compared bit for bit:

    python tools/dump_kernel_outputs.py <repository root> <out.npz>

The package is imported from the given root, so a second checkout (e.g. the parent commit, built) can be dumped by the
same script and the two files compared with numpy.array_equal."""
import os
import sys

import numpy as np


def im2col_layer(x, w, cin, cout, B, T, bias, scale, shift, y):
    """The extractor's first layer: frame t reads rows t .. t + window - 1 of the time-padded planes x as one K = cin
    row (xvb_tdnn_affine_ex with x_batch_stride), + bias -> ReLU -> BN."""
    import ctypes as C
    import torch
    from asv_subtools_b200._lib import BN, RELU, TdnnArgs, check, int_array, lib
    a = TdnnArgs()
    a.x_hi, a.x_lo, a.ldx, a.x_batch_stride = x.hi.data_ptr(), x.lo.data_ptr(), x.ld, x.hi.stride(0)
    a.w_hi, a.w_lo = w.hi.data_ptr(), w.lo.data_ptr()
    a.bias, a.bn_scale, a.bn_shift, a.flags = bias.data_ptr(), scale.data_ptr(), shift.data_ptr(), RELU | BN
    ctx = int_array([0])
    a.context_host, a.ntaps = ctx, 1
    a.y_hi, a.y_lo, a.ldy = y.hi.data_ptr(), y.lo.data_ptr(), y.ld
    a.B, a.T, a.Cin, a.Cout = B, T, cin, cout
    check(lib.xvb_tdnn_affine_ex(C.byref(a), C.c_void_p(torch.cuda.current_stream().cuda_stream)), "im2col layer")


def main():
    root, out = sys.argv[1], sys.argv[2]
    sys.path.insert(0, os.path.abspath(root))
    import torch
    from asv_subtools_b200 import ops
    from asv_subtools_b200._lib import BN, RELU, SIGMOID, TANH  # noqa: F401
    g = torch.Generator(device="cuda").manual_seed(1234)

    def rnd(*shape, scale=1.0):
        return torch.randn(*shape, generator=g, device="cuda") * scale

    res = {}
    # xvb_conv2d / xvb_conv2d_taps: (Cin, Cout, k, stride, F, T, B, taps)
    for i, (cin, cout, k, s, F, T, B, taps) in enumerate([
            (32, 32, 3, 1, 80, 37, 3, None), (64, 128, 3, 2, 40, 51, 2, None), (128, 256, 1, 2, 21, 25, 3, None),
            (256, 256, 3, 2, 39, 149, 4, None), (32, 64, 5, 2, 79, 37, 3, [0, 2, 4, 6, 7, 8, 10, 11, 12, 13, 14, 16, 17, 18,
                                                                            20, 22, 24]),
            (48, 96, 3, 1, 23, 151, 1, [1, 3, 4, 8])]):
        x = ops.split_f32(torch.relu(rnd(B, T, F, cin)).contiguous())
        w = rnd(cout, cin, k, k, scale=1.0 / np.sqrt(cin * k * k))
        To, Fo = (T - 1) // s + 1, (F - 1) // s + 1
        sc, sh = 1 + 0.1 * rnd(cout), 0.1 * rnd(cout)
        res_p = ops.split_f32(rnd(B, To, Fo, cout).contiguous())
        y = ops.SplitPlanes.empty((B, To, Fo, cout), "cuda")
        y2 = ops.SplitPlanes.empty((B, To, Fo, cout), "cuda")
        yf = torch.empty(B, To, Fo, cout, device="cuda")
        ops.conv2d(x, ops.pack_conv2d_weight(w.contiguous(), taps), cout, k, s, sc, sh, res=res_p, relu=True, y=y, y_f32=yf,
                   scale2=sc, shift2=sh, y2=y2, taps=taps)
        res["conv{}_y_hi".format(i)] = y.hi.view(torch.int16).cpu().numpy()
        res["conv{}_y_lo".format(i)] = y.lo.view(torch.int16).cpu().numpy()
        res["conv{}_y2_hi".format(i)] = y2.hi.view(torch.int16).cpu().numpy()
        res["conv{}_f32".format(i)] = yf.cpu().numpy()
    # xvb_tdnn_affine_ex: frame layers with each epilogue, a segment layer (T = 1, split-K), fused pooling
    for i, (B, T, cin, cout, ctx, kw) in enumerate([
            (4, 200, 80, 512, [-2, -1, 0, 1, 2], {"relu": True, "bn": True}),
            (3, 74, 256, 2048, [0], {}), (3, 74, 1536, 128, [0], {"tanh": True}), (5, 37, 128, 96, [-3, 0, 3], {"sigmoid": True}),
            (128, 1, 3072, 256, [0], {"relu": True, "bn": True}), (2, 1, 1024, 8, [0], {"sigmoid": True})]):
        x = ops.split_f32(rnd(B, T, cin))
        span = ctx[-1] - min(ctx[0], 0) + 1
        w = rnd(cout, cin, span, scale=1.0 / np.sqrt(cin * len(ctx)))
        bias = 0.1 * rnd(cout)
        sc, sh = (1 + 0.1 * rnd(cout), 0.1 * rnd(cout)) if kw.get("bn") else (None, None)
        y = ops.SplitPlanes.empty((B, T, cout), "cuda")
        yf = torch.empty(B, T, cout, device="cuda")
        ops.tdnn_affine_ex(x, ops.pack_tdnn_weight(w, ctx), cout, ctx, bias=bias, bn_scale=sc, bn_shift=sh,
                           relu=kw.get("relu", False), tanh=kw.get("tanh", False), sigmoid=kw.get("sigmoid", False), y=y,
                           y_f32=yf)
        res["tdnn{}_y_hi".format(i)] = y.hi.view(torch.int16).cpu().numpy()
        res["tdnn{}_y_lo".format(i)] = y.lo.view(torch.int16).cpu().numpy()
        res["tdnn{}_f32".format(i)] = yf.cpu().numpy()
    x = ops.split_f32(rnd(4, 150, 512))
    w = rnd(1500, 512, 1, scale=1.0 / np.sqrt(512))
    res["pool"] = ops.fused_pool_layer(x, ops.pack_tdnn_weight(w, [0]), 1500, [0], bias=0.1 * rnd(1500)).cpu().numpy()
    # the layer shapes bench.py runs (256 x 200, x-vector spec: the im2col first layer, tdnn2-4, tdnn5 with fused
    # pooling), an ECAPA-sized and a Conformer-sized layer
    B, T = 256, 200
    xin = ops.split_f32(torch.nn.functional.pad(rnd(B, T, 80), (0, 0, 2, 2)).contiguous())   # time-padded planes
    w = rnd(512, 400, 1, scale=1.0 / np.sqrt(400))
    y = ops.SplitPlanes.empty((B, T, 512), "cuda")
    im2col_layer(xin, ops.pack_tdnn_weight(w, [0]), 400, 512, B, T, 0.1 * rnd(512), 1 + 0.1 * rnd(512), 0.1 * rnd(512), y)
    res["bench_tdnn1_y_hi"] = y.hi.view(torch.int16).cpu().numpy()
    res["bench_tdnn1_y_lo"] = y.lo.view(torch.int16).cpu().numpy()
    x = y
    for i, ctx in ((2, [-2, 0, 2]), (3, [-3, 0, 3]), (4, [0])):
        span = ctx[-1] - min(ctx[0], 0) + 1
        w = rnd(512, 512, span, scale=1.0 / np.sqrt(512 * len(ctx)))
        y = ops.SplitPlanes.empty((B, T, 512), "cuda")
        ops.tdnn_affine_ex(x, ops.pack_tdnn_weight(w, ctx), 512, ctx, bias=0.1 * rnd(512), bn_scale=1 + 0.1 * rnd(512),
                           bn_shift=0.1 * rnd(512), relu=True, y=y)
        res["bench_tdnn{}_y_hi".format(i)] = y.hi.view(torch.int16).cpu().numpy()
        res["bench_tdnn{}_y_lo".format(i)] = y.lo.view(torch.int16).cpu().numpy()
        x = y
    w = rnd(1500, 512, 1, scale=1.0 / np.sqrt(512))
    res["bench_tdnn5_pool"] = ops.fused_pool_layer(x, ops.pack_tdnn_weight(w, [0]), 1500, [0], bias=0.1 * rnd(1500),
                                                   bn_scale=1 + 0.1 * rnd(1500), bn_shift=0.1 * rnd(1500)).cpu().numpy()
    for name, (B, T, cin, cout, ctx) in (("ecapa", (64, 200, 1024, 1024, [0])), ("conformer", (128, 74, 256, 2048, [0]))):
        x = ops.split_f32(rnd(B, T, cin))
        w = rnd(cout, cin, 1, scale=1.0 / np.sqrt(cin))
        yf = torch.empty(B, T, cout, device="cuda")
        ops.tdnn_affine_ex(x, ops.pack_tdnn_weight(w, ctx), cout, ctx, bias=0.1 * rnd(cout), relu=True, y_f32=yf)
        res[name + "_f32"] = yf.cpu().numpy()
    # xvb_se_apply (SE scaling + residual, with and without the running sum), a channel-slice view as in ECAPA
    for i, (B, T, C, nxt) in enumerate([(4, 200, 512, True), (3, 37, 1024, False)]):
        z, xin = ops.split_f32(rnd(B, T, 2 * C)).slice(0, C), ops.split_f32(rnd(B, T, C))
        out_p, nxt_p = ops.SplitPlanes.empty((B, T, C), "cuda"), ops.SplitPlanes.empty((B, T, C), "cuda")
        ops.se_apply(z, xin, torch.sigmoid(rnd(B, C)), out_p, nxt_p if nxt else None)
        for name, p in (("out", out_p), ("next", nxt_p)) if nxt else (("out", out_p),):
            res["se_apply{}_{}_hi".format(i, name)] = p.hi.view(torch.int16).cpu().numpy()
            res["se_apply{}_{}_lo".format(i, name)] = p.lo.view(torch.int16).cpu().numpy()
    # the Conformer head conv at both feature strides
    for sf in (2, 1):
        feats = rnd(3, 301, 80)
        F1 = (80 - 1) // 2 if sf == 2 else 80 - 2
        y = ops.SplitPlanes.empty((3, 150, F1, 256), "cuda")
        ops.subsample_head(feats, rnd(256, 1, 3, 3, scale=1.0 / 3), 0.1 * rnd(256), y, stride_f=None if sf == 2 else 1)
        res["subsample_head_sf{}_hi".format(sf)] = y.hi.view(torch.int16).cpu().numpy()
        res["subsample_head_sf{}_lo".format(sf)] = y.lo.view(torch.int16).cpu().numpy()
    # the attention: each d_k, no rope / rope / rope on the values too, softmax and a softmax_plus multiplier
    for dk, H, T, rope_mode, mult in ((32, 8, 98, 0, 1.0), (64, 4, 74, 1, 1.0), (128, 2, 240, 2, 1.0), (64, 4, 74, 2, 0.7391),
                                      (32, 4, 33, 1, 1.3137)):
        qkv = rnd(3, T, 3 * H * dk)
        rope = torch.cat([torch.sin(rnd(T, dk // 2)), torch.cos(rnd(T, dk // 2))], 1).contiguous() if rope_mode else None
        y = ops.SplitPlanes.empty((3, T, H * dk), "cuda")
        ops.rope_attention(qkv, H, dk, y, rope=rope, rope_v=rope_mode == 2, score_mult=mult)
        key = "rope_attention_dk{}_T{}_r{}_m{}".format(dk, T, rope_mode, mult)
        res[key + "_hi"] = y.hi.view(torch.int16).cpu().numpy()
        res[key + "_lo"] = y.lo.view(torch.int16).cpu().numpy()
    # xvb_attn_stats_pool: the Conformer's 1536 channels and ECAPA's 3072, with plane outputs, and a channel tail
    for B, T, C in ((4, 74, 1536), (3, 200, 3072), (2, 33, 200)):
        st, op = ops.attn_stats_pool(rnd(B, T, C), rnd(B, T, C), floor=1e-5, planes=True)
        res["attn_stats_pool_{}x{}x{}".format(B, T, C)] = st.cpu().numpy()
        res["attn_stats_pool_{}x{}x{}_hi".format(B, T, C)] = op.hi.view(torch.int16).cpu().numpy()
    np.savez(out, **res)
    print(out, len(res), "arrays")


if __name__ == "__main__":
    main()
