#!/usr/bin/env python
"""Seeded outputs of the 2-D conv entry points (xvb_conv2d, xvb_conv2d_taps) and the layer kernel (xvb_tdnn_affine_ex,
every existing epilogue flag, the split-K segment path and the fused pooling) written to one .npz, so that two builds of
the library can be compared bit for bit:

    python tools/dump_kernel_outputs.py <repository root> <out.npz>

The package is imported from the given root, so a second checkout (e.g. the parent commit, built) can be dumped by the
same script and the two files compared with numpy.array_equal."""
import os
import sys

import numpy as np


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
    np.savez(out, **res)
    print(out, len(res), "arrays")


if __name__ == "__main__":
    main()
