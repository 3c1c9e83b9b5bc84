#!/usr/bin/env python
"""Per-layer rate of the x-vector frame layers on the layer kernel (xvb_tdnn_affine_ex) at bench.py's shape:
B = 256 utterances x T = 200 frames, 80-d features, the x-vector spec.  tdnn1 runs as the extractor's im2col view
(time-padded planes, K = 5 x 80), tdnn5 with the fused statistics pooling.

    python tools/gemm_layers.py [--root DIR] [--seconds S]

Each layer is launched back to back for about S seconds on rotating inputs and outputs larger than the L2 cache, timed
with CUDA events.  Printed per layer: microseconds per launch, executed TFLOP/s (three bf16 MMAs per MAC), and the
L2 -> shared-memory operand traffic of the launch (128 x 128 tiles x K blocks x the 64 KB four-plane stage every CTA
loads for itself) as GB/s.  All five layers run with BLOCK_N = 128 on one persistent CTA per SM.  The package is
imported from --root, so two builds can be measured by the same script."""
import argparse
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# name, Cin, Cout, context, im2col first layer, fused pooling
LAYERS = [
    ("tdnn1", 80, 512, [-2, -1, 0, 1, 2], True, False),
    ("tdnn2", 512, 512, [-2, 0, 2], False, False),
    ("tdnn3", 512, 512, [-3, 0, 3], False, False),
    ("tdnn4", 512, 512, [0], False, False),
    ("tdnn5", 512, 1500, [0], False, True),
]
L2_BYTES = 50 * 2 ** 20
STAGE_BYTES = 2 * (128 * 64 * 2) + 2 * (128 * 64 * 2)   # frame hi/lo + weight hi/lo, 64 channels of K


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not readable"
    return "{} ({})".format(name, q)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", default=HERE)
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, default=200)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import numpy as np
    import torch
    from asv_subtools_b200 import ops
    from asv_subtools_b200._lib import BN, RELU, TdnnArgs, check, int_array, lib

    B, T = args.B, args.T
    torch.manual_seed(5)
    dev = "cuda"
    tb = C.c_int()
    nblk = lib.xvb_pool_partial_blocks(B, T, C.byref(tb))
    Tb = tb.value
    Bb = 128 // Tb
    m_units = nblk * ((B + Bb - 1) // Bb)
    stream = torch.cuda.current_stream().cuda_stream
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print("card: {}, {} SMs".format(card(), sms))
    print("B={} T={} M tile {} frames x {} utterances, {} M units".format(B, T, Tb, Bb, m_units))
    total_us = 0.0
    for name, cin, cout, ctx, im2col, pool in LAYERS:
        span = ctx[-1] - min(ctx[0], 0) + 1
        w = torch.randn(cout, cin, span, device=dev) / np.sqrt(cin * len(ctx))
        if im2col:    # window of 5 consecutive frames of the time-padded planes = one K = 400 row
            kcin, kctx = cin * len(ctx), [0]
            wp = ops.pack_tdnn_weight(w.permute(0, 2, 1).reshape(cout, kcin, 1).contiguous(), kctx)
            in_shape = (B, T + span - 1, cin)
        else:
            kcin, kctx = cin, ctx
            wp = ops.pack_tdnn_weight(w, ctx)
            in_shape = (B, T, cin)
        bias = 0.1 * torch.randn(cout, device=dev)
        sc, sh = 1 + 0.1 * torch.randn(cout, device=dev), 0.1 * torch.randn(cout, device=dev)
        in_bytes = 4 * int(np.prod(in_shape))
        out_bytes = nblk * B * 2 * cout * 4 if pool else 4 * B * T * cout
        nbuf = max(2, -(-2 * L2_BYTES // (in_bytes + out_bytes)))
        keep, arglist = [], []
        for _ in range(nbuf):
            x = ops.split_f32(torch.randn(*in_shape, device=dev))
            a = TdnnArgs()
            a.x_hi, a.x_lo, a.ldx = x.hi.data_ptr(), x.lo.data_ptr(), x.ld
            if im2col:
                a.x_batch_stride = x.hi.stride(0)
            a.w_hi, a.w_lo = wp.hi.data_ptr(), wp.lo.data_ptr()
            a.bias, a.bn_scale, a.bn_shift = bias.data_ptr(), sc.data_ptr(), sh.data_ptr()
            a.flags = RELU | BN
            c = int_array(kctx)
            a.context_host, a.ntaps = c, len(kctx)
            if pool:
                y = torch.empty(nblk, B, 2 * cout, device=dev)
                a.pool_partial = y.data_ptr()
            else:
                y = ops.SplitPlanes.empty((B, T, cout), dev)
                a.y_hi, a.y_lo, a.ldy = y.hi.data_ptr(), y.lo.data_ptr(), y.ld
            a.B, a.T, a.Cin, a.Cout = B, T, kcin, cout
            keep += [x, y, c]
            arglist.append(a)

        def run(n):
            for i in range(n):
                check(lib.xvb_tdnn_affine_ex(C.byref(arglist[i % nbuf]), C.c_void_p(stream)), name)

        run(3 * nbuf)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        run(20)
        e1.record()
        torch.cuda.synchronize()
        n = max(20, int(args.seconds * 1e3 / (e0.elapsed_time(e1) / 20)))
        e0.record()
        run(n)
        e1.record()
        torch.cuda.synchronize()
        us = e0.elapsed_time(e1) * 1e3 / n
        total_us += us
        tiles = m_units * -(-cout // 128)
        kblocks = len(kctx) * -(-kcin // 64)
        l2_bytes = tiles * kblocks * STAGE_BYTES
        flop = 6.0 * B * T * cout * len(ctx) * cin
        print("{:6s} {:8.1f} us  {:6.1f} TFLOP/s executed  {:6.0f} GB/s L2->SMEM ({:.2f} GB)  {} tiles x {} K blocks, "
              "{:.2f} tiles per CTA  ({} launches)".format(
                  name, us, flop / us * 1e-6, l2_bytes / us * 1e-3, l2_bytes * 1e-9, tiles, kblocks, tiles / sms, n))
    print("frame layers: {:.1f} us per batch".format(total_us))


if __name__ == "__main__":
    main()
