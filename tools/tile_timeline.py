#!/usr/bin/env python
"""Per-tile timeline of the layer kernel on the five frame layers of bench.py's shape (256 x 200), set up as
tools/gemm_layers.py sets them up.

    make -C asv_subtools_b200/csrc timeline
    python tools/tile_timeline.py [--direct-stores] [--B 256] [--T 200]

Needs the timeline build of the library (libxvb200_timeline.so, compiled with -DXVB_TILE_TIMELINE), which this script
loads in place of the default one; that build's kernel is slower than the shipped one, so its times are for the split
between main loop, epilogue and waiting, not for the layer's rate.  Each consumer warpgroup stamps clock64 per tile;
the CTA's head carries %globaltimer and clock64 at both ends, which converts clocks to microseconds per CTA.

Printed per layer, medians over all tiles of one launch (after two warm-up launches): main loop (start to MMAs
retired), epilogue (MMAs retired to epilogue end), the wait on the operand ring's full barriers inside the main loop,
and the share of the CTAs' time during which neither warpgroup had MMAs in flight (from a tile's first operands
arriving to its MMAs retiring).  The epilogue is then split into the time warpgroup thread 0 spent waiting for
the TMA reads of the staging buffer, loading coefficients and on the epilogue's named barriers, on the arithmetic and
staging (or, without staging, the stores), and issuing the TMA stores.  --direct-stores keeps the plans on the direct-store layer epilogue and the fused
pooling epilogue on its general path."""
import argparse
import ctypes as C
import os
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(HERE, "tools"))
HEAD, REC = 8, 12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=256)
    ap.add_argument("--T", type=int, default=200)
    ap.add_argument("--direct-stores", action="store_true")
    args = ap.parse_args()
    tl_lib = os.path.join(HERE, "asv_subtools_b200", "libxvb200_timeline.so")
    if not os.path.exists(tl_lib):
        sys.exit("tile_timeline: {} not found -- make -C asv_subtools_b200/csrc timeline".format(tl_lib))
    os.environ["XVB_LIB"] = tl_lib
    sys.path.insert(0, HERE)
    import numpy as np
    import torch
    from gemm_layers import LAYERS, card
    from asv_subtools_b200 import ops
    from asv_subtools_b200._lib import BN, RELU, TdnnArgs, check, int_array, lib

    lib.xvb_tile_timeline_set.restype = None
    lib.xvb_tile_timeline_set.argtypes = [C.c_void_p, C.c_int, C.c_int]
    B, T = args.B, args.T
    torch.manual_seed(5)
    dev = "cuda"
    tb = C.c_int()
    nblk = lib.xvb_pool_partial_blocks(B, T, C.byref(tb))
    Bb = 128 // tb.value
    m_units = nblk * ((B + Bb - 1) // Bb)
    stream = torch.cuda.current_stream().cuda_stream
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print("card: {}, {} SMs".format(card(), sms))
    print("B={} T={}, {} epilogue of the layer kernel (timeline build)".format(
        B, T, "direct-store / general pooling" if args.direct_stores else "staged TMA-store / full-block pooling"))
    print("{:6s} {:>9s} {:>10s} {:>9s} {:>9s} {:>12s} {:>10s} | {:>9s} {:>10s} {:>9s} {:>9s}".format(
        "layer", "tiles/CTA", "main loop", "epilogue", "op. wait", "no MMA", "CTA time",
        "TMA read", "coef+bar", "arith", "store"))
    for name, cin, cout, ctx, im2col, pool in LAYERS:
        span = ctx[-1] - min(ctx[0], 0) + 1
        w = torch.randn(cout, cin, span, device=dev) / np.sqrt(cin * len(ctx))
        if im2col:
            kcin, kctx = cin * len(ctx), [0]
            wp = ops.pack_tdnn_weight(w.permute(0, 2, 1).reshape(cout, kcin, 1).contiguous(), kctx)
            in_shape = (B, T + span - 1, cin)
        else:
            kcin, kctx = cin, ctx
            wp = ops.pack_tdnn_weight(w, ctx)
            in_shape = (B, T, cin)
        bias = 0.1 * torch.randn(cout, device=dev)
        sc, sh = 1 + 0.1 * torch.randn(cout, device=dev), 0.1 * torch.randn(cout, device=dev)
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
        tiles = m_units * -(-cout // 128)
        grid = min(tiles, sms)
        per_cta = -(-tiles // grid)
        words = HEAD + REC * per_cta
        buf = torch.zeros(grid * words, dtype=torch.int64, device=dev)
        lib.xvb_tile_timeline_set(C.c_void_p(buf.data_ptr()), per_cta, int(args.direct_stores))
        for _ in range(3):      # the last launch's stamps are the ones read back
            check(lib.xvb_tdnn_affine_ex(C.byref(a), C.c_void_p(stream)), name)
        torch.cuda.synchronize()
        lib.xvb_tile_timeline_set(None, 0, 0)
        d = buf.cpu().numpy().reshape(grid, words)
        head, rec = d[:, :HEAD], d[:, HEAD:].reshape(grid, per_cta, REC)
        clk_end = np.maximum(head[:, 3], head[:, 5])
        gt_end = np.maximum(head[:, 2], head[:, 4])
        us_per_clk = (gt_end - head[:, 0]) * 1e-3 / np.maximum(clk_end - head[:, 1], 1)    # per CTA
        main, epi, wait, idle_share, phases = [], [], [], [], [[], [], [], []]
        for cta in range(grid):
            r = rec[cta][rec[cta][:, 7] == 1]
            k = us_per_clk[cta]
            main += list((r[:, 3] - r[:, 0]) * k)
            epi += list((r[:, 4] - r[:, 3]) * k)
            wait += list(r[:, 5] * k)
            for ph in range(4):
                phases[ph] += list(r[:, 8 + ph] * k)
            # union of [first operands, MMAs retired) over both warpgroups' tiles
            busy, end = 0, head[cta, 1]
            for s, e in sorted(zip(r[:, 1], r[:, 3])):
                s = max(s, end)
                if e > s:
                    busy += e - s
                    end = e
            idle_share.append(1.0 - busy / max(clk_end[cta] - head[cta, 1], 1))
        print("{:6s} {:9d} {:7.2f} us {:6.2f} us {:6.2f} us {:10.1f} % {:7.1f} us | {:6.2f} us {:7.2f} us {:6.2f} us {:6.2f} us".format(
            name, per_cta, np.median(main), np.median(epi), np.median(wait), 100 * np.median(idle_share),
            np.median((gt_end - head[:, 0]) * 1e-3), *[np.median(ph) for ph in phases]))


if __name__ == "__main__":
    main()
