#!/usr/bin/env python
"""RepSPK x-vector throughput: the launcher's default model (runRepvggXvector.py:219-262: RepSPK blocks, base width 32,
[2, 4, 14, 1] x [1, 1, 1, 2.5], fc1=False), 80-d features -- a side measurement, not the bench.py line.

    python tools/bench_repvgg.py [rounds] [steps_per_round]

Times, alternating, `steps_per_round` batches per round:
  * at 128 x 200 frames: the native handle (NativeRepVGGExtractor, the default), the Python driver of the same kernels
    (RepVGGExtractor, XVB_REPVGG_NATIVE=0) and the driver with every block given the dense 25-tap list (built as a
    RepVGGExtractor and re-packed inside this script only);
  * at 8 x 200 frames, where launch cost shows: the native handle and the driver.
Reports the median over rounds of the ms per batch of each, frames/s and algorithmic TFLOP/s of the native handle
(2 x the convolution MACs of the 17 kept taps, counted from the shapes; the dense run is rated on the same MAC count, so
the ratio is the time ratio), whether the native and driver embeddings are torch.equal at both sizes, the largest
relative difference between the dense and the 17-tap embeddings, and the card's name and power limit, read in the same
run.  Prints one JSON line."""
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.model.repvgg_xvector import (NativeRepVGGExtractor, RepVGGExtractor, RepVggXvector,  # noqa: E402
                                                    fold_block)
from oracle import nnet as onn  # noqa: E402
import repvgg_oracle as ro  # noqa: E402


def conv_macs(m, F, T, taps_per_block):
    """Multiply-accumulates of the convolutions of one utterance (F x T input): the head (stage0, Cin = 1, dense
    window) and every block at ceil(F/s) x ceil(T/s) outputs with its number of taps."""
    blocks = m.repvgg.blocks()
    head = blocks[0]
    macs = F * T * head.out_channels * head.window ** 2
    for blk, ntaps in zip(blocks[1:], taps_per_block):
        F, T = (F - 1) // blk.stride + 1, (T - 1) // blk.stride + 1
        macs += F * T * blk.in_channels * blk.out_channels * ntaps
    return macs


def timed_rounds(runs, xs, rounds, steps):
    """runs: name -> extractor; every round times each of them in turn.  -> name -> [ms per batch per round]."""
    times = {name: [] for name in runs}
    for _ in range(rounds):
        for name, ex in runs.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for i in range(steps):
                ex.extract(xs[i % len(xs)])
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / steps)
    return times


def main():
    B, T, F, B_SMALL = 128, 200, 80, 8
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    if not torch.cuda.is_available():
        raise SystemExit("bench_repvgg.py needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    m = RepVggXvector(F, 10, training=False, extracted_embedding="near", **ro.LAUNCHER)
    m.load_state_dict(onn.make_state_dict(ro.repvgg_spec(F, ro.LAUNCHER), 401), strict=True)
    m.cuda().eval()
    dev = torch.device("cuda", torch.cuda.current_device())
    native = NativeRepVGGExtractor(m, dev)
    driver = RepVGGExtractor(m, dev)
    dense = RepVGGExtractor(m, dev)             # a third copy, every block re-packed with the dense 25-tap list
    for blk, entry in zip(m.repvgg.blocks()[1:], dense.blocks):
        k = entry["k"]
        entry["taps"] = list(range(k * k))
        entry["w"] = ops.pack_conv2d_weight(fold_block(blk)[0].float().cuda().contiguous(), entry["taps"])
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]
    small = [torch.randn(B_SMALL, T, F, device="cuda") for _ in range(4)]
    with torch.no_grad():
        for ex in (native, driver, dense):
            for i in range(3):
                ex.extract(xs[i % 4])
                ex.extract(small[i % 4])
        torch.cuda.synchronize()
        equal = {n: all(torch.equal(native.extract(x), driver.extract(x)) for x in batch)
                 for n, batch in (("128x200", xs), ("8x200", small))}
        diff = max(float((dense.extract(x) - driver.extract(x)).abs().max() / driver.extract(x).abs().max()) for x in xs)
        native.extract(xs[0])
        launches = native.last_launches
        times = timed_rounds({"native": native, "driver": driver, "dense25": dense}, xs, rounds, steps)
        times_small = timed_rounds({"native": native, "driver": driver}, small, rounds, steps)
    ms = {k: statistics.median(v) for k, v in times.items()}
    ms_small = {k: statistics.median(v) for k, v in times_small.items()}
    macs = conv_macs(m, F, T, [len(b["taps"]) for b in driver.blocks])
    print(json.dumps({
        "model": "RepSPK launcher default (base 32, [2,4,14,1] x [1,1,1,2.5]), F=80", "batch": B, "frames": T,
        "rounds": rounds, "steps_per_round": steps,
        "ms_per_batch": round(ms["native"], 3), "driver_ms_per_batch": round(ms["driver"], 3),
        "frames_per_s": round(B * T / ms["native"] * 1e3),
        "conv_macs_per_frame": macs / T, "tflops_algorithmic": round(2 * macs * B / ms["native"] * 1e-9, 2),
        "native_launches": launches,
        "small_batch": {"batch": B_SMALL, "native_ms_per_batch": round(ms_small["native"], 3),
                        "driver_ms_per_batch": round(ms_small["driver"], 3),
                        "rounds_ms": {k: [round(v, 3) for v in vs] for k, vs in times_small.items()}},
        "native_equals_driver": equal,
        "dense25_ms_per_batch": round(ms["dense25"], 3), "dense25_over_taps17": round(ms["dense25"] / ms["driver"], 3),
        "dense25_conv_macs_per_frame": conv_macs(m, F, T, [25] * len(driver.blocks)) / T,
        "rounds_ms": {k: [round(v, 3) for v in vs] for k, vs in times.items()},
        "embedding_rel_diff_dense_vs_taps17": diff,
        "gpu": smi[0] if smi else "unknown"}))


if __name__ == "__main__":
    main()
