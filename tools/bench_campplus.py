#!/usr/bin/env python
"""CAM++ x-vector throughput: the CamPPConfig default model (FCM head, D-TDNN blocks of 12 / 24 / 16 layers, growth 32,
bn_size 4, embd 512), 80-d features, batches of 128 x 300 frames (one chunk per utterance) -- a side measurement, not
the bench.py line.

    python tools/bench_campplus.py [rounds] [steps_per_round] [--profile]

Alternates the native extractor with the torch restatement of tests/campplus_oracle.py on the same GPU (fp32, TF32 off),
`steps_per_round` batches per round, and reports the median over rounds of the ms per batch of each, frames/s,
algorithmic TFLOP/s (2 x the MACs counted from the shapes), the native path's launches per batch, the largest relative
difference between the two paths' embeddings, and the card's name and power limit, read in the same run.  Prints one
JSON line.

It also times the native handle (NativeCamPPExtractor, the launch sequence in C++) against the Python driver of the same
kernels (CamPPExtractor, one ctypes call per launch) in the same run, alternating them, at 128 x 300 and at 8 x 300
frames, where the per-launch host cost weighs most: ms per batch (median over rounds), frames/s, launches per batch,
and whether the two paths' embeddings are torch.equal.  --profile prints a torch.profiler kernel table of the native path and the share of its GPU time spent in
the BN1 -> ReLU pre-activation kernel (bn_relu_planes_kernel)."""
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from asv_subtools_b200.model.campplus_xvector import (BLOCKS, CamPPExtractor, CamPPXvector,  # noqa: E402
                                                      NativeCamPPExtractor)
import campplus_oracle as co  # noqa: E402


def macs_per_chunk(T, F, m=32, init=128, growth=32, bn_size=4, embd=512):
    """Multiply-accumulates of one T-frame chunk, from the shapes (convolutions, dense layers, masks, transits)."""
    macs, f = T * F * m * 9, F
    for stride in (2, 1, 2, 1):                      # the four BasicResBlocks
        f = (f + 1) // 2 if stride == 2 else f
        macs += T * f * m * m * 9 * 2 + (T * f * m * m if stride == 2 else 0)
    f = (f + 1) // 2
    macs += T * f * m * m * 9                         # conv2
    T2 = (T + 1) // 2
    macs += T2 * m * f * 5 * init                     # tdnn
    bn, c = bn_size * growth, init
    nseg = (T2 + 99) // 100
    for layers, _ in BLOCKS:
        for _ in range(layers):
            macs += T2 * (c * bn + bn * growth * 3) + nseg * (bn * bn // 2 + bn // 2 * growth)
            c += growth
        macs += T2 * c * (c // 2)                     # transit
        c //= 2
    return macs + 2 * c * embd


def handle_vs_driver(m, F, rounds, steps):
    """Native handle against the Python driver, alternating, at 128 x 300 and 8 x 300 frames."""
    dev = torch.device("cuda")
    paths = {"native_handle": NativeCamPPExtractor(m, dev), "python_driver": CamPPExtractor(m, dev)}
    out = {}
    for B, T in ((128, 300), (8, 300)):
        xs = [co.utterances(B, T, F, 950 + i).cuda() for i in range(4)]
        for ex in paths.values():
            for i in range(3):
                ex.extract(xs[i % 4])
        torch.cuda.synchronize()
        equal = all(torch.equal(paths["native_handle"].extract(x), paths["python_driver"].extract(x)) for x in xs)
        times = {k: [] for k in paths}
        for _ in range(rounds):
            for name, ex in paths.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    ex.extract(xs[i % 4])
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / steps)
        r = {"torch_equal": equal}
        for name, ex in paths.items():
            ms = statistics.median(times[name])
            r[name] = {"ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / ms * 1e3), "launches": ex.last_launches,
                       "rounds_ms": [round(v, 3) for v in times[name]]}
        out["{}x{}".format(B, T)] = r
    paths["native_handle"].close()
    return out


def main():
    args = [a for a in sys.argv[1:] if not a.startswith("--")]
    profile = "--profile" in sys.argv
    B, T, F = 128, 300, 80
    rounds = int(args[0]) if len(args) > 0 else 5
    steps = int(args[1]) if len(args) > 1 else 10
    if not torch.cuda.is_available():
        raise SystemExit("bench_campplus.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    keys = np.load(os.path.join(ROOT, "tests", "golden", "campplus.npz"))["keys_default"]
    sd = co.seeded_state_dict(keys, 401)
    m = CamPPXvector(F, 10)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    ex = m.extractor()
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    xs = [co.utterances(B, T, F, 900 + i).cuda() for i in range(4)]

    def oracle(x):
        return co.forward(sd_gpu, x)

    with torch.no_grad():
        for i in range(3):
            ex.extract(xs[i % 4])
            oracle(xs[i % 4])
        torch.cuda.synchronize()
        diff = max(float((ex.extract(x) - oracle(x)).abs().max() / oracle(x).abs().max()) for x in xs)
        if profile:
            from torch.profiler import ProfilerActivity, profile as prof
            with prof(activities=[ProfilerActivity.CUDA]) as p:
                for i in range(steps):
                    ex.extract(xs[i % 4])
                torch.cuda.synchronize()
            avgs = p.key_averages()
            print(avgs.table(sort_by="cuda_time_total", row_limit=25))
            dev_time = lambda e: getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)  # noqa: E731
            total = sum(dev_time(e) for e in avgs if "kernel" in e.key.lower() or "xvb" in e.key or "_kernel" in e.key)
            pre = sum(dev_time(e) for e in avgs if "bn_relu_planes" in e.key)
            print(json.dumps({"bn_relu_planes_share_of_kernel_time": round(pre / total, 4) if total else None,
                              "bn_relu_planes_us_per_batch": round(pre / steps, 1), "gpu": smi[0] if smi else "unknown"}))
            return
        times = {"native": [], "oracle_fp32": []}
        for _ in range(rounds):
            for name, fn in (("native", ex.extract), ("oracle_fp32", oracle)):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(steps):
                    fn(xs[i % 4])
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / steps)
        hvd = handle_vs_driver(m, F, rounds, steps)
    ms = {k: statistics.median(v) for k, v in times.items()}
    macs = macs_per_chunk(T, F)
    print(json.dumps({
        "model": "CAM++ CamPPConfig default (FCM 32ch, D-TDNN 12/24/16, growth 32, bn_size 4, embd 512), F=80", "batch": B,
        "frames": T, "rounds": rounds, "steps_per_round": steps,
        "ms_per_batch": round(ms["native"], 3), "frames_per_s": round(B * T / ms["native"] * 1e3),
        "macs_per_chunk": macs, "tflops_algorithmic": round(2 * macs * B / ms["native"] * 1e-9, 2),
        "launches_per_batch": ex.last_launches,
        "oracle_fp32_ms_per_batch": round(ms["oracle_fp32"], 3),
        "oracle_over_native": round(ms["oracle_fp32"] / ms["native"], 3),
        "rounds_ms": {k: [round(v, 3) for v in vs] for k, vs in times.items()},
        "embedding_rel_diff_vs_oracle": diff,
        "native_handle_vs_python_driver": hvd,
        "gpu": smi[0] if smi else "unknown"}))


if __name__ == "__main__":
    main()
