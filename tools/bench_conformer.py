#!/usr/bin/env python
"""Conformer x-vector throughput: the launcher's model (runTransformerXvector.py:220-286: 6 blocks, attention_dim 256,
4 heads, rot_pos, softmax_plus, transform_out 1536, fc1=False), 80-d features, batches of 128 x 300 frames (one chunk
per utterance) -- a side measurement, not the bench.py line.

    python tools/bench_conformer.py [rounds] [steps_per_round] [--subsampling 4|2] [--profile]

--subsampling 2 measures the same model with input_layer "conv2d2" (SVConv2dSubsampling2, the reference README's
6L-256D-4H-2Sub).  The extractor is the one build_extractor() returns: the native handle, or the Python driver of the
same kernels with XVB_CONFORMER_NATIVE=0.  Alternates it with the torch restatement of tests/conformer_oracle.py on the same GPU (fp32, TF32
off), `steps_per_round` batches per round, and reports the median over rounds of the ms per batch of each, frames/s,
algorithmic TFLOP/s (2 x the MACs counted from the shapes), the native path's launches per batch, the largest relative
difference between the two paths' embeddings, and the card's name and power limit, read in the same run.  Prints one
JSON line.  --profile prints a torch.profiler kernel table of the native path instead."""
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
from asv_subtools_b200.model.transformer_xvector import TransformerXvector  # noqa: E402
import conformer_oracle as co  # noqa: E402
import conformer_2sub_oracle as c2  # noqa: E402


def macs_per_chunk(T, F, D=256, H=4, units=2048, blocks=6, K=15, out_dim=1536, hidden=128, embd=256, subsampling=4):
    """Multiply-accumulates of one T-frame chunk, from the shapes."""
    T1 = (T - 1) // 2
    if subsampling == 4:
        F1 = (F - 1) // 2
        T2, F2 = (T1 - 1) // 2, (F1 - 1) // 2
    else:
        F1 = F - 2
        T2, F2 = T1 - 2, F1 - 2
    m = T1 * F1 * D * 9 + T2 * F2 * D * D * 9 + T2 * F2 * D * D
    per_block = T2 * (2 * 2 * D * units + 3 * D * D + D * D + 2 * D * D + D * K + D * D) + 2 * T2 * T2 * D
    m += blocks * per_block
    m += T2 * D * out_dim + 2 * T2 * out_dim * hidden + 2 * out_dim * embd
    return m


def main():
    argv = sys.argv[1:]
    sub = 4
    if "--subsampling" in argv:
        i = argv.index("--subsampling")
        sub = int(argv[i + 1])
        del argv[i:i + 2]
    if sub not in (4, 2):
        raise SystemExit("--subsampling must be 4 or 2")
    args = [a for a in argv if not a.startswith("--")]
    profile = "--profile" in argv
    B, T, F = 128, 300, 80
    rounds = int(args[0]) if len(args) > 0 else 5
    steps = int(args[1]) if len(args) > 1 else 10
    if not torch.cuda.is_available():
        raise SystemExit("bench_conformer.py needs a GPU")
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    kwargs = co.LAUNCHER if sub == 4 else c2.LAUNCHER_2SUB
    keys = np.load(os.path.join(ROOT, "tests", "golden", "conformer.npz" if sub == 4 else "conformer_2sub.npz"))[
        "keys_launcher" if sub == 4 else "keys_launcher2"]
    sd = co.seeded_state_dict(keys, 401)
    m = TransformerXvector(F, 10, training=False, extracted_embedding="near", **kwargs)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    ex = m.extractor()
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    cfg = co.config(kwargs)
    forward = co.chunk_forward if sub == 4 else c2.chunk_forward
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]

    def oracle(x):
        return forward(sd_gpu, x, cfg, "near")

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
            print(p.key_averages().table(sort_by="cuda_time_total", row_limit=25))
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
    ms = {k: statistics.median(v) for k, v in times.items()}
    macs = macs_per_chunk(T, F, subsampling=sub)
    print(json.dumps({
        "model": "Conformer launcher default (6 blocks, d 256, 4 heads, rot_pos, softmax_plus), F=80, {}x subsampling"
                 .format(sub), "extractor": type(ex).__name__, "batch": B,
        "frames": T, "rounds": rounds, "steps_per_round": steps,
        "ms_per_batch": round(ms["native"], 3), "frames_per_s": round(B * T / ms["native"] * 1e3),
        "macs_per_chunk": macs, "tflops_algorithmic": round(2 * macs * B / ms["native"] * 1e-9, 2),
        "launches_per_batch": ex.last_launches,
        "oracle_fp32_ms_per_batch": round(ms["oracle_fp32"], 3),
        "oracle_over_native": round(ms["oracle_fp32"] / ms["native"], 3),
        "rounds_ms": {k: [round(v, 3) for v in vs] for k, vs in times.items()},
        "embedding_rel_diff_vs_oracle": diff,
        "gpu": smi[0] if smi else "unknown"}))


if __name__ == "__main__":
    main()
