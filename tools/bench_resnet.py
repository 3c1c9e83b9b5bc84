#!/usr/bin/env python
"""ResNet34 x-vector throughput: the online launcher's model (runResnetXvector_online.py:221-275: post-activation blocks
with SE, fc1=False), 80-d features, batches of 128 x 200 frames -- a side measurement, not the bench.py line.

    python tools/bench_resnet.py [steps]

Prints one JSON line: frames/s, ms per batch, algorithmic TFLOP/s (2 x the convolution MACs counted from the shapes
below, head conv and downsamples included; SE and fc2 are per utterance and reported apart) and the card's name and
power limit, read in the same run."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from asv_subtools_b200.model.resnet_xvector import ResNetXvector  # noqa: E402
from oracle import nnet as onn  # noqa: E402
import resnet_oracle as ro  # noqa: E402


def conv_macs(F, T, layers=(3, 4, 6, 3), planes=(32, 64, 128, 256)):
    """Multiply-accumulates of the convolutions of one utterance (F x T input): head 1 -> planes[0] 3x3, then per block
    two 3x3 convs, plus the 1x1 downsample of the first block of layers 2-4, at ceil(F/s) x ceil(T/s) outputs."""
    macs = F * T * planes[0] * 9
    cin = planes[0]
    for li, (n, p) in enumerate(zip(layers, planes)):
        if li:
            F, T = (F + 1) // 2, (T + 1) // 2
            macs += F * T * cin * p                       # downsample
        macs += F * T * (cin * p * 9 + (2 * n - 1) * p * p * 9)
        cin = p
    return macs


def utt_macs(F, planes=(32, 64, 128, 256), layers=(3, 4, 6, 3), se_ratio=4):
    """Per-utterance MACs after the convolutions: the SE blocks' two linears and fc2 on the pooled statistics."""
    se = sum(n * 2 * p * (p // se_ratio) for n, p in zip(layers, planes))
    return se + 2 * ((F + 7) // 8) * planes[3] * planes[3]


def main():
    B, T, F = 128, 200, 80
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    m = ResNetXvector(F, 10, training=False, extracted_embedding="near", **ro.ONLINE)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(F, ro.ONLINE), 301), strict=True)
    m.cuda().eval()
    ex = m.extractor()
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]
    with torch.no_grad():
        for i in range(5):
            ex.extract(xs[i % 4])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(steps):
            ex.extract(xs[i % 4])
        e1.record()
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    macs = conv_macs(F, T)
    print(json.dumps({
        "model": "ResNet34 online launcher (SE, post-activation), F=80", "batch": B, "frames": T, "steps": steps,
        "ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / ms * 1e3),
        "conv_macs_per_frame": macs / T, "tflops_algorithmic": round(2 * macs * B / ms * 1e-9, 2),
        "per_utterance_macs_se_fc2": utt_macs(F),
        "gpu": smi[0] if smi else "unknown"}))


if __name__ == "__main__":
    main()
