#!/usr/bin/env python
"""ResNet34 x-vector throughput: the online launcher's model (runResnetXvector_online.py:221-275: post-activation blocks
with SE, fc1=False), 80-d features, batches of 128 x 200 frames -- a side measurement, not the bench.py line.

    python tools/bench_resnet.py [steps]

Times, alternating in one process over the same inputs: the op-by-op Python driver (ResNetExtractor,
XVB_RESNET_NATIVE=0), the native handle's extract, and its extract_shard over a device-resident shard of 32 batches with
one lane (XVB_LANES=0) and with two.  Prints one JSON line: ms per batch (median of the rounds), frames/s and kernel
launches per batch for each path, algorithmic TFLOP/s (2 x the convolution MACs counted from the shapes below, head conv
and downsamples included; SE and fc2 are per utterance and reported apart), the native workspace in bytes computed
from the shapes, whether native and Python outputs of the timed inputs are bit-identical, and the card's name and power
limit, read in the same run."""
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from asv_subtools_b200.model.resnet_xvector import NativeResNetExtractor, ResNetExtractor, ResNetXvector  # noqa: E402
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


def workspace_bytes(B, T, F, layers=(3, 4, 6, 3), planes=(32, 64, 128, 256), se_ratio=4, emb=256):
    """Bytes of one xvb_resnet workspace at (B, T, F), from the shapes as resnet_extractor.cu sizes it: seven bf16 plane
    pairs of the largest (B, T', F', C) tensor, the last layer's fp32 output, the pooled statistics (planes + fp32), the SE
    mean / hidden / gate and the segment buffers."""
    t, f, big = T, F, B * T * F * planes[0]
    for li, (n, p) in enumerate(zip(layers, planes)):
        if li:
            t, f = (t - 1) // 2 + 1, (f - 1) // 2 + 1
        big = max(big, B * t * f * p)
    pooled = 2 * f * planes[3]
    hidden = max((p // se_ratio + 3) // 4 * 4 for p in planes)
    out = (emb + 7) // 8 * 8
    return (7 * 2 * 2 * big + 4 * B * t * f * planes[3] + B * pooled * (2 * 2 + 4) +
            4 * B * (max(256, max(planes)) + hidden + max(planes)) + 2 * 2 * B * 8 + 4 * B * out)


def main():
    B, T, F = 128, 200, 80
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    rounds, shard_batches = 5, 32
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    m = ResNetXvector(F, 10, training=False, extracted_embedding="near", **ro.ONLINE)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(F, ro.ONLINE), 301), strict=True)
    m.cuda().eval()
    twin, native = ResNetExtractor(m, torch.device("cuda")), NativeResNetExtractor(m, torch.device("cuda"))
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]
    shard = torch.randn(shard_batches * B, T, F, device="cuda")
    shard_out = torch.empty(shard_batches * B, native.embed_dim, device="cuda")
    launches = {}

    def batches(ex):
        def run(i):
            ex.extract(xs[i % 4])
        return run, steps, steps

    def sharded(lanes):
        def run(i):
            os.environ["XVB_LANES"] = lanes
            native.extract_shard(shard, batch=B, out=shard_out)
        return run, 1, shard_batches

    paths = {"python": batches(twin), "native": batches(native), "shard_1lane": sharded("0"), "shard_2lanes": sharded("1")}
    times = {k: [] for k in paths}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with torch.no_grad():
        for name, (run, _, _) in paths.items():   # warm-up: workspaces, modules, second lane
            for i in range(3):
                run(i)
            launches[name] = native.last_launches if name != "python" else None
        torch.cuda.synchronize()
        for _ in range(rounds):
            for name, (run, calls, nb) in paths.items():
                e0.record()
                for i in range(calls):
                    run(i)
                e1.record()
                torch.cuda.synchronize()
                times[name].append(e0.elapsed_time(e1) / nb)
        same = all(torch.equal(native.extract(x), twin.extract(x)) for x in xs)
        ref = torch.cat([twin.extract(shard[i:i + B]) for i in range(0, shard.shape[0], B)])
        for lanes in ("0", "1"):
            os.environ["XVB_LANES"] = lanes
            same = same and torch.equal(native.extract_shard(shard, batch=B), ref)
        native.extract(xs[0])
        launches["python"] = native.last_launches   # the same kernels, one launch per C entry point
    os.environ.pop("XVB_LANES", None)
    macs = conv_macs(F, T)
    res = {"model": "ResNet34 online launcher (SE, post-activation), F=80", "batch": B, "frames": T, "steps": steps,
           "rounds": rounds, "shard_batches": shard_batches}
    for name, ts in times.items():
        ms = sorted(ts)[len(ts) // 2]
        res[name] = {"ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / ms * 1e3),
                     "tflops_algorithmic": round(2 * macs * B / ms * 1e-9, 2),
                     "launches_per_batch": launches[name] // (shard_batches if name.startswith("shard") else 1),
                     "ms_per_batch_all_rounds": [round(t, 3) for t in ts]}
    res.update({"bit_identical_native_vs_python": bool(same), "conv_macs_per_frame": macs / T,
                "per_utterance_macs_se_fc2": utt_macs(F), "workspace_bytes_per_lane": workspace_bytes(B, T, F),
                "gpu": smi[0] if smi else "unknown"})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
