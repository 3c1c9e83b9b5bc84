#!/usr/bin/env python
"""Throughput of an x-vector extractor on a corpus of utterances of different lengths -- a side measurement, not the
bench.py line.

    python tools/bench_mixed_lengths.py [rounds] [--model xvector|resnet|multihead|xivector|xi|ftdnn|campplus|conformer]
                                        [--utts N] [--min-frames A] [--max-frames B] [--batch N] [--dim F]

The corpus is N utterances (default 4000) with frame counts drawn uniformly from [A, B] (default 200 .. 2000) by
numpy.random.RandomState(2026), run through one handle under two batch policies.  --model xvector (the default): an
Xvector(F, far) handle (default F = 23, batch 256).  --model resnet: the online launcher's SE ResNet34 of
tools/bench_resnet.py (post-activation blocks with SE, fc1=False, position near) on 80-d features (--dim is ignored),
batch 128 by default, as bench_resnet.py times it.  --model multihead / xivector / ftdnn: the Python launch sequences of
the golden configurations at 40-d features (--dim is ignored), position far -- the snowdar x-vector with shared-weight
four-head attention pooling (tests/golden/make_golden_snowdar.py "mha_share"), the xi-vector posterior-distribution
pooling ("xi_dist") and the factored F-TDNN (make_golden_ftdnn.py); batch 256, 256 and 128 by default.  --model
campplus: the native CAM++ handle with egrecho's default CamPPConfig (embd_dim 512, init_channels 128, growth_rate 32,
bn_size 4) on 80-d features (--dim is ignored), batch 128 by default, as tools/bench_campplus.py times it; every
utterance of the default corpus is one chunk of its own length under CAM++'s 4000-frame chunk rule.  --model conformer:
the native Conformer handle with the launcher's model as tools/bench_conformer.py builds it (6 blocks, attention_dim 256,
rot_pos, softmax_plus, 4x subsampling) on 80-d features (--dim is ignored), batch 128 by default; every utterance is cut
by the 300-frame chunk rule (chunk_plan) first, and both policies batch the chunks.  Frames/s still counts the corpus
frames.  --model xi: the xi-vector of pytorch/launcher/runSnowdar_Xivector.py (pooling xi-postdist-softplus2, 1500
nodes, hidden_size 256, position far) at 40-d features (--dim is ignored), batch 256 by default, on the native TDNN
handle (AttentionPoolingExtractor.native()); both policies also run on AttentionPoolingExtractor itself, the same
batches, reported as equal_length_python and masked_python.

  * equal_length: today's buckets of xvb-extract / pipeline/extract_embeddings.py without --mixed-lengths -- batches of
    up to `batch` utterances of exactly the same frame count, one xvb_<handle>_extract call each;
  * masked: --mixed-lengths' rule (plan_mixed_batches: ascending length, up to `batch` per batch, padding at most 1/8),
    one xvb_<handle>_extract_lengths call each.

Features come from one resident random buffer (no host copies in the timed region).  Each round times the whole corpus
under each policy with CUDA events, the policies alternating; every launch plan is built in an untimed warm-up pass
first.  Reports per policy the median frames/s over rounds (real frames only: padding does not count), the batch
count and the padded share of the frames computed, with the card's name and power limit read in the same run.
Prints one JSON line."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from asv_subtools_b200.model.xvector import Xvector  # noqa: E402
from asv_subtools_b200.pipeline.extract_embeddings import plan_mixed_batches  # noqa: E402
from oracle import nnet as onn  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import resnet_oracle as ro  # noqa: E402


# the golden configurations of tests/golden/make_golden_snowdar.py that --model multihead / xivector run
SNOWDAR = {"multihead": ("multi-head", {"num_head": 4}, 313),
           "xivector": ("xi-postdist-softplus2", {"hidden_size": 64, "num_nodes": 200}, 320),
           "xi": ("xi-postdist-softplus2", {"num_nodes": 1500, "num_head": 16, "share": True, "affine_layers": 1,
                                            "hidden_size": 256, "context": [0], "temperature": False, "fixed": True}, 321)}


def equal_length_batches(lengths, batch):
    """Exact-length buckets in batches of up to `batch` (the default mode of both CLIs)."""
    buckets = {}
    for i, n in enumerate(lengths):
        buckets.setdefault(n, []).append(i)
    return [idx[k:k + batch] for n in sorted(buckets) for idx in [buckets[n]] for k in range(0, len(idx), batch)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("rounds", nargs="?", type=int, default=5)
    ap.add_argument("--utts", type=int, default=4000)
    ap.add_argument("--min-frames", type=int, default=200)
    ap.add_argument("--max-frames", type=int, default=2000)
    ap.add_argument("--batch", type=int, default=None,
                    help="default 256 (xvector, multihead, xivector, xi) or 128 (resnet, ftdnn, campplus, conformer)")
    ap.add_argument("--dim", type=int, default=23)
    ap.add_argument("--model", choices=["xvector", "resnet", "multihead", "xivector", "xi", "ftdnn", "campplus", "conformer"],
                    default="xvector")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixed_lengths.py needs a GPU")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                          str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    lengths = [int(v) for v in np.random.RandomState(2026).randint(args.min_frames, args.max_frames + 1, args.utts)]
    if args.model == "resnet":
        from asv_subtools_b200.model.resnet_xvector import ResNetXvector
        F = 80
        args.batch = args.batch or 128
        m = ResNetXvector(F, 10, training=False, extracted_embedding="near", **ro.ONLINE)
        m.load_state_dict(onn.make_state_dict(ro.resnet_spec(F, ro.ONLINE), 301), strict=True)
        workload = "online SE ResNet34 (80-d, near)"
    elif args.model in ("multihead", "xivector", "xi"):
        from asv_subtools_b200.model.snowdar_xvector import Xvector as SnowdarXvector
        F = 40
        args.batch = args.batch or 256
        pooling, pp, seed = SNOWDAR[args.model]
        m = SnowdarXvector(F, 10, training=False, extracted_embedding="far", pooling=pooling, pooling_params=pp)
        m.load_state_dict(onn.make_state_dict(onn.snowdar_xvector_spec(F, pooling=pooling, pooling_params=pp), seed),
                          strict=True)
        workload = "snowdar Xvector(40) far, pooling {} {}".format(pooling, pp)
        if args.model == "xi":
            workload = "launcher xi-vector (runSnowdar_Xivector.py, 40-d, far) on the native handle"
    elif args.model == "ftdnn":
        from asv_subtools_b200.model.factored_xvector import Xvector as FactoredXvector
        F = 40
        args.batch = args.batch or 128
        m = FactoredXvector(F, 10, training=False, extracted_embedding="far")
        m.load_state_dict(onn.make_state_dict(onn.factored_xvector_spec(F), 401), strict=True)
        workload = "factored F-TDNN Xvector(40) far"
    elif args.model == "campplus":
        import campplus_oracle as co
        from asv_subtools_b200.model.campplus_xvector import CamPPXvector
        F = 80
        args.batch = args.batch or 128
        if args.max_frames > 4000:
            raise SystemExit("--model campplus: every utterance must be one chunk, --max-frames <= 4000")
        keys = np.load(os.path.join(ROOT, "tests", "golden", "campplus.npz"))["keys_default"]
        m = CamPPXvector(F, 10)
        m.load_state_dict(co.seeded_state_dict(keys, 401), strict=True)
        workload = "CAM++ CamPPConfig defaults (80-d, embd_dim 512)"
    elif args.model == "conformer":
        import conformer_oracle as cfo
        from asv_subtools_b200.model.transformer_xvector import TransformerXvector
        F = 80
        args.batch = args.batch or 128
        keys = np.load(os.path.join(ROOT, "tests", "golden", "conformer.npz"))["keys_launcher"]
        m = TransformerXvector(F, 10, training=False, extracted_embedding="near", **cfo.LAUNCHER)
        m.load_state_dict(cfo.seeded_state_dict(keys, 401), strict=True)
        workload = "launcher Conformer (6 blocks, d 256, rot_pos, softmax_plus, 80-d, near), 300-frame chunks"
    else:
        F = args.dim
        args.batch = args.batch or 256
        m = Xvector(F, 10, training=False, extracted_embedding="far")
        m.load_state_dict(onn.make_state_dict(onn.xvector_spec(F), 7), strict=True)
        workload = "Xvector({}) far".format(F)
    m.cuda().eval()
    ex = m.extractor()
    extractors = {"": ex}
    if args.model == "xi":   # the native handle, and the Python launch sequence it was built from
        extractors = {"": ex.native(), "_python": ex}
    # the items both policies batch: the chunks of the model's own chunk rule where it cuts utterances, else the utterances
    chunks = [n for u in lengths for n in m.chunk_sizes(u)] if args.model == "conformer" else lengths
    base = torch.randn(args.batch * max(chunks) * F, device="cuda")

    policies = {}
    for suffix, e in extractors.items():
        for name, plan in (("equal_length", equal_length_batches(chunks, args.batch)),
                           ("masked", plan_mixed_batches(chunks, args.batch))):
            jobs = []
            for idx in plan:
                lens = [chunks[i] for i in idx]
                B, T = len(lens), max(lens)
                jobs.append((B, T, np.asarray(lens, np.int32) if name == "masked" else None))
            computed = sum(B * T for B, T, _ in jobs)
            policies[name + suffix] = {"jobs": jobs, "ex": e, "batches": len(jobs),
                                       "padded_share": 1.0 - sum(chunks) / computed, "fps": []}

    def run(p):
        ex = p["ex"]
        for B, T, lens in p["jobs"]:
            x = base[:B * T * F].view(B, T, F)
            ex.extract(x) if lens is None else ex.extract(x, lens)

    with torch.no_grad():
        for p in policies.values():          # warm-up: every plan built, every buffer grown
            run(p)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for p in policies.values():
                start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                run(p)
                stop.record()
                stop.synchronize()
                p["fps"].append(sum(lengths) / (start.elapsed_time(stop) / 1e3))
    out = {"workload": "{}, {} utterances uniform over {}..{} frames (RandomState(2026)), batch {}".format(
               workload, args.utts, args.min_frames, args.max_frames, args.batch),
           "frames": sum(lengths), "items": len(chunks), "card": smi, "rounds": args.rounds}
    for name, p in policies.items():
        out[name] = {"frames_per_s": statistics.median(p["fps"]), "frames_per_s_min": min(p["fps"]),
                     "frames_per_s_max": max(p["fps"]), "batches": p["batches"], "padded_share": round(p["padded_share"], 5)}
    out["speedup"] = out["masked"]["frames_per_s"] / out["equal_length"]["frames_per_s"]
    if "masked_python" in out:   # the native handle against the Python launch sequence, per policy
        out["native_vs_python"] = {k: out[k]["frames_per_s"] / out[k + "_python"]["frames_per_s"]
                                   for k in ("equal_length", "masked")}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
