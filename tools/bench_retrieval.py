"""Speaker retrieval at the size of the problem it exists for: M enrolled speakers x N = 10^6 test vectors, D = 256,
k = 10, seeded synthetic length-normalised vectors.  For each M in {1 000, 10 000} and each slab width it times, with
CUDA events (median of --reps after one warm-up):
  retrieve : xvb_retrieve_topk (slab GEMMs + streaming top-k merges, one final NaN check)
  gemm     : xvb_matmul_nt alone over the same slabs into the same buffer -- the GEMM floor of this design
  torch    : xvb_cosine_matrix slab by slab, each slab ranked by torch.topk and merged with torch.topk -- the
             baseline on the same card
and reports algorithmic TFLOP/s (2 M N D over the time), the slab bytes (the matrix written and read once, 8 M N),
whether retrieve and torch agree on every score, and the card name and power limit read in the same run.
Prints one JSON line.  Needs a GPU:  python tools/bench_retrieval.py [--reps 5] [--slabs 16384,65536,262144]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200._lib import check, lib  # noqa: E402


def _p(t):
    return C.c_void_p(t.data_ptr())


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return sorted(times)[len(times) // 2]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def run_case(m, n, d, k, slabs, reps):
    g = torch.Generator(device="cuda").manual_seed(m)
    a = torch.nn.functional.normalize(torch.randn(m, d, device="cuda", generator=g), dim=1).contiguous()
    b = torch.nn.functional.normalize(torch.randn(n, d, device="cuda", generator=g), dim=1).contiguous()
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    out = []
    for slab_cols in slabs:
        slab = torch.empty(lib.xvb_retrieve_topk_slab_bytes(m, slab_cols) // 4, device="cuda")
        sc = torch.empty(m, k, device="cuda")
        ix = torch.empty(m, k, dtype=torch.int64, device="cuda")

        def retrieve():
            check(lib.xvb_retrieve_topk(_p(a), m, _p(b), n, d, None, None, k, _p(slab), slab_cols, _p(sc), _p(ix), stream),
                  "xvb_retrieve_topk")

        def gemm():
            for c0 in range(0, n, slab_cols):
                cols = min(slab_cols, n - c0)
                check(lib.xvb_matmul_nt(_p(a), m, _p(b[c0:]), cols, d, None, None, _p(slab), slab_cols, stream), "xvb_matmul_nt")

        best = {}

        def baseline():
            bs = bi = None
            for c0 in range(0, n, slab_cols):
                cols = min(slab_cols, n - c0)
                s = slab[:m * slab_cols].view(m, slab_cols)
                check(lib.xvb_cosine_matrix(_p(a), m, _p(b[c0:]), cols, d, _p(s), slab_cols, stream), "xvb_cosine_matrix")
                ts, ti = torch.topk(s[:, :cols], k, dim=1)
                if bs is None:
                    bs, bi = ts, ti + c0
                else:
                    bs, o = torch.topk(torch.cat([bs, ts], 1), k, dim=1)
                    bi = torch.gather(torch.cat([bi, ti + c0], 1), 1, o)
            best["s"], best["i"] = bs, bi

        t_ret = _time(retrieve, reps)
        t_gemm = _time(gemm, reps)
        t_torch = _time(baseline, reps)
        flops = 2.0 * m * n * d
        out.append({"M": m, "N": n, "D": d, "k": k, "slab_cols": slab_cols, "retrieve_ms": round(t_ret, 3),
                    "gemm_ms": round(t_gemm, 3), "torch_topk_ms": round(t_torch, 3),
                    "retrieve_tflops": round(flops / t_ret / 1e9, 1), "gemm_tflops": round(flops / t_gemm / 1e9, 1),
                    "slab_bytes_per_call": m * slab_cols * 4, "slab_traffic_gb": round(8.0 * m * n / 1e9, 2),
                    "scores_equal_torch": bool(torch.equal(sc, best["s"]))})
        del slab
        torch.cuda.empty_cache()
    return out


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--slabs", default="16384,65536,262144")
    ap.add_argument("--speakers", default="1000,10000")
    ap.add_argument("--tests", type=int, default=1000000)
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        sys.exit("bench_retrieval needs a GPU")
    name, power = card()
    slabs = [int(s) for s in args.slabs.split(",")]
    cases = []
    for m in (int(x) for x in args.speakers.split(",")):
        cases += run_case(m, args.tests, 256, 10, slabs, args.reps)
    print(json.dumps({"bench": "retrieval", "gpu": name, "power_limit": power, "cases": cases}))


if __name__ == "__main__":
    main()
