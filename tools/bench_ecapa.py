#!/usr/bin/env python
"""ECAPA-TDNN c1024 throughput (BASELINE configs[2]: 80-d fbank, 300-frame chunks, batch 128) --
a side measurement, not the bench.py contract line.

--channels 512: the C512 model (ecapa_params={"channels": 512}, Res2Net width 64) instead; the default, 1024, keeps the
c1024 line.  XVB_ECAPA_NATIVE=0 / XVB_ECAPA_RES2NET=gemm select the twin / its per-scale GEMMs as for the c1024 model.

--pooling mqmha: the roadmap launcher's model (runEcapaXvector_roadmap.py:220-250: MQMHASP 2 queries x 2 heads, hidden
64, share=False, time attention) next to the attentive-pooling model in the same call, and CUDA-event times of its two
attention GEMMs in the layer kernel's grouped mode against their block-diagonal expansions.

--egrecho [--channels 512|1024]: egrecho's EcapaXvector (EcapaConfig's pooling: one head, one query, hidden 128, time
attention) at 128 x 300 on the native handle in its chained form, on its Python twin and as the torch fp32 restatement
(tests/egrecho_ecapa_oracle.py, TF32 off), with the dense ECAPA_TDNN handle of the same width next to it; the four run in
alternating rounds in one process, and each one's median round is reported.

--lawlict [--channels 512|1024]: the ECAPA_TDNN of pytorch/model/ecapa-tdnn-xvector.py (runEcapaXvector.py's model:
attentive pooling without global context, hidden 128) at 128 x 300 on the native handle, on its Python twin and as the
torch fp32 restatement (tests/lawlict_ecapa_oracle.py, TF32 off), with the dense ECAPA_TDNN handle of the same width next
to it, in alternating rounds as for --egrecho."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN  # noqa: E402
from oracle import nnet as onn  # noqa: E402

CANON = dict(training=False, extracted_embedding="near",
             ecapa_params={"channels": 1024, "embd_dim": 192, "mfa_conv": 1536,
                           "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}},
             fc2_params={"nonlinearity": "", "bn": True, "bn_params": {"momentum": 0.5, "affine": False,
                                                                        "track_running_stats": True}})


def _card():
    import subprocess
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=60).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except OSError:
        return torch.cuda.get_device_name()


def _rate(ex, xs, steps):
    for i in range(3):
        ex.extract(xs[i % len(xs)])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = ex.extract(xs[i % len(xs)])
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def _gemm_ms(fn, reps=20):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main_mqmha(steps):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import ecapa_mqmha_oracle as mo
    from asv_subtools_b200 import ops
    from asv_subtools_b200.model.ecapa_tdnn_xvector import _mqmha_attention
    B, T, F = 128, 300, 80
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]
    base = ECAPA_TDNN(F, 10, **CANON)
    base.load_state_dict(onn.make_state_dict(onn.ecapa_spec(F), 201), strict=True)
    kw = mo.ROADMAP_KW
    mq = ECAPA_TDNN(F, 10, training=False, extracted_embedding="near", **kw)
    mq.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kw), 31), strict=True)
    res = {"card": _card(), "workload": "80-d fbank, 300-frame chunks, batch 128, native extractor"}
    for name, m in (("ecpa-attentive", base), ("mqmha", mq)):
        m.cuda().eval()
        ms, out = _rate(m.extractor(), xs, steps)
        res[name] = {"ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / (ms * 1e-3)), "finite": bool(torch.isfinite(out).all())}
    # the two attention GEMMs of the roadmap model at B x T = 128 x 300
    st = mq.stats
    D = st.in_dim
    x = ops.split_f32(torch.randn(B, T, D, device="cuda"))
    a1 = ops.split_f32(torch.randn(B, T, st.hidden_size * st.num_head * st.num_q, device="cuda"))
    recs = {r[0]: r for r in _mqmha_attention(st)}
    for name, src in (("att_x", x), ("att2", a1)):
        _, w, _, _, _, g = recs[name]
        w = torch.from_numpy(w).cuda()
        cout = w.shape[0]
        y = torch.empty(B, T, cout, device="cuda")
        wg, wd = ops.pack_tdnn_weight(w, [0]), ops.pack_tdnn_weight(ops.block_diagonal(w, g).contiguous(), [0])
        tg = _gemm_ms(lambda: ops.tdnn_affine_ex(src, wg, cout, [0], y_f32=y, groups=g))
        td = _gemm_ms(lambda: ops.tdnn_affine_ex(src, wd, cout, [0], y_f32=y))
        res[name + "_gemm_us"] = {"shape": "{}x{}->{} groups {}".format(B * T, src.channels, cout, g),
                                  "grouped": round(tg * 1e3, 1), "block_diagonal": round(td * 1e3, 1)}
    print(json.dumps(res))


def main_egrecho(steps, channels, rounds=5):
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    import egrecho_ecapa_oracle as eo
    from asv_subtools_b200.model import ecapa_tdnn_xvector as etx
    from asv_subtools_b200.model.egrecho_ecapa_xvector import EcapaXvector
    B, T, F = 128, 300, 80
    dev = torch.device("cuda")
    xs = [torch.randn(B, T, F, device=dev) for _ in range(4)]
    m = EcapaXvector(F, 10, channels=channels)
    keys = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    sd = eo.seeded_state_dict(keys, 41)
    m.load_state_dict(sd, strict=True)
    m.to(dev).eval()
    dense = ECAPA_TDNN(F, 10, **dict(CANON, ecapa_params=dict(CANON["ecapa_params"], channels=channels)))
    dense.load_state_dict(onn.make_state_dict(onn.ecapa_spec(F, channels=channels), 201), strict=True)
    dense.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    class Torch:
        def extract(self, x):
            with torch.no_grad():
                return eo.forward(sd_dev, x, {"inputs_dim": F, "channels": channels})[0]

    runs = {"native": m.extractor(), "twin": etx.EcapaExtractor(m, dev), "torch_fp32": Torch(),
            "ecapa_tdnn_dense_native": dense.extractor()}
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for name, ex in runs.items():
            times[name].append(_rate(ex, xs, steps)[0])
    x = xs[0]
    nat, twin, ref = (runs[k].extract(x) for k in ("native", "twin", "torch_fp32"))
    res = {"card": _card(), "workload": "egrecho EcapaXvector C{}, 80-d fbank, 300-frame chunks, batch 128".format(channels),
           "native_equals_twin": bool(torch.equal(nat, twin)),
           "native_vs_torch_rel": float((nat - ref).abs().max() / ref.abs().max()),
           "launches": runs["native"].last_launches}
    for name, v in times.items():
        ms = sorted(v)[len(v) // 2]
        res[name] = {"ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / (ms * 1e-3)),
                     "rounds_ms": [round(t, 3) for t in v]}
    print(json.dumps(res))


def main_lawlict(steps, channels, rounds=5):
    import importlib.util
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(root, "tests"))
    import lawlict_ecapa_oracle as lo
    from asv_subtools_b200.model import ecapa_tdnn_xvector as etx
    spec = importlib.util.spec_from_file_location("lawlict_ecapa_blueprint",
                                                  os.path.join(root, "asv_subtools_b200", "model", "ecapa-tdnn-xvector.py"))
    bp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bp)
    B, T, F = 128, 300, 80
    dev = torch.device("cuda")
    xs = [torch.randn(B, T, F, device=dev) for _ in range(4)]
    kw = lo.kwargs(channels=channels)
    m = bp.ECAPA_TDNN(F, 1211, **kw)
    sd = onn.make_state_dict(lo.spec(F, kw), 41)
    m.load_state_dict(sd, strict=True)
    m.to(dev).eval()
    dense = ECAPA_TDNN(F, 10, **dict(CANON, ecapa_params=dict(CANON["ecapa_params"], channels=channels)))
    dense.load_state_dict(onn.make_state_dict(onn.ecapa_spec(F, channels=channels), 201), strict=True)
    dense.to(dev).eval()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False

    class Torch:
        def extract(self, x):
            with torch.no_grad():
                return lo.forward(sd_dev, x.transpose(1, 2), kw)[:, :, 0]

    runs = {"native": m.extractor(), "twin": etx.EcapaExtractor(m, dev), "torch_fp32": Torch(),
            "ecapa_tdnn_dense_native": dense.extractor()}
    times = {k: [] for k in runs}
    for _ in range(rounds):
        for name, ex in runs.items():
            times[name].append(_rate(ex, xs, steps)[0])
    x = xs[0]
    nat, twin, ref = (runs[k].extract(x) for k in ("native", "twin", "torch_fp32"))
    runs["ecapa_tdnn_dense_native"].extract(x)
    res = {"card": _card(), "workload": "ecapa-tdnn-xvector.py ECAPA_TDNN C{}, 80-d fbank, 300-frame chunks, batch 128".format(
               channels),
           "native_equals_twin": bool(torch.equal(nat, twin)),
           "native_vs_torch_rel": float((nat - ref).abs().max() / ref.abs().max()),
           "launches": runs["native"].last_launches, "dense_launches": runs["ecapa_tdnn_dense_native"].last_launches}
    for name, v in times.items():
        ms = sorted(v)[len(v) // 2]
        res[name] = {"ms_per_batch": round(ms, 3), "frames_per_s": round(B * T / (ms * 1e-3)),
                     "rounds_ms": [round(t, 3) for t in v]}
    print(json.dumps(res))


def macs_per_frame(C, F=80, D=1536, H=128):
    """Contraction MACs per frame from the shapes: layer1 (5 taps), per block bn1 + 7 Res2Net steps (3 taps, width C/8)
    + bn2, mfa, the two attention convs (the per-utterance SE and segment layers are left out)."""
    W = C // 8
    return 5 * F * C + 3 * (2 * C * C + 7 * 3 * W * W) + 3 * C * D + 2 * D * H


def main():
    B, T, F = 128, 300, 80
    steps = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 10
    if "--pooling" in sys.argv and sys.argv[sys.argv.index("--pooling") + 1] == "mqmha":
        return main_mqmha(steps)
    channels = int(sys.argv[sys.argv.index("--channels") + 1]) if "--channels" in sys.argv else 1024
    if channels not in (512, 1024):
        raise SystemExit("--channels takes 512 or 1024")
    if "--egrecho" in sys.argv:
        return main_egrecho(steps, channels)
    if "--lawlict" in sys.argv:
        return main_lawlict(steps, channels)
    kw = dict(CANON, ecapa_params=dict(CANON["ecapa_params"], channels=channels))
    m = ECAPA_TDNN(F, 10, **kw)
    m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(F, channels=channels), 201), strict=True)
    m.cuda().eval()
    if "--profile" in sys.argv:
        os.environ["XVB_ECAPA_NATIVE"] = "0"   # per-op CUDA events live in the op-by-op Python twin
    ex = m.extractor()
    xs = [torch.randn(B, T, F, device="cuda") for _ in range(4)]
    for i in range(3):
        ex.extract(xs[i % 4])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        out = ex.extract(xs[i % 4])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    flop = (25701908 if channels == 1024 else 2 * macs_per_frame(channels)) * B * T  # c1024: SURVEY 8(d)
    if "--profile" in sys.argv:
        import collections
        from asv_subtools_b200.model import ecapa_tdnn_xvector as mod
        agg = collections.OrderedDict()
        for rep in range(5):
            mod._PROFILE = []
            ex.extract(xs[rep % 4])
            torch.cuda.synchronize()
            evs = mod._PROFILE
            for (l0, e0_), (l1, e1_) in zip(evs[:-1], evs[1:]):
                agg.setdefault(l1, []).append(e0_.elapsed_time(e1_))
        mod._PROFILE = None
        tot = 0.0
        for k, v in agg.items():
            per_call = sorted(v)[len(v) // 2]
            n = len(v) // 5
            tot += per_call * n
            print("%-28s x%-3d %8.1f us each %9.1f us total" % (k, n, per_call * 1e3, per_call * n * 1e3))
        print("sum %.1f us" % (tot * 1e3))
    print(json.dumps({"workload": "ECAPA-TDNN c{}, 80-d fbank, 300-frame chunks, batch 128".format(channels),
                      "ms_per_step": ms, "frames_per_s": B * T / (ms * 1e-3),
                      "algorithmic_tflops": flop / (ms * 1e-3) / 1e12, "finite": bool(torch.isfinite(out).all()),
                      "extractor": type(ex).__name__, "launches": getattr(ex, "last_launches", None)}))


if __name__ == "__main__":
    main()
