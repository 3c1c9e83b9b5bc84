#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's ECAPA_TDNN with pooling="mqmha" (pytorch/model/ecapa_tdnn_xvector.py:289-295 over
MQMHASP, pytorch/libs/nnet/pooling.py:589-698) for the cases of tests/ecapa_mqmha_oracle.py -- build container only:
    python tests/golden/make_golden_ecapa_mqmha.py   ->  tests/golden/ecapa_mqmha.npz
Seeded checkpoints from oracle.nnet.make_state_dict(ecapa_mqmha_spec(...)); only outputs are stored.

MQMHASP.forward (pooling.py:636, :654) calls `compute_statistics`, a name libs/nnet/pooling.py neither defines nor
imports: the reference's own model builds but raises NameError at the first forward.  Before any forward this script
sets the module global libs.nnet.pooling.compute_statistics to a function with the semantics of the maintained helper,
subtools2/egrecho/nn/pooling.py:18-65 (dim=-1, keepdim=True, std = sqrt(clamp(sum(m x^2) - mean^2, 1e-5))).  The
keepdim-less variant of pytorch/model/transformer_xvector.py:12 would scramble channels in mean.repeat(1,1,T).view(...)
and is not used.  The roadmap model is also cross-checked against egrecho's own MQMHASP loaded from its file with the
same weights."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import nnet as onn  # noqa: E402
import ecapa_mqmha_oracle as mo  # noqa: E402

REF = "/root/reference"


def compute_statistics(x, m, dim=-1, stddev=True, eps=1e-5):
    mean = torch.sum(m * x, dim=dim, keepdim=True)
    if stddev:
        std = torch.sqrt((torch.sum(m * (x ** 2), dim=dim, keepdim=True) - mean ** 2).clamp_(eps))
    else:
        std = torch.empty(0)
    return mean, std


def egrecho_mqmha():
    """egrecho's MQMHASP class from its file, with the package-level imports it needs stubbed."""
    src = open(os.path.join(REF, "subtools2/egrecho/nn/pooling.py")).read()
    start, end = src.index("class MQMHASP("), src.index('@ASV_POOLINGS.register(name="mqmhasp_linear")')
    mod = types.ModuleType("egrecho_mqmha")
    mod.__dict__.update({"torch": torch, "F": torch.nn.functional, "compute_statistics": compute_statistics,
                         "Literal": __import__("typing").Literal, "BasePooling": torch.nn.Module,
                         "ASV_POOLINGS": types.SimpleNamespace(register=lambda *a, **k: (lambda c: c))})
    exec(src[start:end], mod.__dict__)
    return mod.MQMHASP


def main():
    for name, attrs in (("tkinter", {"N": "n"}), ("tkinter.messagebox", {"NO": "no"}), ("turtle", {"xcor": None})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.path.insert(0, os.path.join(REF, "pytorch"))
    import libs.support.utils as utils
    import libs.nnet.pooling as ref_pooling
    ref_pooling.compute_statistics = compute_statistics
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}
    for case, (kw, frames, positions, sd_seed, feat_seed) in mo.CASES.items():
        spec = mo.ecapa_mqmha_spec(kw)
        sd = onn.make_state_dict(spec, sd_seed)
        for pos in positions:
            model = utils.create_model_from_py(os.path.join(REF, "pytorch/model/ecapa_tdnn_xvector.py"), mo.creation_string(kw, pos))
            ref_sd = model.state_dict()
            ref_keys = [k for k in ref_sd if not k.startswith("loss.")]
            assert ref_keys == [k for k, _, _ in spec], (case, set(ref_keys) ^ set(k for k, _, _ in spec))
            for k, shape, _ in spec:
                assert tuple(ref_sd[k].shape) == tuple(shape), (case, k, ref_sd[k].shape, shape)
            out["keys_" + case] = np.array(["{}:{}".format(k, ",".join(str(d) for d in ref_sd[k].shape)) for k in ref_keys])
            model.load_state_dict(sd, strict=True)
            model.eval()
            if case == "roadmap" and pos == "near":       # egrecho's MQMHASP on the same weights and input
                p = mo.resolve(kw["pooling_params"])
                eg = egrecho_mqmha()(1536, **{k: v for k, v in p.items()})
                eg.load_state_dict({k[len("stats."):]: v for k, v in sd.items() if k.startswith("stats.")}, strict=True)
                eg.eval()
                x = torch.randn(2, 1536, 50)
                with torch.no_grad():
                    diff = (eg(x).reshape(2, -1) - model.stats(x).reshape(2, -1)).abs().max().item()
                assert diff < 1e-5, diff
                print("egrecho MQMHASP cross-check: max abs diff", diff)
            for t in frames:
                feats = onn.synthetic_feats(2, t, 80, feat_seed + t)
                out["{}_{}_{}".format(case, pos, t)] = np.stack([model.extract_embedding(feats[i]).numpy() for i in range(2)])
                print(case, pos, t, flush=True)
    np.savez_compressed(os.path.join(HERE, "ecapa_mqmha.npz"), **out)
    print("ecapa_mqmha.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
