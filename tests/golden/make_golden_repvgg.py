#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's RepVggXvector (pytorch/model/repvgg_xvector.py over libs/nnet/repvgg.py) --
build container only:
    python tests/golden/make_golden_repvgg.py   ->  tests/golden/repvgg.npz
Cases (tests/repvgg_oracle.py CASES): the launcher's default RepSPK model, auto_model RepVGG_A0 at F = 23 (odd spatial
sizes) in all three positions, and a small grouped RepSPK stack with BatchNorm affine=False.  Each seeded checkpoint,
make_state_dict(repvgg_spec(...)), is loaded with strict=True, which asserts the key layout.  The launcher's model is
also converted with the reference's repvgg_model_convert and loaded into a deploy=True model with strict=True (deploy
keys and embeddings).  The npz stores the embeddings of two seeded utterances per (case, position, T), the reference's
state_dict "key:shape" lists and its auto_model table as JSON; no weights."""
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import nnet as onn  # noqa: E402
import repvgg_oracle as ro  # noqa: E402

REF = "/root/reference/pytorch"


def _keys(model):
    return np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in model.state_dict().items()])


def _embeddings(model, case, pos, t, fdim, fseed):
    feats = onn.synthetic_feats(2, t, fdim, fseed + t)
    with torch.no_grad():
        emb = np.stack([model.extract_embedding(feats[i]).numpy() for i in range(2)])
    # a single frame may leave the deep layers input-independent, so T = 1 only has to give a finite, non-constant vector
    assert np.all(np.isfinite(emb)) and emb.std() > 1e-3 and (t == 1 or np.abs(emb[0] - emb[1]).max() > 1e-3), (case, pos, t)
    return emb


def main():
    for name, attrs in (("tkinter", {"N": "n"}), ("tkinter.messagebox", {"NO": "no"}), ("turtle", {"xcor": None})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.path.insert(0, REF)
    import libs.support.utils as utils
    from libs.nnet.repvgg import repvgg_model_convert
    blueprint = os.path.join(REF, "model", "repvgg_xvector.py")
    out = {}
    for case, (kwargs, fdim, frames, positions, seed, fseed) in ro.CASES.items():
        sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
        for pos in positions:
            model = utils.create_model_from_py(blueprint, ro.creation(kwargs, fdim, pos))
            model.load_state_dict(sd, strict=True)
            model.eval()
            out["keys_" + case] = _keys(model)
            for t in frames:
                out["{}_{}_T{}".format(case, pos, t)] = _embeddings(model, case, pos, t, fdim, fseed)
            if case == ro.DEPLOY_CASE:
                dsd = repvgg_model_convert(model).state_dict()
                dmodel = utils.create_model_from_py(blueprint, ro.creation(kwargs, fdim, pos, deploy=True))
                dmodel.load_state_dict(dsd, strict=True)
                dmodel.eval()
                out["keys_{}_deploy".format(case)] = _keys(dmodel)
                for t in frames:
                    out["{}_deploy_{}_T{}".format(case, pos, t)] = _embeddings(dmodel, case + "_deploy", pos, t, fdim, fseed)
    mod = sys.modules[utils.create_model_from_py(blueprint, ro.creation(ro.A0, 23, "near")).__class__.__module__]
    names = ["RepVGG_A0", "RepVGG_A1", "RepVGG_A2", "RepVGG_B0", "RepVGG_B1", "RepVGG_B1g2", "RepVGG_B1g4", "RepVGG_B2",
             "RepVGG_B2g2", "RepVGG_B2g4", "RepVGG_B3", "RepVGG_B3g2", "RepVGG_B3g4", "RepVGG_D2se"]
    out["auto_model_json"] = np.array(json.dumps({n: mod.auto_model(n) for n in names}, sort_keys=True))
    np.savez_compressed(os.path.join(HERE, "repvgg.npz"), **out)
    print("repvgg.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
