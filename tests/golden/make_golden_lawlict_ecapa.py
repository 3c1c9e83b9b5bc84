#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's pytorch/model/ecapa-tdnn-xvector.py (the runEcapaXvector.py launcher's
ECAPA_TDNN) for the cases of tests/lawlict_ecapa_oracle.py -- build container only:
    python tests/golden/make_golden_lawlict_ecapa.py   ->  tests/golden/lawlict_ecapa.npz
The reference blueprint runs unmodified through its own utils.create_model_from_py and the launcher's creation string,
with the module stubs of make_golden_ecapa512.py.  Seeded checkpoints from oracle.nnet.make_state_dict(spec(...)) are
loaded strictly; the npz stores only outputs (two utterances per short length, one per chunked length, through
extract_embedding and its maxChunk = 10000 rule), the state_dict layout "keys_<case>" (training=False), the training
layout "train_keys_<case>" and the parameter counts "params_<case>" and "params_default" (ECAPA_TDNN(80, 1211,
training=False, channels=512)), running statistics left out."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import lawlict_ecapa_oracle as lo  # noqa: E402
from oracle import nnet as onn  # noqa: E402

REF = "/root/reference"


def _keys(sd, skip_loss=True):
    return np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in sd.items()
                     if not (skip_loss and k.startswith("loss."))])


def main():
    for name, attrs in (("tkinter", {"N": "n"}), ("tkinter.messagebox", {"NO": "no"}), ("turtle", {"xcor": None})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.path.insert(0, os.path.join(REF, "pytorch"))
    import libs.support.utils as utils
    blueprint = os.path.join(REF, "pytorch/model/ecapa-tdnn-xvector.py")
    torch.set_num_threads(os.cpu_count() or 1)
    out = {}
    for case, (inputs_dim, kw, short, long, positions, seed, _) in lo.CASES.items():
        spec = lo.spec(inputs_dim, kw)
        sd = onn.make_state_dict(spec, seed)
        train = utils.create_model_from_py(blueprint, lo.creation_string(dict(kw, training=True), inputs_dim))
        out["train_keys_" + case] = _keys(train.state_dict(), skip_loss=False)
        for pos in positions:
            model = utils.create_model_from_py(blueprint, lo.creation_string(kw, inputs_dim, position=pos))
            ref_sd = model.state_dict()
            assert list(ref_sd) == [k for k, _, _ in spec], (case, set(ref_sd) ^ set(k for k, _, _ in spec))
            out["keys_" + case] = _keys(ref_sd)
            out["params_" + case] = np.int64(sum(v.numel() for k, v in ref_sd.items()
                                                 if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))))
            model.load_state_dict(sd, strict=True)
            model.eval()
            for t in short + long:
                feats = lo.utterances(case, t)
                emb = np.stack([model.extract_embedding(f).numpy() for f in feats])
                assert np.all(np.isfinite(emb)) and emb.std() > 1e-3, (case, pos, t)
                out["{}_{}_T{}".format(case, pos, t)] = emb
                print(case, pos, t, float(emb.std()), flush=True)
    default = utils.create_model_from_py(blueprint, "ECAPA_TDNN(80,1211,training=False,channels=512)").state_dict()
    out["params_default"] = np.int64(sum(v.numel() for k, v in default.items()
                                         if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))))
    assert (out["params_default"], out["params_launcher"]) == (lo.PARAMS_DEFAULT, lo.PARAMS_LAUNCHER), \
        (out["params_default"], out["params_launcher"])
    np.savez_compressed(os.path.join(HERE, "lawlict_ecapa.npz"), **out)
    print("lawlict_ecapa.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
