#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's TransformerXvector with input_layer="conv2d2" (SVConv2dSubsampling2,
pytorch/libs/nnet/transformer/subsampling.py:365-415) -- build container only:
    python tests/golden/make_golden_conformer_2sub.py   ->  tests/golden/conformer_2sub.npz
Cases (tests/conformer_2sub_oracle.py CASES): the launcher's model with 2x subsampling at F = 80 (near / near_affine;
T = 300, 37, 7 and the multi-chunk 650, 899) and a small 2Sub model at F = 23 with abs_pos, softmax, a BatchNorm
conv module, relu and fc1 (all three positions; T = 150, 8).  Built exactly as make_golden_conformer.py: the creation
string through create_model_from_py, seeded_state_dict() of the model's own "key:shape" list loaded with strict=True.
The npz stores the embeddings of two seeded utterances per (case, position, T) and the key lists; no weights."""
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
import conformer_oracle as co  # noqa: E402
import conformer_2sub_oracle as c2  # noqa: E402

REF = "/root/reference/pytorch"


def _keys(model):
    return np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in model.state_dict().items()])


def main():
    for name, attrs in (("tkinter", {"N": "n"}), ("tkinter.messagebox", {"NO": "no"}), ("turtle", {"xcor": None})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.path.insert(0, REF)
    import libs.support.utils as utils
    torch.manual_seed(0)
    blueprint = os.path.join(REF, "model", "transformer_xvector.py")
    out = {}
    for case, (kwargs, fdim, frames, positions, seed, fseed) in c2.CASES.items():
        for pos in positions:
            model = utils.create_model_from_py(blueprint, co.creation(kwargs, fdim, pos))
            keys = _keys(model)
            model.load_state_dict(co.seeded_state_dict(keys, seed), strict=True)
            model.eval()
            out["keys_" + case] = keys
            for t in frames:
                feats = onn.synthetic_feats(2, t, fdim, fseed + t)
                with torch.no_grad():
                    emb = np.stack([model.extract_embedding(feats[i]).numpy() for i in range(2)])
                assert np.all(np.isfinite(emb)) and emb.std() > 1e-3 and np.abs(emb[0] - emb[1]).max() > 1e-3, (case, pos, t)
                out["{}_{}_T{}".format(case, pos, t)] = emb
                print(case, pos, t, flush=True)
    np.savez_compressed(os.path.join(HERE, "conformer_2sub.npz"), **out)
    print("conformer_2sub.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
