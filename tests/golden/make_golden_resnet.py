#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's 2-D ResNetXvector (pytorch/model/resnet_xvector.py over libs/nnet/resnet.py) --
build container only:
    python tests/golden/make_golden_resnet.py   ->  tests/golden/resnet.npz
Cases (tests/resnet_oracle.py CASES): the online launcher's model, the pre-activation launcher's model at F = 23 (odd
spatial sizes) and a ResNet18.  Each seeded checkpoint, make_state_dict(resnet_spec(...)), is loaded with strict=True,
which asserts the key layout; the npz stores the embeddings of two seeded utterances per (case, position, T) and the
reference's state_dict "key:shape" list, no weights."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import nnet as onn  # noqa: E402
import resnet_oracle as ro  # noqa: E402


def main():
    for name, attrs in (("tkinter", {"N": "n"}), ("tkinter.messagebox", {"NO": "no"}), ("turtle", {"xcor": None})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m
    sys.path.insert(0, "/root/reference/pytorch")
    import libs.support.utils as utils
    out = {}
    for case, (kwargs, fdim, frames, positions, seed, fseed) in ro.CASES.items():
        sd = onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed)
        for pos in positions:
            model = utils.create_model_from_py("/root/reference/pytorch/model/resnet_xvector.py", ro.creation(kwargs, fdim, pos))
            model.load_state_dict(sd, strict=True)
            model.eval()
            out["keys_" + case] = np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape))
                                            for k, v in model.state_dict().items()])
            for t in frames:
                feats = onn.synthetic_feats(2, t, fdim, fseed + t)
                emb = np.stack([model.extract_embedding(feats[i]).numpy() for i in range(2)])
                # a single frame leaves the synthetic checkpoint's deep layers input-independent (every ReLU of some
                # block is off), so T = 1 only has to give a finite, non-constant vector
                assert np.all(np.isfinite(emb)) and emb.std() > 1e-3 and (t == 1 or np.abs(emb[0] - emb[1]).max() > 1e-3), \
                    (case, pos, t)
                out["{}_{}_T{}".format(case, pos, t)] = emb
    np.savez_compressed(os.path.join(HERE, "resnet.npz"), **out)
    print("resnet.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
