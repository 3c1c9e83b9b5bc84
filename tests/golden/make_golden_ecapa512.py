#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's ECAPA_TDNN at 512 channels (pytorch/model/ecapa_tdnn_xvector.py with
ecapa_params={"channels": 512}: Res2Net width 64) for the cases of tests/ecapa512_cases.py -- build container only:
    python tests/golden/make_golden_ecapa512.py   ->  tests/golden/ecapa512.npz
Seeded checkpoints from oracle.nnet.make_state_dict(ecapa_spec(80, channels=512, ...)), loaded strictly into the
reference model; only outputs and the reference's state_dict layout ("keys_<case>") are stored.  The MQMHA case patches
libs.nnet.pooling.compute_statistics as make_golden_ecapa_mqmha.py does."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ecapa512_cases as c5  # noqa: E402
import ecapa_mqmha_oracle as mo  # noqa: E402
from make_golden_ecapa_mqmha import compute_statistics  # noqa: E402
from oracle import nnet as onn  # noqa: E402

REF = "/root/reference"


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
    for case, (kw, spec, seed, positions, frames, _) in c5.CASES.items():
        sd = onn.make_state_dict(spec, seed)
        for pos in positions:
            model = utils.create_model_from_py(os.path.join(REF, "pytorch/model/ecapa_tdnn_xvector.py"),
                                               mo.creation_string(kw, pos))
            ref_sd = model.state_dict()
            ref_keys = [k for k in ref_sd if not k.startswith("loss.")]
            assert ref_keys == [k for k, _, _ in spec], (case, set(ref_keys) ^ set(k for k, _, _ in spec))
            out["keys_" + case] = np.array(["{}:{}".format(k, ",".join(str(d) for d in ref_sd[k].shape)) for k in ref_keys])
            out["params_" + case] = np.int64(sum(ref_sd[k].numel() for k in ref_keys if not k.endswith(("running_mean",
                                                 "running_var", "num_batches_tracked"))))
            model.load_state_dict(sd, strict=True)
            model.eval()
            for t in frames:
                feats = c5.utterances(case, t)
                out["{}_{}_T{}".format(case, pos, t)] = np.stack([model.extract_embedding(f).numpy() for f in feats])
                print(case, pos, t, flush=True)
    np.savez_compressed(os.path.join(HERE, "ecapa512.npz"), **out)
    print("ecapa512.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
