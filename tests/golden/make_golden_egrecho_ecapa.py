#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's egrecho ECAPA-TDNN (subtools2/egrecho/models/ecapa/) -- build container only:
    python tests/golden/make_golden_egrecho_ecapa.py   ->  tests/golden/egrecho_ecapa.npz

The reference's ecapa_xvector.py, ecapa_config.py, model.py, models/architecture/speaker/xvector.py, nn/components.py,
nn/activation.py, nn/classifier.py and utils/types.py run unmodified.  Stubbed are only the framework bases, with the
stubs of make_golden_campplus.py (imported from it).

Cases (tests/egrecho_ecapa_oracle.py CASES): the recipe config (C1024) at T = 300, 200, 37, 5, 1, the EcapaConfig default
(C512) and its variants (two embedding layers with post_norm, "near" and "far"; MQMHA with 4 heads, 2 queries, share,
one affine layer; the attention without BatchNorm; no time attention; C256) through EcapaXvector.forward, and C512 at
T = 4001, 9000 through EcapaModel.extract_embedding (the 4000-frame chunk rule).  The backbone's state_dict is replaced by
seeded_state_dict() of its own "key:shape" list and loaded with strict=True.  The npz stores the embeddings of two
seeded utterances per (case, position, T), the backbone and EcapaModel key lists and split_chunks' sizes for SPLIT_T; no
weights."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import egrecho_ecapa_oracle as eo  # noqa: E402
import make_golden_campplus as mgc  # noqa: E402


def reference_modules():
    mgc.reference_modules()
    mgc._package("egrecho.models.ecapa")
    cfg = mgc._load("egrecho.models.ecapa.ecapa_config", "models/ecapa/ecapa_config.py")
    mgc._load("egrecho.models.ecapa.ecapa_xvector", "models/ecapa/ecapa_xvector.py")
    model = mgc._load("egrecho.models.ecapa.model", "models/ecapa/model.py")
    xv = sys.modules["egrecho.models.architecture.speaker.xvector"]
    return cfg, model, xv


def main():
    cfg, mod, xv = reference_modules()
    torch.manual_seed(0)
    out = {}
    for case, (config, frames, long_frames, positions, seed, fseed) in eo.CASES.items():
        model = mod.EcapaModel(cfg.EcapaSVConfig(num_classes=10, **config))
        model.eval()
        keys = mgc._keys(model.ecapa)
        model.ecapa.load_state_dict(eo.seeded_state_dict(keys, seed), strict=True)
        out["keys_" + case] = keys
        out["model_keys_" + case] = mgc._keys(model)
        for pos in positions:
            for t in frames + long_frames:
                feats = eo.utterances(2, t, config["inputs_dim"], fseed + t)
                with torch.no_grad():
                    if t in long_frames:
                        emb = np.stack([model.extract_embedding(feats[i:i + 1], position=pos).xvector[0].numpy()
                                        for i in range(2)])
                    else:
                        emb = np.stack([model.ecapa(feats[i:i + 1])[0 if pos == "near" else 1][0].numpy()
                                        for i in range(2)])
                assert np.all(np.isfinite(emb)) and emb.std() > 1e-3 and np.abs(emb[0] - emb[1]).max() > 1e-3, (case, t)
                out["{}_{}_T{}".format(case, pos, t)] = emb
                print(case, pos, t, float(emb.std()), flush=True)
    x = torch.zeros(1, max(eo.SPLIT_T))
    out["split_T"] = np.array(eo.SPLIT_T, np.int64)
    sizes = [xv.XvectorMixin.split_chunks(x[:, :t], max_chunk=eo.MAX_CHUNK)[1] for t in eo.SPLIT_T]
    out["split_sizes"] = np.array([s + [0] * (8 - len(s)) for s in sizes], np.int64)
    np.savez_compressed(os.path.join(HERE, "egrecho_ecapa.npz"), **out)
    print("egrecho_ecapa.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
