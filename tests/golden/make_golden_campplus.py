#!/usr/bin/env python
"""Golden embeddings of the REFERENCE's CAM++ (subtools2/egrecho/models/campplus/) -- build container only:
    python tests/golden/make_golden_campplus.py   ->  tests/golden/campplus.npz

The reference's campplus.py, campplus_config.py, model.py, models/architecture/speaker/xvector.py, nn/components.py,
nn/activation.py, nn/classifier.py and utils/types.py run unmodified.  Stubbed are only the framework bases they derive
from: ModelBase (post_init applies _init_weights), DataclassConfig (from_config / to_dict), the Lightning base
TopVirtualModel (holds the config, no-op save_hyperparameters), and the models/architecture/speaker package __init__
(it imports torchmetrics), whose xvector.py is loaded by file instead.

Cases (tests/campplus_oracle.py CASES): the default config at T = 300, 200, 201, 37, 3 through CamPP.forward and at
T = 4001, 9000 through CamPPModel.extract_embedding (the 4000-frame chunk rule), and a small config at T = 150, 4.  The
backbone's state_dict is replaced by seeded_state_dict() of its own "key:shape" list (BatchNorm statistics and affines
randomised) and loaded with strict=True.  The npz stores the embeddings of two seeded utterances (campplus_oracle.
utterances) per (case, T), the
backbone and CamPPModel key lists and split_chunks' sizes for SPLIT_T; no weights."""
import dataclasses
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import campplus_oracle as co  # noqa: E402

EG = "/root/reference/subtools2/egrecho"


def _package(name):
    m = types.ModuleType(name)
    m.__path__ = []
    sys.modules[name] = m
    return m


def _load(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(EG, rel))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


class ModelBase(torch.nn.Module):
    def post_init(self):
        self.apply(self._init_weights)

    def _init_weights(self, module):
        pass


class DataclassConfig:
    @classmethod
    def from_config(cls, config=None, **kwargs):
        if isinstance(config, cls):
            return config
        return cls(**dict(config or {}, **kwargs))

    def to_dict(self):
        return dataclasses.asdict(self)


class TopVirtualModel(torch.nn.Module):
    CONFIG_CLS = None

    def __init__(self, config, *args, **kwargs):
        super().__init__()
        self.config = config

    def save_hyperparameters(self, *args, **kwargs):
        pass


def reference_modules():
    for name in ("egrecho", "egrecho.core", "egrecho.nn", "egrecho.utils", "egrecho.models", "egrecho.models.campplus",
                 "egrecho.models.architecture"):
        _package(name)
    sys.modules["egrecho.core.model_base"] = types.SimpleNamespace(ModelBase=ModelBase)
    sys.modules["egrecho.core.config"] = types.SimpleNamespace(DataclassConfig=DataclassConfig)
    sys.modules["egrecho.core.module"] = types.SimpleNamespace(TopVirtualModel=TopVirtualModel)
    _load("egrecho.utils.types", "utils/types.py")
    _load("egrecho.nn.activation", "nn/activation.py")
    _load("egrecho.nn.components", "nn/components.py")
    _load("egrecho.nn.classifier", "nn/classifier.py")
    speaker = _package("egrecho.models.architecture.speaker")
    xv = _load("egrecho.models.architecture.speaker.xvector", "models/architecture/speaker/xvector.py")
    speaker.XvectorMixin, speaker.XvectorOutput = xv.XvectorMixin, xv.XvectorOutput
    cfg = _load("egrecho.models.campplus.campplus_config", "models/campplus/campplus_config.py")
    _load("egrecho.models.campplus.campplus", "models/campplus/campplus.py")
    model = _load("egrecho.models.campplus.model", "models/campplus/model.py")
    return cfg, model, xv


def _keys(module):
    return np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in module.state_dict().items()])


def main():
    cfg, mod, xv = reference_modules()
    torch.manual_seed(0)
    out = {}
    for case, (config, frames, long_frames, seed, fseed) in co.CASES.items():
        model = mod.CamPPModel(cfg.CamPPSVConfig(**config))
        model.eval()
        keys = _keys(model.cam)
        model.cam.load_state_dict(co.seeded_state_dict(keys, seed), strict=True)
        out["keys_" + case] = keys
        out["model_keys_" + case] = _keys(model)
        for t in frames + long_frames:
            feats = co.utterances(2, t, config["inputs_dim"], fseed + t)
            with torch.no_grad():
                if t in long_frames:
                    emb = np.stack([model.extract_embedding(feats[i:i + 1]).xvector[0].numpy() for i in range(2)])
                else:
                    emb = np.stack([model.cam(feats[i:i + 1])[0].numpy() for i in range(2)])
            if t > 2:
                assert np.all(np.isfinite(emb)) and emb.std() > 1e-3 and np.abs(emb[0] - emb[1]).max() > 1e-3, (case, t)
            out["{}_T{}".format(case, t)] = emb
            print(case, t, float(emb.std()), flush=True)
    x = torch.zeros(1, max(co.SPLIT_T))
    out["split_T"] = np.array(co.SPLIT_T, np.int64)
    sizes = [xv.XvectorMixin.split_chunks(x[:, :t], max_chunk=co.MAX_CHUNK)[1] for t in co.SPLIT_T]
    out["split_sizes"] = np.array([s + [0] * (8 - len(s)) for s in sizes], np.int64)
    np.savez_compressed(os.path.join(HERE, "campplus.npz"), **out)
    print("campplus.npz", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
