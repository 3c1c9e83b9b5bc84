"""The op-by-op twins (ResNetExtractor, RepVGGExtractor, ConformerExtractor, CamPPExtractor, EcapaExtractor) take their
weights from the records their native handles take, not from the model's modules: with the family's record function
patched to halve one weight, the twin and a handle built after the patch still give the same embeddings bit for bit,
and both differ from the unpatched model's."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import campplus_oracle as cpo  # noqa: E402
import conformer_oracle as co  # noqa: E402
import ecapa_mqmha_oracle as mo  # noqa: E402
import repvgg_oracle as rvo  # noqa: E402
import resnet_oracle as ro  # noqa: E402
from asv_subtools_b200.model import campplus_xvector as cx  # noqa: E402
from asv_subtools_b200.model import ecapa_tdnn_xvector as ex  # noqa: E402
from asv_subtools_b200.model import repvgg_xvector as rv  # noqa: E402
from asv_subtools_b200.model import resnet_xvector as rn  # noqa: E402
from asv_subtools_b200.model import transformer_xvector as tx  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu


def _resnet():
    kw, fdim, _, _, seed, _ = ro.CASES["preact"]
    m = rn.ResNetXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kw), seed), strict=True)
    return rn, "_named_records", rn.ResNetExtractor, rn.NativeResNetExtractor, m, fdim, 30, "resnet.layer2.0.conv2"


def _repvgg():
    kw, fdim, _, _, seed, _ = rvo.CASES["a0"]
    m = rv.RepVggXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(onn.make_state_dict(rvo.repvgg_spec(fdim, kw), seed), strict=True)
    return rv, "_named_records", rv.RepVGGExtractor, rv.NativeRepVGGExtractor, m, fdim, 30, "repvgg.stage2.1"


def _conformer():
    kw, fdim = co.CASES["small"][:2]
    m = tx.TransformerXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    keys = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(co.seeded_state_dict(keys, co.CASES["small"][4]), strict=True)
    return tx, "native_records", tx.ConformerExtractor, tx.NativeConformerExtractor, m, fdim, 40, \
        "transformer.encoders.0.self_attn.linear_qkv"


def _campp():
    kw = dict(cpo.CASES["small"][0])
    fdim = kw.pop("inputs_dim")
    m = cx.CamPPXvector(fdim, 10, **kw)
    keys = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(cpo.seeded_state_dict(keys, cpo.CASES["small"][3]), strict=True)
    return cx, "native_records", cx.CamPPExtractor, cx.NativeCamPPExtractor, m, fdim, 40, "xvector.block2.tdnnd1.linear1"


def _ecapa():
    m = ex.ECAPA_TDNN(80, 10, training=False)
    m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), 201), strict=True)
    return ex, "_named_layers", ex.EcapaExtractor, ex.NativeEcapaExtractor, m, 80, 40, "layer3.res2"


def _ecapa_mqmha():
    kwargs, _, _, seed, _ = mo.CASES["fc1"]
    m = ex.ECAPA_TDNN(80, 10, training=False, extracted_embedding="near", **kwargs)
    m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed), strict=True)
    return ex, "_named_layers", ex.EcapaExtractor, ex.NativeEcapaExtractor, m, 80, 40, "att2"


MODELS = {"resnet": _resnet, "repvgg": _repvgg, "conformer": _conformer, "campp": _campp, "ecapa": _ecapa,
          "ecapa_mqmha": _ecapa_mqmha}


@pytest.mark.parametrize("family", sorted(MODELS))
def test_twin_and_handle_follow_the_records(family, monkeypatch):
    mod, fn, twin_cls, native_cls, m, fdim, frames, target = MODELS[family]()
    m.eval()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(7)
    feats = torch.randn(3, frames, fdim, generator=g).to(dev)
    with torch.no_grad():
        base = native_cls(m, dev).extract(feats).clone()

        records = getattr(mod, fn)
        hits = []

        def halved(model):
            out = []
            for r in records(model):
                if r[0] == target:
                    hits.append(target)
                    r = (r[0], (r[1] * np.float32(0.5)).astype(np.float32)) + tuple(r[2:])
                out.append(r)
            return out

        monkeypatch.setattr(mod, fn, halved)
        native = native_cls(m, dev).extract(feats)
        twin = twin_cls(m, dev).extract(feats)
        torch.cuda.synchronize()
    assert hits, "record {} not found".format(target)
    assert torch.equal(native, twin), (family, float((native - twin).abs().max()))
    assert not torch.equal(native, base), family
    assert not torch.equal(twin, base), family
