"""egrecho's ECAPA-TDNN blueprint on the CPU: the torch restatement against the reference's golden embeddings, the
state_dict layout and loading rules, the records the ECAPA-TDNN handle receives (every backbone tensor carried once, the
head folds in float64), the chunk plan, and the C declaration of the residual-form switch."""
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import egrecho_ecapa_oracle as eo  # noqa: E402
from asv_subtools_b200 import _lib  # noqa: E402
from asv_subtools_b200.model import campplus_xvector as cx  # noqa: E402
from asv_subtools_b200.model import egrecho_ecapa_xvector as eg  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "egrecho_ecapa.npz"))
GOLDEN_KEYS = [(case, pos, t) for case, (_, frames, long_frames, positions, _, _) in eo.CASES.items()
               for pos in positions for t in frames + long_frames]


def _keys(m):
    return ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]


def _model(config, seed, **extra):
    m = eg.EcapaXvector(config["inputs_dim"], 10, **dict(eo.blueprint_kwargs(config), **extra))
    m.load_state_dict(eo.seeded_state_dict(_keys(m), seed), strict=True)
    return m.eval()


@pytest.mark.parametrize("case,pos,t", GOLDEN_KEYS)
def test_oracle_replays_golden(case, pos, t):
    config, _, long_frames, _, seed, fseed = eo.CASES[case]
    sd = eo.seeded_state_dict(GOLDEN["keys_" + case], seed)
    feats = eo.utterances(2, t, config["inputs_dim"], fseed + t)
    with torch.no_grad():
        if t in long_frames:
            got = torch.cat([eo.extract_embedding(sd, feats[i:i + 1], config, pos) for i in range(2)]).numpy()
        else:
            got = torch.cat([eo.forward(sd, feats[i:i + 1], config)[0 if pos == "near" else 1] for i in range(2)]).numpy()
    want = GOLDEN["{}_{}_T{}".format(case, pos, t)]
    assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), (case, pos, t)


@pytest.mark.parametrize("case", sorted(eo.CASES))
def test_state_dict_layout_equals_reference(case):
    config = eo.CASES[case][0]
    m = eg.EcapaXvector(config["inputs_dim"], 10, **eo.blueprint_kwargs(config))
    assert _keys(m) == list(GOLDEN["keys_" + case])


def test_ecapa_model_state_dict_loads_and_foreign_dicts_are_refused():
    config, _, _, _, seed, _ = eo.CASES["c512"]
    m = eg.EcapaXvector(80, 10)
    want = eo.seeded_state_dict(GOLDEN["keys_c512"], seed)
    sd = {k: want[k[6:]] if k.startswith("ecapa.") else torch.zeros(1) for k in
          (key.split(":")[0] for key in GOLDEN["model_keys_c512"])}
    assert any(k.startswith("classifier.") for k in sd)
    m.load_state_dict(sd, strict=True)           # ecapa.* stripped, classifier.* dropped
    got = m.state_dict()
    assert all(torch.equal(got[k], want[k]) for k in want)
    for bad in ({}, {"model.weight": torch.zeros(1)}, {"ecapa.classifier.weight": torch.zeros(1)}):
        with pytest.raises(KeyError):
            m.load_state_dict(bad, strict=False)
    with pytest.raises(NotImplementedError, match="shortcut"):
        m.load_state_dict(dict(want, **{"layer2.shortcut.weight": torch.zeros(1)}), strict=False)


def test_options_that_are_not_built_raise():
    with pytest.raises(NotImplementedError, match="norm_type"):
        eg.EcapaXvector(80, 10, pooling_params={"norm_type": "ln"})
    with pytest.raises(ValueError):
        eg.EcapaXvector(80, 10, pooling_params={"norm_type": "gn"})
    with pytest.raises(TypeError, match="pre_norm"):
        eg.EcapaXvector(80, 10, pooling_params={"pre_norm": True})
    with pytest.raises(ValueError):
        eg.EcapaXvector(80, 10, embd_layer_num=3)
    m = _model(eo.DEFAULT, 5, extracted_embedding="far")
    with pytest.raises(RuntimeError, match="far"):
        m.build_extractor()
    with pytest.raises(NotImplementedError, match="EcapaXvector"):
        m.extract_embedding_batch(torch.zeros(2, 10, 80), lengths=[10, 5])


# small widths: the records are rebuilt once per state_dict tensor
TINY = dict(inputs_dim=24, channels=64, mfa_dim=96, embd_dim=16)
TINY_CASES = {
    "default": dict(TINY, pooling_params=dict(hidden_size=8)),
    "two_layer_near": dict(TINY, embd_layer_num=2, post_norm=True, pooling_params=dict(hidden_size=8)),
    "two_layer_far": dict(TINY, embd_layer_num=2, extracted_embedding="far", pooling_params=dict(hidden_size=8)),
    "mqmha": dict(TINY, pooling_params=dict(num_head=4, num_q=2, share=True, affine_layers=1)),
    "no_norm_no_tatt": dict(TINY, pooling_params=dict(num_head=2, hidden_size=8, norm_type="", time_attention=False)),
}


@pytest.mark.parametrize("case", sorted(TINY_CASES))
def test_records_carry_every_backbone_tensor_once(case):
    """Each state_dict tensor changes exactly one record when perturbed -- the first attention conv's weight two under
    time attention, its x columns (att_x) and its [mean | std] columns (att_gs) -- and every record depends on some
    tensor.  "far" leaves embd2 out."""
    config = dict(TINY_CASES[case])
    m = eg.EcapaXvector(config.pop("inputs_dim"), 10, **config)
    sd = eo.seeded_state_dict(_keys(m), 3)
    m.load_state_dict(sd, strict=True)
    # copies: a record's arrays may share memory with the parameters load_state_dict overwrites
    base = {r[0]: tuple(np.array(a) if isinstance(a, np.ndarray) else a for a in r) for r in eg.native_records(m)}
    touched = set()
    tatt = m.stats.time_attention
    first = "stats.attention.0.weight" if m.stats.affine_layers == 2 else "stats.attention.weight"
    for k in sd:
        if k.endswith("num_batches_tracked"):
            continue
        m.load_state_dict(dict(sd, **{k: sd[k] + 0.5}), strict=True)
        now = {r[0]: r for r in eg.native_records(m)}
        assert now.keys() == base.keys()
        changed = {n for n in base if any(
            (a is None) != (b is None) or (a is not None and not np.array_equal(np.asarray(a), np.asarray(b)))
            for a, b in zip(base[n][1:], now[n][1:]))}
        if k.startswith("embd2.") and m.extracted_embedding == "far":
            assert not changed, k
            continue
        assert len(changed) == (2 if k == first and tatt else 1), (k, changed)
        touched |= changed
    assert touched == set(base)


@pytest.mark.parametrize("case", ["default", "two_layer_near", "two_layer_far"])
def test_head_folds_equal_float64(case):
    config = dict(TINY_CASES[case])
    m = eg.EcapaXvector(config.pop("inputs_dim"), 10, **config)
    sd = eo.seeded_state_dict(_keys(m), 4)
    m.load_state_dict(sd, strict=True)
    recs = {r[0]: r for r in eg.native_records(m)}
    d = {k: v.double() for k, v in sd.items() if v.is_floating_point()}

    def bn(p):
        s = 1.0 / torch.sqrt(d[p + "running_var"] + 1e-5)
        if p + "weight" in d:
            s = s * d[p + "weight"]
        t = -d[p + "running_mean"] * s + (d[p + "bias"] if p + "bias" in d else 0)
        return s, t

    s, t = bn("bn_stats.")
    w1 = d["embd1.linear.weight"][:, :, 0]
    b1 = d.get("embd1.linear.bias", torch.zeros(w1.shape[0], dtype=torch.float64))
    first = "fc2" if m.embd_layer_num == 1 else "fc1"
    _, w, b, ctx, scale, shift, relu = recs[first]
    assert ctx == [0] and relu == (m.embd_layer_num == 2)
    np.testing.assert_allclose(w[:, :, 0], (w1 * s[None, :]).numpy(), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(b, (w1 @ t + b1).numpy(), rtol=1e-6, atol=1e-6)
    if m.embd_layer_num == 2:
        s1, t1 = bn("embd1.nonlinear.1.")
        np.testing.assert_allclose(scale, s1.numpy(), rtol=1e-6)
        np.testing.assert_allclose(shift, t1.numpy(), rtol=1e-6, atol=1e-7)
    if m.embd_layer_num == 2 and m.extracted_embedding == "near":
        _, w, b, _, scale, shift, relu = recs["fc2"]
        np.testing.assert_array_equal(w[:, :, 0], sd["embd2.linear.weight"][:, :, 0].numpy())
        assert not relu and not np.any(b)
        s2, t2 = bn("embd2.nonlinear.1.")
        np.testing.assert_allclose(scale, s2.numpy(), rtol=1e-6)
        np.testing.assert_allclose(shift, t2.numpy(), rtol=1e-6, atol=1e-7)
    assert ("fc2" in recs) == (m.extracted_embedding == "near")


def test_dilated_res2net_taps_spread_over_their_span():
    m = eg.EcapaXvector(24, 10, **{k: v for k, v in TINY.items() if k != "inputs_dim"})
    recs = {r[0]: r for r in eg.native_records(m)}
    for li, d in zip((2, 3, 4), eg.DILATIONS):
        name, w, _, ctx, _, _, relu = recs["layer{}.res3".format(li)]
        src = getattr(m, "layer{}".format(li)).res2net_block.blocks[3].linear.weight.detach().numpy()
        assert ctx == [-d, 0, d] and relu and w.shape == (8, 8, 2 * d + 1)
        np.testing.assert_array_equal(w[:, :, ::d], src)
        assert not np.any(np.delete(w, [0, d, 2 * d], axis=2))


def test_chunk_plan_equals_fixture_and_native_rule():
    for t, row in zip(GOLDEN["split_T"], GOLDEN["split_sizes"]):
        assert eg.chunk_sizes(int(t)) == [int(v) for v in row if v], t
    assert eg.chunk_sizes is cx.chunk_sizes
    out = (_lib.C.c_int * 8)()
    for t in range(1, 20002):
        n = _lib.lib.xvb_campp_chunk_sizes(t, eo.MAX_CHUNK, out, 8)
        assert list(out[:n]) == eg.chunk_sizes(t), t


def test_set_chained_declaration_matches_binding():
    header = open(os.path.join(ROOT, "include", "xvb200.h")).read()
    assert re.search(r"\bint xvb_ecapa_set_chained\(xvb_ecapa_t\* h, int chained\);", header)
    assert _lib.SIGNATURES["xvb_ecapa_set_chained"] == (_lib.C.c_int, [_lib.C.c_void_p, _lib.C.c_int])
    fn = _lib.lib.xvb_ecapa_set_chained
    assert fn.restype is _lib.C.c_int and list(fn.argtypes) == [_lib.C.c_void_p, _lib.C.c_int]
