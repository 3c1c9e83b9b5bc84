"""ECAPA-TDNN with multi-query multi-head attention pooling, CPU side: the oracle against the reference goldens, the
blueprint's state_dict layout and creation string, the hand-over splits of the attention conv, and the options that
raise."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ecapa_mqmha_oracle as mo  # noqa: E402
from oracle import nnet as onn  # noqa: E402
from asv_subtools_b200.model import ecapa_tdnn_xvector as ex  # noqa: E402
from asv_subtools_b200.nnet.pooling import MQMHASP  # noqa: E402
from asv_subtools_b200.pipeline.extract_embeddings import create_model_from_py  # noqa: E402

GOLD = np.load(os.path.join(ROOT, "tests", "golden", "ecapa_mqmha.npz"))
GOLDEN_CASES = [(case, pos, t) for case, (_, frames, positions, _, _) in mo.CASES.items() for pos in positions for t in frames]


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


def _model(case, pos, **kw):
    kwargs = dict(mo.CASES[case][0], **kw)
    m = ex.ECAPA_TDNN(80, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), mo.CASES[case][3]), strict=True)
    return m.eval()


@pytest.mark.parametrize("case,pos,t", GOLDEN_CASES)
def test_oracle_matches_reference_goldens(case, pos, t):
    kwargs, _, _, seed, fseed = mo.CASES[case]
    sd = onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed)
    feats = onn.synthetic_feats(2, t, 80, fseed + t)
    got = np.stack([mo.extract(sd, feats[i], kwargs, pos).numpy() for i in range(2)])
    ref = GOLD["{}_{}_{}".format(case, pos, t)]
    assert _rel(got, ref) < 1e-5, (case, pos, t, _rel(got, ref))


@pytest.mark.parametrize("case", sorted(mo.CASES))
def test_state_dict_layout_is_the_reference_layout(case):
    kwargs, _, positions, _, _ = mo.CASES[case]
    for pos in positions:
        m = ex.ECAPA_TDNN(80, 10, training=False, extracted_embedding=pos, **kwargs)
        mine = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
        assert mine == [str(k) for k in GOLD["keys_" + case]]
        assert [k for k, _, _ in mo.ecapa_mqmha_spec(kwargs)] == list(m.state_dict())


def test_roadmap_creation_string_builds_and_loads_strict():
    kwargs = mo.CASES["roadmap"][0]
    m = create_model_from_py(os.path.join(ROOT, "asv_subtools_b200", "model", "ecapa_tdnn_xvector.py"),
                             mo.creation_string(kwargs, "near"))
    m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), 31), strict=True)
    st = m.stats
    assert isinstance(st, MQMHASP)
    assert (st.num_head, st.num_q, st.hidden_size, st.share, st.affine_layers, st.time_attention, st.stddev) == \
        (2, 2, 64, False, 2, True, True)
    assert st.get_output_dim() == 6144 and m.bn_stats.num_features == 6144 and m.fc2.affine.input_dim == 6144


def test_constructor_defaults_are_the_libs_defaults():
    """ECAPA's pooling defaults (hidden 128, time attention, stddev) over MQMHASP's own (num_q 2, num_head 4, share)."""
    m = ex.ECAPA_TDNN(80, 10, training=False, pooling="mqmha", ecapa_params={"mfa_conv": 256})
    st = m.stats
    assert (st.num_q, st.num_head, st.hidden_size, st.share, st.affine_layers, st.time_attention, st.stddev) == \
        (2, 4, 128, True, 2, True, True)
    bare = MQMHASP(256)
    assert (bare.share, bare.time_attention, bare.num_head) == (True, False, 4)
    # the reference pops `stddev` from ECAPA's pooling_params: MQMHASP keeps its default
    assert ex.ECAPA_TDNN(80, 10, training=False, pooling="mqmha", pooling_params={"stddev": False},
                         ecapa_params={"mfa_conv": 256}).stats.stddev


@pytest.mark.parametrize("case", ["roadmap", "share", "one_layer", "no_tatt"])
def test_attention_handover_float64(case):
    """att_x (x columns) + att_gs (block-diagonal [mean | std] columns) + the bias == the first grouped conv over the
    reference's per-head [x_h | mean_h | std_h] input, in float64."""
    m = _model(case, "near")
    st = m.stats
    recs = {r[0]: r for r in ex._mqmha_attention(st)}
    B, T, C, H = 2, 7, st.in_dim, st.num_head
    x = torch.randn(B, C, T, dtype=torch.float64)
    mean = x.mean(dim=2, keepdim=True)
    std = torch.sqrt((x.pow(2).mean(dim=2, keepdim=True) - mean ** 2).clamp(min=1e-5))
    if st.time_attention:
        parts = [x.view(B, H, -1, T), mean.expand(B, C, T).reshape(B, H, -1, T), std.expand(B, C, T).reshape(B, H, -1, T)]
        x_in = torch.cat(parts, dim=2).reshape(B, -1, T)
    else:
        x_in = x
    ref = torch.nn.functional.conv1d(x_in, st.attention[0].weight.double(), st.attention[0].bias.double(), groups=H)
    _, wx, bx, _, _, gx = recs["att_x"]
    assert gx == H
    dense = ex._block_diagonal(torch.from_numpy(wx).double(), H)
    got = torch.einsum("nc,bct->bnt", dense[:, :, 0], x)
    if st.time_attention:
        _, wg, bg, _, _, _ = recs["att_gs"]
        gstat = torch.cat([mean, std], dim=1)[:, :, 0]
        got = got + (gstat @ torch.from_numpy(wg[:, :, 0]).double().T + torch.from_numpy(bg).double())[:, :, None]
        assert bx is None
    else:
        got = got + torch.from_numpy(bx).double()[None, :, None]
    assert torch.allclose(got, ref, rtol=0, atol=1e-12)
    if st.affine_layers == 2:
        assert recs["att2"][5] == H * st.num_q
        assert np.array_equal(recs["att2"][1], st.attention[4].weight.detach().numpy())
    else:
        assert "att2" not in recs


def test_bn_stats_fold_float64():
    m = _model("fc1", "near_affine")
    recs = ex._segment_layers(m)
    w, b = recs[0][1][:, :, 0].astype(np.float64), recs[0][2].astype(np.float64)
    x = np.random.RandomState(0).standard_normal((3, m.stats.get_output_dim()))
    bn = m.bn_stats
    xb = (x - bn.running_mean.double().numpy()) / np.sqrt(bn.running_var.double().numpy() + bn.eps) * \
        bn.weight.detach().double().numpy() + bn.bias.detach().double().numpy()
    ref = xb @ m.fc1.affine.weight.detach().double().numpy()[:, :, 0].T + m.fc1.affine.bias.detach().double().numpy()
    assert np.abs(x @ w.T + b - ref).max() < 1e-4 * np.abs(ref).max()


def test_block_diagonal_expansion_is_conv1d_groups():
    w = torch.randn(12, 5, 1, dtype=torch.float64)
    x = torch.randn(2, 15, 4, dtype=torch.float64)
    ref = torch.nn.functional.conv1d(x, w, groups=3)
    got = torch.nn.functional.conv1d(x, ex._block_diagonal(w, 3))
    assert torch.equal(got, ref)


@pytest.mark.parametrize("kw,name", [
    (dict(pooling="multi-head"), "multi-head"),
    (dict(pooling="attentive"), "attentive"),
    (dict(pooling="mqmha_linear"), "mqmha_linear"),
    (dict(pooling="mqmha", pooling_params={"norm_type": "layer_norm"}), "layer_norm"),
])
def test_unsupported_options_raise_naming_themselves(kw, name):
    with pytest.raises(NotImplementedError, match=name):
        ex.ECAPA_TDNN(80, 10, training=False, ecapa_params={"mfa_conv": 256}, **kw)
