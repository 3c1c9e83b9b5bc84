"""The Conformer's 2x subsampling (input_layer="conv2d2") and the records the native Conformer extractor receives
(xvb_conformer_set_layer), on the CPU: the 2Sub restatement against the reference's golden embeddings, the blueprint's
2Sub state_dict against the reference's key list, the F - 4 column order, every state_dict tensor carried by exactly one
record, the handed-over tables, and the short-input refusal."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conformer_2sub_oracle as c2
import conformer_oracle as co
from asv_subtools_b200.model import transformer_xvector as tx
from oracle import nnet as onn

CASE_POS = [(c, p) for c in sorted(c2.CASES) for p in c2.CASES[c][3]]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _model(cases, case, pos):
    kwargs, fdim, _, _, seed, _ = cases[case]
    m = tx.TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    keys = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(co.seeded_state_dict(keys, seed), strict=True)
    return m.eval()


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_2sub_restatement_matches_reference_golden(golden, case, pos):
    g = golden("conformer_2sub")
    kwargs, fdim, frames, _, seed, fseed = c2.CASES[case]
    sd = co.seeded_state_dict(g["keys_" + case], seed)
    cfg = co.config(kwargs)
    for t in frames:
        feats = onn.synthetic_feats(2, t, fdim, fseed + t)
        got = np.stack([c2.extract(sd, feats[i], cfg, pos).numpy() for i in range(2)])
        ref = g["{}_{}_T{}".format(case, pos, t)]
        assert rel(got, ref) <= 1e-5, (case, pos, t, rel(got, ref))


@pytest.mark.parametrize("case", sorted(c2.CASES))
def test_2sub_state_dict_matches_reference_keys(golden, case):
    g = golden("conformer_2sub")
    kwargs, fdim, _, positions, _, _ = c2.CASES[case]
    m = tx.TransformerXvector(fdim, 10, training=False, extracted_embedding=positions[-1], **kwargs)
    mine = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    assert mine == list(g["keys_" + case])
    embed = {k: tuple(v.shape) for k, v in m.state_dict().items() if k.startswith("transformer.embed.")}
    d = kwargs["transformer_params"]["attention_dim"]
    assert embed == {"transformer.embed.conv.0.weight": (d, 1, 3, 3), "transformer.embed.conv.0.bias": (d,),
                     "transformer.embed.conv.2.weight": (d, d, 3, 3), "transformer.embed.conv.2.bias": (d,),
                     "transformer.embed.out.0.weight": (d, d * (fdim - 4)), "transformer.embed.out.0.bias": (d,)}
    assert m.transformer.subsampling == 2


def test_2sub_linear_column_order_float64():
    """The Linear over the (B, T', F'', C) conv output flattened f * C + c with permuted columns equals the reference's
    Linear over the c * F'' + f flattening, in float64."""
    torch.manual_seed(0)
    C, fdim, T = 16, 23, 19
    w0, b0 = torch.randn(C, 1, 3, 3, dtype=torch.float64), torch.randn(C, dtype=torch.float64)
    w2, b2 = torch.randn(C, C, 3, 3, dtype=torch.float64), torch.randn(C, dtype=torch.float64)
    lw = torch.randn(C, C * (fdim - 4), dtype=torch.float64)
    x = torch.randn(2, T, fdim, dtype=torch.float64)
    sd = {"transformer.embed.conv.0.weight": w0, "transformer.embed.conv.0.bias": b0,
          "transformer.embed.conv.2.weight": w2, "transformer.embed.conv.2.bias": b2}
    ref = F.linear(c2.head(sd, x), lw)
    h = F.relu(F.conv2d(F.relu(F.conv2d(x.unsqueeze(1), w0, b0, stride=(2, 1))), w2, b2))    # (B, C, T', F'')
    t2, f2 = tx.subsampled_shape(2, T, fdim)
    assert h.shape[2:] == (t2, f2) == (c2.out_frames(T), fdim - 4)
    flat = h.permute(0, 2, 3, 1).reshape(2, t2, f2 * C)                                          # f * C + c
    got = F.linear(flat, lw[:, torch.from_numpy(tx.subsampling_column_order(C, f2))])
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)


ALL_CASES = dict(co.CASES, **c2.CASES)


@pytest.mark.parametrize("case", sorted(ALL_CASES))
def test_native_records_cover_the_state_dict_once(case):
    """Position "near" uses every tensor: each is carried by exactly one record; the other positions hand over a subset."""
    m = _model(ALL_CASES, case, "near" if "near" in ALL_CASES[case][3] else ALL_CASES[case][3][-1])
    recs = tx.native_records(m)
    names = [r[0] for r in recs]
    assert len(names) == len(set(names))
    carried = [k for r in recs for k in r[6]]
    assert len(carried) == len(set(carried))
    sd = m.state_dict()
    assert set(carried) <= set(sd)
    if m.extracted_embedding == "near":
        assert set(carried) == set(sd), set(sd) ^ set(carried)
    else:
        assert set(sd) - set(carried) <= {"fc2.batchnorm.weight", "fc2.batchnorm.bias"}
    by_name = {r[0]: r for r in recs}
    p = "transformer.encoders.0."
    qkv = by_name[p + "self_attn.linear_qkv"]
    a = m.transformer.encoders[0].self_attn
    assert np.array_equal(qkv[1], torch.cat([a.linear_q.weight, a.linear_k.weight, a.linear_v.weight]).detach().numpy())
    conv2 = m.transformer.embed.conv[2].weight.detach()
    d = conv2.shape[0]
    assert np.array_equal(by_name["transformer.embed.conv.2"][1], conv2.transpose(2, 3).reshape(d, 9 * d).numpy())
    cfg = tx.native_config(m)
    assert cfg["subsampling"] == (2 if case in c2.CASES else 4)


@pytest.mark.parametrize("case", ["launcher", "launcher2", "small2", "rotv"])
def test_handed_over_tables_equal_the_python_tables(case):
    kwargs = ALL_CASES[case][0]
    m = _model(ALL_CASES, case, ALL_CASES[case][3][-1])
    by_name = {r[0]: r for r in tx.native_records(m)}
    p = m.transformer.p
    d, h = p["attention_dim"], p["attention_heads"]
    want = tx.rotary_table(d // h) if p["pos_enc_type"] == "rot_pos" else tx.sinusoid_table(d)
    assert np.array_equal(by_name["pos_table"][1], want.numpy()) and want.shape[0] == tx.TABLE_ROWS
    sp = kwargs["transformer_params"].get("attention_norm_args", {}).get("norm_method") == "softmax_plus"
    for i, layer in enumerate(m.transformer.encoders):
        name = "transformer.encoders.{}.self_attn.att_norm".format(i)
        assert (name in by_name) == sp
        if sp:
            mult = by_name[name][1]
            assert mult.shape == (1, tx.TABLE_ROWS)
            for t in (1, 2, 7, 36, 74, 149, 300, 4999):
                assert mult[0, t] == np.float32(tx.softmax_plus_multiplier(t, layer.self_attn.att_norm.train_len)), t


def test_2sub_shortest_input_and_frame_counts():
    m = _model(c2.CASES, "small2", "near")
    with pytest.raises(ValueError, match="at least 7 frames"):
        m.extract_embedding(np.zeros((6, 23), np.float32))
    with pytest.raises(ValueError, match="at least 7 frames"):
        m.extract_embedding_batch(np.zeros((2, 6, 23), np.float32))
    assert [tx.subsampled_shape(2, t, 80) for t in (7, 8, 300)] == [(1, 76), (1, 76), (147, 76)]
    assert [tx.subsampled_shape(4, t, 80) for t in (7, 300)] == [(1, 19), (74, 19)]


def test_other_input_layers_still_raise():
    for layer in ("linear", "re_conv2d", "conv2d6", "conv2d8"):
        kwargs = dict(c2.SMALL_2SUB, transformer_params=dict(c2.SMALL_2SUB["transformer_params"], input_layer=layer))
        with pytest.raises(NotImplementedError, match="input_layer"):
            tx.TransformerXvector(23, 10, training=False, **kwargs)
