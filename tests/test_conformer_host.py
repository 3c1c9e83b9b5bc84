"""CPU side of the Conformer x-vector blueprint (asv_subtools_b200/model/transformer_xvector.py): the torch restatement
against the reference's goldens, state_dict keys, the hand-over arithmetic, the chunk plan and the options that raise."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import conformer_oracle as co  # noqa: E402
from oracle import nnet as onn  # noqa: E402
from asv_subtools_b200.model import transformer_xvector as tx  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "conformer.npz"))


def _model(case, pos, **override):
    kwargs, fdim, _, _, seed, _ = co.CASES[case]
    kwargs = dict(kwargs, **override)
    m = tx.TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(co.seeded_state_dict(GOLD["keys_" + case], seed), strict=True)
    return m.eval()


def _rel(a, b):
    return float(np.abs(a - b).max() / np.abs(b).max())


GOLDEN_CASES = [(case, pos, t) for case, (_, _, frames, positions, _, _) in co.CASES.items()
                for pos in positions for t in frames]


@pytest.mark.parametrize("case,pos,t", GOLDEN_CASES)
def test_restatement_matches_reference_goldens(case, pos, t):
    kwargs, fdim, _, _, seed, fseed = co.CASES[case]
    sd = co.seeded_state_dict(GOLD["keys_" + case], seed)
    cfg = co.config(kwargs)
    feats = onn.synthetic_feats(2, t, fdim, fseed + t)
    got = np.stack([co.extract(sd, feats[i], cfg, pos).numpy() for i in range(2)])
    ref = GOLD["{}_{}_T{}".format(case, pos, t)]
    assert _rel(got, ref) < 1e-5, (case, pos, t, _rel(got, ref))


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_state_dict_keys_match_the_reference(case):
    kwargs, fdim, _, positions, _, _ = co.CASES[case]
    for pos in positions:
        m = tx.TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
        mine = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
        assert mine == [str(k) for k in GOLD["keys_" + case]]


def test_creation_string_and_training_keys():
    m = tx.TransformerXvector(80, 10, training=False, extracted_embedding="near", **co.LAUNCHER)
    assert m.get_model_creation() == co.creation(co.LAUNCHER, 80, "near")
    mt = tx.TransformerXvector(80, 10, **co.LAUNCHER)   # training=True: no loss module, like the other blueprints
    assert list(mt.state_dict()) == list(m.state_dict())
    sd = dict(co.seeded_state_dict(GOLD["keys_launcher"], 11), **{"loss.weight": torch.zeros(10, 256)})
    res = mt.load_state_dict(sd, strict=False)
    assert res.unexpected_keys == ["loss.weight"] and not res.missing_keys


def test_unknown_transformer_params_are_kept():
    m = tx.TransformerXvector(80, 10, training=False, transformer_params={"rotary_value": False, "pos_enc_type": "rot_pos",
                                                                          "not_an_option": 3})
    assert m.transformer.p["rotary_value"] is False and m.transformer.p["not_an_option"] == 3


def test_subsampling_column_order_float64():
    # the reference flattens the conv output (B, C, T', F'') as c * F'' + f; ours is (B, T', F'', C) flattened as f * C + c
    C, Fq, D = 16, 5, 8
    rng = np.random.RandomState(0)
    conv = rng.standard_normal((3, C, 4, Fq))                       # (B, C, T', F'')
    w = rng.standard_normal((D, C * Fq))
    ref = np.einsum("btk,dk->btd", conv.transpose(0, 2, 1, 3).reshape(3, 4, C * Fq), w)
    mine = np.einsum("btk,dk->btd", conv.transpose(0, 2, 3, 1).reshape(3, 4, Fq * C), w[:, tx.subsampling_column_order(C, Fq)])
    np.testing.assert_allclose(mine, ref, rtol=0, atol=1e-12)


def test_qkv_concatenation_float64():
    m = _model("small", "near")
    a = m.transformer.encoders[0].self_attn
    x = torch.randn(5, 128, dtype=torch.float64)
    w = torch.cat([a.linear_q.weight, a.linear_k.weight, a.linear_v.weight]).double()
    b = torch.cat([a.linear_q.bias, a.linear_k.bias, a.linear_v.bias]).double()
    y = x @ w.T + b
    for i, lin in enumerate((a.linear_q, a.linear_k, a.linear_v)):
        assert torch.equal(y[:, 128 * i:128 * (i + 1)], x @ lin.weight.double().T + lin.bias.double())


def test_conv_weight_transpose_matches_conv2d_float64():
    # (C, C, kt, kf) as stored -> (C, C, kf, kt) for the kernel's tap = kf * 3 + kt; the reference convolves (B, 1, T, F)
    w = torch.randn(4, 4, 3, 3, dtype=torch.float64)
    x = torch.randn(1, 4, 9, 7, dtype=torch.float64)                 # (B, C, T, F)
    ref = torch.nn.functional.conv2d(x, w, stride=2)
    wt = w.transpose(2, 3)
    mine = torch.nn.functional.conv2d(x.transpose(2, 3), wt, stride=2).transpose(2, 3)
    assert torch.allclose(mine, ref, rtol=0, atol=1e-12)


@pytest.mark.parametrize("frames", [7, 299, 300, 301, 599, 600, 650, 899, 29999, 100000])
def test_chunk_plan_matches_the_reference_loop(frames):
    lengths, offsets = tx.chunk_plan(frames)
    num_split = (frames + 299) // 300
    split = frames // num_split
    assert lengths == [split] * (num_split - 1) + [frames - split * (num_split - 1)]
    assert offsets == [i * split for i in range(num_split)]
    assert sum(lengths) == frames and lengths == co.chunk_plan(frames)[0]


def test_chunk_plan_worst_case_lengths():
    assert tx.chunk_plan(29999)[0][-1] == 398 and ((398 - 1) // 2 - 1) // 2 == 98
    assert max(((tx.chunk_plan(t)[0][-1] - 1) // 2 - 1) // 2 for t in (100000, 200000)) <= 240


def test_softmax_plus_multiplier_is_the_reference_expression():
    tl = torch.tensor(5.3)
    for t in (1, 74, 98, 240):
        s = torch.ones(1, 1, t)
        mask = (s > -1e4).float()
        ln = torch.sum(mask, dim=-1, keepdim=True).clamp_(1.)
        ref = (torch.log(ln) / tl * mask + 1 - mask)[0, 0, 0]
        assert np.float32(tx.softmax_plus_multiplier(t, tl)) == ref.numpy()


def test_rotary_table_is_the_reference_table():
    abs_rope = co._sin_table(64)
    assert torch.equal(tx.rotary_table(64)[:, :32], abs_rope[:, 0::2])
    assert torch.equal(tx.rotary_table(64)[:, 32:], abs_rope[:, 1::2])
    assert torch.equal(tx.sinusoid_table(256), co._sin_table(256))


def test_short_input_raises():
    m = _model("small", "near")
    with pytest.raises(ValueError, match="at least 7 frames"):
        m.extract_embedding(np.zeros((6, 23), np.float32))
    with pytest.raises(ValueError, match="at least 7 frames"):
        m.extract_embedding_batch(np.zeros((2, 6, 23), np.float32))


def test_far_without_fc1_raises():
    m = _model("launcher", "far")
    with pytest.raises(ValueError, match="fc1"):
        m.build_extractor()


UNSUPPORTED = [
    ({"transformer_type": "transformer"}, "transformer_type"),
    ({"transformer_type": "re_conformer"}, "transformer_type"),
    ({"transformer_params": {"att_type": "gau"}}, "att_type"),
    ({"transformer_params": {"pos_enc_type": "rel_pos"}}, "pos_enc_type"),
    ({"transformer_params": {"pos_enc_type": "rot_pos", "rope_abs_plus": True}}, "rope_abs_plus"),
    ({"transformer_params": {"add_t5rel_bias": True}}, "add_t5rel_bias"),
    ({"transformer_params": {"attention_conv_out": True}}, "attention_conv_out"),
    ({"transformer_params": {"attention_norm_args": {"norm_method": "relu_plus"}}}, "norm_method"),
    ({"transformer_params": {"attention_norm_args": {"scale_adapt": True}}}, "scale_adapt"),
    ({"transformer_params": {"attention_norm_args": {"g_sa": True}}}, "g_sa"),
    ({"transformer_params": {"attention_norm_args": {"diag_mask": True}}}, "diag_mask"),
    ({"transformer_params": {"input_layer": "conv2d6"}}, "input_layer"),
    ({"transformer_params": {"input_layer": "linear"}}, "input_layer"),
    ({"transformer_params": {"mlp_head": True}}, "mlp_head"),
    ({"transformer_params": {"combiner_type": "mfa"}}, "combiner_type"),
    ({"transformer_params": {"combiner_type": "random_frame"}}, "combiner_type"),
    ({"transformer_params": {"convfnn_blocks": 1}}, "convfnn_blocks"),
    ({"transformer_params": {"macaron_style": False}}, "macaron_style"),
    ({"transformer_params": {"use_cnn_module": False}}, "use_cnn_module"),
    ({"transformer_params": {"causal": True}}, "causal"),
    ({"transformer_params": {"normalize_before": False}}, "normalize_before"),
    ({"transformer_params": {"concat_after": True}}, "concat_after"),
    ({"transformer_params": {"norm_type": "batch_norm"}}, "norm_type"),
    ({"transformer_params": {"norm_type": "basic_norm"}}, "norm_type"),
    ({"transformer_params": {"static_chunk_size": 16}}, "static_chunk_size"),
    ({"transformer_params": {"use_dynamic_chunk": True}}, "use_dynamic_chunk"),
    ({"transformer_params": {"activation_balancer": True}}, "activation_balancer"),
    ({"transformer_params": {"re_scale": True}}, "re_scale"),
    ({"transformer_params": {"positionwise_layer_type": "conv1d"}}, "positionwise_layer_type"),
    ({"transformer_params": {"activation_type": "double_swish"}}, "activation_type"),
    ({"transformer_params": {"cnn_module_norm": "basic_norm"}}, "cnn_module_norm"),
    ({"pooling_params": {"time_attention": True}}, "time_attention"),
    ({"pooling_params": {"stddev": False}}, "stddev"),
    ({"tansformer_out": {"bn-relu": True}}, "bn-relu"),
]


@pytest.mark.parametrize("override,name", UNSUPPORTED, ids=[n for _, n in UNSUPPORTED])
def test_unsupported_options_raise(override, name):
    kwargs = dict(co.SMALL)
    for k, v in override.items():
        kwargs[k] = dict(kwargs.get(k, {}), **v) if isinstance(v, dict) else v
    with pytest.raises(NotImplementedError, match=name):
        tx.TransformerXvector(23, 10, training=False, **kwargs)
