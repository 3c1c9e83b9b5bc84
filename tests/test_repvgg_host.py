"""RepVGG / RepSPK x-vector blueprint on the CPU: the oracle replays the reference's golden embeddings in both forms,
the blueprint's state_dict layout equals the reference's in both forms, the hand-over fold equals the three-branch
block in float64, tap pruning keeps the right taps, unsupported options raise, and auto_model equals the reference's
table."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import repvgg_oracle as ro
from asv_subtools_b200.model.repvgg_xvector import RepVggXvector, auto_model, fold_block, kept_taps
from oracle import nnet as onn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# pytorch/launcher/runRepvggXvector.py:219-278 as the launcher writes it into nnet.config, rewritten for extraction
LAUNCHER_CREATION = (
    'RepVggXvector(80,1211,aug_dropout=0.0,tail_dropout=0.0,training=False,extracted_embedding="near",deploy=False,'
    'embd_dim=256,repvgg_config={"auto_model":False,"auto_model_name":"RepVGG_A1","block":"RepSPK","repvgg_params":'
    '{"num_blocks":[2,4,14,1],"strides":[1,1,2,2,2],"base_width":32,"width_multiplier":[1,1,1,2.5],'
    '"override_groups_map":None,"use_se":False,"norm_layer_params":{"momentum":0.5,"affine":True}}},'
    'pooling="statistics",pooling_params={"num_head":1,"share":True,"affine_layers":1,"hidden_size":64,"context":[0],'
    '"stddev":True,"temperature":False,"fixed":True},fc1=False,fc1_params={"nonlinearity":"relu","nonlinearity_params":'
    '{"inplace":True},"bn-relu":False,"bn":True,"bn_params":{"momentum":0.5,"affine":False,"track_running_stats":True}},'
    'fc2_params={"nonlinearity":"","nonlinearity_params":{"inplace":True},"bn-relu":False,"bn":True,"bn_params":'
    '{"momentum":0.5,"affine":False,"track_running_stats":True}},margin_loss=True,margin_loss_params={"method":"am",'
    '"m":0.2,"feature_normalize":True,"s":30,"mhe_loss":False,"mhe_w":0.01},use_step=True,step_params={"margin_warm":'
    'False,"margin_warm_conf":{"start_epoch":1,"end_epoch":1,"offset_margin":-0.0,"init_lambda":1.0},"T":None,"m":True,'
    '"lambda_0":0,"lambda_b":1000,"alpha":5,"gamma":1e-4,"s":False,"s_tuple":(30,12),"s_list":None,"t":False,'
    '"t_tuple":(0.5,1.2),"p":False,"p_tuple":(0.5,0.1)})')
RING = [(0, 1), (0, 3), (1, 0), (1, 4), (3, 0), (3, 4), (4, 1), (4, 3)]   # the RepSPK taps that are always zero


def rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _replay(g, sd, kwargs, case, tag, positions, frames, fdim, fseed):
    for pos in positions:
        for t in frames:
            feats = onn.synthetic_feats(2, t, fdim, fseed + t)
            with torch.no_grad():
                got = ro.repvgg_forward(sd, torch.from_numpy(feats).transpose(1, 2), pos, kwargs).squeeze(2).numpy()
            assert rel(got, g["{}_{}_T{}".format(tag, pos, t)]) < 1e-5, (case, pos, t)


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_oracle_replays_reference_golden(golden, case):
    kwargs, fdim, frames, positions, seed, fseed = ro.CASES[case]
    sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
    _replay(golden("repvgg"), sd, kwargs, case, case, positions, frames, fdim, fseed)


def test_oracle_replays_reference_golden_deploy_form(golden):
    """The reference's repvgg_model_convert, restated in its fp32 order, then the deploy-form forward."""
    kwargs, fdim, frames, positions, seed, fseed = ro.CASES[ro.DEPLOY_CASE]
    dsd = ro.deploy_state_dict(onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed), kwargs)
    assert [(k, tuple(v.shape)) for k, v in dsd.items()] == [(k, s) for k, s, _ in ro.repvgg_spec(fdim, kwargs, deploy=True)]
    _replay(golden("repvgg"), dsd, kwargs, ro.DEPLOY_CASE, ro.DEPLOY_CASE + "_deploy", positions, frames, fdim, fseed)


@pytest.mark.parametrize("case, deploy", [(c, False) for c in sorted(ro.CASES)] + [(ro.DEPLOY_CASE, True)])
def test_blueprint_state_dict_equals_reference_layout(golden, case, deploy):
    kwargs, fdim, _, positions, seed, _ = ro.CASES[case]
    ref = list(golden("repvgg")["keys_" + case + ("_deploy" if deploy else "")])
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding=positions[0], **({"deploy": True} if deploy else {}),
                      **kwargs)
    assert ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()] == ref
    spec = ro.repvgg_spec(fdim, kwargs, deploy=deploy)
    assert [(k, tuple(s)) for k, s, _ in spec] == [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
    m.load_state_dict(ro.deploy_state_dict(sd, kwargs) if deploy else sd, strict=True)
    assert m.get_model_creation() == ro.creation(kwargs, fdim, positions[0], deploy=deploy)


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_fold_equals_three_branch_block_in_float64(case):
    """fold_block (the hand-over) against the block's three-branch forward, every block, float64."""
    kwargs, fdim, _, positions, seed, _ = ro.CASES[case]
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding=positions[0], **kwargs)
    sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
    m.load_state_dict(sd, strict=True)
    sd64 = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    spk = ro._config(kwargs)["spk"]
    g = torch.Generator().manual_seed(seed)
    for (pre, cin, cout, stride, groups), blk in zip(ro._config(kwargs)["blocks"], m.repvgg.blocks()):
        x = torch.randn(2, cin, 11, 9, generator=g, dtype=torch.float64)
        w, b = fold_block(blk)
        assert w.dtype == torch.float64 and tuple(w.shape) == (cout, cin, blk.window, blk.window)
        got = F.relu(F.conv2d(x, w, b, stride=stride, padding=blk.window // 2))
        ref = ro.block_forward(x, sd64, pre, stride, groups, spk)
        assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12), pre


def test_fold_of_deploy_form_equals_fold_of_training_form():
    kwargs, fdim, _, positions, seed, _ = ro.CASES["grouped"]
    sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
    tr = RepVggXvector(fdim, 10, training=False, **kwargs)
    tr.load_state_dict(sd, strict=True)
    de = RepVggXvector(fdim, 10, training=False, deploy=True, **kwargs)
    de.load_state_dict(ro.deploy_state_dict(sd, kwargs), strict=True)
    for a, b in zip(tr.repvgg.blocks(), de.repvgg.blocks()):
        (wa, ba), (wb, bb) = fold_block(a), fold_block(b)
        assert torch.allclose(wa, wb, rtol=1e-6, atol=1e-6) and torch.allclose(ba, bb, rtol=1e-6, atol=1e-6)


def test_tap_pruning_keeps_17_repspk_taps_and_9_repvgg_taps():
    for case, k, expect in (("repspk", 5, ro.REPSPK_TAPS), ("a0", 3, list(range(9))), ("grouped", 5, ro.REPSPK_TAPS)):
        kwargs, fdim, _, _, seed, _ = ro.CASES[case]
        m = RepVggXvector(fdim, 10, training=False, **kwargs)
        m.load_state_dict(onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed), strict=True)
        for blk in m.repvgg.blocks()[1:]:
            assert kept_taps(fold_block(blk)[0].float()) == expect, (case, blk)
    assert sorted(set(range(25)) - set(ro.REPSPK_TAPS)) == sorted(kf * 5 + kt for kf, kt in RING)


def test_tap_pruning_keeps_nonzero_off_pattern_taps_of_a_deploy_file():
    """A deploy checkpoint whose off-pattern taps are not zero keeps them: the result is the dense 5x5 conv."""
    kwargs, fdim, _, _, seed, _ = ro.CASES["repspk"]
    dsd = ro.deploy_state_dict(onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed), kwargs)
    key = "repvgg.stage3.2.rbr_reparam.weight"
    dsd[key] = dsd[key].clone()
    dsd[key][5, 7, 0, 1] = 0.25
    m = RepVggXvector(fdim, 10, training=False, deploy=True, **kwargs)
    m.load_state_dict(dsd, strict=True)
    assert kept_taps(fold_block(m.repvgg.stage3[2])[0].float()) == sorted(ro.REPSPK_TAPS + [1])
    assert kept_taps(fold_block(m.repvgg.stage3[1])[0].float()) == ro.REPSPK_TAPS


def test_launcher_creation_string_builds_and_loads():
    from asv_subtools_b200.pipeline.extract_embeddings import create_model_from_py
    bp = os.path.join(ROOT, "asv_subtools_b200", "model", "repvgg_xvector.py")
    m = create_model_from_py(bp, LAUNCHER_CREATION)
    assert m.get_model_creation().startswith("RepVggXvector(80,1211,aug_dropout=0.0,")
    assert m.extracted_embedding == "near" and m.fc1 is None and not m.fc2.relu and m.fc2.batchnorm.weight is None
    sd = onn.make_state_dict(ro.repvgg_spec(80, ro.LAUNCHER), 401)
    ck = dict(sd, **{"loss.weight": torch.zeros(1211, 256, 1)})   # training checkpoints carry loss.* keys
    m.load_state_dict(ck, strict=False)
    with pytest.raises(RuntimeError):                              # no CPU path
        m.extract_embedding(onn.synthetic_feats(1, 10, 80, 0)[0])


def _rp(**over):
    p = {"num_blocks": [1, 1, 1, 1], "strides": [1, 1, 2, 2, 2], "base_width": 64, "width_multiplier": [0.5, 0.5, 0.5, 0.5],
         "override_groups_map": None, "use_se": False, "norm_layer_params": {"momentum": 0.5, "affine": True}}
    p.update(over)
    return {"repvgg_config": {"block": "RepSPK", "repvgg_params": p}}


@pytest.mark.parametrize("kwargs, exc, word", [
    (_rp(use_se=True), NotImplementedError, "use_se"),
    (dict(repvgg_config={"auto_model": True, "auto_model_name": "RepVGG_D2se"}), NotImplementedError, "use_se"),
    (dict(pooling="attentive"), NotImplementedError, "attentive"),
    (dict(pooling="lde"), NotImplementedError, "lde"),
    (dict(pooling="multi-head"), NotImplementedError, "multi-head"),
    (dict(pooling_params={"stddev": False}), NotImplementedError, "stddev"),
    (_rp(strides=[1, 1, 3, 2, 2]), NotImplementedError, "strides"),
    (_rp(strides=[2, 1, 2, 2, 2]), NotImplementedError, "strides"),
    (_rp(width_multiplier=[0.5, 0.5, 0.5, 0.3]), ValueError, "multiple of 16"),
    (dict(repvgg_config={"block": "RepVGGPlus"}), TypeError, "RepVGGPlus"),
])
def test_unsupported_options_raise(kwargs, exc, word):
    with pytest.raises(exc, match=word):
        RepVggXvector(80, 10, training=False, **kwargs)


def test_far_without_fc1_raises_a_clear_error():
    m = RepVggXvector(80, 10, training=False, extracted_embedding="far")
    with pytest.raises(ValueError, match="fc1"):
        m.build_extractor()


def test_accepts_training_keywords():
    m = RepVggXvector(40, 10, aug_dropout=0.2, tail_dropout=0.1, margin_loss=True, use_step=True, adacos=True,
                      transfer_from="softmax_loss", repvgg_config={"block": "RepVGG"})
    assert len(m.repvgg.blocks()) == 22 and m.stats.get_output_dim() == 2 * 5 * 640


def test_auto_model_table_equals_reference(golden):
    ref = json.loads(str(golden("repvgg")["auto_model_json"]))
    ours = json.loads(json.dumps({n: auto_model(n) for n in ref}, sort_keys=True))
    assert ours == ref
    with pytest.raises(KeyError):
        auto_model("RepVGG_Z9")
