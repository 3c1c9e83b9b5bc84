"""ResNet x-vector blueprint on the CPU: the oracle replays the reference's golden embeddings, the blueprint's state_dict
layout equals the reference's, unsupported options raise, and the pooling-order column permutation equals the
reference's reshape."""
import numpy as np
import pytest
import torch

import resnet_oracle as ro
from asv_subtools_b200.model.resnet_xvector import ResNetXvector, _stats_column_order
from oracle import nnet as onn

# pytorch/launcher/runResnetXvector_online.py:221-275 as the launcher writes it into nnet.config, rewritten for extraction
ONLINE_CREATION = (
    'ResNetXvector(80,1211,aug_dropout=0.0,tail_dropout=0.0,training=False,extracted_embedding="near",'
    'resnet_params={"head_conv":True,"head_conv_params":{"kernel_size":3,"stride":1,"padding":1},"head_maxpool":False,'
    '"head_maxpool_params":{"kernel_size":3,"stride":2,"padding":1},"block":"BasicBlock","layers":[3,4,6,3],'
    '"planes":[32,64,128,256],"use_se":True,"se_ratio":4,"convXd":2,"norm_layer_params":{"momentum":0.5,"affine":True},'
    '"full_pre_activation":False,"zero_init_residual":False},pooling="statistics",pooling_params={"num_head":16,'
    '"share":True,"affine_layers":1,"hidden_size":64,"context":[0],"stddev":True,"temperature":False,"fixed":True},'
    'fc1=False,fc1_params={"nonlinearity":"relu","nonlinearity_params":{"inplace":True},"bn-relu":False,"bn":True,'
    '"bn_params":{"momentum":0.5,"affine":False,"track_running_stats":True}},fc2_params={"nonlinearity":"",'
    '"nonlinearity_params":{"inplace":True},"bn-relu":False,"bn":True,"bn_params":{"momentum":0.5,"affine":False,'
    '"track_running_stats":True}},margin_loss=True,margin_loss_params={"method":"am","m":0.2,"feature_normalize":True,'
    '"s":30,"mhe_loss":False,"mhe_w":0.01},use_step=True,step_params={"margin_warm":False,"margin_warm_conf":'
    '{"start_epoch":1,"end_epoch":1,"offset_margin":-0.0,"init_lambda":1.0},"T":None,"m":True,"lambda_0":0,'
    '"lambda_b":1000,"alpha":5,"gamma":1e-4,"s":False,"s_tuple":(30,12),"s_list":None,"t":False,"t_tuple":(0.5,1.2),'
    '"p":False,"p_tuple":(0.5,0.1)})')


def rel(a, b):
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_oracle_replays_reference_golden(golden, case):
    g = golden("resnet")
    kwargs, fdim, frames, positions, seed, fseed = ro.CASES[case]
    sd = onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed)
    for pos in positions:
        for t in frames:
            feats = onn.synthetic_feats(2, t, fdim, fseed + t)
            with torch.no_grad():
                got = ro.resnet_forward(sd, torch.from_numpy(feats).transpose(1, 2), pos, kwargs).squeeze(2).numpy()
            assert rel(got, g["{}_{}_T{}".format(case, pos, t)]) < 1e-5, (case, pos, t)


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_blueprint_state_dict_equals_reference_layout(golden, case):
    kwargs, fdim, _, positions, seed, _ = ro.CASES[case]
    ref = list(golden("resnet")["keys_" + case])
    m = ResNetXvector(fdim, 10, training=False, extracted_embedding=positions[0], **kwargs)
    assert ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()] == ref
    assert [(k, tuple(s)) for k, s, _ in ro.resnet_spec(fdim, kwargs)] == \
        [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed), strict=True)
    assert m.get_model_creation() == ro.creation(kwargs, fdim, positions[0])


def test_online_launcher_creation_string_builds_and_loads():
    from asv_subtools_b200.pipeline.extract_embeddings import create_model_from_py
    import os
    bp = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "asv_subtools_b200", "model",
                      "resnet_xvector.py")
    m = create_model_from_py(bp, ONLINE_CREATION)
    assert m.get_model_creation().startswith("ResNetXvector(80,1211,aug_dropout=0.0,")
    assert m.extracted_embedding == "near" and m.fc1 is None and not m.fc2.relu and m.fc2.batchnorm.weight is None
    sd = onn.make_state_dict(ro.resnet_spec(80, ro.ONLINE), 301)
    ck = dict(sd, **{"loss.weight": torch.zeros(1211, 256, 1)})   # training checkpoints carry loss.* keys
    m.load_state_dict(ck, strict=False)
    with pytest.raises(RuntimeError):                              # no CPU path
        m.extract_embedding(onn.synthetic_feats(1, 10, 80, 0)[0])


@pytest.mark.parametrize("kwargs, exc, word", [
    (dict(resnet_params={"block": "Bottleneck"}), NotImplementedError, "Bottleneck"),
    (dict(resnet_params={"convXd": 1}), NotImplementedError, "convXd"),
    (dict(resnet_params={"head_maxpool": True}), NotImplementedError, "head_maxpool"),
    (dict(resnet_params={"head_conv": False}), NotImplementedError, "head_conv"),
    (dict(resnet_params={"head_conv_params": {"kernel_size": 3, "stride": 2, "padding": 1}}), NotImplementedError,
     "head_conv_params"),
    (dict(resnet_params={"replace_stride_with_dilation": [False, True, True]}), NotImplementedError, "dilation"),
    (dict(cmvn=True), NotImplementedError, "cmvn"),
    (dict(pooling="attentive"), NotImplementedError, "attentive"),
    (dict(pooling="lde"), NotImplementedError, "lde"),
    (dict(pooling="multi-head"), NotImplementedError, "multi-head"),
    (dict(resnet_params={"planes": [24, 48, 96, 192]}), ValueError, "multiple of 16"),
])
def test_unsupported_options_raise(kwargs, exc, word):
    with pytest.raises(exc, match=word):
        ResNetXvector(80, 10, training=False, **kwargs)


def test_far_without_fc1_raises_a_clear_error():
    m = ResNetXvector(80, 10, training=False, extracted_embedding="far")
    with pytest.raises(ValueError, match="fc1"):
        m.build_extractor()


def test_accepts_training_keywords_and_resnet18():
    m = ResNetXvector(40, 10, aug_dropout=0.2, tail_dropout=0.1, margin_loss=True, use_step=True, jit_compile=True,
                      resnet_params={"layers": [2, 2, 2, 2]})
    assert len(m.resnet.blocks()) == 8 and m.stats.get_output_dim() == 2 * 5 * 256


@pytest.mark.parametrize("c, f, t", [(256, 10, 25), (32, 3, 1), (64, 12, 7)])
def test_pooling_column_permutation_equals_reference_reshape(c, f, t):
    """Frames kept as (B, T', F', C) and pooled over (B, T', F'*C), followed by the first segment layer with permuted
    columns, equal the reference's reshape (B, C*F', T') -> statistics pooling -> the layer (resnet_xvector.py:193)."""
    torch.manual_seed(0)
    x = torch.randn(3, c, f, t, dtype=torch.float64)               # the reference's (B, C, F', T')
    w = torch.randn(16, 2 * c * f, dtype=torch.float64)
    ref = onn.statistics_pooling(x.reshape(3, c * f, t)).squeeze(2) @ w.T
    ours_frames = x.permute(0, 3, 2, 1).reshape(3, t, f * c)          # (B, T', F'*C), column f*C + c
    mean = ours_frames.mean(1)
    std = torch.sqrt(((ours_frames - mean[:, None]) ** 2).mean(1).clamp(min=1e-10))
    got = torch.cat([mean, std], 1) @ w[:, torch.from_numpy(_stats_column_order(c, f))].T
    assert torch.allclose(got, ref, rtol=1e-12, atol=1e-12)
