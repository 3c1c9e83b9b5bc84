"""CPU checks of the CAM++ blueprint (asv_subtools_b200/model/campplus_xvector.py): the torch restatement against the
reference's golden embeddings, the state_dict layout, CamPPModel checkpoints, the chunk plan, the hand-over folds and
the im2col order of the strided tdnn in float64, and the inputs that must raise."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import campplus_oracle as co  # noqa: E402
from asv_subtools_b200.model import campplus_xvector as cx  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "campplus.npz"))


def rel(a, b):
    return float(np.max(np.abs(np.asarray(a) - np.asarray(b))) / np.max(np.abs(np.asarray(b))))


def _model(case):
    cfg = dict(co.CASES[case][0])
    return cx.CamPPXvector(cfg.pop("inputs_dim"), 10, **cfg)


def _keys(module):
    return np.array(["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in module.state_dict().items()])


GOLDEN_CASES = [(case, t) for case, (_, frames, long_frames, _, _) in co.CASES.items() for t in frames + long_frames]


@pytest.mark.parametrize("case,t", GOLDEN_CASES)
def test_oracle_replays_golden(case, t):
    cfg, frames, _, seed, fseed = co.CASES[case]
    sd = co.seeded_state_dict(GOLDEN["keys_" + case], seed)
    feats = co.utterances(2, t, cfg["inputs_dim"], fseed + t)
    with torch.no_grad():
        got = (co.forward(sd, feats) if t in frames else co.extract_embedding(sd, feats)).numpy()
    assert rel(got, GOLDEN["{}_T{}".format(case, t)]) <= 1e-5


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_state_dict_layout_equals_reference(case):
    assert list(_keys(_model(case))) == list(GOLDEN["keys_" + case])


def test_campplus_model_state_dict_loads_and_empty_dict_is_refused():
    m = _model("small")
    sd = co.seeded_state_dict(GOLDEN["model_keys_small"], 5)
    assert any(k.startswith("cam.") for k in sd) and any(k.startswith("classifier.") for k in sd)
    m.load_state_dict(sd, strict=True)
    key = "xvector.block2.tdnnd3.cam_layer.linear1.weight"
    assert torch.equal(m.state_dict()[key], sd["cam." + key])
    for bad in ({"classifier.weight": sd["classifier.weight"]}, {"state_dict": sd, "epoch": 3}, {}):
        with pytest.raises(KeyError):
            m.load_state_dict(bad, strict=False)


def test_chunk_plan_equals_split_chunks():
    for t, sizes in zip(GOLDEN["split_T"], GOLDEN["split_sizes"]):
        assert cx.chunk_sizes(int(t)) == [int(s) for s in sizes if s] == co.chunk_sizes(int(t))
    assert cx.chunk_sizes(9000) == [4000, 2500, 2500] and cx.chunk_sizes(4001) == [2001, 2000]


@pytest.mark.parametrize("T", [11, 12])
def test_tdnn_im2col_order_and_fold_in_float64(T):
    """The (B, T, F'', C) head output, flattened per frame as f * C + c and padded by 2 zero frames, read as 5-frame
    windows every 2 frames against the permuted, BN-folded weight equals relu(BN(Conv1d(k=5, stride=2, padding=2))) on
    the reference's c * F'' + f channel order."""
    g = torch.Generator().manual_seed(T)
    B, C, F8, O = 2, cx.M_CHANNELS, 3, 16
    x = torch.randn(B, T, F8, C, generator=g, dtype=torch.float64)
    w = torch.randn(O, C * F8, 5, generator=g, dtype=torch.float64)
    b = torch.randn(O, generator=g, dtype=torch.float64)
    bn = torch.nn.BatchNorm1d(O).double().eval()
    bn.running_mean.normal_(generator=g)
    bn.running_var.uniform_(0.5, 1.5, generator=g)
    bn.weight.data.normal_(1.0, 0.1, generator=g)
    bn.bias.data.normal_(generator=g)
    ref = F.relu(bn(F.conv1d(x.permute(0, 3, 2, 1).reshape(B, C * F8, T), w, b, stride=2, padding=2)))   # (B, O, T')
    w2, b2 = cx._fold(cx.tdnn_im2col_weight(w, C, F8), bn, b)
    pad = F.pad(x.reshape(B, T, F8 * C), (0, 0, 2, 2))
    T2 = (T + 1) // 2
    win = pad.reshape(B, -1).as_strided((B, T2, 5 * F8 * C), ((T + 4) * F8 * C, 2 * F8 * C, 1))
    got = F.relu(win @ w2.double().T + b2.double())
    assert torch.allclose(got.transpose(1, 2), ref, rtol=1e-5, atol=1e-5)   # the fold itself is fp32


def test_fold_into_linear1_in_float64():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 40, 9, generator=g, dtype=torch.float64)
    w = torch.randn(16, 40, 1, generator=g, dtype=torch.float64)
    bn = torch.nn.BatchNorm1d(16).double().eval()
    bn.running_mean.normal_(generator=g)
    bn.running_var.uniform_(0.5, 1.5, generator=g)
    w2, b2 = cx._fold(w, bn)
    ref = F.relu(bn(F.conv1d(x, w)))
    got = F.relu(F.conv1d(x, w2.double(), b2.double()))
    assert torch.allclose(got, ref, rtol=1e-5, atol=1e-6)


def test_invalid_inputs_raise():
    m = _model("small")
    with pytest.raises(ValueError):
        m.extract_embedding_batch(torch.zeros(1, 2, 40))
    with pytest.raises(ValueError):
        m.extract_embedding_batch(torch.zeros(1, 50, 32))
    with pytest.raises(ValueError):
        cx.CamPPXvector(36, 10)
    with pytest.raises(NotImplementedError, match="growth_rate"):
        cx.CamPPXvector(80, 10, growth_rate=12)
    with pytest.raises(NotImplementedError, match="init_channels"):
        cx.CamPPXvector(80, 10, init_channels=100)
