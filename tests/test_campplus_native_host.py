"""The records the native CAM++ extractor receives (xvb_campp_set_layer) and its chunk plan, on the CPU: every backbone
state_dict tensor carried by exactly one record, the tdnn / transit3 / dense folds in float64, and xvb_campp_chunk_sizes
(host only) against the reference's split_chunks sizes and the Python chunk rule."""
import ctypes as C
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
from asv_subtools_b200 import _lib  # noqa: E402
from asv_subtools_b200.model import campplus_xvector as cx  # noqa: E402

GOLDEN = np.load(os.path.join(HERE, "golden", "campplus.npz"))


def _model(case):
    cfg, _, _, seed, _ = co.CASES[case]
    kw = dict(cfg)
    m = cx.CamPPXvector(kw.pop("inputs_dim"), 10, **kw)
    keys = ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in m.state_dict().items()]
    m.load_state_dict(co.seeded_state_dict(keys, seed), strict=True)
    return m.eval()


def _records(m):
    return {r[0]: r for r in cx.native_records(m)}


def _bn64(sd, p, x, dim):
    """Eval BatchNorm over axis `dim` of x in float64 from the state_dict entries under prefix p."""
    shape = [1] * x.dim()
    shape[dim] = -1
    v = lambda k: sd[p + k].double().view(shape)  # noqa: E731
    y = (x - v("running_mean")) / torch.sqrt(v("running_var") + 1e-5)
    if p + "weight" in sd:
        y = y * v("weight") + v("bias")
    return y


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_records_carry_every_state_dict_tensor_once(case):
    m = _model(case)
    recs = cx.native_records(m)
    names = [r[0] for r in recs]
    assert len(names) == len(set(names))
    keys = [k for r in recs for k in r[6]]
    assert len(keys) == len(set(keys))
    assert sorted(keys) == sorted(m.state_dict())
    cfg = cx.native_config(m)
    assert cfg == dict(feat_dim=co.CASES[case][0]["inputs_dim"], embd_dim=co.CASES[case][0]["embd_dim"],
                       init_channels=co.CASES[case][0]["init_channels"], growth_rate=co.CASES[case][0]["growth_rate"],
                       bn_size=co.CASES[case][0]["bn_size"])
    for name, w, b, s, t, flags, _ in recs:
        assert w is not None or s is not None, name
        for a in (w, b, s, t):
            assert a is None or (a.dtype == np.float32 and np.all(np.isfinite(a))), name


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_tdnn_record_is_conv_bn_folded_and_permuted_float64(case):
    """The record's weight applied to the 5-frame im2col windows of the (T, F'', C) head output equals Conv1d(k = 5,
    stride 2, padding 2) -> BatchNorm -> over channels c * F'' + f, in float64."""
    m = _model(case)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    _, w, b, _, _, flags, _ = _records(m)["xvector.tdnn.linear"]
    assert flags == _lib.RELU
    f8, c = m.inputs_dim // 8, cx.M_CHANNELS
    T = 9
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, T, f8, c, generator=g, dtype=torch.float64)               # the head output, (B, T, F'', C)
    xin = x.permute(0, 3, 2, 1).reshape(1, c * f8, T)                            # channel c * F'' + f
    ref = _bn64(sd, "xvector.tdnn.nonlinear.0.",
                F.conv1d(xin, sd["xvector.tdnn.linear.weight"].double(), sd["xvector.tdnn.linear.bias"].double(), stride=2,
                         padding=2), 1).transpose(1, 2)[0]
    pad = F.pad(x.reshape(1, T, f8 * c), (0, 0, 2, 2))[0]                        # (T + 4, F'' * C)
    T2 = (T + 1) // 2
    win = torch.stack([pad[2 * t:2 * t + 5].reshape(-1) for t in range(T2)])     # row t: frames 2t .. 2t + 4
    got = win @ torch.from_numpy(w).double().T + torch.from_numpy(b).double()
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_transit3_and_dense_folds_float64(case):
    m = _model(case)
    sd = {k: v.detach() for k, v in m.state_dict().items()}
    recs = _records(m)
    g = torch.Generator().manual_seed(4)
    _, w, b, _, _, flags, _ = recs["xvector.transit3.linear"]
    assert flags == _lib.RELU
    x = torch.randn(w.shape[1], 7, generator=g, dtype=torch.float64)            # (C, T)
    ref = torch.relu(_bn64(sd, "xvector.out_nonlinear.batchnorm.", sd["xvector.transit3.linear.weight"].double()[:, :, 0] @ x, 0))
    got = torch.relu(torch.from_numpy(w).double() @ x + torch.from_numpy(b).double()[:, None])
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())
    _, w, b, s, t, flags, _ = recs["xvector.dense.linear"]
    assert flags == _lib.BN and b is None and w.shape == (m.embd_dim, w.shape[1])
    stats = torch.randn(w.shape[1], 3, generator=g, dtype=torch.float64)
    ref = _bn64(sd, "xvector.dense.nonlinear.1.", sd["xvector.dense.linear.weight"].double()[:, :, 0] @ stats, 0)
    got = (torch.from_numpy(w).double() @ stats) * torch.from_numpy(s).double()[:, None] + torch.from_numpy(t).double()[:, None]
    assert float((got - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


def _chunk_sizes(T, max_chunk, cap=64):
    out = (C.c_int * cap)()
    n = _lib.lib.xvb_campp_chunk_sizes(T, max_chunk, out, cap)
    return n, list(out)[:max(n, 0)]


def test_chunk_sizes_equal_reference_split_chunks():
    for t, sizes in zip(GOLDEN["split_T"], GOLDEN["split_sizes"]):
        n, got = _chunk_sizes(int(t), 4000)
        assert got == [int(s) for s in sizes if s], (t, got)


@pytest.mark.parametrize("max_chunk", [4000, 300, 7, 1])
def test_chunk_sizes_equal_python_rule(max_chunk):
    cap = 20001
    out = (C.c_int * cap)()
    for t in range(1, 20002):
        n = _lib.lib.xvb_campp_chunk_sizes(t, max_chunk, out, cap)
        want = cx.chunk_sizes(t, max_chunk)
        assert n == len(want) and out[:n] == want, (t, max_chunk)


def test_chunk_sizes_refuse_bad_arguments():
    """XVB_EINVAL (-1) when cap is too small, T < 1 or max_chunk < 1."""
    assert _chunk_sizes(9000, 4000, cap=2)[0] == -1
    assert "do not fit" in _lib.lib.xvb_last_error().decode()
    assert _chunk_sizes(9000, 4000, cap=3) == (3, [4000, 2500, 2500])
    assert _chunk_sizes(0, 4000)[0] == -1
    assert _chunk_sizes(5, 0)[0] == -1
