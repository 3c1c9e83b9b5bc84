"""GPU tests of the CAM++ path: the reference's golden embeddings through the blueprint, the new kernels against torch
(the (2, 1)-strided conv, the strided tdnn's im2col view, xvb_bn_relu_planes, xvb_cam_gate, xvb_seg_gate_apply), and
batch calls against per-utterance calls."""
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

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(HERE, "golden", "campplus.npz"))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


_MODELS = {}


def _model(case):
    if case not in _MODELS:
        from asv_subtools_b200.model.campplus_xvector import CamPPXvector
        cfg, _, _, seed, _ = co.CASES[case]
        kw = dict(cfg)
        m = CamPPXvector(kw.pop("inputs_dim"), 10, **kw)
        m.load_state_dict(co.seeded_state_dict(GOLDEN["keys_" + case], seed), strict=True)
        _MODELS[case] = m.cuda().eval()
    return _MODELS[case]


def _planes(x):
    from asv_subtools_b200 import ops
    return ops.split_f32(x.contiguous())


GOLDEN_CASES = [(case, t) for case, (_, frames, long_frames, _, _) in co.CASES.items() for t in frames + long_frames]


@pytest.mark.parametrize("case,t", GOLDEN_CASES)
def test_golden(case, t):
    cfg, _, _, _, fseed = co.CASES[case]
    m = _model(case)
    feats = co.utterances(2, t, cfg["inputs_dim"], fseed + t)
    ref = GOLDEN["{}_T{}".format(case, t)]
    got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
    cos = [float(np.dot(got[i], ref[i]) / np.linalg.norm(got[i]) / np.linalg.norm(ref[i])) for i in range(2)]
    print("campplus {} T={}: rel {:.3e}, cosine {}; launches {}".format(case, t, rel(got, ref), cos,
                                                                        m.extractor().last_launches))
    assert rel(got, ref) <= 1e-4 and min(cos) >= 1 - 1e-6


@pytest.mark.parametrize("T,Fd,ksize", [(37, 80, 3), (36, 41, 3), (50, 40, 1), (9, 11, 1)])
def test_conv_stride_2_1(T, Fd, ksize):
    from asv_subtools_b200 import ops
    g = torch.Generator().manual_seed(T * 100 + Fd)
    B, C = 3, 32
    x = torch.randn(B, T, Fd, C, generator=g).cuda()
    w = (torch.randn(C, C, ksize, ksize, generator=g) / (3.0 * ksize)).cuda()
    s, t = (1 + 0.1 * torch.randn(C, generator=g)).cuda(), (0.1 * torch.randn(C, generator=g)).cuda()
    xp = _planes(x)
    Fo = (Fd + 1) // 2
    y = ops.SplitPlanes.empty((B, T, Fo, C), x.device)
    ops.conv2d(xp, ops.pack_conv2d_weight(w), C, ksize, 2, s, t, relu=True, y=y, stride_t=1)
    xin = xp.float().double().permute(0, 3, 2, 1)                  # (B, C, F, T): the reference's layout
    ref = F.relu(F.conv2d(xin, w.double(), stride=(2, 1), padding=ksize // 2) * s.double().view(1, -1, 1, 1) +
                 t.double().view(1, -1, 1, 1)).permute(0, 3, 2, 1)
    assert tuple(ref.shape) == (B, T, Fo, C)
    assert rel(y.float().cpu(), ref.cpu()) <= 3e-5


@pytest.mark.parametrize("T", [37, 38])
def test_strided_tdnn_im2col(T):
    from asv_subtools_b200 import ops
    from asv_subtools_b200.model.campplus_xvector import tdnn_im2col_weight
    g = torch.Generator().manual_seed(T)
    B, C, F8, O = 3, 32, 10, 128
    row = C * F8
    x = torch.randn(B, T, F8, C, generator=g).cuda()
    w = (torch.randn(O, row, 5, generator=g) / 40.0).cuda()
    b = (0.1 * torch.randn(O, generator=g)).cuda()
    xp = _planes(x.reshape(B, T, row))
    pad = ops.SplitPlanes(torch.zeros(B, T + 4, row, dtype=torch.bfloat16, device="cuda"),
                          torch.zeros(B, T + 4, row, dtype=torch.bfloat16, device="cuda"), row)
    pad.hi[:, 2:T + 2] = xp.hi
    pad.lo[:, 2:T + 2] = xp.lo
    T2 = (T + 1) // 2
    win = ops.SplitPlanes(pad.hi.as_strided((B, T2, 2 * row), ((T + 4) * row, 2 * row, 1)),
                          pad.lo.as_strided((B, T2, 2 * row), ((T + 4) * row, 2 * row, 1)), 5 * row)
    wp = ops.pack_tdnn_weight(tdnn_im2col_weight(w, C, F8).unsqueeze(-1).contiguous(), [0])
    y = torch.empty(B, T2, O, dtype=torch.float32, device="cuda")
    ops.tdnn_affine_ex(win, wp, O, [0], bias=b, y_f32=y, x_batch_stride=(T + 4) * row)
    xin = xp.float().double().reshape(B, T, F8, C).permute(0, 3, 2, 1).reshape(B, C * F8, T)   # channel c * F'' + f
    ref = F.conv1d(xin, w.double(), b.double(), stride=2, padding=2).transpose(1, 2)
    assert rel(y.cpu(), ref.cpu()) <= 3e-5


def test_bn_relu_planes():
    from asv_subtools_b200 import ops
    g = torch.Generator().manual_seed(1)
    B, T, W, C = 2, 77, 1024, 424
    buf = _planes(torch.randn(B, T, W, generator=g).cuda())
    s, t = (1 + 0.2 * torch.randn(C, generator=g)).cuda(), (0.3 * torch.randn(C, generator=g)).cuda()
    out = ops.SplitPlanes(torch.full((B, T, W), 7.0, dtype=torch.bfloat16, device="cuda"),
                          torch.full((B, T, W), 7.0, dtype=torch.bfloat16, device="cuda"), W)
    ops.bn_relu_planes(buf.slice(0, C), s, t, out.slice(0, C))
    ref = torch.relu(buf.float()[..., :C].double() * s.double() + t.double())
    assert rel(out.float()[..., :C].cpu(), ref.cpu()) <= 1e-5
    assert bool((out.hi[..., C:] == 7.0).all()) and bool((out.lo[..., C:] == 7.0).all())


@pytest.mark.parametrize("T", [1, 99, 100, 101, 150, 2000])
def test_cam_gate(T):
    from asv_subtools_b200 import ops
    g = torch.Generator().manual_seed(T)
    B, C, R, G = 3, 128, 64, 32
    h = _planes(torch.relu(torch.randn(B, T, C, generator=g)).cuda())
    w1, b1 = torch.randn(R, C, generator=g) / 11.3, 0.1 * torch.randn(R, generator=g)
    w2, b2 = torch.randn(G, R, generator=g) / 8.0, 0.1 * torch.randn(G, generator=g)
    gate = ops.cam_gate(h, w1.cuda(), b1.cuda(), w2.cuda(), b2.cuda(), seg_len=100)
    x = h.float().double().cpu().transpose(1, 2)                   # (B, C, T)
    ctx = x.mean(-1, keepdim=True) + co.seg_pooling(x)
    m = torch.sigmoid(F.conv1d(torch.relu(F.conv1d(ctx, w1.double().unsqueeze(-1), b1.double())),
                               w2.double().unsqueeze(-1), b2.double()))            # (B, G, T)
    nseg = (T + 99) // 100
    assert tuple(gate.shape) == (B, nseg, G)
    ref = m[:, :, ::100].transpose(1, 2)
    assert float((gate.cpu().double() - ref).abs().max()) <= 2e-6


def test_seg_gate_apply_writes_only_its_slice():
    from asv_subtools_b200 import ops
    g = torch.Generator().manual_seed(2)
    B, T, W, G, c0 = 2, 150, 512, 32, 224
    z = _planes(torch.randn(B, T, G, generator=g).cuda())
    gate = torch.rand(B, 2, G, generator=g).cuda()
    buf = ops.SplitPlanes(torch.full((B, T, W), -3.0, dtype=torch.bfloat16, device="cuda"),
                          torch.full((B, T, W), 5.0, dtype=torch.bfloat16, device="cuda"), W)
    ops.seg_gate_apply(z, gate, 100, buf.slice(c0, c0 + G))
    seg = torch.arange(T, device="cuda") // 100
    ref = z.float() * gate[:, seg]
    assert rel(buf.float()[..., c0:c0 + G].cpu(), ref.cpu()) <= 1e-5
    assert bool((buf.hi[..., :c0] == -3.0).all() and (buf.hi[..., c0 + G:] == -3.0).all())
    assert bool((buf.lo[..., :c0] == 5.0).all() and (buf.lo[..., c0 + G:] == 5.0).all())


def test_batch_equals_single_utterance_calls():
    m = _model("default")
    feats = co.utterances(64, 300, 80, 77)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(64)])
    print("campplus batch vs single: rel {:.3e}".format(rel(batch, single)))
    assert np.array_equal(batch, single)


@pytest.mark.parametrize("t", [4001, 9000])
def test_multi_chunk_batch_equals_single_utterance_calls(t):
    m = _model("default")
    feats = co.utterances(3, t, 80, 31)
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(3)])
    print("campplus multi-chunk batch vs single (T={}): rel {:.3e}".format(t, rel(batch, single)))
    assert np.array_equal(batch, single)
