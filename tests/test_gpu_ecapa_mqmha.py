"""ECAPA-TDNN with multi-query multi-head attention pooling on the GPU: the layer kernel's grouped mode, the head-width
pooling map, the whole model (native handle and op-by-op twin) against the reference goldens, shard calls, XVBE0002
model files and bin/xvb-extract."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ecapa_mqmha_oracle as mo  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "ecapa_mqmha.npz"))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosine(a, b):
    a, b = np.asarray(a, dtype=np.float64).reshape(len(a), -1), np.asarray(b, dtype=np.float64).reshape(len(b), -1)
    return float(np.min(np.sum(a * b, 1) / np.linalg.norm(a, axis=1) / np.linalg.norm(b, axis=1)))


def _grouped(ops, x, w, G, bias=None, scale=None, shift=None, relu=False, tanh=False, groups=None):
    B, T, _ = x.shape
    cout = w.shape[0]
    y = torch.empty(B, T, cout, dtype=torch.float32, device="cuda")
    ops.tdnn_affine_ex(ops.split_f32(x), ops.pack_tdnn_weight(w, [0]), cout, [0], bias=bias, bn_scale=scale, bn_shift=shift,
                       relu=relu, tanh=tanh, y_f32=y, groups=G if groups is None else groups)
    return y


GROUPED_SHAPES = [(G, kg, ng) for G in (2, 4, 8) for kg in (64, 768) for ng in (32, 64, 128, 768) if G * kg <= 3072 and G * ng <= 3072]


@pytest.mark.parametrize("G,kg,ng", GROUPED_SHAPES)
def test_grouped_layer_matches_conv1d_groups(G, kg, ng):
    """Ragged B*T (B=3, T=45: tiles cut through utterances and the batch) through each epilogue."""
    from asv_subtools_b200 import ops
    rng = np.random.RandomState(G * 1000 + kg + ng)
    B, T, cin, cout = 3, 45, G * kg, G * ng
    x = torch.from_numpy(rng.standard_normal((B, T, cin)).astype(np.float32)).cuda()
    w = torch.from_numpy((rng.standard_normal((cout, kg, 1)) / np.sqrt(kg)).astype(np.float32)).cuda()
    b = torch.from_numpy((0.1 * rng.standard_normal(cout)).astype(np.float32)).cuda()
    s = torch.from_numpy(rng.uniform(0.5, 1.5, cout).astype(np.float32)).cuda()
    t = torch.from_numpy((0.1 * rng.standard_normal(cout)).astype(np.float32)).cuda()
    ref = F.conv1d(x.double().transpose(1, 2), w.double(), b.double(), groups=G).transpose(1, 2)
    bn = torch.relu(ref) * s.double() + t.double()
    for kw, want in ((dict(), ref), (dict(relu=True, scale=s, shift=t), bn)):
        got = _grouped(ops, x, w, G, bias=b, **kw)
        assert rel(got.cpu().numpy(), want.cpu().numpy()) <= 3e-5, (G, kg, ng, list(kw))
    # tanh is 1-Lipschitz: its error is bounded by the error of its argument, so it is measured on that argument's scale
    # (tanh's own outputs are at most 1, several times smaller than the BatchNorm outputs that the split operands'
    # relative accuracy applies to)
    got = _grouped(ops, x, w, G, bias=b, relu=True, scale=s, shift=t, tanh=True).double().cpu()
    err = float((got - torch.tanh(bn).cpu()).abs().max() / bn.abs().max().cpu())
    assert err <= 3e-5, (G, kg, ng, err)


@pytest.mark.parametrize("G,kg,ng", [(2, 768, 128), (4, 64, 768), (8, 64, 32)])
def test_grouped_mode_equals_its_block_diagonal_expansion(G, kg, ng):
    """The channel blocks outside a group contribute exact zero products, so the dense launch of the expanded weight
    computes the same sums in the same order: equal to within 2 ulp (observed: bit for bit)."""
    from asv_subtools_b200 import ops
    from asv_subtools_b200.model.ecapa_tdnn_xvector import _block_diagonal
    rng = np.random.RandomState(7)
    x = torch.from_numpy(rng.standard_normal((2, 77, G * kg)).astype(np.float32)).cuda()
    w = torch.from_numpy((rng.standard_normal((G * ng, kg, 1)) / np.sqrt(kg)).astype(np.float32)).cuda()
    a = _grouped(ops, x, w, G)
    d = _grouped(ops, x, _block_diagonal(w, G).contiguous(), G, groups=1)
    ulp = (a.view(torch.int32).long() - d.view(torch.int32).long()).abs().max().item()
    print("grouped vs block-diagonal: max ulp difference", ulp)
    assert ulp <= 2


@pytest.mark.parametrize("cin,cout,G,ntaps", [(256, 256, 4, 1),    # Kg = 64, Ng = 64: fits; one tap too many below
                                              (192, 256, 4, 1),    # Kg = 48
                                              (256, 80, 4, 1),     # Ng = 20
                                              (256, 256, 3, 1),    # not divisible
                                              (256, 256, 4, 3)])   # three taps
def test_grouped_constraints_return_einval(cin, cout, G, ntaps):
    from asv_subtools_b200 import _lib, ops
    x = ops.split_f32(torch.zeros(2, 10, cin, device="cuda"))
    ctx = [-1, 0, 1][:ntaps] if ntaps == 3 else [0]
    w = ops.pack_tdnn_weight(torch.zeros(cout, cin // G if cin % G == 0 else cin, len(ctx), device="cuda"), ctx)
    y = torch.empty(2, 10, cout, device="cuda")
    ok = cin % G == 0 and (cin // G) % 64 == 0 and (cout // G) % 32 == 0 and ntaps == 1
    assert ops.tdnn_grouped_fits(cin, cout, G) == (cin % G == 0 and (cin // G) % 64 == 0 and cout % G == 0 and (cout // G) % 32 == 0)
    if ok:
        ops.tdnn_affine_ex(x, w, cout, ctx, y_f32=y, groups=G)
        x2 = ops.split_f32(torch.zeros(2, 10, cin, device="cuda"))
        with pytest.raises(_lib.XvbError, match=r"rc=-1"):            # second source
            ops.tdnn_affine_ex(x, w, cout, ctx, x2=x2, y_f32=y, groups=G)
        with pytest.raises(_lib.XvbError, match=r"rc=-1"):            # swish epilogue
            ops.tdnn_affine_ex(x, w, cout, ctx, y_f32=y, groups=G, swish=True)
        return
    with pytest.raises(_lib.XvbError, match=r"rc=-1"):
        ops.tdnn_affine_ex(x, w, cout, ctx, y_f32=y, groups=G)


@pytest.mark.parametrize("share", [False, True])
def test_head_width_pooling_map_float64(share):
    from asv_subtools_b200 import ops
    rng = np.random.RandomState(3 + share)
    B, T, C, H, Q = 3, 53, 96, 3, 2
    cg = C // H
    nl = H * Q * (1 if share else cg)
    x = torch.from_numpy(rng.standard_normal((B, T, C)).astype(np.float32)).cuda()
    lg = torch.from_numpy(rng.standard_normal((B, T, nl)).astype(np.float32)).cuda()
    got = ops.attn_head_stats_pool_mq(lg, x, Q * C, cg if share else 1, cg, Q).cpu().numpy()
    xd = x.double().cpu().transpose(1, 2)                         # (B, C, T)
    alpha = torch.softmax(lg.double().cpu().transpose(1, 2), dim=2).reshape(B, H, Q, -1, T)
    mean, std = mo.compute_statistics(xd.reshape(B, H, 1, -1, T), alpha)
    want = torch.cat([mean.reshape(B, -1), std.reshape(B, -1)], dim=1).numpy()
    assert rel(got, want) <= 3e-5
    # head_width = C, rep = O / C is the existing map, result for result
    O = 2 * C
    a = ops.attn_head_stats_pool(lg[..., :2], x, O, C, floor=1e-5)
    b = ops.attn_head_stats_pool_mq(lg[..., :2], x, O, C, C, 2)
    assert torch.equal(a, b)


def _model(case, pos):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    kwargs, _, _, seed, _ = mo.CASES[case]
    m = ECAPA_TDNN(80, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed), strict=True)
    return m.cuda().eval()


SHORT = [(c, p, t) for c, (_, frames, positions, _, _) in mo.CASES.items() for p in positions for t in frames if t <= 10000]


@pytest.mark.parametrize("case,pos,t", SHORT)
def test_native_and_twin_match_golden_and_each_other(case, pos, t):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import EcapaExtractor, NativeEcapaExtractor
    m = _model(case, pos)
    feats = torch.from_numpy(onn.synthetic_feats(2, t, 80, mo.CASES[case][4] + t)).cuda()
    ref = GOLD["{}_{}_{}".format(case, pos, t)]
    nat = NativeEcapaExtractor(m, torch.device("cuda")).extract(feats).cpu().numpy()
    twin = EcapaExtractor(m, torch.device("cuda")).extract(feats).cpu().numpy()
    for got in (nat, twin):
        assert rel(got, ref) <= 1e-4 and cosine(got, ref) >= 1 - 1e-6, (case, pos, t, rel(got, ref))
    assert np.array_equal(nat, twin)


def test_chunk_rule_through_the_plugin_call():
    m = _model("roadmap_long", "near")
    feats = onn.synthetic_feats(2, 10050, 80, mo.CASES["roadmap_long"][4] + 10050)
    got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
    ref = GOLD["roadmap_long_near_10050"]
    assert rel(got, ref) <= 1e-4 and cosine(got, ref) >= 1 - 1e-6


def test_stddev_false_pooling_matches_oracle():
    """MQMHASP(stddev=False) (reachable by building the pooling directly: ECAPA's constructor pops `stddev`)."""
    from asv_subtools_b200.model.ecapa_tdnn_xvector import EcapaExtractor, NativeEcapaExtractor
    from asv_subtools_b200.nnet.components import ReluBatchNormTdnnLayer
    from asv_subtools_b200.nnet.pooling import MQMHASP
    m = _model("fc1", "near").cpu()
    p = dict(mo.resolve(mo.CASES["fc1"][0]["pooling_params"]), stddev=False)
    m.stats = MQMHASP(256, **p)
    m.bn_stats = torch.nn.BatchNorm1d(m.stats.get_output_dim())
    m.fc1 = ReluBatchNormTdnnLayer(m.stats.get_output_dim(), 64)
    rng = np.random.RandomState(5)
    sd = m.state_dict()
    for k in sd:
        if k.startswith(("stats.", "bn_stats.", "fc1.")) and sd[k].dtype == torch.float32:
            sd[k] = torch.from_numpy(rng.uniform(0.5, 1.5, sd[k].shape).astype(np.float32) if "running_var" in k
                                     else (rng.standard_normal(sd[k].shape) * 0.1).astype(np.float32))
    m.load_state_dict(sd)
    m.cuda().eval()
    feats = onn.synthetic_feats(2, 60, 80, 77)
    kw = mo.CASES["fc1"][0]
    sdc = {k: v.cpu() for k, v in m.state_dict().items()}
    with torch.no_grad():
        want = torch.stack([mo.ecapa_mqmha_forward(sdc, torch.from_numpy(f).T[None], kw, "near", pooling=p)[0, :, 0]
                            for f in feats]).numpy()
    x = torch.from_numpy(feats).cuda()
    nat = NativeEcapaExtractor(m, torch.device("cuda")).extract(x).cpu().numpy()
    twin = EcapaExtractor(m, torch.device("cuda")).extract(x).cpu().numpy()
    assert rel(nat, want) <= 1e-4 and np.array_equal(nat, twin)


def test_shard_calls_on_two_lanes_equal_per_batch_calls():
    from asv_subtools_b200.model.ecapa_tdnn_xvector import NativeEcapaExtractor
    m = _model("roadmap", "near")
    ex = NativeEcapaExtractor(m, torch.device("cuda"))
    feats = torch.from_numpy(onn.synthetic_feats(256, 300, 80, 41)).cuda()
    shard = ex.extract_shard(feats, batch=128)
    per = torch.cat([ex.extract(feats[:128].contiguous()), ex.extract(feats[128:].contiguous())])
    torch.cuda.synchronize()
    assert torch.equal(shard, per)
    host = np.empty((256, 192), dtype=np.float32)
    pinned = feats.cpu().pin_memory()
    ex.extract_shard_host(pinned.data_ptr(), 256, 300, host.ctypes.data, batch=128)
    assert np.array_equal(host, per.cpu().numpy())


def test_xvbe0002_round_trip_and_rejections(tmp_path):
    from asv_subtools_b200 import _lib
    from asv_subtools_b200.model.ecapa_tdnn_xvector import NativeEcapaExtractor
    m = _model("share", "near")
    ex = NativeEcapaExtractor(m, torch.device("cuda"))
    path = str(tmp_path / "mq.xvbm")
    ex.save(path)
    raw = open(path, "rb").read()
    assert raw[:8] == b"XVBE0002"
    feats = torch.from_numpy(onn.synthetic_feats(3, 90, 80, 9)).cuda()
    assert torch.equal(NativeEcapaExtractor.load(path).extract(feats), ex.extract(feats))
    for name, data in (("trunc", raw[:len(raw) // 2]), ("trunc_header", raw[:40]), ("magic", b"XVBE0003" + raw[8:])):
        bad = str(tmp_path / name)
        open(bad, "wb").write(data)
        with pytest.raises(_lib.XvbError):
            NativeEcapaExtractor.load(bad)
    # a default ECAPA model still writes and reads XVBE0001
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    d = ECAPA_TDNN(80, 10, training=False, ecapa_params={"mfa_conv": 256, "embd_dim": 64})
    d.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, mfa_conv=256, embd_dim=64), 5), strict=False)
    d.cuda().eval()
    e1 = NativeEcapaExtractor(d, torch.device("cuda"))
    p1 = str(tmp_path / "e1.xvbm")
    e1.save(p1)
    assert open(p1, "rb").read(8) == b"XVBE0001"
    assert torch.equal(NativeEcapaExtractor.load(p1).extract(feats), e1.extract(feats))


def test_xvb_extract_binary_runs_an_xvbe0002_file(tmp_path):
    from asv_subtools_b200 import kaldi_io
    m = _model("roadmap", "near")
    kwargs, _, _, seed, _ = mo.CASES["roadmap"]
    sd = onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed)
    model = str(tmp_path / "roadmap.xvbm")
    m.extractor().save(model)
    feats = {"u{}".format(i): onn.synthetic_feats(1, t, 80, 500 + i)[0] for i, t in enumerate([150, 150, 61])}
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "xv.ark")
    run = subprocess.run([BIN, "--batch", "4", model, ark, "ark:" + out], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    for k, v in feats.items():
        want = mo.extract(sd, v, kwargs, "near").numpy()
        assert got[k].shape == (192,) and rel(got[k], want) < 1e-4, k
