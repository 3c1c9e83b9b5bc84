"""ECAPA-TDNN on the GPU: every new epilogue/kernel against the oracle, then the whole model
against the golden fixtures produced by the reference."""
import numpy as np
import pytest
import torch

from oracle import nnet as onn

pytestmark = pytest.mark.gpu
TOL = 3e-5
EMB_TOL = 1e-4

CANON = dict(training=False,
             ecapa_params={"channels": 1024, "embd_dim": 192, "mfa_conv": 1536,
                           "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}},
             pooling="ecpa-attentive", pooling_params={"hidden_size": 128, "time_attention": True, "stddev": True},
             fc1=False, fc2_params={"nonlinearity": "", "nonlinearity_params": {"inplace": True}, "bn-relu": False,
                                    "bn": True, "bn_params": {"momentum": 0.5, "affine": False,
                                                              "track_running_stats": True}})


def rel(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as _ops
    return _ops


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def test_second_source_and_channel_slices(ops):
    """Res2Net step: y = relu_bn(W.(a[:, :, 128:256] + r[:, :, 0:128])) written into a slice of a wider tensor."""
    rng = np.random.RandomState(1)
    B, T, d = 3, 50, 3
    a = rng.standard_normal((B, T, 1024)).astype(np.float32)
    r = rng.standard_normal((B, T, 1024)).astype(np.float32)
    w = (rng.standard_normal((128, 128, 2 * d + 1)) * 0.05).astype(np.float32)
    b = rng.standard_normal(128).astype(np.float32) * 0.1
    sc = rng.uniform(0.5, 1.5, 128).astype(np.float32)
    sh = rng.standard_normal(128).astype(np.float32) * 0.1
    ctx = [-d, 0, d]
    ap, rp = ops.split_f32(cu(a)), ops.split_f32(cu(r))
    out = ops.SplitPlanes(torch.zeros(B, T, 1024, dtype=torch.bfloat16, device="cuda"),
                          torch.zeros(B, T, 1024, dtype=torch.bfloat16, device="cuda"), 1024)
    wp = ops.pack_tdnn_weight(cu(w), ctx)
    ops.tdnn_affine_ex(ap.slice(128, 256), wp, 128, ctx, x2=rp.slice(0, 128), bias=cu(b), bn_scale=cu(sc),
                       bn_shift=cu(sh), relu=True, y=out.slice(256, 384))
    got = out.float().cpu().numpy()
    with torch.no_grad():
        x = torch.from_numpy(a[:, :, 128:256] + r[:, :, 0:128]).transpose(1, 2)
        ref = torch.relu(onn.tdnn_affine(x, torch.from_numpy(w), torch.from_numpy(b), ctx))
        ref = (ref * torch.from_numpy(sc)[None, :, None] + torch.from_numpy(sh)[None, :, None]).transpose(1, 2).numpy()
    assert rel(got[:, :, 256:384], ref) < TOL
    assert np.all(got[:, :, :256] == 0) and np.all(got[:, :, 384:] == 0)   # nothing outside the slice was touched


@pytest.mark.parametrize("B,T,d", [(5, 150, 3), (2, 300, 4), (3, 40, 2), (150, 20, 2)])
def test_res2net_chain_kernel_vs_oracle(ops, B, T, d):
    """The one-kernel Res2Net block (CTA-owned utterances, 7 dependent steps) against the oracle's
    chunk/add/cat restatement, and against the seven-launch GEMM path."""
    from asv_subtools_b200.nnet.components import fold_batchnorm
    rng = np.random.RandomState(40 + d)
    x = rng.standard_normal((B, T, 1024)).astype(np.float32)
    spec = []
    for i in range(7):
        pfx = "blk.blocks.{}".format(i)
        spec += onn._affine_entries(pfx, 128, 128, [-d, 0, d]) + onn._bn_entries(pfx + ".batchnorm", 128)
    sd = onn.make_state_dict(spec, 900 + d)
    with torch.no_grad():
        ref = onn.res2net_block(torch.from_numpy(x).transpose(1, 2), sd, "blk", d).transpose(1, 2).numpy()
    xp = ops.split_f32(cu(x))
    packs, biases, scales, shifts = [], [], [], []
    for i in range(7):
        pfx = "blk.blocks.{}".format(i)
        packs.append(ops.pack_tdnn_weight(sd[pfx + ".affine.weight"].cuda().contiguous(), [-d, 0, d]))
        biases.append(sd[pfx + ".affine.bias"])
        bn = torch.nn.BatchNorm1d(128)
        bn.load_state_dict({k.split(".")[-1]: v for k, v in sd.items() if k.startswith(pfx + ".batchnorm.")})
        sc, sh = fold_batchnorm(bn)
        scales.append(torch.from_numpy(sc))
        shifts.append(torch.from_numpy(sh))
    y = ops.SplitPlanes.empty((B, T, 1024), "cuda")
    ops.res2net_block(xp, torch.cat([p.hi for p in packs]).contiguous(), torch.cat([p.lo for p in packs]).contiguous(),
                      torch.cat(biases).cuda(), torch.cat(scales).cuda(), torch.cat(shifts).cuda(), d, 8, y)
    got = y.float().cpu().numpy()
    assert np.all(np.isfinite(got))
    assert rel(got, ref) < 1e-4            # seven chained layers, each at the 3e-5 GEMM tolerance
    assert np.array_equal(got[:, :, :128], xp.float().cpu().numpy()[:, :, :128])   # chunk 0 passes through


def test_utt_bias_tanh_sigmoid_and_dual_output(ops):
    rng = np.random.RandomState(2)
    B, T, Cin, Cout = 5, 37, 192, 128
    x = rng.standard_normal((B, T, Cin)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, 1)) / np.sqrt(Cin)).astype(np.float32)
    ub = rng.standard_normal((B, Cout)).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    sh = rng.standard_normal(Cout).astype(np.float32) * 0.1
    xp, wp = ops.split_f32(cu(x)), ops.pack_tdnn_weight(cu(w), [0])
    y = ops.SplitPlanes.empty((B, T, Cout), "cuda")
    yf = torch.empty(B, T, Cout, device="cuda")
    ops.tdnn_affine_ex(xp, wp, Cout, [0], utt_bias=cu(ub), bn_scale=cu(sc), bn_shift=cu(sh), relu=True, tanh=True,
                       y=y, y_f32=yf)
    pre = np.einsum("btc,nc->btn", x.astype(np.float64), w[:, :, 0].astype(np.float64)) + ub[:, None, :]
    ref = np.tanh(np.maximum(pre, 0) * sc + sh)
    assert rel(yf.cpu().numpy(), ref) < TOL and rel(y.float().cpu().numpy(), ref) < TOL
    ops.tdnn_affine_ex(xp, wp, Cout, [0], sigmoid=True, y_f32=yf)
    ref = 1 / (1 + np.exp(-np.einsum("btc,nc->btn", x.astype(np.float64), w[:, :, 0].astype(np.float64))))
    assert rel(yf.cpu().numpy(), ref) < TOL


def test_plane_mean_and_se_apply(ops):
    rng = np.random.RandomState(3)
    B, T, C = 4, 61, 1024
    z = rng.standard_normal((B, T, C)).astype(np.float32)
    xin = rng.standard_normal((B, T, C)).astype(np.float32)
    g = rng.uniform(0, 1, (B, C)).astype(np.float32)
    zp, ip = ops.split_f32(cu(z)), ops.split_f32(cu(xin))
    m, mp = ops.plane_mean(zp)
    assert rel(m.cpu().numpy(), z.mean(1)) < 1e-5 and rel(mp.float().cpu().numpy()[:, 0], z.mean(1)) < 1e-5
    cat = ops.SplitPlanes.empty((B, T, 3 * C), "cuda")
    nxt = ops.SplitPlanes.empty((B, T, C), "cuda")
    ops.se_apply(zp, ip, cu(g), cat.slice(C, 2 * C), nxt)
    ref = z * g[:, None, :] + xin
    # split planes carry ~2^-17 relative precision per stored tensor
    assert rel(cat.float().cpu().numpy()[:, :, C:2 * C], ref) < TOL
    assert rel(nxt.float().cpu().numpy(), xin + ref) < TOL
    ops.se_apply(zp, nxt, cu(g), cat.slice(0, C), nxt)          # in place: next = in + out over the same buffer
    assert rel(cat.float().cpu().numpy()[:, :, :C], z * g[:, None, :] + (xin + ref)) < TOL


def test_global_context_stats_and_attentive_pool(ops):
    rng = np.random.RandomState(4)
    B, T, C = 3, 77, 1536
    x = (rng.standard_normal((B, T, C)) * 2 + 0.3).astype(np.float32)
    logits = (rng.standard_normal((B, T, C)) * 3).astype(np.float32)
    g = ops.stats_pool_ex(cu(x), 1e-5, 1).cpu().numpy()
    xt = torch.from_numpy(x).transpose(1, 2)
    assert rel(g[:, :C], xt.mean(2).numpy()) < 2e-6
    assert rel(g[:, C:], torch.sqrt(torch.var(xt, dim=-1) + 1e-5).numpy()) < 2e-6
    out, pl = ops.attn_stats_pool(cu(logits), cu(x), 1e-5, planes=True)
    alpha = torch.softmax(torch.from_numpy(logits).transpose(1, 2), dim=2)
    mean = torch.sum(alpha * xt, dim=2)
    std = torch.sqrt((torch.sum(alpha * xt ** 2, dim=2) - mean ** 2).clamp(min=1e-5))
    ref = torch.cat([mean, std], dim=1).numpy()
    assert rel(out.cpu().numpy(), ref) < 5e-6
    assert rel(pl.float().cpu().numpy()[:, 0], ref) < 2e-5


@pytest.mark.parametrize("B,K,N", [(128, 1024, 128), (128, 128, 1024), (5, 3072, 192), (1, 3072, 128), (37, 64, 20)])
def test_small_affine_rows_vs_float64(ops, B, K, N):
    """xvb_small_affine (segment-level fp32 affine on CUDA cores) against a float64 product, every epilogue flag, ragged
    tile edges (B, N not multiples of the 4 x 4 warp tile), fp32 and split-plane outputs."""
    rng = np.random.RandomState(B + K + N)
    x = rng.standard_normal((B, K)).astype(np.float32)
    w = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32) * 0.1
    s, t = rng.uniform(0.5, 1.5, N).astype(np.float32), rng.standard_normal(N).astype(np.float32) * 0.1
    base = x.astype(np.float64) @ w.astype(np.float64).T + b
    cases = [(dict(), base), (dict(relu=True), np.maximum(base, 0)),
             (dict(relu=True, bn_scale=cu(s), bn_shift=cu(t)), np.maximum(base, 0) * s + t),
             (dict(sigmoid=True), 1 / (1 + np.exp(-base))), (dict(tanh=True), np.tanh(base))]
    for kw, want in cases:
        got = ops.small_affine(cu(x), cu(w), cu(b), **kw)
        assert rel(got.cpu().numpy(), want) < 2e-6, kw
    y, planes = ops.small_affine(cu(x), cu(w), cu(b), planes=True)
    assert rel(planes.float().view(B, -1)[:, :N].cpu().numpy(), base) < 1e-5 and rel(y.cpu().numpy(), base) < 2e-6


def _model(pos, seed=201, default_fc2=False):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    if default_fc2:
        sd = onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), seed)
        m = ECAPA_TDNN(80, 10, training=False)
    else:
        sd = onn.make_state_dict(onn.ecapa_spec(80), seed)
        m = ECAPA_TDNN(80, 10, extracted_embedding=pos, **CANON)
    m.load_state_dict(sd, strict=True)
    return m.cuda().eval(), sd


@pytest.mark.parametrize("pos", ["near", "near_affine"])
def test_ecapa_embeddings_match_reference_golden(golden, pos):
    g = golden("ecapa")
    m, _ = _model(pos)
    feats = onn.synthetic_feats(2, 300, 80, 1201)
    ref = g["ecapa80_{}_emb".format(pos)]
    batch = m.extract_embedding_batch(feats).cpu().numpy()
    single = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
    for i in range(2):
        assert rel(batch[i], ref[i]) < EMB_TOL and rel(single[i], ref[i]) < EMB_TOL
        assert np.dot(batch[i], ref[i]) / (np.linalg.norm(batch[i]) * np.linalg.norm(ref[i])) > 1 - 1e-6


def test_ecapa_default_fc2_and_short_utterances(golden):
    g = golden("ecapa")
    m, _ = _model("near", seed=202, default_fc2=True)
    for T in (2, 40):
        f = onn.synthetic_feats(1, T, 80, 3201 + T)[0]
        assert rel(m.extract_embedding(f).numpy(), g["ecapa80_default_T{}".format(T)]) < EMB_TOL


@pytest.mark.parametrize("native", ["1", "0"])
def test_ecapa_with_fc1_matches_reference_golden(golden, monkeypatch, native):
    """ECAPA_TDNN(fc1=True) in the three positions (far = fc1.affine, near_affine = fc1 -> fc2.affine, near = fc1 -> fc2;
    ecapa_tdnn_xvector.py:412-422) against the reference's own outputs, native extractor and Python twin."""
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    monkeypatch.setenv("XVB_ECAPA_NATIVE", native)
    g = golden("ecapa_fc1")
    sd = onn.make_state_dict(onn.ecapa_spec(80, fc1=True, fc2_bn_affine=True), 203)
    feats = onn.synthetic_feats(2, 120, 80, 1203)
    for pos in ("far", "near_affine", "near"):
        m = ECAPA_TDNN(80, 10, training=False, fc1=True, extracted_embedding=pos)
        m.load_state_dict(sd, strict=True)
        m.cuda().eval()
        assert rel(m.extract_embedding_batch(feats).cpu().numpy(), g["fc1_" + pos]) < EMB_TOL, pos
        assert rel(m.extract_embedding(feats[1]).numpy(), g["fc1_" + pos][1]) < EMB_TOL, pos
        m.invalidate()
    with pytest.raises(AssertionError):
        ECAPA_TDNN(80, 10, training=False, extracted_embedding="far").cuda().eval().extractor()


def test_ecapa_vs_oracle_batch():
    """A batch shape with ragged tiles (B=5, T=83) straight against the oracle."""
    m, sd = _model("near")
    feats = onn.synthetic_feats(5, 83, 80, 555)
    got = m.extract_embedding_batch(feats).cpu().numpy()
    with torch.no_grad():
        ref = onn.ecapa_forward(sd, torch.from_numpy(feats).transpose(1, 2), "near").squeeze(2).numpy()
    for i in range(5):
        assert rel(got[i], ref[i]) < EMB_TOL


def test_ecapa_shard_calls_on_two_lanes_equal_per_batch_extraction(monkeypatch):
    """xvb_ecapa_extract_shard[_host]: batches alternate between the two lanes (twin workspaces, two streams; one lane
    with XVB_LANES=0) and must reproduce independent per-batch calls bit for bit, ragged tail batch, a single batch and
    whole batches included, as must xvb_ecapa_extract_host; C3's full batch size (128 x 300) is checked against
    sub-batches of itself (batch invariance at the BASELINE shape).  One handle serves both settings: XVB_LANES is read
    on every shard call."""
    m, _ = _model("near")
    ex = m.extractor()
    n, t = 11, 47
    feats = torch.from_numpy(onn.synthetic_feats(n, t, 80, 777)).cuda()
    want = torch.cat([ex.extract(feats[i:i + 4]).clone() for i in range(0, n, 4)])         # batches of 4, 4, 3
    for lanes in ("0", "1"):
        monkeypatch.setenv("XVB_LANES", lanes)
        _check_ecapa_shard(ex, feats, want)


def _check_ecapa_shard(ex, feats, want):
    n, t, _ = feats.shape
    assert torch.equal(ex.extract_shard(feats, 4), want)
    assert torch.equal(ex.extract_shard(feats, 4), want)                                    # lanes reused
    assert torch.equal(ex.extract_shard(feats[:3], 4), ex.extract(feats[:3]))               # N <= batch
    assert torch.equal(ex.extract_shard(feats[:8], 4), want[:8])                            # N a multiple of batch
    assert np.array_equal(ex.extract_host(feats[:4].cpu().numpy()), want[:4].cpu().numpy())
    host = torch.empty(n, t, 80, dtype=torch.float32, pin_memory=True)
    host.copy_(feats)
    out = torch.empty(n, ex.embed_dim, dtype=torch.float32, pin_memory=True)
    ex.extract_shard_host(host.data_ptr(), n, t, out.data_ptr(), 4)
    assert torch.equal(out, want.cpu())
    full = torch.from_numpy(onn.synthetic_feats(128, 300, 80, 778)).cuda()
    whole = ex.extract(full).clone()
    assert torch.isfinite(whole).all()
    parts = ex.extract_shard(full, 32)                                                      # 4 sub-batches on 2 lanes
    assert (whole - parts).abs().max() <= 1e-6 * whole.abs().max()      # split-free layers: same arithmetic per utterance
    one = ex.extract(full[77:78]).clone()
    assert (one[0] - whole[77]).abs().max() <= 1e-6 * whole.abs().max()


def test_native_ecapa_extractor_equals_python_orchestration_and_model_file(tmp_path, monkeypatch):
    """xvb_ecapa_t (the launch sequence in C++) against the op-by-op Python twin: same kernels, same order ->
    bit-identical embeddings; and the XVBE0001 model file round trip."""
    from asv_subtools_b200.model import ecapa_tdnn_xvector as mod
    sd = onn.make_state_dict(onn.ecapa_spec(80), 201)
    feats = torch.from_numpy(onn.synthetic_feats(5, 90, 80, 4242)).cuda()
    outs = {}
    for native in ("1", "0"):
        monkeypatch.setenv("XVB_ECAPA_NATIVE", native)
        for pos in ("near", "near_affine"):
            m = mod.ECAPA_TDNN(80, 10, **dict(CANON, extracted_embedding=pos))
            m.load_state_dict(sd, strict=True)
            m.cuda().eval()
            ex = m.extractor()
            assert type(ex).__name__ == ("NativeEcapaExtractor" if native == "1" else "EcapaExtractor")
            outs[native, pos] = ex.extract(feats)
            if native == "1" and pos == "near":
                path = str(tmp_path / "ecapa.xvbm")
                ex.save(path)
                ex2 = mod.NativeEcapaExtractor.load(path)
                assert ex2.feat_dim == 80 and ex2.embed_dim == 192
                assert torch.equal(ex2.extract(feats), outs[native, pos])
                assert ex.last_launches >= 30
            m.invalidate()
    for pos in ("near", "near_affine"):
        assert torch.equal(outs["1", pos], outs["0", pos]), pos
    with open(str(tmp_path / "ecapa.xvbm"), "r+b") as f:
        f.truncate(1000)
    with pytest.raises(RuntimeError):
        mod.NativeEcapaExtractor.load(str(tmp_path / "ecapa.xvbm"))
