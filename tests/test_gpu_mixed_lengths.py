"""Masked batches of utterances of different lengths on the TDNN x-vector handle (xvb_extractor_extract_lengths): equal
to the unmasked call when every length is T, each row equal to the utterance extracted alone, blind to what lies past
an utterance's end; the masked layer epilogue and the length-aware pooling on their own; bad lengths; and xvb-extract /
pipeline/extract_embeddings.py with --mixed-lengths.  Needs an H100 (`-m gpu`)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from asv_subtools_b200 import kaldi_io, ops
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
EMB_TOL = 1e-4


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))


_MODELS = {}


def _model(dim, seed, pos):
    if (dim, seed, pos) not in _MODELS:
        from asv_subtools_b200.model.xvector import Xvector
        sd = onn.make_state_dict(onn.xvector_spec(dim), seed)
        m = Xvector(dim, 10, training=False, extracted_embedding=pos)
        m.load_state_dict(sd, strict=True)
        _MODELS[(dim, seed, pos)] = (m.cuda().eval(), sd)
    return _MODELS[(dim, seed, pos)]


def _padded(rows, T, dim, fill=0.0):
    x = np.full((len(rows), T, dim), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


# ------------------------------------------------------------------ 1. every length == T: bit for bit the unmasked call
@pytest.mark.parametrize("fused", [True, False])
def test_all_lengths_equal_T_is_the_unmasked_call(fused):
    for dim, seed in ((23, 101), (80, 102)):
        m, _ = _model(dim, seed, "far")
        ex = m.extractor()
        ex.set_fused_pooling(fused)
        try:
            for B in (1, 3, 256):
                for T in (1, 3, 37, 200):
                    x = torch.from_numpy(onn.synthetic_feats(B, T, dim, 11 * B + T)).cuda()
                    a = ex.extract(x)
                    b = ex.extract(x, [T] * B)
                    assert torch.equal(a, b), (dim, B, T)
                    assert torch.equal(m.extract_embedding_batch(x, lengths=np.full(B, T)), a), (dim, B, T)
        finally:
            ex.set_fused_pooling(True)


# ------------------------------------------------------------------ 2. mixed lengths: each row == the utterance alone
def _mixed_lengths(seed, B=64, lo=1, hi=300):
    rng = np.random.RandomState(seed)
    lens = rng.randint(lo, hi + 1, B)
    lens[:4] = [1, 2, 3, hi]
    rng.shuffle(lens)
    return [int(v) for v in lens]


@pytest.mark.parametrize("dim,seed", [(23, 101), (80, 102)])
@pytest.mark.parametrize("pos", ["far", "near"])
def test_mixed_batch_rows_equal_solo_extraction(dim, seed, pos):
    m, _ = _model(dim, seed, pos)
    ex = m.extractor()
    lens = _mixed_lengths(seed + (pos == "near"))
    feats = onn.synthetic_feats(64, 300, dim, seed + 500)
    x = torch.from_numpy(feats).cuda()
    for fused in (True, False):
        ex.set_fused_pooling(fused)
        try:
            got = ex.extract(x, lens).cpu().numpy()
            for b, n in enumerate(lens):
                solo = ex.extract(x[b:b + 1, :n].contiguous()).cpu().numpy()[0]
                assert rel(got[b], solo) <= 1e-5, (fused, b, n, rel(got[b], solo))
                assert cos(got[b], solo) >= 1 - 1e-8, (fused, b, n)
        finally:
            ex.set_fused_pooling(True)


def test_mixed_batch_matches_the_oracle():
    m, sd = _model(80, 102, "near")
    lens = [300, 1, 57, 2, 199, 3, 120, 8]
    feats = onn.synthetic_feats(len(lens), 300, 80, 4321)
    got = m.extract_embedding_batch(feats, lengths=lens).cpu().numpy()
    for b, n in enumerate(lens):
        want = onn.extract_embedding(lambda v: onn.xvector_forward(sd, v, "near"), feats[b, :n]).numpy()
        assert rel(got[b], want) < EMB_TOL, (b, n)


# ------------------------------------------------------------------ 3. the reference goldens inside one mixed batch
@pytest.mark.parametrize("dim,seed", [(23, 101), (80, 102)])
def test_xvector_goldens_in_one_mixed_batch(golden, dim, seed):
    g = golden("xvector")
    for pos in ("far", "near"):
        m, _ = _model(dim, seed, pos)
        rows = list(onn.synthetic_feats(4, 200, dim, seed + 1000))
        want = list(g["xv{}_{}_emb".format(dim, pos)])
        if pos == "far":                                            # edge lengths: far position only
            for T in (1, 3, 7):
                rows.append(onn.synthetic_feats(1, T, dim, seed + 3000 + T)[0])
                want.append(g["xv{}_far_T{}".format(dim, T)])
        order = np.random.RandomState(seed).permutation(len(rows))
        rows, want = [rows[i] for i in order], [want[i] for i in order]
        got = m.extract_embedding_batch(_padded(rows, 200, dim), lengths=[r.shape[0] for r in rows]).cpu().numpy()
        for i in range(len(rows)):
            assert rel(got[i], want[i]) < EMB_TOL and cos(got[i], want[i]) >= 1 - 1e-6, (pos, i, rows[i].shape[0])


@pytest.mark.parametrize("cname,extend,seed", [("std", False, 301), ("ext", True, 302)])
def test_snowdar_goldens_in_one_mixed_batch(golden, cname, extend, seed):
    from asv_subtools_b200.model.snowdar_xvector import Xvector
    g = golden("snowdar")
    sd = onn.make_state_dict(onn.snowdar_xvector_spec(40, extend=extend), seed)
    rows = list(onn.synthetic_feats(3, 120, 40, seed + 1000))
    fill = [onn.synthetic_feats(1, t, 40, seed + 7000 + t)[0] for t in (5, 300, 64)]     # other lengths in the batch
    batch = [fill[0], rows[0], fill[1], rows[1], fill[2], rows[2]]
    for pos in ("far", "near_affine", "near"):
        m = Xvector(40, 10, extend=extend, training=False, extracted_embedding=pos)
        m.load_state_dict(sd, strict=True)
        m.cuda().eval()
        got = m.extract_embedding_batch(_padded(batch, 300, 40), lengths=[r.shape[0] for r in batch]).cpu().numpy()
        want = g["{}_{}".format(cname, pos)]
        for i, j in ((1, 0), (3, 1), (5, 2)):
            assert rel(got[i], want[j]) < EMB_TOL and cos(got[i], want[j]) >= 1 - 1e-6, (pos, j)


def test_other_blueprints_refuse_lengths():
    """A snowdar x-vector with LDE pooling runs on the Python launch sequence, not the TDNN handle."""
    from asv_subtools_b200.model.snowdar_xvector import Xvector
    m = Xvector(40, 10, training=False, extracted_embedding="far", pooling="lde")
    m.cuda().eval()
    with pytest.raises(NotImplementedError, match="Xvector"):
        m.extract_embedding_batch(np.zeros((2, 50, 40), np.float32), lengths=[50, 20])


# ------------------------------------------------------------------ 4. what lies past an utterance's end is never read
@pytest.mark.parametrize("dim,seed", [(23, 101), (80, 102)])
def test_pad_content_is_ignored(dim, seed):
    m, _ = _model(dim, seed, "near")
    ex = m.extractor()
    lens = _mixed_lengths(seed + 9, B=16, hi=150)
    rows = list(onn.synthetic_feats(16, 150, dim, seed + 77))
    rows = [r[:n] for r, n in zip(rows, lens)]
    for fused in (True, False):
        ex.set_fused_pooling(fused)
        try:
            ref = ex.extract(_padded(rows, 150, dim, 0.0), lens)
            for fill in (float("nan"), 1e30, -1e30):
                assert torch.equal(ex.extract(_padded(rows, 150, dim, fill), lens), ref), (fused, fill)
        finally:
            ex.set_fused_pooling(True)


# ------------------------------------------------------------------ 5. kernel level
def _layer_inputs(B, T, Cin, Cout, context, seed):
    rng = np.random.RandomState(seed)
    _, _, tot = onn.context_span(context)
    x = rng.standard_normal((B, T, Cin)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, tot)) * np.sqrt(2.0 / (Cin * len(context)))).astype(np.float32)
    b = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, Cout).astype(np.float32)
    shift = (0.1 * rng.standard_normal(Cout)).astype(np.float32)
    return x, w, b, scale, shift


def _oracle_rows(x, lens, w, b, scale, shift, context):
    """Per utterance: F.conv1d (components.py:107-149) on its own frames, ReLU, BN; float64."""
    out = []
    for i, n in enumerate(lens):
        with torch.no_grad():
            y = onn.tdnn_affine(torch.from_numpy(x[i:i + 1, :n]).double().transpose(1, 2), torch.from_numpy(w).double(),
                                torch.from_numpy(b).double(), context)
            y = torch.relu(y) * torch.from_numpy(scale).double()[None, :, None] + torch.from_numpy(shift).double()[None, :, None]
        out.append(y[0].transpose(0, 1).numpy())
    return out


@pytest.mark.parametrize("B,T,Cin,Cout,context", [
    (3, 45, 64, 256, [-2, -1, 0, 1, 2]),         # ragged tile edges
    (5, 200, 512, 512, [-3, 0, 3]),
    (64, 37, 24, 96, [-2, 0, 2]),
])
def test_masked_layer_matches_conv1d_per_utterance(B, T, Cin, Cout, context):
    x, w, b, scale, shift = _layer_inputs(B, T, Cin, Cout, context, B + T)
    lens = [max(1, T - 7 * i) for i in range(B)]
    lens[0] = T
    xz = x.copy()
    for i, n in enumerate(lens):
        xz[i, n:] = 0.0                                # the planes hold zeros past each end
    xp = ops.split_f32(torch.from_numpy(xz).cuda())
    wp = ops.pack_tdnn_weight(torch.from_numpy(w).cuda(), context)
    y = ops.SplitPlanes.empty((B, T, Cout), "cuda")
    yf = torch.full((B, T, Cout), 7.0, device="cuda")
    L = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ops.tdnn_affine_ex(xp, wp, Cout, context, bias=torch.from_numpy(b).cuda(), bn_scale=torch.from_numpy(scale).cuda(),
                       bn_shift=torch.from_numpy(shift).cuda(), relu=True, y=y, y_f32=yf, lengths=L)
    got, planes = yf.cpu().numpy(), y.float().cpu().numpy()
    for i, (n, want) in enumerate(zip(lens, _oracle_rows(x, lens, w, b, scale, shift, context))):
        assert rel(got[i, :n], want) <= 3e-5, (i, n)
        assert rel(planes[i, :n], want) <= 3e-5, (i, n)
        assert np.all(got[i, n:] == 0) and np.all(planes[i, n:] == 0), i


def test_masked_im2col_first_layer_matches_conv1d_per_utterance():
    """The first layer's im2col view (one long row of consecutive taps over time-padded planes), as the extractor runs
    it for 80-dim features, with lengths: B = 3, T = 45."""
    B, T, Cin, Cout, context = 3, 45, 80, 512, [-2, -1, 0, 1, 2]
    x, w, b, scale, shift = _layer_inputs(B, T, Cin, Cout, context, 45)
    lens = [45, 17, 1]
    xz = np.zeros((B, T + 4, Cin), np.float32)
    for i, n in enumerate(lens):
        xz[i, 2:2 + n] = x[i, :n]
    pad = ops.split_f32(torch.from_numpy(xz).cuda())
    win = ops.SplitPlanes(pad.hi.as_strided((B, T, 5 * Cin), ((T + 4) * Cin, Cin, 1)),
                          pad.lo.as_strided((B, T, 5 * Cin), ((T + 4) * Cin, Cin, 1)), 5 * Cin)
    w_im2col = torch.from_numpy(w).permute(0, 2, 1).reshape(Cout, 5 * Cin, 1).contiguous().cuda()
    wp = ops.pack_tdnn_weight(w_im2col, [0])
    yf = torch.full((B, T, Cout), 7.0, device="cuda")
    ops.tdnn_affine_ex(win, wp, Cout, [0], bias=torch.from_numpy(b).cuda(), bn_scale=torch.from_numpy(scale).cuda(),
                       bn_shift=torch.from_numpy(shift).cuda(), relu=True, y_f32=yf, x_batch_stride=(T + 4) * Cin,
                       lengths=torch.tensor(lens, dtype=torch.int32, device="cuda"))
    got = yf.cpu().numpy()
    for i, (n, want) in enumerate(zip(lens, _oracle_rows(x, lens, w, b, scale, shift, context))):
        assert rel(got[i, :n], want) <= 3e-5, (i, n)
        assert np.all(got[i, n:] == 0), i


def _stats64(rows, eps=1e-10):
    out = []
    for r in rows:
        r = np.asarray(r, np.float64)
        mean = r.mean(0)
        out.append(np.concatenate([mean, np.sqrt(np.maximum(((r - mean) ** 2).mean(0), eps))]))
    return np.stack(out)


@pytest.mark.parametrize("B,T", [(3, 45), (40, 8), (2, 300), (9, 1), (16, 200)])
def test_masked_stats_pool_matches_float64(B, T):
    """The last frame layer of a masked batch (fp32 output, zeros past the ends) and the length-aware pooling against
    float64 per-utterance mean / std; the frames past an end hold NaN for the pooling and are never read."""
    Cin, Cout = 512, 1500
    x, w, b, scale, shift = _layer_inputs(B, T, Cin, Cout, [0], 3 * B + T)
    rng = np.random.RandomState(B * T)
    lens = [int(v) for v in rng.randint(1, T + 1, B)]
    lens[0] = T
    xz = x.copy()
    for i, n in enumerate(lens):
        xz[i, n:] = 0.0
    want = _stats64(_oracle_rows(x, lens, w, b, scale, shift, [0]))
    L = torch.tensor(lens, dtype=torch.int32, device="cuda")
    xp = ops.split_f32(torch.from_numpy(xz).cuda())
    wp = ops.pack_tdnn_weight(torch.from_numpy(w).cuda(), [0])
    kw = dict(bias=torch.from_numpy(b).cuda(), bn_scale=torch.from_numpy(scale).cuda(), bn_shift=torch.from_numpy(shift).cuda(),
              relu=True)
    y = torch.empty(B, T, Cout, device="cuda")
    ops.tdnn_affine_ex(xp, wp, Cout, [0], y_f32=y, lengths=L, **kw)
    assert torch.all(torch.stack([torch.all(y[i, n:] == 0) for i, n in enumerate(lens)]))
    for i, n in enumerate(lens):
        y[i, n:] = float("nan")
    out, planes = ops.stats_pool_ex(y, 1e-10, 0, planes=True, lengths=L)
    assert rel(out.cpu().numpy(), want) <= 3e-5
    assert rel(planes.float()[:, 0].cpu().numpy(), want) <= 3e-5
    partial = torch.empty(xvb_blocks(B, T), B, 2 * Cout, device="cuda")
    with pytest.raises(Exception, match="lengths"):                     # the fused pooling takes equal lengths only
        ops.tdnn_affine_ex(xp, wp, Cout, [0], pool_partial=partial, lengths=L, **kw)


def xvb_blocks(B, T):
    tb = C.c_int()
    from asv_subtools_b200._lib import lib
    return lib.xvb_pool_partial_blocks(B, T, C.byref(tb))


# ------------------------------------------------------------------ 6. bad lengths
def test_bad_lengths_are_refused():
    from asv_subtools_b200._lib import XvbError, last_error, lib
    m, _ = _model(23, 101, "far")
    ex = m.extractor()
    x = torch.zeros(3, 20, 23, device="cuda")
    emb = torch.empty(3, 512, device="cuda")
    for bad in ([20, 0, 20], [20, -3, 20], [20, 20, 21]):
        arr = (C.c_int32 * 3)(*bad)
        rc = lib.xvb_extractor_extract_lengths(ex._h, C.c_void_p(x.data_ptr()), arr, 3, 20, C.c_void_p(emb.data_ptr()),
                                               C.c_void_p(torch.cuda.current_stream().cuda_stream))
        bad_at = next(i for i, v in enumerate(bad) if not 1 <= v <= 20)
        assert rc == -1 and "lengths[{}]={}".format(bad_at, bad[bad_at]) in last_error(), (bad, rc, last_error())
        with pytest.raises(XvbError):
            ex.extract(x, bad)
    with pytest.raises(ValueError):
        ex.extract(x, [20, 20])
    torch.cuda.synchronize()
    assert torch.isfinite(ex.extract(x, [20, 1, 7])).all()          # the handle still works


# ------------------------------------------------------------------ 7. the CLIs
def _write_ark(path, feats):
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)


def _corpus(dim):
    rng = np.random.RandomState(2026)
    lens = [1, 2, 3, 12000, 10001] + [int(v) for v in np.exp(rng.uniform(0, np.log(3000), 35))]
    return {"u{:02d}".format(i): onn.synthetic_feats(1, t, dim, 5000 + i)[0] for i, t in enumerate(lens)}


def test_xvb_extract_mixed_lengths(tmp_path):
    m, sd = _model(23, 101, "far")
    model = str(tmp_path / "xv.xvbm")
    m.extractor().save(model)
    feats = _corpus(23)
    assert len(feats) >= 38 and max(v.shape[0] for v in feats.values()) > 10000
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, feats)
    runs = {}
    for name, flag in (("mixed", ["--mixed-lengths"]), ("plain", [])):
        out = str(tmp_path / (name + ".ark"))
        r = subprocess.run([BIN, "--batch", "16"] + flag + [model, "ark:" + ark, "ark:" + out], capture_output=True, text=True,
                           timeout=600)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[name] = (dict(kaldi_io.read_vec_flt_ark(out)), r.stderr)
    got, summary = runs["mixed"]
    assert sorted(got) == sorted(feats)
    s = re.search(r"(\d+) masked batches, (\d+) padded frames \(([0-9.]+) of (\d+) batch frames\)", summary)
    assert s, summary
    assert int(s.group(1)) < len(feats) and float(s.group(3)) <= 0.125
    fwd = lambda v: onn.xvector_forward(sd, v, "far")                           # noqa: E731
    for k, v in feats.items():
        assert rel(got[k], onn.extract_embedding(fwd, v).numpy()) < 1e-4, k
        assert rel(got[k], runs["plain"][0][k]) < 1e-5, k

    # the Python pipeline with the flag: the same vectors per key
    torch.save(sd, str(tmp_path / "final.params"))
    out = str(tmp_path / "py.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--mixed-lengths",
                        "--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", "xvector.py"),
                        "--model-creation", "Xvector(23,10,training=False,extracted_embedding='far')", "--batch-size", "16",
                        str(tmp_path / "final.params"), "ark:" + ark, "ark:" + out],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(py) == sorted(feats) and "masked batches" in r.stderr
    for k in feats:
        assert rel(py[k], got[k]) < 1e-5, k


def test_mixed_lengths_refuses_other_families(tmp_path):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN
    canon = dict(training=False, extracted_embedding="near",
                 ecapa_params={"channels": 1024, "embd_dim": 192, "mfa_conv": 1536,
                               "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}},
                 fc2_params={"nonlinearity": "", "bn": True, "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}})
    m = ECAPA_TDNN(80, 10, **canon)
    m.cuda().eval()
    model = str(tmp_path / "ecapa.xvbm")
    m.extractor().save(model)
    assert open(model, "rb").read(8) == b"XVBE0001"
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, {"a": onn.synthetic_feats(1, 50, 80, 1)[0]})
    r = subprocess.run([BIN, "--mixed-lengths", model, "ark:" + ark, "ark:" + str(tmp_path / "o.ark")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 1 and "ERROR" in r.stderr, r.stdout + r.stderr
    with pytest.raises(NotImplementedError, match="ECAPA_TDNN"):
        m.extract_embedding_batch(np.zeros((2, 50, 80), np.float32), lengths=[50, 20])
