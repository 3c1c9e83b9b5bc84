"""Masked batches of utterances of different lengths on the ResNet x-vector (xvb_resnet_extract_lengths and its op-by-op
twin): equal to the unmasked call when every length is T, each row close to the utterance extracted alone and to the
oracle, the goldens packed into mixed batches, native equal to twin, blind to what lies past an utterance's end; the
masked conv / head conv / SE scaling / plane mean on their own; the position budget; bad lengths; and xvb-extract /
pipeline/extract_embeddings.py with --mixed-lengths on an XVBR0001 file.  Needs an H100 (`-m gpu`)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import resnet_oracle as ro
from asv_subtools_b200 import kaldi_io, ops
from asv_subtools_b200.model.resnet_xvector import NativeResNetExtractor, ResNetExtractor, ResNetXvector
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
CASE_POS = [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosines(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sum(a * b, 1) / (np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1))


_MODELS = {}


def _model(case, pos):
    if (case, pos) not in _MODELS:
        kwargs, fdim, _, _, seed, _ = ro.CASES[case]
        m = ResNetXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
        sd = onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed)
        m.load_state_dict(sd, strict=True)
        _MODELS[(case, pos)] = (m.cuda().eval(), sd)
    return _MODELS[(case, pos)]


def _extractor(monkeypatch, case, pos, native):
    monkeypatch.setenv("XVB_RESNET_NATIVE", "1" if native else "0")
    ex = _model(case, pos)[0].build_extractor()
    assert isinstance(ex, NativeResNetExtractor if native else ResNetExtractor) and ex.TAKES_LENGTHS
    return ex


def _padded(rows, T, fdim, fill=0.0):
    x = np.full((len(rows), T, fdim), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


def _utterances(n, fdim, seed, lo=1, hi=300):
    rng = np.random.RandomState(seed)
    lens = [int(v) for v in rng.randint(lo, hi + 1, n)]
    lens[0], lens[1] = lo, hi
    return [onn.synthetic_feats(1, t, fdim, seed + i)[0] for i, t in enumerate(lens)]


# ------------------------------------------------------------------ 1. every length == T: bit for bit the unmasked call
@pytest.mark.parametrize("case", ["online", "preact"])
@pytest.mark.parametrize("native", [True, False])
def test_all_lengths_equal_T_is_the_unmasked_call(monkeypatch, case, native):
    pos = ro.CASES[case][3][0]
    fdim = ro.CASES[case][1]
    ex = _extractor(monkeypatch, case, pos, native)
    with torch.no_grad():
        for b in (1, 3, 64):
            for t in (1, 2, 37, 200):
                x = torch.from_numpy(onn.synthetic_feats(b, t, fdim, 100 * b + t)).cuda()
                want = ex.extract(x).clone()
                assert torch.equal(ex.extract(x, lengths=[t] * b), want), (case, native, b, t)


# ------------------------------------------------------------------ 2. each row against solo extraction and the oracle
@pytest.mark.parametrize("case, pos", CASE_POS)
def test_rows_match_solo_extraction_and_oracle(monkeypatch, case, pos):
    kwargs, fdim = ro.CASES[case][0], ro.CASES[case][1]
    ex = _extractor(monkeypatch, case, pos, True)
    _, sd = _model(case, pos)
    utts = _utterances(64, fdim, 7000 + len(case))
    T = max(u.shape[0] for u in utts)
    lens = [u.shape[0] for u in utts]
    with torch.no_grad():
        got = ex.extract(_padded(utts, T, fdim), lengths=lens).cpu().numpy()
        worst_rel, worst_cos = 0.0, 1.0
        for i, u in enumerate(utts):
            solo = ex.extract(torch.from_numpy(u[None]).cuda()).cpu().numpy()[0]
            worst_rel = max(worst_rel, rel(got[i], solo))
            worst_cos = min(worst_cos, float(cosines(got[i][None], solo[None])[0]))
        assert worst_rel <= 1e-5 and worst_cos >= 1 - 1e-8, (case, pos, worst_rel, worst_cos)
        for i in (0, 1, 2, 3, 17):
            ref = ro.resnet_forward(sd, torch.from_numpy(utts[i].T[None].copy()), pos, kwargs).numpy()[0, :, 0]
            assert rel(got[i], ref) <= 1e-4, (case, pos, i, lens[i], rel(got[i], ref))


# ------------------------------------------------------------------ 3. goldens packed into mixed batches
@pytest.mark.parametrize("case, pos", CASE_POS)
def test_goldens_in_one_mixed_batch(monkeypatch, golden, case, pos):
    g = golden("resnet")
    _, fdim, frames, _, _, fseed = ro.CASES[case]
    ex = _extractor(monkeypatch, case, pos, True)
    rows, want = [], []
    for t in frames:   # the two golden utterances of every length
        rows += list(onn.synthetic_feats(2, t, fdim, fseed + t))
        want.append(g["{}_{}_T{}".format(case, pos, t)])
    filler = _utterances(5, fdim, 900, 3, max(frames) + 20)
    T = max(r.shape[0] for r in rows + filler)
    got = ex.extract(_padded(filler[:3] + rows + filler[3:], T, fdim),
                     lengths=[r.shape[0] for r in filler[:3] + rows + filler[3:]]).cpu().numpy()[3:3 + len(rows)]
    ref = np.concatenate(want)
    assert rel(got, ref) <= 1e-4 and cosines(got, ref).min() >= 1 - 1e-6, (case, pos, rel(got, ref))


# ------------------------------------------------------------------ 4. native == twin; 5. padding is never read
@pytest.mark.parametrize("case, pos", [("online", "near"), ("preact", "far"), ("resnet18", "near")])
def test_native_equals_twin_and_padding_is_never_read(monkeypatch, case, pos):
    fdim = ro.CASES[case][1]
    native = _extractor(monkeypatch, case, pos, True)
    twin = _extractor(monkeypatch, case, pos, False)
    utts = _utterances(19, fdim, 4000, 1, 133)
    lens = [u.shape[0] for u in utts]
    T = max(lens) + 6
    with torch.no_grad():
        want = native.extract(_padded(utts, T, fdim), lengths=lens).clone()
        assert torch.equal(twin.extract(_padded(utts, T, fdim), lengths=lens), want)
        for fill in (float("nan"), 1e30, -1e30):
            assert torch.equal(native.extract(_padded(utts, T, fdim, fill), lengths=lens), want), fill
            assert torch.equal(twin.extract(_padded(utts, T, fdim, fill), lengths=lens), want), fill


# ------------------------------------------------------------------ 6. kernel level
def _planes(x):
    p = ops.split_f32(x.contiguous())
    return p, p.float()


def _ref_conv(xv, w, stride, k):
    x = xv.double().cpu().permute(0, 3, 2, 1)
    return F.conv2d(x, w.double().cpu(), stride=stride, padding=k // 2).permute(0, 3, 2, 1)


@pytest.mark.parametrize("cin, k, stride, taps", [(32, 3, 1, False), (32, 1, 2, False), (64, 3, 2, False), (64, 3, 1, True),
                                                  (32, 3, 2, True)])
def test_masked_conv2d_vs_per_utterance_conv(cin, k, stride, taps):
    B, T, Fd, cout = 3, 45, 20, 64
    lens = [1, 29, T]
    g = torch.Generator().manual_seed(cin + 10 * k + stride)
    x = torch.randn(B, T, Fd, cin, generator=g)
    for b, L in enumerate(lens):
        x[b, L:] = 0   # the invariant the masked conv relies on: zeros past each input length
    x = x.cuda()
    w = (torch.randn(cout, cin, k, k, generator=g) / (cin * k)).cuda()
    scale, shift = torch.rand(cout, generator=g).cuda() + 0.5, (torch.randn(cout, generator=g) * 0.1).cuda()
    s2, t2 = torch.rand(cout, generator=g).cuda() + 0.5, (torch.rand(cout, generator=g) + 0.1).cuda()   # relu(shift2) > 0
    xp, xv = _planes(x)
    To, Fo = (T - 1) // stride + 1, (Fd - 1) // stride + 1
    tl = list(range(k * k)) if taps else None
    wp = ops.pack_conv2d_weight(w, tl)
    d_lens = torch.tensor(lens, dtype=torch.int32).cuda()
    outs = {}
    for name, ln in (("masked", d_lens), ("plain", None), ("full", torch.full((B,), T, dtype=torch.int32).cuda())):
        y, y2 = ops.SplitPlanes.empty((B, To, Fo, cout), x.device), ops.SplitPlanes.empty((B, To, Fo, cout), x.device)
        for p in (y, y2):
            p.hi.fill_(7.0)
            p.lo.fill_(7.0)
        yf = torch.full((B, To, Fo, cout), 7.0, device=x.device)
        ops.conv2d(xp, wp, cout, k, stride, scale, shift, relu=False, y=y, y_f32=yf, scale2=s2, shift2=t2, y2=y2, taps=tl,
                   lengths=ln)
        outs[name] = (y.float().cpu(), yf.cpu(), y2.float().cpu())
    for a, b in zip(outs["full"], outs["plain"]):
        assert torch.equal(a, b)
    y, yf, y2 = outs["masked"]
    for b, L in enumerate(lens):
        Lo = (L - 1) // stride + 1
        ref = _ref_conv(xv[b:b + 1, :L], w, stride, k)[0] * scale.double().cpu() + shift.double().cpu()
        assert ref.shape[0] == Lo
        assert rel(yf[b, :Lo], ref) <= 3e-5 and rel(y[b, :Lo], ref) <= 3e-5, (b, L)
        ref2 = torch.relu(torch.from_numpy(yf[b, :Lo].numpy()).double() * s2.double().cpu() + t2.double().cpu())
        assert rel(y2[b, :Lo], ref2) <= 3e-5
        for o in (y, yf, y2):
            assert torch.count_nonzero(o[b, Lo:]) == 0, (b, L)


def test_conv2d_valid_refuses_lengths():
    x = ops.SplitPlanes.empty((2, 9, 8, 32), "cuda")
    w = ops.pack_conv2d_weight(torch.randn(32, 32, 3, 3).cuda())
    with pytest.raises(RuntimeError, match="xvb_conv2d_valid: lengths"):
        ops.conv2d(x, w, 32, 3, 1, y=ops.SplitPlanes.empty((2, 7, 6, 32), "cuda"), valid=True,
                   lengths=torch.tensor([9, 4], dtype=torch.int32).cuda())


def test_masked_head_conv_se_residual_and_plane_mean_vs_float64():
    B, T, Fd, C = 3, 23, 12, 32
    lens = [1, 17, T]
    g = torch.Generator().manual_seed(5)
    d_lens = torch.tensor(lens, dtype=torch.int32).cuda()
    # head conv: NaN past each end must not be read
    feats = torch.randn(B, T, Fd, generator=g)
    for b, L in enumerate(lens):
        feats[b, L:] = float("nan")
    w = torch.randn(C, 1, 3, 3, generator=g)
    scale, shift = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    s2, t2 = torch.rand(C, generator=g) + 0.5, torch.rand(C, generator=g) + 0.1
    y, y2 = ops.SplitPlanes.empty((B, T, Fd, C), "cuda"), ops.SplitPlanes.empty((B, T, Fd, C), "cuda")
    ops.conv2d_head(feats.cuda(), w.cuda(), scale.cuda(), shift.cuda(), y, s2.cuda(), t2.cuda(), y2, lengths=d_lens)
    yv, y2v = y.float().cpu(), y2.float().cpu()
    for b, L in enumerate(lens):
        x = feats[b:b + 1, :L].double().permute(0, 2, 1).unsqueeze(1)
        ref = torch.relu(F.conv2d(x, w.double(), padding=1)[0].permute(2, 1, 0) * scale.double() + shift.double())
        assert rel(yv[b, :L], ref) <= 1e-5
        assert rel(y2v[b, :L], torch.relu(ref * s2.double() + t2.double())) <= 1e-5
        assert torch.count_nonzero(yv[b, L:]) == 0 and torch.count_nonzero(y2v[b, L:]) == 0
    # SE scaling + residual
    z = torch.randn(B, T, Fd, C, generator=g)
    ident = torch.randn(B, T, Fd, C, generator=g)
    gate = torch.rand(B, C, generator=g)
    zp, zv = _planes(z.cuda())
    ip, iv = _planes(ident.cuda())
    yo, y2o = ops.SplitPlanes.empty((B, T, Fd, C), "cuda"), ops.SplitPlanes.empty((B, T, Fd, C), "cuda")
    yf = torch.full((B, T, Fd, C), 7.0, device="cuda")
    ops.se_residual(zp, gate.cuda(), ip, relu=True, y=yo, y_f32=yf, scale2=s2.cuda(), shift2=t2.cuda(), y2=y2o, lengths=d_lens)
    ref = torch.relu(zv.double().cpu() * gate.double()[:, None, None, :] + iv.double().cpu())
    for b, L in enumerate(lens):
        assert rel(yf[b, :L].cpu(), ref[b, :L]) <= 1e-6
        assert rel(y2o.float()[b, :L].cpu(), torch.relu(ref[b, :L] * s2.double() + t2.double())) <= 1e-5
        for o in (yo.float(), yf, y2o.float()):
            assert torch.count_nonzero(o[b, L:]) == 0
    # masked plane mean over (B, T*F/k, k*C) rows, k = 4 dividing F
    k = 4
    view = ops.SplitPlanes(zp.hi.view(B, T * Fd // k, k * C), zp.lo.view(B, T * Fd // k, k * C), k * C)
    mean, _ = ops.plane_mean(view, planes=False, lengths=d_lens, rows_per_length=Fd // k)
    for b, L in enumerate(lens):
        want = zv[b, :L].double().cpu().reshape(-1, k * C).mean(0)
        assert rel(mean[b].cpu(), want) <= 1e-6, b


# ------------------------------------------------------------------ 7. position budget; 8. bad lengths
def test_masked_call_over_the_budget_equals_its_groups(monkeypatch):
    """60 utterances padded to 1000 frames x 80 bins are over the 256 * 200 * 80 position budget: groups of 51 and 9."""
    ex = _extractor(monkeypatch, "online", "near", True)
    utts = _utterances(60, 80, 333, 1, 1000)
    lens = [u.shape[0] for u in utts]
    x = _padded(utts, 1000, 80)
    whole = ex.extract(x, lengths=lens)
    parts = torch.cat([ex.extract(x[:51].contiguous(), lengths=lens[:51]), ex.extract(x[51:].contiguous(), lengths=lens[51:])])
    assert torch.equal(whole, parts)


def test_bad_lengths_name_the_first_bad_one(monkeypatch):
    ex = _extractor(monkeypatch, "preact", "near", True)
    x = torch.zeros(4, 30, 23, device="cuda")
    for lens, bad in (([30, 0, 5, 3], "lengths\\[1\\]=0"), ([30, 30, 31, 0], "lengths\\[2\\]=31"), ([-2, 1, 1, 1], "lengths\\[0\\]=-2")):
        with pytest.raises(RuntimeError, match="xvb_resnet_extract_lengths: " + bad):
            ex.extract(x, lengths=lens)
    emb = torch.empty(4, ex.embed_dim, device="cuda")
    arr = (C.c_int32 * 4)(5, 6, 0, 7)
    assert ex._fn("extract_lengths")(ex._h, C.c_void_p(x.data_ptr()), arr, 4, 30, C.c_void_p(emb.data_ptr()),
                                      ex._stream()) == -1   # XVB_EINVAL


# ------------------------------------------------------------------ 9. xvb-extract / the pipeline; 10. other families
def _write_ark(path, feats):
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)


def test_xvb_extract_mixed_lengths_on_a_resnet_model(tmp_path):
    case, pos = "preact", "near"
    kwargs, fdim = ro.CASES[case][0], ro.CASES[case][1]
    m, sd = _model(case, pos)
    model = str(tmp_path / "resnet.xvbm")
    m.extractor().save(model)
    rng = np.random.RandomState(2026)
    lens = [1, 2, 10001] + [int(v) for v in np.exp(rng.uniform(0, np.log(1500), 33))]
    feats = {"u{:02d}".format(i): onn.synthetic_feats(1, t, fdim, 6000 + i)[0] for i, t in enumerate(lens)}
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, feats)
    runs = {}
    for name, flag in (("mixed", ["--mixed-lengths"]), ("plain", [])):
        out = str(tmp_path / (name + ".ark"))
        r = subprocess.run([BIN, "--batch", "16"] + flag + [model, "ark:" + ark, "ark:" + out], capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[name] = (dict(kaldi_io.read_vec_flt_ark(out)), r.stderr)
    got, summary = runs["mixed"]
    assert sorted(got) == sorted(feats)
    s = re.search(r"(\d+) masked batches, (\d+) padded frames \(([0-9.]+) of (\d+) batch frames\)", summary)
    assert s, summary
    assert int(s.group(1)) < len(feats) and float(s.group(3)) <= 0.125
    for k in feats:
        assert rel(got[k], runs["plain"][0][k]) < 1e-5, k
    fwd = lambda v: ro.resnet_forward(sd, v, pos, kwargs)                         # noqa: E731
    with torch.no_grad():
        for k in ("u00", "u01", "u02", "u05", "u11", "u20"):
            assert rel(got[k], onn.extract_embedding(fwd, feats[k]).numpy()) < 1e-4, k

    torch.save(sd, str(tmp_path / "final.params"))
    out = str(tmp_path / "py.ark")
    creation = ro.creation(kwargs, fdim, pos)
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--mixed-lengths",
                        "--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", "resnet_xvector.py"),
                        "--model-creation", creation, "--batch-size", "16",
                        str(tmp_path / "final.params"), "ark:" + ark, "ark:" + out],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(py) == sorted(feats) and "masked batches" in r.stderr
    for k in feats:
        assert rel(py[k], got[k]) < 1e-5, k


def test_other_2d_families_still_refuse_lengths(tmp_path):
    import repvgg_oracle as vo
    from asv_subtools_b200.model.campplus_xvector import CamPPXvector
    from asv_subtools_b200.model.repvgg_xvector import RepVggXvector
    from asv_subtools_b200.model.transformer_xvector import TransformerXvector
    kwargs, fdim, _, positions, seed, _ = vo.CASES["a0"]
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding=positions[0], **kwargs)
    m.load_state_dict(onn.make_state_dict(vo.repvgg_spec(fdim, kwargs), seed), strict=True)
    m.cuda().eval()
    with pytest.raises(NotImplementedError, match="RepVggXvector"):
        m.extract_embedding_batch(np.zeros((2, 50, fdim), np.float32), lengths=[50, 20])
    model = str(tmp_path / "repvgg.xvbm")
    m.extractor().save(model)
    assert open(model, "rb").read(8) == b"XVBV0001"
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, {"a": onn.synthetic_feats(1, 50, fdim, 1)[0]})
    r = subprocess.run([BIN, "--mixed-lengths", model, "ark:" + ark, "ark:" + str(tmp_path / "o.ark")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 1 and "ERROR" in r.stderr, r.stdout + r.stderr
    for cls in (CamPPXvector, TransformerXvector):   # each refuses before it touches the model
        with pytest.raises(NotImplementedError, match=cls.__name__):
            cls.extract_embedding_batch(cls.__new__(cls), np.zeros((2, 50, 80), np.float32), lengths=[50, 20])
