"""Native Conformer x-vector extractor (xvb_conformer_*) and the 2x subsampling on the H100: bit-identical to the op-by-op
Python driver of the same kernels (XVB_CONFORMER_NATIVE=0) over every golden case and position of both subsamplings and
a grid of batch sizes and lengths; the reference's golden embeddings; the stride-(2, 1) head and the stride-1 valid conv
against torch; the new head entry against xvb_subsample_head; workspace reuse; the frame budget; the XVBC0001 model file;
and bin/xvb-extract on Conformer model files without Python."""
import os
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conformer_2sub_oracle as c2
import conformer_oracle as co
from asv_subtools_b200 import kaldi_io
from asv_subtools_b200.model.transformer_xvector import ConformerExtractor, NativeConformerExtractor, TransformerXvector
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
CASES = dict(co.CASES, **c2.CASES)
GOLDEN = {c: ("conformer" if c in co.CASES else "conformer_2sub") for c in CASES}
CASE_POS = [(c, p) for c in ("launcher", "small", "launcher2", "small2") for p in CASES[c][3]]


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _sd(case, golden):
    return co.seeded_state_dict(golden(GOLDEN[case])["keys_" + case], CASES[case][4])


def _model(case, pos, golden):
    kwargs, fdim = CASES[case][:2]
    m = TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(_sd(case, golden), strict=True)
    return m.cuda().eval()


def _extractor(monkeypatch, case, pos, golden, native):
    monkeypatch.setenv("XVB_CONFORMER_NATIVE", "1" if native else "0")
    ex = _model(case, pos, golden).extractor()
    assert isinstance(ex, NativeConformerExtractor if native else ConformerExtractor)
    return ex


def _feats(b, t, fdim, seed):
    return torch.from_numpy(onn.synthetic_feats(b, t, fdim, seed)).cuda()


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_native_equals_python_driver_bit_for_bit(monkeypatch, golden, case, pos):
    fdim = CASES[case][1]
    native = _extractor(monkeypatch, case, pos, golden, True)
    driver = _extractor(monkeypatch, case, pos, golden, False)
    with torch.no_grad():
        for b in (1, 3, 64):
            for t in (7, 8, 37, 300):
                x = _feats(b, t, fdim, 1000 * b + t)
                got, want = native.extract(x), driver.extract(x)
                assert got.shape == (b, native.embed_dim) and native.embed_dim == driver.embed_dim
                assert torch.equal(got, want), (case, pos, b, t, (got - want).abs().max().item())
                assert native.last_launches == driver.last_launches, (native.last_launches, driver.last_launches)


@pytest.mark.parametrize("case, pos", [("launcher", "near"), ("launcher2", "near"), ("small2", "far")])
def test_native_equals_python_driver_through_the_chunk_rule(monkeypatch, golden, case, pos):
    fdim = CASES[case][1]
    models = {}
    for native in (True, False):
        monkeypatch.setenv("XVB_CONFORMER_NATIVE", "1" if native else "0")
        models[native] = _model(case, pos, golden)
        models[native].extractor()    # built while the switch is set
    for t in (650, 899):
        x = onn.synthetic_feats(3, t, fdim, 77 + t)
        got, want = models[True].extract_embedding_batch(x), models[False].extract_embedding_batch(x)
        assert isinstance(models[True].extractor(), NativeConformerExtractor)
        assert isinstance(models[False].extractor(), ConformerExtractor)
        assert torch.equal(got, want), (case, t)


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_native_matches_reference_golden(monkeypatch, golden, case, pos):
    g = golden(GOLDEN[case])
    monkeypatch.setenv("XVB_CONFORMER_NATIVE", "1")
    m = _model(case, pos, golden)
    _, fdim, frames, _, _, fseed = CASES[case]
    for t in frames:
        feats = onn.synthetic_feats(2, t, fdim, fseed + t)
        got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
        ref = g["{}_{}_T{}".format(case, pos, t)]
        cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
        assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (case, pos, t, rel(got, ref), cos)
        batch = m.extract_embedding_batch(feats).cpu().numpy()
        assert rel(batch, ref) <= 1e-4, (case, pos, t, rel(batch, ref))


def test_2sub_head_and_valid_conv_vs_torch():
    """C = 256, F = 78 (so F'' = 74 after both convs): the stride-(2, 1) head and the stride-1 unpadded conv against
    F.conv2d in fp32."""
    from asv_subtools_b200 import ops
    torch.manual_seed(5)
    B, T, Fd, C = 3, 41, 78, 256
    x = torch.randn(B, T, Fd, device="cuda")
    w0, b0 = torch.randn(C, 1, 3, 3, device="cuda") / 3, 0.1 * torch.randn(C, device="cuda")
    w2, b2 = torch.randn(C, C, 3, 3, device="cuda") / 48, 0.1 * torch.randn(C, device="cuda")
    T1, F1 = (T - 1) // 2, Fd - 2
    y1 = ops.SplitPlanes.empty((B, T1, F1, C), "cuda")
    ops.subsample_head(x, w0, b0, y1, stride_f=1)
    ref1 = F.relu(F.conv2d(x.unsqueeze(1), w0, b0, stride=(2, 1))).permute(0, 2, 3, 1)
    assert rel(y1.float().cpu(), ref1.cpu()) <= 3e-5, rel(y1.float().cpu(), ref1.cpu())
    y2 = ops.SplitPlanes.empty((B, T1 - 2, F1 - 2, C), "cuda")
    ops.conv2d(y1, ops.pack_conv2d_weight(w2.transpose(2, 3).contiguous()), C, 3, 1, torch.ones(C, device="cuda"), b2,
               relu=True, y=y2, valid=True)
    ref2 = F.relu(F.conv2d(y1.float().permute(0, 3, 1, 2), w2, b2)).permute(0, 2, 3, 1)
    assert rel(y2.float().cpu(), ref2.cpu()) <= 3e-5, rel(y2.float().cpu(), ref2.cpu())


@pytest.mark.parametrize("B, T, Fd", [(3, 37, 80), (2, 300, 23), (1, 7, 3)])
def test_head_stride_entry_equals_subsample_head(B, T, Fd):
    from asv_subtools_b200 import ops
    torch.manual_seed(T)
    C = 64
    x = torch.randn(B, T, Fd, device="cuda")
    w, b = torch.randn(C, 1, 3, 3, device="cuda"), torch.randn(C, device="cuda")
    shape = (B, (T - 1) // 2, (Fd - 1) // 2, C)
    old, new = ops.SplitPlanes.empty(shape, "cuda"), ops.SplitPlanes.empty(shape, "cuda")
    ops.subsample_head(x, w, b, old)
    ops.subsample_head(x, w, b, new, stride_f=2)
    assert torch.equal(old.hi, new.hi) and torch.equal(old.lo, new.lo)


def test_workspace_reuse_across_shapes(monkeypatch, golden):
    ex = _extractor(monkeypatch, "launcher2", "near", golden, True)
    big, small = _feats(64, 300, 80, 1), _feats(3, 37, 80, 2)
    results = [ex.extract(big).clone(), ex.extract(small).clone(), ex.extract(big).clone()]
    for x, got in zip((big, small, big), results):
        fresh = NativeConformerExtractor(_model("launcher2", "near", golden))
        assert torch.equal(got, fresh.extract(x))
        fresh.close()


def test_frame_budget_groups(monkeypatch, golden):
    """150 x 300 frames is over the 128 * 300 frame budget: the call runs as groups of 128 and 22 utterances and equals
    those two calls."""
    ex = _extractor(monkeypatch, "launcher", "near", golden, True)
    x = _feats(150, 300, 80, 3)
    whole = ex.extract(x)
    assert torch.equal(whole, torch.cat([ex.extract(x[:128].contiguous()), ex.extract(x[128:].contiguous())]))


def test_too_short_and_too_long_chunks_are_refused(monkeypatch, golden):
    ex = _extractor(monkeypatch, "small2", "near", golden, True)
    with pytest.raises(RuntimeError, match="at least 7 frames"):
        ex.extract(_feats(1, 6, 23, 4))
    with pytest.raises(RuntimeError, match="5000"):
        ex.extract(_feats(1, 2 * 5003, 23, 4))   # T' = 5000
    driver = _extractor(monkeypatch, "small2", "near", golden, False)
    with pytest.raises(ValueError, match="5000"):
        driver.extract(_feats(1, 2 * 5003, 23, 4))


@pytest.mark.parametrize("case, pos", [("launcher", "near"), ("launcher2", "near_affine"), ("small2", "far"),
                                       ("small", "near")])
def test_model_file_roundtrip_and_rejects(monkeypatch, golden, tmp_path, case, pos):
    ex = _extractor(monkeypatch, case, pos, golden, True)
    path = str(tmp_path / "conformer.xvbm")
    ex.save(path)
    with open(path, "rb") as f:
        assert f.read(8) == b"XVBC0001"
    loaded = NativeConformerExtractor.load(path)
    fdim = CASES[case][1]
    assert loaded.feat_dim == fdim and loaded.embed_dim == ex.embed_dim
    x = _feats(5, 120, fdim, 6)
    assert torch.equal(loaded.extract(x), ex.extract(x))
    loaded.close()
    data = open(path, "rb").read()
    bad = str(tmp_path / "bad.xvbm")
    inconsistent = bytearray(data)
    inconsistent[8:12] = np.int32(fdim + 8).tobytes()     # feat_dim no longer matches the subsampling Linear
    for blob, msg in ((data[:len(data) // 2], "truncated|corrupt"), (data[:20], "XVBC0001"),
                      (b"XVBR0001" + data[8:], "XVBC0001"), (bytes(inconsistent), "out.0")):
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=msg):
            NativeConformerExtractor.load(bad)


@pytest.mark.parametrize("case", ["launcher", "launcher2"])
def test_xvb_extract_binary_runs_a_conformer_model_file(monkeypatch, golden, tmp_path, case):
    """XVBC0001 model file -> bin/xvb-extract with its default max-chunk (300): mixed lengths 310, 650, 120, 120, 7 and
    899 frames against the oracle under the reference's chunk rule; then a 6-frame utterance ends in ERROR, status 1."""
    kwargs, fdim = CASES[case][:2]
    pos = "near"
    ex = _extractor(monkeypatch, case, pos, golden, True)
    model = str(tmp_path / "conformer.xvbm")
    ex.save(model)
    sd = _sd(case, golden)
    cfg = co.config(kwargs)
    oracle = co if case in co.CASES else c2
    feats = {"c{}".format(i): onn.synthetic_feats(1, t, fdim, 300 + i)[0] for i, t in enumerate([310, 650, 120, 120, 7, 899])}
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "xv.ark")
    run = subprocess.run([BIN, "--batch", "4", model, ark, "ark:" + out], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats)
    for k, v in feats.items():
        want = oracle.extract(sd, v, cfg, pos).numpy()
        assert got[k].shape == (ex.embed_dim,) and rel(got[k], want) < 1e-4, (k, rel(got[k], want))
    short = str(tmp_path / "short.ark")
    with open(short, "wb") as f:
        kaldi_io.write_mat(f, onn.synthetic_feats(1, 6, fdim, 9)[0], key="s")
    run = subprocess.run([BIN, model, short, "ark:" + str(tmp_path / "s.ark")], capture_output=True, text=True, timeout=300)
    assert run.returncode == 1 and "ERROR" in run.stderr, run.stderr
