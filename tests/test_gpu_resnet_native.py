"""Native ResNet x-vector extractor (xvb_resnet_*) on the H100: bit-identical to the op-by-op Python driver of the same
kernels (XVB_RESNET_NATIVE=0) over every golden case, position and a grid of batch sizes and lengths; the reference's
golden embeddings; workspace reuse across shapes; the position budget; the shard calls on one and two lanes; the XVBR0001
model file; and bin/xvb-extract on a ResNet model without Python."""
import os
import subprocess

import numpy as np
import pytest
import torch

import resnet_oracle as ro
from asv_subtools_b200 import kaldi_io
from asv_subtools_b200.model.resnet_xvector import NativeResNetExtractor, ResNetExtractor, ResNetXvector
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
CASE_POS = [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _model(case, pos):
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    m = ResNetXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed), strict=True)
    return m.cuda().eval()


def _extractor(monkeypatch, case, pos, native):
    monkeypatch.setenv("XVB_RESNET_NATIVE", "1" if native else "0")
    ex = _model(case, pos).extractor()
    assert isinstance(ex, NativeResNetExtractor if native else ResNetExtractor)
    return ex


def _feats(b, t, fdim, seed):
    return torch.from_numpy(onn.synthetic_feats(b, t, fdim, seed)).cuda()


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_native_equals_python_twin_bit_for_bit(monkeypatch, case, pos):
    fdim, frames = ro.CASES[case][1], ro.CASES[case][2]
    native = _extractor(monkeypatch, case, pos, True)
    twin = _extractor(monkeypatch, case, pos, False)
    shapes = [(2, t) for t in frames] + [(b, t) for b in (1, 3, 64) for t in (1, 2, 37, 200)]
    with torch.no_grad():
        for b, t in shapes:
            x = _feats(b, t, fdim, 1000 * b + t)
            got, want = native.extract(x), twin.extract(x)
            assert got.shape == (b, native.embed_dim) and native.embed_dim == twin.embed_dim
            assert torch.equal(got, want), (case, pos, b, t, (got - want).abs().max().item())


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_native_matches_reference_golden(monkeypatch, golden, case, pos):
    g = golden("resnet")
    _, fdim, frames, _, _, fseed = ro.CASES[case]
    ex = _extractor(monkeypatch, case, pos, True)
    for t in frames:
        got = ex.extract(torch.from_numpy(onn.synthetic_feats(2, t, fdim, fseed + t)).cuda()).cpu().numpy()
        ref = g["{}_{}_T{}".format(case, pos, t)]
        cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
        assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (case, pos, t, rel(got, ref), cos)


def test_workspace_reuse_across_shapes(monkeypatch):
    ex = _extractor(monkeypatch, "online", "near", True)
    big, small = _feats(64, 200, 80, 1), _feats(3, 37, 80, 2)
    wide = _feats(96, 20, 80, 5)   # the batch grows, the positions shrink: only the per-utterance buffers grow
    results = [ex.extract(big).clone(), ex.extract(small).clone(), ex.extract(big).clone(), ex.extract(wide).clone()]
    for x, got in zip((big, small, big, wide), results):
        fresh = NativeResNetExtractor(_model("online", "near"))
        assert torch.equal(got, fresh.extract(x))
        fresh.close()


def test_position_budget_groups(monkeypatch):
    """60 x 1000 frames x 80 bins is over the 256 * 200 * 80 position budget: the call runs as groups of 51 and 9
    utterances and equals those two calls."""
    ex = _extractor(monkeypatch, "online", "near", True)
    x = _feats(60, 1000, 80, 3)
    whole = ex.extract(x)
    assert torch.equal(whole, torch.cat([ex.extract(x[:51].contiguous()), ex.extract(x[51:].contiguous())]))


@pytest.mark.parametrize("lanes", ["0", "1"])
def test_shard_calls_equal_batch_calls(monkeypatch, lanes):
    monkeypatch.setenv("XVB_LANES", lanes)
    ex = _extractor(monkeypatch, "online", "near", True)
    x = _feats(11, 50, 80, 4)
    want = torch.cat([ex.extract(x[i:i + 4].contiguous()) for i in (0, 4, 8)])
    assert ex.last_launches >= 90
    for _ in range(2):
        assert torch.equal(ex.extract_shard(x, batch=4), want)
    feats = torch.empty(11, 50, 80, pin_memory=True)
    feats.copy_(x.cpu())
    emb = torch.empty(11, ex.embed_dim, pin_memory=True)
    for _ in range(2):
        emb.zero_()
        ex.extract_shard_host(feats.data_ptr(), 11, 50, emb.data_ptr(), batch=4)
        assert torch.equal(emb, want.cpu())


@pytest.mark.parametrize("case, pos", [("online", "near"), ("preact", "far")])
def test_model_file_roundtrip_and_rejects(monkeypatch, tmp_path, case, pos):
    ex = _extractor(monkeypatch, case, pos, True)
    path = str(tmp_path / "resnet.xvbm")
    ex.save(path)
    with open(path, "rb") as f:
        assert f.read(8) == b"XVBR0001"
    loaded = NativeResNetExtractor.load(path)
    fdim = ro.CASES[case][1]
    assert loaded.feat_dim == fdim and loaded.embed_dim == ex.embed_dim == 256
    x = _feats(5, 120, fdim, 6)
    assert torch.equal(loaded.extract(x), ex.extract(x))
    loaded.close()
    data = open(path, "rb").read()
    bad = str(tmp_path / "bad.xvbm")
    for blob in (data[:len(data) // 2], data[:20], b"XVBE0001" + data[8:]):
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match="XVBR0001|truncated|corrupt"):
            NativeResNetExtractor.load(bad)


@pytest.mark.parametrize("case", ["online", "preact"])
def test_xvb_extract_binary_runs_a_resnet_model_file(monkeypatch, tmp_path, case):
    """XVBR0001 model file -> bin/xvb-extract: mixed lengths 120, 120, 75, 1 and 130 frames at --max-chunk 50 (chunks of
    40, 37 / 38, 1 and 43 / 44 frames, batched by length) against the oracle forward under the chunk rule."""
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    pos = "near"
    ex = _extractor(monkeypatch, case, pos, True)
    model = str(tmp_path / "resnet.xvbm")
    ex.save(model)
    sd = onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed)
    feats = {"r{}".format(i): onn.synthetic_feats(1, t, fdim, 400 + i)[0] for i, t in enumerate([120, 120, 75, 1, 130])}
    ark = str(tmp_path / "feats.ark")
    with open(ark, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)
    out = str(tmp_path / "xv.ark")
    run = subprocess.run([BIN, "--batch", "4", "--max-chunk", "50", model, ark, "ark:" + out], capture_output=True,
                         text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats)
    for k, v in feats.items():
        want = onn.extract_embedding(lambda x: ro.resnet_forward(sd, x, pos, kwargs), v, max_chunk=50).numpy()
        assert got[k].shape == (256,) and rel(got[k], want) < 1e-4, (k, rel(got[k], want))
