"""Native CAM++ x-vector extractor (xvb_campp_*) on the H100: bit-identical to the op-by-op Python driver of the same
kernels (XVB_CAMPP_NATIVE=0) over both golden configs and a grid of batch sizes and lengths, and through egrecho's chunk
rule; the reference's golden embeddings; workspace reuse across layouts (the time-padded head copy's zero frames); the
frame budget; input refusals; the XVBP0001 model file; and bin/xvb-extract on CAM++ model files without Python."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import campplus_oracle as co  # noqa: E402
from asv_subtools_b200 import kaldi_io  # noqa: E402
from asv_subtools_b200.model.campplus_xvector import (CamPPExtractor, CamPPXvector, NativeCamPPExtractor,  # noqa: E402
                                                      chunk_sizes)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
GOLDEN = np.load(os.path.join(HERE, "golden", "campplus.npz"))


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _sd(case):
    return co.seeded_state_dict(GOLDEN["keys_" + case], co.CASES[case][3])


def _model(case):
    kw = dict(co.CASES[case][0])
    m = CamPPXvector(kw.pop("inputs_dim"), 10, **kw)
    m.load_state_dict(_sd(case), strict=True)
    return m.cuda().eval()


def _extractor(monkeypatch, case, native):
    monkeypatch.setenv("XVB_CAMPP_NATIVE", "1" if native else "0")
    ex = _model(case).extractor()
    assert isinstance(ex, NativeCamPPExtractor if native else CamPPExtractor)
    return ex


def _feats(b, t, fdim, seed):
    return co.utterances(b, t, fdim, seed).cuda()


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_native_equals_python_driver_bit_for_bit(monkeypatch, case):
    fdim = co.CASES[case][0]["inputs_dim"]
    native = _extractor(monkeypatch, case, True)
    driver = _extractor(monkeypatch, case, False)
    with torch.no_grad():
        for b in (1, 3, 64):
            for t in (3, 4, 37, 200, 201, 300):     # 201: a one-frame last CAM segment
                x = _feats(b, t, fdim, 1000 * b + t)
                got, want = native.extract(x), driver.extract(x)
                assert got.shape == (b, native.embed_dim) and native.embed_dim == driver.embed_dim
                assert torch.equal(got, want), (case, b, t, (got - want).abs().max().item())
                assert native.last_launches == driver.last_launches, (native.last_launches, driver.last_launches)
    if case == "default":
        assert native.last_launches == 284


def test_native_equals_python_driver_through_the_chunk_rule(monkeypatch):
    models = {}
    for native in (True, False):
        monkeypatch.setenv("XVB_CAMPP_NATIVE", "1" if native else "0")
        models[native] = _model("default")
        models[native].extractor()    # built while the switch is set
    for t in (4001, 9000):
        x = co.utterances(3, t, 80, 77 + t)
        got, want = models[True].extract_embedding_batch(x), models[False].extract_embedding_batch(x)
        assert isinstance(models[True].extractor(), NativeCamPPExtractor)
        assert isinstance(models[False].extractor(), CamPPExtractor)
        assert torch.equal(got, want), t


GOLDEN_CASES = [(case, t) for case, (_, frames, long_frames, _, _) in co.CASES.items() for t in frames + long_frames]


@pytest.mark.parametrize("case,t", GOLDEN_CASES)
def test_native_matches_reference_golden(monkeypatch, case, t):
    cfg, _, _, _, fseed = co.CASES[case]
    m = _model(case)
    monkeypatch.setenv("XVB_CAMPP_NATIVE", "1")
    assert isinstance(m.extractor(), NativeCamPPExtractor)
    feats = co.utterances(2, t, cfg["inputs_dim"], fseed + t)
    ref = GOLDEN["{}_T{}".format(case, t)]
    got = np.stack([m.extract_embedding(feats[i]).numpy() for i in range(2)])
    cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (case, t, rel(got, ref), cos)


def test_workspace_reuse_across_layouts(monkeypatch):
    """64x300, 3x37, 5x201, 64x300 on one handle, each equal to a fresh handle's output: a pad frame of the time-padded
    head copy left over from an earlier layout would change the tdnn output."""
    ex = _extractor(monkeypatch, "default", True)
    shapes = [(64, 300), (3, 37), (5, 201), (64, 300)]
    xs = [_feats(b, t, 80, 10 + i) for i, (b, t) in enumerate(shapes)]
    results = [ex.extract(x).clone() for x in xs]
    m = _model("default")
    for x, got in zip(xs, results):
        fresh = NativeCamPPExtractor(m)
        assert torch.equal(got, fresh.extract(x)), tuple(x.shape)
        fresh.close()


def test_frame_budget_groups(monkeypatch):
    """150 x 300 frames is over the 128 * 300 frame budget: the call runs as groups of 128 and 22 utterances and equals
    those two calls; 10 x 4000 runs one utterance per group and equals the per-utterance calls."""
    ex = _extractor(monkeypatch, "default", True)
    x = _feats(150, 300, 80, 3)
    whole = ex.extract(x)
    assert torch.equal(whole, torch.cat([ex.extract(x[:128].contiguous()), ex.extract(x[128:].contiguous())]))
    x = _feats(10, 4000, 80, 4)
    whole = ex.extract(x)
    assert torch.equal(whole, torch.cat([ex.extract(x[i:i + 1].contiguous()) for i in range(10)]))


def test_input_refusals(monkeypatch):
    ex = _extractor(monkeypatch, "small", True)
    with pytest.raises(RuntimeError, match="at least 3 frames"):
        ex.extract(_feats(2, 2, 40, 5))
    with pytest.raises(ValueError, match="feature dim"):
        ex.extract(_feats(2, 50, 80, 5))


@pytest.mark.parametrize("case", sorted(co.CASES))
def test_model_file_roundtrip_and_rejects(monkeypatch, tmp_path, case):
    ex = _extractor(monkeypatch, case, True)
    fdim = co.CASES[case][0]["inputs_dim"]
    path = str(tmp_path / "campplus.xvbm")
    ex.save(path)
    with open(path, "rb") as f:
        assert f.read(8) == b"XVBP0001"
    loaded = NativeCamPPExtractor.load(path)
    assert loaded.feat_dim == fdim and loaded.embed_dim == ex.embed_dim
    x = _feats(5, 120, fdim, 6)
    assert torch.equal(loaded.extract(x), ex.extract(x))
    loaded.close()
    data = open(path, "rb").read()
    bad = str(tmp_path / "bad.xvbm")
    inconsistent = bytearray(data)
    inconsistent[8:12] = np.int32(fdim + 8).tobytes()     # feat_dim no longer matches the tdnn's im2col width
    for blob, msg in ((data[:len(data) // 2], "truncated|corrupt"), (data[:20], "XVBP0001"),
                      (b"XVBC0001" + data[8:], "XVBP0001"), (bytes(inconsistent), "xvector.tdnn.linear")):
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=msg):
            NativeCamPPExtractor.load(bad)


def _write_ark(path, feats):
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, np.ascontiguousarray(v, dtype=np.float32), key=k)


def _run(args, timeout=900):
    return subprocess.run([BIN] + args, capture_output=True, text=True, timeout=timeout)


def test_xvb_extract_binary_runs_a_campplus_model_file(monkeypatch, tmp_path):
    """XVBP0001 file -> bin/xvb-extract --batch 4 with the default 4000-frame chunk rule: the golden utterances of the
    default config (3 .. 9000 frames) against the reference's embeddings; a 2-frame utterance ends in ERROR, status 1."""
    ex = _extractor(monkeypatch, "default", True)
    model = str(tmp_path / "campplus.xvbm")
    ex.save(model)
    feats, want = {}, {}
    for t in (300, 200, 201, 37, 3, 4001, 9000):
        x = co.utterances(2, t, 80, 800 + t).numpy()
        for i in range(2):
            feats["u{}_{}".format(t, i)] = x[i]
            want["u{}_{}".format(t, i)] = GOLDEN["default_T{}".format(t)][i]
    ark, out = str(tmp_path / "feats.ark"), str(tmp_path / "xv.ark")
    _write_ark(ark, feats)
    run = _run(["--batch", "4", model, ark, "ark:" + out])
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(got) == sorted(feats)
    for k in feats:
        assert got[k].shape == (512,) and rel(got[k], want[k]) <= 1e-4, (k, rel(got[k], want[k]))
    short = str(tmp_path / "short.ark")
    _write_ark(short, {"s": co.utterances(1, 2, 80, 9).numpy()[0]})
    run = _run([model, short, "ark:" + str(tmp_path / "s.ark")], timeout=300)
    assert run.returncode == 1 and "ERROR" in run.stderr, run.stderr


def test_xvb_extract_small_config_and_max_chunk(monkeypatch, tmp_path):
    """The small config at 40-d through the binary; --max-chunk 1000 on a 2600-frame utterance keeps egrecho's rule
    (1000, 800, 800) and matches the oracle forward over those chunks."""
    ex = _extractor(monkeypatch, "small", True)
    model = str(tmp_path / "small.xvbm")
    ex.save(model)
    feats = {"u{}_{}".format(t, i): co.utterances(2, t, 40, 850 + t).numpy()[i] for t in (150, 4) for i in range(2)}
    feats["long"] = co.utterances(1, 2600, 40, 5).numpy()[0]
    ark, out = str(tmp_path / "feats.ark"), str(tmp_path / "xv.ark")
    _write_ark(ark, feats)
    run = _run(["--max-chunk", "1000", model, ark, "ark:" + out])
    assert run.returncode == 0, run.stdout + run.stderr
    got = dict(kaldi_io.read_vec_flt_ark(out))
    for t in (150, 4):
        for i in range(2):
            k = "u{}_{}".format(t, i)
            assert rel(got[k], GOLDEN["small_T{}".format(t)][i]) <= 1e-4, k
    sd = _sd("small")
    x = torch.from_numpy(feats["long"])[None]
    sizes = chunk_sizes(2600, 1000)
    assert sizes == [1000, 800, 800]
    acc, off = None, 0
    with torch.no_grad():
        for s in sizes:
            e = co.forward(sd, x[:, off:off + s])
            acc = e * s if acc is None else acc + s * e
            off += s
    want = (acc / 2600)[0].numpy()
    assert rel(got["long"], want) <= 1e-4, rel(got["long"], want)
