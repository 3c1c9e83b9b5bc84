"""Native RepVGG / RepSPK x-vector extractor (xvb_repvgg_*) on the H100: bit-identical to the op-by-op Python driver of
the same kernels (XVB_REPVGG_NATIVE=0) over every golden case and position in both checkpoint forms and a grid of batch
sizes and lengths, and on a deploy checkpoint whose 18 kept taps need two packing pieces; the reference's golden
embeddings; workspace reuse across shapes; the position budget; the XVBV0001 model file; and bin/xvb-extract on a
RepVGG model without Python."""
import os
import subprocess

import numpy as np
import pytest
import torch

import repvgg_oracle as ro
from asv_subtools_b200 import kaldi_io
from asv_subtools_b200.model.repvgg_xvector import NativeRepVGGExtractor, RepVGGExtractor, RepVggXvector
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
CASE_POS = [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]]
SHAPES = [(b, t) for b in (1, 3, 64) for t in (1, 2, 37, 200)]


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / np.max(np.abs(b)))


def _state_dict(case, deploy=False):
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
    return ro.deploy_state_dict(sd, kwargs) if deploy else sd


def _model(case, pos, deploy=False, sd=None):
    kwargs, fdim, _, _, _, _ = ro.CASES[case]
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding=pos, **({"deploy": True} if deploy else {}), **kwargs)
    m.load_state_dict(sd if sd is not None else _state_dict(case, deploy), strict=True)
    return m.cuda().eval()


def _extractor(monkeypatch, case, pos, native, deploy=False, sd=None):
    monkeypatch.setenv("XVB_REPVGG_NATIVE", "1" if native else "0")
    ex = _model(case, pos, deploy, sd).extractor()
    assert isinstance(ex, NativeRepVGGExtractor if native else RepVGGExtractor)
    return ex


def _feats(b, t, fdim, seed):
    return torch.from_numpy(onn.synthetic_feats(b, t, fdim, seed)).cuda()


def _twins_equal(native, twin, fdim, shapes, tag):
    with torch.no_grad():
        for b, t in shapes:
            x = _feats(b, t, fdim, 1000 * b + t)
            got, want = native.extract(x), twin.extract(x)
            assert got.shape == (b, native.embed_dim) and native.embed_dim == twin.embed_dim
            assert torch.equal(got, want), (tag, b, t, (got - want).abs().max().item())


@pytest.mark.parametrize("deploy", [False, True])
@pytest.mark.parametrize("case, pos", CASE_POS)
def test_native_equals_python_twin_bit_for_bit(monkeypatch, case, pos, deploy):
    fdim, frames = ro.CASES[case][1], ro.CASES[case][2]
    native = _extractor(monkeypatch, case, pos, True, deploy)
    twin = _extractor(monkeypatch, case, pos, False, deploy)
    _twins_equal(native, twin, fdim, [(2, t) for t in frames] + SHAPES, (case, pos, deploy))
    if case == "repspk":
        # the head, 21 blocks, the pooling and fc2 (plus fc2's split-K reduce where the kernel takes it)
        for b, t in ((1, 1), (64, 200)):
            native.extract(_feats(b, t, fdim, 5))
            print("repvgg native launches B={} T={}: {}".format(b, t, native.last_launches))
            assert native.last_launches >= 24


def test_deploy_checkpoint_with_a_nonzero_off_pattern_tap(monkeypatch):
    """One block keeps 18 taps, more than one xvb_pack_tdnn_weight call takes: the library packs it in two pieces."""
    kwargs, fdim, _, _, _, _ = ro.CASES["repspk"]
    dsd = _state_dict("repspk", deploy=True)
    key = "repvgg.stage3.2.rbr_reparam.weight"
    dsd[key] = dsd[key].clone()
    dsd[key][5, 7, 0, 1] = 0.25
    native = _extractor(monkeypatch, "repspk", "near", True, True, dsd)
    twin = _extractor(monkeypatch, "repspk", "near", False, True, dsd)
    assert [len(b["taps"]) for b in twin.blocks].count(18) == 1
    _twins_equal(native, twin, fdim, [(1, 1), (3, 37), (64, 200)], "off-pattern")


# The launcher's model at T = 200 and T = 37 misses the 1e-4 bound by the recorded 1.1e-4 (test_gpu_repvgg.py's
# _MISSES): the handle is bit-identical to the driver, so it carries the same strict expected failures.
_MISSES = {(tag, "near", t) for tag in ("repspk", "repspk_deploy") for t in (200, 37)}


def _golden_params(tag, case):
    _, _, frames, positions, _, _ = ro.CASES[case]
    return [pytest.param(case, p, t, marks=pytest.mark.xfail(strict=True, reason="measured 1.1e-4 > 1e-4, see _MISSES"))
            if (tag, p, t) in _MISSES else (case, p, t) for p in positions for t in frames]


def _check_golden(g, ex, tag, fdim, t, pos, fseed):
    feats = _feats(2, t, fdim, fseed + t)
    got = torch.cat([ex.extract(feats[i:i + 1].contiguous()) for i in range(2)]).cpu().numpy()
    ref = g["{}_{}_T{}".format(tag, pos, t)]
    cos = np.sum(got * ref, 1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    assert rel(got, ref) <= 1e-4 and cos.min() >= 1 - 1e-6, (tag, pos, t, rel(got, ref), cos)


@pytest.mark.parametrize("case, pos, t", [x for c in sorted(ro.CASES) for x in _golden_params(c, c)])
def test_native_matches_reference_golden(monkeypatch, golden, case, pos, t):
    _, fdim, _, _, _, fseed = ro.CASES[case]
    _check_golden(golden("repvgg"), _extractor(monkeypatch, case, pos, True), case, fdim, t, pos, fseed)


@pytest.mark.parametrize("case, pos, t", _golden_params(ro.DEPLOY_CASE + "_deploy", ro.DEPLOY_CASE))
def test_native_deploy_form_matches_reference_golden(monkeypatch, golden, case, pos, t):
    _, fdim, _, _, _, fseed = ro.CASES[case]
    ex = _extractor(monkeypatch, case, pos, True, deploy=True)
    _check_golden(golden("repvgg"), ex, case + "_deploy", fdim, t, pos, fseed)


def test_workspace_reuse_across_shapes(monkeypatch):
    ex = _extractor(monkeypatch, "repspk", "near", True)
    big, small = _feats(64, 200, 80, 1), _feats(3, 37, 80, 2)
    results = [ex.extract(big).clone(), ex.extract(small).clone(), ex.extract(big).clone()]
    for x, got in zip((big, small, big), results):
        fresh = NativeRepVGGExtractor(_model("repspk", "near"))
        assert torch.equal(got, fresh.extract(x))
        fresh.close()


def test_position_budget_groups(monkeypatch):
    """60 x 1000 frames x 80 bins is over the 256 * 200 * 80 position budget: the call runs as groups of 51 and 9
    utterances and equals those two calls."""
    ex = _extractor(monkeypatch, "repspk", "near", True)
    x = _feats(60, 1000, 80, 3)
    whole = ex.extract(x)
    assert torch.equal(whole, torch.cat([ex.extract(x[:51].contiguous()), ex.extract(x[51:].contiguous())]))


@pytest.mark.parametrize("case, pos", [("repspk", "near"), ("a0", "far")])
def test_model_file_roundtrip_and_rejects(monkeypatch, tmp_path, case, pos):
    ex = _extractor(monkeypatch, case, pos, True)
    path = str(tmp_path / "repvgg.xvbm")
    ex.save(path)
    data = open(path, "rb").read()
    assert data[:8] == b"XVBV0001"
    loaded = NativeRepVGGExtractor.load(path)
    fdim = ro.CASES[case][1]
    assert loaded.feat_dim == fdim and loaded.embed_dim == ex.embed_dim
    x = _feats(5, 120, fdim, 6)
    assert torch.equal(loaded.extract(x), ex.extract(x))
    loaded.close()
    bad = str(tmp_path / "bad.xvbm")
    ksize = bytearray(data)
    assert ksize[12] in (3, 5)
    ksize[12] = 8 - ksize[12]                          # the configuration's ksize (5 <-> 3) contradicts every block
    for blob, word in ((data[:len(data) // 2], "truncated or corrupt"), (data[:8 + 68], "not an XVBV0001 file"),
                       (b"XVBR0001" + data[8:], "not an XVBV0001 file"), (bytes(ksize), "record 'repvgg.stage0'")):
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=word):
            NativeRepVGGExtractor.load(bad)


def _chunks(t, max_chunk):
    n = (t + max_chunk - 1) // max_chunk
    split = t // n
    return [split] * (n - 1) + [t - split * (n - 1)]


@pytest.mark.parametrize("case", ["a0", "repspk"])
def test_xvb_extract_binary_runs_a_repvgg_model_file(monkeypatch, tmp_path, case):
    """XVBV0001 model file -> bin/xvb-extract: mixed lengths 120, 120, 75, 1 and 130 frames at --max-chunk 50 (chunks of
    40, 37 / 38, 1 and 43 / 44 frames, batched by length) against the oracle forward under the chunk rule (a0 within
    1e-4; the launcher's RepSPK model in cosine, see _MISSES) and against the handle's own per-chunk embeddings."""
    kwargs, fdim, _, _, _, _ = ro.CASES[case]
    pos = "near"
    ex = _extractor(monkeypatch, case, pos, True)
    model = str(tmp_path / "repvgg.xvbm")
    ex.save(model)
    sd = _state_dict(case)
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
        assert got[k].shape == (ex.embed_dim,)
        want = onn.extract_embedding(lambda x: ro.repvgg_forward(sd, x, pos, kwargs), v, max_chunk=50).numpy()
        if case == "a0":
            assert rel(got[k], want) < 1e-4, (k, rel(got[k], want))
        else:
            assert np.dot(got[k], want) / (np.linalg.norm(got[k]) * np.linalg.norm(want)) >= 1 - 1e-6, k
        acc, off = np.zeros(ex.embed_dim, np.float32), 0
        for n in _chunks(len(v), 50):
            acc += np.float32(n) * ex.extract(torch.from_numpy(v[None, off:off + n]).cuda()).cpu().numpy()[0]
            off += n
        assert rel(got[k], acc / np.float32(len(v))) <= 1e-6, (k, rel(got[k], acc / np.float32(len(v))))
