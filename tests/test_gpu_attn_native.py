"""The native TDNN handle with an attention pooling (xvb_extractor_set_attention_pooling): the attentive, multi-head,
multi-resolution and xi-vector models of tests/test_gpu_attn_mixed_lengths.py, built by AttentionPoolingExtractor.native()
from the records its own sequence packed.  Needs an H100 (`-m gpu`).

  * Equal-length and masked batches: torch.equal with AttentionPoolingExtractor.extract at every position; pad content;
    every length equal to T; a call over the frame budget against its groups; masked and unmasked calls alternating on
    one workspace; bad lengths refused by the C entry and by Python, with nothing written.
  * The host-buffer, shard and gather entry points run the attention tail.
  * XVBM0002 files: bytes against an independent writer, load + save round trip, truncated layers refused, the snowdar
    goldens through saved files and bin/xvb-extract (with and without --mixed-lengths) against the goldens and the Python
    CLI; LDE refuses native() and save().
  * Statistics-pooling handles: embeddings equal to the op-by-op sequence of the same kernels, and the launches that
    sequence makes."""
import ctypes as C
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import attn_native_layout as lay  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
EINVAL = -1
EMB_TOL = 1e-4
BUDGET = 256 * 300   # frames per group of an attention model's extract call (extractor.cu kAttnFrameBudget)

# the models of tests/test_gpu_attn_mixed_lengths.py (seeds of tests/golden/make_golden_snowdar.py)
POOLING_CASES = {
    "attn1": ("attentive", {}, 311),
    "attn2": ("attentive", {"affine_layers": 2, "hidden_size": 64}, 312),
    "mha_share": ("multi-head", {"num_head": 4}, 313),
    "mha_full": ("multi-head", {"num_head": 4, "share": False, "affine_layers": 2}, 314),
    "mres": ("multi-resolution", {"num_head": 4, "temperature": True, "affine_layers": 2}, 315),
    "xi_mean": ("xi-postmean-softplus2", {"hidden_size": 64, "num_nodes": 200}, 319),
    "xi_dist": ("xi-postdist-softplus2", {"hidden_size": 64, "num_nodes": 200}, 320),
}
NAMES = sorted(POOLING_CASES)
POSITIONS = ["far", "near_affine", "near"]   # snowdar's "near" is the whole last layer (near_full)
_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    for v in _CACHE.values():
        v[3].close()
    _CACHE.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _model(name, pos):
    """(model on the GPU, state_dict, AttentionPoolingExtractor, its native handle)."""
    if (name, pos) not in _CACHE:
        from asv_subtools_b200.model.snowdar_xvector import Xvector
        pooling, pp, seed = POOLING_CASES[name]
        sd = onn.make_state_dict(onn.snowdar_xvector_spec(40, pooling=pooling, pooling_params=pp), seed)
        m = Xvector(40, 10, training=False, extracted_embedding=pos, pooling=pooling, pooling_params=pp)
        m.load_state_dict(sd, strict=True)
        m.cuda().eval()
        py = m.extractor()
        _CACHE[(name, pos)] = (m, sd, py, py.native())
    return _CACHE[(name, pos)]


def _feats(B, T, seed):
    return torch.from_numpy(onn.synthetic_feats(B, T, 40, seed)).cuda()


def _mixed_lengths(seed, B=64, lo=1, hi=300):
    rng = np.random.RandomState(seed)
    lens = rng.randint(lo, hi + 1, B)
    lens[:4] = [1, 2, 3, hi]
    rng.shuffle(lens)
    return [int(v) for v in lens]


def _padded(rows, T, fill=0.0):
    x = np.full((len(rows), T, 40), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


# ================================================================================================ extraction
@pytest.mark.parametrize("pos", POSITIONS)
@pytest.mark.parametrize("name", NAMES)
def test_handle_equals_python_sequence(name, pos):
    _, _, py, nat = _model(name, pos)
    assert nat.embed_dim == py.embed_dim
    for B in (1, 3, 64):
        for T in (1, 2, 37, 200):
            x = _feats(B, T, 7 * B + T)
            assert torch.equal(nat.extract(x), py.extract(x)), (name, pos, B, T)


@pytest.mark.parametrize("pos", POSITIONS)
@pytest.mark.parametrize("name", NAMES)
def test_masked_batch_equals_python_sequence(name, pos):
    _, _, py, nat = _model(name, pos)
    lens = _mixed_lengths(500 + NAMES.index(name) * 3 + POSITIONS.index(pos))
    x = _feats(64, 300, 1500 + NAMES.index(name))
    got = nat.extract(x, lens)
    assert torch.equal(got, py.extract(x, lens)), (name, pos)
    assert torch.equal(nat.extract(x, [300] * 64), nat.extract(x)), (name, pos)    # every length T: the unmasked call
    rows = [r[:n] for r, n in zip(x.cpu().numpy(), lens)]
    for fill in (float("nan"), 1e30, -1e30):
        assert torch.equal(nat.extract(_padded(rows, 300, fill), lens), got), (name, pos, fill)


@pytest.mark.parametrize("name", ["attn2", "xi_dist"])
def test_calls_over_the_frame_budget_run_as_groups(name):
    _, _, _, nat = _model(name, "near")
    B, T = 300, 300                      # 90 000 frames: groups of 256 and 44 utterances
    assert B * T > BUDGET and (BUDGET // T) == 256
    x = _feats(B, T, 99)
    lens = _mixed_lengths(98, B=B)
    lens[256:] = [T] * (B - 256)         # the second group has nothing to mask: it runs unmasked
    want = torch.cat([nat.extract(x[:256].contiguous(), lens[:256]), nat.extract(x[256:].contiguous())])
    assert torch.equal(nat.extract(x, lens), want), name
    want = torch.cat([nat.extract(x[:256].contiguous()), nat.extract(x[256:].contiguous())])
    assert torch.equal(nat.extract(x), want), name


def test_masked_and_unmasked_calls_share_one_workspace():
    _, _, py, nat = _model("mres", "near_affine")
    calls = [(64, 300, True), (3, 37, False), (64, 300, True), (100, 200, False), (16, 500, True), (64, 300, True),
             (1, 2, False)]
    for i, (B, T, masked) in enumerate(calls):
        x = _feats(B, T, 300 + i)
        lens = _mixed_lengths(400 + i, B=B, hi=T) if masked and B >= 4 else None
        assert torch.equal(nat.extract(x, lens), py.extract(x, lens)), (i, B, T, masked)


@pytest.mark.parametrize("name", ["mha_share", "xi_mean"])
def test_bad_lengths_are_refused_and_write_nothing(name):
    from asv_subtools_b200 import _lib
    _, _, py, nat = _model(name, "far")
    x = _feats(3, 20, 5)
    emb = torch.full((3, nat.embed_dim), 7.0, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    for bad, at in (([20, 0, 20], 1), ([20, -3, 20], 1), ([20, 20, 21], 2)):
        lens = np.array(bad, dtype=np.int32)
        rc = _lib.lib.xvb_extractor_extract_lengths(nat._h, C.c_void_p(x.data_ptr()), lens.ctypes.data_as(C.c_void_p), 3, 20,
                                                    C.c_void_p(emb.data_ptr()), stream)
        assert rc == EINVAL and "lengths[{}]".format(at) in _lib.last_error(), (bad, rc, _lib.last_error())
        with pytest.raises(RuntimeError, match=r"lengths\[{}\]".format(at)):
            nat.extract(x, bad)
        with pytest.raises(ValueError, match=r"lengths\[{}\]".format(at)):
            py.extract(x, bad)
    torch.cuda.synchronize()
    assert bool((emb == 7.0).all())


# ================================================================================================ other entry points
def test_host_shard_and_gather_entry_points_run_the_attention_tail():
    _, _, py, nat = _model("xi_dist", "near")
    N, T, batch = 40, 120, 16
    x = _feats(N, T, 2024)
    want = torch.cat([py.extract(x[i:i + batch].contiguous()) for i in range(0, N, batch)])
    assert np.array_equal(nat.extract_host(x[:batch].cpu().numpy()), want[:batch].cpu().numpy())
    assert torch.equal(nat.extract_shard(x, batch=batch), want)
    feats_host = x.cpu().pin_memory()
    emb_host = torch.empty(N, nat.embed_dim).pin_memory()
    nat.extract_shard_host(feats_host.data_ptr(), N, T, emb_host.data_ptr(), batch=batch)
    assert torch.equal(emb_host.cuda(), want)
    table = torch.full((N + 5, nat.embed_dim), 3.0, device="cuda")
    ptrs = (C.c_void_p * 1)(table.data_ptr())
    nat.set_gather(ptrs, 1, 5, nat.embed_dim)
    try:
        out = nat.extract_shard(x, batch=batch)
        torch.cuda.synchronize()
    finally:
        nat.set_gather(None, 0, 0, 0)
    assert torch.equal(out, want) and torch.equal(table[5:], want) and bool((table[:5] == 3.0).all())


# ================================================================================================ model files
def _records(py):
    def host(v):
        return None if v is None else v.detach().float().cpu().numpy()

    def rec(layer):
        w, b, s, t = (host(v) for v in layer.record)
        return w, b, s, t, layer.context, layer.relu

    att = [rec(layer) for layer in (py.first, py.last) if layer is not None]
    if py.xi is not None:
        kind = lay.POOL_XI_POSTDIST if py.xi[2] else lay.POOL_XI_POSTMEAN
        prior, gdiv, unweighted = (host(py.xi[0]), host(py.xi[1])), 1, False
    else:
        kind, prior, gdiv, unweighted = lay.POOL_ATTENTION, None, py.gdiv, py.unweighted
    return lay.xvbm2(py.feat_dim, py.eps, kind, py.pooled, gdiv, unweighted, prior, [rec(f) for f in py.frames], att,
                     [rec(s) for s in py.segment])


@pytest.mark.parametrize("name", NAMES)
def test_model_file_bytes_roundtrip_and_truncation(tmp_path, name):
    from asv_subtools_b200 import ops
    _, _, py, nat = _model(name, "near_affine")
    path, again, bad = (str(tmp_path / n) for n in ("m.xvbm", "again.xvbm", "bad.xvbm"))
    py.save(path)
    data = open(path, "rb").read()
    assert data[:8] == b"XVBM0002" and data == _records(py)
    loaded = ops.Extractor.load(path)
    assert (loaded.feat_dim, loaded.embed_dim) == (40, nat.embed_dim)
    loaded.save(again)
    assert open(again, "rb").read() == data
    x = _feats(5, 77, 8)
    assert torch.equal(loaded.extract(x), nat.extract(x))
    loaded.close()
    for blob, msg in ((data[:-100], "is truncated in layer"), (data[:len(data) // 2], "is truncated in layer")):
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=msg):
            ops.Extractor.load(bad)


def test_lde_has_no_native_handle_or_file(tmp_path):
    from asv_subtools_b200.model.snowdar_xvector import Xvector
    m = Xvector(40, 10, training=False, extracted_embedding="far", pooling="lde")
    m.cuda().eval()
    ex = m.extractor()
    with pytest.raises(NotImplementedError):
        ex.native()
    with pytest.raises(NotImplementedError):
        ex.save(str(tmp_path / "lde.xvbm"))
    assert not os.path.exists(str(tmp_path / "lde.xvbm"))


@pytest.mark.parametrize("name", NAMES)
def test_goldens_through_saved_files(tmp_path, golden, name):
    from asv_subtools_b200 import ops
    g = golden("snowdar")
    rows = onn.synthetic_feats(3, 120, 40, POOLING_CASES[name][2] + 1000)
    for pos in ("far", "near"):
        path = str(tmp_path / "{}.xvbm".format(pos))
        _model(name, pos)[2].save(path)
        ex = ops.Extractor.load(path)
        got = ex.extract(torch.from_numpy(rows).cuda()).cpu().numpy()
        ex.close()
        want = g["{}_{}".format(name, pos)]
        for j in range(3):
            assert rel(got[j], want[j]) <= EMB_TOL, (name, pos, j, rel(got[j], want[j]))


def _write_ark(path, feats):
    from asv_subtools_b200 import kaldi_io
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)


@pytest.mark.parametrize("name", ["attn2", "mres", "xi_dist"])
def test_xvb_extract_on_xvbm0002(tmp_path, golden, name):
    from asv_subtools_b200 import kaldi_io
    m, sd, py, _ = _model(name, "near")
    g = golden("snowdar")["{}_near".format(name)]
    rows = onn.synthetic_feats(3, 120, 40, POOLING_CASES[name][2] + 1000)
    rng = np.random.RandomState(5)
    feats = {"g{}".format(j): rows[j] for j in range(3)}
    feats["long"] = onn.synthetic_feats(1, 10001, 40, 77)[0]    # past the 10 000-frame chunk: 5000 + 5001
    for i, t in enumerate([1, 2, 9] + [int(v) for v in rng.randint(1, 600, 13)]):
        feats["u{:02d}".format(i)] = onn.synthetic_feats(1, t, 40, 900 + i)[0]
    ark, model = str(tmp_path / "feats.ark"), str(tmp_path / "model.xvbm")
    _write_ark(ark, feats)
    py.save(model)
    torch.save(sd, str(tmp_path / "final.params"))
    pooling, pp, _ = POOLING_CASES[name]
    creation = "Xvector(40,10,training=False,extracted_embedding='near',pooling={!r},pooling_params={!r})".format(pooling, pp)
    ref = str(tmp_path / "python.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--model-blueprint",
                        os.path.join(ROOT, "asv_subtools_b200", "model", "snowdar_xvector.py"), "--model-creation", creation,
                        str(tmp_path / "final.params"), "ark:" + ark, "ark:" + ref],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    want = dict(kaldi_io.read_vec_flt_ark(ref))
    for flag in ([], ["--mixed-lengths"]):
        out = str(tmp_path / "cli.ark")
        r = subprocess.run([BIN, "--batch", "8"] + flag + [model, "ark:" + ark, "ark:" + out], capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-3000:]
        assert ("masked batches" in r.stderr) == bool(flag), r.stderr[-2000:]
        got = dict(kaldi_io.read_vec_flt_ark(out))
        assert sorted(got) == sorted(feats)
        for k in feats:
            assert rel(got[k], want[k]) <= 1e-5, (name, flag, k, rel(got[k], want[k]))
        for j in range(3):
            assert rel(got["g{}".format(j)], g[j]) <= EMB_TOL, (name, flag, j)


# ================================================================================================ statistics pooling
def _splitk(cin, cout, B):
    """Whether the layer kernel runs a segment-level layer (T = 1, one tap, no second source) as split-K, which adds one
    reduce launch: at most 1024 rows, at least 24 channel blocks of 64 and Cout % 4 == 0 (tdnn_gemm.cu splitk_slices)."""
    return B <= 1024 and (cin + 63) // 64 >= 24 and cout % 4 == 0


def _stats_sequence(m, frames, tdnn6, tdnn7, pos):
    """The statistics-pooling handle's launch sequence op by op, as run(feats) -> (embeddings, launches): split, frame
    layers, the last one pooling in its epilogue (+ xvb_pool_finalize), segment layers (+ a split-K reduce where the layer
    kernel splits K); every layer packed here, unpadded as the handle packs it."""
    from asv_subtools_b200 import ops
    dev = torch.device("cuda")

    def packed(layer):
        w, b, s, t, relu = layer.export()
        return ops.PackedAffine(w, dev, layer.affine.context, b, s, t, relu=relu)

    def affine(a):
        return ops.PackedAffine(a.dense_weight(), dev, a.context, a.bias)

    layers = [packed(layer) for layer in frames]
    if pos == "far":
        segs = [affine(tdnn6.affine)]
    else:                                # "near_full": the whole tdnn7 (the snowdar x-vector's "near")
        segs = [packed(tdnn6), packed(tdnn7) if pos == "near_full" else affine(tdnn7.affine)]

    def run(feats):
        B, T, F = feats.shape
        x = ops.split_f32(feats, ld=(F + 7) // 8 * 8)
        n = 1
        for L in layers[:-1]:
            y = ops.SplitPlanes.empty((B, T, L.cout), dev)
            L.run(x, y=y)
            x = y
            n += 1
        top = layers[-1]
        _, x = ops.fused_pool_layer(x, top.w, top.cout, top.context, top.bias, top.scale, top.shift, relu=top.relu,
                                    eps=m.stats.eps, planes=True)
        n += 2
        for i, L in enumerate(segs):
            if i + 1 == len(segs):
                emb = torch.empty(B, 1, L.cout, dtype=torch.float32, device=dev)
                L.run(x, y_f32=emb)
            else:
                y = ops.SplitPlanes.empty((B, 1, L.cout), dev)
                L.run(x, y=y)
            n += 1 + _splitk(x.channels, L.cout, B)
            if i + 1 < len(segs):
                x = y
        return emb.view(B, -1), n

    return run


@pytest.mark.parametrize("kind", ["xvector", "snowdar"])
@pytest.mark.parametrize("pos", ["far", "near"])
def test_statistics_pooling_handles_are_unchanged(kind, pos):
    if kind == "xvector":
        from asv_subtools_b200.model.xvector import Xvector
        spec = onn.xvector_spec(40)
    else:
        from asv_subtools_b200.model.snowdar_xvector import Xvector
        spec = onn.snowdar_xvector_spec(40)
    m = Xvector(40, 10, training=False, extracted_embedding=pos)
    m.load_state_dict(onn.make_state_dict(spec, 606), strict=True)
    m.cuda().eval()
    if kind == "xvector":
        frames = [m.tdnn1, m.tdnn2, m.tdnn3, m.tdnn4, m.tdnn5]
    else:
        frames = [l for l in (m.tdnn1, m.ex_tdnn1, m.tdnn2, m.ex_tdnn2, m.tdnn3, m.ex_tdnn3, m.ex_tdnn4, m.ex_tdnn5, m.tdnn4,
                              m.tdnn5) if l is not None]
    ex = m.extractor()
    sequence = _stats_sequence(m, frames, m.tdnn6, m.tdnn7, "near_full" if kind == "snowdar" and pos == "near" else pos)
    for B, T in ((1, 37), (64, 200), (1100, 3)):     # B = 1100: segment layers without split-K
        x = _feats(B, T, B + T)
        got = ex.extract(x)
        want, n_ops = sequence(x)
        assert torch.equal(got, want), (kind, pos, B, T)
        assert ex.last_launches == n_ops, (kind, pos, B, T, ex.last_launches, n_ops)
