"""Masked batches of utterances of different lengths on the Conformer x-vector (xvb_conformer_extract_lengths and its
op-by-op twin ConformerExtractor): the masked head conv, attention and attentive pooling against the unmasked kernels on
each utterance alone, with the padding poisoned and a fenced spare row; every row of a masked batch bit for bit its solo
extraction on the handle and the twin, handle == twin; what lies past an utterance's end is never read; all lengths
equal to T is the unmasked call; the frame budget; alternating masked and equal-length calls; bad lengths; the goldens
cut by chunk_sizes and packed into masked batches; and xvb-extract / pipeline/extract_embeddings.py with
--mixed-lengths on Conformer models of both subsamplings.  Needs an H100 (`-m gpu`)."""
import ctypes as C
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import conformer_2sub_oracle as c2  # noqa: E402
import conformer_oracle as co  # noqa: E402
from asv_subtools_b200 import kaldi_io, ops  # noqa: E402
from asv_subtools_b200._lib import check, lib  # noqa: E402
from asv_subtools_b200.model.transformer_xvector import (ConformerExtractor, NativeConformerExtractor,  # noqa: E402
                                                         TransformerXvector, rotary_table, subsampled_shape)
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(HERE)
BIN = os.path.join(ROOT, "asv_subtools_b200", "bin", "xvb-extract")
CASES = dict(co.CASES, **c2.CASES)
GOLDEN = {c: np.load(os.path.join(HERE, "golden", "conformer.npz" if c in co.CASES else "conformer_2sub.npz")) for c in CASES}
NAN = float("nan")


@pytest.fixture(autouse=True)
def _no_tf32():
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cosines(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.sum(a * b, -1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))


def _sd(case):
    return co.seeded_state_dict(GOLDEN[case]["keys_" + case], CASES[case][4])


_MODELS = {}


def _model(case, pos):
    if (case, pos) not in _MODELS:
        kwargs, fdim = CASES[case][:2]
        m = TransformerXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
        m.load_state_dict(_sd(case), strict=True)
        _MODELS[case, pos] = m.cuda().eval()
    return _MODELS[case, pos]


def _extractors(case, pos):
    """(handle, twin) on one model, each built directly so that the environment switch is not involved."""
    m = _model(case, pos)
    return NativeConformerExtractor(m), ConformerExtractor(m, torch.device("cuda"))


def _padded(rows, T, fill=0.0):
    x = np.full((len(rows), T, rows[0].shape[1]), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


def _utterances(lens, fdim, seed):
    return [onn.synthetic_feats(1, t, fdim, seed + i)[0] for i, t in enumerate(lens)]


def _fenced_planes(shape):
    """SplitPlanes of `shape` followed by one spare row of 7.0, and the flat buffers that hold them."""
    n, row = int(np.prod(shape)), int(shape[-1])
    hi = torch.full((n + row,), 7.0, dtype=torch.bfloat16, device="cuda")
    lo = torch.full((n + row,), 7.0, dtype=torch.bfloat16, device="cuda")
    return ops.SplitPlanes(hi[:n].view(*shape), lo[:n].view(*shape), shape[-1]), hi, lo


def _fence_intact(buf, n):
    return bool((buf[n:].float() == 7.0).all())


# ------------------------------------------------------------------ 1. the masked kernels against solo calls
HEAD_LENS = [3, 4, 5, 6, 7, 8, 9, 299, 300, 301, 398]


@pytest.mark.parametrize("stride_f", [2, 1])
@pytest.mark.parametrize("C_out", [8, 256])
def test_subsample_head_lengths_rows_equal_solo_calls(stride_f, C_out):
    B, T, F = len(HEAD_LENS), 400, 23
    g = torch.Generator().manual_seed(31 + C_out + stride_f)
    x = torch.randn(B, T, F, generator=g).cuda()
    for b, L in enumerate(HEAD_LENS):
        x[b, L:] = NAN
    w = (torch.randn(C_out, 1, 3, 3, generator=g) / 3).cuda()
    bias = (torch.randn(C_out, generator=g) * 0.1).cuda()
    T1, F1 = (T - 1) // 2, (F - 1) // 2 if stride_f == 2 else F - 2
    y, hi, lo = _fenced_planes((B, T1, F1, C_out))
    n = B * T1 * F1 * C_out
    d_lens = torch.tensor(HEAD_LENS, dtype=torch.int32, device="cuda")
    ops.subsample_head(x, w, bias, y, stride_f=stride_f, lengths=d_lens)
    torch.cuda.synchronize()
    assert _fence_intact(hi, n) and _fence_intact(lo, n)
    for b, L in enumerate(HEAD_LENS):
        L1 = (L - 1) // 2
        solo = ops.SplitPlanes.empty((1, L1, F1, C_out), "cuda")
        ops.subsample_head(x[b:b + 1, :L].contiguous(), w, bias, solo, stride_f=None if stride_f == 2 else 1)
        assert torch.equal(y.hi[b, :L1], solo.hi[0]) and torch.equal(y.lo[b, :L1], solo.lo[0]), (L, stride_f, C_out)
        assert torch.count_nonzero(y.hi[b, L1:].float()) == 0 and torch.count_nonzero(y.lo[b, L1:].float()) == 0, L
    before = hi.clone()
    with pytest.raises(RuntimeError, match="xvb_subsample_head_lengths: null lengths"):
        check(lib.xvb_subsample_head_lengths(x.data_ptr(), B, T, F, None, w.data_ptr(), bias.data_ptr(), C_out, stride_f,
                                             y.hi.data_ptr(), y.lo.data_ptr(), None), "xvb_subsample_head_lengths")
    torch.cuda.synchronize()
    assert torch.equal(hi, before)


ATTN_LENS = [1, 2, 7, 8, 9, 31, 32, 33, 63, 64, 65, 98]


def _mult_table(rows=5000, train_len=300.0):
    t = torch.arange(rows, dtype=torch.float32).clamp(min=1)
    return (torch.log(t) / math.log(train_len)).cuda()


def _check_attention(lens, T, dk, mode, plus):
    H, B = 2, len(lens)
    g = torch.Generator().manual_seed(7 * dk + 3 * mode + int(plus) + T)
    qkv = torch.randn(B, T, 3 * H * dk, generator=g).cuda()
    for b, L in enumerate(lens):
        qkv[b, L:] = NAN
    rope = rotary_table(dk).cuda() if mode else None
    table = _mult_table() if plus else None
    y, hi, lo = _fenced_planes((B, T, H * dk))
    n = B * T * H * dk
    d_lens = torch.tensor(lens, dtype=torch.int32, device="cuda")
    ops.rope_attention(qkv, H, dk, y, rope=rope, rope_v=mode == 2, lengths=d_lens, mult_table=table)
    torch.cuda.synchronize()
    assert _fence_intact(hi, n) and _fence_intact(lo, n)
    for b, L in enumerate(lens):
        solo = ops.SplitPlanes.empty((1, L, H * dk), "cuda")
        ops.rope_attention(qkv[b:b + 1, :L].contiguous(), H, dk, solo, rope=rope, rope_v=mode == 2,
                           score_mult=float(table[L]) if plus else 1.0)
        assert torch.equal(y.hi[b, :L], solo.hi[0]) and torch.equal(y.lo[b, :L], solo.lo[0]), (L, T, dk, mode, plus)
        assert torch.count_nonzero(y.hi[b, L:].float()) == 0 and torch.count_nonzero(y.lo[b, L:].float()) == 0, L
    return qkv, y, hi, d_lens


@pytest.mark.parametrize("plus", [False, True], ids=["softmax", "softmax_plus"])
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["no_rope", "rope", "rope_v"])
@pytest.mark.parametrize("dk", [32, 64, 128])
def test_rope_attention_lengths_rows_equal_solo_calls(dk, mode, plus):
    _check_attention(ATTN_LENS, 98, dk, mode, plus)


def test_rope_attention_lengths_long_and_refusals():
    qkv, y, hi, d_lens = _check_attention([240, 1, 100, 239, 129, 8], 240, 64, 1, True)
    before = hi.clone()
    with pytest.raises(RuntimeError, match="mult_rows=240"):       # mult_table[T] would be outside the table
        ops.rope_attention(qkv, 2, 64, y, lengths=d_lens, mult_table=_mult_table(240))
    with pytest.raises(RuntimeError, match="xvb_rope_attention_lengths: null lengths"):
        check(lib.xvb_rope_attention_lengths(qkv.data_ptr(), qkv.shape[2], qkv.shape[0], 240, 2, 64, None, 0, None, None, 0,
                                             y.hi.data_ptr(), y.lo.data_ptr(), y.ld, None), "xvb_rope_attention_lengths")
    with pytest.raises(ValueError, match="pass lengths"):
        ops.rope_attention(qkv, 2, 64, y, mult_table=_mult_table())
    torch.cuda.synchronize()
    assert torch.equal(hi, before)


POOL_LENS = [1, 7, 8, 9, 31, 32, 33, 63, 64, 65]


@pytest.mark.parametrize("C_in", [132, 260, 1540])
def test_attn_stats_pool_lengths_rows_equal_solo_calls(C_in):
    B, T = len(POOL_LENS), 65
    g = torch.Generator().manual_seed(C_in)
    logits = (torch.randn(B, T, C_in, generator=g) * 3).cuda()
    x = torch.randn(B, T, C_in, generator=g).cuda()
    for b, L in enumerate(POOL_LENS):
        logits[b, L:] = NAN
        x[b, L:] = NAN
    buf = torch.full(((B + 1) * 2 * C_in,), 7.0, device="cuda")       # one spare fenced row after the output
    out = buf[:B * 2 * C_in].view(B, 2 * C_in)
    d_lens = torch.tensor(POOL_LENS, dtype=torch.int32, device="cuda")
    check(lib.xvb_attn_stats_pool_lengths(logits.data_ptr(), C_in, x.data_ptr(), C_in, B, T, C_in, 1e-5, d_lens.data_ptr(),
                                          out.data_ptr(), None, None, 0, None), "xvb_attn_stats_pool_lengths")
    got, planes = ops.attn_stats_pool(logits, x, floor=1e-5, planes=True, lengths=d_lens)
    torch.cuda.synchronize()
    assert torch.equal(buf[B * 2 * C_in:], torch.full((2 * C_in,), 7.0, device="cuda"))
    assert torch.equal(out, got)
    for b, L in enumerate(POOL_LENS):
        solo, sp = ops.attn_stats_pool(logits[b:b + 1, :L].contiguous(), x[b:b + 1, :L].contiguous(), floor=1e-5, planes=True)
        assert torch.equal(out[b], solo[0]), (L, C_in)
        assert torch.equal(planes.hi[b], sp.hi[0]) and torch.equal(planes.lo[b], sp.lo[0]), L
    before = buf.clone()
    with pytest.raises(RuntimeError, match="xvb_attn_stats_pool_lengths: null lengths"):
        check(lib.xvb_attn_stats_pool_lengths(logits.data_ptr(), C_in, x.data_ptr(), C_in, B, T, C_in, 1e-5, None,
                                              out.data_ptr(), None, None, 0, None), "xvb_attn_stats_pool_lengths")
    torch.cuda.synchronize()
    assert torch.equal(buf, before)


# ------------------------------------------------------------------ 2. rows against solo extraction, handle == twin
MIXED = [7, 8, 9, 10, 11, 12, 13, 14, 15, 16, 37, 299, 300, 301, 304, 398, 400]


def _mixed_lengths(n, seed):
    rng = np.random.RandomState(seed)
    lens = MIXED + [int(v) for v in rng.randint(7, 401, n - len(MIXED))]
    rng.shuffle(lens)
    return lens


SOLO_CASES = [("launcher", "near"), ("launcher2", "near_affine"), ("small", "far"), ("small", "near_affine"),
              ("small2", "near"), ("rotv", "near")]


@pytest.mark.parametrize("case, pos", SOLO_CASES)
def test_rows_equal_solo_extraction_on_handle_and_twin(monkeypatch, case, pos):
    """A row whose chunk subsamples to T' = 1 is compared with split-K off in the batch and in the solo call: alone,
    its frame-level linears with Cin >= 1536 (embed_out, the FFNs' w_2) run at T == 1, where the layer kernel splits K,
    which the batch at T' > 1 does not; with split-K off both run the plain K loop (the segment layers too)."""
    fdim, sub = CASES[case][1], _model(case, pos).transformer.subsampling
    native, twin = _extractors(case, pos)
    lens = _mixed_lengths(64, 5 + len(case))
    utts = _utterances(lens, fdim, 3000)
    x = _padded(utts, max(lens))
    got = {}
    with torch.no_grad():
        for splitk in ("1", "0"):
            monkeypatch.setenv("XVB_SPLITK", splitk)
            got_n = native.extract(x, lengths=lens).clone()
            n_launch = native.last_launches
            got_t = twin.extract(x, lengths=lens).clone()
            assert twin.last_launches == n_launch
            assert torch.equal(got_n, got_t), (splitk, (got_n - got_t).abs().max().item())
            got[splitk] = got_n
        for i, u in enumerate(utts):
            splitk = "0" if subsampled_shape(sub, lens[i], fdim)[0] == 1 else "1"
            monkeypatch.setenv("XVB_SPLITK", splitk)
            xs = torch.from_numpy(u[None]).cuda()
            solo_n, solo_t = native.extract(xs), twin.extract(xs)
            row = got[splitk][i]
            assert torch.equal(row, solo_n[0]), (case, i, lens[i], (row - solo_n[0]).abs().max().item())
            assert torch.equal(row, solo_t[0]), (case, i, lens[i])


# ------------------------------------------------------------------ 3. the padding is never read
@pytest.mark.parametrize("case", ["launcher", "small2"])
def test_padding_is_never_read(case):
    fdim = CASES[case][1]
    native, twin = _extractors(case, "near")
    lens = _mixed_lengths(19, 9)[:19]
    utts = _utterances(lens, fdim, 4000)
    T = max(lens) + 7
    with torch.no_grad():
        want = native.extract(_padded(utts, T), lengths=lens).clone()
        for fill in (NAN, 1e30, -1e30):
            assert torch.equal(native.extract(_padded(utts, T, fill), lengths=lens), want), fill
            assert torch.equal(twin.extract(_padded(utts, T, fill), lengths=lens), want), fill


# ------------------------------------------------------------------ 4. the unmasked path, the frame budget, refusals
@pytest.mark.parametrize("case, pos", [("launcher", "near"), ("small", "far"), ("launcher2", "near")])
def test_all_lengths_equal_T_is_the_unmasked_call(case, pos):
    native, twin = _extractors(case, pos)
    fdim = CASES[case][1]
    with torch.no_grad():
        for b in (1, 3):
            for t in (7, 37, 300):
                x = torch.from_numpy(onn.synthetic_feats(b, t, fdim, 10 * b + t)).cuda()
                want = native.extract(x).clone()
                n = native.last_launches
                assert torch.equal(native.extract(x, lengths=[t] * b), want), (case, b, t)
                assert native.last_launches == n
                assert torch.equal(twin.extract(x, lengths=[t] * b), want), (case, b, t)


def test_masked_call_over_the_frame_budget_equals_per_group_calls():
    """200 chunks padded to 300 frames run as groups of 128 (the 128 * 300 frame budget)."""
    native, _ = _extractors("launcher", "near")
    rng = np.random.RandomState(17)
    lens = [300, 7, 299, 150] + [int(v) for v in rng.randint(7, 301, 196)]
    utts = _utterances(lens, 80, 5000)
    x = _padded(utts, 300)
    with torch.no_grad():
        whole = native.extract(x, lengths=lens).clone()
        for a, b in ((0, 128), (128, 200)):
            assert torch.equal(whole[a:b], native.extract(x[a:b].contiguous(), lengths=lens[a:b])), (a, b)


def test_masked_and_equal_length_calls_alternate_on_one_workspace():
    native, twin = _extractors("launcher", "near")
    a = torch.from_numpy(onn.synthetic_feats(8, 300, 80, 61)).cuda()
    lens = [300, 7, 150, 299, 201, 8, 100, 77]
    utts = _utterances(lens, 80, 62)
    with torch.no_grad():
        for ex in (native, twin):
            plain = ex.extract(a).clone()
            masked = ex.extract(_padded(utts, 300), lengths=lens).clone()
            assert torch.equal(ex.extract(a), plain)
            assert torch.equal(ex.extract(_padded(utts, 300), lengths=lens), masked)
            small = torch.from_numpy(onn.synthetic_feats(3, 37, 80, 63)).cuda()
            want = ex.extract(small).clone()
            ex.extract(_padded(utts, 300), lengths=lens)
            assert torch.equal(ex.extract(small), want)


def test_bad_lengths_are_refused_by_the_c_entry_and_python():
    native, twin = _extractors("small", "near")
    x = torch.zeros(4, 30, 23, device="cuda")
    for lens, bad in (([30, 6, 7, 7], r"lengths\[1\]=6"), ([30, 30, 31, 7], r"lengths\[2\]=31"),
                      ([0, 7, 7, 7], r"lengths\[0\]=0")):
        with pytest.raises(RuntimeError, match="xvb_conformer_extract_lengths: " + bad):
            native.extract(x, lengths=lens)
        with pytest.raises(ValueError, match=bad):
            twin.extract(x, lengths=lens)
    emb = torch.full((4, native.embed_dim), 7.0, device="cuda")
    arr = (C.c_int32 * 4)(8, 9, 6, 10)
    assert native._fn("extract_lengths")(native._h, C.c_void_p(x.data_ptr()), arr, 4, 30, C.c_void_p(emb.data_ptr()),
                                         native._stream()) == -1   # XVB_EINVAL, nothing launched
    assert native._fn("extract_lengths")(native._h, C.c_void_p(x.data_ptr()), None, 4, 30, C.c_void_p(emb.data_ptr()),
                                         native._stream()) == -1
    big = torch.zeros(1, 20005, 23, device="cuda")                   # T' = 5000: past the positional tables
    with pytest.raises(RuntimeError, match="5000 subsampled frames|exceeds the positional tables"):
        native.extract(big, lengths=[20005])
    torch.cuda.synchronize()
    assert torch.equal(emb, torch.full_like(emb, 7.0))


# ------------------------------------------------------------------ 5. goldens cut by chunk_sizes, in masked batches
@pytest.mark.parametrize("case", sorted(CASES))
def test_goldens_in_masked_batches(case):
    _, fdim, frames, positions, _, fseed = CASES[case]
    for pos in positions:
        m = _model(case, pos)
        native, twin = _extractors(case, pos)
        chunks, owner, want, total = [], [], [], []
        for t in frames:
            x = onn.synthetic_feats(2, t, fdim, fseed + t)
            for i in range(2):
                off = 0
                for s in m.chunk_sizes(t):
                    chunks.append(x[i, off:off + s])
                    owner.append(len(want))
                    off += s
                want.append(GOLDEN[case]["{}_{}_T{}".format(case, pos, t)][i])
                total.append(t)
        ref = np.stack(want)
        lens = [c.shape[0] for c in chunks]
        for ex in (native, twin):
            emb = ex.extract(_padded(chunks, max(lens)), lengths=lens).cpu().numpy()
            got = np.zeros_like(ref)
            for e, n, u in zip(emb, lens, owner):       # sum(len_i * emb_i) / frames, the reference's average
                got[u] += np.float32(n) * e
            got /= np.asarray(total, np.float32)[:, None]
            assert rel(got, ref) <= 1e-4 and cosines(got, ref).min() >= 1 - 1e-6, (case, pos, type(ex).__name__,
                                                                                     rel(got, ref))


# ------------------------------------------------------------------ 6. xvb-extract and the Python CLI
def _write_ark(path, feats):
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, np.ascontiguousarray(v, dtype=np.float32), key=k)


@pytest.mark.parametrize("case", ["launcher", "launcher2"])
def test_cli_mixed_lengths_on_a_conformer_model(tmp_path, case):
    kwargs, fdim = CASES[case][:2]
    pos = "near"
    m = _model(case, pos)
    sd = _sd(case)
    model = str(tmp_path / "conformer.xvbm")
    NativeConformerExtractor(m).save(model)
    assert open(model, "rb").read(8) == b"XVBC0001"
    lens = [7, 120, 120, 310, 650, 899, 1799]
    assert m.chunk_sizes(1799)[-1] == 304
    feats = {"c{}".format(i): onn.synthetic_feats(1, t, fdim, 300 + i)[0] for i, t in enumerate(lens)}
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, feats)
    runs = {}
    for name, flag in (("mixed", ["--mixed-lengths"]), ("plain", [])):
        out = str(tmp_path / (name + ".ark"))
        r = subprocess.run([BIN, "--batch", "4"] + flag + [model, "ark:" + ark, "ark:" + out], capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        runs[name] = (dict(kaldi_io.read_vec_flt_ark(out)), r.stderr)
    got, summary = runs["mixed"]
    assert sorted(got) == sorted(feats)
    s = re.search(r"(\d+) masked batches, (\d+) padded frames \(([0-9.]+) of (\d+) batch frames\)", summary)
    assert s, summary
    assert float(s.group(3)) <= 0.125
    oracle = co if case in co.CASES else c2
    cfg = co.config(kwargs)
    for k, v in feats.items():
        assert rel(got[k], runs["plain"][0][k]) <= 1e-5, (k, rel(got[k], runs["plain"][0][k]))
        want = oracle.extract(sd, v, cfg, pos).numpy()
        assert rel(got[k], want) <= 1e-4, (k, rel(got[k], want))

    torch.save(sd, str(tmp_path / "final.params"))
    out = str(tmp_path / "py.ark")
    r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings", "--mixed-lengths",
                        "--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", "transformer_xvector.py"),
                        "--model-creation", co.creation(kwargs, fdim, pos), "--batch-size", "4",
                        str(tmp_path / "final.params"), "ark:" + ark, "ark:" + out],
                       capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    py = dict(kaldi_io.read_vec_flt_ark(out))
    assert sorted(py) == sorted(feats) and "masked batches" in r.stderr
    for k in feats:
        assert rel(py[k], got[k]) <= 1e-5, (k, rel(py[k], got[k]))

    short = str(tmp_path / "short.ark")
    _write_ark(short, {"a": feats["c1"], "s": onn.synthetic_feats(1, 6, fdim, 9)[0]})
    r = subprocess.run([BIN, "--mixed-lengths", model, "ark:" + short, "ark:" + str(tmp_path / "s.ark")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 1 and "ERROR" in r.stderr and "lengths" in r.stderr, r.stdout + r.stderr
