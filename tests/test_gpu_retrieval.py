"""Speaker retrieval on the GPU (csrc/retrieval.cu: xvb_retrieve_topk / xvb_topk_merge).  The ranked scores are the
bytes xvb_matmul_nt writes, so every list is checked bit for bit against a stable numpy top-k (score descending,
index ascending) over xvb_matmul_nt's materialised matrix; plus fences, refusals, the reference's golden top-10 file
and mAP, the CLI end to end, and a 1 000 x 300 000 case against torch.topk."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "retrieval.npz")


def _ops():
    from asv_subtools_b200 import ops
    return ops


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _materialised(a, b, row=None, col=None):
    """xvb_matmul_nt over the whole test set in one call (zero-padded to a multiple of 4), as float32 numpy."""
    n = b.shape[0]
    n4 = (n + 3) // 4 * 4
    bp = torch.zeros(n4, b.shape[1], dtype=torch.float32, device=b.device)
    bp[:n] = b
    cp = None
    if col is not None:
        cp = torch.zeros(n4, dtype=torch.float32, device=b.device)
        cp[:n] = col
    return _ops().matmul_nt(a, bp, row_bias=row, col_bias=cp)[:, :n].cpu().numpy()


def _expected(S, k):
    m, n = S.shape
    sc = np.full((m, k), -np.inf, dtype=np.float32)
    ix = np.full((m, k), -1, dtype=np.int64)
    for i in range(m):
        o = np.lexsort((np.arange(n), -S[i]))[:k]
        sc[i, :o.size] = S[i, o]
        ix[i, :o.size] = o
    return sc, ix


def _check_exact(a, b, k, slab, row=None, col=None):
    got_s, got_i = _ops().retrieve_topk(a, b, k, row_bias=row, col_bias=col, slab_cols=slab)
    want_s, want_i = _expected(_materialised(a, b, row, col), k)
    np.testing.assert_array_equal(got_i.cpu().numpy(), want_i)
    assert np.array_equal(got_s.cpu().numpy().view(np.int32), want_s.view(np.int32))


def _cosine(m, n, d, seed, dup=False):
    g = torch.Generator().manual_seed(seed)
    a = torch.nn.functional.normalize(torch.randn(m, d, generator=g), dim=1)
    b = torch.nn.functional.normalize(torch.randn(n, d, generator=g), dim=1)
    if dup and n > 1:                                  # duplicated columns: exact ties
        src = torch.randint(0, n, (n // 3,), generator=g)
        dst = torch.randint(0, n, (n // 3,), generator=g)
        b[dst] = b[src]
    return a.cuda().contiguous(), b.cuda().contiguous()


def _edge_ns(k, slab):
    return sorted({n for n in (1, k - 1, k, slab - 1, slab, slab + 1, 3 * slab + 7) if n >= 1})


EDGE_CASES = [(k, slab, n) for k in (1, 10, 256) for slab in (64, 4096) for n in _edge_ns(k, slab)]


@pytest.mark.parametrize("k,slab,n", EDGE_CASES)
def test_cosine_exact_at_every_edge(k, slab, n):
    a, b = _cosine(5, n, 64, 1000 + n + k, dup=True)
    _check_exact(a, b, k, slab)


@pytest.mark.parametrize("m", [1, 63, 64, 65, 127, 128, 129, 257])
def test_rows_across_row_blocks(m):
    a, b = _cosine(m, 9000, 48, m, dup=True)
    _check_exact(a, b, 10, 4096)


def _plda_operands(m, n, d, seed):
    from asv_subtools_b200.score.plda_train import PLDA
    rng = np.random.RandomState(seed)
    q = rng.randn(d, d)
    model = PLDA(rng.randn(d) * 0.1, q @ q.T / d + np.eye(d), np.diag(rng.rand(d) * 3 + 0.1))
    e = torch.from_numpy(rng.randn(m, d).astype(np.float32)).cuda()
    t = torch.from_numpy(rng.randn(n, d).astype(np.float32)).cuda()
    t[n // 2:n // 2 + n // 5] = t[:n // 5].clone()
    nu = np.arange(1, m + 1, dtype=np.float32)
    return model._operands(model.transform_ivectors(e, nu), nu, model.transform_ivectors(t, None))


@pytest.mark.parametrize("k,n", [(1, 4097), (10, 6143), (10, 9), (256, 12295), (256, 255)])
def test_plda_form_exact(k, n):
    a, row, b, col = _plda_operands(33, n, 40, k + n)
    _check_exact(a, b, k, 2048, row=row, col=col)


def test_all_equal_rows_and_ascending_scores():
    ops = _ops()
    a, b = _cosine(4, 10003, 32, 7)
    a[1] = 0                                           # every score of row 1 is 0: the first k columns win
    col = torch.arange(10003, dtype=torch.float32, device="cuda") * 1e-3   # rising scores: a merge in every round
    for k in (1, 10, 256):
        _check_exact(a, b, k, 4096)
        _check_exact(a, b, k, 4096, col=col)
    s, i = ops.retrieve_topk(a, b, 10, slab_cols=64)
    assert i[1].tolist() == list(range(10)) and bool((s[1] == 0).all())


def test_short_rows_and_fences():
    lib = _ops().lib
    m, n, k = 3, 7, 10
    a, b = _cosine(m, n, 32, 3)
    slab_cols = 8
    nbytes = lib.xvb_retrieve_topk_slab_bytes(m, slab_cols)
    assert nbytes == m * slab_cols * 4
    slab = torch.full((nbytes // 4 + 64,), 7.0, device="cuda")
    sc = torch.full(((m + 2) * k,), 3.5, device="cuda")
    ix = torch.full(((m + 2) * k,), 99, dtype=torch.int64, device="cuda")
    assert lib.xvb_retrieve_topk(_ptr(a), m, _ptr(b), n, 32, None, None, k, _ptr(slab), slab_cols, _ptr(sc), _ptr(ix),
                                 None) == 0
    torch.cuda.synchronize()
    want_s, want_i = _expected(_materialised(a, b), k)
    np.testing.assert_array_equal(ix[:m * k].view(m, k).cpu().numpy(), want_i)
    assert np.array_equal(sc[:m * k].view(m, k).cpu().numpy().view(np.int32), want_s.view(np.int32))
    assert bool((ix[:m * k].view(m, k)[:, n:] == -1).all()) and bool(torch.isneginf(sc[:m * k].view(m, k)[:, n:]).all())
    assert bool((sc[m * k:] == 3.5).all()) and bool((ix[m * k:] == 99).all())
    assert bool((slab[nbytes // 4:] == 7.0).all())


def test_refusals_write_nothing():
    ops = _ops()
    lib = ops.lib
    m, n, k, d = 6, 300, 10, 32
    a, b = _cosine(m, n, d, 5)
    slab = torch.empty(m * 64, device="cuda")
    sc = torch.full((m * k,), 3.5, device="cuda")
    ix = torch.full((m * k,), 99, dtype=torch.int64, device="cuda")

    def call(a_=a, m_=m, b_=b, n_=n, k_=k, slab_=slab, cols=64, sc_=sc, ix_=ix, col=None):
        return lib.xvb_retrieve_topk(_ptr(a_), m_, _ptr(b_), n_, d, None, _ptr(col), k_, _ptr(slab_), cols, _ptr(sc_),
                                     _ptr(ix_), None)

    bad = [dict(k_=0), dict(k_=257), dict(cols=6), dict(cols=0), dict(m_=0), dict(n_=0), dict(a_=None), dict(sc_=None),
           dict(slab_=None)]
    for kw in bad:
        assert call(**kw) == -1, kw
    assert lib.xvb_retrieve_topk_slab_bytes(0, 64) == -1 and lib.xvb_retrieve_topk_slab_bytes(4, 6) == -1
    nan_a = a.clone()
    nan_a[3, 5] = float("nan")
    assert call(a_=nan_a) == -1
    assert "enroll row 3" in ops._lib.last_error()
    col = torch.zeros(n, device="cuda")
    col[250] = float("nan")
    assert call(col=col) == -1
    assert "test row 250" in ops._lib.last_error()
    inf_b = b.clone()
    inf_b[299, 0] = float("inf")                       # in the last, 1..3-row padded slab
    assert call(b_=inf_b) == -1
    assert "test row 299" in ops._lib.last_error()
    torch.cuda.synchronize()
    assert bool((sc == 3.5).all()) and bool((ix == 99).all())
    flag = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    S = torch.zeros(2, 8, device="cuda")
    for args in [(S, 6, 2, 8, 0, 10), (S, 8, 2, 8, 0, 0), (S, 8, 2, 9, 0, 10), (S, 8, 0, 8, 0, 10), (S, 8, 2, 8, -1, 10)]:
        assert lib.xvb_topk_merge(_ptr(args[0]), *args[1:], _ptr(sc), _ptr(ix), _ptr(flag), None) == -1, args
    assert lib.xvb_topk_merge(_ptr(S), 8, 2, 8, 0, 10, _ptr(sc), _ptr(ix), None, None) == -1


def test_merge_flags_nan_scores():
    lib = _ops().lib
    S = torch.randn(5, 4100, device="cuda")
    S[2, 4097] = float("nan")
    S[4, 7] = float("nan")
    sc = torch.full((5, 3), float("-inf"), device="cuda")
    ix = torch.full((5, 3), -1, dtype=torch.int64, device="cuda")
    flag = torch.full((1,), -1, dtype=torch.int64, device="cuda")
    assert lib.xvb_topk_merge(_ptr(S), 4100, 5, 4100, 0, 3, _ptr(sc), _ptr(ix), _ptr(flag), None) == 0
    assert int(flag.item()) == 2
    want_s, want_i = _expected(torch.nan_to_num(S, nan=float("-inf")).cpu().numpy(), 3)
    np.testing.assert_array_equal(ix.cpu().numpy(), want_i)   # a NaN is never ranked


def test_golden_top10_and_map():
    from asv_subtools_b200.score import metrics
    from asv_subtools_b200.score.retrieve import format_topk
    ops = _ops()
    z = np.load(GOLDEN)
    ek, tk = [str(x) for x in z["enroll_keys"]], [str(x) for x in z["test_keys"]]
    e = ops.center_length_norm(torch.from_numpy(z["enroll"]).cuda())
    t = ops.center_length_norm(torch.from_numpy(z["test"]).cuda())
    _, idx = ops.retrieve_topk(e, t, 10)
    idx = idx.cpu().numpy()
    s64 = z["scores64"]
    want = np.stack([np.lexsort((np.arange(r.size), -r))[:10] for r in s64])
    swaps = 0
    for i in range(len(ek)):
        for p in np.flatnonzero(idx[i] != want[i]):   # allowed only between float64 near-ties
            assert abs(s64[i, idx[i, p]] - s64[i, want[i, p]]) < 1e-6, (i, p)
            swaps += 1
    print("golden retrieval: {} near-tie swaps".format(swaps))
    text = format_topk(ek, tk, idx)
    meta = bytes(z["meta"]).decode("utf-8").splitlines(True)
    assert "mAP=%.3f" % metrics.retrieval_map(text.splitlines(True), meta) == str(z["map_line"])
    if swaps == 0:
        assert text.encode("utf-8") == bytes(z["top10"])


def test_cli_end_to_end(tmp_path, capsys):
    from asv_subtools_b200 import kaldi_io
    from asv_subtools_b200.score import retrieve
    z = np.load(GOLDEN)
    for name, keys, x in (("enroll", z["enroll_keys"], z["enroll"]), ("test", z["test_keys"], z["test"])):
        with open(tmp_path / (name + ".ark"), "wb") as f:
            for key, v in zip(keys, x):
                kaldi_io.write_vec_flt(f, v, key=str(key))
    (tmp_path / "test.meta").write_bytes(bytes(z["meta"]))
    out = tmp_path / "out.top10"
    retrieve.main(["--norm", str(tmp_path / "enroll.ark"), str(tmp_path / "test.ark"), str(out),
                   "--test-meta", str(tmp_path / "test.meta")])
    assert out.read_bytes() == bytes(z["top10"])
    assert capsys.readouterr().out.strip() == str(z["map_line"])


def test_cli_plda_with_smoothing_and_num_utts(tmp_path):
    """--plda MODEL --num-utts F --smoothing S ranks by the LLR of the smoothed model, as score.sh `plda` scores it."""
    from asv_subtools_b200 import kaldi_io, ops
    from asv_subtools_b200.score import retrieve
    from asv_subtools_b200.score.plda_train import PLDA
    rng = np.random.RandomState(3)
    d, m, n = 24, 9, 301
    q = rng.randn(d, d)
    model = tmp_path / "plda.ori"
    with open(model, "wb") as f:
        kaldi_io.write_vec_flt(f, (rng.randn(d) * 0.1).astype(np.float32), key="mean")
        kaldi_io.write_vec_flt(f, (q @ q.T / d + np.eye(d)).astype(np.float32).reshape(-1), key="within_var")
        kaldi_io.write_vec_flt(f, np.diag(rng.rand(d) * 3 + 0.1).astype(np.float32).reshape(-1), key="between_var")
    ek = ["spk{:02d}".format(i) for i in (5, 1, 8, 0, 3, 2, 7, 6, 4)]
    tk = ["utt{:03d}".format(j) for j in range(n)]
    e = rng.randn(m, d).astype(np.float32)
    t = rng.randn(n, d).astype(np.float32)
    nu = np.arange(1, m + 1, dtype=np.float32)
    for name, keys, x in (("enroll", ek, e), ("test", tk, t)):
        with open(tmp_path / (name + ".ark"), "wb") as f:
            for key, v in zip(keys, x):
                kaldi_io.write_vec_flt(f, v, key=key)
    (tmp_path / "num_utts").write_text("".join("{} {}\n".format(k, int(c)) for k, c in zip(ek, nu)))
    out = tmp_path / "out.top5"
    retrieve.main(["--top", "5", "--plda", str(model), "--num-utts", str(tmp_path / "num_utts"), "--smoothing", "0.3",
                   str(tmp_path / "enroll.ark"), str(tmp_path / "test.ark"), str(out)])
    plda = PLDA.read_ori(str(model))
    plda.smooth_within_class_covariance(0.3)
    eu = plda.transform_ivectors(torch.from_numpy(e).cuda(), nu)
    tu = plda.transform_ivectors(torch.from_numpy(t).cuda(), None)
    a, row, b, col = plda._operands(eu, nu, tu)
    _, idx = ops.retrieve_topk(a, b, 5, row_bias=row, col_bias=col)
    assert out.read_text() == retrieve.format_topk(ek, tk, idx.cpu().numpy())
    want_s, want_i = _expected(_materialised(a, b, row, col), 5)
    np.testing.assert_array_equal(idx.cpu().numpy(), want_i)


def test_scale_against_torch_topk():
    ops = _ops()
    m, n, d, k, slab = 1000, 300000, 256, 10, 65536
    a, b = _cosine(m, n, d, 11)
    got_s, got_i = ops.retrieve_topk(a, b, k)
    best_s, best_i = None, None
    for c0 in range(0, n, slab):
        cols = min(slab, n - c0)
        s = ops.cosine_matrix(a, b[c0:c0 + cols])
        ts, ti = torch.topk(s, k, dim=1)
        ti = ti + c0
        if best_s is None:
            best_s, best_i = ts, ti
        else:
            cs, ci = torch.cat([best_s, ts], 1), torch.cat([best_i, ti], 1)
            best_s, o = torch.topk(cs, k, dim=1)
            best_i = torch.gather(ci, 1, o)
    assert torch.equal(got_s, best_s)
    same = got_i == best_i
    # torch.topk does not define the order of equal scores; where it differs the scores must be equal
    assert bool((same | (got_s == best_s)).all())
    assert int(same.sum()) >= m * k - 50
