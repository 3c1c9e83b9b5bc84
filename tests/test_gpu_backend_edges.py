"""The back end's CUDA-core kernels (scoring.cu) on the GPU against tests/backend_exact.py, through the C entry points
(so that pitches ops does not expose, lds > ncoh and ldo > N, are reached):

  * Inputs with a pitch hold NaN in the gap past the logical row, which no kernel may read.
  * Outputs are fenced: every output is a view inside a buffer filled with a NaN sentinel, starting 4 elements in;
    everything outside the logical output must be bitwise unchanged.
  * Results are compared bit for bit, except the std of a top-n set whose fp64 sum of squares is not exact (1 ulp) and
    plda_llr_operands' logf row term (the bound of backend_exact.llr_term_ref_and_bound).
  * Refusals return XVB_EINVAL and write nothing."""
import numpy as np
import pytest
import torch

import backend_exact as bx
from gpu_checks import Fenced, equal, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132
EINVAL = -1
LEAD = 4


@pytest.fixture(scope="module")
def lib():
    from asv_subtools_b200 import _lib
    assert torch.cuda.is_available()
    return _lib.lib


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(a):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _p(t):
    return None if t is None else t.data_ptr()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _out(n, dtype=torch.float32):
    """n elements at offset LEAD of a sentinel buffer with 7 more after them"""
    return Fenced((n + LEAD + 7,), dtype, slice(LEAD, LEAD + n))


def _pitched(a, ld):
    """(rows, n) float32 as the first n columns of a (rows, ld) buffer holding NaN in the gap"""
    buf = torch.full((a.shape[0], ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:, :a.shape[1]] = _dev(a)
    return buf


def _exact(f, want, what):
    torch.cuda.synchronize()
    equal(_bits(f.numpy()).reshape(-1), _bits(np.asarray(want, np.float32)).reshape(-1), what)
    f.check(what)


# ------------------------------------------------------------------------------------------------ one warp per row
ROW = sorted(bx.row_cases())


@pytest.mark.parametrize("name", ROW)
def test_center_length_norm(lib, name):
    case = bx.row_cases()[name]
    op = bx.center_length_norm_operands(case, name)
    n, D = case["n"], case["D"]
    x, m, y = _dev(op["x"]), _dev(op["mean"]), _out(n * D)
    assert lib.xvb_center_length_norm(_p(x), _p(m), _p(y.view), n, D, None) == 0
    _exact(y, bx.center_length_norm_ref(op), "center_length_norm " + name)


@pytest.mark.parametrize("name", ROW)
def test_cosine_bilinear_trials(lib, name):
    case = bx.row_cases()[name]
    op = bx.trials_operands(case, name)
    e, t, te, tt, row, col = (_dev(op[k]) for k in ("e", "t", "te", "tt", "row", "col"))
    out = _out(case["n"])
    if case["variant"] == 0:
        rc = lib.xvb_cosine_trials(_p(e), _p(t), case["D"], _p(te), _p(tt), case["n"], _p(out.view), None)
    else:
        rc = lib.xvb_bilinear_trials(_p(e), _p(t), case["D"], _p(te), _p(tt), case["n"], _p(row), _p(col), _p(out.view), None)
    assert rc == 0
    _exact(out, bx.trials_ref(op), "trials " + name)


@pytest.mark.parametrize("name", sorted(bx.plda_terms_cases()))
def test_plda_terms(lib, name):
    case = bx.plda_terms_cases()[name]
    op = bx.plda_terms_operands(case, name)
    x, g, c, term = _dev(op["x"]), _dev(op["gamma"]), _dev(op["c"]), _out(case["n"])
    assert lib.xvb_plda_terms(_p(x), case["n"], case["D"], _p(g), _p(c), _p(term.view), None) == 0
    _exact(term, bx.plda_terms_ref(op), "plda_terms " + name)


@pytest.mark.parametrize("name", ROW)
def test_plda_normalize_rows(lib, name):
    case = bx.row_cases()[name]
    op = bx.plda_normalize_operands(case, name)
    n, D = case["n"], case["D"]
    u = _out(n * D)
    u.view.copy_(_dev(op["x"].reshape(-1)))
    psi, num = _dev(op["psi"]), _dev(op["num"])
    assert lib.xvb_plda_normalize_rows(_p(u.view), _p(psi), _p(num), n, D, op["simple"], None) == 0
    _exact(u, bx.plda_normalize_ref(op), "plda_normalize_rows " + name)


@pytest.mark.parametrize("name", ROW)
def test_plda_llr_operands(lib, name):
    case = bx.row_cases()[name]
    op = bx.llr_operands(case, name)
    n, D = case["n"], case["D"]
    x, psi, num = _dev(op["x"]), _dev(op["psi"]), _dev(op["num"])
    a, term = _out(n * 2 * D), _out(n)
    assert lib.xvb_plda_llr_operands(_p(x), _p(psi), _p(num), n, D, op["side"], _p(a.view), _p(term.view), None) == 0
    want_a, _, _ = bx.llr_emulate(op)
    _exact(a, want_a, "plda_llr_operands operand " + name)
    ref, bound = bx.llr_term_ref_and_bound(op)
    within(term.numpy(), ref, bound, "plda_llr_operands term " + name)
    term.check("plda_llr_operands term " + name)


# ------------------------------------------------------------------------------------------------ column / speaker mean
@pytest.mark.parametrize("name", sorted(bx.column_cases(SMS_FOR_IDS)))
def test_column_mean(lib, sms, name):
    case = bx.column_cases(sms)[name]
    op = bx.column_operands(case, name)
    x, mean = _dev(op["x"]), _out(case["D"])
    assert lib.xvb_column_mean(_p(x), case["rows"], case["D"], _p(mean.view), None) == 0
    _exact(mean, bx.column_ref(op), "column_mean " + name)


@pytest.mark.parametrize("name", sorted(bx.speaker_cases()))
def test_speaker_mean(lib, name):
    case = bx.speaker_cases()[name]
    op = bx.speaker_operands(case, name)
    S, D = len(op["off"]) - 1, case["D"]
    x, off, mem, out = _dev(op["x"]), _dev(op["off"]), _dev(op["members"]), _out(S * D)
    assert lib.xvb_speaker_mean(_p(x), D, _p(off), _p(mem), S, _p(out.view), None) == 0
    _exact(out, bx.speaker_ref(op), "speaker_mean " + name)


# ------------------------------------------------------------------------------------------------ top-n statistics
@pytest.mark.parametrize("name", sorted(bx.topn_cases()))
def test_topn_mean_std(lib, name):
    ncoh = bx.topn_cases()[name]["ncoh"]
    k, vals = bx.topn_rows(ncoh, name)
    R = vals.shape[0]
    S = _pitched(vals, ncoh + 3)
    for top_n in bx.topn_tops(ncoh):
        n = bx.topn_select_n(ncoh, top_n)
        for ddof in (0, 1):
            what = "topn_mean_std {} top_n={} ddof={}".format(name, top_n, ddof)
            mean, std = _out(R), _out(R)
            assert lib.xvb_topn_mean_std_ddof(_p(S), ncoh + 3, R, ncoh, top_n, ddof, _p(mean.view), _p(std.view), None) == 0
            ref = [bx.topn_stats(k[r], n, ddof) for r in range(R)]
            _exact(mean, [m for m, _, _ in ref], what + " mean")
            got = std.numpy()
            for r, (_, sd, exact) in enumerate(ref):
                if np.isnan(sd):
                    assert np.isnan(got[r]), (what, r, got[r])        # n - ddof = 0: NaN, as pandas' std of one value
                elif exact:
                    equal(_bits(got[r:r + 1]), _bits([sd]), what + " std row {} (exact)".format(r))
                else:
                    assert abs(float(got[r]) - float(sd)) <= np.spacing(sd), (what, r, got[r], sd)
            std.check(what + " std")
            if ddof == 1:
                m1, s1 = _out(R), _out(R)
                assert lib.xvb_topn_mean_std(_p(S), ncoh + 3, R, ncoh, top_n, _p(m1.view), _p(s1.view), None) == 0
                torch.cuda.synchronize()
                equal(_bits(m1.numpy()), _bits(mean.numpy()), what + " default-ddof entry mean")
                equal(_bits(s1.numpy()), _bits(std.numpy()), what + " default-ddof entry std")


@pytest.mark.parametrize("name", sorted(bx.topn_idx_cases()))
def test_topn_indices(lib, name):
    ncoh = bx.topn_idx_cases()[name]["ncoh"]
    _, vals = bx.topn_rows(ncoh, "idx" + name)
    R = vals.shape[0]
    S = _pitched(vals, ncoh + 5)
    for top_n in bx.topn_idx_tops(ncoh):
        out = _out(R * top_n, torch.int32)
        assert lib.xvb_topn_indices(_p(S), ncoh + 5, R, ncoh, top_n, _p(out.view), None) == 0
        torch.cuda.synchronize()
        what = "topn_indices {} top_n={}".format(name, top_n)
        equal(out.view.cpu().numpy().reshape(R, top_n), bx.topn_idx_ref(vals, top_n), what)
        out.check(what)


def test_topn_refusals(lib):
    big = torch.zeros(bx.TOPN_MAX + 1, dtype=torch.float32, device="cuda")
    m, s, idx = _out(1), _out(1), _out(bx.TOPN_IDX_MAX + 2, torch.int32)
    c = bx.TOPN_MAX + 1
    ci = bx.TOPN_IDX_MAX + 1
    calls = {
        "topn_mean_std ncoh=32769": lambda: lib.xvb_topn_mean_std_ddof(_p(big), c, 1, c, 5, 1, _p(m.view), _p(s.view), None),
        "topn_mean_std lds < ncoh": lambda: lib.xvb_topn_mean_std_ddof(_p(big), 99, 1, 100, 5, 1, _p(m.view), _p(s.view), None),
        "topn_mean_std ddof=2": lambda: lib.xvb_topn_mean_std_ddof(_p(big), 100, 1, 100, 5, 2, _p(m.view), _p(s.view), None),
        "topn_indices ncoh=16385": lambda: lib.xvb_topn_indices(_p(big), ci, 1, ci, 1, _p(idx.view), None),
        "topn_indices top_n > ncoh": lambda: lib.xvb_topn_indices(_p(big), 100, 1, 100, 101, _p(idx.view), None),
        "topn_indices top_n = 0": lambda: lib.xvb_topn_indices(_p(big), 100, 1, 100, 0, _p(idx.view), None),
    }
    for what, call in calls.items():
        assert call() == EINVAL, what
    torch.cuda.synchronize()
    for f in (m, s, idx):
        assert int((f.bits != f.sent).sum()) == 0, "a refused call wrote its output"


# ------------------------------------------------------------------------------------------------ score normalisation
def _snorm(lib, op, n):
    d = {k: _dev(op[k]) for k in ("s", "te", "tt", "me", "se", "mt", "st")}
    out = _out(n)
    dst = out.buf.data_ptr() + LEAD * 4            # an empty view's data_ptr() is NULL; the call takes any valid pointer
    rc = lib.xvb_snorm_trials(_p(d["s"]), _p(d["te"]), _p(d["tt"]), n, _p(d["me"]), _p(d["se"]), _p(d["mt"]), _p(d["st"]),
                              dst, None)
    return rc, out


@pytest.mark.parametrize("size", ["grid_stride", "small"])
def test_snorm_trials(lib, sms, size):
    n = bx.snorm_trials_count(sms) if size == "grid_stride" else 9
    op = bx.snorm_operands(n, size)
    rc, out = _snorm(lib, op, n)
    assert rc == 0
    _exact(out, bx.snorm_ref(op), "snorm_trials " + size)
    rc, out = _snorm(lib, op, 0)
    assert rc == 0
    torch.cuda.synchronize()
    out.check("snorm_trials with no trials")


@pytest.mark.parametrize("name", sorted(bx.cross_cases()))
def test_snorm_cross_trials(lib, name):
    case = bx.cross_cases()[name]
    op = bx.cross_operands(case, name)
    n, top_n = case["trials"], case["top_n"]
    ld = bx.CROSS_NCOH + 5
    ec, tc = _pitched(op["ec"], ld), _pitched(op["tc"], ld)
    s, te, tt, top_e, top_t = (_dev(op[k]) for k in ("s", "te", "tt", "top_e", "top_t"))
    out = _out(n)

    def call(tn):
        return lib.xvb_snorm_cross_trials(_p(s), _p(te), _p(tt), n, _p(ec), ld, _p(tc), ld, _p(top_e), _p(top_t), tn,
                                          _p(out.view), None)

    assert call(top_n) == 0
    _exact(out, bx.cross_ref(op), "snorm_cross_trials " + name)
    out.bits.fill_(out.sent)
    assert call(1) == EINVAL
    torch.cuda.synchronize()
    assert int((out.bits != out.sent).sum()) == 0, "a refused snorm_cross_trials wrote its output"


# ------------------------------------------------------------------------------------------------ transposed PLDA rows
def _fenced_T(case):
    return Fenced((case["D"] + 1, case["ldo"]), torch.float32, (slice(0, case["D"]), slice(0, case["N"])))


@pytest.mark.parametrize("name", sorted(bx.transpose_cases()))
def test_center_rows_transposed(lib, name):
    case = bx.transpose_cases()[name]
    op = bx.center_T_operands(case, name)
    x, spk, means, sw = (_dev(op[k]) for k in ("x", "spk", "means", "sw"))
    out = _fenced_T(case)
    assert lib.xvb_center_rows_transposed(_p(x), _p(spk), _p(means), _p(sw), case["N"], case["D"], _p(out.buf),
                                          case["ldo"], None) == 0
    _exact(out, bx.center_T_ref(op), "center_rows_transposed " + name)


@pytest.mark.parametrize("name", sorted(bx.transpose_cases()))
def test_plda_em_rows(lib, name):
    case = bx.transpose_cases()[name]
    op = bx.em_operands(case, name)
    u, n, w, psi = (_dev(op[k]) for k in ("u", "n", "w", "psi"))
    what, resid = _fenced_T(case), _fenced_T(case)
    assert lib.xvb_plda_em_rows(_p(u), _p(n), _p(w), _p(psi), case["N"], case["D"], _p(what.buf), _p(resid.buf),
                                case["ldo"], None) == 0
    _, _, a, b = bx.em_emulate(op)
    _exact(what, a, "plda_em_rows what " + name)
    _exact(resid, b, "plda_em_rows resid " + name)
