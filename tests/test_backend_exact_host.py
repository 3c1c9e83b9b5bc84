"""tests/backend_exact.py on the CPU: the catalogue reaches every warp, CTA, block-cap, bitonic-padding, grid-stride and
tile edge of scoring.cu (read from the case lists), every exactness precondition holds, the references are what the
kernels' own order computes, and a kernel that drops a lane tail, a padding slot or a butterfly step would differ."""
import numpy as np
import pytest

import backend_exact as bx

H100_SMS = 132


def test_row_catalogue_reaches_every_lane_and_cta_edge():
    cases = list(bx.row_cases().values())
    assert {c["D"] % 32 for c in cases} >= {0, 1, 31} and min(c["D"] for c in cases) == 1
    assert max(c["D"] for c in cases) > 512 and any(c["D"] > 64 and c["D"] % 32 for c in cases)
    assert {c["n"] % bx.ROWS_PER_CTA for c in cases} >= {0, 1, 7} and min(c["n"] for c in cases) == 1
    assert any(c["n"] > 4000 and c["n"] % 8 == 1 for c in cases) and any(c["n"] > 4000 and c["n"] % 8 == 7 for c in cases)
    for n in bx.ROW_N:          # every optional operand present and absent at every count, and at every D
        assert {c["variant"] for c in cases if c["n"] == n} == {0, 1, 2, 3}
    for D in bx.ROW_D:
        assert {c["variant"] for c in cases if c["D"] == D} == {0, 1, 2, 3}
    terms = list(bx.plda_terms_cases().values())
    assert all(c["D"] % 4 == 0 for c in terms) and {c["D"] % 32 for c in terms} >= {0, 4}


def test_column_and_speaker_catalogue():
    cases = list(bx.column_cases(H100_SMS).values())
    G = 4 * H100_SMS
    assert {c["rows"] for c in cases} >= {1, 2, G - 1, G, G + 1} and max(c["rows"] for c in cases) > 10 * G
    Ds = {c["D"] for c in cases}
    assert {bx.COLUMN_BLOCK_CAP - 1, bx.COLUMN_BLOCK_CAP, bx.COLUMN_BLOCK_CAP + 1} <= Ds and max(Ds) > 2 * bx.COLUMN_BLOCK_CAP
    assert 1 in Ds and any(D % 32 for D in Ds if D < bx.COLUMN_BLOCK_CAP)
    sd = {c["D"] for c in bx.speaker_cases().values()}
    assert {bx.SPEAKER_BLOCK_CAP - 1, bx.SPEAKER_BLOCK_CAP, bx.SPEAKER_BLOCK_CAP + 1, 1} <= sd and max(sd) > 2 * bx.SPEAKER_BLOCK_CAP
    op = bx.speaker_operands(bx.speaker_cases()["D1"], "D1")
    counts = np.diff(op["off"])
    assert counts[0] == 0 and counts[-1] == 0 and 1 in counts and counts.max() > 32
    m = op["members"]
    assert len(np.unique(m)) < len(m) and np.any(np.diff(m) < 0)


def test_column_and_speaker_refs_are_exact():
    for name, case in bx.column_cases(H100_SMS).items():
        if case["rows"] * case["D"] > 2e6:
            continue
        op = bx.column_operands(case, name)
        s = op["x"].astype(np.float64)
        assert np.array_equal(np.cumsum(s[::-1], axis=0)[-1], s.sum(axis=0))   # the order does not matter
        assert np.abs(s).sum(axis=0).max() < 2 ** 40
    for name, case in bx.speaker_cases().items():
        ref = bx.speaker_ref(bx.speaker_operands(case, name))
        assert not ref[0].any() and not ref[3].any() and not ref[-1].any()     # empty speakers write zeros


def test_topn_catalogue_reaches_every_padding_and_cut():
    ncs = [c["ncoh"] for c in bx.topn_cases().values()]
    pads = {bx.next_pow2(c) - c for c in ncs}
    assert 0 in pads and 1 in pads and max(pads) > 10000                       # P = ncoh, P - 1 and far padding
    assert max(ncs) == bx.TOPN_MAX and min(ncs) == 1 and any(c > 16 * bx.TOPN_THREADS for c in ncs)
    assert {bx.next_pow2(c) for c in ncs} >= {bx.TOPN_THREADS // 16, bx.TOPN_THREADS, 2 * bx.TOPN_THREADS}   # P below, at, above the CTA
    for c in ncs:
        tops = bx.topn_tops(c)
        assert {0, 1, c, c + 7} <= set(tops) and (c == 1 or c - 1 in tops)
        assert bx.topn_select_n(c, 0) == c and bx.topn_select_n(c, c + 7) == c
    idx = [c["ncoh"] for c in bx.topn_idx_cases().values()]
    assert max(idx) == bx.TOPN_IDX_MAX and bx.TOPN_IDX_MAX - 1 in idx and 1 in idx
    for c in idx:
        assert {1, c} <= set(bx.topn_idx_tops(c)) and all(t <= c for t in bx.topn_idx_tops(c))


def test_topn_rows_have_ties_across_every_cut_and_exact_stds():
    exact_ns = set()
    for name, case in bx.topn_cases().items():
        c = case["ncoh"]
        k, vals = bx.topn_rows(c, name)
        assert np.array_equal(vals.astype(np.float64) * 8, k)
        srt = np.sort(k[0])[::-1]
        for top_n in bx.topn_tops(c):
            n = bx.topn_select_n(c, top_n)
            if 1 < n < c and c > 40:
                assert srt[n - 1] == srt[n]                                  # the cut falls inside a tie block
            for r in range(k.shape[0]):
                for ddof in (0, 1):
                    mean, std, exact = bx.topn_stats(k[r], n, ddof)
                    assert mean == np.float32(np.sort(vals[r].astype(np.float64))[::-1][:n].mean())
                    if n - ddof == 0:
                        assert np.isnan(std)
                    if exact:
                        exact_ns.add(n)
    assert {1, 2, 32, 512} <= exact_ns and max(exact_ns) >= 16384


def test_topn_idx_ref_orders_ties_by_index():
    row = np.array([1, 3, 3, 2, 3, 1], np.float32)
    assert bx.topn_idx_ref(row[None], 6).tolist() == [[1, 2, 4, 3, 0, 5]]


def test_warp_sum_matches_exact_sums_and_is_order_sensitive():
    rng = np.random.RandomState(3)
    t = bx.f32(rng.randint(-50, 51, (5, 600)))
    assert np.array_equal(bx.warp_sum_f32(t), t.astype(np.float64).sum(axis=1))
    r = bx.f32(rng.uniform(0, 1, (200, 65)))
    assert not np.array_equal(bx.warp_sum_f32(r), r.sum(axis=1, dtype=np.float32))   # the order is what is modelled


def test_exactness_preconditions_hold_for_every_case():
    for name, case in bx.row_cases().items():
        assert bx.fma_free_normalize(bx.plda_normalize_operands(case, name)), name
        assert bx.fma_free_llr(bx.llr_operands(case, name)), name
        bx.center_length_norm_ref(bx.center_length_norm_operands(case, name))   # asserts the integer sums
        bx.trials_ref(bx.trials_operands(case, name))
    for name, case in bx.plda_terms_cases().items():
        bx.plda_terms_ref(bx.plda_terms_operands(case, name))
    for name, case in bx.transpose_cases().items():
        assert bx.fma_free_em(bx.em_operands(case, name)), name
    for name, case in bx.cross_cases().items():
        assert bx.cross_exact(bx.cross_operands(case, name)), name


def test_power_of_four_rows_normalise_exactly():
    case = bx.row_cases()["D65_n9"]
    op = bx.center_length_norm_operands(case, "D65_n9")
    y = bx.center_length_norm_ref(op)
    for r in range(0, 9, 3):
        assert set(np.unique(np.abs(y[r]))) == {0.0, 1.0}


def test_cross_and_transpose_catalogue():
    tops = [c["top_n"] for c in bx.cross_cases().values()]
    assert {31, 32, 33} <= set(tops) and min(tops) == 2 and max(tops) > 256
    assert any(c["trials"] % 8 for c in bx.cross_cases().values()) and max(c["trials"] for c in bx.cross_cases().values()) > 4096
    cases = list(bx.transpose_cases().values())
    for k in ("N", "D"):
        assert {c[k] % bx.TILE for c in cases} >= {0, 1, 31} and max(c[k] for c in cases) > 3 * bx.TILE
    assert all(c["ldo"] > c["N"] for c in cases)
    for N in bx.TRANSPOSE_DIMS:
        assert {c["weighted"] for c in cases if c["N"] == N} == {False, True}


def test_snorm_trials_exceed_one_grid_stride_round():
    assert bx.snorm_trials_count(H100_SMS) > bx.SNORM_THREADS * bx.SNORM_CTAS_PER_SM * H100_SMS
    op = bx.snorm_operands(1000, "host")
    ref = bx.snorm_ref(op)
    assert ref.dtype == np.float32
    s64 = 0.5 * ((op["s"] - op["me"][op["te"]].astype(np.float64)) / op["se"][op["te"]] +
                 (op["s"] - op["mt"][op["tt"]].astype(np.float64)) / op["st"][op["tt"]])
    assert np.max(np.abs(ref - s64)) < 1e-5 * np.max(np.abs(s64))


def _llr_emulated_term(op):
    _, v, q = bx.llr_emulate(op)
    t = np.log(v).astype(np.float32) + q
    s = bx.warp_sum_f32(bx.f32(t))
    return (np.float32(-0.5) if op["side"] == 0 else np.float32(0.5)) * s


def test_llr_bound_holds_for_the_fp32_emulation_and_catches_a_dropped_lane():
    worst = 0.0
    for name, case in bx.row_cases().items():
        if case["n"] > 9:
            continue
        op = bx.llr_operands(case, name)
        ref, bound = bx.llr_term_ref_and_bound(op)
        got = _llr_emulated_term(op)
        worst = max(worst, float(np.max(np.abs(got - ref) / bound)))
        if case["D"] == 33 and op["side"] == 1:       # the tail lane's column dropped leaves the bound
            x = op["x"].copy()
            op2 = dict(op, x=x[:, :32], psi=op["psi"][:32])
            assert np.all(np.abs(_llr_emulated_term(op2) - ref) > 4 * bound)
    assert worst < 1.0


@pytest.mark.parametrize("D", [33, 65, 600])
def test_a_dropped_lane_tail_or_butterfly_step_is_caught(D):
    op = bx.plda_normalize_operands(dict(n=9, D=D, variant=1), "mut{}".format(D))
    ref = bx.plda_normalize_ref(op)
    x = op["x"].copy()
    x[:, 32 * (D // 32):] = 0                                   # the last lane pass skipped
    mut = bx.plda_normalize_ref(dict(op, x=x))
    assert np.any(mut != ref)
    t = bx.f32(op["x"] * op["x"])
    s_full = bx.warp_sum_f32(t)
    lanes = t[:, :32].copy()                                     # one butterfly step (o = 1) missing
    for o in (16, 8, 4, 2):
        lanes = lanes + lanes[:, np.arange(32) ^ o]
    assert np.any(lanes[:, 0] != s_full)
