"""CPU checks of tests/ecapa_exact.py, the operands and references behind test_gpu_ecapa_edges.py: the catalogue holds
the edges it is meant to, every case meets its exactness precondition, every Res2Net weight plane covers all 384 K
positions, and each product term of both sources moves some output."""
import numpy as np
import pytest

import ecapa_exact as ex
import gemm_exact as gx

SM_COUNTS = (132, 114, 78)   # H100 SXM, H100 PCIe, and a smaller part


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_res2net_catalogue_covers_the_edges(sms):
    cases = ex.res2net_cases(sms).values()
    ts = {c["T"] for c in cases}
    assert {1, 2, 127, 128, 129, 255, 256, 257} <= ts and max(ts) >= 24 * 128 - 127
    assert any(c["B"] == 1 and -(-c["T"] // 128) >= 20 for c in cases)
    assert {1, 2, 3, 4, 5} <= {c["d"] for c in cases}
    assert any(c["d"] == c["T"] - 1 for c in cases) and any(c["d"] == c["T"] and c["T"] > 1 for c in cases)
    assert any(c["d"] > 128 and c["T"] > c["d"] for c in cases)
    assert {2, 3, 4, 8, 12, 16} <= {c["scale"] for c in cases}
    bs = {c["B"] for c in cases}
    assert {1, sms - 1, sms, sms + 1, 2 * sms + 1} <= bs
    assert any(c["B"] > 2 * sms and c["T"] > 128 for c in cases)          # several utterances and tiles per CTA
    assert any(c["B"] > sms and c["scale"] == 2 for c in cases)           # one step_bar phase per utterance, repeated
    assert any(c.get("layers") and c["B"] > sms for c in cases) and any(c.get("layers") and c["T"] > 128 for c in cases)
    for c in cases:
        assert c["C"] == 128 * c["scale"]
        assert c["ldx"] % 8 == 0 and c["ldy"] % 8 == 0 and c["ldx"] != c["ldy"]
        assert c["ldx"] >= c["x_c0"] + c["C"] + 8 and c["ldy"] >= c["y_c0"] + c["C"] + 8
        assert c["x_c0"] % 8 == 0 and c["y_c0"] % 8 == 0 and c["x_c0"] > 0


def test_cover_planes_cover_every_k_position():
    for sms in SM_COUNTS:
        for name, case in ex.res2net_cases(sms).items():
            d = ex.make_res2net(case, 3)
            S = case["scale"] - 1
            assert d["w_hi"].shape == d["w_lo"].shape == (S * 128, 384)
            for plane in (d["w_hi"], d["w_lo"]):
                assert set(np.unique(plane)) == {-1.0, 0.0, 1.0}, name
                for st in range(S):
                    p = plane[st * 128:(st + 1) * 128]
                    assert np.all((p != 0).any(axis=0)), "{} step {}: a K position feeds no output row".format(name, st)
            for key in ("bias", "shift"):
                assert np.all(d[key] / gx.GRID == np.round(d[key] / gx.GRID)) and d[key].shape == (S * 128,)
            assert set(np.unique(d["scale"])) <= {-1.0, 1.0}
            # distinct per-step epilogue terms, so a step-index mix-up shows
            if S > 1:
                b = d["bias"].reshape(S, 128)
                assert all(not np.array_equal(b[0], b[i]) for i in range(1, S)), name


def test_res2net_cases_are_exact():
    """Every case, for every SM count: sum |terms| < 2^15 and an fp32-exact epilogue at every step (asserted inside the
    reference); chunk 0 passes through, the outputs are finite and the later chunks carry nonzero lo planes."""
    for sms in SM_COUNTS:
        for name, case in ex.res2net_cases(sms).items():
            d = ex.make_res2net(case, 11)
            yh, yl = ex.res2net_reference(case, d)
            assert yh.shape == (case["B"], case["T"], case["C"]), name
            assert np.array_equal(yh[..., :128], d["x"][0][..., :128]) and np.array_equal(yl[..., :128], d["x"][1][..., :128])
            assert np.all(np.isfinite(yh)) and np.all(np.isfinite(yl))
            assert np.array_equal(gx.bf16_round(yh), yh) and np.array_equal(gx.bf16_round(yl), yl)
            assert np.all(yl / gx.GRID == np.round(yl / gx.GRID)), name          # lo planes stay on the 2^-8 grid
            if case["T"] * case["B"] >= 100:
                assert (yl[..., 128:] != 0).mean() > 0.05, name


def test_res2net_reference_against_plain_chunk_chain():
    """The reference against a direct restatement of the block: for every step, the dilated 3-tap convolution of
    (x hi + x lo) with w_hi plus x hi with w_lo, and the same for the stored planes of the previous step."""
    case = dict(ex.res2net_cases(132)["scale4"], B=2, T=40, d=3)
    d = ex.make_res2net(case, 5)
    yh, yl = ex.res2net_reference(case, d)
    hx, lx = (a.astype(np.float64) for a in d["x"])
    T, dil = case["T"], case["d"]

    def conv(a, w):           # a (B, T, 128), w (128, 384) tap-major -> (B, T, 128)
        out = np.zeros(a.shape[:2] + (128,))
        for tap, off in enumerate((-dil, 0, dil)):
            for t in range(T):
                if 0 <= t + off < T:
                    out[:, t] += a[:, t + off] @ w[:, tap * 128:(tap + 1) * 128].T
        return out

    for st in range(case["scale"] - 1):
        r, k = slice(st * 128, (st + 1) * 128), slice((st + 1) * 128, (st + 2) * 128)
        wh, wl = d["w_hi"][r].astype(np.float64), d["w_lo"][r].astype(np.float64)
        acc = conv(hx[..., k] + lx[..., k], wh) + conv(hx[..., k], wl)
        if st:
            ph, pl = yh[..., r].astype(np.float64), yl[..., r].astype(np.float64)
            acc += conv(ph + pl, wh) + conv(ph, wl)
        v = np.maximum(acc + d["bias"][r], 0) * d["scale"][r] + d["shift"][r]
        h, lo = gx.split_bf16(v.astype(np.float32))
        assert np.array_equal(yh[..., k], h) and np.array_equal(yl[..., k], lo), st


@pytest.mark.parametrize("name", ["T129", "scale3", "scale16", "d_T-1"])
def test_every_product_term_of_both_sources_matters(name):
    """Leaving out any one of hi*w_hi, lo*w_hi, hi*w_lo of x or of the previous step's output changes the block output."""
    case = ex.res2net_cases(132)[name]
    d = ex.make_res2net(case, 7)
    full = ex.res2net_reference(case, d)
    for src in ("x", "y"):
        for term in ("hh", "lh", "hl"):
            try:
                got = ex.res2net_reference(case, d, drop=((src, term),))
            except AssertionError:
                continue      # the dropped term left the exact range: it certainly changed the output
            assert not (np.array_equal(got[0], full[0]) and np.array_equal(got[1], full[1])), (name, src, term)


# ------------------------------------------------------------------------------------------------ SE gate kernels
def test_se_catalogue():
    cases = ex.se_cases()
    assert {8, 24, 1024, 1536} <= {c["C"] for c in cases.values()}
    assert {1, 7, 61, 200} <= {c["T"] for c in cases.values()}
    assert any(c["B"] * c["T"] * c["C"] // 8 > 132 * 32 * 256 for c in cases.values())
    assert any(c.get("inplace") for c in cases.values())
    for c in cases.values():
        lds = (c["ldz"], c["ldin"], c["ldout"], c["ldnext"])
        assert all(ld % 8 == 0 and ld > c["C"] for ld in lds)
        assert len(set(lds)) == (3 if c.get("inplace") else 4)
    segs = ex.seg_gate_cases()
    assert {1, 7, 100} <= {c["seg_len"] for c in segs.values()}
    assert any(c["seg_len"] == c["T"] for c in segs.values()) and any(c["seg_len"] > c["T"] for c in segs.values())
    assert all(c["B"] > 1 for c in segs.values())
    assert {c["with_in"] for c in segs.values()} == {False, True}
    assert any(c["T"] % c["seg_len"] and c["seg_len"] < c["T"] for c in segs.values())


def test_se_reference_rounds_twice():
    """The reference is mul then add (two roundings): it differs from a fused z * g + in (one rounding, computed in
    float64 and rounded once) on ordinary data, so a fused kernel cannot pass the GPU test."""
    rng = np.random.RandomState(0)
    (zh, zl), (ih, il), g = ex.se_operands(rng, 2, 50, 64, 2)
    rows = ex.gate_rows(2, 50, 50)
    out, nxt = ex.se_reference((zh, zl), (ih, il), g, rows)
    z, x = (zh + zl).astype(np.float64), (ih + il).astype(np.float64)
    fused = (z * g[rows] + x).astype(np.float32)
    assert (fused != out).mean() > 0.01
    assert np.array_equal(nxt, out + (ih + il))
    # no residual: +0, whatever the sign of z * g
    z0 = (np.array([-0.0, -1.0, 1.0], np.float32), np.zeros(3, np.float32))
    o, _ = ex.se_reference(tuple(a.reshape(1, 1, 3) for a in z0), None, np.array([[1.0, 0.0, -0.0]], np.float32),
                           np.zeros((1, 1), int))
    assert np.all(o == 0) and not np.any(np.signbit(o))


def test_gate_rows():
    r = ex.gate_rows(2, 5, 2)
    assert r.tolist() == [[0, 0, 1, 1, 2], [3, 3, 4, 4, 5]]
    assert ex.gate_rows(3, 4, 9).tolist() == [[0] * 4, [1] * 4, [2] * 4]


# ------------------------------------------------------------------------------------------------ small affine
def test_small_affine_catalogue_and_exactness():
    cases = ex.small_affine_cases()
    assert set(ex.SA_B) <= {c["B"] for c in cases.values()}
    assert set(ex.SA_N) <= {c["N"] for c in cases.values()}
    assert set(ex.SA_K) <= {c["K"] for c in cases.values()}
    for B in ex.SA_B:
        assert len({c["K"] for c in cases.values() if c["B"] == B}) >= 1
    for name, case in cases.items():
        assert case["ldx"] > case["K"] + case["x_c0"] - 1 and case["ldx"] % 4 == 0 and case["x_c0"] % 4 == 0
        assert case["ldy"] > case["N"] and case["ldp"] >= case["p_c0"] + case["N"]
        d = ex.make_small_affine(case, 3)
        acc = ex.small_affine_acc(d)
        for ep, relu, bn, act in ex.SA_EPILOGUES:
            want, bound = ex.small_affine_reference(case, d, relu, bn, act, acc)
            assert want.shape == (case["B"], case["N"]), (name, ep)
            assert (bound is None) == (act is None)
            if bound is not None:
                assert np.all(bound > 0) and np.all(np.isfinite(want))
