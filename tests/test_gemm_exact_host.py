"""CPU checks of tests/gemm_exact.py, the exact-operand helpers behind test_gpu_gemm_edges.py: its bf16 split against
torch's conversion, and the exactness precondition of every case the GPU file generates."""
import ctypes as C

import numpy as np
import pytest
import torch

import gemm_exact as gx

SM_COUNTS = (132, 114)   # H100 SXM and PCIe


def _torch_bf16(x):
    return torch.from_numpy(x).to(torch.bfloat16).float().numpy()


def test_bf16_round_matches_torch():
    rng = np.random.RandomState(0)
    x = np.concatenate([
        rng.standard_normal(20000).astype(np.float32) * np.float32(2.0) ** rng.randint(-30, 30, 20000).astype(np.float32),
        # exact ties between two bf16 values, on both parities of the last kept bit
        ((rng.randint(1 << 7, 1 << 8, 4000) * 2 + 1).astype(np.float32) * np.float32(2.0 ** -9)) * rng.choice([-1, 1], 4000),
        np.array([0.0, -0.0, np.inf, -np.inf, 3.3895314e38, -3.3895314e38, 1e-40, -1e-40, 2.0 ** -133], dtype=np.float32),
    ]).astype(np.float32)
    got = gx.bf16_round(x)
    want = _torch_bf16(x)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    nan = gx.bf16_round(np.array([np.nan, -np.nan], dtype=np.float32))
    assert np.all(np.isnan(nan))


def test_split_bf16_matches_torch_and_recombines():
    rng = np.random.RandomState(1)
    x = (rng.standard_normal(50000) * 10.0 ** rng.uniform(-6, 6, 50000)).astype(np.float32)
    hi, lo = gx.split_bf16(x)
    assert np.array_equal(hi.view(np.uint32), _torch_bf16(x).view(np.uint32))
    assert np.array_equal(lo.view(np.uint32), _torch_bf16(x - hi).view(np.uint32))
    # hi + lo carries 16 significant bits: within 2^-16 of x, relative
    assert np.all(np.abs((hi.astype(np.float64) + lo) - x) <= 2.0 ** -16 * np.abs(x))
    # values on the grid of the exact cases split without loss
    g = (rng.randint(-2 ** 14, 2 ** 14, 10000) * gx.GRID).astype(np.float32)
    h, l = gx.split_bf16(g)
    assert np.array_equal(h.astype(np.float64) + l, g)
    assert np.array_equal(gx.bf16_bits(np.array([1.0, -2.0], np.float32)), np.array([0x3F80, 0xC000], np.uint16))


def test_operands_are_bf16_exact_and_bounded():
    rng = np.random.RandomState(2)
    hi, lo = gx.frame_planes(rng, (4, 5, 64))
    for a in (hi, lo, gx.pow2_scales(rng, 100)):
        assert np.array_equal(gx.bf16_round(a), a)
    g = gx.grid_values(rng, 1000)            # fp32 epilogue terms: on the 2^-8 grid, not bf16
    assert np.all(g / gx.GRID == np.round(g / gx.GRID)) and np.abs(g).max() <= 2
    assert np.abs(hi).max() <= 2 and np.all(hi == np.round(hi))
    assert np.abs(lo).max() <= 3 * gx.GRID and np.all(lo / gx.GRID == np.round(lo / gx.GRID))
    assert set(np.unique(gx.pow2_scales(rng, 1000))) == {0.5, 1.0, 2.0}
    # the precondition trips where fp32 could round
    with pytest.raises(AssertionError):
        gx.assert_exact_sum(9000, [hi], [lo], hi, lo)
    with pytest.raises(AssertionError):
        gx.exact_f32(np.array([1.0 + 2.0 ** -30]))


def test_every_tb_is_covered():
    """The Tb sweep shapes get the Tb they are named for from the library's own choose_m_tile."""
    from asv_subtools_b200._lib import lib
    for want, (b, t) in gx.TB_SHAPES.items():
        tb = C.c_int()
        lib.xvb_pool_partial_blocks(b, t, C.byref(tb))
        assert tb.value == want, (b, t, tb.value, want)
    pooled = set()
    for b, t, _ in gx.POOL_CASES:
        tb = C.c_int()
        lib.xvb_pool_partial_blocks(b, t, C.byref(tb))
        pooled.add(tb.value)
    assert pooled == {1, 2, 4, 8, 16, 32, 64, 128}
    assert {c % 128 for _, _, c in gx.POOL_CASES} == {4, 64, 124}


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_layer_catalogue_covers_the_issue_shapes(sms):
    cases = gx.layer_cases(sms)
    assert {c["Cin"] % 64 for c in cases.values()} >= {8, 16, 24, 40, 56, 0}
    assert {8, 72, 136, 200, 1544, 3000} <= {c["Cin"] for c in cases.values()}
    assert {1, 33, 129} <= {c["Cout"] for c in cases.values()}
    assert {c.get("inst") for c in cases.values() if c.get("act") == "swish"} == {32, 64, 128}
    assert {c.get("inst") for c in cases.values() if c.get("act") != "swish"} >= {32, 64, 128}
    assert max(c["B"] // 16 * -(-c["Cout"] // 128) for c in cases.values() if c.get("inst") == 128) > 2 * sms
    for c in cases.values():
        assert c["ldx"] % 8 == 0 and c["ldx"] > c["x_c0"] + c["Cin"] and c["ldy"] >= c["y_c0"] + c["Cout"]


def test_layer_cases_are_exact():
    """Every generated layer case meets the precondition (sum |terms| < 2^15) and its epilogue stays in fp32."""
    for sms in SM_COUNTS:
        for name, case in gx.layer_cases(sms).items():
            d = gx.make_layer(case, 7)
            want, bound = gx.layer_reference(case, d)
            assert want.shape == (case["B"], case["T"], case["Cout"]), name
            assert (bound is None) == (case.get("act") is None), name
            if bound is not None:
                assert np.all(bound > 0) and np.all(np.isfinite(want)), name


def test_pool_cases_are_exact():
    for b, t, cout in gx.POOL_CASES:
        case = gx.pool_case(b, t, cout)
        y, bound = gx.layer_reference(case, gx.make_layer(case, 11))
        assert bound is None
        mean, var, mb, vb = gx.pool_reference(y.astype(np.float64), 1)
        assert mean.shape == (b, cout) and np.all(var > 0) and np.all(mb >= 0) and np.all(vb >= 0)


def test_conv_cases_are_exact():
    for sms in SM_COUNTS:
        cases = gx.conv_cases(sms)
        assert {16, 32, 48, 64, 80, 96, 112, 128, 144} <= {c["Cin"] for c in cases.values()}
        assert {16, 48, 80, 144, 272} <= {c["Cout"] for c in cases.values()}
        assert {c.get("inst") for c in cases.values()} >= {32, 64, 128}
        # CAM++'s (2, 1) stride with k = 1 and 3, odd and even F, T > 256; and one (1, 2)
        fcm = [c for c in cases.values() if (c["s"], c["st"]) == (2, 1) and c["Cin"] == c["Cout"] == 32 and c["T"] > 256]
        assert {c["k"] for c in fcm} == {1, 3} and {c["F"] % 2 for c in fcm} == {0, 1}
        assert any((c["s"], c["st"]) == (1, 2) for c in cases.values())
        for name, case in cases.items():
            y, y2 = gx.conv_reference(case, gx.make_conv(case, 5))
            assert y.shape == (case["B"], case["To"], case["Fo"], case["Cout"]), name
            assert (y2 is None) == (not case.get("y2")), name


def test_conv_reference_matches_torch():
    """The im2col reference against F.conv2d (float64) on one strided, one tap-list and one valid case."""
    cases = gx.conv_cases(132)
    for name in ("w32_k3s2_cin80_cout48_res_y2", "taps_k5s2_cin96_cout16", "valid_k3s2_cin96_cout16_odd",
                 "fcm_k3_s2t1_F11_T300", "fcm_k1_s2t1_F10_T270", "k3_s1t2_F9_T41"):
        case = dict(cases[name], relu=False)
        d = gx.make_conv(case, 3)
        for k in ("scale", "res", "scale2"):
            d.pop(k, None)
        y, _ = gx.conv_reference(case, d)
        hx, lx = (torch.from_numpy(a).double().permute(0, 3, 2, 1) for a in d["x"])   # (B, C, F, T): "H" = F, "W" = T
        wh, wl = torch.from_numpy(d["w_int"]).double(), torch.from_numpy(d["w_frac"]).double()
        pad = 0 if case.get("valid") else case["k"] // 2
        conv = torch.nn.functional.conv2d
        stride = (case["s"], case["st"])                                               # (F, T)
        ref = conv(hx + lx, wh, stride=stride, padding=pad) + conv(hx, wl, stride=stride, padding=pad)
        assert np.array_equal(y, ref.permute(0, 3, 2, 1).numpy()), name


def test_score_and_histogram_references():
    for D in gx.SCORE_DIMS + gx.PLDA_DIMS:
        a, b = gx.score_operands(D, (37, 41), D)
        s = gx.int_matmul(a, b)
        assert np.array_equal(s, np.round(s)) and np.abs(s).max() <= 4 * D
    S = np.array([[-3.0, 0.0], [2.0, 7.0]])
    tgt = np.array([[True, False], [False, True]])
    h = gx.histogram_reference(S, tgt, np.ones_like(tgt), -4.5, 16)
    assert h[1, 2] == 1 and h[1, 12] == 1 and h[0, 5] == 1 and h[0, 7] == 1 and h.sum() == 4
