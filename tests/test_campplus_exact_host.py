"""CPU checks of tests/campplus_exact.py, the operands and references behind test_gpu_campplus_edges.py: the catalogue
holds the edges it is meant to, the shared-memory mirror matches the kernel's layout, every case meets its precondition,
the short last segment's divisor matters, and the references agree with a plain float64 restatement of CAMLayer."""
import zlib

import numpy as np
import pytest

import campplus_exact as ce
import gemm_exact as gx

SM_COUNTS = (132, 114, 78)


def test_cam_catalogue_covers_the_edges():
    cases = ce.cam_cases().values()
    b = [c for c in cases if not c["dense"]]
    assert {1, 99, 100, 101, 200, 201, 3000} <= {c["T"] for c in b}
    assert {1, 7, 100} <= {c["seg_len"] for c in b} and any(c["seg_len"] > c["T"] for c in b)
    assert {c["T"] % 100 for c in b if c["seg_len"] == 100 and c["T"] > 1} >= {0, 1, 99}
    assert {8, 424, 512, 2048} <= {c["C"] for c in b}
    assert {ce.cam_lanes(C) for C in (8, 424, 512, 2048)} == {256, 4, 1}
    assert ce.cam_lanes(424) * (424 // 8) < 256                      # idle threads
    assert any(c["smem"] > 48 * 1024 for c in cases) and all(c["smem"] <= ce.MAX_SMEM for c in cases)
    assert all(c["B"] > 1 for c in cases)
    assert any(c["dense"] for c in cases)
    for c in cases:
        assert c["ldh"] % 8 == 0 and c["ldh"] > c["h_c0"] + c["C"] and c["h_c0"] % 8 == 0
        if c["dense"]:
            assert c["T"] & (c["T"] - 1) == 0 and c["seg_len"] & (c["seg_len"] - 1) == 0


def test_cam_smem_mirror():
    """nseg * C contexts + nseg * R hidden + lanes * C partial sums, in floats."""
    assert ce.cam_gate_smem(3000, 512, 100, 256) == (30 * 512 + 30 * 256 + 4 * 512) * 4
    assert ce.cam_gate_smem(1, 8, 7, 16) == (8 + 16 + 256 * 8) * 4
    assert ce.cam_gate_smem(3000, 2048, 1, 16) > ce.MAX_SMEM


@pytest.mark.parametrize("name", sorted(ce.cam_cases()))
def test_cam_cases_are_exact_and_sensitive(name):
    case = ce.cam_cases()[name]
    d = ce.make_cam(case, zlib.crc32(name.encode()) & 0x7FFFFFFF)     # the operands test_gpu_campplus_edges.py runs
    want, bound = ce.cam_reference(case, d)                 # asserts the exact sums inside
    assert want.shape == (case["B"], case["nseg"], case["G"]) and np.all(np.isfinite(want))
    assert np.all(bound > 0)
    # the gates stay off saturation, so a context change shows in them
    assert float(np.mean((want > 1e-3) & (want < 1 - 1e-3))) > 0.5, name
    T, L = case["T"], case["seg_len"]
    if T % L and T > L:
        other, _ = ce.cam_reference(case, d, seg_len=L)
        assert np.any(np.abs(other - want) > 2 * bound), name      # the last segment's own length matters
    if not case["dense"]:
        assert np.all(np.count_nonzero(d["w1"], axis=1) == 1)
    assert np.all(np.count_nonzero(d["w2"], axis=1) == 1)


def test_cam_reference_against_float64_camlayer():
    """context = mean_T(h) + avg_pool1d(h, seg_len, ceil_mode) -> relu(W1 . + b1) -> sigmoid(W2 . + b2), in float64."""
    for name, case in ce.cam_cases().items():
        if case["T"] * case["C"] > 300000:
            continue
        d = ce.make_cam(case, 5)
        h = (d["h_hi"] + d["h_lo"]).astype(np.float64)
        T, L = case["T"], case["seg_len"]
        segs = [h[:, s * L:min(T, (s + 1) * L)].mean(axis=1) for s in range(case["nseg"])]
        ctx = h.mean(axis=1, keepdims=True) + np.stack(segs, axis=1)
        hid = np.maximum(ctx @ d["w1"].T.astype(np.float64) + d["b1"], 0)
        ref = 1 / (1 + np.exp(-(hid @ d["w2"].T.astype(np.float64) + d["b2"])))
        want, bound = ce.cam_reference(case, d)
        # float32 roundings of the mean, the segment mean, their sum, b1 and b2 (a few ulps each, times |W| <= 2)
        assert np.allclose(want, ref, rtol=0, atol=1e-5), name


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_bn_relu_catalogue_and_reference(sms):
    cases = ce.bn_relu_cases(sms)
    assert any(c["C"] == 8 for c in cases.values())
    assert any(c["items"] > sms * 32 * 256 for c in cases.values())
    for name, c in cases.items():
        assert c["x_c0"] != c["y_c0"] and c["ldx"] != c["ldy"] and c["ldx"] % 8 == 0 and c["ldy"] % 8 == 0
        if c["items"] < 100000:
            d = ce.make_bn_relu(c, 1)
            y = ce.bn_relu_reference(d)
            assert (y == 0).mean() > 0.2 and (y > 0).mean() > 0.2, name
            assert np.array_equal(y, np.maximum((d["hi"] + d["lo"]) * d["scale"] + d["shift"], 0)), name
            assert not np.any(np.signbit(y))
    assert gx.GRID == 2.0 ** -8
