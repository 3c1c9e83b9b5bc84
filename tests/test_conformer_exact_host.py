"""CPU checks of tests/conformer_exact.py, the operands and references behind test_gpu_conformer_edges.py: the catalogue
holds the edges it is meant to, every case meets its exactness precondition (k-hot score gaps >= 128 with exact ties,
exact LayerNorm rows, exact GLU gates and conv sums), the host mirrors of the kernels' launch shapes, and the references
against torch float64."""
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conformer_exact as cx
import conformer_oracle as co
import gemm_exact as gx

SM_COUNTS = (132, 114, 78)


def _seed(name):
    """The seed test_gpu_conformer_edges.py gives a case: the preconditions are checked on the operands the GPU runs."""
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


# ------------------------------------------------------------------------------------------------ rotary attention
def test_quarter_rope_rotation_matches_the_oracle_and_inverts():
    rng = np.random.RandomState(0)
    for dk in (32, 64, 128):
        rope = cx.quarter_rope(rng, 50, dk)
        assert {tuple(p) for p in np.stack([rope[:, :dk // 2], rope[:, dk // 2:]], -1).reshape(-1, 2)} == \
            {tuple(p) for p in cx.QUARTER}
        x = rng.standard_normal((2, 3, 50, dk)).astype(np.float32)
        want = co._rotary(torch.from_numpy(x).double(), torch.from_numpy(rope).double()).numpy()
        assert np.array_equal(cx.rotate(x, rope), want.astype(np.float32))
        assert np.array_equal(cx.rotate(cx.unrotate(x, rope), rope), x)
        # the real table (not exact) rotates the same pairs
        real = co.rope_table(dk, 50).numpy()
        np.testing.assert_allclose(cx.rotate(x, real), co._rotary(torch.from_numpy(x), torch.from_numpy(real)).numpy(),
                                   rtol=0, atol=1e-5)


def test_attention_catalogue_covers_the_edges():
    cases = cx.attention_cases().values()
    assert set(cx.ATTN_T) <= {c["T"] for c in cases} and max(c["T"] for c in cases) >= 1500
    assert {(c["dk"], c["rot"]) for c in cases} == {(d, r) for d in (32, 64, 128) for r in ("none", "rope", "rope_v")}
    assert {1, 3, 8} <= {c["H"] for c in cases}
    assert {c["place"] for c in cases} == set(cx.ATTN_PLACES)
    for p in cx.ATTN_PLACES:
        assert any(c["place"] == p and c["T"] % 32 not in (0,) and c["T"] > 32 for c in cases), p
    assert any(c["mult"] != 1.0 for c in cases)
    for c in cases:
        D = c["H"] * c["dk"]
        assert c["ldq"] > c["q_c0"] + 3 * D and c["ldy"] > c["y_c0"] + D and c["ldy"] % 8 == 0


@pytest.mark.parametrize("name", sorted(cx.attention_cases()))
def test_khot_cases_have_exact_ties_and_gaps(name):
    """Every k-hot case: the group's keys tie exactly and score >= 128 above every other key, so expf is exactly 1 / 0."""
    case = cx.attention_cases()[name]
    d = cx.make_attention(case, _seed(name + "khot"), "khot")
    gap, tied = cx.attention_gaps(case, d)
    assert tied and gap >= 128, (gap, tied)
    assert np.float32(np.exp(np.float32(-128.0))) == 0 or gap >= 128
    for b, (gX, gY) in enumerate(d["groups"]):
        nt = -(-case["T"] // 32)
        tiles = {t // 32 for t in gX + gY}
        if case["place"] == "first":
            assert tiles == {0}
        elif case["place"] == "tail":
            assert tiles == {nt - 1}
        elif case["place"] == "later":
            assert 0 not in tiles
        elif nt > 1:
            assert len(tiles) > 1


def _softmax_ref(case, d):
    q, k, v = (torch.from_numpy(np.ascontiguousarray(a)).double() for a in cx._rotated(case, d))
    s = q @ k.transpose(-1, -2) / np.sqrt(case["dk"]) * case["mult"]
    out = torch.softmax(s, -1) @ v
    B, T, H, dk = case["B"], case["T"], case["H"], case["dk"]
    return out.permute(0, 2, 1, 3).reshape(B, T, H * dk).numpy()


@pytest.mark.parametrize("name", ["T65_dk32_H1_rope_v_spread", "edge_T64_dk32_rope_v_later", "T33_dk128_H8_rope_v_first",
                                  "T9_dk32_H1_none_tail"])
def test_attention_references_against_torch(name):
    case = cx.attention_cases()[name]
    for mode in ("uniform", "khot"):
        d = cx.make_attention(case, 3, mode)
        want = cx.attention_exact_reference(case, d, mode)
        ref = _softmax_ref(case, d)
        # float64 softmax differs from the kernel's rounded 1 / count by at most one rounding of each
        np.testing.assert_allclose(want, ref, rtol=2 ** -22, atol=0)
        assert np.all(want != 0)
    d = cx.make_attention(case, 3, "random")
    want, bound = cx.attention_random_bound(case, d)
    assert np.allclose(want, _softmax_ref(case, d), rtol=1e-12, atol=1e-12)
    assert np.all(bound > 0) and np.all(bound < 1e-2)
    # the khot stored operands differ from the rotated ones when a table is used (rotation is exercised)
    if case["rot"] != "none":
        d = cx.make_attention(case, 3, "khot")
        assert not np.array_equal(cx._rotated(case, d)[1], d["k"].transpose(0, 2, 1, 3))


def test_khot_corr_path_needs_the_rescale():
    """In a 'later' case the mid key wins tile 0; without the corr = 0 rescale its v would stay in o (and 1 in l)."""
    case = cx.attention_cases()["edge_T64_dk32_rope_v_later"]
    d = cx.make_attention(case, 5, "khot")
    s = cx.attention_scores(case, d)
    for b in range(case["B"]):
        row = s[b, 0, 0]
        assert row[:32].max() > -1e30 and row.max() - row[:32].max() >= 128


# ------------------------------------------------------------------------------------------------ LayerNorm
def test_ln_rows_per_cta_mirror():
    assert [cx.ln_warps(C) for C in cx.LN_C] == [8, 8, 8, 8, 8, 8, 8, 8, 7, 6, 5, 4, 3, 2, 1, 1]
    assert {cx.ln_warps(C) for C in cx.LN_C} == set(range(1, 9))


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_ln_catalogue_covers_the_edges(sms):
    cases = cx.ln_cases(sms).values()
    assert set(cx.LN_C) <= {c["C"] for c in cases}
    assert any(c["C"] % 32 for c in cases)
    grid = [c for c in cases if c["B"] * c["T"] > sms * 16 * c["warps"]]
    assert {c["warps"] for c in grid} >= {8, 1}
    rows = {c.get("table_rows") for c in cases}
    assert 1 in rows and any(c.get("table_rows") and (c["B"] * c["T"]) % c["table_rows"] for c in cases)
    assert {c["x_out"] for c in cases} == {"inplace", "other", None}
    assert {c.get("second") for c in cases} == {None, "plain", "gamma2"}
    assert {c.get("delta_scale") for c in cases} >= {0.5, 1.0}
    assert {c["act"] for c in cases} == set(cx.LN_ACTS)
    assert any(c["y"] and c["y_f32"] for c in cases)
    for c in cases:
        assert c["ldx"] > c["x_c0"] + c["C"] - 1 and c["ldy"] > c["C"] and c["ldyf"] > c["C"] and c["ldxo"] > c["C"]


def test_ln_cases_are_exact():
    for name, case in cx.ln_cases(132).items():
        d = cx.make_ln(case, _seed(name))
        v = d["x"].astype(np.float32)
        if "table" in d:
            v = v + d["table"][np.arange(case["B"] * case["T"]) % case["table_rows"]].reshape(v.shape)
        if "delta" in d:
            v = v + np.float32(case["delta_scale"]) * d["delta"]
        assert np.array_equal(v, d["row"]), name                 # the kernel's adds rebuild the row exactly
        r = cx.ln_reference(case, d)                                # asserts exact sums inside
        dev = d["row"] - d["row"].mean(axis=-1, keepdims=True)
        assert np.all(dev.sum(axis=-1) == 0) and np.all((dev.astype(np.float64) ** 2).sum(axis=-1) == case["C"] * 4.0 ** d["k"])
        assert np.all(np.isfinite(r["y"]))


def test_ln_reference_against_torch():
    cases = cx.ln_cases(132)
    names = [n for n in cases if n.split("_")[0] in ("C33", "C1025", "C4097")] + ["second_gamma2_C33_swish",
                                                                                 "second_plain_C1024_relu"]
    assert len(names) == 5
    for name in names:
        case = dict(cases[name], act="none")
        d = cx.make_ln(case, 5)
        x = torch.from_numpy(d["row"]).double()
        t = lambda k: torch.from_numpy(d[k]).double() if k in d else None      # noqa: E731
        ref = F.layer_norm(x, (case["C"],), t("gamma"), t("beta"), 0.0)
        if case.get("second"):
            ref = F.layer_norm(ref, (case["C"],), t("gamma2"), t("beta2"), 0.0)
        # torch's float64 statistics round in the last places; the exact rows leave nothing else to differ
        np.testing.assert_allclose(cx.ln_reference(case, d)["y"], ref.numpy(), rtol=1e-12, atol=1e-12, err_msg=name)


def test_ln_random_bound_holds_for_float32_emulation():
    case = dict(B=2, T=7, C=1500)
    x, g, b = cx.make_ln_random(case, 3)
    want, bound = cx.ln_random_bound(x.reshape(-1, 1500), g, b, 1e-5)
    # a float32 evaluation in numpy's own order stays within the bound
    xf = x.reshape(-1, 1500)
    m = xf.mean(axis=-1, keepdims=True, dtype=np.float32)
    dd = xf - m
    y = dd / np.sqrt((dd * dd).mean(axis=-1, keepdims=True, dtype=np.float32) + np.float32(1e-5)) * g + b
    assert np.all(np.abs(y - want) <= bound)
    assert float((bound / np.abs(want).max()).max()) < 1e-2


# ------------------------------------------------------------------------------------------------ convolution module
def test_glu_gates_are_exact():
    b = np.concatenate([np.linspace(20, 60, 50), -np.linspace(100, 200, 50)]).astype(np.float32)
    g = cx.glu_gate_is_exact(b)
    assert np.all(g[:50] == 1) and np.all(g[50:] == 0)


def test_conv_smem_mirror_and_catalogue():
    cmax = cx.conv_max_channels(31)
    assert cx.conv_smem(cmax, 31) <= 200 * 1024 < cx.conv_smem(cmax + 1, 31)
    cases = cx.conv_cases().values()
    assert set(cx.CONV_T) <= {c["T"] for c in cases} and set(cx.CONV_K) <= {c["K"] for c in cases}
    assert {8, 33, 256, cmax} <= {c["C"] for c in cases}
    assert any(c["K"] // 2 > c["T"] for c in cases)
    for norm in ("bn", "ln"):
        assert set(cx.CONV_T) <= {c["T"] for c in cases if c["norm"] == norm}
    for c in cases:
        assert c["ldx"] > c["x_c0"] + 2 * c["C"] and c["ldy"] > c["y_c0"] + c["C"]


def test_conv_cases_are_exact():
    """Every case: exact GLU gates and conv sums (asserted inside), and for the LayerNorm path an exact variance; acts
    none / relu exact, swish within bound."""
    for name, case in cx.conv_cases().items():
        d = cx.make_conv_module(case, _seed(name))
        for act in ("none", "relu", "swish"):
            want, bound = cx.conv_module_reference(case, d, act)
            assert want.shape == (case["B"], case["T"], case["C"]) and np.all(np.isfinite(want)), name
            assert (bound is None) == (act != "swish")
        if case["norm"] == "bn":
            g = cx.glu_gate_is_exact(d["x"][..., case["C"]:])
            assert 0.1 < (g == 0).mean() < 0.4, name              # both gate values occur


@pytest.mark.parametrize("name", ["T15_K3_C33_bn", "T33_K31_C256_ln", "K31_T5_ln", "T32_K15_C33_ln", "K15_T3_bn"])
def test_conv_reference_against_torch(name):
    case = cx.conv_cases()[name]
    d = cx.make_conv_module(case, 4)
    C, K = case["C"], case["K"]
    x = torch.from_numpy(d["x"]).double().transpose(1, 2)
    z = F.conv1d(F.glu(x, dim=1), torch.from_numpy(d["w"]).double().unsqueeze(1), torch.from_numpy(d["b"]).double(),
                 padding=K // 2, groups=C)
    na, nb = torch.from_numpy(d["na"]).double(), torch.from_numpy(d["nb"]).double()
    if case["norm"] == "bn":
        ref = (z * na[:, None] + nb[:, None]).transpose(1, 2)
    else:
        ref = F.layer_norm(z.transpose(1, 2), (C,), na, nb, 0.0)
    want, _ = cx.conv_module_reference(case, d, "none")
    # float64 sigmoid(b) of an open gate is 1 - O(e^-20), not 1: agreement to a few fp32 ulps
    np.testing.assert_allclose(want, ref.numpy(), rtol=0, atol=4 * 2.0 ** -24 * float(np.abs(want).max()))


def test_conv_time_shift_matters():
    """A one-frame shift of the conv window changes the exact outputs of every K > 1 case."""
    for name, case in cx.conv_cases().items():
        if case["K"] == 1 or case["norm"] != "bn" or case["T"] < 2:
            continue
        d = cx.make_conv_module(case, 9)
        w2 = dict(d, w=np.concatenate([d["w"][:, 1:], np.zeros_like(d["w"][:, :1])], axis=1))
        assert not np.array_equal(cx.conv_module_pre(case, d), cx.conv_module_pre(case, w2)), name


# ------------------------------------------------------------------------------------------------ subsampling head
@pytest.mark.parametrize("sms", SM_COUNTS)
def test_subsample_catalogue(sms):
    cases = cx.subsample_cases(sms).values()
    assert {c["sf"] for c in cases} == {1, 2}
    assert {3, 4, 5, 200} <= {c["T"] for c in cases} and {3, 4, 80} <= {c["F"] for c in cases}
    assert {8, 24, 256} <= {c["C"] for c in cases}
    assert {c["sf"] for c in cases if c["items"] > sms * 16 * 256} == {1, 2}


def test_subsample_reference_against_torch():
    for name, case in cx.subsample_cases(132).items():
        d = cx.make_subsample(case, 2)
        want = cx.subsample_reference(case, d)
        if case["items"] < 20000:
            ref = F.relu(F.conv2d(torch.from_numpy(d["x"]).double().unsqueeze(1), torch.from_numpy(d["w"]).double(),
                                  torch.from_numpy(d["b"]).double(), stride=(2, case["sf"]))).permute(0, 2, 3, 1)
            assert np.array_equal(want, ref.numpy()), name
        assert (want > 0).mean() > 0.2 and (want == 0).mean() > 0.1, name
