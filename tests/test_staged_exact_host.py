"""CPU checks of tests/staged_exact.py, the catalogue behind test_gpu_staged_epilogue.py: the exactness precondition of
every case, the Tb and BLOCK_N each case is meant for (the Tb through the library's own choose_m_tile), the edges the
catalogue reaches, and that the integer pooling data makes the fused pooling epilogue's merges exact in fp32."""
import ctypes as C

import numpy as np
import pytest

import gemm_exact as gx
import staged_exact as sx

SM_COUNTS = (132, 114)   # H100 SXM and PCIe


def _lib_tb(B, T):
    from asv_subtools_b200._lib import lib
    tb = C.c_int()
    lib.xvb_pool_partial_blocks(B, T, C.byref(tb))
    return tb.value


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_staged_cases_are_exact(sms):
    """Every case meets gemm_exact's precondition (layer_acc asserts sum |terms| < 2^15, exact_f32 that the epilogue
    stays in fp32), and the masked rows of the reference are +0."""
    for name, case in sx.staged_cases(sms).items():
        d = sx.make_staged(case, 5)
        want, bound = sx.staged_reference(case, d)
        assert want.shape == (case["B"], case["T"], case["Cout"]), name
        assert (bound is None) == (case["act"] is None), name
        if bound is None:
            assert not np.signbit(want[want == 0]).any(), name + ": the kernel stores +0"
        if case.get("lengths"):
            dead = np.arange(case["T"])[None, :] >= np.asarray(case["lengths"])[:, None]
            assert np.all(want[dead] == 0) and not np.signbit(want[dead]).any(), name
            assert dead.any() and not dead.all(), name


def test_named_shapes_get_their_tb():
    """choose_m_tile's host mirror agrees with the library, and every case gets the Tb it is named for."""
    for sms in SM_COUNTS:
        for name, case in sx.staged_cases(sms).items():
            tb = _lib_tb(case["B"], case["T"])
            assert tb == sx.choose_m_tile(case["B"], case["T"]), name
            if "tb" in case:
                assert tb == case["tb"], (name, tb)
    for name, case in sx.pool_cases().items():
        assert _lib_tb(case["B"], case["T"]) == case["tb"], name
    rng = np.random.RandomState(3)
    for B, T in zip(rng.randint(1, 3000, 300), rng.randint(1, 700, 300)):
        assert _lib_tb(int(B), int(T)) == sx.choose_m_tile(int(B), int(T)), (B, T)


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_catalogue_reaches_every_edge(sms):
    cases = sx.staged_cases(sms)
    for name, c in cases.items():
        bn = sx.block_n(c, sms)
        assert bn == c["inst"] and sx.staged_taken(c, bn) == (not name.startswith("odd_")), name
        assert c["ldy"] % 8 == 0 and c["ldy"] > c["y_c0"] + c["Cout"] and c["y_c0"] in (8, 72), name
    assert {cases[n]["Cout"] % 64 for n in sx.ODD_COUT} == {1, 63}
    assert {cases[n]["inst"] for n in sx.ODD_COUT} == {64, 128}
    tails = [c for n, c in cases.items() if n.startswith("tail_")]
    for bn in (64, 128):
        mine = [c for c in tails if c["inst"] == bn]
        assert {c["tb"] for c in mine} == set(sx.TBS)
        assert {c["Cout"] % 64 for c in mine} >= {0, 8, 56}
        assert len({-(-c["Cout"] // 64) for c in mine}) >= 3       # one, two and more 64-channel pieces
        assert any(c["T"] % c["tb"] for c in mine if c["tb"] > 1)
        assert all(c["B"] % (128 // c["tb"]) for c in mine if c["tb"] < 128)
        # a whole 64-row store box past B: the last M tile's utterances end in its first half
        assert any(0 < c["B"] % (128 // c["tb"]) <= 64 // c["tb"] for c in mine if c["tb"] < 128)
        assert any(c["B"] % (128 // c["tb"]) > 64 // c["tb"] for c in mine if c["tb"] < 64)
    masked = [c for n, c in cases.items() if n.startswith("masked_")]
    assert {(c["inst"], c["act"] == "swish", c["tb"]) for c in masked} == \
        {(bn, sw, tb) for bn in (64, 128) for sw in (False, True) for tb in sx.TBS}
    for c in masked:
        T, tb, lens = c["T"], c["tb"], set(c["lengths"])
        assert {1, T - 1, T} <= lens and all(1 <= v <= T for v in lens)
        if tb > 1:
            assert any(v % min(tb, 64) for v in lens if v < T), "no length ends inside a store box"
        if T > tb > 1:
            assert any(v % tb == 0 for v in lens), "no length ends at a tile's edge"
    counts = set()
    for n in ("sms", "sms_p1", "2sms_m1", "3sms_p1"):
        c = cases["tiles_" + n]
        assert sx.num_tiles(c, sms) == c["tiles"] and sx.ping_pong(c["inst"], False)
        counts |= sx.cta_tile_counts(c["tiles"], sms)
    assert counts == {1, 2, 3, 4}
    flags = {k for c in cases.values() for k in ("x2", "im2col", "zero", "groups") if c.get(k)}
    assert flags == {"x2", "im2col", "zero", "groups"}
    assert {c["act"] for c in cases.values()} == {None, "swish", "tanh", "sigmoid"}
    assert {(bool(c.get("relu")), bool(c.get("bn"))) for c in cases.values() if c["act"] is None} == \
        {(a, b) for a in (False, True) for b in (False, True)}
    assert {c["Cout"] // c["groups"] % 128 == 0 for c in cases.values() if c.get("groups")} == {False, True}


@pytest.mark.parametrize("sms", SM_COUNTS)
def test_splitk_case(sms):
    case = sx.splitk_case(sms)
    assert sx.splitk_slices(case["Cin"]) == (7, 7)        # 47 channel blocks: 6 slices of 7 and one of 5
    assert case["B"] <= 1024 and -(-case["B"] // 128) * 7 * 4 >= sms
    want, bound = gx.layer_reference(case, gx.make_layer(case, 9))
    assert bound is None and want.shape == (case["B"], 1, 512)


@pytest.mark.parametrize("name", sorted(sx.pool_cases()))
def test_pool_data_is_exact_in_fp32(name):
    """The integer pooling data: the kernel's merge order, emulated in float32 and in float64, gives the exact block
    statistics in both wherever the merged counts are powers of two: every full 8-frame block (the division-free
    path), and for Tb <= 16 every block whose frame count is a power of two."""
    case = sx.pool_cases()[name]
    d = sx.make_pool(case, 13)
    y, bound = gx.layer_reference(case, d)
    assert bound is None and np.all(y == np.round(y)) and np.abs(y).max() <= 60
    tb = case["tb"]
    exact, counts = sx.block_stats(y, tb)
    e32 = sx.pool_partials_emulated(y, tb, np.float32).astype(np.float64)
    e64 = sx.pool_partials_emulated(y, tb, np.float64)
    claimed = sx.pool_exact_blocks(tb, counts)
    for g, n in enumerate(counts):
        if claimed[g]:
            assert np.array_equal(e32[g], exact[g]) and np.array_equal(e64[g], exact[g]), (name, g, n)
    if tb == 8:
        assert all(claimed[g] for g, n in enumerate(counts) if n == 8), "a full 8-frame block is not compared exactly"
    # where the emulation is not exact, it stays inside the bound the GPU test applies
    gx_bound = sx.pool_block_bounds(y, tb)
    assert np.all(np.abs(e32 - exact) <= gx_bound)
    # the data is not degenerate: blocks of more than one frame have nonzero M2, and the partials are not all equal
    assert (tb == 1 or np.abs(exact[:, :, case["Cout"]:]).max() > 0) and len(np.unique(exact)) > 20


def test_pool_catalogue():
    cases = sx.pool_cases()
    tbs = {c["tb"] for c in cases.values()}
    assert tbs == set(sx.TBS)
    assert {c["Cout"] % 128 for c in cases.values()} == {4, 64, 124}
    blocks = {c["tb"]: set() for c in cases.values()}
    for c in cases.values():
        nb = -(-c["T"] // c["tb"])
        blocks[c["tb"]] |= {min(c["tb"], c["T"] - g * c["tb"]) for g in range(nb)}
    assert {8, 4, 5} <= blocks[8]                          # full blocks, a power-of-two and another partial block
    assert any(c["tb"] == 8 and c["T"] % 8 == 0 for c in cases.values())
    for tb in (2, 4, 16, 32, 64, 128):
        assert tb in blocks[tb], "no full block at Tb={}".format(tb)


def test_merge_emulation_catches_the_full_block_weights():
    """A wrong weight in the full-block path's second merge (x 2 instead of x 4) moves M2 on this data: the exact
    comparison can see it."""
    case, = [c for c in sx.pool_cases().values() if (c["B"], c["T"]) == (16, 24)]
    y, _ = gx.layer_reference(case, sx.make_pool(case, 13))
    exact, _ = sx.block_stats(y, 8)
    blk = y[:, :8].astype(np.float64)
    left, right = blk[:, :4], blk[:, 4:]
    d = right.mean(axis=1) - left.mean(axis=1)
    m2 = ((left - left.mean(axis=1)[:, None]) ** 2).sum(1) + ((right - right.mean(axis=1)[:, None]) ** 2).sum(1)
    assert np.array_equal(m2 + d * d * 4 * 0.5, exact[0, :, case["Cout"]:])
    assert not np.array_equal(m2 + d * d * 2 * 0.5, exact[0, :, case["Cout"]:])
