"""CPU checks of tests/pool_exact.py, the catalogue, references and bounds behind test_gpu_pooling_edges.py: every
listed kernel edge is in the catalogue, every mutant of a case (a kernel mistake of the kinds that go unseen) leaves the
bound by at least 4x, and a correct fp32 computation in two summation orders stays inside it."""
import zlib

import numpy as np
import pytest

import pool_exact as px

FAMILIES = ["stats", "finalize", "attn", "head", "lde", "plane"]
MARGIN = 4.0


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _family(kind):
    return {n: c for n, c in px.all_cases().items() if c["kind"] == kind}


def _flat(case, outs):
    return px.flat_output(case, outs)


def test_catalogue_reaches_every_edge():
    st = px.stats_cases()
    ts = {c["T"] for c in st.values()}
    assert {t % px.BOX for t in ts} >= {0, 1, px.BOX - 1} and {t % px.SLAB for t in ts} >= {0, 1}
    assert ts >= set(px.STATS_T) and {c["C"] for c in st.values()} >= set(px.STATS_C)
    assert {c["ldx"] - c["C"] for c in st.values()} >= set(px.STATS_PAD)
    assert {c["mode"] for c in st.values()} == {0, 1} and {c["eps"] for c in st.values()} == set(px.EPS)
    assert {(c["planes"], c["ldo_pad"]) for c in st.values()} >= {(True, 0), (True, 4), (False, 0)}
    lens = set().union(*(c["lengths"] for c in st.values() if c["lengths"]))
    assert lens >= {1, 40, 41, 200, 201, 400, 401} and any(c["lengths"] and max(c["lengths"]) == c["T"] for c in st.values())
    assert any(c["B"] == 65535 for c in st.values())

    fin = px.finalize_cases()
    assert {(c["nblk"], c["tb"]) for c in fin.values()} == {(n, t) for n in px.FIN_NBLK for t in px.FIN_TB}
    assert all(c["T"] in (c["nblk"] * c["tb"], (c["nblk"] - 1) * c["tb"] + 1) for c in fin.values())
    assert {(c["nblk"], c["tb"], c["T"]) for c in fin.values()} >= {(n, t, (n - 1) * t + 1) for n in px.FIN_NBLK for t in px.FIN_TB}
    assert {c["C"] for c in fin.values()} >= set(px.FIN_C)

    at = px.attn_cases()
    assert {c["T"] for c in at.values()} == set(px.ATTN_T) and {c["C"] for c in at.values()} == set(px.ATTN_C)
    assert all(c["ldl"] > c["C"] and c["ldx"] > c["C"] for c in at.values())
    assert {c["pattern"] for c in at.values()} == set(px.PATTERNS)
    ts = {c["T"] for c in at.values()}
    assert {t % px.ATTN_STRIDE for t in ts} >= {0, 1, px.ATTN_STRIDE - 1} and {t % px.WARPS for t in ts} >= {0, 1, px.WARPS - 1}

    hd = px.head_cases()
    for hmap in px.HEAD_MAPS:
        assert {c["T"] for n, c in hd.items() if n.startswith("head_{}_".format(hmap))} == set(px.ATTN_T), hmap
    assert any(c["gdiv"] == c["C"] and c["O"] == c["C"] for c in hd.values())               # one shared logit
    assert any(c["gdiv"] == 1 and c["O"] == c["C"] for c in hd.values())                    # per channel
    assert any(1 < c["gdiv"] < c["C"] and not c["mq"] for c in hd.values())                # heads
    assert any(c["O"] > c["C"] and c["gdiv"] == c["C"] and not c["mq"] for c in hd.values())  # global heads
    assert any(c["mq"] and c["head_width"] < c["C"] for c in hd.values())
    assert any(c["unweighted"] for c in hd.values()) and any(c["xi"] for c in hd.values())
    assert {c["vector"] for c in hd.values()} == {True, False}
    assert {c["pattern"] for c in hd.values()} == set(px.PATTERNS) | {"softplus"}

    ld = px.lde_cases()
    assert {c["K"] for c in ld.values()} == set(px.LDE_K) and {c["C"] for c in ld.values()} == set(px.LDE_C)
    assert {c["T"] for c in ld.values()} == set(px.LDE_T)
    straddle = [c for c in ld.values() if any((b * c["T"]) // px.LDE_ROWS != (b * c["T"] - 1) // px.LDE_ROWS
                                              for b in range(1, c["B"]))]
    assert straddle, "no weights CTA straddles an utterance boundary"

    pm = px.plane_cases()
    assert {c["C"] for c in pm.values()} >= set(px.PM_C) and {c["T"] for c in pm.values()} >= set(px.PM_T)
    assert any(c["ldx"] > c["C"] for c in pm.values())


def test_softplus_underflow_gets_no_weight():
    l = np.array([-200.0, -110.0, -104.5, -100.0, 0.0, 20.5, 30.0], dtype=np.float32)
    got = px.softplus2log(l)
    assert np.all(got[:3] == -np.inf) and np.all(np.isfinite(got[3:]))
    assert got[5] == 2 * np.log(np.float64(np.float32(20.5))) and got[4] == 2 * np.log(np.log(2.0))
    # an underflowed frame in fp32: expf(l) is 0, so log1pf(expf(l)) is 0 and its log is -inf
    with np.errstate(divide="ignore"):
        assert np.log(np.log1p(np.exp(np.float32(-104.5)))) == -np.inf


@pytest.mark.parametrize("kind", FAMILIES)
def test_mutants_leave_the_bound(kind):
    """Each mutant of each case moves an output past its bound by >= 4x, unless the mutation does not change the exact
    result at all (a frame whose fp32 weight underflows, a duplicated frame that carries all the weight); every mutant
    kind is caught in some case of the family."""
    caught, lines = {}, []
    for name, case in sorted(_family(kind).items()):
        d = px.make_case(case, _seed(name))
        ref = px.reference(case, d)
        want = _flat(case, {k: v[0] for k, v in ref.items()})
        bound = _flat(case, {k: v[1] for k, v in ref.items()})
        scale = np.nanmax(np.abs(want))
        for mname, outs in px.mutants(case, d):
            got = _flat(case, outs)
            r = px.worst_ratio(got, want, bound)
            with np.errstate(invalid="ignore"):
                effect = np.nanmax(np.where(np.isnan(got) & np.isnan(want), 0, np.abs(got - want)))
            lines.append("{:40s} {:28s} {:10.3g}".format(name, mname, r))
            if r >= MARGIN:
                caught[mname] = caught.get(mname, 0) + 1
                continue
            assert effect <= 1e-12 * scale, "{}: mutant '{}' stays within {:.3g} of its bound (change {:.3g})".format(
                name, mname, r, effect)
    print("\n".join(lines))
    kinds = {"drop marker frame", "duplicate marker frame", "split one frame off", "drop one warp's frames", "length - 1",
             "channel block shifted by 4"}
    if kind == "finalize":
        kinds |= {"block split one frame off", "drop block 1's partial"}
    assert kinds <= set(caught), "never caught: {}".format(sorted(kinds - set(caught)))


@pytest.mark.parametrize("kind", FAMILIES)
def test_bounds_hold_for_fp32_orders(kind):
    worst = 0.0
    for name, case in sorted(_family(kind).items()):
        d = px.make_case(case, _seed(name))
        ref = px.reference(case, d)
        want = _flat(case, {k: v[0] for k, v in ref.items()})
        bound = _flat(case, {k: v[1] for k, v in ref.items()})
        for order in ("seq", "pair"):
            got = _flat(case, px.simulate(case, d, order))
            r = px.worst_ratio(got, want, bound)
            assert r <= 1.0, "{} ({} fp32 sums): error {:.3g}x its bound".format(name, order, r)
            worst = max(worst, r)
    print("{}: largest fp32-simulation error / bound = {:.3g}".format(kind, worst))
