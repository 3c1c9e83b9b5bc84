"""The TDNN layer kernel's epilogues (tdnn_gemm.cu) at the edges the staged stores meet, on exact-arithmetic operands
(tests/staged_exact.py, tests/gemm_exact.py):

  * the fused pooling epilogue's full 8-frame blocks, whose partials are staged in shared memory and stored by one TMA
    store per tile through a (Cout, 2, B, time block) map of pool_partial: B not a multiple of 16, Cout 1500, 132 and 4,
    one and many time blocks, and a last time block shorter than 8 frames, which takes the general path in the same
    launch;
  * the staged layer epilogue at Cout % 64 == 32 (the last 64-channel store box half past Cout) on the 64-wide, the
    ping-pong 128-wide (one, two and three tiles per CTA) and the swish instances, masked and unmasked, into channel
    slices at an odd multiple of 8 in a pitch that is an odd multiple of 8.

Outputs are compared bit for bit with the float64 references (staged layers also with the direct-store run of the same
case), inside sentinel-filled buffers that must survive outside the logical output.  test_every_epilogue_edge_ran
checks from the kernel names and the shapes that the cases covered each of these paths."""
import numpy as np
import pytest
import torch

import gemm_exact as gx
import staged_exact as sx
import test_gpu_staged_epilogue as se
from gpu_checks import Fenced, equal, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as _ops
    assert torch.cuda.is_available()
    return _ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------ staged layers
# name -> (BLOCK_N, Cout, Tb, swish, masked, B tail of staged_shape)
LAYER = {
    "w64_cout96_tb8": (64, 96, 8, False, False, "past"),
    "w64_cout224_tb16_masked": (64, 224, 16, False, True, "part"),
    "w128_cout160_tb8": (128, 160, 8, False, False, "part"),
    "w128_cout288_tb4_masked": (128, 288, 4, False, True, "past"),
    "w128_cout160_tb32": (128, 160, 32, False, False, "past"),
    "swish_w128_cout160_tb8": (128, 160, 8, True, False, "past"),
    "swish_w64_cout96_tb16_masked": (64, 96, 16, True, True, "part"),
}
# the ping-pong instance at one, two and three tiles per CTA (both parities of the last tile's warpgroup): B x 8 frames
TILES = {"w128_cout160_tiles1": 1, "w128_cout160_tiles2": 2, "w128_cout160_tiles3": 3}


def layer_cases(sms):
    cases = {}
    for name, (bn, cout, tb, swish, masked, tail) in LAYER.items():
        B, T = sx.staged_shape(sms, tb, bn, cout, tail)
        c = dict(B=B, T=T, Cin=40, Cout=cout, ctx=[-1, 0, 2], relu=not swish, bn=True, inst=bn, tb=tb,
                 act="swish" if swish else None)
        if masked:
            c["lengths"] = sx._lengths(B, T, tb, cout + tb)
        cases[name] = c
    for name, k in TILES.items():
        # Cout 160 = two N blocks per M unit: k tiles per CTA for the 2 * (M units) tiles
        n = -(-(k - 1) * sms // 2) + 1 if k > 1 else sms // 2
        cases[name] = dict(B=16 * n - 5, T=8, Cin=40, Cout=160, ctx=[-1, 0, 1], relu=True, bn=True, inst=128, tb=8,
                           act=None)
    for c in cases.values():
        c["x_c0"] = 8
        c["ldx"] = gx._ru(c["x_c0"] + c["Cin"] + 8, 8)
        c["y_c0"] = 24                                   # an odd multiple of 8 ...
        c["ldy"] = gx._ru(24 + c["Cout"] + 40, 8)
        if (c["ldy"] // 8) % 2 == 0:                     # ... in a pitch that is an odd multiple of 8
            c["ldy"] += 8
        c["yf_c0"], c["ldyf"] = 4, gx._ru(4 + c["Cout"] + 4, 4)
        c["planes"] = True
    return cases


_SEEN = {}


def _layer(ops, sms, name):
    case = layer_cases(sms)[name]
    d = sx.make_staged(case, se._seed(name))
    want, bound = sx.staged_reference(case, d)
    bn, swish = case["inst"], case["act"] == "swish"
    assert se._tb(case["B"], case["T"]) == case["tb"], name
    assert sx.block_n(case, sms) == bn and sx.staged_taken(case, bn), name
    w = se._weight(ops, d, case["ctx"])
    res = {}

    def run():
        res["staged"] = se._run(ops, case, d, w, f32=False)

    seen = se._profiled(run)
    assert se._layer_name(bn, swish=swish) in seen, "{}: saw {}".format(name, sorted(seen))
    staged = res["staged"]
    direct = se._run(ops, case, d, w, f32=True)
    if bound is None:
        wh, wl = gx.split_bf16(want)
        equal(se._bits(staged["hi"].view), gx.bf16_bits(wh), name + " staged hi")
        equal(se._bits(staged["lo"].view), gx.bf16_bits(wl), name + " staged lo")
    else:
        within(direct["f32"].numpy(), want, bound, name + " direct y_f32")
    for k in ("hi", "lo"):
        equal(se._bits(staged[k].view), se._bits(direct[k].view), name + " staged vs direct " + k)
    if case.get("lengths"):
        dead = np.arange(case["T"])[None, :] >= np.asarray(case["lengths"])[:, None]
        for k in ("hi", "lo"):
            assert not se._bits(staged[k].view)[dead].any(), name + ": a masked row is not +0"
    for run_name, outs in (("staged", staged), ("direct", direct)):
        for k, f in outs.items():
            f.check("{} {} {}".format(name, run_name, k))
    _SEEN[("layer", name)] = dict(seen=seen, inst=(bn, swish), masked=bool(case.get("lengths")),
                                  tile_counts=sx.cta_tile_counts(sx.num_tiles(case, sms), sms))


@pytest.mark.parametrize("name", sorted(layer_cases(SMS_FOR_IDS)))
def test_staged_layer_half_box_exact(ops, sms, name):
    _layer(ops, sms, name)


# ------------------------------------------------------------------------------------------------ pooled TMA store
# (B, T, Cout): Tb = 8 for all of them
POOL = [(45, 200, 1500), (29, 200, 132), (21, 8, 4), (16, 8, 132), (43, 200, 4), (29, 21, 132), (13, 21, 1500)]


def pool_cases():
    return {"pool_B{}_T{}_cout{}".format(B, T, c): dict(B=B, T=T, Cin=sx.POOL_CIN, Cout=c, ctx=sx.POOL_CTX, relu=True,
                                                        bn=True, tb=8, x_c0=8, ldx=gx._ru(8 + sx.POOL_CIN + 8, 8))
            for B, T, c in POOL}


def _pool(ops, name):
    case = pool_cases()[name]
    B, T, Cout = case["B"], case["T"], case["Cout"]
    assert sx.choose_m_tile(B, T) == 8 and se._tb(B, T) == 8, name
    d = sx.make_pool(case, se._seed(name))
    y, bound = gx.layer_reference(case, d)
    assert bound is None
    exact, counts = sx.block_stats(y, 8)
    mask = np.broadcast_to(sx.pool_exact_blocks(8, counts)[:, None, None], exact.shape)
    x = se._poisoned(ops, *d["xs"][0], case["x_c0"], case["ldx"])
    w = se._weight(ops, d, case["ctx"])
    nblk = len(counts)
    n = nblk * B * 2 * Cout
    part = Fenced((n + 4 * Cout + 64,), torch.float32, slice(0, n))   # sentinel past the last partial

    def run():
        ops.tdnn_affine_ex(x, w, Cout, case["ctx"], bias=se._dev(d["bias"]), bn_scale=se._dev(d["scale"]),
                           bn_shift=se._dev(d["shift"]), relu=True, pool_partial=part.view)
        torch.cuda.synchronize()

    seen = se._profiled(run)
    assert se._layer_name(128, pool=True) in seen, sorted(seen)
    got = part.numpy().reshape(nblk, B, 2 * Cout)
    part.check(name + " partials")
    # the full 8-frame blocks are exact on this data, and so is a shorter last block of a power-of-two length
    assert mask[:len([c for c in counts if c == 8])].all()
    equal(np.where(mask, got, 0.0), np.where(mask, exact, 0.0), name + " partials (exact blocks)")
    within(got, exact, sx.pool_block_bounds(y, 8), name + " partials")
    _SEEN[("pool", name)] = dict(seen=seen, B=B, Cout=Cout, nblk=nblk, general=counts[-1] != 8)


@pytest.mark.parametrize("name", sorted(pool_cases()))
def test_pooled_tma_store_exact(ops, name):
    _pool(ops, name)


# ------------------------------------------------------------------------------------------------ coverage
def test_every_epilogue_edge_ran(ops, sms):
    """Every layer case ran its staged instance, the ping-pong instance ran with an odd and an even number of tiles per
    CTA, masked and unmasked, and the pooling cases covered B % 16 != 0, Cout
    1500, 132 and 4, one and many time blocks and the general path next to the staged one (cases not yet run in this
    session are run here)."""
    for name in layer_cases(sms):
        if ("layer", name) not in _SEEN:
            _layer(ops, sms, name)
    for name in pool_cases():
        if ("pool", name) not in _SEEN:
            _pool(ops, name)
    layers = {k[1]: v for k, v in _SEEN.items() if k[0] == "layer"}
    for name, v in layers.items():
        assert se._layer_name(v["inst"][0], swish=v["inst"][1]) in v["seen"], name
    assert {(64, False), (128, False), (128, True), (64, True)} <= {v["inst"] for v in layers.values()}
    counts = set().union(*(v["tile_counts"] for v in layers.values() if v["inst"] == (128, False)))
    assert {1, 2, 3} <= counts, sorted(counts)
    assert {v["masked"] for v in layers.values()} == {False, True}
    pools = [v for k, v in _SEEN.items() if k[0] == "pool" and se._layer_name(128, pool=True) in v["seen"]]
    assert len(pools) == len(POOL)
    assert any(v["B"] % 16 for v in pools) and {v["Cout"] for v in pools} == {1500, 132, 4}
    assert {1} <= {v["nblk"] for v in pools} and max(v["nblk"] for v in pools) > 1
    assert any(v["general"] for v in pools) and any(not v["general"] for v in pools)
