"""The staged epilogue of the TDNN layer kernel (tdnn_gemm.cu: outputs staged in shared memory and stored by TMA through
(Cout, T, B) store maps), its ping-pong 128-wide instance, split-K on that instance, and the fused pooling epilogue's
division-free path for full 8-frame blocks, on exact-arithmetic operands (tests/staged_exact.py, tests/gemm_exact.py).

Every layer case runs twice: plane-only, which takes the staged epilogue, and with planes + y_f32, which takes the
direct stores.  The staged planes must equal split_bf16 of the float64 reference bit for bit (or, for swish, tanh and
sigmoid, the direct run's planes, whose fp32 output lies within the derived bound), and bit for bit the direct run's
planes.  Inputs are NaN-poisoned channel slices, outputs are channel slices at channel 8 or 72 of a wider pitch with a
spare utterance, inside buffers filled with a sentinel that must survive outside the logical output: a store map whose
extents were the pitch or the allocation rather than Cout, T and B would write there.  The kernel instance that ran is
read from the kernel names, and test_every_staged_path_ran checks that the cases covered every staged instance at every
Tb, both tile parities of the ping-pong instance, masked and unmasked launches, both pooling paths and split-K."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest
import torch

import gemm_exact as gx
import staged_exact as sx
from gpu_checks import Fenced, equal, profiled, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132        # case names do not depend on the SM count; shapes do (built from multi_processor_count)


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as _ops
    assert torch.cuda.is_available()
    return _ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _tb(B, T):
    from asv_subtools_b200._lib import lib
    tb = C.c_int()
    lib.xvb_pool_partial_blocks(B, T, C.byref(tb))
    return tb.value


_KERNEL = re.compile(r"(tdnn_gemm_bf16x3_kernel)<([^>]*)>")


def _layer_name(block_n, pool=False, swish=False):
    return "tdnn_gemm_bf16x3_kernel<{},{},false,{}>".format(block_n, *("true" if f else "false" for f in (pool, swish)))


def _bits(t):
    """uint16 bit patterns of a bf16 tensor (view allowed)."""
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _poisoned(ops, hi, lo, c0, ld):
    """(B, T, C) planes as the channel slice [c0, c0 + C) of (B + 1, T, ld) buffers that hold NaN everywhere else."""
    B, Cn = hi.shape[0], hi.shape[-1]
    bufs = []
    for a in (hi, lo):
        buf = torch.full((B + 1,) + a.shape[1:-1] + (ld,), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B, ..., c0:c0 + Cn] = _dev(a).to(torch.bfloat16)
        bufs.append(buf)
    return ops.SplitPlanes(bufs[0][:B, ..., c0:c0 + Cn], bufs[1][:B, ..., c0:c0 + Cn], Cn)


def _im2col_input(ops, case, d):
    """The first layer's im2col view: frame t of utterance b is the k * Cin window at b * (T + k - 1) * Cin + t * Cin of
    time-padded planes; the spare utterance after the last one holds NaN."""
    B, T, k, c0 = case["B"], case["T"], case["im2col"], case["cin0"]
    bufs = []
    for p in d["pad"]:
        buf = torch.full((B + 1, T + k - 1, c0), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B] = _dev(p).to(torch.bfloat16)
        bufs.append(buf.as_strided((B, T, k * c0), ((T + k - 1) * c0, c0, 1)))
    return ops.SplitPlanes(bufs[0], bufs[1], k * c0), (T + k - 1) * c0


def _weight(ops, d, ctx):
    wi = ops.pack_tdnn_weight(_dev(d["w_int"]), ctx)
    wf = ops.pack_tdnn_weight(_dev(d["w_frac"]), ctx)
    zero = np.signbit(d["w_int"]).all(axis=(1, 2)) & (d["w_int"] == 0).all(axis=(1, 2))
    if zero.any():             # the signed-zero case: its all -0.0 rows, bit for bit in both packed planes
        rows = torch.from_numpy(zero).cuda()
        for p in (wi.hi, wf.hi):
            p.view(torch.int16)[rows] = -0x8000
    return ops.SplitPlanes(wi.hi, wf.hi, d["w_int"].shape[1])


def _profiled(run):
    """profiled() of gpu_checks, once more when its three captures all came back empty (the profiler's miss)."""
    return profiled(run, _KERNEL) or profiled(run, _KERNEL)


def _run(ops, case, d, w, f32):
    """One launch of a layer case: planes only (f32=False, the staged path) or planes + y_f32 (the direct stores), into
    fenced outputs.  -> {"hi", "lo"[, "f32"]: Fenced}."""
    B, T, Cout = case["B"], case["T"], case["Cout"]
    stride = 0
    if case.get("im2col"):
        x, stride = _im2col_input(ops, case, d)
    else:
        x = _poisoned(ops, *d["xs"][0], case["x_c0"], case["ldx"])
    x2 = _poisoned(ops, *d["xs"][1], case["x2_c0"], case["ldx2"]) if case.get("x2") else None
    idx = (slice(0, B), slice(None), slice(case["y_c0"], case["y_c0"] + Cout))
    outs = {"hi": Fenced((B + 1, T, case["ldy"]), torch.bfloat16, idx),
            "lo": Fenced((B + 1, T, case["ldy"]), torch.bfloat16, idx)}
    y = ops.SplitPlanes(outs["hi"].view, outs["lo"].view, Cout)
    yf = None
    if f32:
        outs["f32"] = Fenced((B + 1, T, case["ldyf"]), torch.float32,
                             (slice(0, B), slice(None), slice(case["yf_c0"], case["yf_c0"] + Cout)))
        yf = outs["f32"].view
    act = case.get("act")
    lengths = torch.tensor(case["lengths"], dtype=torch.int32, device="cuda") if case.get("lengths") else None
    ops.tdnn_affine_ex(x, w, Cout, case["ctx"], x2=x2, bias=_dev(d["bias"]),
                       bn_scale=_dev(d["scale"]) if "scale" in d else None, bn_shift=_dev(d["shift"]) if "shift" in d else None,
                       relu=bool(case.get("relu")), tanh=act == "tanh", sigmoid=act == "sigmoid", swish=act == "swish",
                       y=y, y_f32=yf, groups=case.get("groups", 1), x_batch_stride=stride, lengths=lengths)
    torch.cuda.synchronize()
    return outs


_SEEN = {}   # (group, case name) -> what the case ran: kernel names and the facts the coverage test asks about


# ------------------------------------------------------------------------------------------------ layer cases
def _layer_case(ops, sms, name):
    case = sx.staged_cases(sms)[name]
    d = sx.make_staged(case, _seed(name))
    want, bound = sx.staged_reference(case, d)
    if "tb" in case:
        assert _tb(case["B"], case["T"]) == case["tb"], name
    bn = case["inst"]
    assert sx.block_n(case, sms) == bn, name
    # the plane-only run takes the staged epilogue (unless Cout % 8 != 0) and the planes + y_f32 run the direct stores
    # (prepare_gemm: p.tma_store)
    staged_path = sx.staged_taken(case, bn)
    assert staged_path == (case["Cout"] % 8 == 0) and not sx.staged_taken(dict(case, f32=True), bn), name
    w = _weight(ops, d, case["ctx"])
    res = {}

    def run():
        res["staged"] = _run(ops, case, d, w, f32=False)

    seen = _profiled(run)
    swish = case["act"] == "swish"
    assert _layer_name(bn, swish=swish) in seen, "{}: expected {} to run, saw {}".format(name, _layer_name(bn, swish=swish),
                                                                                        sorted(seen))
    direct = _run(ops, case, d, w, f32=True)
    staged = res["staged"]
    if bound is None:
        wh, wl = gx.split_bf16(want)
        equal(direct["f32"].numpy(), want, name + " direct y_f32")
        equal(_bits(staged["hi"].view), gx.bf16_bits(wh), name + " staged hi")
        equal(_bits(staged["lo"].view), gx.bf16_bits(wl), name + " staged lo")
    else:                      # transcendental epilogue: fp32 within the derived bound, planes = split of that fp32
        got = direct["f32"].numpy()
        within(got, want, bound, name + " direct y_f32")
        wh, wl = gx.split_bf16(got)
        equal(_bits(direct["hi"].view), gx.bf16_bits(wh), name + " direct hi")
        equal(_bits(direct["lo"].view), gx.bf16_bits(wl), name + " direct lo")
    # every output byte of the staged path equals the direct path's
    equal(_bits(staged["hi"].view), _bits(direct["hi"].view), name + " staged hi vs direct")
    equal(_bits(staged["lo"].view), _bits(direct["lo"].view), name + " staged lo vs direct")
    if case.get("lengths"):    # rows past an utterance's end are +0 in both planes
        dead = np.arange(case["T"])[None, :] >= np.asarray(case["lengths"])[:, None]
        for k in ("hi", "lo"):
            assert not _bits(staged[k].view)[dead].any(), name + " staged " + k + ": a masked row is not +0"
    for run_name, outs in (("staged", staged), ("direct", direct)):
        for k, f in outs.items():
            f.check("{} {} {}".format(name, run_name, k))
    tiles = sx.num_tiles(case, sms)
    _SEEN[("layer", name)] = dict(seen=seen, inst=(bn, swish), tb=_tb(case["B"], case["T"]), staged=staged_path,
                                  masked=bool(case.get("lengths")), tile_counts=sx.cta_tile_counts(tiles, sms))
    return case


@pytest.mark.parametrize("name", sorted(sx.staged_cases(SMS_FOR_IDS)))
def test_staged_layer_exact(ops, sms, name):
    case = _layer_case(ops, sms, name)
    if "tiles" in case:
        assert sx.num_tiles(case, sms) == case["tiles"], name


# ------------------------------------------------------------------------------------------------ split-K
def _splitk_case(ops, sms):
    case = sx.splitk_case(sms)
    d = gx.make_layer(case, _seed("splitk_pingpong"))
    want, bound = gx.layer_reference(case, d)
    assert bound is None
    wh, wl = gx.split_bf16(want)
    assert sx.splitk_slices(case["Cin"]) == (7, 7)
    assert -(-case["B"] // 128) * 7 * 4 >= sms, "too few tiles for the 128-wide instance"
    w = _weight(ops, d, case["ctx"])
    seen = {}
    old = os.environ.get("XVB_SPLITK")
    try:
        for flag in ("1", "0"):            # XVB_SPLITK is read per plan
            os.environ["XVB_SPLITK"] = flag
            res = {}

            def run():
                res["out"] = _run(ops, case, d, w, f32=True)

            seen[flag] = _profiled(run)
            what = "splitk B={} XVB_SPLITK={}".format(case["B"], flag)
            out = res["out"]
            equal(out["f32"].numpy(), want, what + " y_f32")
            equal(_bits(out["hi"].view), gx.bf16_bits(wh), what + " hi")
            equal(_bits(out["lo"].view), gx.bf16_bits(wl), what + " lo")
            for k, f in out.items():
                f.check("{} {}".format(what, k))
    finally:
        if old is None:
            os.environ.pop("XVB_SPLITK", None)
        else:
            os.environ["XVB_SPLITK"] = old
    _SEEN[("splitk", "on")] = dict(seen=seen["1"])
    return seen


def test_splitk_on_the_ping_pong_instance(ops, sms):
    """Cin 3000 in 7 slices (6 of 7 channel blocks, one of 5) on the 128-wide ping-pong instance: a CTA with two tiles
    of different K lengths skips the other warpgroup's stages by counting K blocks."""
    seen = _splitk_case(ops, sms)
    assert _layer_name(128) in seen["1"], sorted(seen["1"])


# ------------------------------------------------------------------------------------------------ fused pooling
def _pool_case(ops, name):
    case = sx.pool_cases()[name]
    B, T, Cout, tb = case["B"], case["T"], case["Cout"], case["tb"]
    assert _tb(B, T) == tb, name
    d = sx.make_pool(case, _seed(name))
    y, bound = gx.layer_reference(case, d)
    assert bound is None
    exact, counts = sx.block_stats(y, tb)
    mask = np.broadcast_to(sx.pool_exact_blocks(tb, counts)[:, None, None], exact.shape)
    bnd = sx.pool_block_bounds(y, tb)
    x = _poisoned(ops, *d["xs"][0], case["x_c0"], case["ldx"])
    w = _weight(ops, d, case["ctx"])
    nblk = len(counts)
    n = nblk * B * 2 * Cout
    part = Fenced((n + 64,), torch.float32, slice(0, n))       # sentinel after the last partial
    res = {}

    def run():
        ops.tdnn_affine_ex(x, w, Cout, case["ctx"], bias=_dev(d["bias"]), bn_scale=_dev(d["scale"]),
                           bn_shift=_dev(d["shift"]), relu=True, pool_partial=part.view)
        res["out"], res["planes"] = ops.fused_pool_layer(x, w, Cout, case["ctx"], _dev(d["bias"]), _dev(d["scale"]),
                                                         _dev(d["shift"]), relu=True, planes=True)

    seen = _profiled(run)
    assert _layer_name(128, pool=True) in seen, sorted(seen)
    got = part.numpy().reshape(nblk, B, 2 * Cout)
    part.check(name + " partials")
    # bit for bit where the kernel's merges are exact on this data (every block with a power-of-two count for Tb <= 16,
    # the full 8-frame blocks among them), within the derived bound elsewhere
    equal(np.where(mask, got, 0.0), np.where(mask, exact, 0.0), name + " partials (exact elements)")
    within(got, exact, bnd, name + " partials")
    # the finalized statistics, as test_gpu_gemm_edges checks them
    mean, var, mb, vb = gx.pool_reference(y.astype(np.float64), tb)
    out = res["out"].cpu().numpy()
    within(out[:, :Cout], mean, mb, name + " mean")
    sd = out[:, Cout:].astype(np.float64)
    within(sd * sd, var, vb + 2.0 ** -22 * var, name + " std^2")
    wh, wl = gx.split_bf16(out)
    equal(res["planes"].hi.float().cpu().numpy().reshape(B, -1), wh, name + " planes hi")
    equal(res["planes"].lo.float().cpu().numpy().reshape(B, -1), wl, name + " planes lo")
    full = tb == 8 and 8 in counts
    _SEEN[("pool", name)] = dict(seen=seen, full_block=full, general=any(not (tb == 8 and c == 8) for c in counts))
    return seen


@pytest.mark.parametrize("name", sorted(sx.pool_cases()))
def test_fused_pooling_partials_exact(ops, name):
    _pool_case(ops, name)


# ------------------------------------------------------------------------------------------------ chained launches
def test_chained_staged_layers_match_synchronized(ops, sms):
    """Two staged layers back to back on one stream under the default programmatic dependent launch: the second reads
    the first's TMA-stored planes through TMA.  Bit for bit the same chain with a synchronize between the layers."""
    l1 = dict(sx.staged_cases(sms)["nobn_relu_w128"])
    d1 = sx.make_staged(l1, _seed("chain1"))
    want1, _ = sx.staged_reference(l1, d1)
    w1 = _weight(ops, d1, l1["ctx"])
    rng = np.random.RandomState(_seed("chain2"))
    ctx2, cout2 = [-2, 0, 2], 72
    w2i = gx.int_plane(rng, (cout2, l1["Cout"], 5), 1)
    w2 = ops.SplitPlanes(ops.pack_tdnn_weight(_dev(w2i), ctx2).hi,
                         ops.pack_tdnn_weight(_dev(gx.grid_plane(rng, (cout2, l1["Cout"], 5))), ctx2).hi, l1["Cout"])
    b2 = _dev(gx.grid_values(rng, cout2))
    l2 = dict(B=l1["B"], T=l1["T"], Cout=cout2)
    assert sx.block_n(l2, sms) == 64
    x = _poisoned(ops, *d1["xs"][0], l1["x_c0"], l1["ldx"])

    def chain(sync):
        idx = (slice(0, l1["B"]), slice(None), slice(l1["y_c0"], l1["y_c0"] + l1["Cout"]))
        o1 = [Fenced((l1["B"] + 1, l1["T"], l1["ldy"]), torch.bfloat16, idx) for _ in range(2)]
        idx2 = (slice(0, l1["B"]), slice(None), slice(8, 8 + cout2))
        o2 = [Fenced((l1["B"] + 1, l1["T"], 88), torch.bfloat16, idx2) for _ in range(2)]
        y1 = ops.SplitPlanes(o1[0].view, o1[1].view, l1["Cout"])
        ops.tdnn_affine_ex(x, w1, l1["Cout"], l1["ctx"], bias=_dev(d1["bias"]), relu=True, y=y1)
        if sync:
            torch.cuda.synchronize()
        ops.tdnn_affine_ex(y1, w2, cout2, ctx2, bias=b2, y=ops.SplitPlanes(o2[0].view, o2[1].view, cout2))
        torch.cuda.synchronize()
        return o1, o2

    seen = _profiled(lambda: chain(False))
    assert {_layer_name(128), _layer_name(64)} <= seen, sorted(seen)
    a1, a2 = chain(False)
    s1, s2 = chain(True)
    wh, wl = gx.split_bf16(want1)
    equal(_bits(a1[0].view), gx.bf16_bits(wh), "chained layer 1 hi")
    equal(_bits(a1[1].view), gx.bf16_bits(wl), "chained layer 1 lo")
    for k in range(2):
        equal(_bits(a1[k].view), _bits(s1[k].view), "layer 1 chained vs synchronized")
        equal(_bits(a2[k].view), _bits(s2[k].view), "layer 2 chained vs synchronized")
        for f in (a1[k], a2[k], s1[k], s2[k]):
            f.check("chain")
    assert not np.isnan(a2[0].numpy()).any()


# ------------------------------------------------------------------------------------------------ coverage
def test_every_staged_path_ran(ops, sms):
    """The cases above covered every staged instance at every Tb, tiles per CTA of both parities on the ping-pong
    instance, masked and unmasked staged launches, the full-block and the general pooling paths, and split-K on the
    128-wide instance (cases not yet run in this session are run here)."""
    for name in sx.staged_cases(sms):
        if ("layer", name) not in _SEEN:
            _layer_case(ops, sms, name)
    for name in sx.pool_cases():
        if ("pool", name) not in _SEEN:
            _pool_case(ops, name)
    if ("splitk", "on") not in _SEEN:
        _splitk_case(ops, sms)
    layers = [v for k, v in _SEEN.items()
              if k[0] == "layer" and v["staged"] and _layer_name(v["inst"][0], swish=v["inst"][1]) in v["seen"]]
    want = {(bn, sw, tb) for bn in (64, 128) for sw in (False, True) for tb in sx.TBS}
    got = {(v["inst"][0], v["inst"][1], v["tb"]) for v in layers}
    assert want <= got, "staged (BLOCK_N, swish, Tb) never ran: {}".format(sorted(want - got))
    for bn in (64, 128):
        assert {v["tb"] for v in layers if v["inst"] == (bn, False) and not v["masked"]} == set(sx.TBS), bn
    counts = set().union(*(v["tile_counts"] for v in layers if v["inst"] == (128, False)))
    assert {1, 2, 3, 4} <= counts, "ping-pong tiles per CTA seen: {}".format(sorted(counts))
    assert {v["masked"] for v in layers} == {False, True}
    pools = [v for k, v in _SEEN.items() if k[0] == "pool" and _layer_name(128, pool=True) in v["seen"]]
    assert any(v["full_block"] for v in pools) and any(v["general"] for v in pools)
    assert _layer_name(128) in _SEEN[("splitk", "on")]["seen"]
    print("staged instances and Tb seen:", sorted(got))
