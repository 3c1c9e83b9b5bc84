"""The wgmma GEMM kernels (tdnn_gemm.cu, conv2d.cu) on exact-arithmetic operands, compared bit for bit with a float64
reference (tests/gemm_exact.py), at every channel tail, kernel instance, Tb and buffer edge.

  * Inputs are poisoned: x and x2 are channel slices of wider buffers whose other channels, pitch padding and spare
    last utterance hold NaN (conv inputs: the first B utterances of a B + 1 buffer).  A frame map whose extent were the
    pitch or the allocation instead of Cin and B would multiply NaN into the result.
  * Outputs are fenced: y, y2 and y_f32 are views inside larger buffers filled with a sentinel bit pattern, with a spare
    utterance of rows after the last one; everything outside the logical output must be bitwise unchanged.
  * The kernel instances that ran are read from torch.profiler's kernel names, and every BLOCK_N of the layer, swish,
    pooling, histogram and convolution kernels must have run."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest
import torch

import gemm_exact as gx
from gpu_checks import Fenced as _Fenced, equal as _equal, profiled, within as _within

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


def _poisoned(ops, hi, lo, c0, ld):
    """(B, ..., C) planes as the channel slice [c0, c0 + C) of (B + 1, ..., ld) buffers that hold NaN everywhere else."""
    B, Cn = hi.shape[0], hi.shape[-1]
    bufs = []
    for a in (hi, lo):
        buf = torch.full((B + 1,) + a.shape[1:-1] + (ld,), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B, ..., c0:c0 + Cn] = _dev(a).to(torch.bfloat16)
        bufs.append(buf)
    return ops.SplitPlanes(bufs[0][:B, ..., c0:c0 + Cn], bufs[1][:B, ..., c0:c0 + Cn], Cn)


def _fenced_planes(ops, shape, index, channels):
    hi, lo = _Fenced(shape, torch.bfloat16, index), _Fenced(shape, torch.bfloat16, index)
    return hi, lo, ops.SplitPlanes(hi.view, lo.view, channels)


def _check_planes(hi, lo, want, what):
    """Plane outputs against split_bf16 of the wanted fp32 values, and the fences around them."""
    wh, wl = gx.split_bf16(want)
    _equal(hi.numpy(), wh, what + " hi")
    _equal(lo.numpy(), wl, what + " lo")
    hi.check(what + " hi")
    lo.check(what + " lo")


def _check_packed(wi, wf, w_int, w_frac, ntaps, cin):
    """The packers' layout: (Cout, ntaps * round_up(Cin, 16)), tap-major, the padding columns zero; the bf16-exact parts
    come back unchanged in .hi with .lo zero."""
    cp = (cin + 15) // 16 * 16
    for p, w in ((wi, w_int), (wf, w_frac)):
        hi = p.hi.float().cpu().numpy().reshape(w.shape[0], ntaps, cp)
        _equal(hi[:, :, :cin], w, "packed weight")
        assert not hi[:, :, cin:].any(), "packed weight: padding columns are not zero"
        assert not p.lo.float().cpu().numpy().any(), "packed weight: the lo plane of a bf16-exact weight is not zero"


_KERNEL = re.compile(r"(tdnn_gemm_bf16x3_kernel|conv2d_bf16x3_kernel)<([^>]*)>")


def _profiled(run):
    """The 'tdnn_gemm_bf16x3_kernel<128,false,false,false>'-style names of the GEMM kernels run() launched."""
    return profiled(run, _KERNEL)


def _layer_name(block_n, pool=False, hist=False, swish=False):
    return "tdnn_gemm_bf16x3_kernel<{},{},{},{}>".format(block_n, *("true" if f else "false" for f in (pool, hist, swish)))


_SEEN = {}   # (group, case) -> GEMM kernel instances it launched


# ------------------------------------------------------------------------------------------------ TDNN layer
def _layer_weight(ops, d, ctx, cin):
    wi = ops.pack_tdnn_weight(_dev(d["w_int"]), ctx)
    wf = ops.pack_tdnn_weight(_dev(d["w_frac"]), ctx)
    _check_packed(wi, wf, gx.taps_of(d["w_int"], ctx), gx.taps_of(d["w_frac"], ctx), len(ctx), cin)
    return ops.SplitPlanes(wi.hi, wf.hi, cin)


def _run_layer(ops, case, d, w):
    B, T, Cout = case["B"], case["T"], case["Cout"]
    x = _poisoned(ops, *d["xs"][0], case["x_c0"], case["ldx"])
    x2 = _poisoned(ops, *d["xs"][1], case["x2_c0"], case["ldx2"]) if case.get("x2") else None
    outs = {}
    y = yf = None
    if case.get("planes"):
        idx = (slice(0, B), slice(None), slice(case["y_c0"], case["y_c0"] + Cout))
        outs["hi"], outs["lo"], y = _fenced_planes(ops, (B + 1, T, case["ldy"]), idx, Cout)
    if case.get("f32"):
        outs["f32"] = _Fenced((B + 1, T, case["ldyf"]), torch.float32,
                              (slice(0, B), slice(None), slice(case["yf_c0"], case["yf_c0"] + Cout)))
        yf = outs["f32"].view
    act = case.get("act")
    ops.tdnn_affine_ex(x, w, Cout, case["ctx"], x2=x2, bias=_dev(d["bias"]),
                       bn_scale=_dev(d["scale"]) if "scale" in d else None, bn_shift=_dev(d["shift"]) if "shift" in d else None,
                       utt_bias=_dev(d["utt"]) if "utt" in d else None, row_bias=_dev(d["row"]) if "row" in d else None,
                       relu=bool(case.get("relu")), tanh=act == "tanh", sigmoid=act == "sigmoid", swish=act == "swish",
                       y=y, y_f32=yf)
    torch.cuda.synchronize()
    return outs


def _check_layer(outs, want, bound, what):
    if bound is None:
        if "f32" in outs:
            _equal(outs["f32"].numpy(), want, what + " y_f32")
        if "hi" in outs:
            _check_planes(outs["hi"], outs["lo"], want, what + " y")
    else:                       # transcendental epilogue: fp32 within the derived bound, planes = split of that fp32
        got = outs["f32"].numpy()
        _within(got, want, bound, what + " y_f32")
        if "hi" in outs:
            _check_planes(outs["hi"], outs["lo"], got, what + " y")
    for k, f in outs.items():
        f.check("{} {}".format(what, k))


def _layer_case(ops, sms, name):
    case = gx.layer_cases(sms)[name]
    d = gx.make_layer(case, _seed(name))
    want, bound = gx.layer_reference(case, d)
    if "tb" in case:
        assert _tb(case["B"], case["T"]) == case["tb"]
    w = _layer_weight(ops, d, case["ctx"], case["Cin"])

    def run():
        if not case.get("splitk"):
            _check_layer(_run_layer(ops, case, d, w), want, bound, name)
            return
        # XVB_SPLITK is read per plan: the same call with split-K on and off; exact data makes both bitwise equal
        old = os.environ.get("XVB_SPLITK")
        try:
            for flag in ("1", "0"):
                os.environ["XVB_SPLITK"] = flag
                _check_layer(_run_layer(ops, case, d, w), want, bound, "{} XVB_SPLITK={}".format(name, flag))
        finally:
            if old is None:
                os.environ.pop("XVB_SPLITK", None)
            else:
                os.environ["XVB_SPLITK"] = old

    seen = _profiled(run)
    _SEEN[("layer", name)] = seen
    return case, seen


@pytest.mark.parametrize("name", sorted(gx.layer_cases(SMS_FOR_IDS)))
def test_tdnn_layer_exact(ops, sms, name):
    case, seen = _layer_case(ops, sms, name)
    if "inst" in case:
        want = _layer_name(case["inst"], swish=case.get("act") == "swish")
        assert want in seen, "{}: expected {} to run, saw {}".format(name, want, sorted(seen))


# ------------------------------------------------------------------------------------------------ fused pooling
def _pool_case(ops, B, T, Cout):
    case = gx.pool_case(B, T, Cout)
    d = gx.make_layer(case, _seed("pool{}x{}x{}".format(B, T, Cout)))
    y, _ = gx.layer_reference(case, d)
    tb = _tb(B, T)
    mean, var, mb, vb = gx.pool_reference(y.astype(np.float64), tb)
    x = _poisoned(ops, *d["xs"][0], case["x_c0"], case["ldx"])
    w = _layer_weight(ops, d, case["ctx"], case["Cin"])
    res = {}

    def run():
        res["out"], res["planes"] = ops.fused_pool_layer(x, w, Cout, case["ctx"], _dev(d["bias"]), _dev(d["scale"]),
                                                         _dev(d["shift"]), relu=True, planes=True)

    seen = _profiled(run)
    got, op = res["out"].cpu().numpy(), res["planes"]
    what = "pool B={} T={} Cout={} (Tb={})".format(B, T, Cout, tb)
    _within(got[:, :Cout], mean, mb, what + " mean")
    sd = got[:, Cout:].astype(np.float64)
    _within(sd * sd, var, vb + 2.0 ** -22 * var, what + " std^2")
    wh, wl = gx.split_bf16(got)
    _equal(op.hi.float().cpu().numpy().reshape(B, -1), wh, what + " planes hi")
    _equal(op.lo.float().cpu().numpy().reshape(B, -1), wl, what + " planes lo")
    _SEEN[("pool", (B, T, Cout))] = seen
    return tb, seen


@pytest.mark.parametrize("B,T,Cout", gx.POOL_CASES)
def test_fused_pooling_every_tb(ops, B, T, Cout):
    tb, seen = _pool_case(ops, B, T, Cout)
    assert _layer_name(128, pool=True) in seen, sorted(seen)


# ------------------------------------------------------------------------------------------------ score GEMMs
@pytest.mark.parametrize("D", gx.SCORE_DIMS)
def test_score_matrices_exact(ops, D):
    rng = np.random.RandomState(D)
    a, b, c = gx.score_operands(D, (259, 132, 68), D)
    row, col = gx.int_plane(rng, 259, 5), gx.int_plane(rng, 132, 5)
    got = ops.matmul_nt(_dev(a), _dev(b), row_bias=_dev(row), col_bias=_dev(col)).cpu().numpy()
    _equal(got, gx.exact_f32(gx.int_matmul(a, b) + row[:, None] + col[None, :]), "matmul_nt D={}".format(D))
    _equal(ops.cosine_matrix(_dev(a), _dev(c)).cpu().numpy(), gx.exact_f32(gx.int_matmul(a, c)), "cosine_matrix D={}".format(D))


@pytest.mark.parametrize("D", gx.PLDA_DIMS)
def test_plda_matrix_exact(ops, D):
    rng = np.random.RandomState(100 + D)
    e, t = gx.score_operands(D + 1, (133, 72), D)
    l2 = gx.int_plane(rng, (D, D), 1)
    row, col = gx.int_plane(rng, 133, 5), gx.int_plane(rng, 72, 5)
    got = ops.plda_matrix(_dev(e), _dev(t), _dev(l2), _dev(row), _dev(col)).cpu().numpy()
    el = gx.int_matmul(e, l2)                 # E' = E . L2^T, exact integers
    _equal(got, gx.exact_f32(gx.int_matmul(el, t) + row[:, None] + col[None, :]), "plda_matrix D={}".format(D))


def _hist_case(ops, D):
    """Integer embeddings and row / column terms with unit-width bins starting at lo = -1000.5: every score sits on a bin
    centre, so the counters must equal the float64 histogram exactly.  Symmetric mode over N = 300 or 520 (not a multiple
    of 256: the diagonal exclusion at 128 x 128 tile edges and a ragged last block), and enroll x test."""
    rng = np.random.RandomState(200 + D)
    n = 300 if D in (8, 150) else 520
    lo, nbins = -1000.5, 2048
    hi = lo + (nbins - 2)
    emb, = gx.score_operands(300 + D, (n,), D)
    spk = rng.randint(0, n // 6, n).astype(np.int32)
    row, col = gx.int_plane(rng, n, 5), gx.int_plane(rng, n, 5)
    ne, nt = 333, 301
    e, t = gx.score_operands(400 + D, (ne, nt), D)
    es, ts = rng.randint(0, 40, ne).astype(np.int32), rng.randint(0, 40, nt).astype(np.int32)
    r, c = gx.int_plane(rng, ne, 5), gx.int_plane(rng, nt, 5)

    def run():
        h = ops.trial_histogram(_dev(emb), _dev(spk), _dev(emb), _dev(spk), lo, hi, nbins, row_term=_dev(row),
                                col_term=_dev(col), symmetric=True).cpu().numpy()
        S = gx.int_matmul(emb, emb) + row[:, None] + col[None, :]
        tgt = spk[:, None] == spk[None, :]
        _equal(h, gx.histogram_reference(S, tgt, np.triu(np.ones((n, n), bool), 1), lo, nbins), "symmetric D={} N={}".format(D, n))
        h = ops.trial_histogram(_dev(e), _dev(es), _dev(t), _dev(ts), lo, hi, nbins, row_term=_dev(r),
                                col_term=_dev(c)).cpu().numpy()
        S = gx.int_matmul(e, t) + r[:, None] + c[None, :]
        _equal(h, gx.histogram_reference(S, es[:, None] == ts[None, :], np.ones((ne, nt), bool), lo, nbins),
               "enroll x test D={}".format(D))

    seen = _profiled(run)
    _SEEN[("hist", D)] = seen
    return seen


@pytest.mark.parametrize("D", gx.SCORE_DIMS)
def test_trial_histogram_exact(ops, D):
    seen = _hist_case(ops, D)
    assert _layer_name(128, hist=True) in seen, sorted(seen)


# ------------------------------------------------------------------------------------------------ convolution
def _conv_case(ops, sms, name):
    case = gx.conv_cases(sms)[name]
    d = gx.make_conv(case, _seed(name))
    want, want2 = gx.conv_reference(case, d)
    B, To, Fo, Cin, Cout, k = case["B"], case["To"], case["Fo"], case["Cin"], case["Cout"], case["k"]
    taps = case["taps"]
    kept = taps if taps is not None else list(range(k * k))
    wi = ops.pack_conv2d_weight(_dev(d["w_int"]), taps)
    wf = ops.pack_conv2d_weight(_dev(d["w_frac"]), taps)
    _check_packed(wi, wf, d["w_int"].reshape(Cout, Cin, k * k)[:, :, kept].transpose(0, 2, 1),
                  d["w_frac"].reshape(Cout, Cin, k * k)[:, :, kept].transpose(0, 2, 1), len(kept), Cin)
    w = ops.SplitPlanes(wi.hi, wf.hi, Cin)
    x = _poisoned(ops, *d["x"], 0, Cin)                          # spare utterance B is NaN
    res = _poisoned(ops, *d["res"], 0, Cout) if "res" in d else None
    shape, idx = (B + 1, To, Fo, Cout), (slice(0, B),)
    outs = {}
    y = y2 = yf = None
    if case.get("y"):
        outs["y hi"], outs["y lo"], y = _fenced_planes(ops, shape, idx, Cout)
    if case.get("y2"):
        outs["y2 hi"], outs["y2 lo"], y2 = _fenced_planes(ops, shape, idx, Cout)
    if case.get("yf"):
        outs["y_f32"] = _Fenced(shape, torch.float32, idx)
        yf = outs["y_f32"].view

    def run():
        ops.conv2d(x, w, Cout, k, stride=case["s"], scale=_dev(d["scale"]) if "scale" in d else None,
                   shift=_dev(d["shift"]) if "shift" in d else None, res=res, relu=bool(case.get("relu")), y=y, y_f32=yf,
                   scale2=_dev(d["scale2"]) if "scale2" in d else None, shift2=_dev(d["shift2"]) if "shift2" in d else None,
                   y2=y2, taps=taps, valid=bool(case.get("valid")), stride_t=case["st"] if case["st"] != case["s"] else 0)

    seen = _profiled(run)
    if y is not None:
        _check_planes(outs["y hi"], outs["y lo"], want, name + " y")
    if y2 is not None:
        _check_planes(outs["y2 hi"], outs["y2 lo"], want2, name + " y2")
    if yf is not None:
        _equal(outs["y_f32"].numpy(), want, name + " y_f32")
        outs["y_f32"].check(name + " y_f32")
    _SEEN[("conv", name)] = seen
    return case, seen


@pytest.mark.parametrize("name", sorted(gx.conv_cases(SMS_FOR_IDS)))
def test_conv2d_exact(ops, sms, name):
    case, seen = _conv_case(ops, sms, name)
    if "inst" in case:
        want = "conv2d_bf16x3_kernel<{}>".format(case["inst"])
        assert want in seen, "{}: expected {} to run, saw {}".format(name, want, sorted(seen))


# ------------------------------------------------------------------------------------------------ instance coverage
def test_every_gemm_instance_ran(ops, sms):
    """Every BLOCK_N of the layer kernel, its swish instances, the pooling and histogram instances and every BLOCK_N of
    the convolution ran in the cases above (cases not yet run in this session are run here)."""
    for name in gx.layer_cases(sms):
        if ("layer", name) not in _SEEN:
            _layer_case(ops, sms, name)
    for B, T, Cout in gx.POOL_CASES:
        if ("pool", (B, T, Cout)) not in _SEEN:
            _pool_case(ops, B, T, Cout)
    for D in gx.SCORE_DIMS:
        if ("hist", D) not in _SEEN:
            _hist_case(ops, D)
    for name in gx.conv_cases(sms):
        if ("conv", name) not in _SEEN:
            _conv_case(ops, sms, name)
    assert {_tb(B, T) for B, T, _ in gx.POOL_CASES} == {1, 2, 4, 8, 16, 32, 64, 128}
    assert {c["tb"] for c in gx.layer_cases(sms).values() if "tb" in c} == {1, 2, 4, 8, 16, 32, 64, 128}
    seen = set().union(*_SEEN.values())
    want = {_layer_name(n) for n in (32, 64, 128)} | {_layer_name(n, swish=True) for n in (32, 64, 128)} | \
        {_layer_name(128, pool=True), _layer_name(128, hist=True)} | {"conv2d_bf16x3_kernel<{}>".format(n) for n in (32, 64, 128)}
    assert want <= seen, "never ran: {}".format(sorted(want - seen))
