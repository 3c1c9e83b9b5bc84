"""The ECAPA-TDNN block kernels on the GPU, bit for bit against tests/ecapa_exact.py: the one-kernel Res2Net chain
(res2net.cu) at every frame-tile, dilation, scale, pitch and utterance-round edge, the SE gate and segment gate
(ecapa.cu: xvb_se_apply, xvb_seg_gate_apply) and the segment-level fp32 affine (ecapa.cu: xvb_small_affine).

  * Inputs are poisoned: x, z and in are channel slices of wider buffers whose other channels, pitch padding and spare
    last utterance (row) hold NaN.
  * Outputs are fenced: every output is a view inside a buffer filled with a NaN sentinel, with a spare utterance (row)
    after the last one; everything outside the logical output must be bitwise unchanged.  The Res2Net output's own
    chunks 1 .. scale-1 start as that sentinel too, so a step that read its second source before the previous step stored
    it would carry NaN into the result.
  * Refusals return XVB_EINVAL and write nothing."""
import zlib

import numpy as np
import pytest
import torch

import ecapa_exact as ex
import gemm_exact as gx
from gpu_checks import Fenced, equal, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132        # case names do not depend on the SM count; shapes do (built from multi_processor_count)
EINVAL = -1


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


def _poisoned(ops, hi, lo, c0, ld):
    """(B, T, C) planes as the channel slice [c0, c0 + C) of (B + 1, T, ld) buffers that hold NaN everywhere else."""
    B, Cn = hi.shape[0], hi.shape[-1]
    bufs = []
    for a in (hi, lo):
        buf = torch.full((B + 1,) + a.shape[1:-1] + (ld,), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B, ..., c0:c0 + Cn] = _dev(a).to(torch.bfloat16)
        bufs.append(buf)
    return ops.SplitPlanes(bufs[0][:B, ..., c0:c0 + Cn], bufs[1][:B, ..., c0:c0 + Cn], Cn)


def _fenced_planes(ops, B, T, ld, c0, Cn):
    idx = (slice(0, B), slice(None), slice(c0, c0 + Cn))
    hi, lo = Fenced((B + 1, T, ld), torch.bfloat16, idx), Fenced((B + 1, T, ld), torch.bfloat16, idx)
    return hi, lo, ops.SplitPlanes(hi.view, lo.view, Cn)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _check_planes(hi, lo, want_hi, want_lo, what):
    """Plane outputs bit for bit (the sign of zero included), and the fences around them."""
    equal(_bits(hi.numpy()), _bits(want_hi), what + " hi")
    equal(_bits(lo.numpy()), _bits(want_lo), what + " lo")
    hi.check(what + " hi")
    lo.check(what + " lo")


def _check_values(hi, lo, want_hi, want_lo, what):
    """As _check_planes, with +0 and -0 equal (the GEMM kernels' exact zeros carry no sign the reference fixes)."""
    equal(hi.numpy(), want_hi, what + " hi")
    equal(lo.numpy(), want_lo, what + " lo")
    hi.check(what + " hi")
    lo.check(what + " lo")


# ------------------------------------------------------------------------------------------------ Res2Net chain
def _res2net_params(d):
    return (_dev(d["w_hi"]).to(torch.bfloat16), _dev(d["w_lo"]).to(torch.bfloat16), _dev(d["bias"]), _dev(d["scale"]),
            _dev(d["shift"]))


def _run_layers(ops, case, x, params, y):
    """The block as scale - 1 tdnn_affine_ex calls: step st reads x chunk st + 1 and, from step 1 on, the output chunk
    st as its second source (x2), and writes output chunk st + 1; chunk 0 is copied."""
    wh, wl, bias, scale, shift = params
    ctx = [-case["d"], 0, case["d"]]
    ops.copy_planes(x.slice(0, 128), y.slice(0, 128))
    for st in range(case["scale"] - 1):
        r = slice(st * 128, (st + 1) * 128)
        ops.tdnn_affine_ex(x.slice((st + 1) * 128, (st + 2) * 128), ops.SplitPlanes(wh[r], wl[r], 128), 128, ctx,
                           x2=y.slice(st * 128, (st + 1) * 128) if st else None, bias=bias[r], bn_scale=scale[r],
                           bn_shift=shift[r], relu=True, y=y.slice((st + 1) * 128, (st + 2) * 128))


@pytest.mark.parametrize("name", sorted(ex.res2net_cases(SMS_FOR_IDS)))
def test_res2net_chain_exact(ops, sms, name):
    case = ex.res2net_cases(sms)[name]
    B, T, Cn = case["B"], case["T"], case["C"]
    d = ex.make_res2net(case, _seed(name))
    want_hi, want_lo = ex.res2net_reference(case, d)
    x = _poisoned(ops, *d["x"], case["x_c0"], case["ldx"])
    params = _res2net_params(d)
    yh, yl, y = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], Cn)
    ops.res2net_block(x, *params, case["d"], case["scale"], y)
    torch.cuda.synchronize()
    what = "{} (B={} T={} d={} scale={})".format(name, B, T, case["d"], case["scale"])
    # chunk 0 passes through bit for bit; chunks 1 .. scale-1 are the split planes of the exact steps
    equal(_bits(yh.numpy()[..., :128]), _bits(d["x"][0][..., :128]), what + " chunk 0 hi")
    equal(_bits(yl.numpy()[..., :128]), _bits(d["x"][1][..., :128]), what + " chunk 0 lo")
    _check_values(yh, yl, want_hi, want_lo, what)
    if case.get("layers"):
        lh, ll, ly = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], Cn)
        _run_layers(ops, case, x, params, ly)
        torch.cuda.synchronize()
        _check_planes(lh, ll, yh.numpy(), yl.numpy(), what + " as layer-kernel calls")


def test_res2net_refusals_write_nothing(ops):
    """Bad arguments return XVB_EINVAL before anything is launched: the fenced output (and, for x_hi == y_hi, the
    input) keeps its bits."""
    from asv_subtools_b200._lib import lib
    B, T, scale, dil = 2, 10, 4, 1
    Cn = scale * 128
    case = dict(B=B, T=T, C=Cn, scale=scale, d=dil)
    d = ex.make_res2net(case, 3)
    x = _poisoned(ops, *d["x"], 8, Cn + 16)
    wh, wl, bias, sc, sh = _res2net_params(d)
    yh, yl, y = _fenced_planes(ops, B, T, Cn + 24, 8, Cn)
    xbits = (x.hi.view(torch.int16).clone(), x.lo.view(torch.int16).clone())
    stream = ops._stream()

    def call(xh=None, xl=None, ldx=None, w_hi=None, dil_=dil, scale_=scale, y_hi=None, ldy=None):
        rc = lib.xvb_res2net_block(xh or x.hi.data_ptr(), xl or x.lo.data_ptr(), ldx or x.ld, w_hi or wh.data_ptr(),
                                   wl.data_ptr(), bias.data_ptr(), sc.data_ptr(), sh.data_ptr(), dil_, scale_,
                                   y_hi or y.hi.data_ptr(), y.lo.data_ptr(), ldy or y.ld, B, T, stream)
        torch.cuda.synchronize()
        return rc

    bad = {"scale 1": dict(scale_=1), "scale 17": dict(scale_=17), "dilation 0": dict(dil_=0),
           "ldx not a multiple of 8": dict(ldx=x.ld - 4), "ldx < C": dict(ldx=Cn - 8),
           "ldy not a multiple of 8": dict(ldy=y.ld - 4), "ldy < C": dict(ldy=Cn - 8),
           "misaligned x_hi": dict(xh=x.hi.data_ptr() + 2), "misaligned w_hi": dict(w_hi=wh.data_ptr() + 8),
           "x_hi == y_hi": dict(y_hi=x.hi.data_ptr())}
    for what, kw in bad.items():
        assert call(**kw) == EINVAL, what
        yh.check(what + ": y hi")
        yl.check(what + ": y lo")
        assert int((yh.bits != yh.sent).sum()) == 0 and int((yl.bits != yl.sent).sum()) == 0, what + ": y written"
        assert torch.equal(x.hi.view(torch.int16), xbits[0]) and torch.equal(x.lo.view(torch.int16), xbits[1]), what
    # the same arguments without the fault run and match the reference
    assert call() == 0
    want_hi, want_lo = ex.res2net_reference(case, d)
    _check_values(yh, yl, want_hi, want_lo, "valid call after the refusals")


# ------------------------------------------------------------------------------------------------ SE gate kernels
def _check_se(hi, lo, want, z, xin, g, rows, what):
    """Planes against split_bf16 of the two-rounding reference.  On a mismatch, also says how many of the differing
    elements are instead the planes of a single-rounding (fused) z * g + in, and how many fp32 ulps that value is from
    the two-rounding one there."""
    wh, wl = gx.split_bf16(want)
    gh, gl = hi.numpy(), lo.numpy()
    bad = (_bits(gh) != _bits(wh)) | (_bits(gl) != _bits(wl))
    if bad.any():
        zf = (z[0] + z[1]).astype(np.float64)
        x = 0.0 if xin is None else (xin[0] + xin[1]).astype(np.float64)
        fused = (zf * g[rows] + x).astype(np.float32)
        fh, fl = gx.split_bf16(fused)
        is_fused = bad & (_bits(gh) == _bits(fh)) & (_bits(gl) == _bits(fl))
        ulps = np.abs(fused.astype(np.float64) - want) / np.spacing(np.abs(want)).astype(np.float64)
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("{}: {} of {} elements differ; {} of them are the planes of a fused z * g + in, up to {:.0f} "
                             "fp32 ulps from the two-rounding value; first at {}: got {!r} + {!r}, want {!r} + {!r}"
                             .format(what, int(bad.sum()), bad.size, int(is_fused.sum()),
                                     float(ulps[is_fused].max()) if is_fused.any() else 0.0, i, gh[i], gl[i], wh[i], wl[i]))
    hi.check(what + " hi")
    lo.check(what + " lo")


@pytest.mark.parametrize("name", sorted(ex.se_cases()))
def test_se_apply_exact(ops, name):
    case = ex.se_cases()[name]
    B, T, Cn = case["B"], case["T"], case["C"]
    z, xin, g = ex.se_operands(np.random.RandomState(_seed(name)), B, T, Cn, B)
    rows = ex.gate_rows(B, T, T)
    want_out, want_next = ex.se_reference(z, xin, g, rows)
    zp = _poisoned(ops, *z, 8, case["ldz"])
    oh, ol, out = _fenced_planes(ops, B, T, case["ldout"], 8, Cn)
    if case.get("inplace"):
        # ECAPA's running sum: next is written over in, a fenced view whose contents are the input
        nh, nl, nxt = _fenced_planes(ops, B, T, case["ldin"], 16, Cn)
        nxt.hi.copy_(_dev(xin[0]).to(torch.bfloat16))
        nxt.lo.copy_(_dev(xin[1]).to(torch.bfloat16))
        ip = nxt
    else:
        ip = _poisoned(ops, *xin, 16, case["ldin"])
        nh, nl, nxt = _fenced_planes(ops, B, T, case["ldnext"], 0, Cn)
    ops.se_apply(zp, ip, _dev(g), out, nxt)
    torch.cuda.synchronize()
    _check_se(oh, ol, want_out, z, xin, g, rows, name + " out")
    wh, wl = gx.split_bf16(want_next)
    _check_planes(nh, nl, wh, wl, name + " next")


@pytest.mark.parametrize("name", sorted(ex.seg_gate_cases()))
def test_seg_gate_apply_exact(ops, name):
    case = ex.seg_gate_cases()[name]
    B, T, Cn, seg = case["B"], case["T"], case["C"], case["seg_len"]
    z, xin, g = ex.se_operands(np.random.RandomState(_seed(name)), B, T, Cn, B * case["nseg"])
    if not case["with_in"]:
        xin = None
    rows = ex.gate_rows(B, T, seg)
    want, _ = ex.se_reference(z, xin, g, rows)
    zp = _poisoned(ops, *z, 8, case["ldz"])
    ip = _poisoned(ops, *xin, 16, case["ldin"]) if xin is not None else None
    oh, ol, out = _fenced_planes(ops, B, T, case["ldout"], 8, Cn)
    ops.seg_gate_apply(zp, _dev(g), seg, out, ip)
    torch.cuda.synchronize()
    _check_se(oh, ol, want, z, xin, g, rows, name)


# ------------------------------------------------------------------------------------------------ small affine
@pytest.mark.parametrize("name", sorted(ex.small_affine_cases()))
def test_small_affine_exact(ops, name):
    from asv_subtools_b200._lib import BN, RELU, SIGMOID, TANH, lib
    case = ex.small_affine_cases()[name]
    B, N, K = case["B"], case["N"], case["K"]
    d = ex.make_small_affine(case, _seed(name))
    acc = ex.small_affine_acc(d)
    xbuf = torch.full((B + 1, case["ldx"]), float("nan"), dtype=torch.float32, device="cuda")
    xbuf[:B, case["x_c0"]:case["x_c0"] + K] = _dev(d["x"])
    x = xbuf[:B, case["x_c0"]:]
    w, bias, scale, shift = _dev(d["w"]), _dev(d["bias"]), _dev(d["scale"]), _dev(d["shift"])
    for ep, relu, bn, act in ex.SA_EPILOGUES:
        what = "{} {}".format(name, ep)
        want, bound = ex.small_affine_reference(case, d, relu, bn, act, acc)
        y = Fenced((B + 1, case["ldy"]), torch.float32, (slice(0, B), slice(case["y_c0"], case["y_c0"] + N)))
        pidx = (slice(0, B), slice(case["p_c0"], case["p_c0"] + N))
        ph, pl = Fenced((B + 1, case["ldp"]), torch.bfloat16, pidx), Fenced((B + 1, case["ldp"]), torch.bfloat16, pidx)
        flags = (RELU if relu else 0) | (BN if bn else 0) | {None: 0, "sigmoid": SIGMOID, "tanh": TANH}[act]
        rc = lib.xvb_small_affine(x.data_ptr(), case["ldx"], w.data_ptr(), B, K, N, bias.data_ptr(),
                                  scale.data_ptr() if bn else None, shift.data_ptr() if bn else None, flags,
                                  y.view.data_ptr(), case["ldy"], ph.view.data_ptr(), pl.view.data_ptr(), case["ldp"],
                                  ops._stream())
        assert rc == 0, what
        torch.cuda.synchronize()
        got = y.numpy()
        if bound is None:
            equal(got, want, what + " y")
        else:
            within(got, want, bound, what + " y")
        y.check(what + " y")
        sh, sl = gx.split_bf16(got)
        _check_planes(ph, pl, sh, sl, what + " planes")
