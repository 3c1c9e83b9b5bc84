"""The width-64 Res2Net chain kernel (res2net.cu, xvb_res2net_block_ex with width 64: ECAPA-TDNN C512) on the GPU, bit
for bit against tests/res2net_w64_exact.py at every frame-tile, dilation, scale, pitch and utterance-round edge.

  * Inputs are poisoned: x is a channel slice of a wider buffer whose other channels, pitch padding and spare last
    utterance hold NaN.
  * Outputs are fenced: y is a view inside a buffer filled with a NaN sentinel, with a spare utterance after the last one;
    every column past C and everything else outside the view must be bitwise unchanged.  The output's chunks 1 .. scale-1
    start as that sentinel too, so a step that read its second source before the previous step stored it carries NaN.
  * Refusals return XVB_EINVAL and write nothing."""
import zlib

import numpy as np
import pytest
import torch

import res2net_w64_exact as rx
from gpu_checks import Fenced, equal

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132        # case names do not depend on the SM count; shapes do (built from multi_processor_count)
EINVAL = -1
W = rx.W


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
    return zlib.crc32(("w64 " + name).encode()) & 0x7FFFFFFF


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


def _params(d):
    return (_dev(d["w_hi"]).to(torch.bfloat16), _dev(d["w_lo"]).to(torch.bfloat16), _dev(d["bias"]), _dev(d["scale"]),
            _dev(d["shift"]))


def _run_layers(ops, case, x, params, y):
    """The block as scale - 1 tdnn_affine_ex calls at width 64; chunk 0 is copied."""
    wh, wl, bias, scale, shift = params
    ctx = [-case["d"], 0, case["d"]]
    ops.copy_planes(x.slice(0, W), y.slice(0, W))
    for st in range(case["scale"] - 1):
        r = slice(st * W, (st + 1) * W)
        ops.tdnn_affine_ex(x.slice((st + 1) * W, (st + 2) * W), ops.SplitPlanes(wh[r], wl[r], W), W, ctx,
                           x2=y.slice(st * W, (st + 1) * W) if st else None, bias=bias[r], bn_scale=scale[r],
                           bn_shift=shift[r], relu=True, y=y.slice((st + 1) * W, (st + 2) * W))


@pytest.mark.parametrize("name", sorted(rx.res2net_cases(SMS_FOR_IDS)))
def test_res2net_w64_chain_exact(ops, sms, name):
    case = rx.res2net_cases(sms)[name]
    B, T, Cn = case["B"], case["T"], case["C"]
    d = rx.make_res2net(case, _seed(name))
    want_hi, want_lo = rx.res2net_reference(case, d)
    x = _poisoned(ops, *d["x"], case["x_c0"], case["ldx"])
    params = _params(d)
    yh, yl, y = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], Cn)
    ops.res2net_block(x, *params, case["d"], case["scale"], y, width=W)
    torch.cuda.synchronize()
    what = "{} (B={} T={} d={} scale={})".format(name, B, T, case["d"], case["scale"])
    equal(_bits(yh.numpy()[..., :W]), _bits(d["x"][0][..., :W]), what + " chunk 0 hi")
    equal(_bits(yl.numpy()[..., :W]), _bits(d["x"][1][..., :W]), what + " chunk 0 lo")
    equal(yh.numpy(), want_hi, what + " hi")
    equal(yl.numpy(), want_lo, what + " lo")
    yh.check(what + " hi (sentinel columns past C, pitch padding, spare utterance)")
    yl.check(what + " lo (sentinel columns past C, pitch padding, spare utterance)")
    if case.get("layers"):
        lh, ll, ly = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], Cn)
        _run_layers(ops, case, x, params, ly)
        torch.cuda.synchronize()
        equal(_bits(lh.numpy()), _bits(yh.numpy()), what + " as layer-kernel calls hi")
        equal(_bits(ll.numpy()), _bits(yl.numpy()), what + " as layer-kernel calls lo")


def test_res2net_w64_refusals_write_nothing(ops):
    """Bad arguments to xvb_res2net_block_ex return XVB_EINVAL before anything is launched: the fenced output (and, for
    x_hi == y_hi, the input) keeps its bits.  Widths other than 64 and 128 are refused, and so is a pitch that fits
    scale * 64 at width 64 but not scale * 128."""
    from asv_subtools_b200._lib import lib
    B, T, scale, dil = 2, 10, 4, 1
    Cn = scale * W
    case = dict(B=B, T=T, C=Cn, scale=scale, d=dil)
    d = rx.make_res2net(case, 3)
    x = _poisoned(ops, *d["x"], 8, Cn + 16)
    wh, wl, bias, sc, sh = _params(d)
    yh, yl, y = _fenced_planes(ops, B, T, Cn + 24, 8, Cn)
    xbits = (x.hi.view(torch.int16).clone(), x.lo.view(torch.int16).clone())
    stream = ops._stream()

    def call(xh=None, xl=None, ldx=None, w_hi=None, dil_=dil, scale_=scale, y_hi=None, ldy=None, width=W):
        rc = lib.xvb_res2net_block_ex(xh or x.hi.data_ptr(), xl or x.lo.data_ptr(), ldx or x.ld, w_hi or wh.data_ptr(),
                                      wl.data_ptr(), bias.data_ptr(), sc.data_ptr(), sh.data_ptr(), dil_, scale_,
                                      y_hi or y.hi.data_ptr(), y.lo.data_ptr(), ldy or y.ld, B, T, width, stream)
        torch.cuda.synchronize()
        return rc

    bad = {"width 32": dict(width=32), "width 96": dict(width=96), "width 0": dict(width=0), "width 256": dict(width=256),
           "width 128 with pitches below scale * 128": dict(width=128),
           "scale 1": dict(scale_=1), "scale 17": dict(scale_=17), "dilation 0": dict(dil_=0),
           "ldx not a multiple of 8": dict(ldx=x.ld - 4), "ldx < C": dict(ldx=Cn - 8),
           "ldy not a multiple of 8": dict(ldy=y.ld - 4), "ldy < C": dict(ldy=Cn - 8),
           "misaligned x_hi": dict(xh=x.hi.data_ptr() + 2), "misaligned w_hi": dict(w_hi=wh.data_ptr() + 8),
           "x_hi == y_hi": dict(y_hi=x.hi.data_ptr())}
    assert x.ld < scale * 128 and y.ld < scale * 128
    for what, kw in bad.items():
        assert call(**kw) == EINVAL, what
        yh.check(what + ": y hi")
        yl.check(what + ": y lo")
        assert int((yh.bits != yh.sent).sum()) == 0 and int((yl.bits != yl.sent).sum()) == 0, what + ": y written"
        assert torch.equal(x.hi.view(torch.int16), xbits[0]) and torch.equal(x.lo.view(torch.int16), xbits[1]), what
    # the same arguments without the fault run and match the reference
    assert call() == 0
    want_hi, want_lo = rx.res2net_reference(case, d)
    equal(yh.numpy(), want_hi, "valid call after the refusals hi")
    equal(yl.numpy(), want_lo, "valid call after the refusals lo")
    yh.check("valid call hi")
    yl.check("valid call lo")


def test_res2net_block_is_width_128(ops):
    """xvb_res2net_block and xvb_res2net_block_ex(width = 128) give the same bits on a C1024-shaped block."""
    from asv_subtools_b200._lib import lib
    import ecapa_exact as ex
    case = dict(ex.res2net_cases(SMS_FOR_IDS)["T129"])
    d = ex.make_res2net(case, 21)
    x = _poisoned(ops, *d["x"], case["x_c0"], case["ldx"])
    wh, wl, bias, sc, sh = _params(d)
    outs = []
    for fn in ("xvb_res2net_block", "xvb_res2net_block_ex"):
        hi, lo, y = _fenced_planes(ops, case["B"], case["T"], case["ldy"], case["y_c0"], case["C"])
        args = [x.hi.data_ptr(), x.lo.data_ptr(), x.ld, wh.data_ptr(), wl.data_ptr(), bias.data_ptr(), sc.data_ptr(),
                sh.data_ptr(), case["d"], case["scale"], y.hi.data_ptr(), y.lo.data_ptr(), y.ld, case["B"], case["T"]]
        assert getattr(lib, fn)(*(args + ([128] if fn.endswith("_ex") else []) + [ops._stream()])) == 0
        torch.cuda.synchronize()
        outs.append((_bits(hi.numpy()), _bits(lo.numpy())))
    equal(outs[0][0], outs[1][0], "hi")
    equal(outs[0][1], outs[1][1], "lo")
