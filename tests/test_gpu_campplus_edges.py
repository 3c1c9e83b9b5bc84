"""CAM++'s fp32 CUDA-core kernels (campplus.cu) on the GPU against tests/campplus_exact.py: the context-aware mask at every
segment edge (T % seg_len at 0 and +-1, seg_len 1 and > T), frame-lane count and shared-memory size, and the BN -> ReLU
planes at channel slices, C = 8 and past its grid cap.

  * Inputs are poisoned: h and x are channel slices of wider buffers whose other channels, pitch padding and spare last
    utterance hold NaN.
  * Outputs are fenced: the (B, nseg, G) mask has a spare utterance of sentinel after it, and the planes are slices of
    sentinel-filled buffers; everything outside the logical output must be bitwise unchanged.
  * Refusals return XVB_EINVAL and write nothing."""
import zlib

import numpy as np
import pytest
import torch

import campplus_exact as ce
import gemm_exact as gx
from gpu_checks import Fenced, equal, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132
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


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _poisoned(ops, hi, lo, c0, ld):
    """(B, T, C) planes as the channel slice [c0, c0 + C) of (B + 1, T, ld) buffers that hold NaN everywhere else."""
    B, Cn = hi.shape[0], hi.shape[-1]
    bufs = []
    for a in (hi, lo):
        buf = torch.full((B + 1,) + a.shape[1:-1] + (ld,), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B, ..., c0:c0 + Cn] = _dev(a).to(torch.bfloat16)
        bufs.append(buf)
    return ops.SplitPlanes(bufs[0][:B, ..., c0:c0 + Cn], bufs[1][:B, ..., c0:c0 + Cn], Cn)


@pytest.mark.parametrize("name", sorted(ce.cam_cases()))
def test_cam_gate(ops, name):
    case = ce.cam_cases()[name]
    B, nseg, G = case["B"], case["nseg"], case["G"]
    d = ce.make_cam(case, _seed(name))
    want, bound = ce.cam_reference(case, d)
    h = _poisoned(ops, d["h_hi"], d["h_lo"], case["h_c0"], case["ldh"])
    out = Fenced((B + 1, nseg, G), torch.float32, (slice(0, B),))
    got = ops.cam_gate(h, _dev(d["w1"]), _dev(d["b1"]), _dev(d["w2"]), _dev(d["b2"]), seg_len=case["seg_len"], out=out.view)
    assert got.data_ptr() == out.view.data_ptr()
    torch.cuda.synchronize()
    what = "{} (T={} seg_len={} C={} smem={})".format(name, case["T"], case["seg_len"], case["C"], case["smem"])
    within(out.numpy(), want, bound, what)
    out.check(what)


@pytest.mark.parametrize("name", sorted(ce.bn_relu_cases(SMS_FOR_IDS)))
def test_bn_relu_planes_exact(ops, sms, name):
    case = ce.bn_relu_cases(sms)[name]
    B, T, C = case["B"], case["T"], case["C"]
    d = ce.make_bn_relu(case, _seed(name))
    want = ce.bn_relu_reference(d)
    x = _poisoned(ops, d["hi"], d["lo"], case["x_c0"], case["ldx"])
    idx = (slice(0, B), slice(None), slice(case["y_c0"], case["y_c0"] + C))
    yh, yl = Fenced((B + 1, T, case["ldy"]), torch.bfloat16, idx), Fenced((B + 1, T, case["ldy"]), torch.bfloat16, idx)
    ops.bn_relu_planes(x, _dev(d["scale"]), _dev(d["shift"]), ops.SplitPlanes(yh.view, yl.view, C))
    torch.cuda.synchronize()
    wh, wl = gx.split_bf16(want)
    equal(_bits(yh.numpy()), _bits(wh), name + " hi")
    equal(_bits(yl.numpy()), _bits(wl), name + " lo")
    yh.check(name + " hi")
    yl.check(name + " lo")


def test_cam_gate_refusals_write_nothing(ops):
    """More shared memory than one CTA has, more than 256 channel groups, no channels, or a bad pitch: XVB_EINVAL, and
    the mask keeps its sentinel."""
    from asv_subtools_b200._lib import lib
    st = ops._stream()
    hh = torch.zeros(2, 8, 2064, dtype=torch.bfloat16, device="cuda")
    w = torch.zeros(64 * 2064, device="cuda")
    out = Fenced((3, 8, 16), torch.float32, (slice(0, 2),))

    def call(T=8, C=64, seg=1, ldh=2064, R=16):
        rc = lib.xvb_cam_gate(hh.data_ptr(), hh.data_ptr(), ldh, 2, T, C, seg, w.data_ptr(), w.data_ptr(), R, w.data_ptr(),
                              w.data_ptr(), 16, out.view.data_ptr(), st)
        torch.cuda.synchronize()
        return rc

    assert ce.cam_gate_smem(3000, 2048, 1, 16) > ce.MAX_SMEM
    bad = {"smem > 227 KB": dict(T=3000, C=2048), "C / 8 > 256": dict(C=2056, ldh=2064), "C = 0": dict(C=0),
           "C not a multiple of 8": dict(C=60), "ldh < C": dict(C=64, ldh=56), "ldh not a multiple of 8": dict(ldh=2060),
           "seg_len 0": dict(seg=0)}
    for what, kw in bad.items():
        assert call(**kw) == EINVAL, what
        out.check(what)
        assert int((out.bits != out.sent).sum()) == 0, what + ": mask written"
