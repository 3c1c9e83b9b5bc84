"""The feature front end on the GPU against tests/frontend_exact.py: energy VAD, CMN and voiced-frame selection
(frontend.cu) bit for bit, and fbank / MFCC (fbank.cu) at every FFT size within the bound derived there.  Inputs carry
NaN in the feature columns VAD must not read; every output is a view inside a sentinel-filled buffer whose other
elements must stay unchanged."""
import ctypes as C

import numpy as np
import pytest
import torch

import frontend_exact as fx
from gpu_checks import Fenced, equal, within

pytestmark = pytest.mark.gpu

LEAD = 4
BYTE_SENT = 0xA5


@pytest.fixture(scope="module")
def lib():
    from asv_subtools_b200 import _lib
    assert torch.cuda.is_available()
    return _lib.lib


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _pack(utts, F):
    lens = [u.shape[0] for u in utts]
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    x = np.concatenate(utts, axis=0) if sum(lens) else np.zeros((0, F), np.float32)
    return _dev(x.reshape(-1, F)) if sum(lens) else torch.zeros(1, F, device="cuda"), off, _dev(off)


def _out(n, dtype=torch.float32):
    return Fenced((n + LEAD + 7,), dtype, slice(LEAD, LEAD + n))


class _ByteFence:
    def __init__(self, n):
        self.buf = torch.full((n + LEAD + 7,), BYTE_SENT, dtype=torch.uint8, device="cuda")
        self.view = self.buf[LEAD:LEAD + n]
        self.n = n

    def check(self, what):
        b = self.buf.cpu().numpy()
        assert (b[:LEAD] == BYTE_SENT).all() and (b[LEAD + self.n:] == BYTE_SENT).all(), what + ": written outside"


@pytest.mark.parametrize("name", sorted(fx.vad_cases()))
def test_vad_energy_exact(lib, name):
    case = fx.vad_cases()[name]
    lens, utts = fx.vad_operands(case, name)
    x, off, doff = _pack(utts, 3)
    U = len(utts)
    voiced, counts = _ByteFence(int(off[-1])), _out(U, torch.int32)
    assert lib.xvb_vad_energy(x.data_ptr(), doff.data_ptr(), U, 3, fx.VAD_THRESHOLD, case["scale"], case["context"],
                              case["prop"], voiced.view.data_ptr(), counts.view.data_ptr(), None) == 0
    torch.cuda.synchronize()
    got = voiced.view.cpu().numpy()
    want = [fx.vad_ref(u[:, 0], fx.VAD_THRESHOLD, case["scale"], case["context"], case["prop"]) for u in utts]
    equal(got, np.concatenate(want), "vad decisions " + name)
    equal(counts.view.cpu().numpy(), np.array([w.sum() for w in want], np.int32), "vad counts " + name)
    voiced.check("vad " + name)
    counts.check("vad counts " + name)


@pytest.mark.parametrize("name", sorted(fx.cmn_cases()))
def test_cmn_exact(lib, name):
    case = fx.cmn_cases()[name]
    F, w = case["F"], case["window"]
    utts = fx.cmn_operands(case, name)
    x, off, doff = _pack(utts, F)
    y = _out(int(off[-1]) * F)
    assert lib.xvb_cmn(x.data_ptr(), doff.data_ptr(), len(utts), F, w, y.view.data_ptr(), None) == 0
    torch.cuda.synchronize()
    want = np.concatenate([fx.cmn_ref(u, w) for u in utts], axis=0)
    equal(_bits(y.numpy()), _bits(want).reshape(-1), "cmn " + name)
    y.check("cmn " + name)


@pytest.mark.parametrize("name", sorted(fx.select_cases()))
def test_select_frames_exact(lib, name):
    case = fx.select_cases()[name]
    F = case["F"]
    utts, masks = fx.select_operands(case, name)
    x, off, doff = _pack(utts, F)
    counts = np.array([m.sum() for m in masks])
    out_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    v = _dev(np.concatenate(masks)) if off[-1] else torch.zeros(1, dtype=torch.uint8, device="cuda")
    y = _out(int(out_off[-1]) * F)
    dst = y.buf.data_ptr() + LEAD * 4                  # an empty view's data_ptr() is NULL; the call takes any valid pointer
    assert lib.xvb_select_frames(x.data_ptr(), doff.data_ptr(), v.data_ptr(), _dev(out_off).data_ptr(), len(utts), F,
                                 dst, None) == 0
    torch.cuda.synchronize()
    want = np.concatenate([u[m.astype(bool)] for u, m in zip(utts, masks)], axis=0)
    equal(_bits(y.numpy()), _bits(want).reshape(-1), "select " + name)
    y.check("select " + name)


def _fbank_handle(lib, case):
    from asv_subtools_b200._lib import FbankOpts
    o = FbankOpts()
    lib.xvb_fbank_default_opts(C.byref(o))
    c = case["opts"]
    o.sample_frequency, o.frame_length_ms, o.frame_shift_ms = 16000.0, case["size"] / 16.0, case["shift"] / 16.0
    o.preemphasis_coefficient, o.energy_floor, o.cepstral_lifter = c["preemphasis_coefficient"], c["energy_floor"], c["cepstral_lifter"]
    o.num_mel_bins, o.num_ceps, o.window_type = c["num_mel_bins"], c["num_ceps"], fx.WINDOWS.index(c["window_type"])
    o.use_energy, o.raw_energy, o.remove_dc_offset = int(c["use_energy"]), int(c["raw_energy"]), int(c["remove_dc_offset"])
    o.use_log_fbank, o.use_power, o.htk_compat = int(c["use_log_fbank"]), int(c["use_power"]), int(c["htk_compat"])
    h = C.c_void_p()
    assert lib.xvb_fbank_create(C.byref(h), C.byref(o)) == 0
    return h


@pytest.mark.parametrize("name", sorted(fx.fbank_cases()))
def test_fbank_within_bound(lib, name):
    case = fx.fbank_cases()[name]
    waves = fx.fbank_waves(case, name)
    h = _fbank_handle(lib, case)
    try:
        dim = lib.xvb_fbank_dim(h)
        frames = [int(lib.xvb_fbank_num_frames(h, w.shape[0])) for w in waves]
        soff = np.concatenate([[0], np.cumsum([w.shape[0] for w in waves])]).astype(np.int64)
        foff = np.concatenate([[0], np.cumsum(frames)]).astype(np.int32)
        total = int(foff[-1])
        wave = _dev(np.concatenate(waves).astype(np.float32))
        out = _out(total * dim)
        assert lib.xvb_fbank_compute(h, wave.data_ptr(), _dev(soff).data_ptr(), _dev(foff).data_ptr(), len(waves), total,
                                     out.view.data_ptr(), None) == 0
        torch.cuda.synchronize()
    finally:
        lib.xvb_fbank_destroy(h)
    got = out.numpy().reshape(total, dim)
    for i, w in enumerate(waves):
        ref = fx.fbank_ref(case, w)
        assert ref.shape == (frames[i], dim), (name, i)
        if frames[i]:
            within(got[foff[i]:foff[i + 1]], ref, fx.fbank_bound(case, w), "fbank {} utterance {}".format(name, i))
    out.check("fbank " + name)
