"""XVBM0002 model files of the TDNN x-vector with an attention pooling, on the CPU: xvb_extractor_feat_dim reads them,
and xvb_extractor_load refuses a wrong magic, a bad pooling record and a truncated prior before it creates anything
(the GPU half, tests/test_gpu_attn_native.py, round-trips real models and refuses truncated layers)."""
import ctypes as C
import os
import struct
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import attn_native_layout as lay  # noqa: E402
from asv_subtools_b200 import _lib  # noqa: E402

EINVAL = -1


def _xi_file(kind=lay.POOL_XI_POSTDIST, n_att=2):
    r = np.random.default_rng(3)
    a = lambda *s: r.standard_normal(s).astype(np.float32)   # noqa: E731
    frames = [(a(16, 24, 3), a(16), None, None, [-1, 0, 1], True), (a(32, 16, 1), a(32), a(32), a(32), [0], True)]
    attention = [(a(8, 32, 1), a(8), a(8), a(8), [0], True), (a(32, 8, 1), a(32), None, None, [0], False)][2 - n_att:]
    seg_in = 32 if kind == lay.POOL_XI_POSTMEAN else 64
    segments = [(a(12, seg_in, 1), a(12), None, None, [0], False)]
    return lay.xvbm2(24, 1e-10, kind, 32, 1, False, (a(32), a(32)), frames, attention, segments)


def _load(tmp_path, blob):
    path = str(tmp_path / "model.xvbm")
    with open(path, "wb") as f:
        f.write(blob)
    h = C.c_void_p()
    rc = _lib.lib.xvb_extractor_load(C.byref(h), path.encode())
    assert not h.value
    return rc, _lib.last_error()


def test_new_symbols_are_bound():
    for n in ("xvb_extractor_set_attention_pooling", "xvb_extractor_add_attention_layer"):
        assert n in _lib.SIGNATURES and hasattr(_lib.lib, n), n
    assert (_lib.POOL_ATTENTION, _lib.POOL_XI_POSTMEAN, _lib.POOL_XI_POSTDIST) == (1, 2, 3)


def test_feat_dim_reads_xvbm0002(tmp_path):
    path = str(tmp_path / "m.xvbm")
    with open(path, "wb") as f:
        f.write(_xi_file())
    assert _lib.lib.xvb_extractor_feat_dim(path.encode()) == 24
    with open(path, "wb") as f:
        f.write(b"XVBM0003" + _xi_file()[8:])
    assert _lib.lib.xvb_extractor_feat_dim(path.encode()) == EINVAL


def test_layout_sizes():
    data = _xi_file()
    head = 8 + 16 + 20 + 2 * 32 * 4
    assert struct.unpack_from("<5i", data, 24) == (lay.POOL_XI_POSTDIST, 32, 1, 0, 2)
    assert struct.unpack_from("<7i", data, head) == (16, 24, 3, 3, lay.RELU, 1, 0)


def test_load_refuses_before_creating(tmp_path):
    data = _xi_file()

    def patched(offset, value):
        b = bytearray(data)
        b[offset:offset + 4] = struct.pack("<i", value)
        return bytes(b)

    prior = 8 + 16 + 20
    bad_record = "is not an XVBM0001 file or an XVBM0002 file: bad pooling record"
    cases = [(b"XVBM0003" + data[8:], "is not an XVBM0001 file or an XVBM0002 file"),
             (data[:30], bad_record),                              # cut inside the pooling record
             (patched(24, 0), bad_record),                         # statistics pooling is XVBM0001
             (patched(24, 4), bad_record),                         # no such kind (LDE has no native form)
             (patched(28, 0), bad_record),                         # pooled 0
             (patched(40, 0), bad_record),                         # no attention affine
             (patched(40, 3), bad_record),                         # three attention affines
             (data[:prior + 32 * 4 + 5], "truncated in the xi-vector prior"),
             (patched(16, 0), "bad header")]                       # no frame layer
    for blob, msg in cases:
        rc, err = _load(tmp_path, blob)
        assert rc == EINVAL and msg in err, (msg, rc, err)
