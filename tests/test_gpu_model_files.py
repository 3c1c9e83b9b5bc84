"""The named-record model files of the native ResNet (XVBR0001), Conformer (XVBC0001) and CAM++ (XVBP0001) extractors on
the H100, over every case of the three families' fixtures: save() writes exactly the bytes of a writer of the documented
layout fed the records the handle was built from; load() then save() reproduces the file byte for byte; and corrupt files
are refused with an error naming the magic or the damage, without a crash.  The ECAPA-TDNN files (XVBE0001, XVBE0002
with MQMHA pooling) and the TDNN files (XVBM0001) are checked the same way against writers of their own layouts."""
import struct

import numpy as np
import pytest

import campplus_oracle as po
import conformer_2sub_oracle as c2
import conformer_oracle as co
import ecapa_mqmha_oracle as mo
import resnet_oracle as ro
from asv_subtools_b200 import _lib, ops
from asv_subtools_b200._lib import CamPPConfig, ConformerConfig
from asv_subtools_b200.model.campplus_xvector import CamPPXvector, NativeCamPPExtractor, native_config as campp_config
from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN, NativeEcapaExtractor
from asv_subtools_b200.model.resnet_xvector import NativeResNetExtractor, ResNetXvector
from asv_subtools_b200.model.transformer_xvector import (NativeConformerExtractor, TransformerXvector,
                                                         native_config as conformer_config)
from asv_subtools_b200.nnet.pooling import MQMHASP
from oracle import nnet as onn

pytestmark = pytest.mark.gpu

CONFORMER_CASES = dict(co.CASES, **c2.CASES)
# family -> (magic, shape ints per record, record limit)
FORMATS = {"resnet": (b"XVBR0001", 3, 4096), "conformer": (b"XVBC0001", 2, 65536), "campp": (b"XVBP0001", 2, 65536)}
CASES = ([("resnet", c) for c in sorted(ro.CASES)] + [("conformer", c) for c in sorted(CONFORMER_CASES)] +
         [("campp", c) for c in sorted(po.CASES)])


def _build(family, case, golden):
    """(model, native handle, configuration block) of one fixture case."""
    if family == "resnet":
        kwargs, fdim, _, positions, seed, _ = ro.CASES[case]
        m = ResNetXvector(fdim, 10, training=False, extracted_embedding=positions[0], **kwargs)
        m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed), strict=True)
        m = m.cuda().eval()
        r = m.resnet
        stages = [getattr(r, "layer{}".format(li)) for li in range(1, 5)]
        ints = [m.inputs_dim] + [len(s) for s in stages] + [s[0].conv1.out_channels for s in stages]
        cfg = np.array(ints + [1 if r.full_pre_activation else 0], "<i4").tobytes() + np.float32(m.stats.eps).tobytes()
        return m, NativeResNetExtractor(m), cfg
    if family == "conformer":
        kwargs, fdim, _, positions, seed = CONFORMER_CASES[case][:5]
        npz = "conformer" if case in co.CASES else "conformer_2sub"
        m = TransformerXvector(fdim, 10, training=False, extracted_embedding=positions[0], **kwargs)
        m.load_state_dict(co.seeded_state_dict(golden(npz)["keys_" + case], seed), strict=True)
        m = m.cuda().eval()
        return m, NativeConformerExtractor(m), bytes(ConformerConfig(**conformer_config(m)))
    kw = dict(po.CASES[case][0])
    m = CamPPXvector(kw.pop("inputs_dim"), 10, **kw)
    m.load_state_dict(po.seeded_state_dict(golden("campplus")["keys_" + case], po.CASES[case][3]), strict=True)
    m = m.cuda().eval()
    return m, NativeCamPPExtractor(m), bytes(CamPPConfig(**campp_config(m)))


def _write(magic, cfg, layers):
    """The layout: magic | configuration block | i32 nrec, then per record i32 name_len | name | i32 shape[n] | i32 flags
    | i32 has_w, has_b, has_s | f32 w? | f32 b? | f32 s, t?"""
    out = bytearray(magic + cfg + struct.pack("<i", len(layers)))
    for name, shape, arrays, flags in layers:
        w, b, s, t = [None if a is None else np.ascontiguousarray(a, dtype="<f4") for a in arrays]
        out += struct.pack("<i", len(name)) + name.encode()
        out += np.array(list(shape) + [flags, w is not None, b is not None, s is not None], "<i4").tobytes()
        for a in (w, b, s, t):
            if a is not None:
                out += a.tobytes()
    return bytes(out)


def _records(data, cfg_len, nshape):
    """(start, payload start, end, has_w offset) of each record of a model file."""
    pos = 8 + cfg_len
    (nrec,) = struct.unpack_from("<i", data, pos)
    pos += 4
    out = []
    for _ in range(nrec):
        start = pos
        (nl,) = struct.unpack_from("<i", data, pos)
        hd = np.frombuffer(data, "<i4", nshape + 4, pos + 4 + nl)
        payload = pos + 4 + nl + 4 * (nshape + 4)
        rows = int(hd[0])
        welems = rows * int(hd[1]) * (int(hd[2]) ** 2 if nshape == 3 else 1)
        end = payload + 4 * (welems * int(hd[nshape + 1]) + rows * int(hd[nshape + 2]) + 2 * rows * int(hd[nshape + 3]))
        out.append((start, payload, end, pos + 4 + nl + 4 * (nshape + 1)))
        pos = end
    assert pos == len(data)
    return out


@pytest.mark.parametrize("family, case", CASES)
def test_model_file_bytes_roundtrip_and_rejects(tmp_path, golden, family, case):
    magic, nshape, limit = FORMATS[family]
    m, ex, cfg = _build(family, case, golden)
    cls = type(ex)
    path, again, bad = str(tmp_path / "model.xvbm"), str(tmp_path / "again.xvbm"), str(tmp_path / "bad.xvbm")
    ex.save(path)
    data = open(path, "rb").read()
    assert data == _write(magic, cfg, list(ex._layers(m)))
    loaded = cls.load(path)
    loaded.save(again)
    loaded.close()
    assert open(again, "rb").read() == data

    recs = _records(data, len(cfg), nshape)
    first_w = next(r for r in recs if r[2] - r[1] > 8)
    nrec_at = 8 + len(cfg)

    def patched(offset, value):
        b = bytearray(data)
        b[offset:offset + 4] = struct.pack("<i", value)
        return bytes(b)

    has_w = struct.unpack_from("<i", data, recs[0][3])[0]
    blobs = [(data[:recs[1][0]], "truncated|corrupt"),                    # cut at a record boundary
             (data[:first_w[1] + 6], "truncated|corrupt"),                # cut inside a weight
             (patched(nrec_at, 0), magic.decode()),
             (patched(nrec_at, limit + 1), magic.decode()),
             (patched(recs[0][0], 0), "truncated|corrupt"),               # name length 0
             (patched(recs[0][0], 127), "truncated|corrupt"),             # name length 127
             (patched(recs[0][3], 1 - has_w), "truncated|corrupt")]       # has_w contradicts the shape
    for blob, msg in blobs:
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=msg):
            cls.load(bad)
    ex.close()


def _ecapa_write(ex, m):
    """xvb_ecapa_save's layout: magic | i32 feat_dim, channels, mfa_dim, att_hidden, embed_dim, nlayers | (XVBE0002) i32
    num_head, num_q, hidden, share, affine_layers, time_attention, stddev | per layer i32 name_len | name | i32 Cout, Cin,
    ntaps, tot, flags, has_b, has_s | i32 ctx[ntaps] | f32 w (Cout, Cin, tot) | f32 b? | f32 s, t?"""
    layers = list(ex._layers(m))
    st = m.stats
    mq = isinstance(st, MQMHASP)
    out = bytearray((b"XVBE0002" if mq else b"XVBE0001") + struct.pack("<6i", *ex._create_args(m), len(layers)))
    if mq:
        out += struct.pack("<7i", st.num_head, st.num_q, st.hidden_size, int(st.share), st.affine_layers,
                           int(st.time_attention), int(st.stddev))
    for name, (cout, cin, ctx, ntaps), (w, b, s, t), flags in layers:
        out += struct.pack("<i", len(name)) + name.encode()
        out += struct.pack("<7i", cout, cin, ntaps, w.shape[2], flags, b is not None, s is not None)
        out += struct.pack("<%di" % ntaps, *ctx[:ntaps])
        for a in (w, b, s, t):
            if a is not None:
                out += np.ascontiguousarray(a, dtype="<f4").tobytes()
    return bytes(out)


@pytest.mark.parametrize("magic", ["XVBE0001", "XVBE0002"])
def test_ecapa_model_file_bytes_and_roundtrip(tmp_path, magic):
    if magic == "XVBE0001":
        m = ECAPA_TDNN(80, 10, training=False)
        m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), 201), strict=True)
    else:
        kwargs, _, _, seed, _ = mo.CASES["fc1"]
        m = ECAPA_TDNN(80, 10, training=False, extracted_embedding="near", **kwargs)
        m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed), strict=True)
    m = m.cuda().eval()
    ex = NativeEcapaExtractor(m)
    path, again = str(tmp_path / "model.xvbm"), str(tmp_path / "again.xvbm")
    ex.save(path)
    data = open(path, "rb").read()
    assert data[:8] == magic.encode() and data == _ecapa_write(ex, m)
    loaded = NativeEcapaExtractor.load(path)
    loaded.save(again)
    loaded.close()
    assert open(again, "rb").read() == data
    ex.close()


class _Recorded(ops.Extractor):
    """ops.Extractor keeping what it is handed, for the writer below."""

    def __init__(self, feat_dim):
        super().__init__(feat_dim)
        self.handed = {"frame": [], "segment": []}

    def add_frame_layer(self, weight, bias, context, bn_scale=None, bn_shift=None, relu=True):
        super().add_frame_layer(weight, bias, context, bn_scale, bn_shift, relu)
        self.handed["frame"].append(([int(c) for c in context], weight, bias, bn_scale, bn_shift, relu))

    def add_segment_layer(self, weight, bias, bn_scale=None, bn_shift=None, relu=False):
        super().add_segment_layer(weight, bias, bn_scale, bn_shift, relu)
        self.handed["segment"].append(([0], weight, bias, bn_scale, bn_shift, relu))

    def finalize(self, pooling_eps=1e-10):
        super().finalize(pooling_eps)
        self.eps = pooling_eps


def _xvbm_write(ex):
    """The XVBM0001 layout: magic | i32 feat_dim | f32 pooling_eps | i32 n_frame, n_segment, then per layer, frame layers
    first: i32 Cout, Cin, ntaps, tot_context, flags, has_bias, has_bn | i32 ctx[ntaps] | f32 w (Cout, Cin, tot_context)
    | f32 bias? | f32 scale, shift?"""
    frames, segs = ex.handed["frame"], ex.handed["segment"]
    out = bytearray(b"XVBM0001" + struct.pack("<ifii", ex.feat_dim, ex.eps, len(frames), len(segs)))
    for ctx, w, b, s, t, relu in frames + segs:
        flags = (_lib.RELU if relu else 0) | (_lib.BN if s is not None else 0)
        w3 = np.asarray(w, np.float32).reshape(w.shape[0], w.shape[1], -1)
        out += struct.pack("<7i", w3.shape[0], w3.shape[1], len(ctx), w3.shape[2], flags, b is not None, s is not None)
        out += struct.pack("<%di" % len(ctx), *ctx)
        for a in (w3, b, s, t):
            if a is not None:
                out += np.ascontiguousarray(np.asarray(a, np.float32), dtype="<f4").tobytes()
    return bytes(out)


def _hand_built():
    """Frame layers over the contexts [-2..2], [-2,0,2], [-3,0,3] and [0], with and without bias, BatchNorm and ReLU."""
    r = np.random.default_rng(11)
    w = lambda *s: (r.standard_normal(s) / np.sqrt(np.prod(s[1:]))).astype(np.float32)   # noqa: E731
    v = lambda n: r.standard_normal(n).astype(np.float32)   # noqa: E731
    ex = _Recorded(24)
    ex.add_frame_layer(w(64, 24, 5), v(64), [-2, -1, 0, 1, 2], v(64) + 2, v(64))
    ex.add_frame_layer(w(64, 64, 5), None, [-2, 0, 2])
    ex.add_frame_layer(w(64, 64, 7), v(64), [-3, 0, 3], relu=False)
    ex.add_frame_layer(w(32, 64, 1), v(32), [0], v(32) + 2, v(32))
    ex.add_segment_layer(w(24, 64), v(24), v(24) + 2, v(24), relu=True)
    ex.add_segment_layer(w(16, 24), None)
    ex.finalize(pooling_eps=1e-6)
    return ex


TDNN_CASES = {"xvector_far": ("xvector", 23, 101, "far"), "xvector_near": ("xvector", 23, 101, "near"),
              "extended_near": ("extended", 80, 103, "near"), "snowdar_near_full": ("snowdar", 40, 301, "near"),
              "hand_built": None}


def _tdnn(case, monkeypatch):
    if TDNN_CASES[case] is None:
        return _hand_built()
    kind, dim, seed, pos = TDNN_CASES[case]
    if kind == "xvector":
        from asv_subtools_b200.model.xvector import Xvector as cls
        spec = onn.xvector_spec(dim)
    elif kind == "extended":
        from asv_subtools_b200.model.extended_xvector import ExtendedXvector as cls
        spec = onn.extended_xvector_spec(dim)
    else:   # the snowdar Xvector's "near" is the whole last layer (built as near_full)
        from asv_subtools_b200.model.snowdar_xvector import Xvector as cls
        spec = onn.snowdar_xvector_spec(dim)
    m = cls(dim, 10, training=False, extracted_embedding=pos)
    m.load_state_dict(onn.make_state_dict(spec, seed), strict=True)
    monkeypatch.setattr(ops, "Extractor", _Recorded)   # build_tdnn_extractor hands its layers to a _Recorded
    ex = m.cuda().eval().extractor()
    assert isinstance(ex, _Recorded)
    return ex


@pytest.mark.parametrize("case", sorted(TDNN_CASES))
def test_tdnn_model_file_bytes_roundtrip_and_rejects(tmp_path, monkeypatch, case):
    ex = _tdnn(case, monkeypatch)
    path, again, bad = str(tmp_path / "model.xvbm"), str(tmp_path / "again.xvbm"), str(tmp_path / "bad.xvbm")
    ex.save(path)
    data = open(path, "rb").read()
    assert data == _xvbm_write(ex)
    loaded = _Recorded.load(path)
    assert (loaded.feat_dim, loaded.embed_dim) == (ex.feat_dim, ex.embed_dim)
    loaded.save(again)
    assert open(again, "rb").read() == data

    def patched(offset, value):
        b = bytearray(data)
        b[offset:offset + 4] = struct.pack("<i", value)
        return bytes(b)

    layer0 = 24   # after magic, feat_dim, pooling_eps, n_frame, n_segment
    blobs = [(data[:-100], "is truncated in layer"),                      # cut inside the last layer's arrays
             (data[:layer0 + 52], "is truncated in layer 0"),             # cut inside the first weight
             (data[:layer0 + 10], "bad layer 0 header"),                  # cut inside the first layer's ints
             (patched(layer0, 0), "bad layer 0 header"),                  # Cout 0
             (patched(layer0 + 8, 17), "bad layer 0 header"),             # more taps than XVB_MAX_TAPS
             (patched(layer0 + 12, 4096), "bad layer 0 header"),          # tot_context out of range
             (patched(16, 0), "bad header"),                              # no frame layer
             (b"XVBM0002" + data[8:], "is not an XVBM0001 file")]
    for blob, msg in blobs:
        with open(bad, "wb") as f:
            f.write(blob)
        with pytest.raises(RuntimeError, match=msg):
            _Recorded.load(bad)
