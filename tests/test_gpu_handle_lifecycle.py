"""The lifecycle all six native extractor handles share (csrc/records.cuh, Handle): a draft from create until finalize
succeeds, then an immutable model.  A draft refuses every extract, extract_host and save entry point with XVB_EINVAL; a
finalized handle refuses set_layer / add_*_layer; destroy(NULL) is a no-op; and a finalize refused for a missing block
record leaves a draft that, once given the record, finalizes to exactly the model a fresh handle builds from the same
records in the same order: the same embeddings bit for bit, the same launch count and the same model file."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import campplus_oracle as cpo  # noqa: E402
import conformer_oracle as co  # noqa: E402
import ecapa_mqmha_oracle as mo  # noqa: E402
import repvgg_oracle as rvo  # noqa: E402
import resnet_oracle as ro  # noqa: E402
from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200._lib import XvbError, check, int_array, last_error, lib  # noqa: E402
from asv_subtools_b200.model.campplus_xvector import CamPPXvector, NativeCamPPExtractor  # noqa: E402
from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN, NativeEcapaExtractor  # noqa: E402
from asv_subtools_b200.model.repvgg_xvector import NativeRepVGGExtractor, RepVggXvector  # noqa: E402
from asv_subtools_b200.model.resnet_xvector import NativeResNetExtractor, ResNetXvector  # noqa: E402
from asv_subtools_b200.model.transformer_xvector import NativeConformerExtractor, TransformerXvector  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu

EINVAL, XVB_ESTATE = -1, -4
FAMILIES = ["extractor", "ecapa", "resnet", "repvgg", "conformer", "campp"]


def _resnet():
    kw, fdim, _, _, seed, _ = ro.CASES["preact"]
    m = ResNetXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kw), seed), strict=True)
    return NativeResNetExtractor, m, fdim, 30, "resnet.layer2.0.conv2"


def _repvgg():
    kw, fdim, _, _, seed, _ = rvo.CASES["a0"]
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(onn.make_state_dict(rvo.repvgg_spec(fdim, kw), seed), strict=True)
    return NativeRepVGGExtractor, m, fdim, 30, "repvgg.stage2.1"


def _conformer():
    kw, fdim = co.CASES["small"][:2]
    g = np.load(os.path.join(HERE, "golden", "conformer.npz"))
    m = TransformerXvector(fdim, 10, training=False, extracted_embedding="near", **kw)
    m.load_state_dict(co.seeded_state_dict(g["keys_small"], co.CASES["small"][4]), strict=True)
    return NativeConformerExtractor, m, fdim, 40, "transformer.encoders.0.self_attn.linear_qkv"


def _campp():
    kw = dict(cpo.CASES["small"][0])
    fdim = kw.pop("inputs_dim")
    g = np.load(os.path.join(HERE, "golden", "campplus.npz"))
    m = CamPPXvector(fdim, 10, **kw)
    m.load_state_dict(cpo.seeded_state_dict(g["keys_small"], cpo.CASES["small"][3]), strict=True)
    return NativeCamPPExtractor, m, fdim, 40, "xvector.block2.tdnnd1.linear1"


def _ecapa(mqmha, held):
    """ECAPA-TDNN (the default model, or MQMHA pooling with fc1) holding back `held`: "mfa" is refused after the Res2Net
    stacks are built, "layer4.res6" while the last one is."""
    def make():
        if mqmha:
            kwargs, _, _, seed, _ = mo.CASES["fc1"]
            m = ECAPA_TDNN(80, 10, training=False, extracted_embedding="near", **kwargs)
            m.load_state_dict(onn.make_state_dict(mo.ecapa_mqmha_spec(kwargs), seed), strict=True)
        else:
            m = ECAPA_TDNN(80, 10, training=False)
            m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), 201), strict=True)
        return NativeEcapaExtractor, m, 80, 40, held
    return make


RECORD_MODELS = {"resnet": _resnet, "repvgg": _repvgg, "conformer": _conformer, "campp": _campp}
RETRY_MODELS = dict(RECORD_MODELS, **{"ecapa{}-{}".format("_mqmha" if mq else "", held): _ecapa(mq, held)
                                     for mq in (False, True) for held in ("mfa", "layer4.res6")})


def _draft(cls, m):
    """A handle of cls between create (and the family's configuration) and finalize, driven record by record."""
    ex = cls.__new__(cls)
    ex._lib, ex._check, ex._h = lib, check, C.c_void_p()
    ex._call("create", C.byref(ex._h), *ex._create_args(m))
    ex._configure(m)
    return ex


def _set(ex, rec):
    name, shape, arrays, flags = rec
    arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float32) for a in arrays]
    ptr = [None if a is None else a.ctypes.data_as(C.c_void_p) for a in arrs]
    return ex._fn("set_layer")(ex._h, name.encode(), *shape, *ptr, flags)


def _finalize(ex):
    rc = ex._fn("finalize")(ex._h)
    if rc == 0:
        ex.feat_dim, ex.embed_dim = ex._fn("feat_dim")(ex._h), ex._fn("embed_dim")(ex._h)
    return rc


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _draft_of(family):
    """A new draft handle of `family` (the record families with their configuration only) and its feature dim."""
    h = C.c_void_p()
    if family == "extractor":
        check(lib.xvb_extractor_create(C.byref(h), 24), "xvb_extractor_create")
        return h, 24
    if family == "ecapa":
        check(lib.xvb_ecapa_create(C.byref(h), 80, 1024, 1536, 128, 192), "xvb_ecapa_create")
        return h, 80
    cls, m, fdim, _, _ = RECORD_MODELS[family]()
    ex = _draft(cls, m)
    h, ex._h = ex._h, None
    return h, fdim


@pytest.mark.parametrize("family", FAMILIES)
def test_a_draft_refuses_every_extract_and_save(family, tmp_path):
    h, fdim = _draft_of(family)
    fn = lambda name: getattr(lib, "xvb_{}_{}".format(family, name))   # noqa: E731
    B, T = 2, 40
    x, y = torch.zeros(B, T, fdim, device="cuda"), torch.zeros(B, 512, device="cuda")
    feats, emb = C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr())
    host_feats, host_emb = np.zeros((B, T, fdim), np.float32), np.zeros((B, 512), np.float32)
    hp = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731
    lens = (C.c_int32 * B)(T, T - 1)
    calls = {"extract": lambda: fn("extract")(h, feats, B, T, emb, _stream())}
    if family in ("extractor", "resnet"):
        calls["extract_lengths"] = lambda: fn("extract_lengths")(h, feats, lens, B, T, emb, _stream())
    if family in ("extractor", "ecapa", "resnet"):
        calls["extract_host"] = lambda: fn("extract_host")(h, hp(host_feats), B, T, hp(host_emb), _stream())
        calls["extract_shard"] = lambda: fn("extract_shard")(h, feats, B, T, 1, emb, _stream())
        calls["extract_shard_host"] = lambda: fn("extract_shard_host")(h, hp(host_feats), B, T, 1, hp(host_emb), _stream())
    if family == "extractor":
        calls["submit_host"] = lambda: fn("submit_host")(h, hp(host_feats), B, T, hp(host_emb), 0, _stream())
    calls["save"] = lambda: fn("save")(h, str(tmp_path / "draft.bin").encode())
    try:
        for name, call in calls.items():
            assert call() == EINVAL, (family, name)
            assert "xvb_{}_{}".format(family, name) in last_error(), (family, name, last_error())
        assert not os.path.exists(tmp_path / "draft.bin")
        # each family's own answer for a draft: ECAPA-TDNN and CAM++ read the configured width, the TDNN has no
        # segment layer yet, the others refuse
        assert fn("embed_dim")(h) == {"extractor": XVB_ESTATE, "ecapa": 192, "campp": 192}.get(family, EINVAL), family
    finally:
        fn("destroy")(h)


@pytest.mark.parametrize("family", FAMILIES)
def test_destroy_null_is_a_no_op(family):
    getattr(lib, "xvb_{}_destroy".format(family))(None)


def _tdnn_layers(seed=5):
    r = np.random.default_rng(seed)
    w = lambda *s: (r.standard_normal(s) / np.sqrt(np.prod(s[1:]))).astype(np.float32)   # noqa: E731
    b = lambda n: r.standard_normal(n).astype(np.float32)   # noqa: E731
    frame = [(w(64, 24, 5), b(64), [-2, -1, 0, 1, 2]), (w(64, 64, 1), b(64), [0])]
    seg = [(w(32, 128), b(32))]
    return frame, seg


def test_tdnn_finalize_retries_after_the_missing_segment_layer(tmp_path):
    frame, seg = _tdnn_layers()
    retried, fresh = ops.Extractor(24), ops.Extractor(24)
    for wt, b, ctx in frame:
        retried.add_frame_layer(wt, b, ctx)
        fresh.add_frame_layer(wt, b, ctx)
    with pytest.raises(XvbError, match="need >=1 frame and >=1 segment layer"):
        retried.finalize()
    for wt, b in seg:
        retried.add_segment_layer(wt, b)
        fresh.add_segment_layer(wt, b)
    retried.finalize()
    fresh.finalize()
    x = torch.from_numpy(onn.synthetic_feats(3, 50, 24, 9)).cuda()
    got, want = retried.extract(x), fresh.extract(x)
    assert torch.equal(got, want) and retried.last_launches == fresh.last_launches
    retried.save(tmp_path / "retried.bin")
    fresh.save(tmp_path / "fresh.bin")
    assert (tmp_path / "retried.bin").read_bytes() == (tmp_path / "fresh.bin").read_bytes()
    wt, b, ctx = frame[0]
    w_np = np.ascontiguousarray(wt)
    for h in (retried, fresh):   # finalized: no more layers
        assert lib.xvb_extractor_add_frame_layer(h._h, 64, int_array(ctx), len(ctx), w_np.ctypes.data_as(C.c_void_p),
                                                 None, None, None, 0) == EINVAL
        assert lib.xvb_extractor_add_segment_layer(h._h, 32, w_np.ctypes.data_as(C.c_void_p), None, None, None,
                                                   0) == EINVAL


def test_ecapa_set_layer_refuses_a_finalized_handle():
    m = ECAPA_TDNN(80, 10, training=False)
    m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), 201), strict=True)
    ex = NativeEcapaExtractor(m.cuda().eval())
    name, shape, arrays, flags = next(iter(ex._layers(m)))
    w = np.ascontiguousarray(arrays[0], dtype=np.float32)
    assert lib.xvb_ecapa_set_layer(ex._h, b"extra", shape[0], shape[1], shape[2], shape[3], w.ctypes.data_as(C.c_void_p),
                                   None, None, None, 0) == EINVAL
    assert lib.xvb_ecapa_set_mqmha(ex._h, 1, 1, 128, 0, 2, 1, 1) == EINVAL
    assert ex.extract(torch.from_numpy(onn.synthetic_feats(2, 40, 80, 3)).cuda()).shape == (2, 192)


@pytest.mark.parametrize("family", sorted(RETRY_MODELS))
def test_finalize_after_a_missing_record_equals_a_fresh_handle(family, tmp_path):
    cls, m, fdim, T, held = RETRY_MODELS[family]()
    m = m.cuda().eval()
    records = list(cls.__new__(cls)._layers(m))
    order = [r for r in records if r[0] != held] + [r for r in records if r[0] == held]
    assert len(order) == len(records) and order[-1][0] == held

    retried = _draft(cls, m)
    for rec in order[:-1]:
        assert _set(retried, rec) == 0, last_error()
    assert _finalize(retried) == EINVAL
    what = "layer" if family.startswith("ecapa") else "record"
    assert "{} '{}' is missing".format(what, held) in last_error(), last_error()
    assert _set(retried, order[-1]) == 0, last_error()
    assert _finalize(retried) == 0, last_error()

    fresh = _draft(cls, m)
    for rec in order:
        assert _set(fresh, rec) == 0, last_error()
    assert _finalize(fresh) == 0, last_error()

    assert (retried.feat_dim, retried.embed_dim) == (fresh.feat_dim, fresh.embed_dim)
    with torch.no_grad():
        for b, t in ((1, T), (3, T + 7)):
            x = torch.from_numpy(onn.synthetic_feats(b, t, fdim, 100 + b)).cuda()
            got = retried.extract(x)
            n_got = retried.last_launches
            want = fresh.extract(x)
            assert torch.equal(got, want), (family, b, t, (got - want).abs().max().item())
            assert n_got == fresh.last_launches, (family, n_got, fresh.last_launches)
    retried.save(tmp_path / "retried.bin")
    fresh.save(tmp_path / "fresh.bin")
    assert (tmp_path / "retried.bin").read_bytes() == (tmp_path / "fresh.bin").read_bytes()
    assert _set(retried, order[0]) == EINVAL             # finalized: no more records
    assert "finalized" in last_error()
    assert _finalize(retried) == EINVAL
