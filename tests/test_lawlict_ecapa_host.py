"""The ECAPA-TDNN of pytorch/model/ecapa-tdnn-xvector.py (the runEcapaXvector.py launcher's model) on the CPU: the torch
restatement against the reference's golden embeddings, the blueprint's state_dict layout and creation string, the
records the ECAPA-TDNN handle receives (every tensor carried once; in float64, in the handle's launch order, they equal
the restatement, which checks the Res2Net chunk rotation and the bn_stats fold), the poolings that are not built, and
the C declaration of the attention switch."""
import importlib.util
import os
import re
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import lawlict_ecapa_oracle as lo  # noqa: E402
from asv_subtools_b200 import _lib  # noqa: E402
from asv_subtools_b200.pipeline import extract_embeddings  # noqa: E402
from oracle import nnet as onn  # noqa: E402

BLUEPRINT = os.path.join(ROOT, "asv_subtools_b200", "model", "ecapa-tdnn-xvector.py")
GOLDEN = np.load(os.path.join(HERE, "golden", "lawlict_ecapa.npz"))


def _load_blueprint():
    spec = importlib.util.spec_from_file_location("lawlict_ecapa_blueprint", BLUEPRINT)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


bp = _load_blueprint()


def _keys(sd):
    return ["{}:{}".format(k, ",".join(str(d) for d in v.shape)) for k, v in sd.items()]


def _params(sd):
    return sum(v.numel() for k, v in sd.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))


def _model(inputs_dim, kw, position="near"):
    return bp.ECAPA_TDNN(inputs_dim, 1211, **dict(kw, extracted_embedding=position))


@pytest.mark.parametrize("key", lo.keys())
def test_oracle_replays_golden(key):
    case, rest = key.split("_", 1)
    pos, t = rest.rsplit("_T", 1)
    t = int(t)
    _, kw, short, _, _, _, _ = lo.CASES[case]
    sd = lo.state_dict(case)
    feats = lo.utterances(case, t)
    with torch.no_grad():
        if t in short:
            got = torch.cat([lo.forward(sd, torch.from_numpy(f.T.copy())[None], kw, pos)[:, :, 0] for f in feats]).numpy()
        else:
            got = np.stack([lo.extract_embedding(sd, f, kw, pos).numpy() for f in feats])
    want = GOLDEN[key]
    assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), key


@pytest.mark.parametrize("case", sorted(lo.CASES))
def test_state_dict_layout_equals_reference(case):
    inputs_dim, kw, _, _, _, _, _ = lo.CASES[case]
    m = _model(inputs_dim, kw)
    assert _keys(m.state_dict()) == list(GOLDEN["keys_" + case])
    assert _params(m.state_dict()) == int(GOLDEN["params_" + case])
    train = _model(inputs_dim, dict(kw, training=True))
    assert _keys(train.state_dict()) == list(GOLDEN["train_keys_" + case])
    m.load_state_dict(lo.state_dict(case), strict=True)


def test_parameter_counts():
    assert _params(bp.ECAPA_TDNN(80, 1211, training=False, channels=512).state_dict()) == int(GOLDEN["params_default"]) \
        == lo.PARAMS_DEFAULT
    assert _params(_model(80, lo.LAUNCHER).state_dict()) == lo.PARAMS_LAUNCHER
    soft = bp.ECAPA_TDNN(80, 10, margin_loss=False)
    assert [k for k in soft.state_dict() if k.startswith("loss.")] == ["loss.affine.weight", "loss.affine.bias"]


def test_launcher_creation_string_builds_through_blueprint_dir(tmp_path):
    """nnet.config names the reference's subtools/pytorch/model/ecapa-tdnn-xvector.py with the launcher's creation string
    (training=True); --blueprint-dir swaps in this file by its name and the creation string evaluates unchanged.  The
    launcher's training checkpoint, loss layer included, loads strictly."""
    creation = lo.creation_string(dict(lo.LAUNCHER, training=True))
    cfg = tmp_path / "nnet.config"
    cfg.write_text('model_blueprint;"subtools/pytorch/model/ecapa-tdnn-xvector.py"\nmodel_creation;"{}"\n'.format(
        creation.replace('"', '""')))
    blueprint, got_creation = extract_embeddings.read_nnet_config(str(cfg))
    assert got_creation == creation
    swapped = os.path.join(ROOT, "asv_subtools_b200", "model", os.path.basename(blueprint))
    assert os.path.exists(swapped)
    m = extract_embeddings.create_model_from_py(swapped, creation)
    assert type(m).__name__ == "ECAPA_TDNN" and m.extracted_embedding == "near" and m.channels == 512
    assert type(m).__module__ == "ecapa-tdnn-xvector"
    sd = dict(lo.state_dict("launcher"), **{"loss.weight": torch.zeros(1211, 192, 1)})
    m.load_state_dict(sd, strict=True)
    assert _keys(m.state_dict()) == list(GOLDEN["train_keys_launcher"])


@pytest.mark.parametrize("pooling", ["attentive", "multi-head", "global-multi", "multi-resolution", "statistics", "lde"])
def test_unbuilt_poolings_raise_naming_the_option(pooling):
    with pytest.raises(NotImplementedError, match="pooling='{}'".format(pooling)):
        bp.ECAPA_TDNN(80, 10, pooling=pooling, training=False)


def test_positions():
    m = _model(80, lo.LAUNCHER, "far")
    with pytest.raises(AssertionError, match="fc1"):
        m.build_extractor()
    with pytest.raises(TypeError, match="position"):
        _model(80, lo.LAUNCHER, "middle").build_extractor()


# small widths: the records are rebuilt once per state_dict tensor
TINY = {
    "near": (24, lo.kwargs(channels=64, embd_dim=16), "near"),
    "fc1_near": (24, lo.kwargs(channels=64, embd_dim=16, fc1=True), "near"),
    "fc1_near_affine": (24, lo.kwargs(channels=64, embd_dim=16, fc1=True), "near_affine"),
    "fc1_far": (24, lo.kwargs(channels=64, embd_dim=16, fc1=True), "far"),
}


@pytest.mark.parametrize("case", sorted(TINY))
def test_records_read_every_tensor_once(case):
    """Each state_dict tensor changes exactly one record when perturbed, and every record depends on some tensor; what the
    position leaves out (fc1's BatchNorm and fc2 at "far", fc2's BatchNorm at "near_affine") changes none."""
    inputs_dim, kw, pos = TINY[case]
    m = _model(inputs_dim, kw, pos)
    sd = onn.make_state_dict(lo.spec(inputs_dim, kw), 3)
    m.load_state_dict(sd, strict=True)
    base = {r[0]: tuple(np.array(a) if isinstance(a, np.ndarray) else a for a in r) for r in bp.native_records(m)}
    assert "att_gs" not in base
    touched = set()
    for k in sd:
        if k.endswith("num_batches_tracked"):
            continue
        m.load_state_dict(dict(sd, **{k: sd[k] + 0.5}), strict=True)
        now = {r[0]: r for r in bp.native_records(m)}
        assert now.keys() == base.keys()
        changed = {n for n in base if any(
            (a is None) != (b is None) or (a is not None and not np.array_equal(np.asarray(a), np.asarray(b)))
            for a, b in zip(base[n][1:], now[n][1:]))}
        unused = (pos == "far" and k.startswith(("fc2.", "fc1.batchnorm."))) or \
            (pos == "near_affine" and k.startswith("fc2.batchnorm."))
        if unused:
            assert not changed, k
            continue
        assert len(changed) == 1, (k, changed)
        touched |= changed
    assert touched == set(base)


def _apply(rec, x):
    """One record over x (T, Cin) in float64: taps at the record's context (zero padding), bias, ReLU, BatchNorm."""
    _, w, b, ctx, s, t, relu = rec
    w = np.asarray(w, np.float64).reshape(w.shape[0], w.shape[1], -1)
    T = x.shape[0]
    y = np.zeros((T, w.shape[0]))
    for c in ctx:
        xs = np.zeros_like(x)
        lo_, hi = max(0, -c), min(T, T - c)
        if hi > lo_:
            xs[lo_:hi] = x[lo_ + c:hi + c]
        y += xs @ w[:, :, c - ctx[0]].T
    if b is not None:
        y += np.asarray(b, np.float64)
    if relu:
        y = np.maximum(y, 0)
    if s is not None:
        y = y * np.asarray(s, np.float64) + np.asarray(t, np.float64)
    return y


def _launch_order(recs, x, floor):
    """The records in the handle's launch order (ecapa_extractor.cu, xvb_ecapa_set_attention(h, 0, floor)), float64:
    layer1; per block bn1, the chain (chunk 0 passed through, y[i+1] = f_i(x[i+1] (+ y[i] for i >= 1))), bn2, SE gate,
    z * gate + block input into the MFA slot and the running sum; mfa; att_x (tanh, no utt bias), att2, softmax over T,
    weighted mean and std floored at `floor`; [fc1] [fc2]."""
    r = {rec[0]: rec for rec in recs}
    cur = _apply(r["layer1"], x)
    C = cur.shape[1]
    W = C // lo.SCALE
    run, slots = cur, []
    for li in (2, 3, 4):
        p = "layer{}.".format(li)
        h = _apply(r[p + "bn1"], cur)
        y = np.empty_like(h)
        y[:, :W] = h[:, :W]
        for i in range(lo.SCALE - 1):
            a = h[:, (i + 1) * W:(i + 2) * W] + (y[:, i * W:(i + 1) * W] if i >= 1 else 0)
            y[:, (i + 1) * W:(i + 2) * W] = _apply(r[p + "res{}".format(i)], a)
        z = _apply(r[p + "bn2"], y)
        g = _apply(r[p + "se1"], z.mean(0, keepdims=True))
        g = 1 / (1 + np.exp(-_apply(r[p + "se2"], g)))
        out = z * g + cur
        slots.append(out)
        run = run + out if li > 2 else cur + out
        cur = run
    m = _apply(r["mfa"], np.concatenate(slots, axis=1))
    a = _apply(r["att2"], np.tanh(_apply(r["att_x"], m)))
    a = np.exp(a - a.max(0))
    a /= a.sum(0)
    mean = (a * m).sum(0)
    std = np.sqrt(np.maximum((a * m * m).sum(0) - mean ** 2, floor))
    v = np.concatenate([mean, std])[None]
    for name in ("fc1", "fc2"):
        if name in r:
            v = _apply(r[name], v)
    return v[0]


@pytest.mark.parametrize("case,t", [("near", 23), ("fc1_near", 9), ("fc1_near_affine", 1), ("fc1_far", 4),
                                    ("launcher", 17)])
def test_records_in_launch_order_equal_oracle_float64(case, t):
    if case == "launcher":
        inputs_dim, kw, pos = 80, lo.LAUNCHER, "near"
    else:
        inputs_dim, kw, pos = TINY[case]
    sd = onn.make_state_dict(lo.spec(inputs_dim, kw), 21)
    m = _model(inputs_dim, kw, pos).double()
    m.load_state_dict(sd, strict=True)
    cfg = bp.native_config(m)
    assert cfg["attention"] == (0, 1e-9) and cfg["mqmha"] is None and not cfg["chained"]
    assert cfg["create"] == (inputs_dim, kw["channels"], 3 * kw["channels"], 128, kw["embd_dim"])
    x = onn.synthetic_feats(1, t, inputs_dim, 99 + t)[0].astype(np.float64)
    got = _launch_order(bp.native_records(m), x, 1e-9)
    with torch.no_grad():
        want = lo.forward({k: v.double() if v.is_floating_point() else v for k, v in sd.items()},
                          torch.from_numpy(x.T.copy())[None], kw, pos)[0, :, 0].numpy()
    # the records are fp32, so compare against the float64 restatement at fp32 weight rounding
    assert np.abs(got - want).max() <= 1e-5 * max(1.0, np.abs(want).max()), (case, np.abs(got - want).max())


def test_rotation_is_the_chunk_map():
    perm = bp.rotation(512)
    W = 64
    assert list(perm[:W]) == list(range(7 * W, 8 * W)) and list(perm[W:]) == list(range(7 * W))


def test_set_attention_declaration_matches_binding():
    header = open(os.path.join(ROOT, "include", "xvb200.h")).read()
    assert re.search(r"\bint xvb_ecapa_set_attention\(xvb_ecapa_t\* h, int global_context, float floor\);", header)
    assert _lib.SIGNATURES["xvb_ecapa_set_attention"] == (_lib.C.c_int, [_lib.C.c_void_p, _lib.C.c_int, _lib.C.c_float])
    fn = _lib.lib.xvb_ecapa_set_attention
    assert fn.restype is _lib.C.c_int and list(fn.argtypes) == [_lib.C.c_void_p, _lib.C.c_int, _lib.C.c_float]
