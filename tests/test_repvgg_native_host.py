"""Records the RepVGG / RepSPK x-vector hands to the native extractor (xvb_repvgg_set_layer), on the CPU: every
state_dict tensor the extracted position uses is covered by exactly one record, in the training and the deploy form;
block records are the fp32 folds; the first segment record carries the pooling-order column permutation; the
configuration block matches the model; and the library's tap rule (xvb_conv2d_kept_taps, host only) equals kept_taps."""
import ctypes as C

import numpy as np
import pytest
import torch

import repvgg_oracle as ro
from asv_subtools_b200 import _lib
from asv_subtools_b200.model.repvgg_xvector import (RepVggXvector, _named_records, fold_block, kept_taps,
                                                    native_config)
from asv_subtools_b200.model.resnet_xvector import _stats_column_order
from oracle import nnet as onn

CASE_POS = [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]]


def _model(case, pos, deploy=False, sd=None):
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    if sd is None:
        sd = onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed)
        sd = ro.deploy_state_dict(sd, kwargs) if deploy else sd
    m = RepVggXvector(fdim, 10, training=False, extracted_embedding=pos, **({"deploy": True} if deploy else {}), **kwargs)
    m.load_state_dict(sd, strict=True)
    return m.eval()


def _unused(sd, pos):
    """state_dict keys of the segment layer the position does not run at all: fc2 for far (near_affine runs fc2.affine
    alone, under the record "fc2"; test_first_segment_record_is_column_permuted pins which arrays it carries)."""
    return {k for k in sd if k.startswith("fc2.")} if pos == "far" else set()


@pytest.mark.parametrize("deploy", [False, True])
@pytest.mark.parametrize("case, pos", CASE_POS)
def test_records_cover_the_state_dict(case, pos, deploy):
    m = _model(case, pos, deploy)
    recs = _named_records(m)
    names = [r[0] for r in recs]
    assert len(names) == len(set(names))
    sd = m.state_dict()
    seen = []
    for name, *_ in recs:
        keys = [k for k in sd if k.startswith(name + ".")]
        assert keys, "record {} names no state_dict module".format(name)
        seen += keys
    assert len(seen) == len(set(seen)), "a key is consumed twice"
    assert set(seen) == set(sd) - _unused(sd, pos), set(sd) ^ set(seen)
    blocks = m.repvgg.blocks()
    assert names[:len(blocks)] == ["repvgg.stage0"] + ["repvgg.stage{}.{}".format(s, i) for s in range(1, 5)
                                                       for i in range(len(getattr(m.repvgg, "stage{}".format(s))))]
    for (name, w, b, scale, shift, relu), blk in zip(recs, blocks):
        fw, fb = fold_block(blk)
        assert w.dtype == np.float32 and np.array_equal(w, fw.float().numpy()), name
        assert np.array_equal(b, fb.float().numpy()) and scale is None and shift is None and relu, name
        assert w.shape == (blk.out_channels, blk.in_channels, blk.window, blk.window)


def test_training_and_deploy_records_have_the_same_shapes():
    tr, de = _named_records(_model("grouped", "near")), _named_records(_model("grouped", "near", deploy=True))
    assert [(r[0], r[1].shape) for r in tr] == [(r[0], r[1].shape) for r in de]


@pytest.mark.parametrize("case, pos", CASE_POS)
def test_first_segment_record_is_column_permuted(case, pos):
    m = _model(case, pos)
    recs = _named_records(m)
    seg = [r for r in recs if r[0] in ("fc1", "fc2")]
    first = seg[0]
    assert first[0] == ("fc1" if m.fc1 is not None else "fc2")
    assert len(seg) == (1 if pos == "far" else 1 + (m.fc1 is not None))
    layer = getattr(m, first[0])
    perm = _stats_column_order(m.repvgg.get_output_planes(), m.out_freq)
    whole = pos != "far" and (first[0] == "fc1" or pos == "near")
    w = layer.export()[0].numpy()[:, :, 0] if whole else layer.affine.weight.detach().numpy()[:, :, 0]
    assert np.array_equal(first[1], w[:, perm])
    assert not np.array_equal(first[1], w)
    for rec in seg[1:]:
        w2 = m.fc2.export()[0].numpy()[:, :, 0] if pos == "near" else m.fc2.affine.weight.detach().numpy()[:, :, 0]
        assert np.array_equal(rec[1], w2)


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_config_block_matches_the_model(case):
    kwargs, fdim, _, positions, _, _ = ro.CASES[case]
    m = _model(case, positions[0])
    cfg = ro._config(kwargs)
    c = native_config(m)
    blocks = cfg["blocks"]
    assert c["feat_dim"] == fdim and c["ksize"] == (5 if cfg["spk"] else 3)
    assert c["widths"] == [blocks[0][2]] + [next(b[2] for b in blocks if b[0].startswith("repvgg.stage{}.".format(s)))
                                            for s in range(1, 5)]
    assert c["strides"] == [blocks[0][3]] + [next(b[3] for b in blocks if b[0] == "repvgg.stage{}.0".format(s))
                                             for s in range(1, 5)]
    assert c["num_blocks"] == [sum(b[0].startswith("repvgg.stage{}.".format(s)) for b in blocks) for s in range(1, 5)]
    assert c["pooling_eps"] == m.stats.eps
    # the XVBV0001 configuration block is the C struct: 16 int32s in declaration order, then the f32 eps
    st = _lib.RepVGGConfig(feat_dim=c["feat_dim"], ksize=c["ksize"], pooling_eps=c["pooling_eps"])
    for f in ("num_blocks", "strides", "widths"):
        getattr(st, f)[:] = c[f]
    raw = bytes(st)
    assert len(raw) == 68
    ints = [c["feat_dim"], c["ksize"]] + c["num_blocks"] + c["strides"] + c["widths"]
    assert raw == np.array(ints, "<i4").tobytes() + np.array([c["pooling_eps"]], "<f4").tobytes()


def _lib_taps(w, cap=25):
    w = np.ascontiguousarray(w, dtype=np.float32)
    out = (C.c_int * cap)()
    n = _lib.lib.xvb_conv2d_kept_taps(w.ctypes.data_as(C.c_void_p), w.shape[0], w.shape[1], w.shape[-1], out, cap)
    return n, list(out)[:max(n, 0)]


def _folds(case, deploy_sd=None):
    m = _model(case, ro.CASES[case][3][0], deploy=deploy_sd is not None, sd=deploy_sd)
    return [fold_block(b)[0].float() for b in m.repvgg.blocks()[1:]]


@pytest.mark.parametrize("case, expect", [("repspk", 17), ("a0", 9), ("grouped", 17)])
def test_library_tap_rule_equals_kept_taps_on_folds(case, expect):
    for w in _folds(case):
        want = kept_taps(w)
        assert len(want) == expect
        assert _lib_taps(w.numpy()) == (len(want), want)


def test_library_tap_rule_on_a_grouped_fold_and_an_all_zero_kernel():
    m = _model("grouped", "near")
    grouped = [fold_block(b)[0].float() for b in m.repvgg.blocks()[1:] if b.groups > 1]
    assert grouped
    for w in grouped:
        assert _lib_taps(w.numpy()) == (len(kept_taps(w)), kept_taps(w))
    for k in (3, 5):
        z = torch.zeros(32, 16, k, k)
        assert kept_taps(z) == [k * k // 2] and _lib_taps(z.numpy()) == (1, [k * k // 2])
    z = torch.zeros(16, 16, 5, 5)
    z[3, 9, 4, 0] = -0.0                     # negative zero is zero
    z[0, 0, 1, 3] = 1e-30
    assert kept_taps(z) == [8] and _lib_taps(z.numpy()) == (1, [8])


def test_library_tap_rule_keeps_a_nonzero_off_pattern_tap_of_a_deploy_file():
    kwargs, fdim, _, _, seed, _ = ro.CASES["repspk"]
    dsd = ro.deploy_state_dict(onn.make_state_dict(ro.repvgg_spec(fdim, kwargs), seed), kwargs)
    key = "repvgg.stage3.2.rbr_reparam.weight"
    dsd[key] = dsd[key].clone()
    dsd[key][5, 7, 0, 1] = 0.25
    m = _model("repspk", "near", deploy=True, sd=dsd)
    w = fold_block(m.repvgg.stage3[2])[0].float()
    want = kept_taps(w)
    assert len(want) == 18 and _lib_taps(w.numpy()) == (18, want)


def test_library_tap_rule_refuses_too_small_a_cap_and_bad_shapes():
    w = _folds("repspk")[0].numpy()
    assert _lib_taps(w, cap=16)[0] == -1
    assert "do not fit" in _lib.last_error()
    assert _lib_taps(w, cap=17)[0] == 17
    out = (C.c_int * 25)()
    assert _lib.lib.xvb_conv2d_kept_taps(None, 4, 4, 3, out, 25) == -1
    x = np.zeros((4, 4, 3, 3), np.float32)
    assert _lib.lib.xvb_conv2d_kept_taps(x.ctypes.data_as(C.c_void_p), 0, 4, 3, out, 25) == -1
    assert "bad arguments" in _lib.last_error()
