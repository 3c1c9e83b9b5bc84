"""Records the ResNet x-vector hands to the native extractor (xvb_resnet_set_layer), on the CPU: every convolution,
BatchNorm, SE and fc tensor of the state_dict is covered by exactly the record named after its module, with its values,
and the first segment record carries the pooling-order column permutation."""
import numpy as np
import pytest
import torch

import resnet_oracle as ro
from asv_subtools_b200.model.resnet_xvector import ResNetXvector, _named_records, _stats_column_order
from asv_subtools_b200.nnet.components import fold_batchnorm
from oracle import nnet as onn


def _model(case, pos):
    kwargs, fdim, _, _, seed, _ = ro.CASES[case]
    m = ResNetXvector(fdim, 10, training=False, extracted_embedding=pos, **kwargs)
    m.load_state_dict(onn.make_state_dict(ro.resnet_spec(fdim, kwargs), seed), strict=True)
    return m.eval(), kwargs


def _module(m, name):
    mod = m
    for part in name.split("."):
        mod = getattr(mod, part) if not part.isdigit() else mod[int(part)]
    return mod


@pytest.mark.parametrize("case", sorted(ro.CASES))
def test_records_cover_the_state_dict(case):
    m, kwargs = _model(case, "near")
    recs = _named_records(m)
    names = [r[0] for r in recs]
    assert len(names) == len(set(names))
    sd = m.state_dict()
    covered = set()
    for name, w, b, scale, shift, relu in recs:
        keys = {k for k in sd if k.startswith(name + ".")}
        assert keys, "record {} names no state_dict module".format(name)
        covered |= keys
        if name in ("fc1", "fc2"):
            continue
        mod = _module(m, name)
        if isinstance(mod, torch.nn.BatchNorm2d):
            s, t = fold_batchnorm(mod)
            assert w is None and b is None and np.array_equal(scale, s) and np.array_equal(shift, t), name
        else:
            assert np.array_equal(w, sd[name + ".weight"].numpy()), name
            assert (b is None) == (name + ".bias" not in sd), name
            if b is not None:
                assert np.array_equal(b, sd[name + ".bias"].numpy()), name
            assert scale is None and shift is None and not relu, name
    assert covered == set(sd), set(sd) ^ covered
    convs = [n for n in names if n.endswith(("conv1", "conv2", "downsample.0"))]
    cfg = ro._config(kwargs)
    assert len(convs) == 1 + 2 * sum(cfg["layers"]) + 3
    assert sum(n.endswith("se.fc_1") for n in names) == (sum(cfg["layers"]) if cfg["use_se"] else 0)


@pytest.mark.parametrize("case, pos", [(c, p) for c in sorted(ro.CASES) for p in ro.CASES[c][3]])
def test_first_segment_record_is_column_permuted(case, pos):
    m, _ = _model(case, pos)
    recs = _named_records(m)
    seg = [r for r in recs if r[0] in ("fc1", "fc2")]
    first = seg[0]
    assert first[0] == ("fc1" if m.fc1 is not None else "fc2")
    assert len(seg) == (1 if pos == "far" else 1 + (m.fc1 is not None))
    layer = getattr(m, first[0])
    perm = _stats_column_order(m.resnet.layer4[0].conv1.out_channels, m.out_freq)
    stored = layer.affine.weight.detach().numpy()[:, :, 0]
    assert first[1].shape == stored.shape
    whole = pos != "far" and (first[0] == "fc1" or pos == "near")
    w = layer.export()[0].numpy()[:, :, 0] if whole else stored
    assert np.array_equal(first[1], w[:, perm])
    assert not np.array_equal(first[1], w)
    for rec in seg[1:]:                                 # later layers keep their stored column order
        w2 = m.fc2.export()[0].numpy()[:, :, 0] if pos == "near" else m.fc2.affine.weight.detach().numpy()[:, :, 0]
        assert np.array_equal(rec[1], w2)
