"""The grow-only workspace of the TDNN and ECAPA-TDNN native handles: a handle reused over a sequence of shapes, in which
each class of buffer (per frame, per utterance, fused-pooling partials, masked-call lengths) grows while the others do
not and a shape whose launch plan was cached before a growth comes back, computes every call bit for bit as a fresh
handle does, with the same launch count.  Needs an H100 (`-m gpu`)."""
import numpy as np
import pytest
import torch

from oracle import nnet as onn

pytestmark = pytest.mark.gpu


def _feats(b, t, seed):
    return torch.from_numpy(onn.synthetic_feats(b, t, 80, seed)).cuda()


def _xvector():
    from asv_subtools_b200.model.xvector import Xvector
    m = Xvector(80, 10, training=False, extracted_embedding="far")
    m.load_state_dict(onn.make_state_dict(onn.xvector_spec(80), 102), strict=True)
    return m.cuda().eval()


def test_tdnn_handle_reused_across_growing_shapes_equals_fresh_handles(monkeypatch):
    m = _xvector()
    ex = m.extractor()

    def check(feats, lengths=None, fused=True):
        got = ex.extract(feats, lengths).clone()
        launches = ex.last_launches
        fresh = m.build_extractor()
        fresh.set_fused_pooling(fused)
        assert torch.equal(got, fresh.extract(feats, lengths))
        assert launches == fresh.last_launches
        fresh.close()

    check(_feats(8, 200, 1))     # first call: every buffer grows
    check(_feats(32, 50, 2))     # the batch grows, the frames stay (8 x 200 = 32 x 50)
    check(_feats(8, 200, 3))     # a shape whose plan was cached before that growth
    check(_feats(4, 500, 4))     # the frames grow, the batch does not
    lens = np.random.RandomState(5).randint(1, 41, size=40)
    lens[0] = 17
    check(_feats(40, 40, 5), lens)  # masked, a batch larger than any so far: the lengths buffer grows
    check(_feats(8, 200, 6))
    ex.set_fused_pooling(False)  # no pooling partials from here on
    check(_feats(8, 200, 7), fused=False)
    monkeypatch.setenv("XVB_LANES", "1")
    feats = _feats(20, 200, 8)
    want = torch.cat([ex.extract(feats[i:i + 8]).clone() for i in range(0, 20, 8)])
    assert torch.equal(ex.extract_shard(feats, 8), want)


@pytest.mark.parametrize("im2col", ["0", "1"])
def test_ecapa_handle_reused_across_growing_shapes_equals_fresh_handles(monkeypatch, im2col):
    from asv_subtools_b200.model.ecapa_tdnn_xvector import ECAPA_TDNN, NativeEcapaExtractor
    monkeypatch.setenv("XVB_IM2COL", im2col)   # read when a handle is finalized
    m = ECAPA_TDNN(80, 10, training=False)
    m.load_state_dict(onn.make_state_dict(onn.ecapa_spec(80, fc2_bn_affine=True), 201), strict=True)
    m.cuda().eval()
    ex = m.extractor()
    assert isinstance(ex, NativeEcapaExtractor)
    # the batch grows with the frames staying, a shape seen before that growth, then the frames grow
    for i, (b, t) in enumerate(((4, 300), (16, 75), (4, 300), (2, 700))):
        feats = _feats(b, t, 20 + i)
        got = ex.extract(feats).clone()
        launches = ex.last_launches
        fresh = NativeEcapaExtractor(m, torch.cuda.current_device())
        assert torch.equal(got, fresh.extract(feats)), (b, t)
        assert launches == fresh.last_launches
        fresh.close()
