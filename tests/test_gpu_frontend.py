"""Front-end kernels (energy VAD, CMN, voiced-frame selection) on ragged batches vs the oracle."""
import numpy as np
import pytest
import torch

from oracle import frontend as ofe

pytestmark = pytest.mark.gpu


def _utts(seed, lens, F=24):
    rng = np.random.RandomState(seed)
    out = []
    for T in lens:
        f = rng.standard_normal((T, F)).astype(np.float32)
        f[:, 0] = rng.uniform(2.0, 9.0, T).astype(np.float32) + 2.0 * np.sin(np.arange(T) / 7.0)   # log-energy column
        out.append(f)
    return out


def test_vad_cmn_select_match_oracle():
    from asv_subtools_b200 import frontend as fe
    utts = _utts(0, [1, 7, 200, 333, 64])
    x, off = fe.pack(utts)
    for ctx, prop, scale in ((0, 0.6, 0.5), (2, 0.12, 0.5), (5, 0.6, 0.0)):
        voiced, counts = fe.vad_energy(x, off, 5.5, scale, ctx, prop)
        v = voiced.cpu().numpy()
        o = off.cpu().numpy()
        for i, u in enumerate(utts):
            ref = ofe.vad_energy(u, 5.5, scale, ctx, prop)
            got = v[o[i]:o[i + 1]]
            assert (got != ref).mean() <= 0.01, (ctx, prop, i)     # energies next to the threshold: summation order of the mean
            assert counts[i].item() == got.sum()
        y, new_off = fe.select_frames(x, off, voiced, counts)
        parts = fe.unpack(y, new_off)
        for i, u in enumerate(utts):
            assert np.array_equal(parts[i].cpu().numpy(), ofe.select_voiced(u, v[o[i]:o[i + 1]]))
    for i, (a, u) in enumerate(zip(fe.unpack(fe.cmn(x, off, 0), off), utts)):
        assert np.allclose(a.cpu().numpy(), ofe.cmn_utterance(u), atol=2e-6)
    for w in (300, 50, 8):
        for a, u in zip(fe.unpack(fe.cmn(x, off, w), off), utts):
            ref = ofe.cmn_sliding(u, w) if u.shape[0] > w else ofe.cmn_utterance(u)
            assert np.allclose(a.cpu().numpy(), ref, atol=5e-6), w


def test_frontend_feeds_the_extractor():
    """VAD -> CMN -> select -> bucket by length -> extractor == the same steps through the oracle."""
    from asv_subtools_b200 import frontend as fe
    from asv_subtools_b200.model.xvector import Xvector
    from oracle import nnet as onn
    utts = _utts(3, [120, 150, 120], F=24)
    x, off = fe.pack(utts)
    voiced, counts = fe.vad_energy(x, off, 5.5, 0.5, 0, 0.6)
    y, noff = fe.select_frames(fe.cmn(x, off, 0), off, voiced, counts)
    sd = onn.make_state_dict(onn.xvector_spec(24), 9)
    m = Xvector(24, 10, training=False)
    m.load_state_dict(sd, strict=True)
    m.cuda().eval()
    for i, part in enumerate(fe.unpack(y, noff)):
        got = m.extract_embedding(part.cpu().numpy()).numpy()
        v = voiced.cpu().numpy()[off.cpu().numpy()[i]:off.cpu().numpy()[i + 1]]
        ref_feats = ofe.select_voiced(ofe.cmn_utterance(utts[i]), v)
        ref = onn.extract_embedding(lambda z: onn.xvector_forward(sd, z, "far"), ref_feats).numpy()
        assert np.max(np.abs(got - ref)) / np.max(np.abs(ref)) < 1e-4
