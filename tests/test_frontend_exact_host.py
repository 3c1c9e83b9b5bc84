"""tests/frontend_exact.py on the CPU: the catalogue reaches every block, window, ballot and FFT-size edge of frontend.cu
and fbank.cu (read from the case lists), the exactness preconditions hold, the references equal the oracle, the fp32
emulation of the fbank kernel stays inside the bound and each mutant of it leaves the bound by at least 4x."""
import numpy as np
import pytest

import frontend_exact as fx
from oracle import frontend as ofe


def test_vad_catalogue_and_exactness():
    cases = list(fx.vad_cases().values())
    assert {c["context"] for c in cases} >= {0, 1, 5} and max(c["context"] for c in cases) >= max(fx.VAD_T)
    assert {c["scale"] for c in cases} == {0.0, 0.5}
    at_thr = ties = 0
    for name, case in fx.vad_cases().items():
        lens, utts = fx.vad_operands(case, name)
        assert {fx.VAD_THREADS - 1, fx.VAD_THREADS, fx.VAD_THREADS + 1, 1, 2} <= set(lens)
        assert 0 in lens[1:-1]                                              # an empty utterance between two others
        for u in utts:
            e = u[:, 0]
            if not len(e):
                continue
            assert fx.vad_exact(e) and np.isnan(u[:, 1:]).all()
            thr = fx.vad_threshold(e, fx.VAD_THRESHOLD, case["scale"])
            assert np.float64(thr) == fx.VAD_THRESHOLD + case["scale"] * e.astype(np.float64).mean()   # exact threshold
            at_thr += int((e == thr).sum())
            if len(e) <= 300 or case["context"] <= 12:
                ref = ofe.vad_energy(u, fx.VAD_THRESHOLD, case["scale"], case["context"], case["prop"])
                assert np.array_equal(fx.vad_ref(e, fx.VAD_THRESHOLD, case["scale"], case["context"], case["prop"]), ref)
            if case["context"] == 12 and case["prop"] == 0.6 and len(e) >= 25:
                above = np.convolve(e > thr, np.ones(25, int), "valid")
                ties += int((above == 15).sum())
    assert at_thr > 100 and ties > 0


def test_vad_proportion_tie_is_decided_in_fp32():
    """15 voiced frames of 25 at p = 0.6: 25 * 0.6f = 15.000001 > 15, so the frame is unvoiced (the reference keeps the
    proportion in a float); a float64 product would say voiced"""
    e = np.zeros((25, 1), np.float32)
    e[:15, 0] = 9.0
    e[15:, 0] = 1.0
    got = ofe.vad_energy(e, 5.0, 0.0, 12, 0.6)
    assert got[12] == 0 and 15 >= 25 * 0.6
    assert fx.vad_ref(e[:, 0], 5.0, 0.0, 12, 0.6)[12] == 0
    assert fx.vad_ref(e[:, 0], 5.0, 0.0, 12, 0.5)[12] == 1


def test_cmn_catalogue_and_reference():
    cases = list(fx.cmn_cases().values())
    Fs = {c["F"] for c in cases}
    assert {fx.CMN_BLOCK_CAP - 1, fx.CMN_BLOCK_CAP, fx.CMN_BLOCK_CAP + 1, 1, 31, 32, 33} <= Fs and max(Fs) > 2 * fx.CMN_BLOCK_CAP
    ws = {c["window"] for c in cases}
    assert min(ws) < 0 and 0 in ws and {1, 2, 3, 8, 300} <= ws
    for w in ws:
        if w > 0:
            lens = fx.cmn_lens(w)
            assert {w - 1, w, w + 1, 3 * w} - {0} <= set(lens) and 0 in lens
    for name in ("w8_F33", "w3_F1", "w300_F31", "w0_F129", "w-3_F1"):
        case = fx.cmn_cases()[name]
        for u in fx.cmn_operands(case, name):
            k = u.astype(np.float64) * 8
            assert np.array_equal(k, np.round(k)) and np.abs(k).sum(axis=0).max() < 2 ** 45
            if not len(u):
                continue
            w = case["window"]
            want = ofe.cmn_sliding(u, w) if 0 < w < u.shape[0] else ofe.cmn_utterance(u)
            assert np.array_equal(fx.cmn_ref(u, w), want), (name, u.shape)


def test_select_catalogue():
    for name, case in fx.select_cases().items():
        utts, masks = fx.select_operands(case, name)
        lens = [u.shape[0] for u in utts]
        assert {1, 31, 32, 33, 64} <= set(lens) and max(lens) > 32 * 30 and lens[0] == 0 and lens[-1] == 0 and 0 in lens[1:-1]
    assert {c["mask"] for c in fx.select_cases().values()} >= {"all", "none", "alternating"}
    assert {c["F"] for c in fx.select_cases().values()} == {1, 80}


def test_fbank_catalogue_reaches_every_fft_size_and_option():
    cases = fx.fbank_cases()
    Ns = {}
    for name, c in cases.items():
        assert fx.kernel_geometry(c["size"], c["shift"]) == (c["size"], c["shift"]), name
        Ns.setdefault(fx.padded(c["size"]), set()).add(c["size"] - fx.padded(c["size"]))
    assert sorted(Ns) == [2 ** k for k in range(1, 13)]
    for N, offs in Ns.items():
        assert 0 in offs and (N == 2 or -N // 2 + 1 in offs or N - 1 <= 2)   # 2^k and 2^(k-1) + 1 land on N
    opts = [c["opts"] for c in cases.values()]
    assert {o["window_type"] for o in opts} == set(fx.WINDOWS)
    assert {o["preemphasis_coefficient"] for o in opts} >= {0.0, 1.0}
    for k in ("remove_dc_offset", "raw_energy", "use_energy", "htk_compat", "use_power", "use_log_fbank"):
        assert {bool(o[k]) for o in opts} == {False, True}, k
    assert {o["energy_floor"] for o in opts} == {0.0, 1.0}
    assert {o["num_mel_bins"] for o in opts} == set(fx.FBANK_MEL)
    ceps = {o["num_ceps"] for o in opts if o["num_ceps"]}
    assert {1, 13, 32, 33} <= ceps and any(o["num_ceps"] == o["num_mel_bins"] for o in opts)
    assert any(o["htk_compat"] and o["num_ceps"] and not o["use_energy"] for o in opts)
    assert any(o["htk_compat"] and o["num_ceps"] and o["use_energy"] for o in opts)
    assert any(o["htk_compat"] and not o["num_ceps"] and o["use_energy"] for o in opts)
    assert any(not o["htk_compat"] and not o["num_ceps"] and o["use_energy"] for o in opts)
    # bands without any FFT bin at small N; the M = 1 path
    W = ofe.kaldi_mel_banks(4, 4, 16000.0, 20.0, 0.0)
    assert not W[0].any()
    assert any(fx.padded(c["size"]) == 2 for c in cases.values())


def test_fbank_shared_slices_are_aligned_and_fit():
    for N in (2 ** k for k in range(1, 13)):
        assert fx.warp_floats(N) % 4 == 0 and fx.warp_floats(N) >= N + N // 2 + 4 + 128
    assert fx.FBANK_WARPS * fx.warp_floats(4096) * 4 == 200832 <= fx.FBANK_MAX_SMEM
    assert (2 + 1 + 4 + 128) % 4 != 0                       # N = 2 is the size the rounding exists for


def test_fbank_ragged_batches():
    cases = fx.fbank_cases()
    big = [n for n, c in cases.items() if c["utts"] >= 32]
    assert big
    for name, c in cases.items():
        lens = [w.shape[0] for w in fx.fbank_waves(c, name)]
        frames = [ofe.kaldi_num_frames(n, c["size"], c["shift"]) for n in lens]
        assert frames[0] == 0 and frames[-1] == 0 and 1 in frames and max(frames) > 1
        if c["utts"] == 5:
            assert 0 in frames[1:-1]


@pytest.mark.parametrize("name", sorted(fx.fbank_cases()))
def test_fbank_emulation_inside_bound(name):
    case = fx.fbank_cases()[name]
    worst = 0.0
    for w in fx.fbank_waves(case, name):
        ref = fx.fbank_ref(case, w)
        if not ref.shape[0]:
            continue
        em = fx.fbank_emulate(case, w)
        b = fx.fbank_bound(case, w)
        assert em.shape == ref.shape == b.shape
        err = np.abs(em - ref)
        assert np.all(err <= b), (name, float(np.max(err / np.where(b > 0, b, 1))))
        with np.errstate(divide="ignore", invalid="ignore"):
            worst = max(worst, float(np.max(np.where(err > 0, err / b, 0))))
    assert worst < 1.0


def test_each_fbank_mutant_leaves_the_bound_by_4x():
    caught = dict.fromkeys(fx.MUTANTS, 0.0)
    for name, case in fx.fbank_cases().items():
        for w in fx.fbank_waves(case, name):
            ref = fx.fbank_ref(case, w)
            if not ref.shape[0]:
                continue
            b = fx.fbank_bound(case, w)
            for m in fx.MUTANTS:
                err = np.abs(fx.fbank_emulate(case, w, m) - ref)
                with np.errstate(divide="ignore", invalid="ignore"):
                    r = np.where(err > 0, err / b, 0.0)
                caught[m] = max(caught[m], float(np.nanmax(r)))
    for m, r in caught.items():
        assert r >= 4.0, (m, r)
