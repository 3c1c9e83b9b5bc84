"""Oracle (NumPy) restatement of the feature-side front-end.  TEST INFRASTRUCTURE ONLY.

  vad_energy      : TorchAsvExtractor::ComputeVadEnergy, runtime/extractor/torch_asv_extractor.cc:14-62
  cmn_utterance   : `input_feats - input_feats.mean(0)`, torch_asv_extractor.cc:99-101
  select_voiced   : index_select(0, nonzero(vad)), torch_asv_extractor.cc:103-107
  cmn_sliding     : Kaldi apply-cmvn-sliding --norm-vars=false --center=true (call site
                    pytorch/pipeline/extract_xvectors_for_pytorch.sh:105-111).  PARITY UNPINNED: Kaldi is not
                    vendored; the window rule is restated from Kaldi's SlidingWindowCmn.
The C++ runtime cannot be built here (libtorch/gflags are fetched from the network), so these are
pinned by code reading only; the functions are a handful of lines each."""
import numpy as np


def vad_energy(feats, energy_threshold=5.0, energy_mean_scale=0.5, frames_context=0, proportion_threshold=0.6):
    T = feats.shape[0]
    log_energy = feats[:, 0].astype(np.float32)
    thr = np.float32(energy_threshold)
    if energy_mean_scale != 0.0:
        thr = np.float32(thr + np.float32(energy_mean_scale) * np.float32(log_energy.sum(dtype=np.float32)) / np.float32(T))
    out = np.zeros(T, dtype=np.uint8)
    for t in range(T):
        num = den = 0
        for t2 in range(t - frames_context, t + frames_context + 1):
            if 0 <= t2 < T:
                den += 1
                if log_energy[t2] > thr:
                    num += 1
        out[t] = 1 if np.float32(num) >= np.float32(den) * np.float32(proportion_threshold) else 0   # float, as the reference
    return out


def cmn_utterance(feats):
    return feats - feats.mean(axis=0, dtype=np.float64).astype(np.float32)


def cmn_sliding(feats, window=300):
    T = feats.shape[0]
    out = np.empty_like(feats)
    csum = np.concatenate([np.zeros((1, feats.shape[1])), np.cumsum(feats.astype(np.float64), axis=0)])
    for t in range(T):
        b = t - window // 2
        e = b + window
        if b < 0:
            e -= b
            b = 0
        if e > T:
            b -= e - T
            e = T
            if b < 0:
                b = 0
        out[t] = feats[t] - ((csum[e] - csum[b]) / (e - b)).astype(np.float32)
    return out


def select_voiced(feats, voiced):
    return feats[np.flatnonzero(voiced)]


# ---------------------------------------------------------------- Kaldi fbank / MFCC from waveforms
# The reference's online path computes features with `KaldiFeature` (pytorch/libs/egs/kaldi_features.py:
# 69-135), which calls torchaudio.compliance.kaldi.fbank / .mfcc (third-party, torchaudio 2.11.0 in this
# image) with the `kaldi_featset` of the run (runtime/test/feat_conf.yaml; launcher/runEcapaXvector_online.py
# :380-381 forces dither = 0.0) and then `InputSequenceNormalization` (:12-66).  Restated in float64 from
# torchaudio's published algorithm (_get_window, get_mel_banks, fbank, mfcc); pinned by tests/golden/fbank.npz,
# which is produced by the reference's own KaldiFeature (tests/golden/make_golden_fbank.py).
FBANK_DEFAULTS = dict(blackman_coeff=0.42, dither=0.0, energy_floor=1.0, frame_length=25.0, frame_shift=10.0,
                      high_freq=0.0, htk_compat=False, low_freq=20.0, num_mel_bins=23, preemphasis_coefficient=0.97,
                      raw_energy=True, remove_dc_offset=True, round_to_power_of_two=True, sample_frequency=16000.0,
                      snip_edges=True, use_energy=False, use_log_fbank=True, use_power=True, window_type="povey",
                      num_ceps=13, cepstral_lifter=22.0)
_EPS32 = float(np.finfo(np.float32).eps)


def _mel(f):
    return 1127.0 * np.log(1.0 + np.asarray(f, dtype=np.float64) / 700.0)


def kaldi_window(window_type, n, blackman_coeff=0.42):
    i = np.arange(n, dtype=np.float64)
    a = 2.0 * np.pi / (n - 1)
    if window_type == "hanning":
        return 0.5 - 0.5 * np.cos(a * i)
    if window_type == "hamming":
        return 0.54 - 0.46 * np.cos(a * i)
    if window_type == "povey":
        return (0.5 - 0.5 * np.cos(a * i)) ** 0.85
    if window_type == "rectangular":
        return np.ones(n)
    if window_type == "blackman":
        return blackman_coeff - 0.5 * np.cos(a * i) + (0.5 - blackman_coeff) * np.cos(2 * a * i)
    raise ValueError("Invalid window type " + window_type)


def kaldi_mel_banks(num_bins, padded, sample_freq, low_freq, high_freq):
    """get_mel_banks with vtln_warp = 1 -> (num_bins, padded/2 + 1), last column zero (fbank pads it)."""
    nyquist = 0.5 * sample_freq
    if high_freq <= 0.0:
        high_freq += nyquist
    assert 0.0 <= low_freq < nyquist and 0.0 < high_freq <= nyquist and low_freq < high_freq
    lo, hi = _mel(low_freq), _mel(high_freq)
    delta = (hi - lo) / (num_bins + 1)
    b = np.arange(num_bins, dtype=np.float64)[:, None]
    left, center, right = lo + b * delta, lo + (b + 1.0) * delta, lo + (b + 2.0) * delta
    mel = _mel(sample_freq / padded * np.arange(padded // 2))[None, :]
    bins = np.maximum(0.0, np.minimum((mel - left) / (center - left), (right - mel) / (right - center)))
    return np.pad(bins, ((0, 0), (0, 1)))


def kaldi_num_frames(num_samples, window_size, window_shift):
    return 0 if num_samples < window_size else 1 + (num_samples - window_size) // window_shift


def kaldi_fbank(wave, **kw):
    """torchaudio.compliance.kaldi.fbank on a 1-D waveform (snip_edges, dither 0, no VTLN) -> (m, bins[+1])."""
    o = dict(FBANK_DEFAULTS)
    o.update(kw)
    assert o["snip_edges"] and o["dither"] == 0.0 and o["round_to_power_of_two"]
    x = np.asarray(wave, dtype=np.float64).reshape(-1)
    sf = o["sample_frequency"]
    shift, size = int(sf * o["frame_shift"] * 0.001), int(sf * o["frame_length"] * 0.001)
    padded = 1 << (size - 1).bit_length()
    m = kaldi_num_frames(x.shape[0], size, shift)
    idx = np.arange(m)[:, None] * shift + np.arange(size)[None, :]
    fr = x[idx]
    if o["remove_dc_offset"]:
        fr = fr - fr.mean(axis=1, keepdims=True)

    def log_energy(z):
        e = np.log(np.maximum((z ** 2).sum(axis=1), _EPS32))
        return e if o["energy_floor"] == 0.0 else np.maximum(e, np.log(o["energy_floor"]))

    if o["raw_energy"]:
        energy = log_energy(fr)
    if o["preemphasis_coefficient"] != 0.0:
        prev = np.concatenate([fr[:, :1], fr[:, :-1]], axis=1)
        fr = fr - o["preemphasis_coefficient"] * prev
    fr = fr * kaldi_window(o["window_type"], size, o["blackman_coeff"])[None, :]
    fr = np.pad(fr, ((0, 0), (0, padded - size)))
    if not o["raw_energy"]:
        energy = log_energy(fr)
    spec = np.abs(np.fft.rfft(fr, axis=1))
    if o["use_power"]:
        spec = spec ** 2
    out = spec @ kaldi_mel_banks(o["num_mel_bins"], padded, sf, o["low_freq"], o["high_freq"]).T
    if o["use_log_fbank"]:
        out = np.log(np.maximum(out, _EPS32))
    if o["use_energy"]:
        out = np.concatenate([out, energy[:, None]] if o["htk_compat"] else [energy[:, None], out], axis=1)
    return out


def kaldi_mfcc(wave, **kw):
    """torchaudio.compliance.kaldi.mfcc: log-mel -> orthonormal DCT-II (first basis = sqrt(1/N)) -> lifter."""
    o = dict(FBANK_DEFAULTS)
    o.update(kw)
    nb, nc = o["num_mel_bins"], o["num_ceps"]
    assert nc <= nb
    fo = {k: v for k, v in o.items() if k not in ("num_ceps", "cepstral_lifter")}
    fo.update(use_log_fbank=True, use_power=True)
    feat = kaldi_fbank(wave, **fo)
    if o["use_energy"]:
        energy = feat[:, nb if o["htk_compat"] else 0]
        off = 0 if o["htk_compat"] else 1
        feat = feat[:, off:off + nb]
    n = np.arange(nb, dtype=np.float64)[:, None]
    k = np.arange(nb, dtype=np.float64)[None, :]
    dct = np.cos(np.pi / nb * (n + 0.5) * k) * np.sqrt(2.0 / nb)     # torchaudio.functional.create_dct(.., 'ortho')
    dct[:, 0] = np.sqrt(1.0 / nb)
    feat = feat @ dct[:, :nc]
    if o["cepstral_lifter"] != 0.0:
        i = np.arange(nc, dtype=np.float64)
        feat = feat * (1.0 + 0.5 * o["cepstral_lifter"] * np.sin(np.pi * i / o["cepstral_lifter"]))[None, :]
    if o["use_energy"]:
        feat[:, 0] = energy
    if o["htk_compat"]:
        e = feat[:, :1] * (1.0 if o["use_energy"] else np.sqrt(2.0))
        feat = np.concatenate([feat[:, 1:], e], axis=1)
    return feat


def sequence_normalize(feats, mean_norm=True, std_norm=False):
    """InputSequenceNormalization, kaldi_features.py:39-66 (torch.std is unbiased; floor 1e-10)."""
    x = np.asarray(feats, dtype=np.float64)
    mean = x.mean(axis=0) if mean_norm else 0.0
    std = np.maximum(x.std(axis=0, ddof=1), 1e-10) if std_norm else 1.0
    return (x - mean) / std


def synthetic_wave(num_samples, seed, scale=3000.0, sample_frequency=16000.0):
    """Deterministic speech-like test signal: a few drifting tones + noise + DC offset, Kaldi (int16) scale."""
    rng = np.random.RandomState(seed)
    t = np.arange(num_samples, dtype=np.float64) / sample_frequency
    x = np.zeros(num_samples)
    for _ in range(5):
        f0, am = rng.uniform(80, 3500), rng.uniform(0.2, 1.0)
        x += am * np.sin(2 * np.pi * (f0 * t + rng.uniform(20, 200) * t * t) + rng.uniform(0, 6.28))
    x = x * (0.6 + 0.4 * np.sin(2 * np.pi * 3.1 * t)) + 0.3 * rng.standard_normal(num_samples) + 0.05
    return (scale * x).astype(np.float32)
