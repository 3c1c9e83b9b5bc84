"""Case catalogue, exact operands, references and bounds for the feature front end: energy VAD, CMN and voiced-frame
selection (csrc/frontend.cu), and the one-warp-per-frame fbank / MFCC (csrc/fbank.cu).

VAD.  Log energies are multiples of 2^-4 well below 2^19, so the kernel's fp32 sum of them is exact in any order, and the
threshold threshold + mean_scale * sum / T rounds the same in numpy fp32.  Utterances carry energies equal to the
threshold (the comparison is strict) and windows whose proportion ties in real arithmetic (15 of 25 at p = 0.6): there
the fp32 product 25 * 0.6f = 15.000001 decides, as in the reference and the kernel.  Decisions and counts are exact.
CMN.  Features are multiples of 2^-3 below 2^12: every fp64 window sum is exact, so fl32(s / n) is the kernel's mean.
Select.  A copy: exact.

fbank.  Checked against the float64 oracle (oracle/frontend.kaldi_fbank / kaldi_mfcc) within `fbank_bound`, derived once
per frame from the operation count: the fp32 roundings before the FFT, an FFT error of FFT_C (log2 N + 2) u per bin on
the scale ||y||_2 sqrt(N), then |X_k|^2 (or |X_k|), the fp32 mel weights with their sequential fmaf sum, log(max(., eps)),
the DCT and the lifter.  `fbank_emulate` is a numpy fp32 restatement of the kernel (the half-size complex DIF FFT with
fp32 twiddles and the bit-reversed even / odd recombination) that stays inside the bound; its mutants (a twiddle index
without the stage stride, the half-size transform's Nyquist bin Z[M/2] dropped, the mel start off by one, the energy
column swapped, c0 without sqrt 2 under htk_compat) leave it.

Plain numpy (no torch, no GPU)."""
import zlib

import numpy as np

from oracle import frontend as ofe

U32 = 2.0 ** -24
EPS32 = float(np.finfo(np.float32).eps)
VAD_THREADS = 256
CMN_BLOCK_CAP = 128
FBANK_MAX_SMEM = 200 * 1024
FBANK_WARPS = 8


def rng_for(name):
    return np.random.RandomState(zlib.crc32(name.encode()) & 0x7FFFFFFF)


def f32(a):
    return np.asarray(a, dtype=np.float32)


# ------------------------------------------------------------------------------------------------ VAD
VAD_T = (1, 2, 255, 256, 257, 1000)
VAD_THRESHOLD = 5.5


def vad_cases():
    """context 0, 1, 5 and >= T; mean_scale 0 and 0.5; proportions 0.6 (ties 15 / 25 at context 12) and 0.5 (exact ties
    num = den / 2 are voiced).  Every case holds every T of VAD_T with an empty utterance between two others."""
    cases = {}
    for ctx in (0, 1, 5, 12, 1000):
        for scale in (0.0, 0.5):
            for prop in (0.6, 0.5):
                cases["c{}_s{}_p{}".format(ctx, scale, prop)] = dict(context=ctx, scale=scale, prop=prop)
    return cases


def vad_operands(case, name, F=3):
    """(lens, feats list) with the energy column on the 2^-4 grid and the other columns NaN.  With mean_scale 0.5 the last
    frame makes the sum T m with m on the grid, so the threshold is exact and frames can equal it."""
    rng = rng_for("vad" + name)
    lens = list(VAD_T[:3]) + [0] + list(VAD_T[3:])
    utts = []
    for T in lens:
        m = rng.randint(20, 70) / 8.0                         # 0.5 m stays on the 2^-4 grid
        thr = VAD_THRESHOLD + case["scale"] * m
        e = rng.randint(0, 200, T) / 16.0
        e[rng.rand(T) < 0.25] = thr                        # exactly at the threshold: unvoiced
        if T and case["scale"]:
            e[-1] = T * m - e[:-1].sum()
        f = np.full((T, F), np.nan, np.float32)
        f[:, 0] = e
        utts.append(f)
    return lens, utts


def vad_threshold(e, threshold, scale):
    T = e.shape[0]
    thr = np.float32(threshold)
    if scale != 0.0 and T:
        thr = np.float32(thr + np.float32(scale) * np.float32(e.astype(np.float64).sum()) / np.float32(T))
    return thr


def vad_ref(e, threshold, scale, context, prop):
    """vectorised fp32 restatement of the kernel (== oracle.frontend.vad_energy)"""
    T = e.shape[0]
    thr = vad_threshold(e, threshold, scale)
    above = np.concatenate([[0], np.cumsum(e > thr)])
    t = np.arange(T)
    lo, hi = np.maximum(t - context, 0), np.minimum(t + context + 1, T)
    num, den = above[hi] - above[lo], hi - lo
    return (f32(num) >= f32(den) * np.float32(prop)).astype(np.uint8)


def vad_exact(e):
    """the energies are on the 2^-4 grid and their sum stays far inside fp32's 24 bits"""
    k = e.astype(np.float64) * 16
    return bool(np.array_equal(k, np.round(k)) and np.abs(k).sum() < 2 ** 23)


# ------------------------------------------------------------------------------------------------ CMN
CMN_F = (1, 31, 32, 33, 127, 128, 129, 300)
CMN_W = (0, -3, 1, 2, 3, 8, 300)


def cmn_cases():
    """every window with every F; each case holds utterances of T = 0, 1, W - 1, W, W + 1, 2 W + 1 and 3 W frames"""
    return {"w{}_F{}".format(w, F): dict(window=w, F=F) for w in CMN_W for F in CMN_F}


def cmn_lens(w):
    if w <= 0:
        return [1, 0, 7, 40]
    return sorted({1, max(w - 1, 1), w, w + 1, 2 * w + 1, 3 * w}) + [0, 2]


def cmn_operands(case, name):
    rng = rng_for("cmn" + name)
    return [f32(rng.randint(-16000, 16001, (T, case["F"])) / 8.0) for T in cmn_lens(case["window"])]


def cmn_ref(x, window):
    """the kernel's window rule with exact fp64 sums (integers / 8): fl32(fl64(s / n)) subtracted in fp32"""
    T = x.shape[0]
    if window <= 0 or window >= T:
        return x - f32(x.astype(np.float64).sum(axis=0) / T) if T else x.copy()
    c = np.concatenate([np.zeros((1, x.shape[1])), np.cumsum(x.astype(np.float64), axis=0)])
    out = np.empty_like(x)
    for t in range(T):
        b = t - window // 2
        e = b + window
        if b < 0:
            e -= b
            b = 0
        if e > T:
            b -= e - T
            e = T
            b = max(b, 0)
        out[t] = x[t] - f32((c[e] - c[b]) / (e - b))
    return out


# ------------------------------------------------------------------------------------------------ select
SELECT_T = (1, 31, 32, 33, 64, 1000)


def select_cases():
    return {"{}_F{}".format(m, F): dict(mask=m, F=F) for m in ("all", "none", "alternating", "random") for F in (1, 80)}


def select_operands(case, name):
    rng = rng_for("sel" + name)
    lens = [0] + list(SELECT_T[:3]) + [0] + list(SELECT_T[3:]) + [0]
    utts, masks = [], []
    for T in lens:
        utts.append(f32(rng.standard_normal((T, case["F"]))))
        m = {"all": np.ones(T), "none": np.zeros(T), "alternating": np.arange(T) % 2,
             "random": rng.rand(T) < 0.5}[case["mask"]]
        masks.append(np.asarray(m, np.uint8))
    return utts, masks


# ------------------------------------------------------------------------------------------------ fbank
WINDOWS = ("povey", "hamming", "hanning", "rectangular", "blackman")
FBANK_MEL = (4, 23, 31, 32, 33, 80, 128)


def fbank_sizes():
    out = []
    for k in range(1, 13):
        for s in (2 ** k - 1, 2 ** k, 2 ** k + 1):
            if 2 <= s <= 4096 and s not in out:
                out.append(s)
    return out


def padded(size):
    return 1 << (size - 1).bit_length()


def warp_floats(N):
    """shared floats per warp (fbank_warp_floats): 16-byte aligned"""
    return (N + (N // 2 + 4) + 128 + 3) & ~3


def kernel_geometry(size, shift):
    """(window, shift) as xvb_fbank_create computes them in fp32 from frame_length_ms = size / 16 at 16 kHz"""
    def g(n):
        return int(np.float32(np.float32(16000.0) * np.float32(n / 16.0)) * np.float32(0.001))
    return g(size), g(shift)


def fbank_cases():
    """every window size 2^k - 1, 2^k, 2^k + 1 in [2, 4096] (every FFT size N = 2 .. 4096), the options cycling over the
    catalogue: window type, pre-emphasis 0 / 0.97 / 1, remove_dc, raw_energy, energy floor 0 / 1, use_energy, htk_compat,
    use_power off, use_log off, MFCC with num_ceps in {1, 13, 32, 33, num_mel}; plus one ragged batch of 37 utterances."""
    cases = {}
    for i, size in enumerate(fbank_sizes()):
        nm = FBANK_MEL[i % len(FBANK_MEL)]
        mfcc = i % 3 == 1
        choices = [c for c in (1, 13, 32, 33, nm) if c <= nm]
        ceps = choices[(i // 3) % len(choices)]
        o = dict(window_type=WINDOWS[i % 5], preemphasis_coefficient=(0.97, 0.0, 1.0)[i % 3],
                 remove_dc_offset=bool(i % 4 != 3), raw_energy=bool(i % 2), energy_floor=(1.0, 0.0)[(i // 2) % 2],
                 use_energy=bool(i % 4 in (1, 2)), htk_compat=bool((i // 4) % 2), num_mel_bins=nm,
                 use_power=not (not mfcc and i % 5 == 4), use_log_fbank=not (not mfcc and i % 7 == 5),
                 num_ceps=ceps if mfcc else 0, cepstral_lifter=(22.0, 0.0)[(i // 5) % 2])
        cases["s{}_{}".format(size, "mfcc" if mfcc else "fbank")] = dict(size=size, shift=max(1, size // 2), opts=o, utts=5)
    cases["ragged37_s400"] = dict(size=400, shift=160, utts=37,
                                  opts=dict(window_type="povey", preemphasis_coefficient=0.97, remove_dc_offset=True,
                                            raw_energy=True, energy_floor=0.0, use_energy=True, htk_compat=False,
                                            num_mel_bins=80, use_power=True, use_log_fbank=True, num_ceps=0,
                                            cepstral_lifter=22.0))
    return cases


def fbank_waves(case, name):
    """utterance lengths: empty first, in the middle and last; exactly one frame; a few frames; one frame short of two"""
    rng = rng_for("fb" + name)
    size, shift = case["size"], case["shift"]
    if case["utts"] == 5:
        lens = [0, size, size + 3 * shift + 1, size - 1, size + 2 * shift - 1, 0]
    else:
        lens = [[0, size, size + rng.randint(0, 9) * shift][rng.randint(0, 3)] for _ in range(case["utts"])]
        lens[0] = lens[-1] = 0
    return [ofe.synthetic_wave(n, int(rng.randint(1 << 30)), scale=float(rng.choice([1.0, 3000.0])))
            if n else np.zeros(0, np.float32) for n in lens]


def oracle_kw(case):
    o = dict(case["opts"])
    kw = dict(frame_length=case["size"] / 16.0, frame_shift=case["shift"] / 16.0, sample_frequency=16000.0, **o)
    return kw


def fbank_ref(case, wave):
    kw = oracle_kw(case)
    if kw["num_ceps"]:
        return ofe.kaldi_mfcc(wave, **kw)
    kw = {k: v for k, v in kw.items() if k not in ("num_ceps", "cepstral_lifter")}
    return ofe.kaldi_fbank(wave, **kw)


FFT_C = 6.0          # per-stage error of a radix-2 butterfly with fp32 twiddles, in u, on the L2 scale
LOG_ULPS = 2.0       # logf in ulps of its result


def _frames(case, wave):
    size, shift = case["size"], case["shift"]
    m = ofe.kaldi_num_frames(wave.shape[0], size, shift)
    idx = np.arange(m)[:, None] * shift + np.arange(size)[None, :]
    return wave.astype(np.float64)[idx]


def _log_err(val, err, eps=EPS32):
    """bound on |log(max(a, eps)) - log(max(val, eps))| for |a - val| <= err, plus the logf rounding"""
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.log(np.maximum(val, eps))
        e = np.maximum(np.log(np.maximum(val + err, eps)) - c, c - np.log(np.maximum(val - err, eps)))
    return e + LOG_ULPS * np.spacing(np.abs(f32(c))).astype(np.float64)


def fbank_bound(case, wave):
    """(frames, dim) bound on |kernel - float64 oracle| (see the module docstring)"""
    o = case["opts"]
    size = case["size"]
    N = padded(size)
    x = _frames(case, wave)
    if x.shape[0] == 0:
        return np.zeros((0, 1))
    p = o["preemphasis_coefficient"]
    depth = -(-size // 32) + 6
    mean = x.mean(axis=1, keepdims=True) if o["remove_dc_offset"] else np.zeros((x.shape[0], 1))
    e_mean = depth * U32 * np.abs(x).mean(axis=1, keepdims=True) if o["remove_dc_offset"] else 0.0
    v = x - mean
    e_v = e_mean + U32 * np.abs(v)
    vp = np.concatenate([v[:, :1], v[:, :-1]], axis=1)
    e_vp = np.concatenate([e_v[:, :1], e_v[:, :-1]], axis=1)
    w = np.abs(ofe.kaldi_window(o["window_type"], size))[None, :]
    y = (v - p * vp) * w
    e_y = w * (e_v + p * e_vp + 4 * U32 * (np.abs(v) + p * np.abs(vp)))
    ypad = np.pad(y, ((0, 0), (0, N - size)))
    X = np.abs(np.fft.rfft(ypad, axis=1))
    e_X = e_y.sum(axis=1, keepdims=True) + FFT_C * (np.log2(N) + 2) * U32 * np.sqrt(N) * np.sqrt((y ** 2).sum(axis=1, keepdims=True))
    if o["use_power"] or o["num_ceps"]:
        P, e_P = X ** 2, 2 * X * e_X + e_X ** 2 + 3 * U32 * X ** 2
    else:
        P, e_P = X, e_X + 2 * U32 * X
    nm = o["num_mel_bins"]
    W = ofe.kaldi_mel_banks(nm, N, 16000.0, 20.0, 0.0)
    lens = np.array([(np.ptp(np.flatnonzero(r)) + 1) if r.any() else 0 for r in W])
    acc = P @ W.T
    e_acc = (e_P + U32 * P) @ W.T + (lens[None, :] + 1) * U32 * acc
    if o["use_log_fbank"] or o["num_ceps"]:
        lm, e_lm = np.log(np.maximum(acc, EPS32)), _log_err(acc, e_acc)
    else:
        lm, e_lm = acc, e_acc
    # log energy
    if o["raw_energy"]:
        E, e_E = (v ** 2).sum(axis=1), (2 * np.abs(v) * e_v).sum(axis=1) + depth * U32 * (v ** 2).sum(axis=1)
    else:
        E, e_E = (y ** 2).sum(axis=1), (2 * np.abs(y) * e_y).sum(axis=1) + depth * U32 * (y ** 2).sum(axis=1)
    e_en = _log_err(E, e_E)
    if o["num_ceps"]:
        nc = o["num_ceps"]
        n = np.arange(nm)[:, None]
        k = np.arange(nc)[None, :]
        dct = np.abs(np.where(k == 0, np.sqrt(1.0 / nm), np.cos(np.pi / nm * (n + 0.5) * k) * np.sqrt(2.0 / nm)))
        lift = (1.0 + 0.5 * o["cepstral_lifter"] * np.sin(np.pi * np.arange(nc) / o["cepstral_lifter"])) if o["cepstral_lifter"] else np.ones(nc)
        mag = np.abs(lm) @ dct
        e_c = (e_lm @ dct + (nm + 2) * U32 * mag) * np.abs(lift)[None, :] + 2 * U32 * mag * np.abs(lift)[None, :]
        if o["use_energy"]:
            e_c[:, 0] = e_en
        if o["htk_compat"]:
            c0 = e_c[:, :1] * (1.0 if o["use_energy"] else np.sqrt(2.0)) + (0 if o["use_energy"] else 2 * U32 * mag[:, :1] * np.sqrt(2) * lift[0])
            e_c = np.concatenate([e_c[:, 1:], c0], axis=1)
        return e_c
    out = e_lm
    if o["use_energy"]:
        out = np.concatenate([out, e_en[:, None]] if o["htk_compat"] else [e_en[:, None], out], axis=1)
    return out


# fp32 emulation of fbank_kernel
def _tables(case):
    o = case["opts"]
    size = case["size"]
    N = padded(size)
    M = N // 2
    k = np.arange(max(M // 2, 1))
    twm = (f32(np.cos(-2 * np.pi * k / M)), f32(np.sin(-2 * np.pi * k / M)))
    k = np.arange(M + 1)
    twn = (f32(np.cos(-2 * np.pi * k / N)), f32(np.sin(-2 * np.pi * k / N)))
    W = f32(ofe.kaldi_mel_banks(o["num_mel_bins"], N, 16000.0, 20.0, 0.0)[:, :M])
    return N, M, twm, twn, W


def _bitrev(k, bits):
    out = np.zeros_like(k)
    for b in range(bits):
        out |= ((k >> b) & 1) << (bits - 1 - b)
    return out


MUTANTS = ("twiddle_stride", "half_nyquist", "mel_start", "energy_column", "htk_sqrt2")


def fbank_emulate(case, wave, mutant=None):
    """numpy fp32 restatement of fbank_kernel for one utterance -> (frames, dim) float32"""
    o = case["opts"]
    size = case["size"]
    N, M, twm, twn, W = _tables(case)
    x = f32(_frames(case, f32(wave)))
    T = x.shape[0]
    nm, nc = o["num_mel_bins"], o["num_ceps"]
    dim = nc if nc else nm + (1 if o["use_energy"] else 0)
    if T == 0:
        return np.zeros((0, dim), np.float32)
    one = np.float32(1.0)
    mean = (x.sum(axis=1, dtype=np.float32) / np.float32(size))[:, None] if o["remove_dc_offset"] else np.float32(0)
    v = x - mean
    energy = (v * v).sum(axis=1, dtype=np.float32)
    win = f32(ofe.kaldi_window(o["window_type"], size))
    vp = np.concatenate([v[:, :1], v[:, :-1]], axis=1)
    y = (v - np.float32(o["preemphasis_coefficient"]) * vp) * win[None, :]
    if not o["raw_energy"]:
        energy = (y * y).sum(axis=1, dtype=np.float32)
    log_floor = np.float32(-np.inf) if o["energy_floor"] == 0 else np.float32(np.log(np.float32(o["energy_floor"])))
    log_energy = np.maximum(np.log(np.maximum(energy, np.float32(EPS32))), log_floor)
    yp = np.zeros((T, N), np.float32)
    yp[:, :size] = y
    zr, zi = yp[:, 0::2].copy(), yp[:, 1::2].copy()
    h, tstep = M >> 1, 1
    while h >= 1:
        j = np.arange(M >> 1)
        pos = j & (h - 1)
        i0 = ((j - pos) << 1) + pos
        i1 = i0 + h
        ti = pos if mutant == "twiddle_stride" else pos * tstep
        wr, wi = twm[0][ti], twm[1][ti]
        ar, ai, br, bi = zr[:, i0], zi[:, i0], zr[:, i1], zi[:, i1]
        dx, dy = ar - br, ai - bi
        zr[:, i0], zi[:, i0] = ar + br, ai + bi
        zr[:, i1], zi[:, i1] = dx * wr - dy * wi, dx * wi + dy * wr
        h >>= 1
        tstep <<= 1
    log2m = M.bit_length() - 1
    if mutant == "half_nyquist" and M >= 2:
        zr[:, 1] = zi[:, 1] = 0                              # Z[M/2] sits at bitrev(M/2) = 1
    k = np.arange(M + 1)
    k0, k1 = k & (M - 1), (M - k) & (M - 1)
    ia, ic = (_bitrev(k0, log2m), _bitrev(k1, log2m)) if log2m else (k0 * 0, k1 * 0)
    half = np.float32(0.5)
    ax, ay, cx, cy = zr[:, ia], zi[:, ia], zr[:, ic], zi[:, ic]
    ex, ey = half * (ax + cx), half * (ay - cy)
    ox, oy = half * (ay + cy), np.float32(-0.5) * (ax - cx)
    xr = ex + (twn[0] * ox - twn[1] * oy)
    xi = ey + (twn[0] * oy + twn[1] * ox)
    P = xr * xr + xi * xi
    if not o["use_power"]:
        P = np.sqrt(P)
    if mutant == "mel_start":
        P = np.concatenate([P[:, 1:], np.zeros((T, 1), np.float32)], axis=1)
    acc = np.zeros((T, nm), np.float32)
    for j in range(M):
        acc = acc + W[:, j][None, :] * P[:, j:j + 1]
    if o["use_log_fbank"]:
        acc = np.log(np.maximum(acc, np.float32(EPS32)))
    htk = o["htk_compat"]
    if not nc:
        if not o["use_energy"]:
            return acc
        if mutant == "energy_column":
            htk = not htk
        return np.concatenate([acc, log_energy[:, None]] if htk else [log_energy[:, None], acc], axis=1)
    n = np.arange(nm)[:, None]
    kk = np.arange(nc)[None, :]
    dct = f32(np.where(kk == 0, np.sqrt(1.0 / nm), np.cos(np.pi / nm * (n + 0.5) * kk) * np.sqrt(2.0 / nm)))
    L = o["cepstral_lifter"]
    lift = f32((1.0 + 0.5 * L * np.sin(np.pi * np.arange(nc) / L)) if L else np.ones(nc))
    c = np.zeros((T, nc), np.float32)
    for b in range(nm):
        c = c + acc[:, b:b + 1] * dct[b][None, :]
    c = c * lift[None, :]
    if o["use_energy"]:
        c[:, 0] = log_energy
    if htk:
        c0 = c[:, :1] if (o["use_energy"] or mutant == "htk_sqrt2") else c[:, :1] * np.float32(1.41421356237309515)
        c = np.concatenate([c[:, 1:], c0], axis=1)
    return c
