"""Exact-arithmetic operands, case catalogue and float64 reference for the width-64 instance of the Res2Net chain kernel
(csrc/res2net.cu, xvb_res2net_block_ex with width = 64: ECAPA-TDNN C512, scale 8 x 64 channels).

The construction is tests/ecapa_exact.py's at width W = 64 instead of 128: x hi planes hold integers in [-2, 2] and lo
planes multiples of 2^-8; each weight plane of a step is +-1 on a signed cover of the 3 * W (tap, channel) K positions,
3 per output row (a balanced hi / lo pair past scale 8, so the chain stays below 2^15); bias and BN shift on the 2^-8
grid, BN scale +-1.  Every fp32 sum is then exact in any order (asserted for every output of every step), so the kernel
must match the reference bit for bit.  A dropped product term, a wrong tap, box or K offset, or a read of a chunk before
the previous step stored it moves an output by at least 2^-8.

Plain numpy (no torch, no GPU): test_gpu_res2net_w64_edges.py moves the operands to the device, and
test_ecapa_c512_host.py checks the helpers, the catalogue and the precondition of every case on the CPU."""
import numpy as np

import ecapa_exact as ex
import gemm_exact as gx

W = 64                   # Res2Net width: channels per chunk
K3 = 3 * W               # K positions of one step: 3 taps x 64 channels, tap-major (the packed weight layout)
CTAS_PER_SM = 1          # Res2Cfg<64>::kCtas in csrc/res2net.cu: a round of utterances is sms * CTAS_PER_SM


def cover_plane(rng):
    """(64, 192) float32 weight plane: +-1 on a random partition of the 192 K positions into 64 rows of 3."""
    w = np.zeros((W, K3), np.float32)
    cols = rng.permutation(K3).reshape(W, 3)
    w[np.arange(W)[:, None], cols] = rng.choice([-1.0, 1.0], (W, 3)).astype(np.float32)
    return w


def balanced_planes(rng):
    """(w_hi, w_lo) on one cover: w_lo = -w_hi on half of the rows, one sign kept on the others (ecapa_exact's rule)."""
    wh = cover_plane(rng)
    wl = -wh
    for r in np.nonzero(rng.rand(W) < 0.5)[0]:
        c = np.nonzero(wh[r])[0]
        wl[r, c[rng.randint(3)]] *= -1
    return wh, wl


def res2net_cases(sms):
    """name -> width-64 chain case for a GPU with `sms` SMs (the grid is min(B, sms * CTAS_PER_SM) CTAs, each owning
    utterances b = blockIdx.x, blockIdx.x + grid, ...)."""
    D = dict
    rnd = sms * CTAS_PER_SM
    cases = {}
    # T on both sides of the 64- and 128-frame edges (the A tile is 128 frames; 64 is one consumer warpgroup's half)
    for t in (1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257):
        cases["T{}".format(t)] = D(B=3, T=t, d=2, scale=8)
    cases["T3000_one_utt"] = D(B=1, T=3000, d=3, scale=8)
    # dilation 1 .. 5, side taps wholly outside the utterance (d >= T) and d > 128
    for d in (1, 2, 3, 4, 5):
        cases["d{}".format(d)] = D(B=2, T=140, d=d, scale=8)
    cases["d_T-1"] = D(B=3, T=50, d=49, scale=8)
    cases["d_T"] = D(B=3, T=50, d=50, scale=8)
    cases["d_T+7"] = D(B=2, T=30, d=37, scale=8)
    cases["d_T_T1"] = D(B=2, T=1, d=1, scale=4)
    cases["d130_T300"] = D(B=2, T=300, d=130, scale=8)
    cases["d200_T257"] = D(B=2, T=257, d=200, scale=4)
    # scale: C = scale * 64 and the weight map height; scale 2 is a single step with no second source
    for s in (2, 3, 4, 5, 12, 16):
        cases["scale{}".format(s)] = D(B=3, T=150, d=2, scale=s)
    # utterance rounds: several utterances per CTA carry the stage ring and the step_bar parity across utterances
    cases["B1"] = D(B=1, T=5, d=1, scale=8)
    cases["B_round-1"] = D(B=rnd - 1, T=5, d=1, scale=8)
    cases["B_round"] = D(B=rnd, T=5, d=2, scale=3)
    cases["B_round+1_scale2"] = D(B=rnd + 1, T=6, d=1, scale=2)
    cases["B_2round+1"] = D(B=2 * rnd + 1, T=7, d=2, scale=3)
    cases["B_2round+1_T130"] = D(B=2 * rnd + 1, T=130, d=3, scale=8)
    # the same block as scale - 1 layer-kernel calls must give the same bits
    for name in ("T129", "scale3", "B_2round+1"):
        cases[name]["layers"] = True
    for c in cases.values():
        C = c["scale"] * W
        c["C"] = C
        # x: the channel slice at 8 of a NaN buffer; y: a fenced slice at 16 of another pitch (both wider than C)
        c["x_c0"], c["ldx"] = 8, ex._ru(8 + C + 8, 8)
        c["y_c0"], c["ldy"] = 16, ex._ru(16 + C + 24, 8)
    return cases


def make_res2net(case, seed):
    """Operands: x planes (B, T, C), stacked weight planes ((scale-1) * 64, 192), per-step bias / scale / shift."""
    rng = np.random.RandomState(seed)
    B, T, C, S = case["B"], case["T"], case["C"], case["scale"] - 1
    x = gx.frame_planes(rng, (B, T, C))
    if case["scale"] > 8:
        w = [balanced_planes(rng) for _ in range(S)]
    else:
        w = [(cover_plane(rng), cover_plane(rng)) for _ in range(S)]
    return {"x": x, "w_hi": np.concatenate([a for a, _ in w]), "w_lo": np.concatenate([b for _, b in w]),
            "bias": gx.grid_values(rng, S * W, 1.0),
            "scale": rng.choice([-1.0, 1.0], S * W).astype(np.float32),
            "shift": gx.grid_values(rng, S * W, 1.0)}


def _splice(a, d):
    """(B, T, 64) -> (B * T, 192): frames t - d, t, t + d side by side, zero outside the utterance"""
    return np.concatenate([gx.shift_time(a, c) for c in (-d, 0, d)], axis=2).reshape(-1, K3).astype(np.float64)


def step_acc(srcs, wh, wl, d, drop=()):
    """float64 sum over sources and K of hi*w_hi + lo*w_hi + hi*w_lo -> (acc, sum |terms|), both (B * T, 64)."""
    wh64, wl64 = wh.astype(np.float64).T, wl.astype(np.float64).T
    acc = 0.0
    mag = 0.0
    for name, hi, lo in srcs:
        sh, sl = _splice(hi, d), _splice(lo, d)
        for term, a, w in (("hh", sh, wh64), ("lh", sl, wh64), ("hl", sh, wl64)):
            mag = mag + np.abs(a) @ np.abs(w)
            if (name, term) not in drop:
                acc = acc + a @ w
    return acc, mag


def res2net_reference(case, d, drop=()):
    """-> (y_hi, y_lo) float32 (B, T, C).  Asserts, for every output of every step, sum |terms| < 2^15."""
    B, T, C, dil = case["B"], case["T"], case["C"], case["d"]
    hx, lx = d["x"]
    yh, yl = np.zeros((B, T, C), np.float32), np.zeros((B, T, C), np.float32)
    yh[..., :W], yl[..., :W] = hx[..., :W], lx[..., :W]
    for st in range(case["scale"] - 1):
        r, k = slice(st * W, (st + 1) * W), slice((st + 1) * W, (st + 2) * W)
        srcs = [("x", hx[..., k], lx[..., k])]
        if st:
            srcs.append(("y", yh[..., r], yl[..., r]))
        acc, mag = step_acc(srcs, d["w_hi"][r], d["w_lo"][r], dil, drop)
        peak = float(mag.max())
        assert peak < gx.EXACT_SUM_LIMIT, "step {}: sum of |terms| reaches {} >= 2^15".format(st, peak)
        v = np.maximum(acc + d["bias"][r], 0.0) * d["scale"][r].astype(np.float64) + d["shift"][r]
        h, lo = gx.split_bf16(gx.exact_f32(v))
        yh[..., k], yl[..., k] = h.reshape(B, T, W), lo.reshape(B, T, W)
    return yh, yl
