"""Exact-arithmetic operands, case catalogue and float64 references for the ECAPA-TDNN block kernels: the one-kernel
Res2Net chain (csrc/res2net.cu, xvb_res2net_block), the SE gate and segment gate (csrc/ecapa.cu, xvb_se_apply and
xvb_seg_gate_apply) and the segment-level fp32 affine (csrc/ecapa.cu, xvb_small_affine).

Res2Net chain.  Step st (0 .. scale-2) of the block computes
    y[st+1] = BN(ReLU(W_st * splice(x[st+1], [-d, 0, d]) + [st >= 1] W_st * splice(y[st], [-d, 0, d]) + b_st))
from bf16 planes: hi*w_hi + lo*w_hi + hi*w_lo of both sources into fp32 accumulators, and stores y[st+1] as split_bf16
planes that step st+1 reads back.  The operands keep every step exact in fp32:
  * x: hi planes hold integers in [-2, 2], lo planes multiples of 2^-8 in +-3 * 2^-8;
  * W_st: both planes hold +-1 on a signed sparse cover of the 384 (tap, channel) K positions (every position feeds
    exactly one output row of each plane), so a swizzle, K-offset or tap mistake cannot hide behind zero weights.  Up to
    scale 8 the two planes are independent covers.  Each row then sums about six hi terms of the previous step's output,
    and the chain grows by about 1.9x per step, past 2^15 by step 14.  So at scale 12 and 16 the lo plane shares the hi
    plane's partition and cancels it (w_lo = -w_hi) on half of the rows and on two of the three positions of the others:
    hi * (w_hi + w_lo) vanishes there, but each of the three products still moves the output when it is dropped,
    misplaced or read from the wrong tap;
  * bias and BN shift are on the 2^-8 grid, BN scale is +-1.
Every product is then a multiple of 2^-8: a step's output v is on the 2^-8 grid, and so are both planes of
split_bf16(v) (hi = rn(v) rounds to a grid at least as coarse as 2^-8 unless v is exact in bf16, and lo = rn(v - hi)
likewise).  As long as the sum of |terms| of every output stays below 2^15 (asserted for every output of every step) the
fp32 sums are exact in any order, and the reference models the split of each step's output exactly (gemm_exact.split_bf16)
before feeding it to the next step.  A dropped product term, a wrong tap or K offset, a read of a chunk before the
previous step stored it or a step-index mix-up of the epilogue terms moves an output by at least 2^-8.

SE gate kernels.  out = z * g + in is computed as two fp32 roundings (multiply, then add), and next = out + in as one;
both are stored as split_bf16 planes.  The reference is float32 numpy, which rounds each operation once, so the
comparison is bit for bit on arbitrary (normal) data.

Small affine.  x on the 2^-8 grid with |x| <= 2, W small integers: with K <= 3072 every FMA chain stays a multiple of
2^-8 below 2^15 and is exact in any order; bias, ReLU and BN with power-of-two scales keep the epilogue exact; sigmoid and
tanh are within the bounds derived in gemm_exact.layer_reference.

Plain numpy (no torch, no GPU): test_gpu_ecapa_edges.py moves these operands to the device, and test_ecapa_exact_host.py
checks the helpers, the catalogue and the precondition of every case on the CPU."""
import numpy as np

import gemm_exact as gx

RW = 128                 # Res2Net width: channels per chunk
K3 = 3 * RW              # K positions of one step: 3 taps x 128 channels, tap-major (the packed weight layout)


def _ru(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ Res2Net chain
def cover_plane(rng):
    """(128, 384) float32 weight plane: +-1 on a random partition of the 384 K positions into 128 rows of 3."""
    w = np.zeros((RW, K3), np.float32)
    cols = rng.permutation(K3).reshape(RW, 3)
    w[np.arange(RW)[:, None], cols] = rng.choice([-1.0, 1.0], (RW, 3)).astype(np.float32)
    return w


def balanced_planes(rng):
    """(w_hi, w_lo) on one cover: w_lo = -w_hi on half of the rows; on the others it keeps the sign of w_hi at one of
    the row's three positions and flips it at the other two."""
    wh = cover_plane(rng)
    wl = -wh
    for r in np.nonzero(rng.rand(RW) < 0.5)[0]:
        c = np.nonzero(wh[r])[0]
        wl[r, c[rng.randint(3)]] *= -1
    return wh, wl


def res2net_cases(sms):
    """name -> Res2Net chain case for a GPU with `sms` SMs (the grid is min(B, sms) CTAs, each owning utterances
    b = blockIdx.x, blockIdx.x + grid, ...)."""
    D = dict
    cases = {}
    # T on both sides of the 128-frame tile edges; the long utterance is 24 tiles through one CTA
    for t in (1, 2, 127, 128, 129, 255, 256, 257):
        cases["T{}".format(t)] = D(B=3, T=t, d=2, scale=8)
    cases["T3000_one_utt"] = D(B=1, T=3000, d=3, scale=8)
    # dilation: 1 .. 5, side taps wholly outside the utterance (d = T - 1 reaches one frame, d = T none), and d > 128
    for d in (1, 2, 3, 4, 5):
        cases["d{}".format(d)] = D(B=2, T=140, d=d, scale=8)
    cases["d_T-1"] = D(B=3, T=50, d=49, scale=8)
    cases["d_T"] = D(B=3, T=50, d=50, scale=8)
    cases["d_T_T1"] = D(B=2, T=1, d=1, scale=4)
    cases["d130_T300"] = D(B=2, T=300, d=130, scale=8)
    cases["d200_T257"] = D(B=2, T=257, d=200, scale=4)
    # scale: C = scale * 128 and the weight map height; scale 2 is a single step with no second source
    for s in (2, 3, 4, 12, 16):
        cases["scale{}".format(s)] = D(B=3, T=150, d=2, scale=s)
    # utterance rounds: several utterances per CTA carry the stage ring and the step_bar parity across utterances
    cases["B1"] = D(B=1, T=5, d=1, scale=8)
    cases["B_sms-1"] = D(B=sms - 1, T=5, d=1, scale=8)
    cases["B_sms"] = D(B=sms, T=5, d=2, scale=3)
    cases["B_sms+1_scale2"] = D(B=sms + 1, T=6, d=1, scale=2)
    cases["B_2sms+1"] = D(B=2 * sms + 1, T=7, d=2, scale=3)
    cases["B_2sms+1_T130"] = D(B=2 * sms + 1, T=130, d=3, scale=4)
    # the same block as scale - 1 layer-kernel calls must give the same bits
    for name in ("T129", "scale3", "B_2sms+1"):
        cases[name]["layers"] = True
    for c in cases.values():
        C = c["scale"] * RW
        c["C"] = C
        # x: the channel slice at 8 of a NaN buffer; y: a fenced slice at 16 of another pitch
        c["x_c0"], c["ldx"] = 8, _ru(8 + C + 8, 8)
        c["y_c0"], c["ldy"] = 16, _ru(16 + C + 24, 8)
        assert c["ldx"] != c["ldy"]
    return cases


def make_res2net(case, seed):
    """Operands of a Res2Net case: x planes (B, T, C), stacked weight planes ((scale-1) * 128, 384) and per-step
    bias / scale / shift ((scale-1) * 128,)."""
    rng = np.random.RandomState(seed)
    B, T, C, S = case["B"], case["T"], case["C"], case["scale"] - 1
    x = gx.frame_planes(rng, (B, T, C))
    if case["scale"] > 8:
        w = [balanced_planes(rng) for _ in range(S)]
    else:
        w = [(cover_plane(rng), cover_plane(rng)) for _ in range(S)]
    return {"x": x, "w_hi": np.concatenate([a for a, _ in w]), "w_lo": np.concatenate([b for _, b in w]),
            "bias": gx.grid_values(rng, S * RW, 1.0),
            "scale": rng.choice([-1.0, 1.0], S * RW).astype(np.float32),
            "shift": gx.grid_values(rng, S * RW, 1.0)}


def _splice(a, d):
    """(B, T, 128) -> (B * T, 384): frames t - d, t, t + d side by side, zero outside the utterance"""
    return np.concatenate([gx.shift_time(a, c) for c in (-d, 0, d)], axis=2).reshape(-1, K3).astype(np.float64)


def res2net_step_acc(srcs, wh, wl, d, drop=()):
    """float64 sum over sources and K of hi*w_hi + lo*w_hi + hi*w_lo -> ((B * T, 128) acc, (B * T, 128) sum |terms|).
    srcs: [(name, hi, lo)] with name 'x' or 'y'; drop: (name, term) pairs left out, term in 'hh', 'lh', 'hl'."""
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
    """-> (y_hi, y_lo) float32 (B, T, C): the block output planes.  Chunk 0 is x's chunk 0; chunk st+1 is split_bf16 of
    step st's output.  Asserts, for every output of every step, that the sum of |terms| is below 2^15 and that the
    epilogue value is exact in fp32.  drop: product terms to leave out (test_ecapa_exact_host.py shows each matters)."""
    B, T, C, dil = case["B"], case["T"], case["C"], case["d"]
    hx, lx = d["x"]
    yh, yl = np.zeros((B, T, C), np.float32), np.zeros((B, T, C), np.float32)
    yh[..., :RW], yl[..., :RW] = hx[..., :RW], lx[..., :RW]
    for st in range(case["scale"] - 1):
        r, k = slice(st * RW, (st + 1) * RW), slice((st + 1) * RW, (st + 2) * RW)
        srcs = [("x", hx[..., k], lx[..., k])]
        if st:
            srcs.append(("y", yh[..., r], yl[..., r]))
        acc, mag = res2net_step_acc(srcs, d["w_hi"][r], d["w_lo"][r], dil, drop)
        peak = float(mag.max())
        assert peak < gx.EXACT_SUM_LIMIT, "step {}: sum of |terms| reaches {} >= 2^15".format(st, peak)
        v = np.maximum(acc + d["bias"][r], 0.0) * d["scale"][r].astype(np.float64) + d["shift"][r]
        h, lo = gx.split_bf16(gx.exact_f32(v))
        yh[..., k], yl[..., k] = h.reshape(B, T, RW), lo.reshape(B, T, RW)
    return yh, yl


def res2net_peak(case, d):
    """Largest sum of |terms| over every output of every step (the precondition's margin)."""
    B, T, C, dil = case["B"], case["T"], case["C"], case["d"]
    yh, yl = res2net_reference(case, d)
    hx, lx = d["x"]
    peak = 0.0
    for st in range(case["scale"] - 1):
        r, k = slice(st * RW, (st + 1) * RW), slice((st + 1) * RW, (st + 2) * RW)
        srcs = [("x", hx[..., k], lx[..., k])] + ([("y", yh[..., r], yl[..., r])] if st else [])
        peak = max(peak, float(res2net_step_acc(srcs, d["w_hi"][r], d["w_lo"][r], dil)[1].max()))
    return peak


# ------------------------------------------------------------------------------------------------ SE gate kernels
def se_cases():
    """name -> xvb_se_apply case.  Pitches are distinct and NaN-gapped: z at channel 8 of ldz, in at 16 of ldin, out
    fenced at 8 of ldout, next fenced at 0 of ldnext."""
    D = dict
    cases = {}
    for C in (8, 24, 1024, 1536):
        for T in (1, 7, 61, 200):
            cases["C{}_T{}".format(C, T)] = D(B=3, T=T, C=C)
    # more than sms * 32 * 256 eight-channel items: the grid-stride loop runs more than one round
    cases["grid_stride_B64_T200_C1024"] = D(B=64, T=200, C=1024)
    # ECAPA's running sum: next is the same buffer as in
    cases["inplace_C1024_T61"] = D(B=4, T=61, C=1024, inplace=True)
    cases["inplace_C24_T7"] = D(B=3, T=7, C=24, inplace=True)
    for c in cases.values():
        C = c["C"]
        c["ldz"], c["ldin"], c["ldout"], c["ldnext"] = _ru(8 + C + 8, 8), _ru(16 + C + 16, 8), _ru(8 + C + 40, 8), C + 8
        if c.get("inplace"):
            c["ldnext"] = c["ldin"]
    return cases


def seg_gate_cases():
    """name -> xvb_seg_gate_apply case: seg_len 1, 7, 100 (CAM++), T and > T, T not a multiple of seg_len, B > 1."""
    D = dict
    cases = {}
    for seg in (1, 7, 100, "T", "T+3"):
        for with_in in (False, True):
            T = 250
            s = {"T": T, "T+3": T + 3}.get(seg, seg)
            cases["seg{}_{}".format(seg, "in" if with_in else "noin")] = D(B=3, T=T, C=136, seg_len=s, with_in=with_in)
    cases["seg7_T61_C8_in"] = D(B=5, T=61, C=8, seg_len=7, with_in=True)
    for c in cases.values():
        C = c["C"]
        c["ldz"], c["ldin"], c["ldout"] = _ru(8 + C + 8, 8), _ru(16 + C + 16, 8), _ru(8 + C + 40, 8)
        c["nseg"] = -(-c["T"] // c["seg_len"])
    return cases


def se_operands(rng, B, T, C, rows):
    """(z planes, in planes, gate): z and in are split_bf16 of random normal fp32 values (full 16-bit planes), a few of
    them +-0; gate (rows, C) fp32 in [0, 1) with a few +-0."""
    def planes():
        v = (rng.standard_normal((B, T, C)) * 2.0 ** rng.randint(-4, 5, (B, T, C))).astype(np.float32)
        v[rng.rand(B, T, C) < 0.02] = 0.0
        v[rng.rand(B, T, C) < 0.02] = -0.0
        return gx.split_bf16(v)
    g = rng.uniform(0, 1, (rows, C)).astype(np.float32)
    g[rng.rand(rows, C) < 0.02] = 0.0
    g[rng.rand(rows, C) < 0.02] = -0.0
    return planes(), planes(), g


def gate_rows(B, T, seg_len):
    """(B, T) index of the gate row of frame t of utterance b: b * nseg + t // seg_len"""
    nseg = -(-T // seg_len)
    return np.arange(B)[:, None] * nseg + np.arange(T)[None, :] // seg_len


def se_reference(z, xin, g, rows):
    """float32: out = (z * g) + in, next = out + in, each operation rounded once.  z, xin: (hi, lo) planes or None for
    xin (no residual: out = z * g + 0).  -> (out, next) float32 (B, T, C)."""
    zf = z[0] + z[1]
    gate = g[rows]
    with np.errstate(all="ignore"):
        prod = zf * gate
    if xin is None:
        return prod + np.float32(0.0), None
    x = xin[0] + xin[1]
    out = prod + x
    return out, out + x


# ------------------------------------------------------------------------------------------------ small affine
SA_B = (1, 15, 16, 17, 64, 65, 1000)
SA_N = (1, 3, 4, 5, 8, 9, 129, 1536)
SA_K = (4, 124, 128, 132, 3072)


def small_affine_cases():
    """name -> xvb_small_affine case.  Every B, N and K value appears, every B and N against several K; the CTA tile is
    16 rows x 8 outputs, a warp's 4 x 4, and the lanes stride K by 128."""
    cases = {}
    for i, B in enumerate(SA_B):
        for j, N in enumerate(SA_N):
            if (i + j) % 3:
                continue
            K = SA_K[(i + 2 * j) % len(SA_K)]
            cases["B{}_N{}_K{}".format(B, N, K)] = dict(B=B, N=N, K=K)
    cases.update({"B1000_N129_K3072": dict(B=1000, N=129, K=3072), "B65_N1536_K3072": dict(B=65, N=1536, K=3072),
                  "B17_N9_K4": dict(B=17, N=9, K=4), "B16_N5_K132": dict(B=16, N=5, K=132),
                  "B15_N3_K124": dict(B=15, N=3, K=124), "B64_N8_K128": dict(B=64, N=8, K=128)})
    for c in cases.values():
        # x: the slice at 4 of a NaN (B + 1, ldx) buffer; y / planes: fenced slices of wider pitches
        c["x_c0"], c["ldx"] = 4, _ru(4 + c["K"] + 8, 4)
        c["y_c0"], c["ldy"] = 3, c["N"] + 7
        c["p_c0"], c["ldp"] = 8, _ru(8 + c["N"] + 8, 8)
    return cases


# epilogue flag sets run on every case: (name, relu, bn, act)
SA_EPILOGUES = [("bias", False, False, None), ("relu", True, False, None), ("relu_bn", True, True, None),
                ("bn", False, True, None), ("sigmoid", False, False, "sigmoid"), ("relu_bn_tanh", True, True, "tanh")]


def make_small_affine(case, seed):
    rng = np.random.RandomState(seed)
    B, N, K = case["B"], case["N"], case["K"]
    return {"x": gx.grid_values(rng, (B, K), 2.0), "w": gx.int_plane(rng, (N, K), 2), "bias": gx.grid_values(rng, N),
            "scale": (gx.pow2_scales(rng, N) * rng.choice([-1.0, 1.0], N)).astype(np.float32),
            "shift": gx.grid_values(rng, N)}


def small_affine_acc(d):
    """float64 x . W^T, asserting that every partial sum is exact in fp32 (multiples of 2^-8, sum |terms| < 2^15)."""
    x, w = d["x"].astype(np.float64), d["w"].astype(np.float64)
    peak = float((np.abs(x) @ np.abs(w).T).max())
    assert peak < gx.EXACT_SUM_LIMIT, "sum of |terms| reaches {} >= 2^15".format(peak)
    return x @ w.T


def small_affine_reference(case, d, relu, bn, act, acc=None):
    """-> (want, bound) as gemm_exact.layer_reference: float32 and None when exact, else float64 and its bound."""
    acc = small_affine_acc(d) if acc is None else acc
    layer = dict(B=case["B"], T=1, relu=relu, act=act)
    dd = {"bias": d["bias"]}
    if bn:
        dd["scale"], dd["shift"] = d["scale"], d["shift"]
    want, bound = gx.layer_reference(layer, dd, acc[:, None, :])
    return want[:, 0], (None if bound is None else bound[:, 0])
