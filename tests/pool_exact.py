"""Edge catalogue, operands, float64 references and per-element error bounds for the time-pooling kernels:
csrc/pooling.cu (stats_pool_tma_kernel, pool_finalize_kernel) and the pooling half of csrc/ecapa.cu
(attn_stats_pool_kernel, attn_head_stats_pool_kernel, lde_weights_kernel + lde_encode_kernel, plane_mean_kernel).

Catalogue.  Every family has cases on both sides of each of its kernel constants: the 40-frame TMA boxes and 200-frame
slabs of the statistics kernel, the 8-warp / 32-frame strides of the attention kernels, the 128-frame x 32-channel
weights tiles and 64-frame weight staging of LDE, the 128- and 256-channel CTAs.

Operands.  Ordinary frames are N(0, 1) plus a per-channel offset (so a channel block read 4 channels off moves every
mean).  Large-magnitude markers sit where kernels go wrong: the first and last frame of every TMA box, slab, time block
and weight stage, the first frame each warp handles, the last frame of each utterance, and the first and last channel of
every CTA.  Attention logits follow one of five patterns: random, increasing (a rescale at every frame), decreasing,
one +60 spike over a floor of -50 (every other weight underflows in fp32) and a per-channel range of up to +-80.

References are float64 and follow the formulas the kernels cite: StatisticsPooling (pooling.py:58-67) with its clamp
(mode 0) or the ECAPA global context's sqrt(unbiased var + eps) (mode 1, ecapa_tdnn_xvector.py:177-178); the
attentive E[x^2] - mu^2 with its floor (ecapa_tdnn_xvector.py:183-188, and mean_T((x - mu)^2) for
stddev_attention=False); the xi-vector prior element and 2 log softplus (pooling.py:165-212); LDE (pooling.py:148-159).

Bounds, per output element, u = 2^-24; one constant K per family, written once below and never tuned per case.
  * Plain means (stats, finalize, plane mean).  A sum of n terms in any order, then a multiply by a rounded 1/n and at
    most a few Chan merges (each a convex combination, <= 4u of the larger mean): |d mean| <= K (n + 8) u mean|x|.
    pool_finalize_kernel only merges nblk fp32 partials (each rounded once): n is nblk there, and mean|x| the largest
    over the prefixes that end at a block boundary (the running mean each merge rounds).
  * Two-pass / Chan variances.  Each slab's sum of (x - m)^2 is a sum of n non-negative terms, each with 3 roundings:
    (n + 8) u sum (x - mu)^2.  The mean's error dm enters a Chan merge through d^2 n_a n_b / n, with |d| <= 2 max|x - mu|
    and sum n_a n_b / n <= n, and the pass-2 centre through n dm^2:  |d M2| <= K (n + 8) u S2 + 4 n R dm + n dm^2, with
    S2 = sum (x - mu)^2, R = max|x - mu|; the variance divides by n (mode 0) or n - 1 (mode 1) and rounds twice more.
  * Softmax-weighted moments.  A weight exp(l - m) picks up a relative error of about u |l - m| from the rounded
    argument, a few ulp from expf, and one rounding per online rescale (at most n of them); a common relative error of
    all weights cancels in sum(w x) / sum(w), so only its spread matters, against x - mu.  The sums themselves add
    n u sum w|x|.  With L = max|l - max l| (+8 for expf and the argument, +16 more for 2 log softplus):
      |d mu| <= K u ((n + L) sum w|x - mu| + n sum w|x|),   |d E[x^2]| <= K u ((n + L) sum w|x^2 - E[x^2]| + n sum w x^2),
    and E[x^2] - mu^2 adds (2|mu| + dmu) dmu and the cancellation term K u (E[x^2] + mu^2).  The unweighted variance
    (u2 - 2 mu u1) / T + mu^2 adds K u n (sum x^2 + 2|mu| sum|x|) / T for its plain sums and 2 |mu - mean x| dmu.
  * LDE.  d[t,k] = sum_c (x - mu)^2 has (C + 3) u d of error, so the logit beta d is off by |beta| (C + 3) u d; a softmax
    weight's relative error is then at most rho_t = 4 max_k (|beta_k| (C + 3) u d[t,k] + 2u |l[t,k]|) + (K + 8) u.  The
    encode sum adds (T + 3) u per term:  |d e| <= K (1/T) sum_t w |x - mu| (rho_t + (T + 3) u).
  * A std's error is the variance's error over (sd + sqrt(floor)) (or its square root, if smaller), plus 2u sd.

Plain numpy (no torch, no GPU): test_gpu_pooling_edges.py runs the kernels on these operands, and
test_pooling_edges_host.py shows on the CPU that every mutant of a case leaves its bound and every fp32 simulation
stays inside it."""
import math

import numpy as np

U = 2.0 ** -24
K_STATS = 2.0        # stats_pool_tma_kernel and pool_finalize_kernel
K_ATTN = 4.0         # attn_stats_pool_kernel and attn_head_stats_pool_kernel
K_LDE = 4.0          # lde_weights_kernel + lde_encode_kernel
K_PLANE = 2.0        # plane_mean_kernel

BOX, SLAB, WARPS, ATTN_STRIDE = 40, 200, 8, 32
LDE_ROWS, LDE_CHUNK, LDE_STAGE = 128, 32, 64
MARK = 64.0          # marker magnitude (stats, attention, plane mean)
LDE_MARK = 4.0       # LDE markers stay moderate: a logit error grows with d = sum (x - mu)^2


# ------------------------------------------------------------------------------------------------ catalogue
STATS_T = [1, 2, 8, 9, 39, 40, 41, 199, 200, 201, 240, 241, 399, 400, 401, 1001]
STATS_C = [4, 124, 128, 132, 256, 260, 512, 1500, 1536]
STATS_PAD = [0, 4, 124]
EPS = [1e-10, 0.0, 1e-5]
MASKED_LENGTHS = [
    (401, [1, 40, 41, 200, 201, 400, 401, 7]),
    (1001, [1001, 241, 240, 199, 39, 2]),
]
FIN_NBLK = [1, 2, 7, 50]
FIN_TB = [1, 8, 32, 128]
FIN_C = [4, 508, 512, 516, 1500]
ATTN_T = [1, 2, 7, 8, 9, 31, 32, 33, 64, 65, 200, 1001]
ATTN_C = [4, 124, 128, 132, 1536]
PATTERNS = ["random", "inc", "dec", "spike", "range80"]
HEAD_MAPS = ["shared", "gdiv1", "heads", "global", "global_gdiv1", "mq", "mq_gdiv1", "xi", "unweighted"]
HEAD_C = [128, 132, 4, 256]
LDE_K = [1, 2, 7, 8, 9, 16, 17, 56, 57, 63, 64]
LDE_C = [1, 3, 31, 32, 33, 127, 128, 129, 200]
LDE_T = [1, 63, 64, 65, 127, 128, 129]
PM_C = [8, 248, 256, 264, 1536]
PM_T = [1, 7, 8, 9, 200]


def stats_cases():
    cases = {}
    for i, T in enumerate(STATS_T):
        C = STATS_C[i % len(STATS_C)]
        pad = STATS_PAD[i % 3]
        B = 3 if T * C < 200000 else 2
        cases["stats_T{}_C{}".format(T, C)] = dict(
            kind="stats", B=B, T=T, C=C, ldx=C + pad, c0=0 if pad == 0 else (4 if pad == 4 else 60), mode=i % 2,
            eps=EPS[(i // 2) % 3], planes=(i // 3) % 2 == 0, ldo_pad=4 * ((i // 2) % 2), lengths=None)
    cases["stats_T1_mode1"] = dict(kind="stats", B=2, T=1, C=132, ldx=136, c0=4, mode=1, eps=1e-5, planes=True, ldo_pad=4,
                                   lengths=None)
    for j, (T, lens) in enumerate(MASKED_LENGTHS):
        C = (260, 132)[j]
        cases["stats_masked_T{}".format(T)] = dict(kind="stats", B=len(lens), T=T, C=C, ldx=C + 4 * (1 + j), c0=4, mode=j,
                                                    eps=(1e-10, 1e-5)[j], planes=True, ldo_pad=4 * j, lengths=list(lens))
    cases["stats_B65535"] = dict(kind="stats", B=65535, T=2, C=4, ldx=8, c0=4, mode=0, eps=1e-10, planes=True, ldo_pad=0,
                                 lengths=None)
    return cases


def finalize_cases():
    cases, i = {}, 0
    for nblk in FIN_NBLK:
        for tb in FIN_TB:
            for T in sorted({nblk * tb, (nblk - 1) * tb + 1}):
                C = FIN_C[i % len(FIN_C)] if T <= 1000 else (4, 508)[i % 2]
                cases["fin_n{}_tb{}_T{}_C{}".format(nblk, tb, T, C)] = dict(
                    kind="finalize", B=2, T=T, C=C, nblk=nblk, tb=tb, mode=i % 2, eps=EPS[i % 3], planes=i % 3 != 1,
                    ldo_pad=4 * (i % 2))
                i += 1
    return cases


def attn_cases():
    cases = {}
    for i, T in enumerate(ATTN_T):
        C = ATTN_C[i % len(ATTN_C)]
        pat = PATTERNS[(i + i // 5) % len(PATTERNS)]
        cases["attn_T{}_C{}_{}".format(T, C, pat)] = dict(
            kind="attn", B=2, T=T, C=C, G=C, O=C, gdiv=1, ldl=C + 4 * (1 + i % 2), ldx=C + 4 * (2 - i % 2), l0=4, x0=4,
            pattern=pat, floor=1e-5, planes=i % 2 == 0)
    return cases


def _head_case(hmap, T, C, i):
    pat = PATTERNS[(i + i // 5) % len(PATTERNS)]
    O, gdiv, hw, rep, unw, xi = C, 1, C, 1, False, False
    if hmap == "shared":
        gdiv = C
    elif hmap == "heads":
        gdiv = C // 4 if C >= 16 else 2
    elif hmap == "global":
        O, gdiv = 2 * C, C
    elif hmap == "global_gdiv1":
        O = 2 * C
    elif hmap in ("mq", "mq_gdiv1"):
        hw = 4 if C == 4 else (44 if C == 132 else 32)
        rep = 2
        O = rep * C
        gdiv = hw if hmap == "mq" else 1
    elif hmap == "xi":
        xi, pat = True, "softplus"
    elif hmap == "unweighted":
        unw, gdiv = True, (1 if i % 2 else C)
    if not hmap.startswith("mq"):
        hw, rep = C, O // C
    G = (O - 1) // gdiv + 1
    return dict(kind="head", B=2, T=T, C=C, O=O, G=G, gdiv=gdiv, head_width=hw, rep=rep, unweighted=unw, xi=xi,
                mq=hmap.startswith("mq"), ldl=G + 4 * (1 + i % 2), ldx=C + 4, l0=0, x0=4, pattern=pat,
                floor=(1e-10, 1e-5)[i % 2], planes=i % 2 == 1, vector=gdiv == 1)


def head_cases():
    cases = {}
    for j, hmap in enumerate(HEAD_MAPS):
        for i, T in enumerate(ATTN_T):
            C = HEAD_C[(i + j) % len(HEAD_C)]
            if T * C > 70000:
                C = 132
            cases["head_{}_T{}_C{}".format(hmap, T, C)] = _head_case(hmap, T, C, i + j)
    return cases


def lde_cases():
    cases = {}
    for i, K in enumerate(LDE_K):
        C, T = LDE_C[i % len(LDE_C)], LDE_T[i % len(LDE_T)]
        B = 3 if T % 128 else 2
        cases["lde_K{}_C{}_T{}".format(K, C, T)] = dict(kind="lde", B=B, T=T, C=C, K=K, ldx=C + (0, 1, 5)[i % 3],
                                                        x0=(0, 1, 3)[i % 3], planes=i % 2 == 0, ldo_pad=3 * (i % 2))
    return cases


def plane_cases():
    cases = {}
    for i, C in enumerate(PM_C):
        for j, T in enumerate(PM_T):
            cases["plane_T{}_C{}".format(T, C)] = dict(kind="plane", B=2, T=T, C=C, ldx=C + (0, 8, 24)[(i + j) % 3],
                                                       planes=(i + j) % 2 == 0, ldo_pad=8 * ((i + j) % 2))
    for k in (1, 2, 4):       # the ResNet SE gate's (B, P, C) planes read as (B, P / k, k C)
        cases["plane_resnet_k{}".format(k)] = dict(kind="plane", B=3, T=16 // k, C=256 * k, ldx=256 * k, planes=k == 2,
                                                    ldo_pad=0)
    return cases


def all_cases():
    out = {}
    for f in (stats_cases, finalize_cases, attn_cases, head_cases, lde_cases, plane_cases):
        out.update(f())
    return out


# ------------------------------------------------------------------------------------------------ operands
def _lengths(case):
    return np.array(case["lengths"] if case.get("lengths") else [case["T"]] * case["B"], dtype=np.int64)


def _offsets(C):
    return ((np.arange(C) % 13) - 6) * 0.25


def marker_frames(case):
    """(B, T + 1) bool: the frames that hold markers."""
    B, T = case["B"], case["T"]
    t = np.arange(T + 1)
    kind = case["kind"]
    if kind == "stats":
        m = (t % BOX == 0) | (t % BOX == BOX - 1) | (t % SLAB == SLAB - 1) | (t % SLAB < WARPS)
    elif kind == "finalize":
        m = (t % case["tb"] == 0) | (t % case["tb"] == case["tb"] - 1)
    elif kind in ("attn", "head"):
        m = (t < WARPS) | (t % ATTN_STRIDE == 0) | (t % ATTN_STRIDE == ATTN_STRIDE - 1)
    elif kind == "lde":
        m = (t % LDE_STAGE == 0) | (t % LDE_STAGE == LDE_STAGE - 1)
    else:
        m = t < WARPS
    m = np.broadcast_to(m, (B, T + 1)).copy()
    if kind == "lde":
        rows = np.arange(B)[:, None] * T + t[None, :]
        m |= (rows % LDE_ROWS == 0) | (rows % LDE_ROWS == LDE_ROWS - 1)
    lens = _lengths(case)
    m[np.arange(B), lens - 1] = True
    return m


def marker_channels(case, C):
    c = np.arange(C)
    cta = {"stats": 128, "finalize": 512, "attn": 128, "head": 128, "lde": 128, "plane": 256}[case["kind"]]
    m = (c % cta == 0) | (c % cta == cta - 1) | (c == C - 1)
    if case["kind"] == "lde":
        m |= (c % LDE_CHUNK == 0) | (c % LDE_CHUNK == LDE_CHUNK - 1)
    return m


def make_x(case, rng, C=None):
    """(B, T + 1, C) float32 frames (one spare frame past T for the length + 1 mutant)."""
    B, T = case["B"], case["T"]
    C = case["C"] if C is None else C
    mark = LDE_MARK if case["kind"] == "lde" else MARK
    x = rng.standard_normal((B, T + 1, C))
    ch = marker_channels(case, C)
    x[:, :, ch] *= 4.0 if case["kind"] == "lde" else 16.0
    fr = marker_frames(case)
    sign = np.where(rng.random_sample((B, T + 1, C)) < 0.5, -1.0, 1.0)
    x = np.where(fr[:, :, None], mark * sign + 0.5 * x, x)
    return (x + _offsets(C)).astype(np.float32)


def spike_frame(T):
    """The spike's frame: the last 32-frame stride start (warp 0's frame of its last round), or the last frame if T <= 32."""
    return ATTN_STRIDE * ((T - 1) // ATTN_STRIDE) if T > ATTN_STRIDE else T - 1


def make_logits(case, rng, G):
    B, T, pat = case["B"], case["T"], case["pattern"]
    t = np.arange(T + 1, dtype=np.float64)[None, :, None]
    g = np.arange(G)[None, None, :]
    if pat == "random":
        l = rng.standard_normal((B, T + 1, G)) * 2.0
    elif pat == "inc":
        l = t * (1 + g % 3) * min(0.5, 40.0 / T) + 0.1 * rng.standard_normal((B, T + 1, G))
    elif pat == "dec":
        l = -t * (1 + g % 3) * min(0.5, 40.0 / T) + 0.1 * rng.standard_normal((B, T + 1, G))
    elif pat == "spike":
        l = rng.standard_normal((B, T + 1, G)) - 50.0
        l[:, spike_frame(T), :] = 60.0
    elif pat == "range80":
        l = rng.uniform(-1, 1, (B, T + 1, G)) * 80.0 * (1 + g % 5) / 5.0
    else:                   # softplus: raw logits, some above the threshold 20, some below -104 (softplus underflows)
        l = np.clip(rng.standard_normal((B, T + 1, G)) * 2.0, -10, 10)
        r = rng.random_sample((B, T + 1, G))
        l = np.where(r < 0.15, rng.uniform(21, 40, l.shape), l)
        l = np.where(r > 0.8, rng.uniform(-200, -110, l.shape), l)
        l[:, :, 1 % G] = rng.uniform(-200, -110, (B, T + 1))   # a channel whose frames all underflow: the prior alone
    if pat in ("random", "dec", "range80"):
        l[:, T - 1] = l[:, :T].max(axis=1)       # the last frame carries weight, so a frame too few or too many shows
    return l.astype(np.float32)


def make_case(case, seed):
    rng = np.random.RandomState(seed)
    k = case["kind"]
    d = {"lengths": _lengths(case)}
    if k in ("stats", "finalize", "plane"):
        d["x"] = make_x(case, rng)
    elif k in ("attn", "head"):
        d["x"] = make_x(case, rng)
        d["l"] = make_logits(case, rng, case["G"])
        if case.get("xi"):
            d["prior_l"] = rng.uniform(-1, 3, case["C"]).astype(np.float32)
            d["prior_x"] = (rng.standard_normal(case["C"]) + _offsets(case["C"])).astype(np.float32)
    else:
        d["x"] = make_x(case, rng)
        C, K = case["C"], case["K"]
        d["mu"] = (_offsets(C)[:, None] + 0.5 * rng.standard_normal((C, K))).astype(np.float32)
        d["neg_beta"] = (-(rng.uniform(0.05, 0.3, K) ** 2 + 1e-5)).astype(np.float32)
    if k == "plane":                                # bf16 planes; hi + lo is exact in fp32
        from gemm_exact import split_bf16
        d["hi"], d["lo"] = split_bf16(d["x"])
        d["x"] = (d["hi"].astype(np.float64) + d["lo"]).astype(np.float32)
    if k == "finalize":
        d["partial"] = finalize_partials(d["x"][:, :case["T"]].astype(np.float64), case["tb"])
    return d


def finalize_partials(x, tb, shift=0):
    """(nblk, B, 2C) fp32 [mean | M2] of the time blocks of tb frames, in float64 then rounded.  shift moves every block
    boundary one frame later (the split mutant) while the finaliser keeps the nominal counts."""
    B, T, C = x.shape
    nblk = -(-T // tb)
    p = np.zeros((nblk, B, 2 * C))
    for k in range(nblk):
        lo, hi = min(T, k * tb + (shift if k else 0)), min(T, (k + 1) * tb + shift)
        if k == nblk - 1:
            hi = T
        blk = x[:, lo:hi]
        n = max(hi - lo, 1)
        m = blk.sum(axis=1) / n
        p[k, :, :C] = m
        p[k, :, C:] = ((blk - m[:, None]) ** 2).sum(axis=1)
    return p.astype(np.float32)


# ------------------------------------------------------------------------------------------------ references
def _chan(x, lens, mult, block):
    """float64 mean and M2 of utterance b's first lens[b] frames, frame t counted mult[b, t] times, in blocks of `block`
    frames merged with Chan's update (the counts stay the nominal ones, as a kernel's would)."""
    B, T, C = x.shape
    run_n = np.zeros((B, 1))
    run_m = np.zeros((B, C))
    run_q = np.zeros((B, C))
    for k in range(-(-T // block)):
        t = np.arange(k * block, min(T, (k + 1) * block))
        inb = t[None, :] < lens[:, None]
        nk = inb.sum(axis=1)[:, None].astype(np.float64)
        w = np.where(inb, mult[:, t], 0.0)[:, :, None]
        xk = x[:, t]
        mk = (w * xk).sum(axis=1) / np.maximum(nk, 1)
        qk = (w * (xk - mk[:, None]) ** 2).sum(axis=1)
        tot = run_n + nk
        wb = np.where(tot > 0, nk / np.maximum(tot, 1), 0.0)
        d = mk - run_m
        run_m = run_m + d * wb
        run_q = run_q + qk + d * d * run_n * wb
        run_n = tot
    return run_m, run_q


def _std(q, n, mode, eps):
    with np.errstate(divide="ignore", invalid="ignore"):
        if mode == 0:
            return np.sqrt(np.maximum(q / n, eps))
        return np.sqrt(q / (n - 1) + eps)


def _std_bound(bvar, sd, floor):
    with np.errstate(divide="ignore", invalid="ignore"):
        b = np.minimum(bvar / (sd + math.sqrt(floor)), np.sqrt(bvar)) + 2 * U * sd
    return np.where(np.isnan(b), 0.0, b)


def stats_reference(case, d, x=None, lens=None, mult=None, block=None):
    """(mean, std), each (B, C) float64, of xvb_stats_pool_ex / _lengths (or of pool_finalize over d's data)."""
    x = d["x"].astype(np.float64) if x is None else x
    lens = d["lengths"] if lens is None else lens
    T = int(lens.max())
    x = x[:, :T]
    mult = np.ones(x.shape[:2]) if mult is None else mult
    m, q = _chan(x, lens, mult, block or (SLAB if case["kind"] == "stats" else case["tb"]))
    n = lens[:, None].astype(np.float64)
    return m, _std(q, n, case["mode"], case["eps"])


def stats_bound(case, d):
    x = d["x"][:, :case["T"]].astype(np.float64)
    lens = d["lengths"]
    inb = (np.arange(case["T"])[None, :] < lens[:, None])[:, :, None]
    n = lens[:, None].astype(np.float64)
    mean, sd = stats_reference(case, d)
    A = np.where(inb, np.abs(x), 0).sum(axis=1) / n
    nt = n
    if case["kind"] == "finalize":      # fp32 partials (one rounding each) and nblk merges: A is the largest block's mean|x|
        tb = case["tb"]
        nt = float(case["nblk"])
        ends = np.minimum(np.arange(tb, case["T"] + tb, tb), case["T"])
        A = (np.cumsum(np.abs(x), axis=1)[:, ends - 1] / ends[None, :, None]).max(axis=1)
    dev = np.where(inb, np.abs(x - mean[:, None]), 0)
    S2, R = (dev ** 2).sum(axis=1), dev.max(axis=1)
    bmean = K_STATS * (nt + 8) * U * A
    bq = K_STATS * (nt + 8) * U * S2 + 4 * n * R * bmean + n * bmean ** 2
    with np.errstate(divide="ignore", invalid="ignore"):
        nd = n if case["mode"] == 0 else n - 1
        var = S2 / nd
        bvar = bq / nd + 2 * U * var
    return bmean, _std_bound(bvar, sd, case["eps"])


def _head_maps(case):
    o = np.arange(case["O"])
    hw, rep = case.get("head_width", case["C"]), case.get("rep", 1)
    return (o // (rep * hw)) * hw + o % hw, o // case["gdiv"]


def softplus2log(l):
    """2 log softplus(l) (Softplus(beta=1, threshold=20)) in float64, -inf where fp32's softplus underflows to 0."""
    l = np.asarray(l, dtype=np.float64)
    with np.errstate(over="ignore", divide="ignore"):
        sp = np.where(l > 20, l, np.log1p(np.exp(np.minimum(l, 20))))
        out = 2 * np.log(sp)
    return np.where(np.exp(l) < 2.0 ** -150, -np.inf, out)


def attn_operands(case, d, mult=None, x=None, chshift=0):
    """Per output channel (B, n, O) float64 logits and values (prior appended as element n - 1), and multiplicities."""
    x = d["x"] if x is None else x
    T = case["T"]
    cmap, gmap = _head_maps(case)
    if chshift:
        cmap, gmap = _shift_block(cmap, chshift, case["C"]), (_shift_block(gmap, chshift, case["G"]) if case["gdiv"] == 1 else gmap)
    X = x[:, :T].astype(np.float64)[:, :, cmap]
    Lg = d["l"][:, :T].astype(np.float64)[:, :, gmap]
    mult = np.ones((case["B"], T)) if mult is None else mult[:, :T]
    if case.get("xi"):
        Lg = softplus2log(Lg)
        B, O = case["B"], case["O"]
        X = np.concatenate([X, np.broadcast_to(d["prior_x"].astype(np.float64)[cmap], (B, 1, O))], axis=1)
        Lg = np.concatenate([Lg, np.broadcast_to(d["prior_l"].astype(np.float64)[cmap], (B, 1, O))], axis=1)
        mult = np.concatenate([mult, np.ones((B, 1))], axis=1)
    return Lg, X, mult


def _shift_block(idx, s, n):
    """The first CTA's 128 outputs read index + s (clamped to the last valid one): a channel block 4 off."""
    idx = idx.copy()
    idx[:128] = np.minimum(idx[:128] + s, n - 1)
    return idx


def _softmax_w(Lg, mult):
    with np.errstate(invalid="ignore", over="ignore"):
        mx = np.where(mult[:, :, None] > 0, Lg, -np.inf).max(axis=1, keepdims=True)
        e = np.where(mult[:, :, None] > 0, np.exp(Lg - mx), 0.0) * mult[:, :, None]
        return e / e.sum(axis=1, keepdims=True), mx


def attn_reference(case, d, **kw):
    Lg, X, mult = attn_operands(case, d, **kw)
    w, _ = _softmax_w(Lg, mult)
    mu = (w * X).sum(axis=1)
    if case.get("unweighted"):
        var = (mult[:, :, None] * (X - mu[:, None]) ** 2).sum(axis=1) / case["T"]
    else:
        var = (w * X * X).sum(axis=1) - mu * mu
    return mu, np.sqrt(np.maximum(var, case["floor"]))


def attn_bound(case, d):
    Lg, X, mult = attn_operands(case, d)
    w, mx = _softmax_w(Lg, mult)
    n = X.shape[1]
    fin = np.isfinite(Lg)
    L = np.where(fin, mx - Lg, 0).max(axis=1) + 8 + (16 if case.get("xi") else 0)
    mu, sd = attn_reference(case, d)
    E2 = (w * X * X).sum(axis=1)
    dx = np.abs(X - mu[:, None])
    bmu = K_ATTN * U * ((n + L) * (w * dx).sum(axis=1) + n * (w * np.abs(X)).sum(axis=1))
    if case.get("unweighted"):
        T = case["T"]
        s2, s1 = (X * X).sum(axis=1), X.sum(axis=1)
        bvar = K_ATTN * U * (n * (s2 + 2 * np.abs(mu) * np.abs(X).sum(axis=1)) / T + s2 / T + 2 * np.abs(mu * s1) / T
                             + mu * mu) + 2 * np.abs(mu - s1 / T) * bmu + bmu * bmu
    else:
        bE2 = K_ATTN * U * ((n + L) * (w * np.abs(X * X - E2[:, None])).sum(axis=1) + n * E2)
        bvar = bE2 + (2 * np.abs(mu) + bmu) * bmu + K_ATTN * U * (E2 + mu * mu)
    return bmu, _std_bound(bvar, sd, case["floor"])


def lde_terms(case, d, x=None, mult=None, lens=None):
    x = (d["x"] if x is None else x).astype(np.float64)
    T = case["T"] if lens is None else int(lens[0])
    x = x[:, :T]
    mu, nb = d["mu"].astype(np.float64), d["neg_beta"].astype(np.float64)
    r = x[:, :, :, None] - mu[None, None]                       # (B, T, C, K)
    dist = (r * r).sum(axis=2)                                   # (B, T, K)
    l = nb * dist
    e = np.exp(l - l.max(axis=2, keepdims=True))
    w = e / e.sum(axis=2, keepdims=True)
    if mult is not None:
        w = w * mult[:, :T, None]
    return r, dist, l, w, T


def lde_reference(case, d, **kw):
    r, _, _, w, T = lde_terms(case, d, **kw)
    return ((w[:, :, None, :] * r).sum(axis=1) / T).reshape(case["B"], -1)


def lde_bound(case, d):
    r, dist, l, w, T = lde_terms(case, d)
    C, K = case["C"], case["K"]
    nb = np.abs(d["neg_beta"].astype(np.float64))
    rho = 4 * (nb * (C + 3) * U * dist + 2 * U * np.abs(l)).max(axis=2) + (K + 8) * U      # (B, T)
    # + 2^-125 |x - mu|: a weight that underflows to a subnormal keeps only its absolute accuracy
    b = K_LDE * ((w[:, :, None, :] * (rho + (T + 3) * U)[:, :, None, None] + 2.0 ** -125) * np.abs(r)).sum(axis=1) / T
    return b.reshape(case["B"], -1)


def plane_reference(case, d, x=None, mult=None):
    T = case["T"]
    x = (d["x"] if x is None else x)[:, :T].astype(np.float64)
    if mult is not None:
        x = x * mult[:, :T, None]
    return x.sum(axis=1) / T


def plane_bound(case, d):
    T = case["T"]
    return K_PLANE * (T + 4) * U * np.abs(d["x"][:, :T].astype(np.float64)).mean(axis=1)


def finalize_reference(case, partial, drop=None):
    """float64 Chan merge of fp32 partials with the nominal block counts (drop: skip one block's partial)."""
    nblk, B, C2 = partial.shape
    C, T, tb = C2 // 2, case["T"], case["tb"]
    p = partial.astype(np.float64)
    n, m, q = 0.0, np.zeros((B, C)), np.zeros((B, C))
    for k in range(nblk):
        if k == drop:
            continue
        nk = min(tb, T - k * tb)
        tot = n + nk
        dd = p[k, :, :C] - m
        m = m + dd * (nk / tot)
        q = q + p[k, :, C:] + dd * dd * n * nk / tot
        n = tot
    return m, _std(q, T, case["mode"], case["eps"])


def reference(case, d):
    """{output name: (want float64, bound float64)} for a case."""
    k = case["kind"]
    if k in ("stats", "finalize"):
        (m, s), (bm, bs) = stats_reference(case, d), stats_bound(case, d)
        return {"mean": (m, bm), "std": (s, bs)}
    if k in ("attn", "head"):
        (m, s), (bm, bs) = attn_reference(case, d), attn_bound(case, d)
        return {"mean": (m, bm), "std": (s, bs)}
    if k == "lde":
        return {"e": (lde_reference(case, d), lde_bound(case, d))}
    return {"mean": (plane_reference(case, d), plane_bound(case, d))}


def flat_output(case, outs):
    """The kernel's fp32 output row layout: [mean | std] or the single output."""
    if "e" in outs:
        return outs["e"]
    if "std" in outs:
        return np.concatenate([outs["mean"], outs["std"]], axis=1)
    return outs["mean"]


# ------------------------------------------------------------------------------------------------ mutants
def mutants(case, d):
    """(name, {output: float64}) for each kernel mistake that applies to the case: a marker frame dropped or duplicated,
    the first CTA's channel block read 4 channels off, an utterance one frame shorter or longer, a box / slab / block /
    stage boundary read one frame late (the boundary frame replaced by the one before it), one warp's frames dropped."""
    k, B, T = case["kind"], case["B"], case["T"]
    lens = d["lengths"]
    fr = marker_frames(case)
    out = []
    b = int(np.argmax(lens))
    L = int(lens[b])
    # how much each frame of utterance b can move an output: its largest softmax weight for the attention kernels
    # (an underflowed weight cannot), 1 elsewhere; the mutants pick the frames that matter, the middle ones on ties
    imp = dup = np.ones(L)
    if k in ("attn", "head"):        # dropping the heaviest frame moves the most; duplicating one moves w (1 - w) |x - mu|
        Lg, X, mult = attn_operands(case, d)
        w = _softmax_w(Lg, mult)[0][b, :L]
        mu = attn_reference(case, d)[0][b]
        imp = w.max(axis=1)
        dup = (w * (1 - w) * np.abs(X[b, :L] - mu)).max(axis=1)
    closeness = -np.abs(np.arange(L) - L / 2) * 1e-9

    def mult_with(t, v):
        mm = np.ones((B, T + 1))
        mm[b, t] = v
        return mm

    tm = [t for t in range(L) if fr[b, t]]
    t_mark = max(tm, key=lambda t: imp[t] + closeness[t])
    t_dup = max(tm, key=lambda t: dup[t] + closeness[t])
    muts = [("drop marker frame", dict(mult=mult_with(t_mark, 0.0))),
            ("duplicate marker frame", dict(mult=mult_with(t_dup, 2.0)))]
    edge = {"stats": BOX, "finalize": case.get("tb"), "attn": WARPS, "head": WARPS, "lde": LDE_STAGE, "plane": WARPS}[k]
    if L > edge:
        e = max(range(edge, L, edge), key=lambda e: imp[e] + imp[e - 1] + closeness[e])
        mm = np.ones((B, T + 1))
        mm[:, e] -= 1
        mm[:, e - 1] += 1
        muts.append(("split one frame off", dict(mult=mm)))
    if L > 1:
        mm = np.ones((B, T + 1))
        mm[:, np.arange(T + 1) % WARPS == t_mark % WARPS] = 0.0
        muts.append(("drop one warp's frames", dict(mult=mm)))
    muts.append(("length - 1" if L > 1 else "length + 1", dict(dlen=-1 if L > 1 else 1)))
    muts.append(("channel block shifted by 4", dict(shift=4)))

    for name, mu in muts:
        res = _mutant_eval(case, d, **mu)
        if res is not None:
            out.append((name, res))
    if k == "finalize" and case["nblk"] > 1:
        x = d["x"][:, :T].astype(np.float64)
        out.append(("block split one frame off", _fin_out(case, finalize_partials(x, case["tb"], shift=1))))
        out.append(("drop block 1's partial", _fin_out(case, d["partial"], drop=1)))
    return out


def _fin_out(case, partial, drop=None):
    m, s = finalize_reference(case, partial, drop=drop)
    return {"mean": m, "std": s}


def _shifted_x(x, s, C):
    x = x.copy()
    hi = min(128, C)
    src = np.minimum(np.arange(hi) + s, C - 1)
    x[:, :, :hi] = x[:, :, src]
    return x


def _mutant_eval(case, d, mult=None, dlen=0, shift=0):
    k = case["kind"]
    x = d["x"]
    lens = d["lengths"]
    if shift:
        C = case["C"]
        if k in ("attn", "head"):
            m, s = attn_reference(case, d, chshift=shift)
            return {"mean": m, "std": s}
        x = _shifted_x(x, shift, C)
    if dlen:
        lens = lens.copy()
        b = int(np.argmax(lens))
        lens[b] += dlen
    if k in ("stats", "finalize"):
        m, s = stats_reference(case, d, x=x.astype(np.float64), lens=lens, mult=mult)
        return {"mean": m, "std": s}
    if k in ("attn", "head"):
        if dlen:
            mm = np.ones((case["B"], case["T"] + 1))
            if dlen < 0:
                mm[:, case["T"] - 1] = 0.0
                return dict(zip(("mean", "std"), attn_reference(case, d, mult=mm)))
            return None     # T = 1: one frame more is a different case
        m, s = attn_reference(case, d, x=x, mult=mult)
        return {"mean": m, "std": s}
    if k == "lde":
        if dlen:
            c2 = dict(case, T=case["T"] + dlen)
            return {"e": lde_reference(c2, d) * (case["T"] + dlen) / case["T"]}
        return {"e": lde_reference(case, d, x=x, mult=mult)}
    if dlen:
        c2 = dict(case, T=case["T"] + dlen)
        return {"mean": plane_reference(c2, d, x=x) * (case["T"] + dlen) / case["T"]}
    return {"mean": plane_reference(case, d, x=x, mult=mult)}


def worst_ratio(got, want, bound):
    """max |got - want| / bound over the elements (NaN where both are NaN counts as equal; NaN in one is inf)."""
    got, want, bound = (np.asarray(a, dtype=np.float64) for a in (got, want, bound))
    both = np.isnan(got) & np.isnan(want)
    with np.errstate(invalid="ignore", divide="ignore"):
        r = np.abs(got - want) / bound
    r = np.where(both, 0.0, np.where(np.isnan(r), np.inf, r))
    r = np.where((got == want) & ~both, 0.0, r)
    return float(r.max()) if r.size else 0.0


# ------------------------------------------------------------------------------------------------ fp32 simulations
def _sum32(a, axis, order):
    a = np.moveaxis(np.asarray(a, dtype=np.float32), axis, 0)
    if order == "seq":
        s = np.zeros(a.shape[1:], np.float32)
        for v in a:
            s = (s + v).astype(np.float32)
        return s
    n = a.shape[0]
    p = 1
    while p < n:
        p *= 2
    a = np.concatenate([a, np.zeros((p - n,) + a.shape[1:], np.float32)])
    while a.shape[0] > 1:
        a = (a[0::2] + a[1::2]).astype(np.float32)
    return a[0]


def simulate(case, d, order):
    """The case's outputs computed in numpy float32 with a plausible summation order ('seq' or 'pair')."""
    k = case["kind"]
    f = np.float32
    if k in ("stats", "finalize"):
        if k == "finalize":
            p = d["partial"]
            parts = [(min(case["tb"], case["T"] - j * case["tb"]), p[j, :, :case["C"]], p[j, :, case["C"]:])
                     for j in range(p.shape[0])]
            lens = np.full(case["B"], case["T"])
        else:
            lens = d["lengths"]
            parts = None
        B, C = case["B"], case["C"]
        m_out, s_out = np.zeros((B, C), f), np.zeros((B, C), f)
        for n in np.unique(lens):               # the utterances of one length together
            b = np.nonzero(lens == n)[0]
            n = int(n)
            if parts is None:
                xb = d["x"][b, :n]
                pb = []
                for t0 in range(0, n, SLAB):
                    blk = xb[:, t0:t0 + SLAB]
                    mk = (_sum32(blk, 1, order) * f(1.0 / blk.shape[1])).astype(f)
                    dv = (blk - mk[:, None]).astype(f)
                    pb.append((blk.shape[1], mk, _sum32(dv * dv, 1, order)))
            else:
                pb = [(nk, mk[b], qk[b]) for nk, mk, qk in parts]
            rn, rm, rq = f(0), np.zeros((len(b), C), f), np.zeros((len(b), C), f)
            for nk, mk, qk in pb:
                tot = f(rn + nk)
                wb = f(f(nk) / tot)
                cross = f(rn * wb)
                dd = (mk - rm).astype(f)
                rm = (rm + dd * wb).astype(f)
                rq = (rq + (qk + (dd * dd).astype(f) * cross).astype(f)).astype(f)
                rn = tot
            m_out[b] = rm
            with np.errstate(divide="ignore", invalid="ignore"):
                if case["mode"] == 0:
                    s_out[b] = np.sqrt(np.maximum(rq * f(1.0 / n), f(case["eps"])))
                else:
                    s_out[b] = np.sqrt(rq * f(1.0 / (n - 1)) + f(case["eps"]) if n > 1 else rq * f(np.inf) + f(case["eps"]))
        return {"mean": m_out, "std": s_out}
    if k in ("attn", "head"):
        Lg, X, mult = attn_operands(case, d)
        Lg, X = Lg.astype(f), X.astype(f)
        n = X.shape[1]
        with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
            if order == "seq":            # online softmax, frame by frame
                m = np.full(X.shape[::2], -np.inf, f)
                s0, s1, s2 = (np.zeros(X.shape[::2], f) for _ in range(3))
                for t in range(n):
                    l = Lg[:, t]
                    ok = np.isfinite(l)
                    mn = np.where(ok, np.maximum(m, l), m)
                    sc = np.exp((m - mn).astype(f)).astype(f)
                    sc = np.where(np.isnan(sc), f(0), sc)
                    e = np.where(ok, np.exp((l - mn).astype(f)).astype(f), f(0))
                    xv = X[:, t]
                    s0 = (s0 * sc + e).astype(f)
                    s1 = (s1 * sc + (e * xv).astype(f)).astype(f)
                    s2 = (s2 * sc + ((e * xv).astype(f) * xv).astype(f)).astype(f)
                    m = mn
            else:                          # max first, then pairwise sums
                mx = np.where(np.isfinite(Lg), Lg, -np.inf).max(axis=1, keepdims=True)
                e = np.where(np.isfinite(Lg), np.exp((Lg - mx).astype(f)), 0).astype(f)
                s0 = _sum32(e, 1, order)
                s1 = _sum32((e * X).astype(f), 1, order)
                s2 = _sum32(((e * X).astype(f) * X).astype(f), 1, order)
            mu = (s1 / s0).astype(f)
            if case.get("unweighted"):
                T = case["T"]
                u1, u2 = _sum32(X, 1, order), _sum32((X * X).astype(f), 1, order)
                var = (((u2 - (f(2) * mu * u1).astype(f)).astype(f) / f(T)).astype(f) + (mu * mu).astype(f)).astype(f)
            else:
                var = ((s2 / s0).astype(f) - (mu * mu).astype(f)).astype(f)
            return {"mean": mu, "std": np.sqrt(np.maximum(var, f(case["floor"])))}
    if k == "lde":
        T = case["T"]
        x = d["x"][:, :T]
        mu, nb = d["mu"], d["neg_beta"]
        r = (x[:, :, :, None] - mu[None, None]).astype(f)
        dist = _sum32((r * r).astype(f), 2, order)
        l = (nb * dist).astype(f)
        e = np.exp((l - l.max(axis=2, keepdims=True)).astype(f)).astype(f)
        w = (e / _sum32(e, 2, order)[:, :, None]).astype(f)
        acc = _sum32((w[:, :, None, :] * r).astype(f), 1, order)
        return {"e": (acc * f(1.0 / T)).astype(f).reshape(case["B"], -1)}
    T = case["T"]
    return {"mean": (_sum32(d["x"][:, :T], 1, order) / f(T)).astype(f)}
