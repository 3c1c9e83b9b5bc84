"""Exact-arithmetic operands, case catalogue and references for the back end's CUDA-core kernels (csrc/scoring.cu):
center_length_norm, column_mean, speaker_mean, cosine / bilinear trials, the plda_terms row term, topn_mean_std(_ddof),
topn_indices, snorm_trials, snorm_cross_trials, center_rows_transposed, plda_em_rows, plda_normalize_rows and
plda_llr_operands.

Every operand is chosen so that each sum a kernel forms is exact in any order: small integers or multiples of 2^-3, far
below 2^24 (fp32 sums) or 2^53 (fp64 sums).  What is left, the divisions, square roots and conversions, is correctly
rounded in IEEE fp32 / fp64, and numpy rounds it the same way in the kernel's order, so the references below are bit
patterns, not tolerances.  The library builds with nvcc's -fmad=true, so the compiler may fuse a * b + c; every product
that could be fused is exact here (`fma_free_*` assert it), which makes the fused and the unfused result the same.  Two
places keep a rounding that depends on the order: plda_normalize_rows' Kaldi weights 1 / (psi + 1 / n) are arbitrary
fp32 values, so `warp_sum_f32` reproduces the kernel's order (each lane adds its columns in turn, then the xor
butterfly), and topn_mean_std's fp64 sum of squared deviations, which is exact only where `topn_stats` says so
(else within 1 ulp of the fp64 result rounded to fp32).  Only logf in plda_llr_operands' row term gets a bound
(`llr_term_ref_and_bound`).

Plain numpy (no torch, no GPU): test_gpu_backend_edges.py moves these operands to the device, and
test_backend_exact_host.py checks the catalogue, the preconditions and the references on the CPU."""
import zlib

import numpy as np

U32 = 2.0 ** -24
WARP = 32
ROWS_PER_CTA = 8                 # one warp per row / trial, 256-thread CTAs
TOPN_THREADS = 512
TOPN_MAX = 32768                 # cohort entries one CTA sorts (xvb_topn_mean_std)
TOPN_IDX_MAX = 16384             # (score, index) pairs one CTA sorts (xvb_topn_indices)
SNORM_THREADS, SNORM_CTAS_PER_SM = 256, 16
COLUMN_PARTIALS_PER_SM = 4
COLUMN_BLOCK_CAP, SPEAKER_BLOCK_CAP = 512, 256
TILE = 32                        # center_rows_transposed / plda_em_rows: 32 x 32 tiles, 32 x 8 threads

ROW_D = (1, 31, 32, 33, 64, 65, 192, 600)
ROW_N = (1, 7, 8, 9, 4095, 4097)
PLDA_TERMS_D = (4, 32, 36, 64, 192, 600)          # xvb_plda_terms takes D % 4 == 0 (its GEMM)
COLUMN_D = (1, 33, 511, 512, 513, 1500)
SPEAKER_D = (1, 255, 256, 257, 600)
TOPN_NCOH = (1, 2, 3, 31, 32, 33, 511, 512, 513, 16385, 32767, 32768)
TOPN_IDX_NCOH = (1, 2, 3, 33, 1000, 16383, 16384)
CROSS_TOP_N = (2, 31, 32, 33, 64, 300)
TRANSPOSE_DIMS = (1, 31, 32, 33, 100)


def rng_for(name):
    return np.random.RandomState(zlib.crc32(name.encode()) & 0x7FFFFFFF)


def f32(a):
    return np.asarray(a, dtype=np.float32)


def next_pow2(n):
    p = 1
    while p < n:
        p <<= 1
    return p


def warp_sum_f32(t):
    """(rows, D) fp32 terms -> (rows,) fp32 in the order of a one-warp-per-row kernel: lane l adds t[:, l], t[:, l + 32],
    ... in turn starting from 0, then s += shfl_xor(s, o) for o = 16, 8, 4, 2, 1 (every lane ends with the same value)."""
    rows, D = t.shape
    L = -(-D // WARP) * WARP
    pad = np.zeros((rows, L), np.float32)
    pad[:, :D] = t
    lanes = np.zeros((rows, WARP), np.float32)
    for j in range(L // WARP):
        lanes = lanes + pad[:, j * WARP:(j + 1) * WARP]
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[:, np.arange(WARP) ^ o]
    return lanes[:, 0]


def exact_in_f32(a):
    """float64 values that fp32 holds exactly"""
    a = np.asarray(a, dtype=np.float64)
    return bool(np.array_equal(a.astype(np.float32).astype(np.float64), a))


# ------------------------------------------------------------------------------------------------ one warp per row
def row_cases():
    """name -> one-warp-per-row case: every D of ROW_D with every row / trial count of ROW_N (the last CTA of 8 warps is
    partial at 1, 7, 9, 4095 and 4097), with the optional operands cycling so that each is present and absent at every
    count."""
    return {"D{}_n{}".format(D, n): dict(D=D, n=n, variant=(i + j) % 4) for i, D in enumerate(ROW_D) for j, n in enumerate(ROW_N)}


def plda_terms_cases():
    return {"D{}_n{}".format(D, n): dict(D=D, n=n) for D in PLDA_TERMS_D for n in ROW_N}


def center_length_norm_operands(case, name):
    """x = v + m with integer v (every row nonzero) and integer m (or no mean, variant odd).  Every third row is a
    power-of-4 row, v = +-2^j on one column, whose norm is exact end to end (y = +-1)."""
    rng = rng_for("cln" + name)
    n, D = case["n"], case["D"]
    v = rng.randint(-8, 9, (n, D)).astype(np.float32)
    for r in range(0, n, 3):
        v[r] = 0
        v[r, (r // 3) % D] = (-1) ** r * 2.0 ** (r % 5)
    zero = ~v.any(axis=1)
    v[zero, 0] = 1
    mean = None if case["variant"] % 2 else f32(rng.randint(-4, 5, D))
    x = v + (mean if mean is not None else 0)
    return dict(x=f32(x), mean=mean, v=v)


def center_length_norm_ref(op):
    v = op["v"]
    ss = (v.astype(np.float64) ** 2).sum(axis=1)
    assert ss.max() < 2 ** 24 and exact_in_f32(ss)       # integer sum: exact in any order, fmaf or not
    inv = np.float32(1.0) / np.sqrt(f32(ss))
    return v * inv[:, None]


TRIAL_SETS = 37


def trials_operands(case, name):
    """Integer embeddings and row / column terms.  variant 0: cosine_trials (no terms); 1: row term only; 2: column term
    only; 3: both."""
    rng = rng_for("trials" + name)
    D, n, var = case["D"], case["n"], case["variant"]
    e = f32(rng.randint(-8, 9, (TRIAL_SETS, D)))
    t = f32(rng.randint(-8, 9, (TRIAL_SETS + 5, D)))
    te = rng.randint(0, TRIAL_SETS, n).astype(np.int32)
    tt = rng.randint(0, TRIAL_SETS + 5, n).astype(np.int32)
    row = f32(rng.randint(-100, 101, TRIAL_SETS)) if var in (1, 3) else None
    col = f32(rng.randint(-100, 101, TRIAL_SETS + 5)) if var in (2, 3) else None
    return dict(e=e, t=t, te=te, tt=tt, row=row, col=col)


def trials_ref(op):
    s = (op["e"][op["te"]].astype(np.float64) * op["t"][op["tt"]]).sum(axis=1)
    if op["row"] is not None:
        s = s + op["row"][op["te"]]
    if op["col"] is not None:
        s = s + op["col"][op["tt"]]
    assert np.abs(s).max() < 2 ** 24
    return f32(s)


def plda_terms_operands(case, name):
    rng = rng_for("terms" + name)
    D, n = case["D"], case["n"]
    g = rng.randint(-2, 3, (D, D))
    return dict(x=f32(rng.randint(-3, 4, (n, D))), gamma=f32(np.triu(g) + np.triu(g, 1).T), c=f32(rng.randint(-4, 5, D)))


def plda_terms_ref(op):
    x = op["x"].astype(np.float64)
    y = x @ op["gamma"].astype(np.float64).T           # the GEMM: exact integers well below 2^24, bf16 hi planes exact
    assert np.abs(y).max() < 256 * 64 and exact_in_f32(op["x"]) and np.abs(op["gamma"]).max() <= 2
    term = (x * (y + op["c"])).sum(axis=1)
    assert np.abs(term).max() < 2 ** 24 and np.abs(y + op["c"]).max() < 2 ** 24
    return f32(term)


def plda_normalize_operands(case, name):
    """x in {-2..2} (nonzero rows), so x * x in {0, 1, 4} and x * x * r is exact for any fp32 r.  variant & 1: Kaldi form
    (simple 0); variant & 2: num_examples given (arbitrary fp32 counts)."""
    rng = rng_for("pnorm" + name)
    n, D, var = case["n"], case["D"], case["variant"]
    x = f32(rng.randint(-2, 3, (n, D)))
    x[~x.any(axis=1), 0] = 2
    psi = f32(rng.uniform(0.0, 3.0, D))
    num = f32(rng.uniform(1.0, 20.0, n)) if var & 2 else None
    return dict(x=x, psi=psi, num=num, simple=0 if var & 1 else 1)


def fma_free_normalize(op):
    """x * x * r rounds to itself: the fused x * x * r + s equals the unfused one."""
    x2 = op["x"].astype(np.float64) ** 2
    return set(np.unique(x2)) <= {0.0, 1.0, 4.0}


def plda_normalize_ref(op):
    x = op["x"]
    n, D = x.shape
    if op["simple"]:
        t = x * x
    else:
        inv_n = np.float32(1.0) / op["num"] if op["num"] is not None else np.ones(n, np.float32)
        r = np.float32(1.0) / (op["psi"][None, :] + inv_n[:, None])
        t = (x * x) * r
    s = warp_sum_f32(f32(t))
    f = np.sqrt(np.float32(D) / s)
    return x * f[:, None]


# plda_llr_operands
LLR_NP = (0.0, 0.5, 1.0, 1.5, 3.0, 7.0)


def llr_operands(case, name):
    """side = variant & 1; num_examples given when variant & 2.  n and psi are dyadic with n * psi in LLR_NP, so
    nn * p + 1 is the same fused or not (`fma_free_llr`); x are integers."""
    rng = rng_for("llr" + name)
    n, D, var = case["n"], case["D"], case["variant"]
    psi = f32(rng.choice([0.0, 0.5, 1.0, 1.5, 3.0], D))
    num = f32(rng.choice([1.0, 2.0], n)) if var & 2 else None
    return dict(x=f32(rng.randint(-8, 9, (n, D))), psi=psi, num=num, side=var & 1)


def fma_free_llr(op):
    nn = op["num"] if (op["side"] == 0 and op["num"] is not None) else np.ones(op["x"].shape[0], np.float32)
    prod = nn.astype(np.float64)[:, None] * op["psi"].astype(np.float64)[None, :]
    return exact_in_f32(prod)


def llr_emulate(op):
    """-> (operand (n, 2D) fp32 bit-exact, log arguments (n, D) fp32, other addends (n, D) fp32) in the kernel's order."""
    x, p = op["x"], op["psi"][None, :]
    n, D = x.shape
    if op["side"] == 0:
        nn = (op["num"] if op["num"] is not None else np.ones(n, np.float32))[:, None]
        den = nn * p + np.float32(1.0)
        m = nn * p / den * x
        v = np.float32(1.0) + p / den
        a = np.concatenate([np.float32(-0.5) / v, m / v], axis=1)
        return a, v, m * m / v
    q = p + np.float32(1.0)
    return np.concatenate([x * x, x], axis=1), np.broadcast_to(q, x.shape), x * x / q


LLR_LOGF_ULPS = 2.0       # logf's error in ulps of its result (CUDA documents 1)
LLR_SUM_SLACK = 2.0       # over the first-order bound of the fp32 summation


def ulp32(a):
    a = np.abs(np.asarray(a, dtype=np.float32))
    return (np.spacing(a).astype(np.float64))


def llr_term_ref_and_bound(op):
    """term = -+1/2 sum_d (log v_d + q_d) in fp64 from the kernel's own fp32 v and q; bound = 1/2 (sum of logf errors +
    summation error): each addend passes through one add with q, ceil(D / 32) lane adds and 5 butterfly adds."""
    _, v, q = llr_emulate(op)
    lg = np.log(v.astype(np.float64))
    terms = lg + q
    D = v.shape[1]
    depth = 1 + -(-D // WARP) + 5
    ref = 0.5 * terms.sum(axis=1) * (-1.0 if op["side"] == 0 else 1.0)
    bound = 0.5 * (LLR_LOGF_ULPS * ulp32(lg).sum(axis=1) +
                   LLR_SUM_SLACK * depth * U32 * (np.abs(lg) + np.abs(q)).sum(axis=1))
    return ref, bound


# ------------------------------------------------------------------------------------------------ column / speaker mean
def column_cases(sms):
    """rows on both sides of G = 4 SMs partial rows (and far above it), D on both sides of the 512-thread block cap"""
    G = COLUMN_PARTIALS_PER_SM * sms
    rows = {"1": 1, "2": 2, "Gm1": G - 1, "G": G, "Gp1": G + 1, "10Gp3": 10 * G + 3}
    return {"r{}_D{}".format(k, D): dict(rows=r, D=D, G=G) for k, r in rows.items() for D in COLUMN_D}


def column_operands(case, name):
    return dict(x=f32(rng_for("col" + name).randint(-512, 513, (case["rows"], case["D"])) / 8.0))


def column_ref(op):
    s = op["x"].astype(np.float64).sum(axis=0)          # multiples of 1/8 below 2^20: exact in any order
    return f32(s / op["x"].shape[0])


SPEAKER_COUNTS = (0, 1, 5, 0, 40, 2, 1, 0)


def speaker_cases():
    return {"D{}".format(D): dict(D=D) for D in SPEAKER_D}


def speaker_operands(case, name):
    """50 rows of multiples of 1/8; speakers with 0, 1 and many members (first, middle and last ones empty or not),
    member lists unsorted with repeats."""
    rng = rng_for("spk" + name)
    N, D = 50, case["D"]
    counts = np.array(SPEAKER_COUNTS)
    members = rng.randint(0, N, counts.sum()).astype(np.int32)
    members[1:3] = members[0]                           # repeats
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    return dict(x=f32(rng.randint(-800, 801, (N, D)) / 8.0), off=off, members=members)


def speaker_ref(op):
    x, off, mem = op["x"].astype(np.float64), op["off"], op["members"]
    out = np.zeros((len(off) - 1, x.shape[1]), np.float32)
    for s in range(len(off) - 1):
        if off[s + 1] > off[s]:
            out[s] = f32(x[mem[off[s]:off[s + 1]]].sum(axis=0) / (off[s + 1] - off[s]))
    return out


# ------------------------------------------------------------------------------------------------ top-n statistics
def topn_tops(ncoh):
    return sorted({0, 1, 2, 3, max(ncoh - 1, 0), ncoh, ncoh + 7})


def topn_cases():
    return {"c{}".format(c): dict(ncoh=c) for c in TOPN_NCOH}


def topn_rows(ncoh, name, unit=8):
    """rows (unit = 1 / 8 grid) as integers k: 0 random in [-8, 8] (ties at every cut), 1 all equal, 2 distinct (a
    permutation), 3 descending with a tie block centred on ncoh / 2.  Returned as integers and as fp32 k / unit."""
    rng = rng_for("topn" + name)
    k = np.empty((4, ncoh), np.int64)
    k[0] = rng.randint(-8, 9, ncoh)
    k[1] = 3
    k[2] = rng.permutation(ncoh) - ncoh // 2
    k[3] = np.sort(rng.randint(-8, 9, ncoh))[::-1]
    k[3, max(0, ncoh // 2 - 2):ncoh // 2 + 3] = 1
    return k, f32(k / float(unit))


def topn_stats(k, n, ddof, unit=8):
    """(mean fp32, std fp32 reference, std exact?) of the n largest of the integer row k (values k / unit).  The kernel's
    fp64 sum is exact (integers / 8), so mu = fl64(s1 / n) is the kernel's mu and the mean is bit-exact.  The sum of
    squares of d = x - mu is exact in any order when mu is exact (n a power of two) and the scaled total
    sum (n k - s1)^2 fits 53 bits; then the std is bit-exact, otherwise the fp64 value is the reference within 1 ulp."""
    top = np.sort(k)[::-1][:n]
    K = int(top.sum())
    mu = (K / unit) / n
    scaled = [int(n * int(t) - K) for t in top]         # d * unit * n, integers
    ss = sum(v * v for v in scaled)
    pow2 = n & (n - 1) == 0
    exact = pow2 and ss < 2 ** 53
    s2 = ss / float(unit * n) ** 2                      # correctly rounded (exact when `exact`)
    with np.errstate(invalid="ignore", divide="ignore"):
        std = np.sqrt(np.float64(s2) / np.float64(n - ddof))
    return np.float32(mu), np.float32(std), exact


def topn_select_n(ncoh, top_n):
    return top_n if 0 < top_n < ncoh else ncoh


def topn_idx_cases():
    return {"c{}".format(c): dict(ncoh=c) for c in TOPN_IDX_NCOH}


def topn_idx_tops(ncoh):
    return sorted({1, min(2, ncoh), ncoh})


def topn_idx_ref(rows, top_n):
    return np.stack([np.argsort(-r, kind="stable")[:top_n] for r in rows]).astype(np.int32)


# ------------------------------------------------------------------------------------------------ score normalisation
def snorm_trials_count(sms):
    """more trials than one grid-stride round of the capped grid covers"""
    return SNORM_THREADS * SNORM_CTAS_PER_SM * sms + 12345


def snorm_operands(n, name):
    """arbitrary fp32 scores and statistics: the kernel's expression has no product next to a sum, so numpy's fp32
    evaluation in the same order is its bit pattern"""
    rng = rng_for("snorm" + name)
    Ne, Nt = 300, 211
    return dict(s=f32(rng.standard_normal(n) * 3), te=rng.randint(0, Ne, n).astype(np.int32),
                tt=rng.randint(0, Nt, n).astype(np.int32), me=f32(rng.standard_normal(Ne)), se=f32(rng.uniform(0.5, 2, Ne)),
                mt=f32(rng.standard_normal(Nt)), st=f32(rng.uniform(0.5, 2, Nt)))


def snorm_ref(op):
    v = op["s"]
    return np.float32(0.5) * ((v - op["me"][op["te"]]) / op["se"][op["te"]] + (v - op["mt"][op["tt"]]) / op["st"][op["tt"]])


CROSS_NCOH = 700
CROSS_TRIALS = (1, 7, 8, 9, 4097, 300)


def cross_cases():
    return {"n{}_t{}".format(top_n, nt): dict(top_n=top_n, trials=nt) for top_n, nt in zip(CROSS_TOP_N, CROSS_TRIALS)}


def _pair_sets(rng, rows, top_n):
    """index sets of top_n cohort entries made of pairs (3m, 3m + 1) and, for odd top_n, one 3m + 2, shuffled"""
    out = np.empty((rows, top_n), np.int32)
    for r in range(rows):
        m = rng.choice(CROSS_NCOH // 3, top_n // 2 + 1, replace=False)
        idx = np.concatenate([3 * m[:-1], 3 * m[:-1] + 1] + ([[3 * m[-1] + 2]] if top_n % 2 else []))
        out[r] = rng.permutation(idx)
    return out


def cross_operands(case, name):
    """Cohort rows c + a w_j with w_j = +1, -1, 0 for j = 0, 1, 2 mod 3, integer c and a power of two a; every top-n set
    is whole (+1, -1) pairs plus at most one w = 0 entry, so each set's fp64 sum is top_n c exactly, its mean c, its
    deviations +-a and 0 and their squares exact: only the final sqrt, divisions and conversion round."""
    rng = rng_for("cross" + name)
    top_n, n = case["top_n"], case["trials"]
    Ne, Nt = 40, 30
    w = np.array([1.0, -1.0, 0.0])[np.arange(CROSS_NCOH) % 3]

    def cohort(rows):
        c = rng.randint(-20, 21, rows).astype(np.float64)
        a = 2.0 ** rng.randint(-1, 3, rows)
        return c, a, f32(c[:, None] + a[:, None] * w[None, :])

    ce, ae, ec = cohort(Ne)
    ct, at, tc = cohort(Nt)
    return dict(s=f32(rng.standard_normal(n) * 4), te=rng.randint(0, Ne, n).astype(np.int32),
                tt=rng.randint(0, Nt, n).astype(np.int32), ec=ec, tc=tc, top_e=_pair_sets(rng, Ne, top_n),
                top_t=_pair_sets(rng, Nt, top_n), top_n=top_n, ce=ce, ae=ae, ct=ct, at=at)


def cross_ref(op):
    n = op["top_n"]

    def stats(row, idx):
        vals = row[idx].astype(np.float64)
        assert vals.sum() == n * vals.mean() and exact_in_f32(vals)
        mu = vals.sum() / n
        s2 = ((vals - mu) ** 2).sum()
        return mu, np.sqrt(s2 / (n - 1))

    out = np.empty(len(op["s"]), np.float32)
    for i, (e, t) in enumerate(zip(op["te"], op["tt"])):
        me, se = stats(op["ec"][e], op["top_t"][t])
        mt, st = stats(op["tc"][t], op["top_e"][e])
        v = np.float64(op["s"][i])
        out[i] = np.float32(0.5 * ((v - me) / se + (v - mt) / st))
    return out


def cross_exact(op):
    """every top-n set's mean is its row's c and its deviations are +-a or 0"""
    for row_c, row_a, rows, sets_of in ((op["ce"], op["ae"], op["ec"], op["top_t"]), (op["ct"], op["at"], op["tc"], op["top_e"])):
        for r in range(rows.shape[0]):
            for idx in sets_of:
                d = rows[r, idx].astype(np.float64) - row_c[r]
                if d.sum() != 0 or not set(np.unique(np.abs(d))) <= {0.0, row_a[r]}:
                    return False
    return True


# ------------------------------------------------------------------------------------------------ transposed PLDA rows
def transpose_cases():
    """N (or S), D over TRANSPOSE_DIMS (both sides of the 32 x 32 tile), weights absent / given alternately"""
    cases = {}
    i = 0
    for N in TRANSPOSE_DIMS:
        for D in TRANSPOSE_DIMS:
            cases["N{}_D{}".format(N, D)] = dict(N=N, D=D, weighted=bool(i % 2), ldo=N + 5)
            i += 1
    return cases


def center_T_operands(case, name):
    rng = rng_for("cT" + name)
    N, D, S = case["N"], case["D"], 5
    return dict(x=f32(rng.randint(-50, 51, (N, D))), spk=rng.randint(0, S, N).astype(np.int32),
                means=f32(rng.randint(-20, 21, (S, D))), sw=f32(rng.uniform(0.1, 3.0, S)) if case["weighted"] else None)


def center_T_ref(op):
    y = op["x"] - op["means"][op["spk"]]               # integers: exact
    if op["sw"] is not None:
        y = y * op["sw"][op["spk"]][:, None]
    return np.ascontiguousarray(f32(y).T)


EM_NK = (1.0, 3.0, 7.0, 15.0)


def em_operands(case, name):
    """psi in {0, 1} and n in {1, 3, 7, 15}: n psi / (1 + n psi) is 0 or 1 - 2^-j, so what = q u is exact for integer u
    and u - what is exact: fused or not, the same (`fma_free_em`).  Weights arbitrary fp32."""
    rng = rng_for("em" + name)
    S, D = case["N"], case["D"]
    return dict(u=f32(rng.randint(-64, 65, (S, D))), n=f32(rng.choice(EM_NK, S)),
                w=f32(rng.uniform(0.1, 4.0, S)) if case["weighted"] else None, psi=f32(rng.randint(0, 2, D)))


def em_emulate(op):
    nk = op["n"][:, None]
    p = op["psi"][None, :]
    wk = (op["w"] if op["w"] is not None else np.ones(len(op["n"]), np.float32))[:, None]
    q = nk * p / (np.float32(1.0) + nk * p)
    wh = q * op["u"]
    a = np.sqrt(wk) * wh
    b = np.sqrt(wk * nk) * (op["u"] - wh)
    return q, wh, np.ascontiguousarray(a.T), np.ascontiguousarray(b.T)


def fma_free_em(op):
    q, wh, _, _ = em_emulate(op)
    u = op["u"].astype(np.float64)
    return exact_in_f32(q.astype(np.float64) * u) and exact_in_f32(u - wh) and exact_in_f32(op["n"][:, None].astype(np.float64) * op["psi"][None, :])
