"""Exact-arithmetic operands, shape catalogue and float64 references for the two wgmma GEMM kernels (csrc/tdnn_gemm.cu:
the TDNN layer, fused pooling, score matrices and trial histogram; csrc/conv2d.cu: the 2-D convolution).

The kernels compute hi*hi + lo*hi + hi*lo from bf16 planes into fp32 accumulators.  The operands here are chosen so
that every one of those sums is exact in any order:
  * frame planes: hi holds integers with |hi| <= 2, lo holds multiples of 2^-8 with |lo| <= 3 * 2^-8;
  * weights: an integer part (|w| <= 2) and a 2^-8 part (|w| <= 3 * 2^-8), each bf16-exact, packed separately so that
    the real packer's layout is used and each part comes back as its own .hi plane;
  * every product is then a multiple of 2^-8, and as long as the sum of the absolute values of an output's terms stays
    below 2^15 (assert_exact_sum), every partial sum is a multiple of 2^-8 below 2^16: 24 significant bits, which
    fp32 holds exactly.  That allows K up to about 8000 (tdnn6's 3000 x 1 and the 3-tap layers fit);
  * bias, row / utterance terms, BN shifts and residuals are on the 2^-8 grid and BN scales are powers of two, so the
    epilogue is exact as well (exact_f32 asserts it for every reference).
The reference is sum(hx*hw + lx*hw + hx*lw) in float64; lo*lo is left out because the kernels never compute it.  Any
dropped term, shifted K step, wrong tap, swizzle or tile-edge mistake then moves an output by at least 2^-8.

Plain numpy (no torch, no GPU): the GPU file (test_gpu_gemm_edges.py) moves these operands to the device, and
test_gemm_exact_host.py checks the helpers and the precondition of every generated case on the CPU."""
import math

import numpy as np

GRID = 2.0 ** -8
EXACT_SUM_LIMIT = 2.0 ** 15     # sum of |terms| of one output, in units where the terms are multiples of 2^-8
U32 = 2.0 ** -24                # unit roundoff of fp32


# ------------------------------------------------------------------------------------------------ bf16 split
def bf16_round(x):
    """float32 -> nearest bf16 value (ties to even), as float32: __float2bfloat16_rn.  NaN maps to a quiet NaN."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) & 0xFFFF
    r = np.where(np.isnan(x), (u >> 16) | 0x40, r)
    return (r.astype(np.uint32) << 16).view(np.float32)


def split_bf16(x):
    """split_bf16 of common.cuh: hi = rn(x), lo = rn(x - hi), both as float32 arrays of bf16 values."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hi = bf16_round(x)
    lo = bf16_round(x - hi)      # x - hi is exact in fp32
    return hi, lo


def bf16_bits(x):
    """uint16 bit patterns of bf16-exact float32 values."""
    return (np.ascontiguousarray(x, dtype=np.float32).view(np.uint32) >> 16).astype(np.uint16)


# ------------------------------------------------------------------------------------------------ operands
def int_plane(rng, shape, lim=2):
    return rng.randint(-lim, lim + 1, shape).astype(np.float32)


def grid_plane(rng, shape, lim=3):
    """multiples of 2^-8 in [-lim, lim] * 2^-8"""
    return (rng.randint(-lim, lim + 1, shape) * GRID).astype(np.float32)


def grid_values(rng, shape, lim=2.0):
    """multiples of 2^-8 in [-lim, lim]: biases, shifts, row / utterance terms"""
    n = int(lim / GRID)
    return (rng.randint(-n, n + 1, shape) * GRID).astype(np.float32)


def pow2_scales(rng, n):
    return (2.0 ** rng.randint(-1, 2, n)).astype(np.float32)


def frame_planes(rng, shape):
    return int_plane(rng, shape), grid_plane(rng, shape)


def assert_exact_sum(k_eff, his, los, w_hi, w_lo):
    """Precondition: every output of a K = k_eff contraction has sum |terms| < 2^15.  Bounded from above by
    k_eff * (max|hx| max|hw| + max|lx| max|hw| + max|hx| max|lw|), which is what is asserted."""
    mh = max(float(np.max(np.abs(h))) for h in his)
    ml = max(float(np.max(np.abs(lo))) for lo in los)
    bound = k_eff * (mh * float(np.max(np.abs(w_hi))) + ml * float(np.max(np.abs(w_hi))) + mh * float(np.max(np.abs(w_lo))))
    assert bound < EXACT_SUM_LIMIT, "sum of |terms| may reach {} >= 2^15: fp32 accumulation would round".format(bound)
    return bound


def exact_f32(v):
    """float64 reference -> float32, asserting that no rounding happens (the epilogue stays exact)."""
    f = np.asarray(v, dtype=np.float64).astype(np.float32)
    assert np.array_equal(f.astype(np.float64), v), "reference not representable in fp32: the case is not exact"
    return f


def context_span(context):
    left = context[0] if context[0] < 0 else 0
    right = context[-1] if context[-1] > 0 else 0
    return left, right, right - left + 1


def shift_time(x, c):
    """x (B, T, C) -> x[:, t + c] with zeros outside [0, T) (F.pad of TdnnAffine)"""
    out = np.zeros_like(x)
    T = x.shape[1]
    lo, hi = max(0, -c), min(T, T - c)
    if hi > lo:
        out[:, lo:hi] = x[:, lo + c:hi + c]
    return out


# ------------------------------------------------------------------------------------------------ TDNN layer
def _ru(x, m):
    return (x + m - 1) // m * m


def _cdiv(a, b):
    return -(-a // b)


def layer_cases(sms):
    """name -> TDNN layer case for a GPU with `sms` SMs.  Shapes that target a kernel instance use T = 8 and B = 16 k:
    Tb = 8 x Bb = 16 then tiles the frames with no padding, so there are exactly k M tiles, and gemm_plan_build picks
    BLOCK_N 128 when Cout >= 128 and k * ceil(Cout / 128) >= sms, else 64 when Cout >= 64 and k * ceil(Cout / 64) >=
    sms / 2, else 32.  `inst` is the instance the shape is meant for (checked on the GPU from the kernel names)."""
    h = sms // 2
    D = dict
    ctx5 = [-2, -1, 0, 1, 2]
    cases = {
        # Cout tails on the 32-wide instance, odd Cout through the single-column stores, context span > T
        "w32_cin8_cout1_T2": D(B=5, T=2, Cin=8, Cout=1, ctx=[-3, 0, 3], relu=True, bn=True, planes=True, f32=True, inst=32),
        "w32_cin80_cout33_x2": D(B=4, T=29, Cin=80, Cout=33, ctx=ctx5, x2=True, relu=True, planes=True, f32=True, inst=32),
        "w32_cin56_cout48": D(B=32, T=8, Cin=56, Cout=48, ctx=ctx5, relu=True, bn=True, planes=True, inst=32),
        # 64-wide: N tails of 16 and 1
        "w64_cin40_cout80": D(B=16 * _cdiv(h, 2), T=8, Cin=40, Cout=80, ctx=[-3, 0, 3], relu=True, planes=True, f32=True, inst=64),
        "w64_cin24_cout129": D(B=16 * _cdiv(h, 3), T=8, Cin=24, Cout=129, ctx=[0], relu=True, bn=True, planes=True, f32=True,
                               inst=64),
        # 128-wide: N tails of 1 and 72
        "w128_cin136_cout129": D(B=16 * _cdiv(sms, 2), T=8, Cin=136, Cout=129, ctx=[-1, 0, 1], relu=True, planes=True,
                                 f32=True, inst=128),
        "w128_cin200_cout200": D(B=16 * _cdiv(sms, 2), T=8, Cin=200, Cout=200, ctx=[0], relu=True, bn=True, f32=True, inst=128),
        # more than 2 x sms tiles: the persistent loop runs several rounds
        "w128_persistent_cin72": D(B=16 * (sms + 1), T=8, Cin=72, Cout=256, ctx=[-1, 0, 1], relu=True, bn=True, planes=True,
                                   inst=128),
        # swish instances, one per width
        "swish32_cin200": D(B=3, T=21, Cin=200, Cout=40, ctx=[-2, 0, 2], relu=True, act="swish", bn=True, planes=True,
                            f32=True, inst=32),
        "swish64_cin16": D(B=16 * _cdiv(h, 2), T=8, Cin=16, Cout=72, ctx=[0], act="swish", planes=True, f32=True, inst=64),
        "swish128_cin64": D(B=16 * _cdiv(sms, 2), T=8, Cin=64, Cout=136, ctx=[0], act="swish", bn=True, planes=True,
                            f32=True, inst=128),
        # other epilogue flags
        "tanh_cin88": D(B=3, T=17, Cin=88, Cout=72, ctx=[-1, 0, 1], bn=True, act="tanh", planes=True, f32=True),
        "sigmoid_cin120": D(B=2, T=23, Cin=120, Cout=36, ctx=ctx5, act="sigmoid", planes=True, f32=True),
        "utt_row_cin104": D(B=3, T=19, Cin=104, Cout=100, ctx=[-2, 0, 2], utt=True, row=True, relu=True, bn=True,
                            planes=True, f32=True),
        "cin128_ctx_sparse": D(B=2, T=31, Cin=128, Cout=96, ctx=[-2, 0, 2], relu=True, planes=True),
        "cin64_T1_span": D(B=6, T=1, Cin=64, Cout=64, ctx=[-3, 0, 3], relu=True, planes=True, f32=True),
        # segment level, split-K (Cin tails of 8 and 56); run with XVB_SPLITK on and off
        "splitk_cin1544": D(B=9, T=1, Cin=1544, Cout=260, ctx=[0], relu=True, bn=True, planes=True, f32=True, splitk=True),
        "splitk_cin3000": D(B=130, T=1, Cin=3000, Cout=512, ctx=[0], relu=True, bn=True, f32=True, splitk=True),
    }
    # every frames-per-tile Tb of choose_m_tile (1 .. 128), ragged in T or B
    for tb, (b, t) in TB_SHAPES.items():
        cases["tb{}_B{}_T{}".format(tb, b, t)] = D(B=b, T=t, Cin=16, Cout=64, ctx=[-2, 0, 1] if t > 1 else [0],
                                                   relu=True, planes=True, f32=True, tb=tb)
    for c in cases.values():
        c.setdefault("ctx", [0])
        # poisoned channel slices: x starts at channel 8 of a wider buffer with NaN on both sides
        c["x_c0"] = 8
        c["ldx"] = _ru(c["x_c0"] + c["Cin"] + 8, 8)
        if c.get("x2"):
            c["x2_c0"] = 16
            c["ldx2"] = _ru(c["x2_c0"] + c["Cin"] + 24, 8)
            assert c["ldx2"] != c["ldx"]
        # fenced outputs: a channel slice at 8 (planes) / 4 (fp32) of a padded pitch, one spare utterance of rows
        c["y_c0"], c["ldy"] = 8, _ru(8 + c["Cout"] + 8, 8)
        c["yf_c0"], c["ldyf"] = 4, _ru(4 + c["Cout"] + 4, 4)
    return cases


# (B, T) -> Tb of choose_m_tile (tdnn_gemm.cu), read back through xvb_pool_partial_blocks by the tests
TB_SHAPES = {1: (100, 3), 2: (65, 2), 4: (70, 3), 8: (17, 7), 16: (10, 13), 32: (5, 27), 64: (3, 50), 128: (2, 97)}


def make_layer(case, seed):
    """Operands of a layer case: dict of numpy arrays."""
    rng = np.random.RandomState(seed)
    B, T, Cin, Cout, ctx = case["B"], case["T"], case["Cin"], case["Cout"], case["ctx"]
    _, _, tot = context_span(ctx)
    d = {"xs": [frame_planes(rng, (B, T, Cin)) for _ in range(2 if case.get("x2") else 1)],
         "w_int": int_plane(rng, (Cout, Cin, tot)), "w_frac": grid_plane(rng, (Cout, Cin, tot)),
         "bias": grid_values(rng, Cout)}
    if case.get("bn"):
        d["scale"], d["shift"] = pow2_scales(rng, Cout), grid_values(rng, Cout)
    if case.get("utt"):
        d["utt"] = grid_values(rng, (B, Cout))
    if case.get("row"):
        d["row"] = grid_values(rng, B * T)
    return d


def taps_of(w, context):
    """(Cout, Cin, tot) reference weight -> (Cout, ntaps, Cin) of the kept taps"""
    left, _, _ = context_span(context)
    return np.ascontiguousarray(w[:, :, [c - left for c in context]].transpose(0, 2, 1))


def layer_acc(d, context):
    """float64 sum of hx*hw + lx*hw + hx*lw over sources, taps and channels: (B, T, Cout)"""
    wh, wl = taps_of(d["w_int"], context), taps_of(d["w_frac"], context)
    B, T, Cin = d["xs"][0][0].shape
    assert_exact_sum(len(d["xs"]) * len(context) * Cin, [h for h, _ in d["xs"]], [lo for _, lo in d["xs"]], wh, wl)
    acc = np.zeros((B * T, wh.shape[0]))
    for hi, lo in d["xs"]:
        for j, c in enumerate(context):
            sh = shift_time(hi, c).reshape(-1, Cin).astype(np.float64)
            sl = shift_time(lo, c).reshape(-1, Cin).astype(np.float64)
            acc += (sh + sl) @ wh[:, j].T.astype(np.float64) + sh @ wl[:, j].T.astype(np.float64)
    return acc.reshape(B, T, -1)


def layer_reference(case, d, acc=None):
    """-> (want, bound): the float64 output of the layer epilogue (+bias, row / utterance terms -> ReLU -> swish -> BN ->
    tanh / sigmoid), and None when it is exact (float32 array then) or the per-element bound of a transcendental one.
    acc: the (B, T, Cout) float64 contraction when it is not layer_acc's (grouped layers)."""
    v = (layer_acc(d, case["ctx"]) if acc is None else acc) + d["bias"][None, None, :].astype(np.float64)
    B, T = case["B"], case["T"]
    if "row" in d:
        v = v + d["row"].reshape(B, T)[:, :, None]
    if "utt" in d:
        v = v + d["utt"][:, None, :]
    if case.get("relu"):
        v = np.maximum(v, 0.0)
    act = case.get("act")
    scale = d["scale"].astype(np.float64) if "scale" in d else None
    if act is None:
        if scale is not None:
            v = v * scale + d["shift"]
        return exact_f32(v), None
    pre = exact_f32(v).astype(np.float64)      # everything before the activation is exact
    if act == "swish":
        # swish(u) = u / (1 + expf(-u)).  expf is within 2 ulp (CUDA C Programming Guide, single-precision functions),
        # i.e. a relative error <= 2^-22; 1 + e and the division each round once (<= 2^-24 relative), so the result is
        # within 2^-22 + 2 * 2^-24 < 2^-21 of swish(u), relative.  Where expf(-u) overflows (u < -88.7) the kernel returns
        # -0 for a true value below 2^-120 in magnitude.  The BN that follows multiplies that error by |scale| and adds
        # one fp32 rounding of its own result (fmaf, <= 2^-24 relative).
        sw = pre / (1.0 + np.exp(-pre))
        err = 2.0 ** -21 * np.abs(sw) + 2.0 ** -120
        if scale is not None:
            out = sw * scale + d["shift"]
            return out, err * scale + 2.0 ** -24 * np.abs(out)
        return sw, err
    if scale is not None:
        pre = pre * scale + d["shift"]          # exact: power-of-two scale, 2^-8 shift
        exact_f32(pre)
    if act == "tanh":
        # tanhf is within 2 ulp; ulp(y) <= 2^-23 |y| for normal y, and |tanh(u)| >= 2^-10 / 2 for the nonzero grid values
        out = np.tanh(pre)
        return out, 2.0 * 2.0 ** -23 * np.abs(out) + 2.0 ** -126
    if act == "sigmoid":
        # 1 / (1 + expf(-u)): expf within 2 ulp (2^-22 relative), its error shrinks by e / (1 + e) < 1 in 1 + e, which
        # rounds once (2^-24), and the division rounds once (2^-24): < 2^-21 relative.  Overflow of expf(-u)
        # (u < -88.7) returns 0 for a true value below 2^-120.
        out = 1.0 / (1.0 + np.exp(-pre))
        return out, 2.0 ** -21 * out + 2.0 ** -120
    raise ValueError(act)


# ------------------------------------------------------------------------------------------------ fused pooling
# (B, T, Cout): every Tb, plus T = 1 (the Tb == 1 single-frame path); Cout % 128 in {4, 64, 124}
POOL_CASES = [(5, 1, 132), (100, 3, 192), (65, 2, 124), (70, 3, 132), (17, 7, 192), (10, 13, 124), (5, 27, 132),
              (3, 50, 192), (2, 97, 124), (1, 137, 132)]
POOL_CIN, POOL_CTX = 72, [-1, 0, 1]


def pool_case(B, T, Cout):
    return dict(B=B, T=T, Cin=POOL_CIN, Cout=Cout, ctx=POOL_CTX, relu=True, bn=True, x_c0=8, ldx=_ru(8 + POOL_CIN + 8, 8))


def pool_reference(y, tb, eps=1e-10):
    """Statistics of the exact layer output y (B, T, C) float64 -> (mean, var, mean_bound, var_bound), per (b, c).

    The kernel pools in fp32 through Chan et al.'s merge: pairs of frames, then tree merges inside a time block of Tb
    frames (log2 Tb levels, two of them quad shuffles), then xvb_pool_finalize merges the nblk = ceil(T / Tb) blocks one
    after the other.  An element passes through at most L = log2(Tb) + nblk + 2 merges.
      mean: a merge is the convex combination mean_a + (mean_b - mean_a) * wb; with wb, the difference and the fma each
        rounded once it adds at most 4 u max|y| to the larger of its inputs' errors (u = 2^-24), so
        |d mean| <= 4 L u max|y|; asserted with a factor of 2 to spare.
      M2: M2_a + M2_b + d^2 n_a n_b / (n_a + n_b).  The roundings of the sums and the product are relative to terms that
        add up to at most T max|y|^2 (<= 7 L u T max|y|^2 in all), and the error of d (<= 2 |d mean|) enters as
        2 |d| |dd| min(n_a, n_b) <= 32 L u max|y|^2 min(n_a, n_b).  Summed over the merge tree, min(n_a, n_b) adds up to
        at most T (log2 Tb + 2).  Divided by T: |d var| <= (32 (log2 Tb + 2) + 7) L u max|y|^2, asserted with 2x.
    The std is checked through its square: sqrt and squaring add 2^-22 relative."""
    B, T, C = y.shape
    nblk = -(-T // tb)
    L = math.log2(tb) + nblk + 2
    m = np.abs(y).max(axis=1)
    mean = y.mean(axis=1)
    var = np.maximum(((y - mean[:, None, :]) ** 2).mean(axis=1), eps)
    return mean, var, 8 * L * U32 * m, 2 * (32 * (math.log2(tb) + 2) + 7) * L * U32 * m * m


# ------------------------------------------------------------------------------------------------ score GEMMs
SCORE_DIMS = [8, 40, 150, 200]
PLDA_DIMS = [8, 40, 148, 200]    # xvb_plda_matrix needs D % 4 == 0 (its first GEMM writes a (Ne, D) fp32 matrix)


def score_operands(seed, n_rows, D, lim=2):
    rng = np.random.RandomState(seed)
    return [int_plane(rng, (n, D), lim) for n in n_rows]


def int_matmul(a, b):
    """float64 a . b^T for integer operands, asserting the fp32 accumulation of the kernel is exact (|sums| < 2^23)."""
    bound = a.shape[1] * float(np.abs(a).max()) * float(np.abs(b).max())
    assert bound < 2.0 ** 23, bound
    return a.astype(np.float64) @ b.astype(np.float64).T


def histogram_reference(S, tgt, mask, lo, nbins):
    """Scores on the bin centres of unit-width bins starting at lo: bin = 1 + floor(s - lo), clamped to [0, nbins-1];
    (2, nbins) int64 [nontarget | target] of the masked entries."""
    b = np.clip(1 + np.floor(S - lo), 0, nbins - 1).astype(np.int64)
    out = np.zeros((2, nbins), dtype=np.int64)
    for cls in (0, 1):
        sel = mask & (tgt == bool(cls))
        out[cls] = np.bincount(b[sel], minlength=nbins)
    return out


# ------------------------------------------------------------------------------------------------ convolution
# taps of a re-parameterised RepSPK 5x5 block with 8 taps that are always zero (17 kept: more than one packing piece)
REPSPK_TAPS = [j for j in range(25) if j not in (0, 4, 20, 24, 2, 10, 14, 22)]


def conv_cases(sms):
    """name -> convolution case.  Shapes that target BLOCK_N 64 / 128 use To = Fo = 16, which choose_conv_tile tiles as
    Fb = 16 x Tb = 8 with no padding: 2 M tiles per utterance, and conv2d_run picks 128 when Cout >= 128 and m_tiles *
    ceil(Cout / 128) >= sms, else 64 when Cout >= 64 and m_tiles * ceil(Cout / 64) >= sms / 2, else 32."""
    h = sms // 2
    D = dict
    cases = {
        "w32_k3s1_cin48_cout16_odd": D(B=2, T=13, F=11, Cin=48, Cout=16, k=3, s=1, scale=True, relu=True, y=True, yf=True,
                                      inst=32),
        "w32_k3s2_cin80_cout48_res_y2": D(B=3, T=15, F=9, Cin=80, Cout=48, k=3, s=2, scale=True, res=True, relu=True,
                                          y=True, y2=True, inst=32),
        "w32_k1s2_cin64_cout80": D(B=2, T=9, F=7, Cin=64, Cout=80, k=1, s=2, scale=True, y=True, yf=True, inst=32),
        "w64_k3s1_cin112_cout80": D(B=_cdiv(_cdiv(h, 2), 2), T=16, F=16, Cin=112, Cout=80, k=3, s=1, scale=True, relu=True,
                                    y=True, y2=True, inst=64),
        "w64_k3s1_cin144_cout144": D(B=_cdiv(_cdiv(h, 3), 2), T=16, F=16, Cin=144, Cout=144, k=3, s=1, scale=True, res=True,
                                     relu=True, y=True, yf=True, inst=64),
        "w128_k3s1_cin16_cout144": D(B=_cdiv(_cdiv(sms, 2), 2), T=16, F=16, Cin=16, Cout=144, k=3, s=1, scale=True,
                                     relu=True, y=True, y2=True, inst=128),
        "w128_k3s2_cin32_cout272": D(B=_cdiv(_cdiv(sms, 3), 2), T=32, F=32, Cin=32, Cout=272, k=3, s=2, scale=True,
                                     res=True, relu=True, y=True, yf=True, inst=128),
        "taps_k5_cin80_cout48": D(B=2, T=9, F=12, Cin=80, Cout=48, k=5, s=1, taps=REPSPK_TAPS, scale=True, relu=True,
                                  y=True, yf=True),
        "taps_k5s2_cin96_cout16": D(B=2, T=11, F=7, Cin=96, Cout=16, k=5, s=2, taps=REPSPK_TAPS, y=True),
        "valid_k3s2_cin96_cout16_odd": D(B=3, T=15, F=13, Cin=96, Cout=16, k=3, s=2, valid=True, scale=True, relu=True,
                                         y=True, yf=True),
        "k1s1_cin128_cout16_odd": D(B=2, T=7, F=5, Cin=128, Cout=16, k=1, s=1, yf=True, y2=True),
        "k3s1_cin32_cout64_res": D(B=2, T=10, F=9, Cin=32, Cout=64, k=3, s=1, scale=True, res=True, relu=True, y=True),
        # CAM++'s FCM front end: feature stride 2, time stride 1 (st), over T > 256 (several time blocks), odd and even F
        "fcm_k3_s2t1_F11_T300": D(B=2, T=300, F=11, Cin=32, Cout=32, k=3, s=2, st=1, scale=True, relu=True, y=True, yf=True),
        "fcm_k3_s2t1_F10_T257": D(B=2, T=257, F=10, Cin=32, Cout=32, k=3, s=2, st=1, scale=True, res=True, relu=True,
                                  y=True),
        "fcm_k1_s2t1_F11_T300": D(B=2, T=300, F=11, Cin=32, Cout=32, k=1, s=2, st=1, scale=True, y=True, yf=True),
        "fcm_k1_s2t1_F10_T270": D(B=3, T=270, F=10, Cin=32, Cout=32, k=1, s=2, st=1, scale=True, y=True),
        # the other mixed stride the API takes: feature stride 1, time stride 2
        "k3_s1t2_F9_T41": D(B=2, T=41, F=9, Cin=32, Cout=48, k=3, s=1, st=2, scale=True, relu=True, y=True, yf=True),
    }
    for c in cases.values():
        c.setdefault("taps", None)
        c.setdefault("st", c["s"])
        pad = 0 if c.get("valid") else c["k"] // 2
        c["To"] = (c["T"] + 2 * pad - c["k"]) // c["st"] + 1
        c["Fo"] = (c["F"] + 2 * pad - c["k"]) // c["s"] + 1
    return cases


def make_conv(case, seed):
    rng = np.random.RandomState(seed)
    B, T, F, Cin, Cout, k = case["B"], case["T"], case["F"], case["Cin"], case["Cout"], case["k"]
    d = {"x": frame_planes(rng, (B, T, F, Cin)), "w_int": int_plane(rng, (Cout, Cin, k, k)),
         "w_frac": grid_plane(rng, (Cout, Cin, k, k))}
    taps = case["taps"]
    if taps is not None:     # the dropped taps of a RepSPK kernel are zero in the stored weight
        keep = np.zeros(k * k, bool)
        keep[taps] = True
        for key in ("w_int", "w_frac"):
            d[key].reshape(Cout, Cin, k * k)[:, :, ~keep] = 0
    if case.get("scale"):
        d["scale"], d["shift"] = pow2_scales(rng, Cout), grid_values(rng, Cout)
    if case.get("res"):
        d["res"] = frame_planes(rng, (B, case["To"], case["Fo"], Cout))
    if case.get("y2"):
        d["scale2"], d["shift2"] = pow2_scales(rng, Cout), grid_values(rng, Cout)
    return d


def conv_reference(case, d):
    """-> (y, y2): float32 outputs of the conv epilogue (BN -> + residual -> ReLU; y2 = relu(y * scale2 + shift2))."""
    k, s, st = case["k"], case["s"], case.get("st", case["s"])      # st: the time stride
    pad = 0 if case.get("valid") else k // 2
    taps = case["taps"] if case["taps"] is not None else list(range(k * k))
    hx, lx = d["x"]
    B, T, F, Cin = hx.shape
    To, Fo = case["To"], case["Fo"]
    wh = d["w_int"].reshape(d["w_int"].shape[0], Cin, k * k)
    wl = d["w_frac"].reshape(d["w_frac"].shape[0], Cin, k * k)
    assert_exact_sum(len(taps) * Cin, [hx], [lx], wh, wl)
    ph = np.pad(hx, ((0, 0), (pad, pad), (pad, pad), (0, 0))).astype(np.float64)
    pl = np.pad(lx, ((0, 0), (pad, pad), (pad, pad), (0, 0))).astype(np.float64)
    acc = np.zeros((B * To * Fo, wh.shape[0]))
    for j in taps:
        kf, kt = divmod(j, k)   # tap = kf * k + kt; "H" is the feature axis, "W" is time
        sh = ph[:, kt:kt + st * (To - 1) + 1:st, kf:kf + s * (Fo - 1) + 1:s].reshape(-1, Cin)
        sl = pl[:, kt:kt + st * (To - 1) + 1:st, kf:kf + s * (Fo - 1) + 1:s].reshape(-1, Cin)
        acc += (sh + sl) @ wh[:, :, j].T.astype(np.float64) + sh @ wl[:, :, j].T.astype(np.float64)
    v = acc.reshape(B, To, Fo, -1)
    if "scale" in d:
        v = v * d["scale"] + d["shift"]
    if "res" in d:
        v = v + d["res"][0] + d["res"][1]
    if case.get("relu"):
        v = np.maximum(v, 0.0)
    y = exact_f32(v)
    y2 = exact_f32(np.maximum(v * d["scale2"] + d["shift2"], 0.0)) if "scale2" in d else None
    return y, y2
