"""Exact-arithmetic operands, case catalogue and references for the Conformer's fp32 CUDA-core kernels (csrc/conformer.cu):
rotary self-attention (xvb_rope_attention), residual + LayerNorm (xvb_layer_norm), the convolution module's middle
(xvb_conv_module) and the subsampling's first conv (xvb_subsample_head[_stride]).

Rotary attention.  The rotary tables hold only quarter turns, (sin, cos) in {(0, 1), (1, 0), (0, -1), (-1, 0)}, varying
with the frame and the pair: each rotated element is one product by +-1 or 0 minus / plus another, so rotation is exact and
`rotate` (float32 numpy, the kernel's operation order) reproduces it bit for bit.  Operands are built in the rotated
domain and rotated back (`unrotate`), so the stored q, k, v differ frame by frame.  Three operand sets:
  * uniform: q = 0, so every score is 0, every p = expf(0) = 1, l = T and o = sum_t v_t over integer v (exact in any
    order).  The output is fl32(o * fl32(1 / T)).  A key dropped or counted twice at a tile edge moves it.
  * k-hot: queries and keys are integers.  Each query is of type X or Y; X queries score 64 * 64 against the keys of group
    X, Y queries against those of group Y, and far less against every other key (integer noise in +-1 on the other
    dimensions, a mid key at 24 * 64): after the division by sqrt(dk) and the multiplier the tied keys of a query's
    group score at least 128 above every other key (asserted for every case by `attention_gaps`), so expf gives exactly 1
    for them and exactly 0 for every other key, and every corr of a tile that brings the group's keys is exactly 0 when
    an earlier tile held a lower maximum.  The output is fl32(sum of the group's v * fl32(1 / k)).  Placements put the
    groups in the first tile, only in the tail tile, in a later tile than a lower earlier maximum (a "mid" key in tile
    0 that the corr = 0 rescale has to wipe out), or spread over the tiles.
  * random: normal q, k, v and a multiplier != 1, checked within the bound derived in `attention_random_bound`.
v is nonzero with a fixed sign per dimension, so no exact output is zero and the bits include the sign.

LayerNorm.  With eps = 0, a row m + d_c whose integer deviations have sum d = 0 and sum d^2 = C 4^k normalises exactly:
the mean is m, the variance 4^k, sqrtf 2^k and its reciprocal 2^-k.  Deviations are built from pairs (2, -2) and
blocks (3, -3, 1, -1, 0) (which makes odd C possible: C = 5 + 2n), scaled by 2^j and permuted over the channels.  Each
block carries a sign s_c, and gamma = s_c 2^p with a constant beta makes the first norm's output an exact row again (the
deviations s_c 2^(p-k) d_c still sum to 0 within each block), which the second norm of `second` normalises exactly.  x is
built so that x + table + delta_scale * delta is the row exactly.  Rows with eps = 1e-5 and random data are checked
within the bound of `ln_random_bound`.

Convolution module.  GLU gates are >= 20 or <= -100: 1 / (1 + expf(-b)) is then exactly 1 or exactly 0 in fp32
(`glu_gate_is_exact`), so the GLU is a or +-0.  The depthwise conv on grid weights and biases is exact.  The scale / shift
norm uses power-of-two scales.  The LayerNorm path (eps = 0) has a[t, c] = alpha_t u_c with u an exact-row deviation,
weights w[c, k] = s_c omega_k with s_c the block signs of u and a constant bias beta: each output row is beta +
A_t s_c u_c with A_t = sum_k omega_k alpha_(t+k-pad) > 0, whose variance A_t^2 C 4^k has an exact sqrt; the reciprocal,
the normalised value and the affine fmaf each round once, which `ln_emulate` reproduces in float32.

Subsampling head.  Grid x, w and bias: exact.

Plain numpy (no torch, no GPU): test_gpu_conformer_edges.py moves these operands to the device, and
test_conformer_exact_host.py checks the helpers, the catalogue and every case's precondition on the CPU."""
import math

import numpy as np

import gemm_exact as gx

U = gx.U32
QUARTER = np.array([(0.0, 1.0), (1.0, 0.0), (0.0, -1.0), (-1.0, 0.0)], np.float32)   # (sin, cos)
ATTN_TILE = 32           # keys staged per tile (kAttnK)
ATTN_Q = 8               # queries per CTA (kAttnQ)
CONV_ROWS = 16           # frames per conv-module CTA (kConvRows)
CONV_MAX_SMEM = 200 * 1024


def _ru(x, m):
    return (x + m - 1) // m * m


# ------------------------------------------------------------------------------------------------ rotary attention
def quarter_rope(rng, T, dk):
    """(T, dk) float32 [sin | cos] table of quarter turns, varying with the frame and the pair"""
    q = QUARTER[rng.randint(0, 4, (T, dk // 2))]
    return np.concatenate([q[..., 0], q[..., 1]], axis=1)


def rotate(x, rope):
    """The kernel's rotate_pair over x (..., T, dk): pairs (2j, 2j+1), x1 * cos - x2 * sin and x2 * cos + x1 * sin, each
    product and the sum rounded in float32 (exact for quarter turns)."""
    dk = x.shape[-1]
    s, c = rope[:, :dk // 2], rope[:, dk // 2:]
    a, b = x[..., 0::2], x[..., 1::2]
    out = np.empty_like(x)
    out[..., 0::2] = a * c - b * s
    out[..., 1::2] = b * c + a * s
    return out


def unrotate(y, rope):
    """The inverse quarter turn: rotate(unrotate(y)) == y for quarter-turn tables."""
    dk = y.shape[-1]
    s, c = rope[:, :dk // 2], rope[:, dk // 2:]
    a, b = y[..., 0::2], y[..., 1::2]
    out = np.empty_like(y)
    out[..., 0::2] = a * c + b * s
    out[..., 1::2] = b * c - a * s
    return out


ATTN_T = (1, 7, 8, 9, 31, 32, 33, 63, 64, 65, 257, 1500)
ATTN_PLACES = ("first", "tail", "later", "spread")


def attention_cases():
    """name -> rope_attention case.  Every T runs every dk at least once across the catalogue, and each (dk, rotary
    mode) pair appears; H in {1, 3, 8}.  q / k / v are the channel slice at 8 of a NaN buffer of a wider pitch (a NaN
    gap between the slice and the next row), y a fenced slice at 8 of a pitch > H dk."""
    D = dict
    cases = {}
    rots = ("none", "rope", "rope_v")
    i = 0
    for T in ATTN_T:
        for dk in (32, 64, 128):
            if T == 1500 and dk != 64:
                continue
            H = (1, 3, 8)[i % 3] if T < 1500 else 2
            place = ATTN_PLACES[i % 4]
            if T <= ATTN_TILE and place in ("later", "spread"):
                place = ("first", "tail")[i % 2]
            rot = rots[(i + T) % 3]
            cases["T{}_dk{}_H{}_{}_{}".format(T, dk, H, rot, place)] = D(
                B=2, T=T, dk=dk, H=H, rot=rot, place=place, mult=(1.0, 1.375)[(i // 3) % 2])
            i += 1
    # every placement at a tile edge on each head size, with every rotary mode
    for T, dk, rot in ((64, 32, "rope_v"), (65, 128, "rope"), (96, 64, "none"), (33, 128, "rope_v")):
        for place in ATTN_PLACES:
            cases["edge_T{}_dk{}_{}_{}".format(T, dk, rot, place)] = D(B=3, T=T, dk=dk, H=3, rot=rot, place=place, mult=1.0)
    for c in cases.values():
        D_ = c["H"] * c["dk"]
        c["q_c0"], c["ldq"] = 8, 8 + 3 * D_ + 12
        c["y_c0"], c["ldy"] = 8, _ru(8 + D_ + 8, 8)
    return cases


def _groups(rng, T, place):
    """Positions of the two tied groups (X, Y) and of the mid key (or None) for a placement."""
    nt = -(-T // ATTN_TILE)
    last = (nt - 1) * ATTN_TILE

    def pick(lo, hi, k):
        return list(rng.choice(np.arange(lo, hi), size=min(k, hi - lo), replace=False))

    mid = None
    if place == "first":
        pos = pick(0, min(T, ATTN_TILE), 4)
    elif place == "tail":
        pos = pick(last, T, 4)
    elif place == "later":
        mid = int(rng.randint(0, ATTN_TILE))
        pos = pick(ATTN_TILE, T, 4)
    else:                          # one key per tile, the last tile included
        pos = [int(rng.randint(t * ATTN_TILE, min(T, (t + 1) * ATTN_TILE))) for t in range(nt)]
        pos = list(dict.fromkeys(pos + pick(0, T, 2)))
    rng.shuffle(pos)
    if len(pos) == 1:
        return pos, pos, mid       # one key: both groups share it
    k = max(1, min(3, len(pos) // 2))
    return pos[:k], pos[k:2 * k] if len(pos) >= 2 * k else pos[:k], mid


def make_attention(case, seed, mode):
    """-> dict(q, k, v (B, T, H, dk) stored float32, rope or None, and for k-hot: groups, qtype (B, T) 0 / 1)."""
    rng = np.random.RandomState(seed)
    B, T, H, dk = case["B"], case["T"], case["H"], case["dk"]
    rope = quarter_rope(rng, T, dk) if case["rot"] != "none" else None
    sign = rng.choice([-1.0, 1.0], (B, H, dk)).astype(np.float32)
    v = (rng.randint(1, 9, (B, T, H, dk)) * sign[:, None]).astype(np.float32)
    d = {"rope": rope}
    if mode == "uniform":
        qr, kr = np.zeros((B, T, H, dk), np.float32), gx.int_plane(rng, (B, T, H, dk), 3)
    elif mode == "khot":
        qtype = rng.randint(0, 2, (B, T))
        qr = rng.randint(-1, 2, (B, T, H, dk)).astype(np.float32)
        qr[..., 0:2] = 0
        qr[..., 0] = np.where(qtype == 0, 64, 0)[..., None]
        qr[..., 1] = np.where(qtype == 1, 64, 0)[..., None]
        kr = rng.randint(-1, 2, (B, T, H, dk)).astype(np.float32)
        kr[..., 0:2] = rng.randint(-2, 3, (B, T, H, 2))
        groups = []
        for b in range(B):
            gX, gY, mid = _groups(rng, T, case["place"])
            for g in (gX, gY):
                kr[b, g, :, :] = kr[b, g[0], :, :]          # the group's keys are one rotated vector
                kr[b, g, :, 0:2] = 0
            kr[b, gX, :, 0] = 64                            # a lone key shared by both groups scores 64 * 64 for both
            kr[b, gY, :, 1] = 64
            if mid is not None and mid not in gX and mid not in gY:
                kr[b, mid, :, 0:2] = 24
            groups.append((gX, gY))
        d["groups"], d["qtype"] = groups, qtype
    else:
        qr = rng.standard_normal((B, T, H, dk)).astype(np.float32)
        kr = rng.standard_normal((B, T, H, dk)).astype(np.float32)
        v = rng.standard_normal((B, T, H, dk)).astype(np.float32)
    if rope is not None:
        # stored values are the rotated-domain operands turned back; the kernel turns them forward again
        qs = unrotate(qr.transpose(0, 2, 1, 3), rope).transpose(0, 2, 1, 3)
        ks = unrotate(kr.transpose(0, 2, 1, 3), rope).transpose(0, 2, 1, 3)
        vs = unrotate(v.transpose(0, 2, 1, 3), rope).transpose(0, 2, 1, 3) if case["rot"] == "rope_v" else v
    else:
        qs, ks, vs = qr, kr, v
    d.update(q=np.ascontiguousarray(qs), k=np.ascontiguousarray(ks), v=np.ascontiguousarray(vs))
    return d


def _rotated(case, d):
    """(q, k, v) as the kernel sees them after rotation, (B, H, T, dk) float32"""
    q, k, v = (a.transpose(0, 2, 1, 3) for a in (d["q"], d["k"], d["v"]))
    if d["rope"] is not None:
        q, k = rotate(q, d["rope"]), rotate(k, d["rope"])
        if case["rot"] == "rope_v":
            v = rotate(v, d["rope"])
    return q, k, v


def attention_scores(case, d):
    """(B, H, T, T) float32 scores as the kernel forms them: an exact integer dot (asserted below 2^24), then
    fl32(fl32(d / sqrtf(dk)) * mult)."""
    q, k, _ = _rotated(case, d)
    dot = np.einsum("bhqd,bhkd->bhqk", q.astype(np.float64), k.astype(np.float64))
    mag = np.einsum("bhqd,bhkd->bhqk", np.abs(q).astype(np.float64), np.abs(k).astype(np.float64))
    assert mag.max() < 2.0 ** 24 and np.array_equal(dot, np.round(dot)), "score dots are not exact"
    return (dot.astype(np.float32) / np.sqrt(np.float32(case["dk"]))) * np.float32(case["mult"])


def attention_gaps(case, d):
    """k-hot precondition: for every query, the smallest score of its group's keys minus the largest of the other keys
    (inf when there are none), and whether the group's scores are all equal.  -> (min gap, all tied)"""
    s = attention_scores(case, d)
    gap, tied = np.inf, True
    for b, (gX, gY) in enumerate(d["groups"]):
        for t in range(case["T"]):
            g = (gX, gY)[d["qtype"][b, t]]
            mask = np.zeros(case["T"], bool)
            mask[g] = True
            for h in range(case["H"]):
                row = s[b, h, t]
                tied &= bool(np.all(row[mask] == row[mask][0]))
                if (~mask).any():
                    gap = min(gap, float(row[mask].min() - row[~mask].max()))
    return gap, tied


def attention_exact_reference(case, d, mode):
    """uniform / k-hot: (B, T, H * dk) float32 output, fl32(exact sum of v over the attended keys * fl32(1 / count))."""
    B, T, H, dk = case["B"], case["T"], case["H"], case["dk"]
    _, _, v = _rotated(case, d)                          # (B, H, T, dk)
    v = v.astype(np.float64)
    out = np.empty((B, H, T, dk), np.float32)
    for b in range(B):
        if mode == "uniform":
            sums, counts = np.broadcast_to(v[b].sum(axis=1)[:, None], (H, T, dk)), np.full(T, T)
        else:
            gX, gY = d["groups"][b]
            sx, sy = v[b][:, gX].sum(axis=1), v[b][:, gY].sum(axis=1)
            typ = d["qtype"][b]
            sums = np.where((typ == 0)[None, :, None], sx[:, None], sy[:, None])
            counts = np.where(typ == 0, len(gX), len(gY))
        inv = np.float32(1.0) / counts.astype(np.float32)
        out[b] = gx.exact_f32(sums) * inv[None, :, None]
    return np.ascontiguousarray(out.transpose(0, 2, 1, 3).reshape(B, T, H * dk))


def attention_random_bound(case, d):
    """(want float64 (B, T, H dk), bound).  Scores: the fp32 dot over dk terms errs by <= dk u sum|q k|, the division and
    the multiplier by 2u |s| more, and s - m by u |s - m|: delta = max over keys.  The softmax weights then err by
    <= exp(2 delta) - 1 relative (a common shift cancels), expf by 2^-22, and each of the ceil(T / 32) rescales multiplies
    the earlier weights by corr (within 2^-22 + u) for o and l alike.  o and l accumulate T terms (<= T u relative each)
    and 1 / l and o * inv round once each.  The stored planes keep 16 of the 24 bits: + 2^-16 |y|.  Everything is taken
    twice for margin."""
    B, T, H, dk = case["B"], case["T"], case["H"], case["dk"]
    q, k, v = (a.astype(np.float64) for a in _rotated(case, d))
    s64 = np.einsum("bhqd,bhkd->bhqk", q, k) / math.sqrt(dk) * case["mult"]
    mag = np.einsum("bhqd,bhkd->bhqk", np.abs(q), np.abs(k)) / math.sqrt(dk) * case["mult"]
    m = s64.max(axis=-1, keepdims=True)
    delta = (dk * U * mag + 2 * U * np.abs(s64) + U * np.abs(s64 - m) * 2).max(axis=-1)
    w = np.exp(s64 - m)
    w /= w.sum(axis=-1, keepdims=True)
    want = np.einsum("bhqk,bhkd->bhqd", w, v)
    wabs = np.einsum("bhqk,bhkd->bhqd", w, np.abs(v))
    nt = -(-T // ATTN_TILE)
    eta = np.expm1(2 * delta) + 2.0 ** -22 * (1 + nt) + 2 * U * nt
    bound = 2 * ((2 * eta[..., None] + 2 * T * U) * wabs + 3 * U * np.abs(want)) + 2.0 ** -16 * np.abs(want) + 2.0 ** -120
    tr = lambda a: np.ascontiguousarray(a.transpose(0, 2, 1, 3).reshape(B, T, H * dk))   # noqa: E731
    return tr(want), tr(bound)


def qkv_rows(d):
    """(B, T, 3 H dk) float32 [q | k | v] rows, heads contiguous within each third (the fused projection's layout)"""
    B, T, H, dk = d["q"].shape
    return np.concatenate([a.reshape(B, T, H * dk) for a in (d["q"], d["k"], d["v"])], axis=2)


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_warps(C):
    """Rows per CTA of xvb_layer_norm: clamp(8192 / C, 1, 8) warps, one row each (the staged rows fit 32 KB)."""
    return max(1, min(8, 8192 // C))


def deviation_blocks(rng, C, max_j=2):
    """A random exact-row pattern for C channels: -> (d (C,) float64 integers, block sign s (C,) +-1, k, block id (C,))
    with sum d = 0 within every block, sum d^2 = C 4^k.  Blocks: (2, -2) pairs and (3, -3, 1, -1, 0) fives (one for odd C, two for even
    C >= 10), all scaled by 2^j and permuted over the channels."""
    assert C >= 2 and C != 3
    blocks = []
    fives = 1 if C % 2 else (2 if C >= 10 else 0)
    blocks += [[3, -3, 1, -1, 0]] * fives
    blocks += [[2, -2]] * ((C - 5 * fives) // 2)
    j = int(rng.randint(0, max_j + 1))
    d, s, ids = np.zeros(C), np.zeros(C), np.zeros(C, int)
    perm = rng.permutation(C)
    i = 0
    for n, blk in enumerate(blocks):
        idx = perm[i:i + len(blk)]
        d[idx] = np.array(blk, float) * rng.choice([-1.0, 1.0]) * 2.0 ** j
        s[idx] = rng.choice([-1.0, 1.0])
        ids[idx] = n
        i += len(blk)
    assert i == C
    return d, s, 1 + j, ids


def ln_emulate(v, g, b, eps, what="row"):
    """The kernel's warp_layer_norm over float32 rows v (..., C) whose sums are exact in any order (asserted: every
    element on a grid of 2^-e and the largest sum of |terms| below 2^(24 - e)): the mean fl32(sum / C), d = v - mean
    (asserted exact), the variance fl32(sum d^2 / C) + eps, fl32(sqrt), fl32(1 / .), fl32(d * rstd), then fmaf(y, g, b)
    rounded once.  -> float32."""
    v = np.asarray(v, np.float32)
    C = v.shape[-1]
    e = 0
    while not np.array_equal(v * 2.0 ** e, np.round(v * 2.0 ** e)):
        e += 1
        assert e <= 12, what + ": values off the grid"
    assert float(np.abs(v.astype(np.float64)).sum(axis=-1).max()) * 2.0 ** e < 2.0 ** 24, what + ": sum not exact"
    mean = (v.astype(np.float64).sum(axis=-1, keepdims=True).astype(np.float32) / np.float32(C)).astype(np.float32)
    dd = v - mean
    assert np.array_equal(dd.astype(np.float64), v.astype(np.float64) - mean), what + ": v - mean rounds"
    sq = (dd.astype(np.float64) ** 2)
    e2 = 0
    while not np.array_equal(sq * 2.0 ** e2, np.round(sq * 2.0 ** e2)):
        e2 += 1
        assert e2 <= 24, what + ": squares off the grid"
    q = sq.sum(axis=-1, keepdims=True)
    assert float(q.max()) * 2.0 ** e2 < 2.0 ** 24, what + ": sum of squares not exact"
    var = q.astype(np.float32) / np.float32(C) + np.float32(eps)
    rstd = np.float32(1.0) / np.sqrt(var)
    y = dd * rstd
    if g is not None:
        y = (y.astype(np.float64) * g.astype(np.float64) + b.astype(np.float64)).astype(np.float32)
    return y


def ln_random_bound(v, g, b, eps):
    """(want float64, bound) of a LayerNorm of arbitrary float32 rows.  The mean errs by <= C u mean|v| + u |mean|
    (sum, division), d by that plus u |d|; the variance by 2 |dmean| mean|d| + (C + 2) u var; rstd by half the relative
    variance error plus 3 u (sqrt, reciprocal); y = d rstd by |dd| rstd + |d| drstd + u |y|; the affine multiplies by |g|
    and rounds once more.  Twice that."""
    v = np.asarray(v, np.float64)
    C = v.shape[-1]
    mean = v.mean(axis=-1, keepdims=True)
    d = v - mean
    var = (d * d).mean(axis=-1, keepdims=True)
    r = 1.0 / np.sqrt(var + eps)
    y = d * r
    dmean = C * U * np.abs(v).mean(axis=-1, keepdims=True) + U * np.abs(mean)
    dd = dmean + U * np.abs(d)
    dvar = 2 * dmean * np.abs(d).mean(axis=-1, keepdims=True) + (C + 2) * U * var
    dr = r * (0.5 * dvar / (var + eps) + 3 * U)
    dy = dd * r + np.abs(d) * dr + U * np.abs(y)
    if g is not None:
        out = y * g + b
        return out, 2 * (dy * np.abs(g) + U * np.abs(out))
    return y, 2 * dy


LN_C = (2, 8, 31, 32, 33, 100, 1023, 1024, 1025, 1200, 1500, 2000, 2730, 4096, 4097, 8192)
LN_ACTS = ("none", "relu", "swish", "tanh")


def ln_cases(sms):
    """name -> layer_norm case for a GPU with `sms` SMs (the grid is min(ceil(rows / warps), 16 sms) CTAs, so rows >
    16 sms warps make the grid-stride loop go round again)."""
    D = dict
    cases = {}
    for i, C in enumerate(LN_C):
        B, T = 2, (5, 3, 7)[i % 3]
        rows = B * T
        c = D(B=B, T=T, C=C, act=LN_ACTS[i % 4], gamma=i % 5 != 1)
        if i % 2 == 0:
            c["table_rows"] = 1 if i % 4 == 0 else T + 1       # 1, or a count that does not divide the rows
        if i % 3 != 1:
            c["delta_scale"] = (0.5, 1.0)[i % 2]
        c["x_out"] = ("inplace", "other", None)[i % 3]
        if i % 4 == 3:
            c["second"] = "gamma2" if i % 8 == 3 else "plain"
        c["y"] = i % 5 != 4
        c["y_f32"] = i % 5 != 2 or not c["y"]
        assert rows > 0
        cases["C{}_{}".format(C, c["act"])] = c
    cases["second_gamma2_C33_swish"] = D(B=3, T=4, C=33, act="swish", gamma=True, second="gamma2", table_rows=5,
                                         delta_scale=0.5, x_out="other", y=True, y_f32=True)
    cases["second_plain_C1024_relu"] = D(B=2, T=9, C=1024, act="relu", gamma=False, second="plain", delta_scale=1.0,
                                         x_out="inplace", y=True, y_f32=True)
    cases["grid_stride_C100"] = D(B=1, T=sms * 16 * 8 + 37, C=100, act="relu", gamma=True, table_rows=7, delta_scale=1.0,
                                  x_out="inplace", y=True, y_f32=True)
    cases["grid_stride_C4097"] = D(B=1, T=sms * 16 + 5, C=4097, act="none", gamma=True, second="gamma2", delta_scale=0.5,
                                   x_out="other", y=True, y_f32=False)
    for c in cases.values():
        C = c["C"]
        c["warps"] = ln_warps(C)
        c["x_c0"], c["ldx"] = 3, C + 5
        c["d_c0"], c["ldd"] = 1, C + 9
        c["xo_c0"], c["ldxo"] = 2, C + 7
        c["y_c0"], c["ldy"] = 8, _ru(8 + C + 8, 8)
        c["yf_c0"], c["ldyf"] = 4, C + 6
    return cases


def make_ln(case, seed):
    """Exact operands: rows (B, T, C) = m + d (per row, m on the 2^-4 grid in [-4, 4]), table and delta on the 2^-4 grid,
    x = row - table - delta_scale * delta; gamma / beta on the 2^-8 grid, or for `second` gamma = s_c 2^p (the block
    signs) and a constant beta.  One deviation pattern (blocks and signs) per case, each row negating blocks at random."""
    rng = np.random.RandomState(seed)
    B, T, C = case["B"], case["T"], case["C"]
    rows = B * T
    dev, s, k, blk = deviation_blocks(rng, C)
    flip = rng.choice([-1.0, 1.0], (rows, blk.max() + 1))[:, blk]      # each row negates whole blocks
    m = (rng.randint(-64, 65, (rows, 1)) / 16.0)
    v = (m + flip * dev[None]).astype(np.float32)
    d = {"row": v.reshape(B, T, C), "k": k, "s": s.astype(np.float32)}
    x = v.astype(np.float64)
    if case.get("table_rows"):
        d["table"] = (rng.randint(-32, 33, (case["table_rows"], C)) / 16.0).astype(np.float32)
        x = x - d["table"][np.arange(rows) % case["table_rows"]]
    if "delta_scale" in case:
        d["delta"] = (rng.randint(-32, 33, (rows, C)) / 16.0).astype(np.float32)
        x = x - case["delta_scale"] * d["delta"].astype(np.float64)
        d["delta"] = d["delta"].reshape(B, T, C)
    d["x"] = gx.exact_f32(x).reshape(B, T, C)
    if case.get("second"):
        if case["gamma"]:
            d["gamma"] = (s * 2.0 ** rng.randint(-1, 2)).astype(np.float32)
            d["beta"] = np.full(C, rng.randint(-16, 17) / 8.0, np.float32)
        if case["second"] == "gamma2":
            d["gamma2"], d["beta2"] = gx.grid_values(rng, C), gx.grid_values(rng, C)
    elif case["gamma"]:
        d["gamma"], d["beta"] = gx.grid_values(rng, C), gx.grid_values(rng, C)
    return d


def ln_reference(case, d):
    """-> dict(x_out float32 or None, y float32 or float64, y_bound or None).  Everything before the activation is exact
    (ln_emulate asserts it); swish and tanh carry the bounds of gemm_exact.layer_reference."""
    B, T, C = case["B"], case["T"], case["C"]
    v = d["row"].reshape(-1, C)
    n1 = ln_emulate(v, d.get("gamma"), d.get("beta"), 0.0, "first norm")
    if case.get("second"):
        xo, n = n1, ln_emulate(n1, d.get("gamma2"), d.get("beta2"), 0.0, "second norm")
    else:
        xo, n = v, n1
    assert np.array_equal(gx.exact_f32(n.astype(np.float64)), n)
    y, bound = act_reference(n.astype(np.float64), case["act"])
    sh = (B, T, C)
    return {"x_out": xo.reshape(sh), "y": y.reshape(sh), "bound": None if bound is None else bound.reshape(sh)}


def act_reference(pre, act):
    """activate() over exact float64 inputs -> (float32 exact, None) or (float64, bound) (bounds of
    gemm_exact.layer_reference: expf / tanhf within 2 ulp, each further operation one rounding)."""
    if act == "none":
        return pre.astype(np.float32), None
    if act == "relu":
        return np.maximum(pre, 0.0).astype(np.float32), None
    if act == "swish":
        with np.errstate(over="ignore"):
            sw = pre / (1.0 + np.exp(-pre))
        return sw, 2.0 ** -21 * np.abs(sw) + 2.0 ** -120
    if act == "tanh":
        out = np.tanh(pre)
        return out, 2.0 * 2.0 ** -23 * np.abs(out) + 2.0 ** -126
    raise ValueError(act)


def make_ln_random(case, seed):
    rng = np.random.RandomState(seed)
    B, T, C = case["B"], case["T"], case["C"]
    x = (rng.standard_normal((B, T, C)) * 3 + 0.5).astype(np.float32)
    g = (1 + 0.1 * rng.standard_normal(C)).astype(np.float32)
    b = (0.1 * rng.standard_normal(C)).astype(np.float32)
    return x, g, b


# ------------------------------------------------------------------------------------------------ convolution module
def glu_gate_is_exact(b):
    """fp32 1 / (1 + expf(-b)) is exactly 1 (b >= 20) or exactly 0 (b <= -100) -> the float32 gate values."""
    b = np.asarray(b, np.float32)
    with np.errstate(over="ignore"):
        g = np.float32(1.0) / (np.float32(1.0) + np.exp(-b))
    assert np.all((g == 1.0) | (g == 0.0))
    return g


def conv_smem(C, K):
    """Dynamic shared memory of xvb_conv_module: (16 + K - 1) GLU rows and 16 output rows of C floats."""
    return (2 * CONV_ROWS + K - 1) * C * 4


def conv_max_channels(K):
    return CONV_MAX_SMEM // ((2 * CONV_ROWS + K - 1) * 4)


CONV_T = (1, 15, 16, 17, 31, 32, 33, 100)
CONV_K = (1, 3, 15, 31)
CONV_ACTS = ("relu", "swish")


def conv_cases():
    """name -> conv_module case: every T with every K and C in turn and both norms, K / 2 > T, and the largest C whose
    staging fits 200 KB at K = 31.  x is the slice at 4 of a NaN buffer of pitch > 2C (NaN gap, NaN spare utterance); y
    is a fenced slice at 8 of a pitch > C."""
    D = dict
    cases = {}
    Cs = (8, 33, 256)
    for i, T in enumerate(CONV_T):
        for j, norm in enumerate(("bn", "ln")):
            K = CONV_K[(i + j) % 4]
            C = Cs[(i + 2 * j) % 3]
            cases["T{}_K{}_C{}_{}".format(T, K, C, norm)] = D(B=3, T=T, K=K, C=C, norm=norm, act=CONV_ACTS[(i + j) % 2])
    cmax = conv_max_channels(31)
    for norm in ("bn", "ln"):
        cases["Cmax{}_K31_T40_{}".format(cmax, norm)] = D(B=2, T=40, K=31, C=cmax, norm=norm, act="swish")
        cases["K31_T5_{}".format(norm)] = D(B=2, T=5, K=31, C=33, norm=norm, act="relu")
        cases["K15_T3_{}".format(norm)] = D(B=2, T=3, K=15, C=8, norm=norm, act="swish")
    for c in cases.values():
        c["x_c0"], c["ldx"] = 4, 4 + 2 * c["C"] + 6
        c["y_c0"], c["ldy"] = 8, _ru(8 + c["C"] + 8, 8)
    return cases


def make_conv_module(case, seed):
    """Operands of a conv-module case: x (B, T, 2C) [a | gate input], dw_w (C, K), dw_b (C,), norm_a / norm_b (C,)."""
    rng = np.random.RandomState(seed)
    B, T, C, K = case["B"], case["T"], case["C"], case["K"]
    gate_in = rng.uniform(20, 40, (B, T, C)).astype(np.float32)
    if case["norm"] == "bn":
        a = (rng.randint(-48, 49, (B, T, C)) / 16.0).astype(np.float32)
        closed = rng.rand(B, T, C) < 0.25
        gate_in[closed] = -rng.uniform(100, 140, int(closed.sum())).astype(np.float32)
        w = (rng.randint(-32, 33, (C, K)) / 16.0).astype(np.float32)
        bias = gx.grid_values(rng, C)
        na = (gx.pow2_scales(rng, C) * rng.choice([-1.0, 1.0], C)).astype(np.float32)
        nb = gx.grid_values(rng, C)
    else:
        dev, s, _, blk = deviation_blocks(rng, C, max_j=0)     # sum d^2 = A_t^2 C 4 <= 62^2 * 825 * 4 < 2^24
        flips = rng.choice([-1.0, 1.0], (B, blk.max() + 1))[:, blk]                # per utterance, whole blocks
        alpha = rng.randint(1, 3, (B, T, 1)).astype(np.float64)
        a = (alpha * (flips * dev)[:, None, :]).astype(np.float32)
        omega = rng.randint(1, 3, K) if K <= 15 else np.ones(K)
        w = (s[:, None] * omega[None, :]).astype(np.float32)
        bias = np.full(C, rng.randint(-16, 17) / 4.0, np.float32)
        na, nb = gx.grid_values(rng, C), gx.grid_values(rng, C)
    x = np.concatenate([a, gate_in], axis=2)
    return {"x": x, "w": w, "b": bias, "na": na, "nb": nb}


def conv_module_pre(case, d):
    """The depthwise conv of the GLU, float64 in the kernel's tap order from 0 (fmaf(w, g, s), exact), + bias:
    (B, T, C), asserted exact in fp32 (multiples of 2^-8 below 2^15)."""
    B, T, C, K = case["B"], case["T"], case["C"], case["K"]
    x = d["x"]
    g = glu_gate_is_exact(x[..., C:])
    with np.errstate(invalid="ignore"):
        glu = (x[..., :C] * g).astype(np.float64)             # a * 1 or a * 0 (+-0)
    pad = K // 2
    s = np.zeros((B, T, C))
    mag = np.zeros((B, T, C))
    for k in range(K):
        sh = gx.shift_time(glu, k - pad)
        s = s + d["w"][:, k].astype(np.float64) * sh
        mag = mag + np.abs(d["w"][:, k]) * np.abs(sh)
    assert float(mag.max()) < gx.EXACT_SUM_LIMIT
    return gx.exact_f32(s + d["b"])


def conv_module_reference(case, d, act):
    """-> (want, bound): float32 and None when exact (act none / relu), else float64 and the bound of act_reference."""
    C = case["C"]
    y = conv_module_pre(case, d)
    if case["norm"] == "bn":
        n = gx.exact_f32(y.astype(np.float64) * d["na"] + d["nb"])
    else:
        n = ln_emulate(y.reshape(-1, C), d["na"], d["nb"], 0.0, "conv LayerNorm").reshape(y.shape)
    return act_reference(n.astype(np.float64), act)


# ------------------------------------------------------------------------------------------------ subsampling head
def subsample_cases(sms):
    """name -> subsample_head case: both feature strides over T in {3, 4, 5, 200}, F in {3, 4, 80}, C in {8, 24, 256},
    and one shape with more than 16 sms * 256 (position, 8-channel) items, so the grid-stride loop runs again."""
    D = dict
    cases = {}
    i = 0
    for sf in (1, 2):
        for T in (3, 4, 5, 200):
            for F in (3, 4, 80):
                if (T == 200) and F == 80 and sf == 2:
                    continue
                C = (8, 24, 256)[i % 3]
                cases["sf{}_T{}_F{}_C{}".format(sf, T, F, C)] = D(B=2, T=T, F=F, C=C, sf=sf)
                i += 1
    cases["grid_stride_sf1"] = D(B=4, T=200, F=80, C=256, sf=1)
    cases["grid_stride_sf2"] = D(B=9, T=200, F=80, C=256, sf=2)
    for c in cases.values():
        c["T1"] = (c["T"] - 3) // 2 + 1
        c["F1"] = (c["F"] - 3) // c["sf"] + 1
        c["items"] = c["B"] * c["T1"] * c["F1"] * c["C"] // 8
    assert cases["grid_stride_sf1"]["items"] > sms * 16 * 256 and cases["grid_stride_sf2"]["items"] > sms * 16 * 256
    return cases


def make_subsample(case, seed):
    rng = np.random.RandomState(seed)
    return {"x": (rng.randint(-64, 65, (case["B"], case["T"], case["F"])) / 16.0).astype(np.float32),
            "w": (rng.randint(-32, 33, (case["C"], 1, 3, 3)) / 16.0).astype(np.float32),
            "b": gx.grid_values(rng, case["C"])}


def subsample_reference(case, d):
    """relu(conv2d(x, w, stride (2, sf)) + b) -> (B, T1, F1, C) float32, exact (grid operands, 9 terms)."""
    x, w = d["x"].astype(np.float64), d["w"][:, 0].astype(np.float64)
    T1, F1, sf = case["T1"], case["F1"], case["sf"]
    acc = np.zeros((case["B"], T1, F1, case["C"]))
    for kt in range(3):
        for kf in range(3):
            win = x[:, kt:kt + 2 * (T1 - 1) + 1:2, kf:kf + sf * (F1 - 1) + 1:sf]
            acc += win[..., None] * w[:, kt, kf]
    return gx.exact_f32(np.maximum(acc + d["b"], 0.0))
