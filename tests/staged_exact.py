"""Case catalogue and float64 references for the staged epilogue of the TDNN layer kernel (csrc/tdnn_gemm.cu): the
plane-only layers whose outputs leave through shared memory and TMA stores, the ping-pong 128-wide instance, split-K on
it, and the fused pooling epilogue's partials.

Operands, the bf16 split and the layer reference are gemm_exact's, so every layer output is exact in fp32.  What this
module adds:
  * host mirrors of choose_m_tile, of the BLOCK_N dispatch of gemm_plan_build and of the condition under which a launch
    takes the staged epilogue (prepare_gemm: p.tma_store), so that each case states which instance, Tb and path it is
    meant for; the GPU file confirms the instance from the kernel names and test_staged_exact_host.py the Tb through the
    library's own xvb_pool_partial_blocks;
  * a shape search that gives a case its Tb, BLOCK_N, ragged T and B and tile count on a GPU with `sms` SMs (the case
    names do not depend on it);
  * masked batches (lengths), grouped 1x1 layers, the im2col view of a first layer and a signed-zero case;
  * integer-valued pooling data, on which the fused pooling epilogue's Chan merges are exact wherever the merged counts
    are powers of two, and an fp32 emulation of the epilogue's merge order that says where that is the case.

Plain numpy (no torch, no GPU)."""
import numpy as np

import gemm_exact as gx

TBS = (1, 2, 4, 8, 16, 32, 64, 128)


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------------ host mirrors
def choose_m_tile(B, T):
    """choose_m_tile of tdnn_gemm.cu: Tb frames x 128 / Tb utterances per M tile, the fewest padded rows, larger Tb on
    ties; T == 1 is always Tb = 1."""
    if T == 1:
        return 1
    best, bt = -1, 128
    for tb in (128, 64, 32, 16, 8, 4, 2, 1):
        rows = _cdiv(T, tb) * tb * _cdiv(B, 128 // tb) * (128 // tb)
        if best < 0 or rows < best:
            best, bt = rows, tb
    return bt


def m_tiles(B, T):
    tb = choose_m_tile(B, T)
    return _cdiv(T, tb) * _cdiv(B, 128 // tb)


def block_n(case, sms):
    """The BLOCK_N gemm_plan_build's dispatch picks for a (non-split-K) layer case."""
    cout, g = case["Cout"], case.get("groups", 1)
    if g > 1:
        ng = cout // g
        return 128 if ng % 128 == 0 else 64 if ng % 64 == 0 else 32
    m = m_tiles(case["B"], case["T"])
    if cout >= 128 and m * _cdiv(cout, 128) >= sms:
        return 128
    if cout >= 64 and m * _cdiv(cout, 64) >= sms // 2:
        return 64
    return 32


def num_tiles(case, sms):
    return m_tiles(case["B"], case["T"]) * _cdiv(case["Cout"], block_n(case, sms))


def cta_tile_counts(tiles, sms):
    """Tiles per CTA of a persistent launch (grid = min(tiles, sms), CTA i takes tiles i, i + grid, ...)."""
    grid = min(tiles, sms)
    return {_cdiv(tiles - i, grid) for i in range(grid)}


def staged_taken(case, bn, splitk=False):
    """Mirrors the condition of p.tma_store in prepare_gemm (tdnn_gemm.cu): the staged epilogue runs for a 64- or
    128-wide layer that writes planes only, with no fp32 output, split-K, row or utterance term, and Cout % 8 == 0."""
    return bn % 64 == 0 and not case.get("f32") and not splitk and not case.get("row") and not case.get("utt") and \
        case["Cout"] % 8 == 0


def ping_pong(bn, swish):
    """ping_pong() of tdnn_gemm.cu: the 128-wide layer instance without swish runs its warpgroups ping-pong."""
    return bn == 128 and not swish


# ------------------------------------------------------------------------------------------------ shape search
def _width_ok(bn, cout, m, sms):
    if bn == 128:
        return cout >= 128 and m * _cdiv(cout, 128) >= sms
    return cout >= 64 and not (cout >= 128 and m * _cdiv(cout, 128) >= sms) and m * _cdiv(cout, 64) >= sms // 2


def staged_shape(sms, tb, bn, cout, b_tail="past", min_T=1):
    """(B, T) with choose_m_tile's Tb == tb, BLOCK_N == bn for this Cout, T not a multiple of Tb (Tb > 1) and B not a
    multiple of Bb = 128 / Tb.  b_tail "past": the last M tile's utterances end in its first 64-row half, so the second
    half's store box lies wholly past B (Tb <= 64); "part": they end inside the second half.  The first such shape in
    (T, B) order."""
    bb = 128 // tb
    need_m = _cdiv(sms, _cdiv(cout, 128)) if bn == 128 else _cdiv(sms // 2, _cdiv(cout, 64))
    t_range = [1] if tb == 1 and min_T == 1 else range(max(2, min_T), 5 * tb + 2)
    # ragged T first; where choose_m_tile never picks this Tb for a ragged T with enough tiles (Tb = 2: T odd pads a
    # frame per utterance, which Tb = 1 or 4 avoids), T a multiple of Tb
    for ragged in (True, False):
        for T in t_range:
            if tb > 1 and (T % tb != 0) != ragged:
                continue
            first = (_cdiv(need_m, _cdiv(T, tb)) - 1) * bb + 1       # the fewest utterances that give need_m tiles
            for B in range(first, first + 2 * bb):
                r = B % bb
                if bb > 1 and r == 0:
                    continue
                if bb > 2 and (b_tail == "past") != (r <= bb // 2):
                    continue
                if choose_m_tile(B, T) == tb and _width_ok(bn, cout, _cdiv(T, tb) * _cdiv(B, bb), sms):
                    return B, T
    raise ValueError("no shape for Tb={} BLOCK_N={} Cout={}".format(tb, bn, cout))


# Cout of the tail sweep per Tb: Cout % 64 in {0, 8, 56} (the staged path needs Cout % 8 == 0), one or several 64-channel
# pieces per tile
TAIL_COUT = {64: (72, 120, 64, 200, 248, 136, 256, 184), 128: (136, 184, 256, 264, 312, 200, 128, 392)}
# odd Cout (% 64 in {1, 63}) on both widths: plane-only launches that keep the direct stores and must not write past Cout
ODD_COUT = {"odd_w64_tb4_cout65": (4, 64, 65), "odd_w64_tb1_cout127": (1, 64, 127), "odd_w128_tb16_cout129": (16, 128, 129),
            "odd_w128_tb32_cout191": (32, 128, 191)}


def _lengths(B, T, tb, seed):
    """Lengths of a masked batch: 1, T - 1 and T, lengths that end inside a 64-row store box and at its end, and at a
    tile's edge in time (multiples of Tb); the rest random."""
    box = min(tb, 64)
    special = [T, 1, max(1, T - 1)]
    special += [v for v in (box // 2 + 1, box, tb, 2 * tb, tb + box // 2 + 1, 64, 64 + 13) if 1 <= v <= T]
    rng = np.random.RandomState(seed)
    lens = np.concatenate([special * (1 + B // len(special)), rng.randint(1, T + 1, B)])[:B]
    rng.shuffle(lens)
    lens[0] = T
    return [int(v) for v in lens]


def staged_cases(sms):
    """name -> layer case.  Keys beyond gemm_exact's: inst (BLOCK_N it is meant for), tb, lengths, groups, im2col, zero
    (the signed-zero case), y_c0 (8 or 72: the output's first channel in a wider pitch)."""
    D = dict
    cases = {}
    # 1. both staged widths x every Tb, ragged T and B, Cout % 64 in {0, 1, 8, 63}; B's tail alternates between a store
    #    box wholly past B and one that B ends in
    for bn in (64, 128):
        for i, tb in enumerate(TBS):
            cout = TAIL_COUT[bn][i]
            B, T = staged_shape(sms, tb, bn, cout, "past" if i % 2 == 0 else "part")
            cases["tail_w{}_tb{}_cout{}".format(bn, tb, cout)] = D(
                B=B, T=T, Cin=24, Cout=cout, ctx=[-2, 0, 1] if T > 1 else [0], relu=True, bn=i % 3 == 0, inst=bn, tb=tb)
    # 4. masked rows at every Tb on all four staged instances (the two layer and the two swish ones)
    for bn in (64, 128):
        for swish in (False, True):
            for i, tb in enumerate(TBS):
                cout = TAIL_COUT[bn][(i + 3) % 8]
                B, T = staged_shape(sms, tb, bn, cout, "part" if i % 2 == 0 else "past", min_T=2 if tb == 1 else 1)
                name = "masked_{}w{}_tb{}".format("swish_" if swish else "", bn, tb)
                cases[name] = D(B=B, T=T, Cin=16, Cout=cout, ctx=[-1, 0, 2], relu=not swish, bn=i % 2 == 1, inst=bn,
                                tb=tb, lengths=_lengths(B, T, tb, 7 * tb + bn + swish), act="swish" if swish else None)
    # 2. tiles per CTA on the ping-pong instance: warpgroup 1 idle, one CTA with two tiles, odd counts of both parities
    for nm, n in (("sms", sms), ("sms_p1", sms + 1), ("2sms_m1", 2 * sms - 1), ("3sms_p1", 3 * sms + 1)):
        cases["tiles_" + nm] = D(B=16 * n - (3 if n % 2 else 0), T=8, Cin=40, Cout=128, ctx=[-1, 0, 1], relu=True, bn=True,
                                 inst=128, tb=8, tiles=n)
    # 3. epilogue variants on the staged path
    v = {
        "bn_relu_w64": (16, 64, 72, D(relu=True, bn=True)),
        "bn_norelu_w64": (32, 64, 120, D(bn=True)),
        "nobn_relu_w128": (8, 128, 136, D(relu=True)),
        "nobn_norelu_w128": (4, 128, 184, D()),
        "swish_w64": (8, 64, 72, D(act="swish", relu=True)),
        "swish_bn_w128": (16, 128, 136, D(act="swish", bn=True)),
        "tanh_bn_w64": (8, 64, 80, D(act="tanh", bn=True)),
        "tanh_w128": (2, 128, 136, D(act="tanh", relu=True)),
        "sigmoid_w64": (64, 64, 120, D(act="sigmoid")),
        "sigmoid_bn_w128": (8, 128, 200, D(act="sigmoid", bn=True)),
        "x2_w128": (8, 128, 136, D(x2=True, relu=True, bn=True)),
        "x2_w64": (128, 64, 72, D(x2=True, relu=True)),
        "im2col_w128": (8, 128, 256, D(im2col=5, relu=True, bn=True)),
        "im2col_w64": (4, 64, 72, D(im2col=5, relu=True)),
        "zero_w128": (8, 128, 136, D(zero=True)),
        "zero_w64": (16, 64, 120, D(zero=True)),
    }
    v.update({name: (tb, bn, cout, D(relu=True, bn=True)) for name, (tb, bn, cout) in ODD_COUT.items()})
    for name, (tb, bn, cout, extra) in v.items():
        B, T = staged_shape(sms, tb, bn, cout, "past" if tb % 32 else "part")
        cin = 64 if extra.get("zero") else 24 if extra.get("im2col") else 40
        ctx = [0] if extra.get("im2col") else [-1, 0, 1]
        cases[name] = D(B=B, T=T, Cin=cin, Cout=cout, ctx=ctx, inst=bn, tb=tb, **extra)
    # grouped 1x1: Cout / G a multiple of 128 (ping-pong) and of 64; Cin / G multiples of 64
    cases["grouped_g2_ng128"] = D(B=7, T=29, Cin=128, Cout=256, ctx=[0], groups=2, relu=True, bn=True, inst=128)
    cases["grouped_g4_ng64"] = D(B=9, T=21, Cin=256, Cout=256, ctx=[0], groups=4, relu=True, inst=64)
    for i, (name, c) in enumerate(sorted(cases.items())):
        c.setdefault("act", None)
        if c.get("im2col"):
            c["cin0"], c["Cin"] = c["Cin"], c["im2col"] * c["Cin"]
        c["x_c0"] = 8
        c["ldx"] = gx._ru(c["x_c0"] + c["Cin"] + 8, 8)
        if c.get("x2"):
            c["x2_c0"], c["ldx2"] = 16, gx._ru(16 + c["Cin"] + 24, 8)
        c["y_c0"] = 8 if i % 2 == 0 else 72
        c["ldy"] = gx._ru(c["y_c0"] + c["Cout"] + 8, 8)
        c["yf_c0"], c["ldyf"] = 4, gx._ru(4 + c["Cout"] + 4, 4)
        c["planes"] = True
    return cases


def make_staged(case, seed):
    """Operands of a staged case (gemm_exact.make_layer, then what the case's flags change)."""
    d = gx.make_layer(dict(case, Cin=case.get("cin0", case["Cin"])) if case.get("im2col") else case, seed)
    B, T = case["B"], case["T"]
    if case.get("groups", 1) > 1:
        g = case["groups"]
        d["w_int"], d["w_frac"] = d["w_int"][:, :case["Cin"] // g], d["w_frac"][:, :case["Cin"] // g]
    if case.get("im2col"):
        # the first layer's im2col view: utterance b's frames padded by k // 2 zeros on both sides, frame t the window of
        # k consecutive frames; the reference sees the windows as one (B, T, k * Cin) input and a one-tap weight
        k, c0 = case["im2col"], case["cin0"]
        pads = []
        for hi_lo in d["xs"][0]:
            p = np.zeros((B, T + k - 1, c0), np.float32)
            p[:, k // 2:k // 2 + T] = hi_lo
            pads.append(p)
        d["pad"] = tuple(pads)
        d["xs"] = [tuple(np.stack([p[:, t:t + k].reshape(B, k * c0) for t in range(T)], axis=1) for p in pads)]
        rng = np.random.RandomState(seed + 1)
        d["w_int"] = gx.int_plane(rng, (case["Cout"], case["Cin"], 1))
        d["w_frac"] = gx.grid_plane(rng, (case["Cout"], case["Cin"], 1))
    if case.get("zero"):
        # every third output channel has an all -0.0 weight row and a -0.0 bias; non-negative frames make each of its
        # products -0, so the kernel's accumulator is -0 and -0 + -0 = -0 unless the epilogue adds a +0
        d["xs"] = [(np.abs(h), np.abs(lo)) for h, lo in d["xs"]]
        z = np.arange(case["Cout"]) % 3 == 0
        d["w_int"][z], d["w_frac"][z] = -0.0, -0.0
        d["bias"][z] = -0.0
    return d


def staged_reference(case, d):
    """-> (want, bound) as gemm_exact.layer_reference; masked rows (t >= lengths[b]) are +0."""
    acc = None
    g = case.get("groups", 1)
    if g > 1:
        kg, ng = case["Cin"] // g, case["Cout"] // g
        hi, lo = d["xs"][0]
        acc = np.concatenate([gx.layer_acc({"xs": [(hi[..., j * kg:(j + 1) * kg], lo[..., j * kg:(j + 1) * kg])],
                                            "w_int": d["w_int"][j * ng:(j + 1) * ng],
                                            "w_frac": d["w_frac"][j * ng:(j + 1) * ng]}, case["ctx"])
                              for j in range(g)], axis=2)
    want, bound = gx.layer_reference(case, d, acc)
    if bound is None:
        # the kernel adds its row term (+0 when absent) to every sum, so an exact -0 (a -0 bias on a -0 sum) stores +0
        want = want + np.float32(0.0)
    if case.get("lengths") is not None:
        dead = np.arange(case["T"])[None, :] >= np.asarray(case["lengths"])[:, None]
        want = np.where(dead[:, :, None], np.float32(0.0), want).astype(want.dtype)
        if bound is not None:
            bound = np.where(dead[:, :, None], 0.0, bound)
    return want, bound


# ------------------------------------------------------------------------------------------------ split-K
def splitk_case(sms):
    """tdnn6-like segment layer on the ping-pong instance with split-K: Cin 3000 = 47 channel blocks in 7 slices of
    7, 7, 7, 7, 7, 7 and 5 blocks, Cout 512 = 4 N blocks of 128, and ceil(B / 128) * 7 * 4 >= sms tiles."""
    B = 128 * _cdiv(sms, 28) - 37
    assert B <= 1024
    return dict(B=B, T=1, Cin=3000, Cout=512, ctx=[0], relu=True, bn=True, act=None, planes=True, f32=True, inst=128,
                x_c0=8, ldx=gx._ru(8 + 3000 + 8, 8), y_c0=8, ldy=gx._ru(8 + 512 + 8, 8), yf_c0=4, ldyf=gx._ru(4 + 512 + 4, 4))


def splitk_slices(cin):
    """(slices, channel blocks per slice) of splitk_slices in tdnn_gemm.cu for a layer that may split."""
    ncb = _cdiv(cin, 64)
    s = min(8, ncb // 6)
    kb = _cdiv(ncb, s)
    return _cdiv(ncb, kb), kb


# ------------------------------------------------------------------------------------------------ fused pooling
# (B, T) -> the Tb they are meant to get: Tb = 8 with only full blocks, Tb = 8 with a partial block (8, 8, 4 and
# 4 x 8 + 5); per other Tb two full blocks and a partial one of Tb / 2 frames (Tb = 2: 1 frame), and partial blocks of
# 3 and 27 frames
POOL_SHAPES = {(16, 24): 8, (48, 200): 8, (13, 20): 8, (11, 37): 8, (100, 3): 1, (49, 5): 2, (25, 10): 4, (7, 40): 16,
               (4, 80): 32, (2, 160): 64, (1, 320): 128, (70, 3): 4, (5, 27): 32}
POOL_COUTS = (132, 192, 252)          # Cout % 128 in {4, 64, 124}
POOL_CIN, POOL_CTX = 8, [-1, 0, 1]


def pool_cases():
    return {"pool_B{}_T{}_cout{}".format(B, T, POOL_COUTS[i % 3]): dict(
        B=B, T=T, Cin=POOL_CIN, Cout=POOL_COUTS[i % 3], ctx=POOL_CTX, relu=True, bn=True, tb=tb, x_c0=8,
        ldx=gx._ru(8 + POOL_CIN + 8, 8)) for i, ((B, T), tb) in enumerate(sorted(POOL_SHAPES.items()))}


def make_pool(case, seed):
    """Integer-valued layer outputs: frames and weights in {-1, 0, 1} (lo planes zero), integer bias and shift, BN
    scales 1 or 2.  Every output is then an integer of magnitude <= 2 * (Cin * ntaps + 4) + 4 = 60."""
    rng = np.random.RandomState(seed)
    B, T, Cin, Cout = case["B"], case["T"], case["Cin"], case["Cout"]
    tot = gx.context_span(case["ctx"])[2]
    return {"xs": [(gx.int_plane(rng, (B, T, Cin), 1), np.zeros((B, T, Cin), np.float32))],
            "w_int": gx.int_plane(rng, (Cout, Cin, tot), 1), "w_frac": np.zeros((Cout, Cin, tot), np.float32),
            "bias": gx.int_plane(rng, Cout, 4), "scale": (2.0 ** rng.randint(0, 2, Cout)).astype(np.float32),
            "shift": gx.int_plane(rng, Cout, 4)}


def block_stats(y, tb):
    """Exact per-time-block statistics of y (B, T, C): (nblk, B, 2C) float64 [mean | M2] and the valid count of each
    block."""
    B, T, C = y.shape
    nblk = _cdiv(T, tb)
    out = np.zeros((nblk, B, 2 * C))
    counts = []
    for g in range(nblk):
        blk = y[:, g * tb:min(T, (g + 1) * tb)].astype(np.float64)
        mean = blk.mean(axis=1)
        out[g, :, :C], out[g, :, C:] = mean, ((blk - mean[:, None]) ** 2).sum(axis=1)
        counts.append(blk.shape[1])
    return out, counts


def _fma(a, b, c, dt):
    if dt == np.float32:      # a * b is exact in float64 and, on the data here, so is the sum: one rounding, as fmaf
        return (a.astype(np.float64) * b + c.astype(np.float64)).astype(np.float32)
    return a * b + c


def _chan_merge(s, o, dt):
    """chan_merge of tdnn_gemm.cu on (n, mean, M2) arrays in dtype dt, every operation rounded in its order."""
    n, mean, m2 = s
    nb, meanb, m2b = o
    tot = (n + nb).astype(dt)
    live = tot > 0
    safe = np.where(live, tot, dt(1))
    d = (meanb - mean).astype(dt)
    wb = (nb / safe).astype(dt)
    nmean = _fma(d, wb, mean, dt)
    nm2 = (m2 + (m2b + ((d * d).astype(dt) * n).astype(dt) * wb).astype(dt)).astype(dt)
    return tot, np.where(live, nmean, mean).astype(dt), np.where(live, nm2, m2).astype(dt)


def pool_partials_emulated(y, tb, dt=np.float32):
    """The fused pooling epilogue's partials of y (B, T, C) in dtype dt, in the kernel's merge order: per lane q4 of a
    quad, the pairs of frames (8 i + 2 q4, + 1) of its chunks merged one after the other, then with lane q4 ^ 1 (Tb >= 4)
    and with lane q4 ^ 2 (Tb >= 8); lane 0 (of each 4-frame block for Tb = 4) emits.  Full 8-frame blocks take the
    kernel's division-free path, which is the same sequence with the counts folded.  -> (nblk, B, 2C)."""
    y = np.asarray(y, dt)
    B, T, C = y.shape
    nblk = _cdiv(T, tb)
    out = np.zeros((nblk, B, 2 * C), dt)
    z = np.zeros((B, C), dt)
    for g in range(nblk):
        t0 = g * tb
        nv = min(tb, T - t0)
        if tb == 1:
            out[g, :, :C] = y[:, t0]
            continue
        lanes = []
        for q in range(4 if tb >= 8 else tb // 2):
            s = (z, z, z)
            for i in range(max(1, tb // 8)):
                j = 8 * i + 2 * q
                v0, v1 = j < nv, j + 1 < nv
                x0 = y[:, t0 + j] if v0 else z
                x1 = y[:, t0 + j + 1] if v1 else z
                pn = np.full((B, C), dt(v0) + dt(v1), dt)
                pm = (dt(0.5) * (x0 + x1)).astype(dt) if v1 else (x0 if v0 else z)
                pm2 = ((dt(0.5) * (x0 - x1)).astype(dt) * (x0 - x1)).astype(dt) if v1 else z
                s = _chan_merge(s, (pn, pm, pm2), dt)
            lanes.append(s)
        if tb >= 4:
            lanes = [_chan_merge(lanes[k], lanes[k + 1], dt) for k in range(0, len(lanes), 2)]
        if tb >= 8:
            lanes = [_chan_merge(lanes[0], lanes[1], dt)]
        out[g, :, :C], out[g, :, C:] = lanes[0][1], lanes[0][2]
    return out


def pool_exact_blocks(tb, counts):
    """The blocks whose partials the kernel computes exactly on integer data, whatever the compiler contracts into
    fmas: those in which every merge weight is a power of two (or zero), i.e. a power-of-two frame count with Tb <= 16.
    Above that a lane merges its 2-frame pairs one after the other (counts 4 + 2, 6 + 2, ...), with weights 1/3, 1/5,
    ... that round.  -> bool per block."""
    return np.array([n & (n - 1) == 0 and tb <= 16 for n in counts])


def pool_block_bounds(y, tb):
    """Per-element bounds of the partials from gemm_exact.pool_reference's derivation, applied to each block on its own
    (a block is one pooling of at most Tb frames): |d mean| <= mean bound, |d M2| <= n x var bound."""
    B, T, C = y.shape
    nblk = _cdiv(T, tb)
    out = np.zeros((nblk, B, 2 * C))
    for g in range(nblk):
        blk = y[:, g * tb:min(T, (g + 1) * tb)].astype(np.float64)
        _, _, mb, vb = gx.pool_reference(blk, tb)
        out[g, :, :C], out[g, :, C:] = mb, blk.shape[1] * vb
    return out
