"""Operands, case catalogue and references for CAM++'s fp32 CUDA-core kernels (csrc/campplus.cu): the context-aware mask
(xvb_cam_gate) and the BN -> ReLU over split planes (xvb_bn_relu_planes).

cam_gate, in the kernel's order: per segment, every frame lane sums its frames and the lanes are reduced in a fixed
order (S[s, c]); total = sum_s S; mean = fl32(total / T); ctx = fl32(mean + fl32(S / n)) with n the segment's own length
(the last segment may be short); hid = relu(W1 ctx + b1); gate = sigmoid(W2 hid + b2).  h holds multiples of 2^-8 whose
sums stay below 2^16 (asserted), so S and total are exact in any order, and numpy float32 then reproduces the mean and the
contexts bit for bit.  Two weight sets:
  (a) T and the segment lengths are powers of two and h is on a coarse grid: the contexts are exact, and a dense
      small-integer W1 sums them exactly (asserted from the grid and the sum of |terms|).
  (b) any T: W1 holds one +-2^e per row, so each hidden value is one exact product plus one rounded add of b1, which
      float32 reproduces.
W2 holds one +-2^e per row in both, so W2 hid + b2 rounds once (float32 again), and the sigmoid 1 / (1 + expf(-z)) is
checked within 2^-21 relative (gemm_exact.layer_reference's sigmoid bound).

bn_relu_planes: relu(fmaf(x, scale, shift)) on grid planes, power-of-two scales and grid shifts: exact.

Plain numpy (no torch, no GPU): test_gpu_campplus_edges.py runs these on the device and test_campplus_exact_host.py
checks them on the CPU."""
import numpy as np

import gemm_exact as gx

GATE_THREADS = 256
MAX_SMEM = 227 * 1024


def _ru(x, m):
    return (x + m - 1) // m * m


def cam_gate_smem(T, C, seg_len, R):
    """Dynamic shared memory of xvb_cam_gate: nseg x C contexts, nseg x R hidden values, lanes x C partial sums with
    lanes = 256 / (C / 8) frame lanes."""
    nseg = -(-T // seg_len)
    return (nseg * C + nseg * R + (GATE_THREADS // (C // 8)) * C) * 4


def cam_lanes(C):
    return GATE_THREADS // (C // 8)


def cam_cases():
    """name -> cam_gate case.  (b) covers T in {1, 99, 100, 101, 200, 201, 3000} (T % 100 at 0 and +-1), seg_len 1, 7,
    100 and > T, and C in {8, 424, 512, 2048} (256, 4, 4 and 1 frame lanes; at 424 = 53 groups, 44 threads idle); (a)
    covers power-of-two T and segment lengths with dense W1.  h is the slice at 8 of a NaN buffer of pitch > C; the
    (B, nseg, G) output sits in a buffer with a spare utterance of sentinel after it."""
    D = dict
    cases = {}
    Cs = (8, 424, 512, 2048)
    i = 0
    for j, T in enumerate((1, 99, 100, 101, 200, 201, 3000)):
        for k, seg in enumerate((1, 7, 100, T + 5)):
            C, R, G = Cs[(j + k) % 4], (16, 64, 128)[i % 3], (24, 128, 32)[i % 3]
            i += 1
            if cam_gate_smem(T, C, seg, R) > MAX_SMEM:
                continue                        # more segments than one CTA's shared memory holds (refused)
            cases["b_T{}_seg{}_C{}".format(T, seg, C)] = D(B=2, T=T, C=C, seg_len=seg, R=R, G=G, dense=False)
    for T, seg, C in ((64, 16, 8), (256, 64, 512), (256, 512, 2048), (64, 1, 424), (4, 2, 2048)):
        cases["a_T{}_seg{}_C{}".format(T, seg, C)] = D(B=3, T=T, C=C, seg_len=seg, R=32, G=40, dense=True)
    cases["b_B5_T3000_seg100_C512_R256"] = D(B=5, T=3000, C=512, seg_len=100, R=256, G=512, dense=False)
    for c in cases.values():
        c["nseg"] = -(-c["T"] // c["seg_len"])
        c["smem"] = cam_gate_smem(c["T"], c["C"], c["seg_len"], c["R"])
        c["h_c0"], c["ldh"] = 8, _ru(8 + c["C"] + 8, 8)
    return cases


def make_cam(case, seed):
    """-> dict(h_hi, h_lo (B, T, C) planes, w1 (R, C), b1 (R,), w2 (G, R), b2 (G,))"""
    rng = np.random.RandomState(seed)
    B, T, C, R, G = case["B"], case["T"], case["C"], case["R"], case["G"]
    if case["dense"]:
        hi = gx.int_plane(rng, (B, T, C), 2)
        lo = (rng.randint(-1, 2, (B, T, C)) * 0.25).astype(np.float32)    # 2^-2 grid: bf16-exact, so h = hi + lo
        w1 = rng.randint(-1, 2, (R, C)).astype(np.float32)
        b1 = (rng.randint(-8, 9, R) * 0.25).astype(np.float32)
    else:
        hi, lo = gx.frame_planes(rng, (B, T, C))
        w1 = np.zeros((R, C), np.float32)
        w1[np.arange(R), rng.randint(0, C, R)] = (rng.choice([-1.0, 1.0], R) * 2.0 ** rng.randint(-1, 2, R))
        b1 = gx.grid_values(rng, R, 1.0)
    w2 = np.zeros((G, R), np.float32)
    w2[np.arange(G), rng.randint(0, R, G)] = rng.choice([-1.0, 1.0], G) * 2.0 ** rng.randint(-4 if case["dense"] else -1, 1, G)
    b2 = gx.grid_values(rng, G, 1.0)
    return {"h_hi": hi, "h_lo": lo, "w1": w1, "b1": b1, "w2": w2, "b2": b2}


def cam_contexts(case, d, seg_len=None):
    """(B, nseg, C) float32 contexts in the kernel's order.  seg_len: a different segment length for the short last
    segment's divisor (None: the kernel's own n) -- only to show that the choice matters."""
    B, T, C, L = case["B"], case["T"], case["C"], case["seg_len"]
    h = (d["h_hi"] + d["h_lo"]).astype(np.float64)
    assert np.array_equal(h, (d["h_hi"] + d["h_lo"]).astype(np.float32)), "h = hi + lo rounds"
    assert np.all(h * 256 == np.round(h * 256)) and float(np.abs(h).sum(axis=1).max()) < 2.0 ** 16, "segment sums round"
    nseg = case["nseg"]
    S = np.stack([h[:, s * L:min(T, (s + 1) * L)].sum(axis=1) for s in range(nseg)], axis=1)       # exact
    total = S.sum(axis=1, keepdims=True)
    mean = total.astype(np.float32) / np.float32(T)
    n = np.array([min(T, (s + 1) * L) - s * L for s in range(nseg)], np.float32)
    if seg_len is not None:
        n[-1] = seg_len
    return mean + S.astype(np.float32) / n[None, :, None]


def cam_hidden(case, d, ctx):
    """relu(W1 ctx + b1) (B, nseg, R) float32: dense W1 exactly (asserted), one entry per row as one product + one add."""
    w1 = d["w1"]
    if case["dense"]:
        c64 = ctx.astype(np.float64)
        e = 0
        while not np.array_equal(c64 * 2.0 ** e, np.round(c64 * 2.0 ** e)):
            e += 1
        mag = np.abs(c64) @ np.abs(w1.astype(np.float64)).T
        assert float(mag.max()) * 2.0 ** max(e, 2) < 2.0 ** 24, "dense W1 sums round"
        acc = gx.exact_f32(c64 @ w1.astype(np.float64).T + d["b1"])
        return np.maximum(acc, np.float32(0.0))
    col = np.argmax(w1 != 0, axis=1)
    w = w1[np.arange(w1.shape[0]), col]
    acc = ctx[..., col] * w                                   # exact: a power of two
    return np.maximum(acc + d["b1"], np.float32(0.0))


def cam_reference(case, d, seg_len=None):
    """-> (gate float64 (B, nseg, G), bound)"""
    hid = cam_hidden(case, d, cam_contexts(case, d, seg_len))
    w2 = d["w2"]
    col = np.argmax(w2 != 0, axis=1)
    z = hid[..., col] * w2[np.arange(w2.shape[0]), col] + d["b2"]       # one exact product, one rounded add (float32)
    with np.errstate(over="ignore"):
        out = 1.0 / (1.0 + np.exp(-z.astype(np.float64)))
    return out, 2.0 ** -21 * out + 2.0 ** -120


# ------------------------------------------------------------------------------------------------ bn_relu_planes
def bn_relu_cases(sms):
    """name -> bn_relu_planes case: channel slices of x and y at different pitches and offsets, C = 8, and one shape
    with more than 32 sms * 256 eight-channel items (the grid-stride loop goes round again)."""
    D = dict
    cases = {"C8": D(B=3, T=17, C=8), "C64_T1": D(B=5, T=1, C=64), "C136": D(B=2, T=33, C=136),
             "C512": D(B=2, T=100, C=512),
             "grid_stride_C64": D(B=2, T=sms * 32 * 256 // 16 + 77, C=64)}
    for c in cases.values():
        C = c["C"]
        c["x_c0"], c["ldx"] = 8, _ru(8 + C + 16, 8)
        c["y_c0"], c["ldy"] = 16, _ru(16 + C + 8, 8) + 8
        assert c["ldx"] != c["ldy"]
        c["items"] = c["B"] * c["T"] * C // 8
    return cases


def make_bn_relu(case, seed):
    rng = np.random.RandomState(seed)
    C = case["C"]
    hi, lo = gx.frame_planes(rng, (case["B"], case["T"], C))
    return {"hi": hi, "lo": lo, "scale": (gx.pow2_scales(rng, C) * rng.choice([-1.0, 1.0], C)).astype(np.float32),
            "shift": gx.grid_values(rng, C)}


def bn_relu_reference(d):
    v = (d["hi"].astype(np.float64) + d["lo"]) * d["scale"] + d["shift"]
    return gx.exact_f32(np.maximum(v, 0.0))
