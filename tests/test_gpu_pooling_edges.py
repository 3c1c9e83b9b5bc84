"""The time-pooling kernels (csrc/pooling.cu, the pooling half of csrc/ecapa.cu) through the C ABI at every box, slab,
warp and channel edge of tests/pool_exact.py, each output element within its float64-derived bound.

  * Inputs are poisoned: x and the logits are channel slices of wider buffers whose other channels, pitch padding and
    spare last utterance hold NaN; in a masked batch the frames past each utterance's length are NaN too.
  * Outputs are fenced: out, out_hi and out_lo are views inside sentinel-filled buffers with a spare row; everything
    outside them must be bitwise unchanged.
  * Exact identities: plane outputs are split_bf16 of the fp32 output; a masked stats_pool row equals an unmasked call
    on that utterance alone; the vector- and scalar-logit branches of attn_head_stats_pool_kernel agree bit for bit,
    and so do its <1>, <2> and <4> instances (XVB_ATTN_ROWS is read once per process, so <2> and <4> run in child
    processes that write their outputs for this one to compare).
  * Refusals return XVB_EINVAL and write nothing.

Run directly (python tests/test_gpu_pooling_edges.py OUT.npz) it is the child: it runs the attention head cases under
whatever XVB_ATTN_ROWS it was given and saves their outputs and the kernel instances that ran."""
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    _here = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [_here, os.path.dirname(_here)]

import gemm_exact as gx
import pool_exact as px
from gpu_checks import Fenced, equal, profiled, within

pytestmark = pytest.mark.gpu

EINVAL = -1
_ATTN_KERNEL = re.compile(r"(attn_head_stats_pool_kernel)<\s*(\d+)\s*>")
WORST = {}          # family -> largest error / bound seen


@pytest.fixture(scope="module")
def lib():
    from asv_subtools_b200 import ops  # noqa: F401  (loads and checks the library)
    from asv_subtools_b200._lib import lib as _lib
    assert torch.cuda.is_available()
    return _lib


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _poisoned(a, ld, c0, lengths=None):
    """(B, T, C) float32 as the slice [c0, c0 + C) of a NaN (B + 1, T, ld) buffer; frames past lengths[b] NaN too.
    Returns (buffer, address of element [0, 0, c0])."""
    B, T, Cn = a.shape
    buf = torch.full((B + 1, T, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:B, :, c0:c0 + Cn] = _dev(a)
    if lengths is not None:
        for b, n in enumerate(lengths):
            buf[b, n:] = float("nan")
    return buf, buf.data_ptr() + 4 * c0


class _Out:
    """A fenced fp32 (B, W) output and, with planes, fenced (B, ldo) bf16 planes holding the row at column `off`."""

    def __init__(self, B, W, planes, ldo_pad):
        self.W = W
        self.f = Fenced((B + 1, W), torch.float32, slice(0, B))
        self.hi = self.lo = None
        self.ldo = W + ldo_pad
        if planes:
            idx = (slice(0, B), slice(ldo_pad, ldo_pad + W))
            self.hi = Fenced((B + 1, self.ldo), torch.bfloat16, idx)
            self.lo = Fenced((B + 1, self.ldo), torch.bfloat16, idx)

    def ptrs(self):
        if self.hi is None:
            return self.f.view.data_ptr(), None, None, self.ldo
        return self.f.view.data_ptr(), self.hi.view.data_ptr(), self.lo.view.data_ptr(), self.ldo

    def result(self, what):
        """The fp32 output, after the fences and the planes = split_bf16(fp32) identity are checked."""
        torch.cuda.synchronize()
        got = self.f.numpy()
        self.f.check(what + " out")
        if self.hi is not None:
            wh, wl = gx.split_bf16(got)
            nan = np.isnan(got)           # a NaN output (unbiased std of one frame) splits into NaN planes, any payload
            for f, w, p in ((self.hi, wh, " out_hi"), (self.lo, wl, " out_lo")):
                g = f.numpy()
                assert np.isnan(g[nan]).all(), what + p + ": a NaN output did not split into NaN"
                equal(np.where(nan, 0, g), np.where(nan, 0, w), what + p)
            self.hi.check(what + " out_hi")
            self.lo.check(what + " out_lo")
        return got


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ------------------------------------------------------------------------------------------------ launches
def _run_stats(lib, case, d, x=None, B=None, T=None, lengths=None):
    B = case["B"] if B is None else B
    T = case["T"] if T is None else T
    x = d["x"][:, :T] if x is None else x
    buf, xp = _poisoned(x, case["ldx"], case["c0"], lengths)
    out = _Out(B, 2 * case["C"], case["planes"], case["ldo_pad"])
    o, h, l, ldo = out.ptrs()
    if lengths is None:
        rc = lib.xvb_stats_pool_ex(xp, case["ldx"], B, T, case["C"], case["eps"], case["mode"], o, h, l, ldo, None)
    else:
        lens = _dev(np.asarray(lengths, dtype=np.int32))
        rc = lib.xvb_stats_pool_lengths(xp, case["ldx"], B, T, case["C"], case["eps"], case["mode"], lens.data_ptr(), o, h,
                                        l, ldo, None)
    assert rc == 0
    return out, buf


def _run_finalize(lib, case, d):
    p = _dev(d["partial"])
    out = _Out(case["B"], 2 * case["C"], case["planes"], case["ldo_pad"])
    o, h, l, ldo = out.ptrs()
    rc = lib.xvb_pool_finalize(p.data_ptr(), case["nblk"], case["tb"], case["B"], case["T"], case["C"], case["eps"],
                               case["mode"], o, h, l, ldo, None)
    assert rc == 0
    return out, p


def _run_attn(lib, case, d, ldl=None):
    B, T, C = case["B"], case["T"], case["C"]
    ldl = case["ldl"] if ldl is None else ldl
    lb, lp = _poisoned(d["l"][:, :T], ldl, case["l0"])
    xb, xp = _poisoned(d["x"][:, :T], case["ldx"], case["x0"])
    out = _Out(B, 2 * case["O"], case["planes"], 0)
    o, h, l, ldo = out.ptrs()
    k = case["kind"]
    if k == "attn":
        rc = lib.xvb_attn_stats_pool(lp, ldl, xp, case["ldx"], B, T, C, case["floor"], o, h, l, ldo, None)
    elif case["mq"]:
        rc = lib.xvb_attn_head_stats_pool_mq(lp, ldl, case["G"], xp, case["ldx"], B, T, C, case["O"], case["gdiv"],
                                             case["head_width"], case["rep"], case["floor"], int(case["unweighted"]), o, h,
                                             l, ldo, None)
    else:
        keep = []
        pl = px_ = None
        if case["xi"]:
            keep = [_dev(d["prior_l"]), _dev(d["prior_x"])]
            pl, px_ = keep[0].data_ptr(), keep[1].data_ptr()
        rc = lib.xvb_attn_head_stats_pool_prior(lp, ldl, case["G"], xp, case["ldx"], B, T, C, case["O"], case["gdiv"],
                                                case["floor"], int(case["unweighted"]), pl, px_, int(case["xi"]), o, h, l,
                                                ldo, None)
        torch.cuda.synchronize()
    assert rc == 0
    return out, (lb, xb)


def _run_lde(lib, case, d):
    B, T, C, K = case["B"], case["T"], case["C"], case["K"]
    xb, xp = _poisoned(d["x"][:, :T], case["ldx"], case["x0"])
    mu, nb = _dev(d["mu"]), _dev(d["neg_beta"])
    w = torch.full((B * T, K), float("nan"), dtype=torch.float32, device="cuda")
    out = _Out(B, C * K, case["planes"], case["ldo_pad"])
    o, h, l, ldo = out.ptrs()
    rc = lib.xvb_lde_pool(xp, case["ldx"], B, T, C, mu.data_ptr(), K, nb.data_ptr(), w.data_ptr(), o, h, l, ldo, None)
    assert rc == 0
    return out, (xb, mu, nb, w)


def _run_plane(lib, case, d):
    B, T, C, ld = case["B"], case["T"], case["C"], case["ldx"]
    c0 = (ld - C) // 2 // 8 * 8
    bufs = []
    for a in (d["hi"], d["lo"]):
        buf = torch.full((B + 1, T, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
        buf[:B, :, c0:c0 + C] = _dev(a[:, :T]).to(torch.bfloat16)
        bufs.append(buf)
    out = _Out(B, C, case["planes"], case["ldo_pad"])
    o, h, l, ldo = out.ptrs()
    rc = lib.xvb_plane_mean(bufs[0].data_ptr() + 2 * c0, bufs[1].data_ptr() + 2 * c0, ld, B, T, C, o, h, l, ldo, None)
    assert rc == 0
    return out, bufs


def _run(lib, case, d):
    k = case["kind"]
    if k == "stats":
        return _run_stats(lib, case, d, lengths=case["lengths"])
    if k == "finalize":
        return _run_finalize(lib, case, d)
    if k in ("attn", "head"):
        return _run_attn(lib, case, d)
    if k == "lde":
        return _run_lde(lib, case, d)
    return _run_plane(lib, case, d)


def _check(lib, name):
    case = px.all_cases()[name]
    d = px.make_case(case, _seed(name))
    ref = px.reference(case, d)
    out, keep = _run(lib, case, d)
    got = out.result(name)
    want = px.flat_output(case, {k: v[0] for k, v in ref.items()})
    bound = px.flat_output(case, {k: v[1] for k, v in ref.items()})
    r = within(got, want, bound, name)
    WORST[case["kind"]] = max(WORST.get(case["kind"], 0.0), r)
    return case, d, got


# ------------------------------------------------------------------------------------------------ values
@pytest.mark.parametrize("name", sorted(px.stats_cases()))
def test_stats_pool(lib, name):
    case, d, got = _check(lib, name)
    if case["lengths"]:
        # row b of the masked batch = an unmasked call on utterance b alone: the same frames in the same order
        for b, n in enumerate(case["lengths"]):
            out, _ = _run_stats(lib, case, d, x=d["x"][b:b + 1, :n], B=1, T=n)
            equal(_bits(out.result("{} utterance {}".format(name, b))), _bits(got[b:b + 1]),
                  "{}: masked row {} vs its own call".format(name, b))


@pytest.mark.parametrize("name", sorted(px.finalize_cases()))
def test_pool_finalize(lib, name):
    _check(lib, name)


@pytest.mark.parametrize("name", sorted(px.attn_cases()))
def test_attn_stats_pool(lib, name):
    _check(lib, name)


@pytest.mark.parametrize("name", sorted(px.head_cases()))
def test_attn_head_stats_pool(lib, name):
    case, d, got = _check(lib, name)
    if case["vector"]:
        # the same logits at a pitch that is not a multiple of 4: the scalar-logit branch, bit for bit
        out, _ = _run_attn(lib, case, d, ldl=case["G"] + 1)
        equal(_bits(out.result(name + " scalar logits")), _bits(got), name + ": scalar vs vector logit branch")


@pytest.mark.parametrize("name", sorted(px.lde_cases()))
def test_lde_pool(lib, name):
    _check(lib, name)


@pytest.mark.parametrize("name", sorted(px.plane_cases()))
def test_plane_mean(lib, name):
    _check(lib, name)


# ------------------------------------------------------------------------------------------------ kernel instances
def _head_outputs(lib):
    """Every attention head case's fp32 output, and the attn_head_stats_pool_kernel instances that ran."""
    outs = {}

    def run():
        for name, case in sorted(px.head_cases().items()):
            out, _ = _run_attn(lib, case, px.make_case(case, _seed(name)))
            outs[name] = out.result(name)

    seen = profiled(run, _ATTN_KERNEL)
    return outs, seen


def test_attn_rows_instances_are_bitwise_equal(lib, tmp_path):
    """XVB_ATTN_ROWS = 1 (this process), 2 and 4 (child processes): each warp adds frames w, w + 8, w + 16, ... in the
    same order in every instance, so the outputs must agree bit for bit, and each instance must have run."""
    outs, seen = _head_outputs(lib)
    assert "attn_head_stats_pool_kernel<1>" in seen, sorted(seen)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for rows in (2, 4):
        dst = tmp_path / "rows{}.npz".format(rows)
        env = dict(os.environ, XVB_ATTN_ROWS=str(rows))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), str(dst)], cwd=root, env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, "XVB_ATTN_ROWS={} child failed:\n{}\n{}".format(rows, r.stdout[-3000:], r.stderr[-3000:])
        got = np.load(dst)
        assert "attn_head_stats_pool_kernel<{}>".format(rows) in set(got["__seen__"].tolist()), got["__seen__"]
        for name, want in outs.items():
            equal(_bits(got[name]), _bits(want), "{}: XVB_ATTN_ROWS={} vs 1".format(name, rows))


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals_return_einval_and_write_nothing(lib):
    B, T, C = 2, 8, 128
    x = torch.zeros(B + 1, T, C + 8, device="cuda")
    lens = torch.full((65536,), T, dtype=torch.int32, device="cuda")
    out = Fenced((B + 1, 4 * C), torch.float32, slice(0, B))
    hi = Fenced((B + 1, 4 * C), torch.bfloat16, slice(0, B))
    lo = Fenced((B + 1, 4 * C), torch.bfloat16, slice(0, B))
    p, o, h, l = x.data_ptr(), out.view.data_ptr(), hi.view.data_ptr(), lo.view.data_ptr()
    part = torch.zeros(4, B, 2 * C, device="cuda")
    mu, nb, w = torch.zeros(C, 64, device="cuda"), torch.zeros(65, device="cuda"), torch.zeros(B * T, 65, device="cuda")
    ld = C + 8
    calls = {
        "stats_pool_ex B=65536": lambda: lib.xvb_stats_pool_ex(p, ld, 65536, 1, 4, 1e-10, 0, o, h, l, 8, None),
        "stats_pool_lengths B=65536": lambda: lib.xvb_stats_pool_lengths(p, ld, 65536, 1, 4, 1e-10, 0, lens.data_ptr(), o, h,
                                                                         l, 8, None),
        "pool_finalize B=65536": lambda: lib.xvb_pool_finalize(part.data_ptr(), 1, 1, 65536, 1, 4, 1e-10, 0, o, h, l, 8, None),
        "attn_stats_pool B=65536": lambda: lib.xvb_attn_stats_pool(p, ld, p, ld, 65536, 1, 4, 1e-5, o, h, l, 8, None),
        "attn_head B=65536": lambda: lib.xvb_attn_head_stats_pool(p, ld, 4, p, ld, 65536, 1, 4, 4, 1, 1e-5, 0, o, h, l, 8, None),
        "attn_head_prior B=65536": lambda: lib.xvb_attn_head_stats_pool_prior(p, ld, 4, p, ld, 65536, 1, 4, 4, 1, 1e-5, 0, None,
                                                                              None, 0, o, h, l, 8, None),
        "attn_head_mq B=65536": lambda: lib.xvb_attn_head_stats_pool_mq(p, ld, 4, p, ld, 65536, 1, 4, 4, 1, 4, 1, 1e-5, 0, o, h,
                                                                        l, 8, None),
        "lde_pool B=65536": lambda: lib.xvb_lde_pool(p, ld, 65536, 1, 4, mu.data_ptr(), 4, nb.data_ptr(), w.data_ptr(), o, h, l,
                                                     16, None),
        "plane_mean B=65536": lambda: lib.xvb_plane_mean(p, p, ld, 65536, 1, 8, o, h, l, 8, None),
        "lde_pool K=0": lambda: lib.xvb_lde_pool(p, ld, B, T, C, mu.data_ptr(), 0, nb.data_ptr(), w.data_ptr(), o, h, l, 0,
                                                 None),
        "lde_pool K=65": lambda: lib.xvb_lde_pool(p, ld, B, T, 4, mu.data_ptr(), 65, nb.data_ptr(), w.data_ptr(), o, None,
                                                  None, 0, None),
        "stats_pool_ex C=130": lambda: lib.xvb_stats_pool_ex(p, ld, B, T, 130, 1e-10, 0, o, h, l, 260, None),
        "stats_pool_lengths C=126": lambda: lib.xvb_stats_pool_lengths(p, ld, B, T, 126, 1e-10, 0, lens.data_ptr(), o, h, l,
                                                                       252, None),
        "attn_stats_pool C=130": lambda: lib.xvb_attn_stats_pool(p, ld, p, ld, B, T, 130, 1e-5, o, h, l, 260, None),
        "attn_head C=130": lambda: lib.xvb_attn_head_stats_pool(p, ld, 130, p, ld, B, T, 130, 130, 1, 1e-5, 0, o, h, l, 260,
                                                                None),
        "pool_finalize 4 x 8 frames for T=33": lambda: lib.xvb_pool_finalize(part.data_ptr(), 4, 8, B, 33, C, 1e-10, 0, o, h,
                                                                             l, 2 * C, None),
        "pool_finalize 4 x 8 frames for T=24": lambda: lib.xvb_pool_finalize(part.data_ptr(), 4, 8, B, 24, C, 1e-10, 0, o, h,
                                                                             l, 2 * C, None),
        "stats_pool_ex ldo < 2C": lambda: lib.xvb_stats_pool_ex(p, ld, B, T, C, 1e-10, 0, o, h, l, 2 * C - 4, None),
        "stats_pool_lengths ldo < 2C": lambda: lib.xvb_stats_pool_lengths(p, ld, B, T, C, 1e-10, 0, lens.data_ptr(), o, h, l,
                                                                          2 * C - 4, None),
        "pool_finalize ldo < 2C": lambda: lib.xvb_pool_finalize(part.data_ptr(), 1, 8, B, T, C, 1e-10, 0, o, h, l, 2 * C - 4,
                                                                None),
        "attn_stats_pool ldo < 2C": lambda: lib.xvb_attn_stats_pool(p, ld, p, ld, B, T, C, 1e-5, o, h, l, 2 * C - 4, None),
        "attn_head ldo < 2O": lambda: lib.xvb_attn_head_stats_pool(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 0, o, h, l, 2 * C - 4,
                                                                   None),
        "attn_head_mq ldo < 2O": lambda: lib.xvb_attn_head_stats_pool_mq(p, ld, C, p, ld, B, T, C, C, 1, 32, 1, 1e-5, 0, o, h,
                                                                         l, 2 * C - 4, None),
    }
    for what, call in calls.items():
        assert call() == EINVAL, what
    torch.cuda.synchronize()
    for f, what in ((out, "out"), (hi, "out_hi"), (lo, "out_lo")):
        f.check("refusals " + what)
        assert int((f.bits[:B] != f.sent).sum()) == 0, "a refused call wrote " + what


def test_report_worst_ratio():
    """The largest error / bound seen per kernel family in this session (printed with -s)."""
    for k, v in sorted(WORST.items()):
        print("{:10s} largest error / bound = {:.3g}".format(k, v))


if __name__ == "__main__":
    from asv_subtools_b200._lib import lib as _lib
    outs, seen = _head_outputs(_lib)
    np.savez(sys.argv[1], __seen__=np.array(sorted(seen)), **outs)
