"""The Conformer's fp32 CUDA-core kernels (conformer.cu) on the GPU against tests/conformer_exact.py: rotary attention at
every key-tile edge, head size and rotary mode, LayerNorm at every rows-per-CTA count, lane tail and grid round, the
convolution module at every frame-block edge, and the subsampling head over both strides.

  * Inputs are poisoned: q / k / v, x, delta and the conv-module input are channel slices of wider buffers whose other
    channels, pitch padding and spare last utterance hold NaN.
  * Outputs are fenced: every output is a view inside a buffer filled with a NaN sentinel, with a spare utterance after
    the last one; everything outside the logical output must be bitwise unchanged.
  * Exact results are compared bit for bit (planes as split_bf16 of the reference, the sign of zero included);
    transcendental ones elementwise within the bounds derived in conformer_exact.
  * Refusals return XVB_EINVAL and write nothing; ops refuses tables that are too short and views whose rows do not
    collapse.
  * The kernel instances are read from torch.profiler in a child process, so this file starts no profiler session in the
    test process (the GEMM edge files' captures then start from the same state as without it)."""
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

import conformer_exact as cx
import gemm_exact as gx
from gpu_checks import Fenced, equal, profiled, within

pytestmark = pytest.mark.gpu

SMS_FOR_IDS = 132
EINVAL = -1
ACT = {"none": 0, "relu": 1, "swish": 2, "tanh": 3}


@pytest.fixture(scope="module")
def ops():
    from asv_subtools_b200 import ops as _ops
    assert torch.cuda.is_available()
    return _ops


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _seed(name):
    return zlib.crc32(name.encode()) & 0x7FFFFFFF


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _poisoned_f32(a, c0, ld):
    """(B, T, C) float32 as the slice [c0, c0 + C) of a (B + 1, T, ld) buffer that holds NaN everywhere else"""
    B, T, Cn = a.shape
    buf = torch.full((B + 1, T, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:B, :, c0:c0 + Cn] = _dev(a)
    return buf[:B, :, c0:c0 + Cn]


def _fenced_planes(ops, B, T, ld, c0, Cn):
    idx = (slice(0, B), slice(None), slice(c0, c0 + Cn))
    hi, lo = Fenced((B + 1, T, ld), torch.bfloat16, idx), Fenced((B + 1, T, ld), torch.bfloat16, idx)
    return hi, lo, ops.SplitPlanes(hi.view, lo.view, Cn)


def _check_planes(hi, lo, want, what):
    """Plane outputs bit for bit against split_bf16 of an exact float32 reference, and the fences around them."""
    wh, wl = gx.split_bf16(want)
    equal(_bits(hi.numpy()), _bits(wh), what + " hi")
    equal(_bits(lo.numpy()), _bits(wl), what + " lo")
    hi.check(what + " hi")
    lo.check(what + " lo")


def _check_planes_within(hi, lo, want, bound, what):
    """Planes of a transcendental result: hi + lo keeps 16 of fp32's 24 bits (+ 2^-16 relative)."""
    within(hi.numpy() + lo.numpy(), want, bound + 2.0 ** -16 * np.abs(want), what)
    hi.check(what + " hi")
    lo.check(what + " lo")


# ------------------------------------------------------------------------------------------------ rotary attention
_ATTN_SEEN = set()
_ATTN_PAT = re.compile(r"(rope_attention_kernel)<(\d+)>")


def _run_attention(ops, case, d, what, check, profile=False):
    B, T, H, dk = case["B"], case["T"], case["H"], case["dk"]
    qkv = _poisoned_f32(cx.qkv_rows(d), case["q_c0"], case["ldq"])
    yh, yl, y = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], H * dk)
    rope = _dev(d["rope"]) if d["rope"] is not None else None

    def run():
        ops.rope_attention(qkv, H, dk, y, rope=rope, rope_v=case["rot"] == "rope_v", score_mult=case["mult"])

    if profile:
        _ATTN_SEEN.update(profiled(run, _ATTN_PAT))
    else:
        run()
    torch.cuda.synchronize()
    check(yh, yl, what)


@pytest.mark.parametrize("name", sorted(cx.attention_cases()))
def test_rope_attention_exact(ops, name):
    case = cx.attention_cases()[name]
    for mode in ("uniform", "khot"):
        d = cx.make_attention(case, _seed(name + mode), mode)
        want = cx.attention_exact_reference(case, d, mode)
        _run_attention(ops, case, d, "{} {}".format(name, mode), lambda h, l, w: _check_planes(h, l, want, w))
    d = cx.make_attention(case, _seed(name + "random"), "random")
    want, bound = cx.attention_random_bound(case, d)
    _run_attention(ops, case, d, name + " random", lambda h, l, w: _check_planes_within(h, l, want, bound, w))


def _attention_instances(ops):
    """One exact k-hot case of each dk under torch.profiler -> the rope_attention_kernel<DK> names that ran."""
    cases = cx.attention_cases()
    for dk in (32, 64, 128):
        name = next(n for n in sorted(cases) if cases[n]["dk"] == dk and cases[n]["T"] > 32)
        d = cx.make_attention(cases[name], 1, "khot")
        want = cx.attention_exact_reference(cases[name], d, "khot")
        _run_attention(ops, cases[name], d, name, lambda h, l, w: _check_planes(h, l, want, w), profile=True)
    return _ATTN_SEEN


def test_every_attention_instance_ran(tmp_path):
    """The kernel names torch.profiler records: every rope_attention_kernel<DK> instance runs (one exact case of each dk,
    in a child process)."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    dst = tmp_path / "seen.txt"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(dst)], cwd=root, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, "child failed:\n{}\n{}".format(r.stdout[-3000:], r.stderr[-3000:])
    seen = set(dst.read_text().split())
    want = {"rope_attention_kernel<{}>".format(n) for n in (32, 64, 128)}
    assert want <= seen, "never ran: {}".format(sorted(want - seen))


# ------------------------------------------------------------------------------------------------ LayerNorm
def _ln_buffers(ops, case, d):
    B, T, C = case["B"], case["T"], case["C"]
    bufs = {"x": _poisoned_f32(d["x"], case["x_c0"], case["ldx"])}
    if "delta" in d:
        bufs["delta"] = _poisoned_f32(d["delta"], case["d_c0"], case["ldd"])
    fx = None
    if case["x_out"] == "other":
        fx = Fenced((B + 1, T, case["ldxo"]), torch.float32, (slice(0, B), slice(None), slice(case["xo_c0"], case["xo_c0"] + C)))
        bufs["x_out"] = fx.view
    elif case["x_out"] == "inplace":
        bufs["x_out"] = bufs["x"]
    planes = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], C) if case["y"] else None
    fy = Fenced((B + 1, T, case["ldyf"]), torch.float32, (slice(0, B), slice(None), slice(case["yf_c0"], case["yf_c0"] + C))) \
        if case["y_f32"] else None
    return bufs, fx, planes, fy


@pytest.mark.parametrize("name", sorted(cx.ln_cases(SMS_FOR_IDS)))
def test_layer_norm_exact(ops, sms, name):
    case = cx.ln_cases(sms)[name]
    d = cx.make_ln(case, _seed(name))
    ref = cx.ln_reference(case, d)
    bufs, fx, planes, fy = _ln_buffers(ops, case, d)
    t = lambda k: _dev(d[k]) if k in d else None      # noqa: E731
    second = None
    if case.get("second"):
        second = (t("gamma2"), t("beta2"))
    ops.layer_norm(bufs["x"], t("gamma"), t("beta"), eps=0.0, delta=bufs.get("delta"), delta_scale=case.get("delta_scale", 1.0),
                   table=t("table"), x_out=bufs.get("x_out"), second=second, act=ACT[case["act"]],
                   y=planes[2] if planes else None, y_f32=fy.view if fy else None)
    torch.cuda.synchronize()
    what = "{} (C={} rows={} warps={})".format(name, case["C"], case["B"] * case["T"], case["warps"])
    if case["x_out"] is not None:
        got = bufs["x_out"].cpu().numpy()
        equal(_bits(got), _bits(ref["x_out"]), what + " x_out")
        if fx is not None:
            fx.check(what + " x_out")
    else:
        equal(_bits(bufs["x"].cpu().numpy()), _bits(d["x"]), what + " x unchanged")
    if ref["bound"] is None:
        if fy is not None:
            equal(_bits(fy.numpy()), _bits(ref["y"]), what + " y_f32")
            fy.check(what + " y_f32")
        if planes:
            _check_planes(planes[0], planes[1], ref["y"], what + " y")
    else:
        if fy is not None:
            within(fy.numpy(), ref["y"], ref["bound"], what + " y_f32")
            fy.check(what + " y_f32")
            if planes:
                _check_planes(planes[0], planes[1], fy.numpy(), what + " y planes of y_f32")
        elif planes:
            _check_planes_within(planes[0], planes[1], ref["y"], ref["bound"], what + " y")


@pytest.mark.parametrize("C", [33, 1500, 8192])
def test_layer_norm_random_rows_within_bound(ops, C):
    case = dict(B=3, T=11, C=C)
    x, g, b = cx.make_ln_random(case, C)
    want, bound = cx.ln_random_bound(x.reshape(-1, C), g, b, 1e-5)
    xs = _poisoned_f32(x, 3, C + 5)
    fy = Fenced((4, 11, C + 6), torch.float32, (slice(0, 3), slice(None), slice(4, 4 + C)))
    ops.layer_norm(xs, _dev(g), _dev(b), eps=1e-5, y_f32=fy.view)
    torch.cuda.synchronize()
    within(fy.numpy().reshape(-1, C), want, bound, "random rows C={}".format(C))
    fy.check("random rows")


# ------------------------------------------------------------------------------------------------ convolution module
@pytest.mark.parametrize("name", sorted(cx.conv_cases()))
def test_conv_module_exact(ops, name):
    case = cx.conv_cases()[name]
    B, T, C = case["B"], case["T"], case["C"]
    d = cx.make_conv_module(case, _seed(name))
    x = _poisoned_f32(d["x"], case["x_c0"], case["ldx"])
    w, b, na, nb = _dev(d["w"]), _dev(d["b"]), _dev(d["na"]), _dev(d["nb"])
    for act in ("none", case["act"]):
        want, bound = cx.conv_module_reference(case, d, act)
        yh, yl, y = _fenced_planes(ops, B, T, case["ldy"], case["y_c0"], C)
        ops.conv_module(x, w, b, na, nb, y, batch_norm=case["norm"] == "bn", eps=0.0, act=ACT[act])
        torch.cuda.synchronize()
        what = "{} act {}".format(name, act)
        if bound is None:
            _check_planes(yh, yl, want, what)
        else:
            _check_planes_within(yh, yl, want, bound, what)


# ------------------------------------------------------------------------------------------------ subsampling head
@pytest.mark.parametrize("name", sorted(cx.subsample_cases(SMS_FOR_IDS)))
def test_subsample_head_exact(ops, sms, name):
    case = cx.subsample_cases(sms)[name]
    B, T, F, C, T1, F1 = case["B"], case["T"], case["F"], case["C"], case["T1"], case["F1"]
    d = cx.make_subsample(case, _seed(name))
    want = cx.subsample_reference(case, d)
    xb = torch.full((B + 1, T, F), float("nan"), device="cuda")
    xb[:B] = _dev(d["x"])
    idx = (slice(0, B),)
    yh, yl = Fenced((B + 1, T1, F1, C), torch.bfloat16, idx), Fenced((B + 1, T1, F1, C), torch.bfloat16, idx)
    ops.subsample_head(xb[:B], _dev(d["w"]), _dev(d["b"]), ops.SplitPlanes(yh.view, yl.view, C),
                       stride_f=None if case["sf"] == 2 else 1)
    torch.cuda.synchronize()
    _check_planes(yh, yl, want, name)


# ------------------------------------------------------------------------------------------------ refusals
def _untouched(fences, what):
    for f in fences:
        f.check(what)
        assert int((f.bits != f.sent).sum()) == 0, what + ": output written"


def test_refusals_write_nothing(ops):
    """Bad arguments return XVB_EINVAL before any launch: every output stays sentinel."""
    from asv_subtools_b200._lib import LayerNormArgs, lib
    import ctypes as C
    st = ops._stream()
    x = torch.zeros(4, 64, device="cuda")
    yf = Fenced((5, 64), torch.float32, (slice(0, 4),))
    yh, yl = Fenced((5, 64), torch.bfloat16, (slice(0, 4),)), Fenced((5, 64), torch.bfloat16, (slice(0, 4),))
    tab = torch.zeros(3, 64, device="cuda")

    def ln(**kw):
        a = LayerNormArgs()
        a.rows, a.C, a.eps, a.x, a.ldx = 4, 64, 1e-5, x.data_ptr(), 64
        a.y_f32, a.ldyf = yf.view.data_ptr(), 64
        for k, v in kw.items():
            setattr(a, k, v)
        rc = lib.xvb_layer_norm(C.byref(a), st)
        torch.cuda.synchronize()
        return rc

    assert ln() == 0
    yf.bits.fill_(yf.sent)
    for what, kw in {"C > 8192": dict(C=8193), "ldx < C": dict(ldx=63), "ldyf < C": dict(ldyf=60),
                     "table_rows = 0": dict(table=tab.data_ptr(), table_rows=0)}.items():
        assert ln(**kw) == EINVAL, what
        _untouched([yf], "layer_norm " + what)

    qkv = torch.zeros(2, 9, 3 * 2 * 64, device="cuda")
    rope = torch.zeros(9, 64, device="cuda")

    def attn(dk=64, ldq=3 * 2 * 64, rope_p=rope.data_ptr(), rope_v=0):
        rc = lib.xvb_rope_attention(qkv.data_ptr(), ldq, 2, 9, 2, dk, rope_p, rope_v, 1.0, yh.view.data_ptr(),
                                    yl.view.data_ptr(), 128, st)
        torch.cuda.synchronize()
        return rc

    for what, kw in {"dk 48": dict(dk=48), "dk 256": dict(dk=256), "ldq < 3 H dk": dict(ldq=3 * 128 - 8),
                     "rope_v without rope": dict(rope_p=None, rope_v=1)}.items():
        assert attn(**kw) == EINVAL, what
        _untouched([yh, yl], "rope_attention " + what)

    xc = torch.zeros(2, 5, 2 * 64, device="cuda")
    w = torch.zeros(64, 31, device="cuda")
    v64 = torch.zeros(8192, device="cuda")

    def conv(Cn=64, K=3, ldx=128):
        rc = lib.xvb_conv_module(xc.data_ptr(), ldx, 2, 5, Cn, w.data_ptr(), v64.data_ptr(), K, v64.data_ptr(),
                                 v64.data_ptr(), 1, 1e-5, 0, yh.view.data_ptr(), yl.view.data_ptr(), Cn, st)
        torch.cuda.synchronize()
        return rc

    cmax = cx.conv_max_channels(31)
    for what, kw in {"even K": dict(K=4), "smem > 200 KB": dict(Cn=cmax + 1, K=31, ldx=2 * (cmax + 1))}.items():
        assert conv(**kw) == EINVAL, what
        _untouched([yh, yl], "conv_module " + what)

    feats = torch.zeros(2, 9, 10, device="cuda")
    sw = torch.zeros(64 * 9, device="cuda")

    def head(B=2, T=9, F=10, Cn=8):
        rc = lib.xvb_subsample_head_stride(feats.data_ptr(), B, T, F, sw.data_ptr(), sw.data_ptr(), Cn, 1,
                                           yh.view.data_ptr(), yl.view.data_ptr(), st)
        torch.cuda.synchronize()
        return rc

    # 65536 x 6000 x 98 x 1 items >= 2^31: refused on the host before any launch
    for what, kw in {"T < 3": dict(T=2), "F < 3": dict(F=2), ">= 2^31 items": dict(B=65536, T=12001, F=100)}.items():
        assert head(**kw) == EINVAL, what
        _untouched([yh, yl], "subsample_head " + what)


def test_ops_refuses_short_tables_and_non_collapsing_views(ops):
    """ops checks what the kernels cannot: the rotary table covers T frames of dk, the positional table has C columns, and
    the rows of every fp32 operand collapse to (row * pitch) addressing."""
    B, T, H, dk = 2, 9, 2, 32
    qkv = torch.zeros(B, T, 3 * H * dk, device="cuda")
    y = ops.SplitPlanes.empty((B, T, H * dk), "cuda")
    for bad in (torch.zeros(T - 1, dk, device="cuda"), torch.zeros(T, dk // 2, device="cuda"),
                torch.zeros(T, dk, 2, device="cuda")):
        with pytest.raises(ValueError, match="rope"):
            ops.rope_attention(qkv, H, dk, y, rope=bad)
    ops.rope_attention(qkv, H, dk, y, rope=torch.zeros(T + 3, dk, device="cuda"))     # a longer table is fine
    x = torch.zeros(B, T, 40, device="cuda")
    for bad in (torch.zeros(T, 39, device="cuda"), torch.zeros(T, 41, device="cuda"), torch.zeros(40, device="cuda")):
        with pytest.raises(ValueError, match="table"):
            ops.layer_norm(x, table=bad, y_f32=torch.empty_like(x))
    # a time slice of a longer buffer: row (b, t) is not at (b T + t) * pitch
    long = torch.zeros(B, T + 4, 3 * H * dk, device="cuda")
    with pytest.raises(ValueError, match="collapse"):
        ops.rope_attention(long[:, :T], H, dk, y)
    xl = torch.zeros(B, T + 1, 40, device="cuda")
    for kw in (dict(x=xl[:, :T]), dict(x=x, delta=xl[:, :T]), dict(x=x, x_out=xl[:, :T]), dict(x=x, y_f32=xl[:, :T])):
        kw.setdefault("y_f32", torch.empty_like(x))
        with pytest.raises(ValueError, match="collapse"):
            ops.layer_norm(**kw)
    cm = torch.zeros(B, T + 2, 2 * 16, device="cuda")
    with pytest.raises(ValueError, match="collapse"):
        ops.conv_module(cm[:, :T], torch.zeros(16, 3, device="cuda"), torch.zeros(16, device="cuda"),
                        torch.ones(16, device="cuda"), torch.zeros(16, device="cuda"), ops.SplitPlanes.empty((B, T, 16), "cuda"))
    # channel slices and size-1 dimensions still collapse
    ops.layer_norm(torch.zeros(B, 1, 40, device="cuda")[..., :20], y_f32=torch.empty(B, 1, 20, device="cuda"))
    ops.layer_norm(torch.zeros(B, T, 80, device="cuda")[..., 8:48], y_f32=torch.empty_like(x))


if __name__ == "__main__":
    from asv_subtools_b200 import ops as _ops
    with open(sys.argv[1], "w") as f:
        f.write("\n".join(sorted(_attention_instances(_ops))))
