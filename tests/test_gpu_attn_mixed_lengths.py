"""Masked batches of utterances of different lengths on the Python launch sequences: the attention-pooling and xi-vector
TDNN x-vectors (AttentionPoolingExtractor) and the F-TDNN (FtdnnExtractor).  Needs an H100 (`-m gpu`).

  * Kernel: each row of xvb_attn_head_stats_pool_lengths is bit-identical to an unmasked call on that utterance alone,
    for every head map, both variance branches and the xi-vector form with and without a prior; inputs past each end
    are NaN, outputs are fenced; every length equal to T gives the unmasked entry's bytes; the XVB_ATTN_ROWS = 1 / 2 / 4
    instances, each in a child process, give the same bytes; bad arguments return XVB_EINVAL and write nothing.
  * Staging: xvb_split_frames_lengths equals xvb_split_frames inside each length and writes zeros past it.
  * Extractors: rows of 64-utterance batches against solo extraction, a subset against the oracle, the goldens packed
    into mixed batches, every length equal to T, pad content, bad lengths, the LDE refusal.
  * CLI: pipeline/extract_embeddings.py --mixed-lengths.

Run directly (python tests/test_gpu_attn_mixed_lengths.py OUT.npz) it is the child: it runs the kernel cases under
whatever XVB_ATTN_ROWS it was given and saves their outputs and the kernel instances that ran."""
import gc
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

if __name__ == "__main__":
    _here = os.path.dirname(os.path.abspath(__file__))
    sys.path[:0] = [_here, os.path.dirname(_here)]

from gpu_checks import Fenced, equal, profiled  # noqa: E402
from oracle import nnet as onn  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -1
EMB_TOL = 1e-4
_ATTN_KERNEL = re.compile(r"(attn_head_stats_pool_kernel)<\s*(\d+)\s*>")

# the attention poolings of tests/golden/make_golden_snowdar.py (LDE excluded: it does not take lengths)
POOLING_CASES = {
    "attn1": ("attentive", {}, 311),
    "attn2": ("attentive", {"affine_layers": 2, "hidden_size": 64}, 312),
    "mha_share": ("multi-head", {"num_head": 4}, 313),
    "mha_full": ("multi-head", {"num_head": 4, "share": False, "affine_layers": 2}, 314),
    "mres": ("multi-resolution", {"num_head": 4, "temperature": True, "affine_layers": 2}, 315),
    "xi_mean": ("xi-postmean-softplus2", {"hidden_size": 64, "num_nodes": 200}, 319),
    "xi_dist": ("xi-postdist-softplus2", {"hidden_size": 64, "num_nodes": 200}, 320),
}
MODELS = sorted(POOLING_CASES) + ["ftdnn"]
WORST = {}          # (model, pos) -> (largest |masked - solo| / max |solo|, every row bit-identical)


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def cos(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return float(np.dot(a, b) / (np.linalg.norm(a) * np.linalg.norm(b)))


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ================================================================================================ kernel
KT = 70
KLENS = [1, 7, 8, 9, 31, 32, 33, KT]
KC = 68                     # C % 128 != 0: inactive lanes; 68 / 4 heads = 17-channel heads
# name -> (O, G, gdiv, unweighted, xi: 0 none / 1 softplus2log without prior / 2 with prior)
KCASES = {
    "shared": (KC, 1, KC, 0, 0),
    "shared_unweighted": (KC, 1, KC, 1, 0),
    "heads_shared": (KC, 4, KC // 4, 0, 0),
    "per_channel": (KC, KC, 1, 0, 0),
    "per_channel_unweighted": (KC, KC, 1, 1, 0),
    "global_shared": (4 * KC, 4, KC, 0, 0),
    "global_per_channel": (4 * KC, 4 * KC, 1, 0, 0),
    "global_unweighted": (4 * KC, 4, KC, 1, 0),
    "xi_no_prior": (KC, KC, 1, 0, 1),
    "xi_prior": (KC, KC, 1, 0, 2),
}


def _kdata(name):
    O, G, _, _, xi = KCASES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    d = {"x": (rng.standard_normal((len(KLENS), KT, KC)) * 1.5 + 0.3).astype(np.float32),
         "l": (rng.standard_normal((len(KLENS), KT, G)) * 2.0).astype(np.float32)}
    if xi == 2:
        d["prior_l"] = rng.standard_normal(KC).astype(np.float32)
        d["prior_x"] = rng.standard_normal(KC).astype(np.float32)
    return d


def _poisoned(a, ld, c0, lengths=None):
    """(B, T, C) as the slice [c0, c0 + C) of a NaN (B + 1, T, ld) buffer, frames past lengths[b] NaN too."""
    B, T, Cn = a.shape
    buf = torch.full((B + 1, T, ld), float("nan"), dtype=torch.float32, device="cuda")
    buf[:B, :, c0:c0 + Cn] = _dev(a)
    if lengths is not None:
        for b, n in enumerate(lengths):
            buf[b, n:] = float("nan")
    return buf, buf.data_ptr() + 4 * c0


class _Out:
    """Fenced fp32 (B, 2O) output and fenced (B, 2O) planes at pitch 2O + 8 (one spare row each)."""

    def __init__(self, B, W):
        self.f = Fenced((B + 1, W), torch.float32, slice(0, B))
        self.ldo = W + 8
        self.hi = Fenced((B + 1, self.ldo), torch.bfloat16, (slice(0, B), slice(0, W)))
        self.lo = Fenced((B + 1, self.ldo), torch.bfloat16, (slice(0, B), slice(0, W)))

    def ptrs(self):
        return self.f.view.data_ptr(), self.hi.view.data_ptr(), self.lo.view.data_ptr(), self.ldo

    def result(self, what):
        """(fp32, hi bits, lo bits) after the fences are checked."""
        torch.cuda.synchronize()
        for f, n in ((self.f, " out"), (self.hi, " out_hi"), (self.lo, " out_lo")):
            f.check(what + n)
        return (self.f.numpy(), self.hi.view.view(torch.int16).cpu().numpy(), self.lo.view.view(torch.int16).cpu().numpy())


def _run_kernel(lib, name, d, lengths=None, rows=None, T=None, entry="lengths"):
    """One call on utterances `rows` (default all) over T frames; lengths None: an unmasked call."""
    O, G, gdiv, unw, xi = KCASES[name]
    rows = list(range(len(KLENS))) if rows is None else rows
    T = KT if T is None else T
    B = len(rows)
    ldl = (G + 7) // 8 * 8 + 4 * (G % 2 == 0)          # a pitch that keeps 16-byte logit rows when G allows it
    lb, lp = _poisoned(d["l"][rows, :T], ldl, 0, lengths)
    xb, xp = _poisoned(d["x"][rows, :T], KC + 12, 4, lengths)
    keep = [lb, xb]
    pl = pxp = None
    if xi == 2:
        keep += [_dev(d["prior_l"]), _dev(d["prior_x"])]
        pl, pxp = keep[-2].data_ptr(), keep[-1].data_ptr()
    out = _Out(B, 2 * O)
    o, h, l, ldo = out.ptrs()
    args = (lp, ldl, G, xp, KC + 12, B, T, KC, O, gdiv, 1e-10, unw)
    if lengths is not None:
        lens = _dev(np.asarray(lengths, dtype=np.int32))
        keep.append(lens)
        rc = lib.xvb_attn_head_stats_pool_lengths(*args, pl, pxp, int(xi > 0), lens.data_ptr(), o, h, l, ldo, None)
    elif entry == "plain":
        rc = lib.xvb_attn_head_stats_pool(*args, o, h, l, ldo, None)
    else:
        rc = lib.xvb_attn_head_stats_pool_prior(*args, pl, pxp, int(xi > 0), o, h, l, ldo, None)
    assert rc == 0, name
    res = out.result(name)
    del keep
    return res


@pytest.fixture(scope="module")
def lib():
    from asv_subtools_b200 import ops  # noqa: F401  (loads and checks the library)
    from asv_subtools_b200._lib import lib as _lib
    assert torch.cuda.is_available()
    return _lib


@pytest.mark.parametrize("name", sorted(KCASES))
def test_masked_rows_equal_their_own_unmasked_call(lib, name):
    d = _kdata(name)
    got = _run_kernel(lib, name, d, lengths=KLENS)
    assert np.isfinite(got[0]).all(), name
    for b, n in enumerate(KLENS):
        solo = _run_kernel(lib, name, d, rows=[b], T=n)
        for k, what in enumerate(("out", "out_hi", "out_lo")):
            g = _bits(got[0][b:b + 1]) if k == 0 else got[k][b:b + 1]
            s = _bits(solo[0]) if k == 0 else solo[k]
            equal(g, s, "{} row {} ({} frames) {}".format(name, b, n, what))


@pytest.mark.parametrize("name", sorted(KCASES))
def test_all_lengths_T_is_the_unmasked_entry(lib, name):
    d = _kdata(name)
    got = _run_kernel(lib, name, d, lengths=[KT] * len(KLENS))
    entries = ["prior"] + (["plain"] if KCASES[name][4] == 0 else [])
    for entry in entries:
        want = _run_kernel(lib, name, d, entry=entry)
        equal(_bits(got[0]), _bits(want[0]), name + " vs " + entry)
        equal(got[1], want[1], name + " hi vs " + entry)
        equal(got[2], want[2], name + " lo vs " + entry)


def _kernel_outputs(lib):
    return {name: _run_kernel(lib, name, _kdata(name), lengths=KLENS)[0] for name in sorted(KCASES)}


def test_attn_rows_instances_are_bitwise_equal(lib, tmp_path):
    """XVB_ATTN_ROWS = 1, 2 and 4 walk each utterance's frames in the same order.  XVB_ATTN_ROWS is read once per process,
    so each instance runs in a child process, under the profiler there to name the instance that ran; the profiler is
    never started in this process, whose later files take their own profiles.  Each child's outputs must equal this
    process's (default instance) bit for bit."""
    outs = _kernel_outputs(lib)
    for rows in (1, 2, 4):
        dst = tmp_path / "rows{}.npz".format(rows)
        env = dict(os.environ, XVB_ATTN_ROWS=str(rows))
        r = subprocess.run([sys.executable, os.path.abspath(__file__), str(dst)], cwd=ROOT, env=env, capture_output=True,
                           text=True, timeout=600)
        assert r.returncode == 0, "XVB_ATTN_ROWS={} child failed:\n{}\n{}".format(rows, r.stdout[-3000:], r.stderr[-3000:])
        got = np.load(dst)
        assert "attn_head_stats_pool_kernel<{}>".format(rows) in set(got["__seen__"].tolist()), got["__seen__"]
        for name, want in outs.items():
            equal(_bits(got[name]), _bits(want), "{}: XVB_ATTN_ROWS={} vs this process".format(name, rows))


def test_kernel_refusals_return_einval_and_write_nothing(lib):
    B, T, C = 2, 8, 128
    x = torch.zeros(B + 1, T, C + 8, device="cuda")
    lens = torch.full((65536,), T, dtype=torch.int32, device="cuda")
    pri = torch.zeros(C, device="cuda")
    out = Fenced((B + 1, 4 * C), torch.float32, slice(0, B))
    hi = Fenced((B + 1, 4 * C), torch.bfloat16, slice(0, B))
    lo = Fenced((B + 1, 4 * C), torch.bfloat16, slice(0, B))
    p, o, h, l, n, q = x.data_ptr(), out.view.data_ptr(), hi.view.data_ptr(), lo.view.data_ptr(), lens.data_ptr(), pri.data_ptr()
    ld = C + 8
    f = lib.xvb_attn_head_stats_pool_lengths
    calls = {
        "NULL lengths": lambda: f(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 0, None, None, 0, None, o, h, l, 2 * C, None),
        "NULL lengths, xi": lambda: f(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 0, q, q, 1, None, o, h, l, 2 * C, None),
        "B=65536": lambda: f(p, ld, 4, p, ld, 65536, 1, 4, 4, 1, 1e-5, 0, None, None, 0, n, o, h, l, 8, None),
        "C=130": lambda: f(p, ld, 130, p, ld, B, T, 130, 130, 1, 1e-5, 0, None, None, 0, n, o, h, l, 260, None),
        "prior with unweighted": lambda: f(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 1, q, q, 1, n, o, h, l, 2 * C, None),
        "one prior array": lambda: f(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 0, q, None, 1, n, o, h, l, 2 * C, None),
        "head map past G": lambda: f(p, ld, 4, p, ld, B, T, C, C, 1, 1e-5, 0, None, None, 0, n, o, h, l, 2 * C, None),
        "ldo < 2O": lambda: f(p, ld, C, p, ld, B, T, C, C, 1, 1e-5, 0, None, None, 0, n, o, h, l, 2 * C - 4, None),
        "split_frames NULL lengths": lambda: lib.xvb_split_frames_lengths(p, B, T, C, h, l, 4 * C, 0, 0, None, None),
    }
    for what, call in calls.items():
        assert call() == EINVAL, what
    torch.cuda.synchronize()
    for fz, what in ((out, "out"), (hi, "out_hi"), (lo, "out_lo")):
        fz.check("refusals " + what)
        assert int((fz.bits[:B] != fz.sent).sum()) == 0, "a refused call wrote " + what


# ================================================================================================ staging
@pytest.mark.parametrize("C,pads", [(40, (0, 0)), (40, (2, 3)), (23, (0, 0)), (23, (1, 4))])
def test_split_frames_lengths(lib, C, pads):
    lens = [1, 7, 40, 8, 33]
    B, T = len(lens), 40
    ld = (C + 7) // 8 * 8 + 8
    Tp = pads[0] + T + pads[1]
    x = np.random.RandomState(C + pads[0]).standard_normal((B, T, C)).astype(np.float32)
    for b, n in enumerate(lens):
        x[b, n:] = np.nan
    xd = _dev(x)
    res = {}
    for masked in (False, True):
        hi = Fenced((B + 1, Tp, ld), torch.bfloat16, slice(0, B))
        lo = Fenced((B + 1, Tp, ld), torch.bfloat16, slice(0, B))
        keep = _dev(np.asarray(lens, np.int32))
        args = (xd.data_ptr(), B, T, C, hi.view.data_ptr(), lo.view.data_ptr(), ld, pads[0], pads[1])
        rc = lib.xvb_split_frames_lengths(*args, keep.data_ptr(), None) if masked else lib.xvb_split_frames(*args, None)
        assert rc == 0
        torch.cuda.synchronize()
        hi.check("hi")
        lo.check("lo")
        res[masked] = (hi.view.view(torch.int16).cpu().numpy(), lo.view.view(torch.int16).cpu().numpy())
    for k in range(2):
        for b, n in enumerate(lens):
            inside = slice(pads[0], pads[0] + n)
            equal(res[True][k][b, inside], res[False][k][b, inside], "plane {} utterance {} inside".format(k, b))
            past = np.concatenate([res[True][k][b, :pads[0]], res[True][k][b, pads[0] + n:]])
            assert (past == 0).all(), "plane {} utterance {}: nonzero past its end".format(k, b)


# ================================================================================================ extractors
_MODEL_CACHE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    """The sixteen models built here, their extractors and the activations they cached go when this file is done, so
    the files that run after it in the same process start from the device state they would have without it."""
    yield
    _MODEL_CACHE.clear()
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _model(name, pos):
    """(model on the GPU, float32 state_dict, oracle forward of one (1, F, T) utterance)."""
    if (name, pos) not in _MODEL_CACHE:
        if name == "ftdnn":
            from asv_subtools_b200.model.factored_xvector import Xvector
            sd = onn.make_state_dict(onn.factored_xvector_spec(40), 401)
            m = Xvector(40, 10, training=False, extracted_embedding=pos)
            fwd = lambda v: onn.factored_xvector_forward(sd, v, pos)  # noqa: E731
        else:
            from asv_subtools_b200.model.snowdar_xvector import Xvector
            pooling, pp, seed = POOLING_CASES[name]
            sd = onn.make_state_dict(onn.snowdar_xvector_spec(40, pooling=pooling, pooling_params=pp), seed)
            m = Xvector(40, 10, training=False, extracted_embedding=pos, pooling=pooling, pooling_params=pp)
            fwd = lambda v: onn.snowdar_xvector_forward(sd, v, pos, pooling=pooling, pooling_params=pp)  # noqa: E731
        m.load_state_dict(sd, strict=True)
        _MODEL_CACHE[(name, pos)] = (m.cuda().eval(), sd, fwd)
    return _MODEL_CACHE[(name, pos)]


def _mixed_lengths(seed, B=64, lo=1, hi=300):
    rng = np.random.RandomState(seed)
    lens = rng.randint(lo, hi + 1, B)
    lens[:4] = [1, 2, 3, hi]
    rng.shuffle(lens)
    return [int(v) for v in lens]


def _padded(rows, T, dim=40, fill=0.0):
    x = np.full((len(rows), T, dim), fill, dtype=np.float32)
    for i, r in enumerate(rows):
        x[i, :r.shape[0]] = r
    return torch.from_numpy(x).cuda()


def test_extractors_take_lengths():
    from asv_subtools_b200.model.factored_xvector import FtdnnExtractor
    from asv_subtools_b200.nnet.framework import AttentionPoolingExtractor
    for name in MODELS:
        ex = _model(name, "far")[0].extractor()
        assert isinstance(ex, FtdnnExtractor if name == "ftdnn" else AttentionPoolingExtractor) and ex.TAKES_LENGTHS, name


@pytest.mark.parametrize("pos", ["far", "near"])
@pytest.mark.parametrize("name", MODELS)
def test_mixed_batch_rows_equal_solo_extraction(name, pos):
    m = _model(name, pos)[0]
    ex = m.extractor()
    seed = MODELS.index(name) * 2 + (pos == "near")
    lens = _mixed_lengths(900 + seed)
    x = torch.from_numpy(onn.synthetic_feats(64, 300, 40, 1900 + seed)).cuda()
    got = ex.extract(x, lens).cpu().numpy()
    worst, same = 0.0, True
    for b, n in enumerate(lens):
        solo = ex.extract(x[b:b + 1, :n].contiguous()).cpu().numpy()[0]
        r = rel(got[b], solo)
        # the F-TDNN's solo call pools in layer10's fused epilogue, a masked batch with the standalone pooling: at one
        # frame the two differ by up to 1.3e-5 of the largest component (measured on the H100); the attention models run
        # the same kernels either way
        assert r <= (2e-5 if name == "ftdnn" and n == 1 else 1e-5), (name, pos, b, n, r)
        assert cos(got[b], solo) >= 1 - 1e-8, (name, pos, b, n)
        worst, same = max(worst, r), same and np.array_equal(_bits(got[b]), _bits(solo))
    WORST[(name, pos)] = (worst, same)


@pytest.mark.parametrize("pos", ["far", "near"])
@pytest.mark.parametrize("name", MODELS)
def test_mixed_batch_matches_the_oracle(name, pos):
    m, _, fwd = _model(name, pos)
    # no 2..7-frame rows here: there the attention poolings' weighted variance (sum alpha x^2 - mean^2) cancels, and the
    # unmasked path and the fp32 oracle differ by up to 2e-4 already; the masked rows equal the unmasked ones bit for bit
    lens = [300, 1, 57, 9, 199, 8]
    feats = onn.synthetic_feats(len(lens), 300, 40, 4321)
    got = m.extract_embedding_batch(feats, lengths=lens).cpu().numpy()
    for b, n in enumerate(lens):
        want = onn.extract_embedding(fwd, feats[b, :n]).numpy()
        assert rel(got[b], want) < EMB_TOL, (name, pos, b, n, rel(got[b], want))


@pytest.mark.parametrize("name", MODELS)
def test_goldens_in_one_mixed_batch(golden, name):
    if name == "ftdnn":
        g, rows, key = golden("ftdnn"), list(onn.synthetic_feats(2, 90, 40, 1401)), "{pos}"
    else:
        seed = POOLING_CASES[name][2]
        g, rows, key = golden("snowdar"), list(onn.synthetic_feats(3, 120, 40, seed + 1000)), name + "_{pos}"
    fill = [onn.synthetic_feats(1, t, 40, 7000 + t)[0] for t in (5, 300, 64)]
    batch, where = [], []
    for i, r in enumerate(rows):
        batch.append(fill[i % 3])
        where.append(len(batch))
        batch.append(r)
    for pos in ("far", "near"):
        m = _model(name, pos)[0]
        got = m.extract_embedding_batch(_padded(batch, 300), lengths=[r.shape[0] for r in batch]).cpu().numpy()
        want = g[key.format(pos=pos)]
        for j, i in enumerate(where):
            assert rel(got[i], want[j]) < EMB_TOL and cos(got[i], want[j]) >= 1 - 1e-6, (name, pos, j)


@pytest.mark.parametrize("name", MODELS)
def test_all_lengths_T_is_the_unmasked_call(name):
    for pos in ("far", "near"):
        m = _model(name, pos)[0]
        ex = m.extractor()
        for B, T in ((1, 1), (3, 37), (16, 200)):
            x = torch.from_numpy(onn.synthetic_feats(B, T, 40, 11 * B + T)).cuda()
            a = ex.extract(x)
            assert torch.equal(ex.extract(x, [T] * B), a), (name, pos, B, T)
            assert torch.equal(m.extract_embedding_batch(x, lengths=np.full(B, T)), a), (name, pos, B, T)


@pytest.mark.parametrize("name", MODELS)
def test_pad_content_is_ignored(name):
    ex = _model(name, "near")[0].extractor()
    lens = _mixed_lengths(77 + MODELS.index(name), B=16, hi=150)
    rows = [r[:n] for r, n in zip(onn.synthetic_feats(16, 150, 40, 177), lens)]
    ref = ex.extract(_padded(rows, 150), lens)
    for fill in (float("nan"), 1e30, -1e30):
        assert torch.equal(ex.extract(_padded(rows, 150, fill=fill), lens), ref), (name, fill)


@pytest.mark.parametrize("name", ["mha_share", "xi_dist", "ftdnn"])
def test_bad_lengths_raise(name):
    ex = _model(name, "far")[0].extractor()
    x = torch.zeros(3, 20, 40, device="cuda")
    for bad, at in (([20, 0, 20], 1), ([20, -3, 20], 1), ([20, 20, 21], 2)):
        with pytest.raises(ValueError, match=r"lengths\[{}\]".format(at)):
            ex.extract(x, bad)
    with pytest.raises(ValueError):
        ex.extract(x, [20, 20])
    assert torch.isfinite(ex.extract(x, [20, 1, 7])).all()


def test_lde_still_refuses_lengths():
    from asv_subtools_b200.model.snowdar_xvector import Xvector
    m = Xvector(40, 10, training=False, extracted_embedding="far", pooling="lde")
    m.cuda().eval()
    ex = m.extractor()
    assert ex.TAKES_LENGTHS is False
    with pytest.raises(NotImplementedError):
        ex.extract(torch.zeros(2, 50, 40, device="cuda"), [50, 20])


def test_report_masked_vs_solo():
    """The largest |masked - solo| / max |solo| per model and position, and whether every row was bit-identical (-s)."""
    for (name, pos), (worst, same) in sorted(WORST.items()):
        print("{:10s} {:4s} largest difference {:.3g}  rows bit-identical: {}".format(name, pos, worst, same))


# ================================================================================================ CLI
def _write_ark(path, feats):
    from asv_subtools_b200 import kaldi_io
    with open(path, "wb") as f:
        for k, v in feats.items():
            kaldi_io.write_mat(f, v, key=k)


@pytest.mark.parametrize("name", ["mha_share", "xi_dist", "ftdnn"])
def test_pipeline_mixed_lengths(tmp_path, name):
    from asv_subtools_b200 import kaldi_io
    _, sd, fwd = _model(name, "far")
    rng = np.random.RandomState(2027)
    lens = [1, 2, 1200] + [int(v) for v in rng.randint(1, 1201, 37)]
    feats = {"u{:02d}".format(i): onn.synthetic_feats(1, t, 40, 6000 + i)[0] for i, t in enumerate(lens)}
    ark = str(tmp_path / "feats.ark")
    _write_ark(ark, feats)
    torch.save(sd, str(tmp_path / "final.params"))
    if name == "ftdnn":
        bp, creation = "factored_xvector.py", "Xvector(40,10,training=False,extracted_embedding='far')"
    else:
        pooling, pp, _ = POOLING_CASES[name]
        bp = "snowdar_xvector.py"
        creation = "Xvector(40,10,training=False,extracted_embedding='far',pooling={!r},pooling_params={!r})".format(pooling, pp)
    runs = {}
    for run, flag in (("mixed", ["--mixed-lengths"]), ("plain", [])):
        out = str(tmp_path / (run + ".ark"))
        r = subprocess.run([sys.executable, "-m", "asv_subtools_b200.pipeline.extract_embeddings"] + flag +
                           ["--model-blueprint", os.path.join(ROOT, "asv_subtools_b200", "model", bp), "--model-creation",
                            creation, "--batch-size", "16", str(tmp_path / "final.params"), "ark:" + ark, "ark:" + out],
                           capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT), cwd=ROOT, timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        runs[run] = (dict(kaldi_io.read_vec_flt_ark(out)), r.stderr)
    got, err = runs["mixed"]
    assert sorted(got) == sorted(feats) and "masked batches" in err, err[-2000:]
    for i, (k, v) in enumerate(sorted(feats.items())):
        assert rel(got[k], runs["plain"][0][k]) < 1e-5, (name, k)
        n = v.shape[0]
        # against the oracle: not the 2..7-frame rows (see test_mixed_batch_matches_the_oracle), and for the F-TDNN (slow
        # on the CPU) every fourth utterance
        if (n == 1 or n >= 8) and (name != "ftdnn" or i % 4 == 0):
            assert rel(got[k], onn.extract_embedding(fwd, v).numpy()) < EMB_TOL, (name, k)


if __name__ == "__main__":
    from asv_subtools_b200._lib import lib as _lib
    outs = {}

    def run():
        outs.update(_kernel_outputs(_lib))

    seen = profiled(run, _ATTN_KERNEL)
    np.savez(sys.argv[1], __seen__=np.array(sorted(seen)), **outs)
