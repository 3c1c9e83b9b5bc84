"""Masked batches of the attention-pooling, xi-vector and F-TDNN x-vectors, checked without a GPU.

  * The definition: a float64 masked-batch forward -- every frame layer's output zeroed past each utterance's end, the
    attention logits set to -inf there (the xi-vector's softmax then runs over lengths[b] frames + the prior), the
    statistics over each utterance's own frames -- equals the oracle's forward of each utterance alone, for every
    attention pooling of tests/golden/make_golden_snowdar.py (not LDE) and for the F-TDNN, at lengths 1..300.  This is
    what the GPU path computes in fp32.
  * The ctypes prototypes of xvb_attn_head_stats_pool_lengths and xvb_split_frames_lengths match include/xvb200.h.
  * nvcc builds the two changed sources for sm_90a, and the three attn_head_stats_pool_kernel instances keep no stack
    and no spills."""
import ctypes as C
import importlib.util
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nnet as onn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LENGTHS = [1, 2, 7, 8, 9, 31, 32, 33, 150, 300]
T = 300


def _pooling_cases():
    spec = importlib.util.spec_from_file_location("make_golden_snowdar", os.path.join(ROOT, "tests", "golden",
                                                                                      "make_golden_snowdar.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return {k: v for k, v in mod.POOLING_CASES.items() if v[0] != "lde"}


POOLING_CASES = _pooling_cases()


def _f64(sd):
    return {k: v.double() for k, v in sd.items()}


def _mask(lengths, t):
    """(B, 1, T) float64: 1 on each utterance's own frames, 0 past its end."""
    return (torch.arange(t)[None, :] < torch.tensor(lengths)[:, None]).double().unsqueeze(1)


def _padded(feats, lengths):
    """(B, T, F) float32 frames -> (B, F, T) float64 with zeros past each end."""
    return torch.from_numpy(feats).double().transpose(1, 2) * _mask(lengths, feats.shape[1])


# ------------------------------------------------------------------------------------------------ masked references
def _masked_attention(x, sd, pooling, params, m):
    """The attention poolings of oracle.snowdar_pooling over a masked batch: logits -inf past each end, so the softmax
    over T is each utterance's own."""
    p = dict(onn.ATTENTION_DEFAULTS)
    p.update(params)
    if pooling == "attentive":
        heads, split, share, bias, temp, glob = 1, True, True, True, False, False
    elif pooling == "multi-head":
        heads, split, share, bias, temp, glob = p["num_head"], True, p["share"], False, p["temperature"], False
    else:
        heads, split, share, bias, temp, glob = p["num_head"], False, p["share"], True, True, True
    first, last, _ = onn.attention_layout(x.shape[1], heads, split, share, p["affine_layers"], p["hidden_size"], bias)
    pre, ctx = "stats.attention", list(p["context"])
    h = x
    if first is not None:
        h = F.relu(onn.tdnn_affine(h, sd[pre + ".first_affine.weight"], sd.get(pre + ".first_affine.bias"), ctx, first[2])) * m
    logits = onn.tdnn_affine(h, sd[pre + ".last_affine.weight"], sd.get(pre + ".last_affine.bias"), ctx, last[2])
    if heads > 1 and temp:
        b, _, t = logits.shape
        tt = sd[pre + ".t"] if p["fixed"] else 1 + sd[pre + ".t"] ** 2
        logits = (logits.reshape(b, heads, -1, t) / tt).reshape(b, -1, t)
    alpha = torch.softmax(logits.masked_fill(m == 0, float("-inf")), dim=2)
    return onn.attention_pooling(x, alpha, heads, glob)


def _masked_xi(x, sd, stddev, m):
    """xi_vector_pooling over a masked batch: frame log-precisions -inf past each end (weight 0 in the softmax over the
    utterance's own frames and the prior)."""
    h = onn.relu_bn_tdnn_layer(x, sd, "stats.lin1_relu_bn", [0]) * m
    logprec = 2.0 * torch.log(F.softplus(onn.tdnn_affine(h, sd["stats.lin2.weight"], sd["stats.lin2.bias"], [0]), beta=1,
                                         threshold=20))
    logprec = logprec.masked_fill(m == 0, float("-inf"))
    b = x.shape[0]
    pl = sd["stats.prior_logprec"].repeat(b, 1).unsqueeze(2)
    pm = sd["stats.prior_mean"].repeat(b, 1).unsqueeze(2)
    w = torch.softmax(torch.cat((logprec, pl), 2), dim=2)
    xx = torch.cat((x, pm), 2)
    phi = torch.sum(xx * w, dim=2)
    if not stddev:
        return phi.unsqueeze(2)
    sigma = torch.sqrt(torch.clamp(torch.sum(xx.pow(2) * w, dim=2) - phi ** 2, min=1.0e-10))
    return torch.cat((phi, sigma), dim=1).unsqueeze(2)


def _masked_stats(x, m, eps=1.0e-10):
    n = m.sum(dim=2, keepdim=True)
    mean = (x * m).sum(dim=2, keepdim=True) / n
    var = (((x - mean) ** 2) * m).sum(dim=2, keepdim=True) / n
    return torch.cat((mean, torch.sqrt(var.clamp(min=eps))), dim=1)


def masked_snowdar_forward(sd, x, lengths, pos, pooling, params):
    """snowdar_xvector_forward of a masked batch x (B, F, T), zeros past each end."""
    m = _mask(lengths, x.shape[2])
    for name, ctx in onn.snowdar_layers(False):
        x = onn.relu_bn_tdnn_layer(x, sd, name, ctx) * m
    if pooling.startswith("xi-"):
        x = _masked_xi(x, sd, pooling == "xi-postdist-softplus2", m)
    else:
        x = _masked_attention(x, sd, pooling, params, m)
    if pos == "far":
        return onn.tdnn_affine(x, sd["tdnn6.affine.weight"], sd["tdnn6.affine.bias"], [0])
    x = onn.relu_bn_tdnn_layer(x, sd, "tdnn6", [0])
    return onn.relu_bn_tdnn_layer(x, sd, "tdnn7", [0])


def masked_ftdnn_forward(sd, x, lengths, pos):
    """factored_xvector_forward of a masked batch: each FTdnnBlock's factor output is zeroed past the end too, since the
    affine after it reads frames t .. t + c."""
    m = _mask(lengths, x.shape[2])

    def blk(i, v):
        _, _, c, bypass = onn.FTDNN_BLOCKS[i]
        p = "layer{:02d}".format(i)
        c1, c2 = ([-c, 0], [0, c]) if c > 0 else ([0], [0])
        out = onn.tdnn_affine(v, sd[p + ".factor.weight"], None, c1) * m
        out = onn.tdnn_affine(out, sd[p + ".affine.weight"], sd[p + ".affine.bias"], c2)
        out = onn.batchnorm_eval(F.relu(out), sd, p + ".bn") * m
        return out + bypass * v if bypass != 0 else out

    x1 = onn.relu_bn_tdnn_layer(x, sd, "layer01", [-2, -1, 0, 1, 2]) * m
    x2 = blk(2, x1)
    x3 = blk(3, x2)
    x4 = blk(4, x3)
    x5 = blk(5, x3)
    x6 = blk(6, x5)
    x7 = blk(7, torch.cat((x2, x4), 1))
    x8 = blk(8, x7)
    x9 = blk(9, torch.cat((x4, x6, x8), 1))
    v = _masked_stats(onn.relu_bn_tdnn_layer(x9, sd, "layer10", [0]) * m, m)
    if pos == "far":
        return onn.tdnn_affine(v, sd["embedding1.affine.weight"], sd["embedding1.affine.bias"], [0])
    v = onn.relu_bn_tdnn_layer(v, sd, "embedding1", [0])
    return onn.tdnn_affine(v, sd["embedding2.affine.weight"], sd["embedding2.affine.bias"], [0])


def _rel(a, b):
    return float((a - b).abs().max() / b.abs().max())


@pytest.mark.parametrize("name", sorted(POOLING_CASES))
def test_masked_snowdar_reference_equals_solo_oracle(name):
    pooling, params, seed = POOLING_CASES[name]
    sd = _f64(onn.make_state_dict(onn.snowdar_xvector_spec(40, pooling=pooling, pooling_params=params), seed))
    lengths = list(np.random.RandomState(seed).permutation(LENGTHS))
    feats = onn.synthetic_feats(len(lengths), T, 40, seed + 2000)
    x = _padded(feats, lengths)
    with torch.no_grad():
        for pos in ("far", "near"):
            got = masked_snowdar_forward(sd, x, lengths, pos, pooling, params).squeeze(2)
            for b, n in enumerate(lengths):
                want = onn.snowdar_xvector_forward(sd, x[b:b + 1, :, :n], pos, pooling=pooling, pooling_params=params)
                assert _rel(got[b], want[0, :, 0]) < 1e-10, (name, pos, b, n)


def test_masked_ftdnn_reference_equals_solo_oracle():
    sd = _f64(onn.make_state_dict(onn.factored_xvector_spec(40), 401))
    lengths = [1, 9, 33, 300, 8, 150]
    feats = onn.synthetic_feats(len(lengths), T, 40, 2401)
    x = _padded(feats, lengths)
    with torch.no_grad():
        for pos in ("far", "near"):
            got = masked_ftdnn_forward(sd, x, lengths, pos).squeeze(2)
            for b, n in enumerate(lengths):
                want = onn.factored_xvector_forward(sd, x[b:b + 1, :, :n], pos)
                assert _rel(got[b], want[0, :, 0]) < 1e-10, (pos, b, n)


# ------------------------------------------------------------------------------------------------ C ABI
_CTYPES = {"const float*": C.c_void_p, "float*": C.c_void_p, "const int*": C.c_void_p, "uint16_t*": C.c_void_p,
           "void*": C.c_void_p, "int64_t": C.c_int64, "int": C.c_int, "float": C.c_float}


def _header_prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "xvb200.h")).read(), flags=re.S)
    m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)\s*;", text)
    assert m, name
    args = []
    for a in m.group(1).split(","):
        a = " ".join(a.split())
        typ = re.sub(r"\s*\b\w+$", "", a).replace(" *", "*")
        args.append(_CTYPES[typ])
    return args


@pytest.mark.parametrize("name", ["xvb_attn_head_stats_pool_lengths", "xvb_split_frames_lengths"])
def test_ctypes_prototypes_match_the_header(name):
    from asv_subtools_b200 import _lib
    res, args = _lib.SIGNATURES[name]
    assert res is C.c_int
    assert args == _header_prototype(name), name
    # the lengths entry is the _prior entry with the lengths pointer before the outputs
    if name == "xvb_attn_head_stats_pool_lengths":
        prior = _lib.SIGNATURES["xvb_attn_head_stats_pool_prior"][1]
        assert args == prior[:15] + [C.c_void_p] + prior[15:]
    else:
        assert args == _lib.SIGNATURES["xvb_split_frames"][1][:-1] + [C.c_void_p, C.c_void_p]


NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.mark.skipif(not (os.path.exists(NVCC) or shutil.which("nvcc")), reason="needs nvcc")
def test_changed_sources_build_for_sm90a_without_spills(tmp_path):
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    csrc = os.path.join(ROOT, "asv_subtools_b200", "csrc")
    flags = ["-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a"]
    for src in ("core.cu", "ecapa.cu"):
        obj = str(tmp_path / (src + ".o"))
        r = subprocess.run([nvcc] + flags + ["-Xptxas", "-v", "-c", os.path.join(csrc, src), "-o", obj], capture_output=True,
                           text=True, timeout=1200)
        assert r.returncode == 0, r.stderr[-3000:]
        syms = subprocess.run(["nm", "-g", "--defined-only", obj], capture_output=True, text=True).stdout
        want = "xvb_split_frames_lengths" if src == "core.cu" else "xvb_attn_head_stats_pool_lengths"
        assert re.search(r"\bT\s+" + want + r"\b", syms), want
        if src == "ecapa.cu":
            seen = 0
            for block in re.split(r"(?=ptxas info\s+: Compiling entry function)", r.stderr):
                if "attn_head_stats_pool_kernel" not in block.split("\n")[0]:
                    continue
                seen += 1
                assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, block
            assert seen == 3, r.stderr[-3000:]
