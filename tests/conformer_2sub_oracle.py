"""torch-CPU restatement of the reference's TransformerXvector with input_layer="conv2d2" (SVConv2dSubsampling2,
pytorch/libs/nnet/transformer/subsampling.py:365-415), and the golden cases of tests/golden/make_golden_conformer_2sub.py.

The 2x subsampling differs from Conv2dSubsampling4 only in its two convolutions: Conv2d(1, C, 3, stride (2, 1)) + ReLU,
then Conv2d(C, C, 3, 1) + ReLU, so T' = (T - 1) // 2 - 2 and F'' = F - 4; the Linear, the positional encoding and
everything after are the same.  chunk_forward runs conformer_oracle.chunk_forward with those two strides."""
import copy
import types

import torch
import torch.nn.functional as F

import conformer_oracle as co

MIN_FRAMES = 7

LAUNCHER_2SUB = copy.deepcopy(co.LAUNCHER)
LAUNCHER_2SUB["transformer_params"]["input_layer"] = "conv2d2"

# abs_pos, softmax, a BatchNorm conv module, relu, transform_out with BatchNorm and fc1
SMALL_2SUB = copy.deepcopy(co.SMALL)
SMALL_2SUB["transformer_params"]["input_layer"] = "conv2d2"

# name -> (kwargs, feat_dim, frame counts, positions, state_dict seed, feature seed), as conformer_oracle.CASES
CASES = {
    "launcher2": (LAUNCHER_2SUB, 80, (300, 37, 7, 650, 899), ("near", "near_affine"), 21, 800),
    "small2": (SMALL_2SUB, 23, (150, 8), ("far", "near_affine", "near"), 22, 900),
}


def out_frames(t):
    """T' of SVConv2dSubsampling2."""
    return (t - 1) // 2 - 2


def head(sd, x):
    """SVConv2dSubsampling2 up to its Linear: x (B, T, F) -> (B, T', C * F'') with the reference's c * F'' + f columns."""
    p = "transformer.embed."
    h = F.relu(F.conv2d(x.unsqueeze(1), sd[p + "conv.0.weight"], sd[p + "conv.0.bias"], stride=(2, 1)))
    h = F.relu(F.conv2d(h, sd[p + "conv.2.weight"], sd[p + "conv.2.bias"], stride=1))
    b, c, t, f = h.size()
    return h.transpose(1, 2).contiguous().view(b, t, c * f)


def _functional_2sub():
    """torch.nn.functional with conv2d's first call at stride (2, 1) and its second at stride 1: the two subsampling
    convolutions of conformer_oracle.chunk_forward (its only conv2d calls) become SVConv2dSubsampling2's."""
    calls = []

    def conv2d(x, w, b=None, stride=1, **kw):
        calls.append(None)
        return F.conv2d(x, w, b, stride=(2, 1) if len(calls) == 1 else 1, **kw)

    ns = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith("__")})
    ns.conv2d = conv2d
    return ns


def chunk_forward(sd, x, cfg, position):
    """One chunk of the 2Sub model: x (B, T, F) fp32 -> (B, embd_dim)."""
    saved = co.F
    co.F = _functional_2sub()
    try:
        return co.chunk_forward(sd, x, cfg, position)
    finally:
        co.F = saved


def extract(sd, feats, cfg, position):
    """feats (T, F) -> embedding under the maxChunk = 300 chunk rule (conformer_oracle.extract)."""
    x = torch.as_tensor(feats).unsqueeze(0)
    lengths, offsets = co.chunk_plan(x.shape[1])
    acc = 0.
    with torch.no_grad():
        for n, o in zip(lengths[:-1], offsets[:-1]):
            acc = acc + n * chunk_forward(sd, x[:, o:o + n], cfg, position)
        last = chunk_forward(sd, x[:, offsets[-1]:], cfg, position)
    return ((acc + lengths[-1] * last) / x.shape[1])[0]
