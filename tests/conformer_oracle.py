"""torch-CPU restatement of the reference's TransformerXvector with the Conformer encoder at extraction
(pytorch/model/transformer_xvector.py:321-346 over pytorch/libs/nnet/transformer/), the golden cases of
tests/golden/make_golden_conformer.py and the seeded state_dict rule both sides share.

Written from the reference's arithmetic, in its operation order, for the options the native blueprint supports: conv2d
subsampling, abs_pos / rot_pos (rotary_value either way) / no_pos, softmax / softmax_plus, the convolution module with
LayerNorm or BatchNorm, swish or relu, transform_out with LayerNorm or BatchNorm, AttentiveStatsPool, fc1 on or off,
positions far / near_affine / near, and the maxChunk = 300 chunk rule of for_extract_embedding."""
import copy
import math
import zlib

import numpy as np
import torch
import torch.nn.functional as F

MAX_CHUNK = 300

_FC1_LAUNCHER = {"nonlinearity": 'relu', "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                 "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}}
_FC2_LAUNCHER = {"nonlinearity": '', "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                 "ln_replace": True, "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}

# runTransformerXvector.py:220-286 without training / extracted_embedding
LAUNCHER = dict(
    wenet_transfer=True, embd_dim=256, transformer_type="conformer",
    transformer_params={"attention_dim": 256, "attention_heads": 4, "num_blocks": 6, "combiner_type": "norm",
                        "aux_layer_period": 2, "aux_layer_start": 3, "dropout_rate": 0.1, "layer_dropout": 0.,
                        "linear_units": 2048, "positional_dropout_rate": 0.1, "attention_dropout_rate": 0.1,
                        "attention_norm_args": {"norm_method": "softmax_plus", "train_len": 300},
                        "input_layer": "conv2d", "cnn_module_kernel": 15, "pos_enc_type": "rot_pos", "convfnn_blocks": 0},
    pooling="ecpa-attentive", pooling_params={"hidden_size": 128, "time_attention": False, "stddev": True},
    fc1=False, fc1_params=_FC1_LAUNCHER, fc2_params=_FC2_LAUNCHER,
    margin_loss=True, margin_loss_params={"method": "aam", "m": 0.2, "feature_normalize": True, "s": 30,
                                          "mhe_loss": False, "mhe_w": 0.01},
    use_step=False)

# the other options: abs_pos, softmax, BatchNorm in the conv module, relu, transform_out with BatchNorm, fc1 with a
# LayerNorm without affine
SMALL = dict(
    embd_dim=128, transformer_type="conformer",
    transformer_params={"attention_dim": 128, "attention_heads": 2, "num_blocks": 2, "linear_units": 512,
                        "pos_enc_type": "abs_pos", "attention_norm_args": {"norm_method": "softmax"},
                        "cnn_module_norm": "batch_norm", "activation_type": "relu", "input_layer": "conv2d"},
    tansformer_out={"out_dim": 384, "ln_replace": False},
    pooling="ecpa-attentive", pooling_params={"hidden_size": 64},
    fc1=True, fc1_params=_FC1_LAUNCHER, fc2_params=_FC2_LAUNCHER)

# rot_pos without the rotary value, one block
ROTV = copy.deepcopy(LAUNCHER)
ROTV["transformer_params"].update({"num_blocks": 1, "rotary_value": False})

# name -> (kwargs, feat_dim, frame counts, positions, state_dict seed, feature seed)
CASES = {
    "launcher": (LAUNCHER, 80, (300, 37, 7, 650, 899), ("near", "near_affine"), 11, 500),
    "small": (SMALL, 23, (150, 8), ("far", "near_affine", "near"), 12, 600),
    "rotv": (ROTV, 80, (300, 29999), ("near",), 13, 700),
}


def creation(kwargs, inputs_dim, position):
    """Creation string of TransformerXvector(inputs_dim, 10, training=False, extracted_embedding=position, **kwargs)."""
    args = dict(training=False, extracted_embedding=position, **kwargs)
    return "TransformerXvector({},10,{})".format(inputs_dim, ",".join("{}={!r}".format(k, v) for k, v in args.items()))


def seeded_state_dict(keys, seed):
    """Deterministic weights for a "key:shape" list, independent of the key order: norm gains 1 + 0.1 N(0,1), every
    1-D bias 0.1 N(0,1), running_var U(0.5, 1.5), train_len = ln U(150, 600), weights N(0,1) / sqrt(fan_in)."""
    sd = {}
    for entry in keys:
        key, shape = str(entry).split(":")
        shape = tuple(int(d) for d in shape.split(",")) if shape else ()
        g = torch.Generator().manual_seed(seed * 1000003 + zlib.crc32(key.encode()))
        if key.endswith("num_batches_tracked"):
            sd[key] = torch.tensor(0, dtype=torch.long)
        elif key.endswith("running_var"):
            sd[key] = 0.5 + torch.rand(shape, generator=g)
        elif key.endswith("train_len"):
            sd[key] = torch.log(150. + 450. * torch.rand(shape, generator=g))
        elif len(shape) == 1 and key.endswith(".weight"):
            sd[key] = 1. + 0.1 * torch.randn(shape, generator=g)
        elif len(shape) == 1:
            sd[key] = 0.1 * torch.randn(shape, generator=g)
        else:
            sd[key] = torch.randn(shape, generator=g) / math.sqrt(float(np.prod(shape[1:])))
    return sd


def _assign(defaults, given, unknown=False):
    out = copy.deepcopy(defaults)
    for k, v in (given or {}).items():
        if k in out:
            out[k] = _assign(out[k], v, unknown) if isinstance(out[k], dict) and isinstance(v, dict) else v
        elif unknown:
            out[k] = v
    return out


def config(kwargs):
    """The option values the forward depends on (defaults of transformer_xvector.py:98-149 and encoder.py:536-581)."""
    tp = _assign({"attention_dim": 256, "attention_heads": 4, "num_blocks": 6, "linear_units": 2048,
                  "attention_norm_args": {"norm_method": "softmax", "train_len": 300.}, "pos_enc_type": "abs_pos",
                  "cnn_module_kernel": 15, "cnn_module_norm": "layer_norm", "rotary_value": True,
                  "activation_type": "swish"}, kwargs.get("transformer_params", {}), unknown=True)
    to = _assign({"out_dim": 1536, "bn": True, "ln_replace": True}, kwargs.get("tansformer_out", {}))
    fc = {"nonlinearity": 'relu', "bn": True, "ln_replace": True, "bn_params": {"affine": True}}
    return dict(tp=tp, to=to, fc1=kwargs.get("fc1", False), fc1_params=_assign(fc, kwargs.get("fc1_params", {})),
                fc2_params=_assign(fc, kwargs.get("fc2_params", {})))


def _act(x, name):
    return F.silu(x) if name == "swish" else F.relu(x)


def _ln(x, sd, prefix, dim=-1):
    w, b = sd.get(prefix + ".weight"), sd.get(prefix + ".bias")
    if dim == -1:
        return F.layer_norm(x, (x.shape[-1],), w, b, 1e-5)
    return F.layer_norm(x.transpose(1, -1), (x.shape[1],), w, b, 1e-5).transpose(1, -1)


def _bn(x, sd, prefix):
    return F.batch_norm(x, sd[prefix + ".running_mean"], sd[prefix + ".running_var"], sd.get(prefix + ".weight"),
                        sd.get(prefix + ".bias"), False, 0.0, 1e-5)


def _sin_table(dim, max_len=5000):
    pe = torch.zeros(max_len, dim)
    position = torch.arange(0, max_len, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def rope_table(dk, max_len=5000):
    """RoPositionalEncoding.pe (embedding.py:162-177): (max_len, dk) = [sin | cos]."""
    abs_rope = _sin_table(dk, max_len)
    freq = torch.zeros_like(abs_rope)
    freq[:, 0:dk // 2] = abs_rope[:, 0::2]
    freq[:, dk // 2:] = abs_rope[:, 1::2]
    return freq


def _rotary(x, pos):
    sin, cos = pos.chunk(2, dim=-1)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack([x1 * cos - x2 * sin, x2 * cos + x1 * sin], dim=-1).flatten(-2, -1)


def _tdnn_layer(x, sd, prefix, params, affine_only=False):
    """ReluBatchNormTdnnLayer on (B, C, 1 or T): affine [-> activation -> LayerNorm / BatchNorm] (components.py:410-431)."""
    x = F.conv1d(x, sd[prefix + ".affine.weight"], sd.get(prefix + ".affine.bias"))
    if affine_only:
        return x
    if params["nonlinearity"] == "relu":
        x = F.relu(x)
    elif params["nonlinearity"] == "swish":
        x = F.silu(x)
    if params["bn"]:
        x = _ln(x, sd, prefix + ".batchnorm", dim=1) if params["ln_replace"] else _bn(x, sd, prefix + ".batchnorm")
    return x


def chunk_forward(sd, x, cfg, position):
    """One chunk: x (B, T, F) fp32 -> (B, embd_dim), extract_embedding's body (transformer_xvector.py:322-346)."""
    tp = cfg["tp"]
    D, H = tp["attention_dim"], tp["attention_heads"]
    dk = D // H
    p = "transformer."
    # Conv2dSubsampling4 (subsampling.py:132-141) + positional encoding
    h = F.relu(F.conv2d(x.unsqueeze(1), sd[p + "embed.conv.0.weight"], sd[p + "embed.conv.0.bias"], stride=2))
    h = F.relu(F.conv2d(h, sd[p + "embed.conv.2.weight"], sd[p + "embed.conv.2.bias"], stride=2))
    b, c, t, f = h.size()
    h = F.linear(h.transpose(1, 2).contiguous().view(b, t, c * f), sd[p + "embed.out.0.weight"], sd[p + "embed.out.0.bias"])
    pos = tp["pos_enc_type"]
    rope = None
    if pos == "abs_pos":
        h = h * math.sqrt(D) + _sin_table(D)[:t].to(h.device).unsqueeze(0)
    elif pos == "rot_pos":
        h = h * math.sqrt(D)
        rope = rope_table(dk)[:t].to(h.device).unsqueeze(0)
    norm_method = tp["attention_norm_args"]["norm_method"]
    act = tp["activation_type"]
    for i in range(tp["num_blocks"]):
        q = "{}encoders.{}.".format(p, i)

        def ffn(z, name):
            z = F.linear(z, sd[q + name + ".w_1.weight"], sd[q + name + ".w_1.bias"])
            return F.linear(_act(z, act), sd[q + name + ".w_2.weight"], sd[q + name + ".w_2.bias"])

        h = h + 0.5 * ffn(_ln(h, sd, q + "norm_ff_macaron"), "feed_forward_macaron")
        z = _ln(h, sd, q + "norm_mha")
        a = q + "self_attn."
        qq, kk, vv = (F.linear(z, sd[a + n + ".weight"], sd[a + n + ".bias"]).view(b, -1, H, dk).transpose(1, 2)
                      for n in ("linear_q", "linear_k", "linear_v"))
        if rope is not None:
            qq, kk = _rotary(qq, rope), _rotary(kk, rope)
            if tp["rotary_value"]:
                vv = _rotary(vv, rope)
        scores = torch.matmul(qq, kk.transpose(-2, -1)) / torch.tensor(math.sqrt(dk))
        if norm_method == "softmax_plus":
            mask = (scores > -1e4).float()
            ln = torch.sum(mask, dim=-1, keepdim=True).clamp_(1.)
            scores = scores * (torch.log(ln) / sd[a + "att_norm.train_len"] * mask + 1 - mask)
        z = torch.matmul(torch.softmax(scores, dim=-1), vv).transpose(1, 2).contiguous().view(b, -1, D)
        h = h + F.linear(z, sd[a + "linear_out.weight"], sd[a + "linear_out.bias"])
        # convolution module (convolution.py:87-130)
        m = q + "conv_module."
        z = _ln(h, sd, q + "norm_conv").transpose(1, 2)
        z = F.glu(F.conv1d(z, sd[m + "pointwise_conv1.weight"], sd[m + "pointwise_conv1.bias"]), dim=1)
        kk = sd[m + "depthwise_conv.weight"].shape[-1]
        z = F.conv1d(z, sd[m + "depthwise_conv.weight"], sd[m + "depthwise_conv.bias"], padding=kk // 2, groups=D)
        z = _ln(z, sd, m + "norm", dim=1) if tp["cnn_module_norm"] == "layer_norm" else _bn(z, sd, m + "norm")
        z = F.conv1d(_act(z, act), sd[m + "pointwise_conv2.weight"], sd[m + "pointwise_conv2.bias"])
        h = h + z.transpose(1, 2)
        h = h + 0.5 * ffn(_ln(h, sd, q + "norm_ff"), "feed_forward")
        h = _ln(h, sd, q + "norm_final")
    h = _ln(h, sd, p + "after_norm").transpose(1, 2)
    to = dict(cfg["to"], nonlinearity="swish")
    h = _tdnn_layer(h, sd, "transform_out", to)
    # AttentiveStatsPool (transformer_xvector.py:53-87)
    s = "stats.attention."
    alpha = F.relu(F.conv1d(h, sd[s + "0.weight"], sd[s + "0.bias"]))
    alpha = torch.tanh(_ln(alpha, sd, s + "2", dim=1))
    alpha = torch.softmax(F.conv1d(alpha, sd[s + "4.weight"], sd[s + "4.bias"]), dim=2)
    mean = (alpha * h).sum(2)
    std = torch.sqrt((torch.sum(alpha * (h ** 2), dim=2) - mean ** 2).clamp(1e-5))
    z = _ln(torch.cat([mean, std], dim=1).unsqueeze(2), sd, "stats.norm_stats", dim=1)
    if position == "far":
        return _tdnn_layer(z, sd, "fc1", cfg["fc1_params"], affine_only=True)[:, :, 0]
    if cfg["fc1"]:
        z = _tdnn_layer(z, sd, "fc1", cfg["fc1_params"])
    return _tdnn_layer(z, sd, "fc2", cfg["fc2_params"], affine_only=position == "near_affine")[:, :, 0]


def chunk_plan(num_frames, max_chunk=MAX_CHUNK):
    """for_extract_embedding's split (framework.py:34-47): (chunk lengths, offsets)."""
    num_split = (num_frames + max_chunk - 1) // max_chunk
    split = num_frames // num_split
    lengths = [split] * (num_split - 1) + [num_frames - split * (num_split - 1)]
    offsets = [i * split for i in range(num_split)]
    return lengths, offsets


def extract(sd, feats, cfg, position):
    """feats (T, F) -> embedding, the chunk rule with maxChunk = 300 and its weighted average in fp32."""
    x = torch.as_tensor(feats).unsqueeze(0)
    lengths, offsets = chunk_plan(x.shape[1])
    acc = 0.
    with torch.no_grad():
        for n, o in zip(lengths[:-1], offsets[:-1]):
            acc = acc + n * chunk_forward(sd, x[:, o:o + n], cfg, position)
        last = chunk_forward(sd, x[:, offsets[-1]:], cfg, position)
    return ((acc + lengths[-1] * last) / x.shape[1])[0]
