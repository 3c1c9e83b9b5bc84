"""torch-CPU restatement of the reference's egrecho ECAPA-TDNN at extraction (subtools2/egrecho/models/ecapa/
ecapa_xvector.py EcapaXvector.forward :420-438, MQMHASP.forward :109-149, model.py EcapaModel.extract_embedding :72-103
with XvectorMixin.split_chunks), and the golden cases of tests/golden/make_golden_egrecho_ecapa.py.

Written from the reference's arithmetic, in its operation order, over a backbone state_dict (`layer1.*`, ..., `embd2.*`):
TDNNBlock = conv (zero padding (k - 1) / 2 * dilation) -> ReLU -> BatchNorm, three chained SE-Res2Net blocks (each adds
its input back), mfa over [x1 | x2 | x3], MQMHASP (time attention over each head's [x | mean | std] with the biased
variance clamped at 1e-5), bn_stats, embd1 [-> embd2].  The seeded state_dict rule is conformer_oracle's and the test
utterances are campplus_oracle's."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from campplus_oracle import MAX_CHUNK, SPLIT_T, chunk_sizes, utterances  # noqa: E402,F401  (shared with the generator)
from conformer_oracle import seeded_state_dict  # noqa: E402,F401

DILATIONS = (2, 3, 4)
SCALE = 8
# EcapaConfig's pooling defaults over MQMHASP's constructor defaults
POOLING = {"num_q": 1, "num_head": 1, "time_attention": True, "hidden_size": 128, "stddev": True, "share": False,
           "affine_layers": 2, "norm_type": "bn"}

RECIPE = dict(inputs_dim=80, channels=1024)          # recipes/voxcelebSRC/config/train_ecapa.yaml
DEFAULT = dict(inputs_dim=80, channels=512)          # EcapaConfig()

# name -> (EcapaConfig fields, frame counts through EcapaXvector.forward, frame counts through
# EcapaModel.extract_embedding, positions, sd seed, feature seed)
CASES = {
    "c1024": (RECIPE, (300, 200, 37, 5, 1), (), ("near",), 41, 900),
    "c512": (DEFAULT, (300, 37), (4001, 9000), ("near",), 42, 910),
    "two_layer": (dict(DEFAULT, embd_layer_num=2, post_norm=True), (200, 37), (), ("near", "far"), 43, 920),
    "mqmha": (dict(DEFAULT, pooling_params=dict(num_head=4, num_q=2, share=True, affine_layers=1)), (200, 37), (),
              ("near",), 44, 930),
    "no_norm": (dict(DEFAULT, pooling_params=dict(num_head=2, norm_type="")), (200, 37), (), ("near",), 45, 940),
    "no_tatt": (dict(DEFAULT, pooling_params=dict(time_attention=False)), (200, 37), (), ("near",), 46, 950),
    "c256": (dict(DEFAULT, channels=256), (150, 37), (), ("near",), 47, 960),
}


def blueprint_kwargs(config):
    """EcapaXvector(inputs_dim, num_targets, **kwargs) arguments of an EcapaConfig field dict."""
    return {k: v for k, v in config.items() if k != "inputs_dim"}


def _bn(x, sd, p, eps=1e-5):
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd.get(p + "weight"), sd.get(p + "bias"),
                        False, 0.0, eps)


def _tdnn(x, sd, p, dilation=1, relu=True):
    """TDNNBlock (relu) or DenseLayer (no nonlinearity, BatchNorm when the state_dict has one)."""
    w = sd[p + "linear.weight"]
    x = F.conv1d(x, w, sd.get(p + "linear.bias"), padding=(w.shape[2] - 1) // 2 * dilation, dilation=dilation)
    if relu:
        x = F.relu(x)
    return _bn(x, sd, p + "nonlinear.1.") if p + "nonlinear.1.running_mean" in sd else x


def _block(x, sd, p, dilation):
    h = _tdnn(x, sd, p + "conv_relu_bn1.")
    spx = torch.chunk(h, SCALE, dim=1)
    y, sp = [spx[0]], None
    for i in range(SCALE - 1):
        sp = spx[i + 1] if i == 0 else sp + spx[i + 1]
        sp = _tdnn(sp, sd, p + "res2net_block.blocks.{}.".format(i), dilation)
        y.append(sp)
    h = _tdnn(torch.cat(y, dim=1), sd, p + "conv_relu_bn2.")
    s = F.relu(F.linear(h.mean(dim=2), sd[p + "se.linear1.weight"], sd[p + "se.linear1.bias"]))
    s = torch.sigmoid(F.linear(s, sd[p + "se.linear2.weight"], sd[p + "se.linear2.bias"]))
    return h * s.unsqueeze(2) + x


def _stats(x, m, stddev):
    mean = torch.sum(m * x, dim=-1, keepdim=True)
    std = torch.sqrt((torch.sum(m * x ** 2, dim=-1, keepdim=True) - mean ** 2).clamp(1e-5)) if stddev else None
    return mean, std


def _mqmha(x, sd, pool):
    B, C, T = x.shape
    H, Q = pool["num_head"], pool["num_q"]
    if pool["time_attention"]:
        mean, std = _stats(x, torch.full((B, 1, T), 1.0 / T, device=x.device), pool["stddev"])
        parts = [x.view(B, H, -1, T), mean.repeat(1, 1, T).view(B, H, -1, T)]
        if pool["stddev"]:
            parts.append(std.repeat(1, 1, T).view(B, H, -1, T))
        x_in = torch.cat(parts, dim=2).reshape(B, -1, T)
    else:
        x_in = x
    if pool["affine_layers"] == 2:
        a = F.relu(F.conv1d(x_in, sd["stats.attention.0.weight"], sd["stats.attention.0.bias"], groups=H))
        if "stats.attention.2.running_mean" in sd:
            a = _bn(a, sd, "stats.attention.2.")
        a = F.conv1d(torch.tanh(a), sd["stats.attention.4.weight"], sd["stats.attention.4.bias"], groups=H * Q)
    else:
        a = F.conv1d(x_in, sd["stats.attention.weight"], sd["stats.attention.bias"], groups=H)
    alpha = F.softmax(a, dim=2).reshape(B, H, Q, -1, T)
    mean, std = _stats(x.reshape(B, H, 1, -1, T), alpha, pool["stddev"])
    return torch.cat([mean.reshape(B, -1), std.reshape(B, -1)], dim=1) if pool["stddev"] else mean.reshape(B, -1)


def forward(sd, feats, config):
    """EcapaXvector.forward: feats (B, T, F) fp32 -> (embd, embd_far); embd_far is None with one embedding layer."""
    pool = dict(POOLING, **config.get("pooling_params", {}))
    x = _tdnn(feats.permute(0, 2, 1), sd, "layer1.")
    outs = []
    for li, d in zip((2, 3, 4), DILATIONS):
        x = _block(x, sd, "layer{}.".format(li), d)
        outs.append(x)
    x = _tdnn(torch.cat(outs, dim=1), sd, "mfa.")
    x = _bn(_mqmha(x, sd, pool), sd, "bn_stats.").unsqueeze(2)
    if config.get("embd_layer_num", 1) == 1:
        return _tdnn(x, sd, "embd1.", relu=False).squeeze(2), None
    far = _tdnn(x, sd, "embd1.")
    return _tdnn(far, sd, "embd2.", relu=False).squeeze(2), far.squeeze(2)


def extract_embedding(sd, feats, config, position="near"):
    """EcapaModel.extract_embedding: sum_i size_i * emb_i / sum_i size_i over the chunks of chunk_sizes(T)."""
    acc, off = None, 0
    sizes = chunk_sizes(feats.shape[1])
    for s in sizes:
        near, far = forward(sd, feats[:, off:off + s], config)
        e = near if position == "near" else far
        acc = e * s if acc is None else acc + s * e
        off += s
    return acc / sum(sizes)
