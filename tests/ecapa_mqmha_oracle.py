"""torch-CPU restatement of the reference's ECAPA_TDNN with pooling="mqmha" (pytorch/model/ecapa_tdnn_xvector.py:289-295,
:326-333, :403-426 over MQMHASP, pytorch/libs/nnet/pooling.py:589-698), the golden cases of
tests/golden/make_golden_ecapa_mqmha.py and the state_dict layout both sides share.

MQMHASP.forward calls `compute_statistics`, which libs/nnet/pooling.py neither defines nor imports; the arithmetic here is
that of the maintained copy of the helper (subtools2/egrecho/nn/pooling.py:18-65): mean = sum(m x), std =
sqrt(clamp(sum(m x^2) - mean^2, 1e-5)), keepdim over time.  Everything up to the mfa layer is oracle.nnet's ECAPA."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nnet as onn  # noqa: E402

# MQMHASP's own constructor defaults (pooling.py:596-606) under ECAPA's pooling defaults (ecapa_tdnn_xvector.py:213-217);
# ECAPA pops `stddev` before building the pooling (:274), so MQMHASP always keeps stddev=True there
MQ_DEFAULTS = {"num_q": 2, "num_head": 4, "hidden_size": 128, "share": True, "affine_layers": 2, "time_attention": True,
               "stddev": True}

# runEcapaXvector_roadmap.py:220-250 without training / extracted_embedding
ROADMAP = {"hidden_size": 64, "num_q": 2, "share": False, "num_head": 2, "affine_layers": 2, "time_attention": True,
           "stddev": True}
_FC_LAUNCHER = {"nonlinearity": '', "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}}
ROADMAP_KW = dict(ecapa_params={"channels": 1024, "embd_dim": 192, "mfa_conv": 1536,
                                "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}},
                  pooling="mqmha", pooling_params=ROADMAP, fc1=False, fc2_params=_FC_LAUNCHER)

# name -> (creation kwargs, frame counts, positions, state_dict seed, feature seed); feat_dim 80 throughout
CASES = {
    "roadmap": (ROADMAP_KW, (300, 37, 2), ("near", "near_affine"), 31, 3100),
    "roadmap_long": (ROADMAP_KW, (10050,), ("near",), 31, 3200),       # two chunks of the maxChunk = 10000 rule
    "share": (dict(ecapa_params={"mfa_conv": 256, "embd_dim": 64}, pooling="mqmha",
                   pooling_params={"hidden_size": 32, "num_q": 2, "num_head": 4, "share": True}), (120, 5), ("near",), 32, 3300),
    "one_layer": (dict(ecapa_params={"mfa_conv": 256, "embd_dim": 64}, pooling="mqmha",
                       pooling_params={"num_q": 2, "num_head": 2, "share": False, "affine_layers": 1}), (90,), ("near",), 33, 3400),
    "no_tatt": (dict(ecapa_params={"mfa_conv": 256, "embd_dim": 64}, pooling="mqmha",
                     pooling_params={"hidden_size": 64, "num_q": 1, "num_head": 2, "share": False, "time_attention": False}),
                (90,), ("near",), 34, 3500),
    "fc1": (dict(ecapa_params={"mfa_conv": 256, "embd_dim": 64}, pooling="mqmha", fc1=True,
                 pooling_params={"hidden_size": 64, "num_q": 2, "num_head": 2, "share": False}),
            (70,), ("far", "near_affine", "near"), 35, 3600),
}


def resolve(pooling_params):
    p = dict(MQ_DEFAULTS)
    p.update(pooling_params or {})
    p["stddev"] = True
    return p


def creation_string(kwargs, pos, feat_dim=80):
    return "ECAPA_TDNN({},10,training=False,extracted_embedding={!r},{})".format(
        feat_dim, pos, ",".join("{}={!r}".format(k, v) for k, v in kwargs.items()))


def mqmha_spec(in_dim, p):
    """stats.attention.* keys of MQMHASP(in_dim, **p) (pooling.py:609-619, :665-698); fan-in = one group's inputs."""
    H, Q, hs = p["num_head"], p["num_q"], p["hidden_size"]
    cg = in_dim // H
    idim = ((3 if p["stddev"] else 2) if p["time_attention"] else 1) * cg      # per head
    odim = (1 if p["share"] else cg) * H * Q
    if p["affine_layers"] == 2:
        hid = hs * H * Q
        return [("stats.attention.0.weight", (hid, idim, 1), ("w", idim)), ("stats.attention.0.bias", (hid,), ("b", 0))] + \
            onn._bn_entries("stats.attention.2", hid) + \
            [("stats.attention.4.weight", (odim, hs, 1), ("w", hs)), ("stats.attention.4.bias", (odim,), ("b", 0))]
    return [("stats.attention.0.weight", (odim, idim, 1), ("w", idim)), ("stats.attention.0.bias", (odim,), ("b", 0))]


def ecapa_mqmha_spec(kwargs, inputs_dim=80):
    """Keys/shapes of ECAPA_TDNN(inputs_dim, N, training=False, **kwargs).state_dict() for pooling="mqmha"."""
    ep = dict({"channels": 1024, "embd_dim": 192, "mfa_conv": 1536}, **kwargs.get("ecapa_params", {}))
    p = resolve(kwargs.get("pooling_params"))
    fc1 = kwargs.get("fc1", False)
    fc2_affine = kwargs.get("fc2_params", {}).get("bn_params", {}).get("affine", True)
    D, E = ep["mfa_conv"], ep["embd_dim"]
    base = onn.ecapa_spec(inputs_dim, channels=ep["channels"], embd_dim=E, mfa_conv=D)
    spec = [e for e in base if not e[0].startswith(("stats.", "bn_stats", "fc1", "fc2"))]
    pooled = D * p["num_q"] * (2 if p["stddev"] else 1)
    spec += mqmha_spec(D, p) + onn._bn_entries("bn_stats", pooled)
    if fc1:
        spec += onn._affine_entries("fc1", pooled, E, [0]) + onn._bn_entries("fc1.batchnorm", E)
    spec += onn._affine_entries("fc2", E if fc1 else pooled, E, [0]) + onn._bn_entries("fc2.batchnorm", E, affine=fc2_affine)
    return spec


def compute_statistics(x, m, stddev=True, eps=1e-5):
    """egrecho/nn/pooling.py:18-65 (dim=-1, keepdim)."""
    mean = torch.sum(m * x, dim=-1, keepdim=True)
    std = torch.sqrt((torch.sum(m * x ** 2, dim=-1, keepdim=True) - mean ** 2).clamp(min=eps)) if stddev else None
    return mean, std


def mqmha_pool(x, sd, p, prefix="stats"):
    """MQMHASP.forward without a mask (pooling.py:627-663): x (B, C, T) -> (B, pooled)."""
    B, C, T = x.shape
    H, Q = p["num_head"], p["num_q"]
    if p["time_attention"]:
        mean, std = compute_statistics(x, torch.full((B, 1, T), 1.0 / T, dtype=x.dtype), p["stddev"])
        parts = [x.view(B, H, -1, T), mean.expand(B, C, T).reshape(B, H, -1, T)]
        if p["stddev"]:
            parts.append(std.expand(B, C, T).reshape(B, H, -1, T))
        x_in = torch.cat(parts, dim=2).reshape(B, -1, T)
    else:
        x_in = x
    w0, b0 = sd[prefix + ".attention.0.weight"], sd[prefix + ".attention.0.bias"]
    a = F.conv1d(x_in, w0.to(x.dtype), b0.to(x.dtype), groups=H)
    if p["affine_layers"] == 2:
        a = torch.tanh(onn.batchnorm_eval(F.relu(a), sd, prefix + ".attention.2"))
        a = F.conv1d(a, sd[prefix + ".attention.4.weight"].to(x.dtype), sd[prefix + ".attention.4.bias"].to(x.dtype), groups=H * Q)
    alpha = torch.softmax(a, dim=2).reshape(B, H, Q, -1, T)
    mean, std = compute_statistics(x.reshape(B, H, 1, -1, T), alpha, p["stddev"])
    out = [mean.reshape(B, -1)] + ([std.reshape(B, -1)] if p["stddev"] else [])
    return torch.cat(out, dim=1)


def ecapa_mqmha_forward(sd, x, kwargs, extracted_embedding="near", pooling=None):
    """ECAPA_TDNN.extract_embedding body (:403-426) with the MQMHASP pooling; x (B, F, T) -> (B, E, 1).  `pooling`
    (resolved MQMHASP options) overrides what the creation kwargs give, for a pooling built directly."""
    p = pooling or resolve(kwargs.get("pooling_params"))
    fc1 = kwargs.get("fc1", False)
    fc2_relu = kwargs.get("fc2_params", {}).get("nonlinearity", "relu") == "relu"
    h = onn.relu_bn_tdnn_layer(x, sd, "layer1", [-2, -1, 0, 1, 2])
    x1 = onn.se_res2block(h, sd, "layer2", 2)
    x2 = onn.se_res2block(h + x1, sd, "layer3", 3)
    x3 = onn.se_res2block(h + x1 + x2, sd, "layer4", 4)
    h = onn.relu_bn_tdnn_layer(torch.cat([x1, x2, x3], dim=1), sd, "mfa", [0])
    h = onn.batchnorm_eval(mqmha_pool(h, sd, p), sd, "bn_stats").unsqueeze(2)
    if extracted_embedding == "far":
        return onn.tdnn_affine(h, sd["fc1.affine.weight"], sd["fc1.affine.bias"], [0])
    if fc1:
        h = onn.relu_bn_tdnn_layer(h, sd, "fc1", [0])
    if extracted_embedding == "near_affine":
        return onn.tdnn_affine(h, sd["fc2.affine.weight"], sd["fc2.affine.bias"], [0])
    return onn.relu_bn_tdnn_layer(h, sd, "fc2", [0], relu=fc2_relu)


def extract(sd, feats, kwargs, pos):
    """One utterance (T, F) ndarray through the maxChunk = 10000 rule -> 1-D tensor."""
    return onn.extract_embedding(lambda x: ecapa_mqmha_forward(sd, x, kwargs, pos), feats)
