"""The ECAPA-TDNN of pytorch/model/ecapa-tdnn-xvector.py (the runEcapaXvector.py launcher's model) restated in torch, in
the reference's own channel order, for tests/golden/make_golden_lawlict_ecapa.py, test_lawlict_ecapa_host.py,
test_gpu_lawlict_ecapa.py and tools/bench_ecapa.py --lawlict.

spec() lists the state_dict of ECAPA_TDNN(inputs_dim, N, training=False, ...) for oracle.nnet.make_state_dict; forward()
is extract_embedding's body (:308-329) over such a dict: Conv1dReluBn = conv (no bias) -> ReLU -> BN; Res2Conv1dReluBn
passes its last chunk through, out_i = f_i(spx[i] + out_{i-1}); SE_Connect = mean over T -> Linear -> ReLU -> Linear ->
sigmoid -> x * gate; dense residual sums; conv -> ReLU -> bn_conv; AttentiveStatsPool without global context and with the
std floored at variance 1e-9; bn_stats -> [fc1 ->] fc2 at positions far / near_affine / near."""
import copy

import torch
import torch.nn.functional as F

from oracle import nnet as onn

SCALE = 8
HIDDEN = 128
MAX_CHUNK = 10000

_FC_OFF = {"momentum": 0.5, "affine": False, "track_running_stats": True}
# model_params of pytorch/launcher/runEcapaXvector.py:197-236 (training=False, as its extraction stage rewrites it)
LAUNCHER = {
    "aug_dropout": 0., "tail_dropout": 0., "training": False, "extracted_embedding": "near",
    "channels": 512, "embd_dim": 192,
    "pooling": "ecpa-attentive",
    "pooling_params": {"num_head": 16, "share": True, "affine_layers": 1, "hidden_size": 64, "context": [0], "stddev": True,
                       "temperature": True, "fixed": True},
    "fc1": False,
    "fc1_params": {"nonlinearity": "relu", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                   "bn_params": _FC_OFF},
    "fc2_params": {"nonlinearity": "", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                   "bn_params": _FC_OFF},
    "margin_loss": True,
    "margin_loss_params": {"method": "am", "m": 0.2, "feature_normalize": True, "s": 30, "mhe_loss": False, "mhe_w": 0.01},
    "use_step": True,
    "step_params": {"T": None, "m": True, "lambda_0": 0, "lambda_b": 1000, "alpha": 5, "gamma": 1e-4, "s": False,
                    "s_tuple": (30, 12), "s_list": None, "t": False, "t_tuple": (0.5, 1.2), "p": False,
                    "p_tuple": (0.5, 0.1)},
}


def kwargs(**over):
    """The launcher's model_params with some entries replaced."""
    kw = copy.deepcopy(LAUNCHER)
    kw.update(over)
    return kw


def creation_string(kw, inputs_dim=80, num_targets=1211, position=None):
    """`ECAPA_TDNN(inputs_dim,num_targets,**model_params)` as the launcher writes it to nnet.config (repr of the values),
    with the extraction position replaced."""
    kw = dict(kw, extracted_embedding=position or kw["extracted_embedding"])
    return "ECAPA_TDNN({},{},{})".format(inputs_dim, num_targets, ",".join("{}={!r}".format(k, v) for k, v in kw.items()))


# case -> (inputs_dim, kwargs, short frame counts, chunked frame counts (one utterance each), positions, sd seed, feat seed)
CASES = {
    "launcher": (80, kwargs(), (300, 200, 129, 37, 2, 1), (10050,), ("near",), 631, 6310),
    "fc1": (80, kwargs(fc1=True), (120,), (), ("far", "near_affine", "near"), 632, 6320),
    "c1024": (80, kwargs(channels=1024), (300, 37), (), ("near",), 633, 6330),
    "feat30": (30, kwargs(embd_dim=96), (57, 3), (), ("near", "near_affine"), 634, 6340),
    "c256": (80, kwargs(channels=256), (150, 5), (), ("near",), 635, 6350),
}
# parameters without the running statistics: ECAPA_TDNN(80, 1211, training=False, channels=512) with the constructor's
# fc defaults, and the launcher's model, whose fc2 BatchNorm has no affine parameters (2 x 192 fewer)
PARAMS_DEFAULT = 5796032
PARAMS_LAUNCHER = 5795648


def _relu(params):
    return params["nonlinearity"] == "relu"


def _bn_affine(params):
    return params["bn_params"]["affine"]


def spec(inputs_dim, kw):
    """(key, shape, (kind, fan_in)) of the model's state_dict, training=False, for oracle.nnet.make_state_dict."""
    C, E = kw["channels"], kw["embd_dim"]
    W, D = C // SCALE, 3 * C
    out = [("layer1.conv.weight", (C, inputs_dim, 5), ("w", inputs_dim * 5))] + onn._bn_entries("layer1.bn", C)
    for li in (2, 3, 4):
        p = "layer{}.".format(li)
        out += [(p + "0.conv.weight", (C, C, 1), ("w", C))] + onn._bn_entries(p + "0.bn", C)
        out += [(p + "1.convs.{}.weight".format(i), (W, W, 3), ("w", 3 * W)) for i in range(SCALE - 1)]
        for i in range(SCALE - 1):
            out += onn._bn_entries(p + "1.bns.{}".format(i), W)
        out += [(p + "2.conv.weight", (C, C, 1), ("w", C))] + onn._bn_entries(p + "2.bn", C)
        out += [(p + "3.linear1.weight", (C // 4, C), ("w", C)), (p + "3.linear1.bias", (C // 4,), ("b", 0)),
                (p + "3.linear2.weight", (C, C // 4), ("w", C // 4)), (p + "3.linear2.bias", (C,), ("b", 0))]
    out += [("conv.weight", (D, D, 1), ("w", D)), ("conv.bias", (D,), ("b", 0))] + onn._bn_entries("bn_conv", D)
    out += [("stats.linear1.weight", (HIDDEN, D, 1), ("w", D)), ("stats.linear1.bias", (HIDDEN,), ("b", 0)),
            ("stats.linear2.weight", (D, HIDDEN, 1), ("w", HIDDEN)), ("stats.linear2.bias", (D,), ("b", 0))]
    out += onn._bn_entries("bn_stats", 2 * D)
    if kw["fc1"]:
        out += onn._affine_entries("fc1", 2 * D, E, [0]) + onn._bn_entries("fc1.batchnorm", E, _bn_affine(kw["fc1_params"]))
    out += onn._affine_entries("fc2", E if kw["fc1"] else 2 * D, E, [0]) + \
        onn._bn_entries("fc2.batchnorm", E, _bn_affine(kw["fc2_params"]))
    return out


def _conv_relu_bn(x, sd, p, padding=0, dilation=1):
    y = F.conv1d(x, sd[p + "conv.weight"], None, padding=padding, dilation=dilation)
    return onn.batchnorm_eval(F.relu(y), sd, p + "bn")


def _se_res2block(x, sd, p, d):
    h = _conv_relu_bn(x, sd, p + "0.")
    spx = torch.chunk(h, SCALE, dim=1)
    out, sp = [], None
    for i in range(SCALE - 1):
        sp = spx[i] if i == 0 else sp + spx[i]
        sp = F.conv1d(sp, sd[p + "1.convs.{}.weight".format(i)], None, padding=d, dilation=d)
        sp = onn.batchnorm_eval(F.relu(sp), sd, p + "1.bns.{}".format(i))
        out.append(sp)
    out.append(spx[SCALE - 1])
    z = _conv_relu_bn(torch.cat(out, dim=1), sd, p + "2.")
    g = F.relu(F.linear(z.mean(dim=2), sd[p + "3.linear1.weight"], sd[p + "3.linear1.bias"]))
    g = torch.sigmoid(F.linear(g, sd[p + "3.linear2.weight"], sd[p + "3.linear2.bias"]))
    return z * g.unsqueeze(2)


def _fc(x, sd, name, params, full):
    y = onn.tdnn_affine(x, sd[name + ".affine.weight"], sd[name + ".affine.bias"], [0])
    if not full:
        return y
    if _relu(params):
        y = F.relu(y)
    return onn.batchnorm_eval(y, sd, name + ".batchnorm")


def forward(sd, x, kw, position="near"):
    """x (N, F, T) -> (N, embd_dim, 1): ECAPA_TDNN.extract_embedding's body at `position`."""
    out1 = _conv_relu_bn(x, sd, "layer1.", padding=2)
    out2 = _se_res2block(out1, sd, "layer2.", 2) + out1
    out3 = _se_res2block(out1 + out2, sd, "layer3.", 3) + out1 + out2
    out4 = _se_res2block(out1 + out2 + out3, sd, "layer4.", 4) + out1 + out2 + out3
    out = torch.cat([out2, out3, out4], dim=1)
    out = onn.batchnorm_eval(F.relu(F.conv1d(out, sd["conv.weight"], sd["conv.bias"])), sd, "bn_conv")
    alpha = torch.tanh(F.conv1d(out, sd["stats.linear1.weight"], sd["stats.linear1.bias"]))
    alpha = torch.softmax(F.conv1d(alpha, sd["stats.linear2.weight"], sd["stats.linear2.bias"]), dim=2)
    mean = torch.sum(alpha * out, dim=2)
    residuals = torch.sum(alpha * out ** 2, dim=2) - mean ** 2
    std = torch.sqrt(residuals.clamp(min=1e-9))
    x = onn.batchnorm_eval(torch.cat([mean, std], dim=1), sd, "bn_stats").unsqueeze(2)
    if position == "far":
        assert kw["fc1"]
        return _fc(x, sd, "fc1", kw["fc1_params"], False)
    if kw["fc1"]:
        x = _fc(x, sd, "fc1", kw["fc1_params"], True)
    if position == "near_affine":
        return _fc(x, sd, "fc2", kw["fc2_params"], False)
    if position == "near":
        return _fc(x, sd, "fc2", kw["fc2_params"], True)
    raise TypeError("Expected far or near position, but got {}".format(position))


def state_dict(case):
    inputs_dim, kw, _, _, _, seed, _ = CASES[case]
    return onn.make_state_dict(spec(inputs_dim, kw), seed)


def utterances(case, frames):
    """(n, frames, F) float32 ndarray: two utterances, one for a chunked length."""
    inputs_dim, _, short, _, _, _, fseed = CASES[case]
    return onn.synthetic_feats(2 if frames in short else 1, frames, inputs_dim, fseed + frames)


def extract_embedding(sd, feats, kw, position="near"):
    """One (T, F) utterance through the maxChunk = 10000 rule (oracle.nnet.extract_embedding): 1-D tensor."""
    return onn.extract_embedding(lambda x: forward(sd, x, kw, position), feats, MAX_CHUNK)


def keys():
    """Every golden key "<case>_<pos>_T<frames>", in a stable order."""
    return ["{}_{}_T{}".format(case, pos, t) for case, (_, _, short, long, poss, _, _) in CASES.items()
            for pos in poss for t in short + long]
