"""Oracle (torch-CPU) restatement of the reference's RepVGG / RepSPK x-vector (pytorch/model/repvgg_xvector.py
extract_embedding :181-208 over pytorch/libs/nnet/repvgg.py), in both forms: the three-branch training form and the
re-parameterised deploy form, plus the deploy conversion itself (get_equivalent_kernel_bias, repvgg.py:112-152 and
:226-275, in the reference's fp32 order), the state_dict layouts and the golden cases of tests/golden/repvgg.npz.  Test
infrastructure only: written from the model's semantics with F.conv2d / F.batch_norm, layer helpers shared with
oracle/nnet.py."""
import os
import sys
from collections import OrderedDict

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nnet as onn  # noqa: E402

_FC_NO_RELU_BN_FIXED = {"nonlinearity": "", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                        "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}}
# pytorch/launcher/runRepvggXvector.py:219-262: RepSPK, base width 32, [2, 4, 14, 1] x [1, 1, 1, 2.5], fc1 off, fc2
# without nonlinearity and with BatchNorm affine=False
LAUNCHER = dict(embd_dim=256,
                repvgg_config={"auto_model": False, "auto_model_name": "RepVGG_A1", "block": "RepSPK",
                               "repvgg_params": {"num_blocks": [2, 4, 14, 1], "strides": [1, 1, 2, 2, 2], "base_width": 32,
                                                 "width_multiplier": [1, 1, 1, 2.5], "override_groups_map": None,
                                                 "use_se": False, "norm_layer_params": {"momentum": 0.5, "affine": True}}},
                pooling="statistics", fc1=False,
                fc1_params=dict(_FC_NO_RELU_BN_FIXED, nonlinearity="relu"), fc2_params=_FC_NO_RELU_BN_FIXED)
# auto_model RepVGG_A0 (RepVGG block, widths 48 / 96 / 192 / 1280), fc1 on, fc1 / fc2 with their defaults
A0 = dict(repvgg_config={"auto_model": True, "auto_model_name": "RepVGG_A0", "block": "RepVGG"}, fc1=True)
# a small grouped RepSPK stack with BatchNorm affine=False
GROUPED = dict(embd_dim=128,
               repvgg_config={"block": "RepSPK",
                              "repvgg_params": {"num_blocks": [1, 2, 2, 1], "strides": [1, 1, 2, 2, 2], "base_width": 64,
                                                "width_multiplier": [0.5, 0.5, 0.5, 0.5],
                                                "override_groups_map": {2: 2, 3: 4, 5: 2}, "use_se": False,
                                                "norm_layer_params": {"momentum": 0.5, "affine": False}}},
               fc1=False)

# name -> (creation kwargs, feature dim, frame counts, positions, checkpoint seed, feature seed); "repspk" also has a
# deploy form (the same checkpoint after repvgg_model_convert), stored as "repspk_deploy"
CASES = {
    "repspk": (LAUNCHER, 80, (200, 37, 1), ("near",), 401, 1401),
    "a0": (A0, 23, (150, 2), ("far", "near_affine", "near"), 402, 1402),
    "grouped": (GROUPED, 40, (64,), ("near",), 403, 1403),
}
DEPLOY_CASE = "repspk"

# RepVGG_A0 of repvgg_xvector.py's auto_model table
_AUTO = {"RepVGG_A0": {"num_blocks": [2, 4, 14, 1], "strides": [1, 1, 2, 2, 2], "base_width": 64,
                       "width_multiplier": [0.75, 0.75, 0.75, 2.5], "override_groups_map": None,
                       "norm_layer_params": {"momentum": 0.5, "affine": True}}}
# the RepSPK taps that stay: the 3x3 core and the dilation-2 ring (kf * 5 + kt)
REPSPK_TAPS = [0, 2, 4, 6, 7, 8, 10, 11, 12, 13, 14, 16, 17, 18, 20, 22, 24]


def creation(kwargs, inputs_dim, position, deploy=False):
    """Creation string of RepVggXvector(inputs_dim, 10, training=False, extracted_embedding=position, [deploy=True,]
    **kwargs)."""
    args = dict(training=False, extracted_embedding=position, **({"deploy": True} if deploy else {}), **kwargs)
    return "RepVggXvector({},10,{})".format(inputs_dim, ",".join("{}={!r}".format(k, v) for k, v in args.items()))


def _config(kwargs):
    rc = kwargs.get("repvgg_config", {})
    rp = _AUTO[rc["auto_model_name"]] if rc.get("auto_model") else rc["repvgg_params"]
    wm = [w * rp["base_width"] / 64. for w in rp["width_multiplier"]]
    widths = [min(64, int(64 * wm[0]))] + [int(c * w) for c, w in zip((64, 128, 256, 512), wm)]
    groups = rp.get("override_groups_map") or {}
    blocks = [("repvgg.stage0", 1, widths[0], rp["strides"][0], 1)]      # (prefix, cin, cout, stride, groups)
    inp, layer = widths[0], 1
    for si in range(4):
        for i in range(rp["num_blocks"][si]):
            blocks.append(("repvgg.stage{}.{}".format(si + 1, i), inp, widths[si + 1], rp["strides"][si + 1] if i == 0 else 1,
                           groups.get(layer, 1)))
            inp, layer = widths[si + 1], layer + 1
    dm = 1
    for s in rp["strides"]:
        dm *= s
    fc = {"nonlinearity": "relu", "bn-relu": False, "bn": True, "bn_params": {"affine": True}}
    fc1 = dict(fc, **kwargs.get("fc1_params", {}))
    fc2 = dict(fc, **kwargs.get("fc2_params", {}))
    return dict(spk=rc.get("block", "RepSPK") == "RepSPK", blocks=blocks, dm=dm, out_planes=inp,
                bn_affine=rp["norm_layer_params"].get("affine", True), embd=kwargs.get("embd_dim", 256),
                fc1=kwargs.get("fc1", False), fc1_relu=fc1["nonlinearity"] == "relu", fc1_bn=fc1["bn"],
                fc1_bn_affine=fc1["bn_params"].get("affine", True), fc1_bn_relu=fc1["bn-relu"],
                fc2_relu=fc2["nonlinearity"] == "relu", fc2_bn=fc2["bn"], fc2_bn_affine=fc2["bn_params"].get("affine", True),
                fc2_bn_relu=fc2["bn-relu"])


def repvgg_spec(inputs_dim, kwargs, deploy=False):
    """(key, shape, init kind) of RepVggXvector(inputs_dim, N, training=False, deploy=deploy, **kwargs).state_dict() for
    onn.make_state_dict, in registration order (repvgg.py:54-64, :200-210, :326-336; repvgg_xvector.py:93-120)."""
    c = _config(kwargs)
    aff, k = c["bn_affine"], 5 if c["spk"] else 3
    spec = []
    for pre, cin, cout, stride, g in c["blocks"]:
        pre += "."
        if deploy:
            spec += [(pre + "rbr_reparam.weight", (cout, cin // g, k, k), ("w", cin // g * 9)),
                     (pre + "rbr_reparam.bias", (cout,), ("b", 0))]
            continue
        if cin == cout and stride == 1:
            spec += onn._bn_entries(pre + "rbr_identity", cin, aff)
        spec += [(pre + "rbr_dense.conv.weight", (cout, cin // g, 3, 3), ("w", cin // g * 9))]
        spec += onn._bn_entries(pre + "rbr_dense.bn", cout, aff)
        second, ks = ("rbr_dense_dilation", 3) if c["spk"] else ("rbr_1x1", 1)
        spec += [(pre + second + ".conv.weight", (cout, cin // g, ks, ks), ("w", cin // g * ks * ks))]
        spec += onn._bn_entries(pre + second + ".bn", cout, aff)
    stats = 2 * ((inputs_dim + c["dm"] - 1) // c["dm"]) * c["out_planes"]
    emb = c["embd"]
    if c["fc1"]:
        spec += onn._affine_entries("fc1", stats, emb, [0])
        spec += onn._bn_entries("fc1.batchnorm", emb, c["fc1_bn_affine"]) if c["fc1_bn"] else []
    spec += onn._affine_entries("fc2", emb if c["fc1"] else stats, emb, [0])
    spec += onn._bn_entries("fc2.batchnorm", emb, c["fc2_bn_affine"]) if c["fc2_bn"] else []
    return spec


def _bn(x, sd, prefix):
    return onn.batchnorm_eval(x, sd, prefix)


def block_forward(x, sd, prefix, stride, groups, spk):
    """One block, either form (RepVGGBlock.forward :67-79, RepSPKBlock.forward :213-225)."""
    if prefix + ".rbr_reparam.weight" in sd:
        w = sd[prefix + ".rbr_reparam.weight"]
        return F.relu(F.conv2d(x, w, sd[prefix + ".rbr_reparam.bias"], stride=stride, padding=w.shape[-1] // 2,
                               groups=groups))
    y = _bn(F.conv2d(x, sd[prefix + ".rbr_dense.conv.weight"], stride=stride, padding=1, groups=groups), sd,
            prefix + ".rbr_dense.bn")
    if spk:
        y = y + _bn(F.conv2d(x, sd[prefix + ".rbr_dense_dilation.conv.weight"], stride=stride, padding=2, dilation=2,
                             groups=groups), sd, prefix + ".rbr_dense_dilation.bn")
    else:
        y = y + _bn(F.conv2d(x, sd[prefix + ".rbr_1x1.conv.weight"], stride=stride, groups=groups), sd, prefix + ".rbr_1x1.bn")
    if prefix + ".rbr_identity.running_mean" in sd:
        y = y + _bn(x, sd, prefix + ".rbr_identity")
    return F.relu(y)


def repvgg_forward(sd, x, extracted_embedding, kwargs):
    """RepVggXvector.extract_embedding (:181-208) on (B, F, T) features -> (B, D, 1); sd in either form."""
    c = _config(kwargs)
    x = x.unsqueeze(1)
    for pre, _, _, stride, g in c["blocks"]:
        x = block_forward(x, sd, pre, stride, g, c["spk"])
    x = x.reshape(x.shape[0], x.shape[1] * x.shape[2], x.shape[3])       # :191, channel index c*F' + f
    x = onn.statistics_pooling(x)

    def fc(v, name, full):
        if not full:
            return onn.tdnn_affine(v, sd[name + ".affine.weight"], sd[name + ".affine.bias"], [0])
        return onn.relu_bn_tdnn_layer(v, sd, name, [0], relu=c[name + "_relu"], bn=c[name + "_bn"],
                                      bn_relu=c[name + "_bn_relu"])

    if extracted_embedding == "far":
        assert c["fc1"], "far needs fc1 (repvgg_xvector.py:194-196)"
        return fc(x, "fc1", False)
    if c["fc1"]:
        x = fc(x, "fc1", True)
    return fc(x, "fc2", extracted_embedding == "near")


def _fuse(sd, prefix, kernel=None):
    """_fuse_bn_tensor (repvgg.py:124-152): (kernel * gamma / std, beta - mean * gamma / std); BN without affine has
    gamma 1 and beta 0."""
    kernel = sd[prefix.rsplit(".", 1)[0] + ".conv.weight"] if kernel is None else kernel
    std = (sd[prefix + ".running_var"] + onn.BN_EPS).sqrt()
    gamma = sd.get(prefix + ".weight", torch.ones_like(std))
    beta = sd.get(prefix + ".bias", torch.zeros_like(std))
    return kernel * (gamma / std).reshape(-1, 1, 1, 1), beta - sd[prefix + ".running_mean"] * gamma / std


def deploy_state_dict(sd, kwargs):
    """repvgg_model_convert (repvgg.py:378-386) of a training-form state_dict, in its fp32 order."""
    c = _config(kwargs)
    out = OrderedDict()
    for pre, cin, cout, stride, g in c["blocks"]:
        k3, b3 = _fuse(sd, pre + ".rbr_dense.bn")
        if c["spk"]:
            kd, bd = _fuse(sd, pre + ".rbr_dense_dilation.bn")
            k = torch.zeros(kd.shape[0], kd.shape[1], 5, 5, dtype=kd.dtype)
            k[:, :, ::2, ::2] = kd
            kernel, bias = k + F.pad(k3, [1, 1, 1, 1]), b3 + bd
        else:
            k1, b1 = _fuse(sd, pre + ".rbr_1x1.bn")
            kernel, bias = k3 + F.pad(k1, [1, 1, 1, 1]), b3 + b1
        if pre + ".rbr_identity.running_mean" in sd:
            ks = kernel.shape[-1]
            idt = torch.zeros(cin, cin // g, ks, ks)
            for i in range(cin):
                idt[i, i % (cin // g), ks // 2, ks // 2] = 1
            ki, bi = _fuse(sd, pre + ".rbr_identity", idt)
            kernel, bias = kernel + ki, bias + bi
        out[pre + ".rbr_reparam.weight"] = kernel
        out[pre + ".rbr_reparam.bias"] = bias
    for key, v in sd.items():
        if not key.startswith("repvgg."):
            out[key] = v
    return out
