"""Oracle (torch-CPU, fp32) restatement of the reference's 2-D ResNet x-vector (pytorch/model/resnet_xvector.py
extract_embedding :183-208 over pytorch/libs/nnet/resnet.py BasicBlock / ResNet), its state_dict layout, and the golden
cases of tests/golden/resnet.npz.  Test infrastructure only: written from the model's semantics with F.conv2d /
F.batch_norm, layer helpers shared with oracle/nnet.py."""
import os
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import nnet as onn  # noqa: E402

# The online launcher's model (pytorch/launcher/runResnetXvector_online.py:221-275): post-activation blocks with SE,
# fc1=False, fc2 without nonlinearity and with BatchNorm affine=False.
ONLINE = dict(resnet_params={"head_conv": True, "head_conv_params": {"kernel_size": 3, "stride": 1, "padding": 1},
                             "head_maxpool": False, "block": "BasicBlock", "layers": [3, 4, 6, 3],
                             "planes": [32, 64, 128, 256], "use_se": True, "se_ratio": 4, "convXd": 2,
                             "norm_layer_params": {"momentum": 0.5, "affine": True}, "full_pre_activation": False,
                             "zero_init_residual": False},
              pooling="statistics", fc1=False,
              fc2_params={"nonlinearity": "", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                          "bn_params": {"momentum": 0.5, "affine": False, "track_running_stats": True}})
# runResnetXvector.py:196-246: pre-activation blocks without SE, fc1=True, fc1 / fc2 with ReLU and affine BatchNorm.
PREACT = dict(resnet_params={"head_conv": True, "head_conv_params": {"kernel_size": 3, "stride": 1, "padding": 1},
                             "head_maxpool": False, "block": "BasicBlock", "layers": [3, 4, 6, 3],
                             "planes": [32, 64, 128, 256], "convXd": 2,
                             "norm_layer_params": {"momentum": 0.5, "affine": True}, "full_pre_activation": True,
                             "zero_init_residual": False},
              pooling="statistics", fc1=True,
              fc1_params={"nonlinearity": "relu", "bn-relu": False, "bn": True,
                          "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}},
              fc2_params={"nonlinearity": "relu", "bn-relu": False, "bn": True,
                          "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}})
# ResNet18 with pre-activation SE blocks (se_ratio 16: a hidden width that is not a multiple of 4), BatchNorm
# affine=False in the backbone, fc2 with its constructor defaults.
RESNET18 = dict(resnet_params={"layers": [2, 2, 2, 2], "planes": [32, 64, 128, 256], "use_se": True, "se_ratio": 16,
                               "norm_layer_params": {"momentum": 0.5, "affine": False}, "full_pre_activation": True},
                fc1=False)

# name -> (creation kwargs, feature dim, frame counts, positions, checkpoint seed, feature seed)
CASES = {
    "online": (ONLINE, 80, (200, 37, 1), ("near", "near_affine"), 301, 1301),
    "preact": (PREACT, 23, (150, 2), ("far", "near"), 302, 1302),
    "resnet18": (RESNET18, 40, (64,), ("near",), 303, 1303),
}


def creation(kwargs, inputs_dim, position):
    """Creation string of ResNetXvector(inputs_dim, 10, training=False, extracted_embedding=position, **kwargs)."""
    args = dict(training=False, extracted_embedding=position, **kwargs)
    return "ResNetXvector({},10,{})".format(inputs_dim, ",".join("{}={!r}".format(k, v) for k, v in args.items()))


def _config(kwargs):
    rp = dict(kwargs.get("resnet_params", {}))
    fc = {"nonlinearity": "relu", "bn-relu": False, "bn": True, "bn_params": {"affine": True}}
    fc1 = dict(fc, **kwargs.get("fc1_params", {}))
    fc2 = dict(fc, **kwargs.get("fc2_params", {}))
    return dict(layers=rp.get("layers", [3, 4, 6, 3]), planes=rp.get("planes", [32, 64, 128, 256]),
                pre=rp.get("full_pre_activation", True), use_se=rp.get("use_se", False), se_ratio=rp.get("se_ratio", 4),
                bn_affine=rp.get("norm_layer_params", {}).get("affine", True), fc1=kwargs.get("fc1", False),
                fc1_relu=fc1["nonlinearity"] == "relu", fc1_bn=fc1["bn"], fc1_bn_affine=fc1["bn_params"].get("affine", True),
                fc1_bn_relu=fc1["bn-relu"], fc2_relu=fc2["nonlinearity"] == "relu", fc2_bn=fc2["bn"],
                fc2_bn_affine=fc2["bn_params"].get("affine", True), fc2_bn_relu=fc2["bn-relu"])


def resnet_spec(inputs_dim, kwargs):
    """(key, shape, init kind) of ResNetXvector(inputs_dim, N, training=False, **kwargs).state_dict() for
    onn.make_state_dict, in registration order (resnet.py:221-347, BasicBlock :23-66, resnet_xvector.py:87-119)."""
    c = _config(kwargs)
    aff = c["bn_affine"]
    spec = [("resnet.conv1.weight", (c["planes"][0], 1, 3, 3), ("w", 9))] + onn._bn_entries("resnet.bn1", c["planes"][0], aff)
    inp = c["planes"][0]
    for li, (n, p) in enumerate(zip(c["layers"], c["planes"])):
        for i in range(n):
            pre = "resnet.layer{}.{}.".format(li + 1, i)
            cin = inp if i == 0 else p
            if i == 0 and (li > 0 or inp != p):
                spec += [(pre + "downsample.0.weight", (p, inp, 1, 1), ("w", inp))] + onn._bn_entries(pre + "downsample.1", p, aff)
            conv1 = [(pre + "conv1.weight", (p, cin, 3, 3), ("w", 9 * cin))]
            conv2 = [(pre + "conv2.weight", (p, p, 3, 3), ("w", 9 * p))]
            if c["pre"]:
                spec += onn._bn_entries(pre + "bn1", cin, aff) + conv1 + onn._bn_entries(pre + "bn2", p, aff) + conv2
            else:
                spec += conv1 + onn._bn_entries(pre + "bn1", p, aff) + conv2 + onn._bn_entries(pre + "bn2", p, aff)
            if c["use_se"]:
                h = p // c["se_ratio"]
                spec += [(pre + "se.fc_1.weight", (h, p), ("w", p)), (pre + "se.fc_1.bias", (h,), ("b", 0)),
                         (pre + "se.fc_2.weight", (p, h), ("w", h)), (pre + "se.fc_2.bias", (p,), ("b", 0))]
        inp = p
    emb = c["planes"][3]
    stats = 2 * ((inputs_dim + 7) // 8) * emb
    if c["fc1"]:
        spec += onn._affine_entries("fc1", stats, emb, [0])
        spec += onn._bn_entries("fc1.batchnorm", emb, c["fc1_bn_affine"]) if c["fc1_bn"] else []
    spec += onn._affine_entries("fc2", emb if c["fc1"] else stats, emb, [0])
    spec += onn._bn_entries("fc2.batchnorm", emb, c["fc2_bn_affine"]) if c["fc2_bn"] else []
    return spec


def _bn(x, sd, prefix):
    return onn.batchnorm_eval(x, sd, prefix)


def _se(x, sd, prefix):
    """SEBlock_2D.forward (components.py:626-639): mean over all F' x T' positions -> Linear -> ReLU -> Linear ->
    sigmoid -> scale."""
    s = x.mean(dim=(2, 3))
    s = F.relu(F.linear(s, sd[prefix + ".fc_1.weight"], sd[prefix + ".fc_1.bias"]))
    s = torch.sigmoid(F.linear(s, sd[prefix + ".fc_2.weight"], sd[prefix + ".fc_2.bias"]))
    return x * s[:, :, None, None]


def _block(x, sd, prefix, stride, pre):
    ident = x
    if prefix + ".downsample.0.weight" in sd:    # 1x1 conv (stride, no padding) + BN of the un-activated input
        ident = _bn(F.conv2d(x, sd[prefix + ".downsample.0.weight"], stride=stride), sd, prefix + ".downsample.1")
    if pre:      # resnet.py:87-104: bn1 -> relu -> conv1 -> bn2 -> relu -> conv2 -> se; + identity, nothing after
        h = F.conv2d(F.relu(_bn(x, sd, prefix + ".bn1")), sd[prefix + ".conv1.weight"], stride=stride, padding=1)
        z = F.conv2d(F.relu(_bn(h, sd, prefix + ".bn2")), sd[prefix + ".conv2.weight"], padding=1)
        if prefix + ".se.fc_1.weight" in sd:
            z = _se(z, sd, prefix + ".se")
        return z + ident
    # resnet.py:70-85: conv1 -> bn1 -> relu -> conv2 -> bn2 -> se; relu(. + identity)
    h = F.relu(_bn(F.conv2d(x, sd[prefix + ".conv1.weight"], stride=stride, padding=1), sd, prefix + ".bn1"))
    z = _bn(F.conv2d(h, sd[prefix + ".conv2.weight"], padding=1), sd, prefix + ".bn2")
    if prefix + ".se.fc_1.weight" in sd:
        z = _se(z, sd, prefix + ".se")
    return F.relu(z + ident)


def resnet_frames(sd, x, pre):
    """ResNet._forward_impl (resnet.py:351-367) on (B, F, T) features: (B, C, F', T')."""
    x = x.unsqueeze(1)                                                     # resnet_xvector.py:191
    x = F.relu(_bn(F.conv2d(x, sd["resnet.conv1.weight"], padding=1), sd, "resnet.bn1"))
    for li in range(1, 5):
        i = 0
        while "resnet.layer{}.{}.conv1.weight".format(li, i) in sd:
            x = _block(x, sd, "resnet.layer{}.{}".format(li, i), 2 if (li > 1 and i == 0) else 1, pre)
            i += 1
    return x


def resnet_forward(sd, x, extracted_embedding, kwargs):
    """ResNetXvector.extract_embedding (:183-208) on (B, F, T) features -> (B, D, 1)."""
    c = _config(kwargs)
    x = resnet_frames(sd, x, c["pre"])
    x = x.reshape(x.shape[0], x.shape[1] * x.shape[2], x.shape[3])       # :193, channel index c*F' + f
    x = onn.statistics_pooling(x)

    def fc(v, name, full):
        if not full:
            return onn.tdnn_affine(v, sd[name + ".affine.weight"], sd[name + ".affine.bias"], [0])
        return onn.relu_bn_tdnn_layer(v, sd, name, [0], relu=c[name + "_relu"], bn=c[name + "_bn"],
                                      bn_relu=c[name + "_bn_relu"])

    if extracted_embedding == "far":
        assert c["fc1"], "far needs fc1 (resnet_xvector.py:196-198)"
        return fc(x, "fc1", False)
    if c["fc1"]:
        x = fc(x, "fc1", True)
    return fc(x, "fc2", extracted_embedding == "near")
