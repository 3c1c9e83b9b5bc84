# -*- coding:utf-8 -*-
"""The second ECAPA-TDNN blueprint of the reference, pytorch/model/ecapa-tdnn-xvector.py (the model of
pytorch/launcher/runEcapaXvector.py, after github.com/lawlict/ECAPA-TDNN) -- drop-in under the same file name, so that
`--blueprint-dir` and integration/extract_xvectors_b200.sh take it for an nnet.config naming that file.  The module name
has a hyphen: the pipeline imports it with __import__ by basename, as the reference's create_model_from_py does; load it
by path otherwise.

Same constructor signature and defaults, creation string and state_dict keys as the reference (ECAPA_TDNN.init :146-261):
`layer1.conv` (no bias) / `layer1.bn`, `layerN.0.conv/bn`, `layerN.1.convs.i` (no bias) / `layerN.1.bns.i`,
`layerN.2.conv/bn`, `layerN.3.linear1/linear2` (nn.Linear), `conv` / `bn_conv` (the 3C-wide MFA layer), `stats.linear1/
linear2` (AttentiveStatsPool(3C, 128)), `bn_stats`, `[fc1.*]`, `fc2.*`, and with training=True the loss layer's `loss.*`
(margin loss: `loss.weight`; softmax: `loss.affine.*`).  Training-only keywords (dropouts, mixup, step and margin
parameters) are accepted and do nothing at extraction.  Built: pooling="ecpa-attentive" (the launcher's), any channel
count, embd_dim, fc1 on or off, positions far / near_affine / near.  Every other pooling raises NotImplementedError.

It runs on the ECAPA-TDNN extractors of ecapa_tdnn_xvector.py (the native handle at 512 or 1024 channels, else or with
XVB_ECAPA_NATIVE=0 the Python twin); what differs from ECAPA_TDNN is handed over as records and one switch:
  * Conv1dReluBn is conv -> ReLU -> BN like ReluBatchNormTdnnLayer; its conv has no bias, so the records have none;
  * Res2Conv1dReluBn (:20-54) passes its LAST chunk through and computes out_i = f_i(spx[i] + out_{i-1}), where the chain
    kernel passes chunk 0 through and computes y[i+1] = f_i(x[i+1] + y[i]).  With the block's channels rotated by
    perm = [7W..8W) + [0..7W) -- the rows (and BatchNorm) of bn1 and the input columns of bn2 -- the kernel computes the
    reference's chunks in rotated order and bn2 reads them back in the reference's order.  The residual and the SE read
    the block's input and bn2's output, whose order is unchanged;
  * SE_Connect's Linear layers are the se1 / se2 records (bottleneck C / 4); the residual sums are ECAPA_TDNN's dense form;
  * AttentiveStatsPool (:120-134) has no global context: alpha = softmax(linear2(tanh(linear1(x)))) without ReLU or BN,
    and std = sqrt(clamp(var, 1e-9)) -- xvb_ecapa_set_attention(h, 0, 1e-9f), which leaves out the global statistics
    pass and "att_gs"; XVBE0003 model files hold it for bin/xvb-extract;
  * bn_stats -> [fc1 ->] fc2 is ECAPA_TDNN's head (ecapa_tdnn_xvector._segment_layers folds bn_stats in float64).
extract_embedding keeps the reference's maxChunk = 10000 rule (:307)."""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200.model import ecapa_tdnn_xvector as etx  # noqa: E402
from asv_subtools_b200.nnet import ReluBatchNormTdnnLayer, TdnnAffine, TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402

SCALE = 8
DILATIONS = (2, 3, 4)      # layer2 .. layer4, kernel size 3, padding = dilation
ATT_HIDDEN = 128           # AttentiveStatsPool(cat_channels, 128)
STD_FLOOR = 1e-9           # std = sqrt(residuals.clamp(min=1e-9))


class Conv1dReluBn(nn.Module):
    def __init__(self, inputs_dim, out_channels, kernel_size=1, stride=1, padding=0, dilation=1, bias=False):
        super().__init__()
        self.conv = nn.Conv1d(inputs_dim, out_channels, kernel_size, stride, padding, dilation, bias=bias)
        self.bn = nn.BatchNorm1d(out_channels)


class Res2Conv1dReluBn(nn.Module):
    def __init__(self, channels, kernel_size=1, stride=1, padding=0, dilation=1, bias=False, scale=4):
        super().__init__()
        assert channels % scale == 0, "{} % {} != 0".format(channels, scale)
        self.scale, self.width = scale, channels // scale
        self.nums = scale if scale == 1 else scale - 1
        self.convs = nn.ModuleList([nn.Conv1d(self.width, self.width, kernel_size, stride, padding, dilation, bias=bias)
                                    for _ in range(self.nums)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(self.width) for _ in range(self.nums)])


class SE_Connect(nn.Module):
    def __init__(self, channels, s=4):
        super().__init__()
        assert channels % s == 0, "{} % {} != 0".format(channels, s)
        self.linear1 = nn.Linear(channels, channels // s)
        self.linear2 = nn.Linear(channels // s, channels)


def SE_Res2Block(channels, kernel_size, stride, padding, dilation, scale):
    return nn.Sequential(
        Conv1dReluBn(channels, channels, kernel_size=1, stride=1, padding=0),
        Res2Conv1dReluBn(channels, kernel_size, stride, padding, dilation, scale=scale),
        Conv1dReluBn(channels, channels, kernel_size=1, stride=1, padding=0),
        SE_Connect(channels))


class AttentiveStatsPool(nn.Module):
    def __init__(self, in_dim, bottleneck_dim):
        super().__init__()
        self.in_dim = in_dim
        self.linear1 = nn.Conv1d(in_dim, bottleneck_dim, kernel_size=1)
        self.linear2 = nn.Conv1d(bottleneck_dim, in_dim, kernel_size=1)


class _MarginLoss(nn.Module):
    """The parameter of the reference's MarginSoftmaxLoss (libs/nnet/loss.py:220-233): weight (num_targets, input_dim, 1)."""

    def __init__(self, input_dim, num_targets):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(num_targets, input_dim, 1))


class _SoftmaxLoss(nn.Module):
    """The parameters of the reference's SoftmaxLoss: its TdnnAffine(input_dim, num_targets)."""

    def __init__(self, input_dim, num_targets):
        super().__init__()
        self.affine = TdnnAffine(input_dim, num_targets)


class ECAPA_TDNN(TopVirtualNnet):
    def init(self, inputs_dim, num_targets, channels=512, embd_dim=192,
             aug_dropout=0., tail_dropout=0., training=True,
             extracted_embedding="near", mixup=False, mixup_alpha=1.0,
             pooling="ecpa-attentive", pooling_params={}, fc1=False, fc1_params={}, fc2_params={},
             margin_loss=True, margin_loss_params={}, use_step=False, step_params={}, transfer_from="softmax_loss"):
        if pooling != "ecpa-attentive":
            raise NotImplementedError("pooling={!r} is not built for pytorch/model/ecapa-tdnn-xvector.py; its native path "
                                      "runs pooling='ecpa-attentive' (the launcher's)".format(pooling))
        default_fc = {"nonlinearity": "relu", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                      "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        fc1_params = etx._merge(default_fc, fc1_params)
        fc2_params = etx._merge(default_fc, fc2_params)
        self.inputs_dim, self.channels, self.embd_dim = inputs_dim, channels, embd_dim
        self.use_step, self.step_params = use_step, step_params
        self.extracted_embedding = extracted_embedding
        self.layer1 = Conv1dReluBn(inputs_dim, channels, kernel_size=5, padding=2)
        self.layer2, self.layer3, self.layer4 = (
            SE_Res2Block(channels, kernel_size=3, stride=1, padding=d, dilation=d, scale=SCALE) for d in DILATIONS)
        cat_channels = channels * 3
        self.conv = nn.Conv1d(cat_channels, cat_channels, kernel_size=1)
        self.bn_conv = nn.BatchNorm1d(cat_channels)
        self.stats = AttentiveStatsPool(cat_channels, ATT_HIDDEN)
        self.bn_stats = nn.BatchNorm1d(cat_channels * 2)
        self.fc1 = ReluBatchNormTdnnLayer(cat_channels * 2, embd_dim, **fc1_params) if fc1 else None
        self.fc2 = ReluBatchNormTdnnLayer(embd_dim if fc1 else cat_channels * 2, embd_dim, **fc2_params)
        if training:
            self.loss = _MarginLoss(embd_dim, num_targets) if margin_loss else _SoftmaxLoss(embd_dim, num_targets)
            self.transform_keys = ["layer2", "layer3", "layer4", "conv", "stats", "fc1", "fc2"]
            if margin_loss and transfer_from == "softmax_loss":
                self.rename_transform_keys = {"loss.affine.weight": "loss.weight"}

    def build_extractor(self):
        if self.extracted_embedding == "far":
            assert self.fc1 is not None, "extracted_embedding='far' needs fc1 (ecapa-tdnn-xvector.py:318-320)"
        elif self.extracted_embedding not in ("near", "near_affine"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        dev = self.device_for_extraction()
        if os.environ.get("XVB_ECAPA_NATIVE", "1") == "0" or self.channels not in etx.NATIVE_CHANNELS:
            return etx.EcapaExtractor(self, dev)       # op-by-op twin; also the path for other channel counts
        return etx.NativeEcapaExtractor(self, dev)

    def native_records(self):
        return native_records(self)

    def native_config(self):
        return native_config(self)


def native_config(m):
    """The ECAPA-TDNN handle's configuration (ecapa_tdnn_xvector.native_config's form): attentive pooling without global
    context and with the 1e-9 variance floor, dense blocks."""
    return {"create": (m.inputs_dim, m.channels, 3 * m.channels, ATT_HIDDEN, m.embd_dim), "mqmha": None, "chained": False,
            "attention": (0, STD_FLOOR)}


def rotation(channels, scale=SCALE):
    """The block channel permutation that maps Res2Conv1dReluBn onto the chain kernel: new chunk 0 is old chunk
    scale - 1, new chunk j + 1 is old chunk j."""
    w = channels // scale
    return np.concatenate([np.arange((scale - 1) * w, scale * w), np.arange(0, (scale - 1) * w)])


def _f(t):
    return t.detach().float().cpu().numpy()


def _conv_relu_bn(name, blk, rows=None, cols=None):
    """A Conv1dReluBn (or a Res2Conv1dReluBn conv + its BatchNorm) as a (name, w (Cout, Cin, span), bias, context, scale,
    shift, relu) record: a dilated kernel's taps spread over its span with zeros between them, output rows (and their
    BatchNorm) taken in the order `rows`, input columns in the order `cols`."""
    conv, bn = blk
    w = _f(conv.weight)
    k, d = w.shape[2], conv.dilation[0]
    half = (k - 1) // 2
    context = [d * (i - half) for i in range(k)]
    if d > 1:
        spread = np.zeros(w.shape[:2] + (d * (k - 1) + 1,), dtype=np.float32)
        spread[:, :, ::d] = w
        w = spread
    s, t = fold_batchnorm(bn)
    b = _f(conv.bias) if conv.bias is not None else None
    if rows is not None:
        w, s, t = w[rows], s[rows], t[rows]
        b = b[rows] if b is not None else None
    if cols is not None:
        w = w[:, cols]
    return (name, np.ascontiguousarray(w), b, context, np.ascontiguousarray(s), np.ascontiguousarray(t), True)


def native_records(m):
    """Records for xvb_ecapa_set_layer and EcapaExtractor under ECAPA_TDNN's names: layer1, layerN.bn1 (rows rotated),
    layerN.res0..res6 ([-d, 0, d], zero bias: the convs have none and the chain kernel takes one), layerN.bn2 (columns
    rotated), layerN.se1 / se2, mfa, att_x (linear1 with its bias, no BN), att2, then [fc1] [fc2] with bn_stats folded in."""
    perm = rotation(m.channels)
    out = [_conv_relu_bn("layer1", (m.layer1.conv, m.layer1.bn))]
    for li, blk in zip((2, 3, 4), (m.layer2, m.layer3, m.layer4)):
        p = "layer{}.".format(li)
        out.append(_conv_relu_bn(p + "bn1", (blk[0].conv, blk[0].bn), rows=perm))
        res = blk[1]
        for i, (conv, bn) in enumerate(zip(res.convs, res.bns)):
            name, w, _, ctx, s, t, relu = _conv_relu_bn(p + "res{}".format(i), (conv, bn))
            out.append((name, w, np.zeros(w.shape[0], dtype=np.float32), ctx, s, t, relu))
        out.append(_conv_relu_bn(p + "bn2", (blk[2].conv, blk[2].bn), cols=perm))
        se = blk[3]
        out.append((p + "se1", _f(se.linear1.weight)[:, :, None], _f(se.linear1.bias), [0], None, None, True))
        out.append((p + "se2", _f(se.linear2.weight)[:, :, None], _f(se.linear2.bias), [0], None, None, False))
    out.append(_conv_relu_bn("mfa", (m.conv, m.bn_conv)))
    out.append(("att_x", _f(m.stats.linear1.weight), _f(m.stats.linear1.bias), [0], None, None, False))
    out.append(("att2", _f(m.stats.linear2.weight), _f(m.stats.linear2.bias), [0], None, None, False))
    return out + etx._segment_layers(m)


# Test.
if __name__ == "__main__":
    print(ECAPA_TDNN(80, 10, training=False))
