# -*- coding:utf-8 -*-
"""ResNet x-vector (2-D) blueprint for the native path -- drop-in for pytorch/model/resnet_xvector.py (ResNetXvector.init
:18-141, extract_embedding :183-208) over pytorch/libs/nnet/resnet.py (BasicBlock :23-110, ResNet :221-347).

Same constructor signature and defaults, creation string and state_dict keys (`resnet.conv1.weight`, `resnet.bn1.*`,
`resnet.layerL.i.{conv1,bn1,conv2,bn2}.*`, `resnet.layerL.0.downsample.{0,1}.*`, `resnet.layerL.i.se.fc_{1,2}.*`, `fc1.*`,
`fc2.*`).  Supported: convXd=2 BasicBlocks in both block orders (full_pre_activation True / False), SE blocks with any
ratio, the 3x3 stride-1 head conv without max pooling, statistics pooling, fc1 on or off, positions far / near_affine /
near.  Other options raise NotImplementedError; training-only keywords are accepted and ignored.

Every convolution runs on the 2-D wgmma kernel (csrc/conv2d.cu, xvb_conv2d) with eval BatchNorm, ReLU, the residual
add and the next pre-activation block's BN-ReLU in its epilogue; the head conv and the SE scaling have kernels of their
own; pooling and fc1 / fc2 reuse the TDNN path's kernels.  Activations stay channel-contiguous (B, T, F, C) split planes
throughout, so the reshape before pooling (:193, pooled channel c*F' + f) becomes a permutation of the input columns of
the first segment layer, made once when the weights are handed over.

The launch sequence runs in the native handle (NativeResNetExtractor over xvb_resnet_*, csrc/resnet_extractor.cu), which
also writes XVBR0001 model files for bin/xvb-extract.  XVB_RESNET_NATIVE=0 selects ResNetExtractor, the Python driver of
the same kernels in the same order, whose embeddings are bit-identical.  Both take a masked batch of utterances of
different lengths (extract(feats, lengths)): every position tensor then holds exact zeros past each utterance's length at
its own time resolution, which is what the next conv's taps must read."""
import copy
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.native import ShardExtractor, host_lengths  # noqa: E402
from asv_subtools_b200.nnet import ReluBatchNormTdnnLayer, StatisticsPooling, TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402
from asv_subtools_b200.nnet.framework import from_record  # noqa: E402


def _assign(defaults, given):
    """utils.assign_params_dict (utils.py:319-356) as the reference calls it: known keys override the defaults
    (recursively for sub-dicts), unknown keys are dropped."""
    out = copy.deepcopy(defaults)
    for k, v in (given or {}).items():
        if k in out:
            out[k] = _assign(out[k], v) if isinstance(out[k], dict) and isinstance(v, dict) else v
    return out


class SEBlock_2D(nn.Module):
    """Parameter container of components.py:613-639: avg pool -> Linear(C, C/r) -> ReLU -> Linear(C/r, C) -> sigmoid."""

    def __init__(self, in_planes, ratio=16):
        super().__init__()
        self.in_planes = in_planes
        self.fc_1 = nn.Linear(in_planes, in_planes // ratio)
        self.fc_2 = nn.Linear(in_planes // ratio, in_planes)


class BasicBlock(nn.Module):
    """Parameter container of resnet.py:23-66 (same attribute names, so the same state_dict keys)."""

    def __init__(self, inplanes, planes, stride=1, downsample=None, norm_layer_params={}, full_pre_activation=True,
                 use_se=False, se_ratio=4):
        super().__init__()
        self.downsample = downsample
        self.stride = stride
        self.full_pre_activation = full_pre_activation
        conv3x3 = lambda cin, cout, s=1: nn.Conv2d(cin, cout, 3, stride=s, padding=1, bias=False)  # noqa: E731
        if full_pre_activation:
            self.bn1 = nn.BatchNorm2d(inplanes, **norm_layer_params)
            self.conv1 = conv3x3(inplanes, planes, stride)
            self.bn2 = nn.BatchNorm2d(planes, **norm_layer_params)
            self.conv2 = conv3x3(planes, planes)
        else:
            self.conv1 = conv3x3(inplanes, planes, stride)
            self.bn1 = nn.BatchNorm2d(planes, **norm_layer_params)
            self.conv2 = conv3x3(planes, planes)
            self.bn2 = nn.BatchNorm2d(planes, **norm_layer_params)
        self.se = SEBlock_2D(planes, se_ratio) if use_se else None


class ResNet(nn.Module):
    """Parameter container of resnet.py:221-347 for convXd=2 BasicBlocks with the 3x3 stride-1 head conv."""

    def __init__(self, layers, planes, full_pre_activation, use_se, se_ratio, norm_layer_params):
        super().__init__()
        self.conv1 = nn.Conv2d(1, planes[0], kernel_size=3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes[0], **norm_layer_params)
        self.full_pre_activation = full_pre_activation
        inplanes = planes[0]
        for li, (n, p) in enumerate(zip(layers, planes)):
            stride = 1 if li == 0 else 2
            ds = None
            if stride != 1 or inplanes != p:          # resnet.py:324-328
                ds = nn.Sequential(nn.Conv2d(inplanes, p, kernel_size=1, stride=stride, bias=False),
                                   nn.BatchNorm2d(p, **norm_layer_params))
            blocks = [BasicBlock(inplanes, p, stride, ds, norm_layer_params, full_pre_activation, use_se, se_ratio)]
            blocks += [BasicBlock(p, p, 1, None, norm_layer_params, full_pre_activation, use_se, se_ratio)
                       for _ in range(1, n)]
            setattr(self, "layer{}".format(li + 1), nn.Sequential(*blocks))
            inplanes = p

    def blocks(self):
        return [b for li in range(1, 5) for b in getattr(self, "layer{}".format(li))]


class ResNetXvector(TopVirtualNnet):
    """A resnet x-vector framework (2-D, BasicBlock)."""

    def init(self, inputs_dim, num_targets, aug_dropout=0., tail_dropout=0., training=True, extracted_embedding="near",
             cmvn=False, cmvn_params={}, resnet_params={}, pooling="statistics", pooling_params={}, fc1=False, fc1_params={},
             fc2_params={}, margin_loss=False, margin_loss_params={}, use_step=False, step_params={},
             transfer_from="softmax_loss", jit_compile=False):
        default_resnet_params = {                                                          # :28-41
            "head_conv": True, "head_conv_params": {"kernel_size": 3, "stride": 1, "padding": 1},
            "head_maxpool": False, "head_maxpool_params": {"kernel_size": 3, "stride": 1, "padding": 1},
            "block": "BasicBlock", "layers": [3, 4, 6, 3], "planes": [32, 64, 128, 256], "use_se": False, "se_ratio": 4,
            "convXd": 2, "norm_layer_params": {"momentum": 0.5, "affine": True}, "full_pre_activation": True,
            "zero_init_residual": False}
        default_pooling_params = {"num_head": 1, "hidden_size": 64, "share": True, "affine_layers": 1, "context": [0],
                                  "stddev": True, "temperature": False, "fixed": True}     # :43-52
        default_fc_params = {"nonlinearity": 'relu', "nonlinearity_params": {"inplace": True}, "bn-relu": False,
                             "bn": True, "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}  # :54-59
        if cmvn:
            raise NotImplementedError("cmvn=True is not on the native ResNet path (apply CMN to the features instead)")
        if any(resnet_params.get("replace_stride_with_dilation") or []):
            raise NotImplementedError("replace_stride_with_dilation is not on the native ResNet path")
        rp = _assign(default_resnet_params, resnet_params)
        pp = _assign(default_pooling_params, pooling_params)
        fc1_params = _assign(default_fc_params, fc1_params)
        fc2_params = _assign(default_fc_params, fc2_params)
        if rp["convXd"] != 2:
            raise NotImplementedError("convXd={} is not on the native ResNet path (convXd=2 only)".format(rp["convXd"]))
        if rp["block"] != "BasicBlock":
            raise NotImplementedError("block={!r} is not on the native ResNet path (BasicBlock only)".format(rp["block"]))
        if not rp["head_conv"]:
            raise NotImplementedError("head_conv=False is not on the native ResNet path (resnet.py:235 fails on it too)")
        if dict(rp["head_conv_params"]) != {"kernel_size": 3, "stride": 1, "padding": 1}:
            raise NotImplementedError("head_conv_params={} is not on the native ResNet path (kernel_size 3, stride 1, "
                                      "padding 1 only)".format(rp["head_conv_params"]))
        if rp["head_maxpool"]:
            raise NotImplementedError("head_maxpool=True is not on the native ResNet path")
        if pooling != "statistics":
            raise NotImplementedError("pooling={!r} is not on the native ResNet path (statistics only)".format(pooling))
        if not pp["stddev"]:
            raise NotImplementedError("stddev=False is not on the native ResNet path")
        planes, layers = list(rp["planes"]), list(rp["layers"])
        if len(planes) != 4 or len(layers) != 4:
            raise ValueError("layers and planes need four entries, got {} and {}".format(layers, planes))
        if any(p % 16 for p in planes):
            raise ValueError("every plane count must be a multiple of 16 for the 2-D conv kernel, got {}".format(planes))
        self.inputs_dim = inputs_dim
        self.extracted_embedding = extracted_embedding
        self.use_step, self.step_params = use_step, step_params
        self.convXd = 2
        self.resnet = ResNet(layers, planes, bool(rp["full_pre_activation"]), bool(rp["use_se"]), rp["se_ratio"],
                             rp["norm_layer_params"])
        self.out_freq = (inputs_dim + 7) // 8                                               # :99-100
        self.stats = StatisticsPooling(self.out_freq * planes[3], stddev=True)
        self.fc1 = ReluBatchNormTdnnLayer(self.stats.get_output_dim(), planes[3], **fc1_params) if fc1 else None
        self.fc2 = ReluBatchNormTdnnLayer(planes[3] if fc1 else self.stats.get_output_dim(), planes[3], **fc2_params)
        self.embd_dim = planes[3]
        self.transform_keys = ["resnet", "stats", "fc1", "fc2", "loss.weight"]
        if margin_loss and transfer_from == "softmax_loss":
            self.rename_transform_keys = {"loss.affine.weight": "loss.weight"}

    def build_extractor(self):
        if self.extracted_embedding == "far" and self.fc1 is None:
            raise ValueError("extracted_embedding='far' needs fc1=True (resnet_xvector.py:196-198 asserts it)")
        if self.extracted_embedding not in ("far", "near_affine", "near"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        dev = self.device_for_extraction()
        if os.environ.get("XVB_RESNET_NATIVE", "1") == "0":
            return ResNetExtractor(self, dev)       # op-by-op twin of the native handle
        return NativeResNetExtractor(self, dev)


def _stats_column_order(c, f):
    """Index map from the pooled columns of (B, T', F', C) frames ([mean | std], column f*C + c) to the reference's
    reshape (B, C*F', T') (:193, column c*F' + f): out[:, j] = ref[:, perm[j]]."""
    half = np.arange(c * f).reshape(c, f).T.reshape(-1)
    return np.concatenate([half, half + c * f])


def _segment_chain(m, channels=None):
    """The segment layers the extracted position uses (:194-206) as (name, w, b, scale, shift, relu): "far" = fc1.affine
    alone, otherwise [fc1 whole ->] fc2 whole ("near") or fc2.affine ("near_affine"); whole layers through export()
    (BatchNorm folded to scale / shift, or into the weight for "bn-relu"), the first layer's input columns permuted to the
    pooling order of (B, T', F', C) frames.  Shared by the ResNet and RepVGG records; RepVGG passes the channel count of
    its last stage (default: the ResNet's last conv2)."""
    if channels is None:
        channels = m.resnet.blocks()[-1].conv2.out_channels
    perm = torch.from_numpy(_stats_column_order(channels, m.out_freq))
    pos = m.extracted_embedding
    chain = ([("fc1", m.fc1, pos != "far")] if m.fc1 is not None else []) + \
            ([("fc2", m.fc2, pos == "near")] if pos != "far" else [])
    out = []
    for i, (name, layer, full) in enumerate(chain):
        if full:
            w, b, scale, shift, relu = layer.export()
        else:
            w, b, scale, shift, relu = layer.affine.dense_weight(), layer.affine.bias.detach().float(), None, None, False
        if i == 0:
            w = w[:, perm]
        out.append((name, w.contiguous(), b, scale, shift, relu))
    return out


def native_config(m):
    """The arguments of xvb_resnet_create for model m."""
    r = m.resnet
    stages = [getattr(r, "layer{}".format(li)) for li in range(1, 5)]
    return {"feat_dim": m.inputs_dim, "layers": [len(s) for s in stages], "planes": [s[0].conv1.out_channels for s in stages],
            "pre_activation": r.full_pre_activation, "pooling_eps": float(m.stats.eps)}


def _named_records(m):
    """(name, w, bias, scale, shift, relu) records for xvb_resnet_set_layer, named by state_dict module path:
    convolution weights as stored (Cout, Cin, k, k), BatchNorm folded to (scale, shift) with no weight, the SE linears
    as stored, and the segment layers of _segment_chain with their (Cout, Cin, 1) weight as (Cout, Cin).  The library
    only packs and pads these."""
    f = lambda t: t.detach().float().cpu().numpy()  # noqa: E731
    r = m.resnet
    out = []

    def conv(name, c):
        out.append((name, f(c.weight), None, None, None, False))

    def bn(name, b):
        scale, shift = fold_batchnorm(b)
        out.append((name, None, None, scale, shift, False))

    conv("resnet.conv1", r.conv1)
    bn("resnet.bn1", r.bn1)
    for li in range(1, 5):
        for i, blk in enumerate(getattr(r, "layer{}".format(li))):
            p = "resnet.layer{}.{}.".format(li, i)
            conv(p + "conv1", blk.conv1)
            bn(p + "bn1", blk.bn1)
            conv(p + "conv2", blk.conv2)
            bn(p + "bn2", blk.bn2)
            if blk.downsample is not None:
                conv(p + "downsample.0", blk.downsample[0])
                bn(p + "downsample.1", blk.downsample[1])
            if blk.se is not None:
                out.append((p + "se.fc_1", f(blk.se.fc_1.weight), f(blk.se.fc_1.bias), None, None, False))
                out.append((p + "se.fc_2", f(blk.se.fc_2.weight), f(blk.se.fc_2.bias), None, None, False))
    for name, w, b, scale, shift, relu in _segment_chain(m):
        out.append((name, f(w)[:, :, 0], f(b) if b is not None else None, scale, shift, relu))
    return out


def _se_rows(w1, b1, w2, b2, device):
    """SE weights (the se.fc_1 / se.fc_2 records) for xvb_small_affine (K % 4 == 0): the hidden width C/r is zero-padded
    to a multiple of 4; the padded units are relu(0) = 0 and meet zero columns of fc_2, so the gate is unchanged.  fc_1
    also comes as w1k[k] = [w1 / k, ..., w1 / k] (k copies, k a power of two, k * C <= 256): fc_1 applied to the mean of
    k-position groups (see ResNetExtractor._se_gate), which is fc_1 of the mean over all positions."""
    w1, b1, w2, b2 = (torch.from_numpy(a) for a in (w1, b1, w2, b2))
    pad = (-w1.shape[0]) % 4
    if pad:
        w1 = torch.cat([w1, torch.zeros(pad, w1.shape[1])])
        b1 = torch.cat([b1, torch.zeros(pad)])
        w2 = torch.cat([w2, torch.zeros(w2.shape[0], pad)], 1)
    w1k = {}
    k = 1
    while k * w1.shape[1] <= 256:
        w1k[k] = torch.cat([w1 / k] * k, 1).to(device).contiguous()
        k *= 2
    return w1k, b1.to(device), w2.to(device).contiguous(), b2.to(device)


class ResNetExtractor:
    """Packed weights on one device + the launch sequence of ResNetXvector.extract_embedding (:183-208), driven from Python
    like AttentionPoolingExtractor: per block two convs (+ a 1x1 stride-2 downsample in the first block of layers 2-4)
    [+ plane mean, two small affines and the SE scaling], then statistics pooling and the segment layers.  The weights
    are the records and configuration the native handle takes (_named_records, native_config)."""

    TAKES_LENGTHS = True

    def __init__(self, m, device):
        recs = {r[0]: r[1:] for r in _named_records(m)}
        cfg = native_config(m)
        dev = lambda a: torch.from_numpy(a).to(device)  # noqa: E731
        conv = lambda name: ops.pack_conv2d_weight(dev(recs[name][0]).contiguous())  # noqa: E731
        bn = lambda name: (dev(recs[name][2]), dev(recs[name][3]))  # noqa: E731
        self.feat_dim = cfg["feat_dim"]
        self.pre = cfg["pre_activation"]
        self.head_w = dev(recs["resnet.conv1"][0]).contiguous()
        self.head_bn = bn("resnet.bn1")
        self.blocks = []
        for li, (n, co) in enumerate(zip(cfg["layers"], cfg["planes"])):
            for i in range(n):
                p = "resnet.layer{}.{}.".format(li + 1, i)
                self.blocks.append({
                    "stride": 2 if li > 0 and i == 0 else 1, "cout": co,
                    "conv1": conv(p + "conv1"), "conv2": conv(p + "conv2"), "bn1": bn(p + "bn1"), "bn2": bn(p + "bn2"),
                    "ds": (conv(p + "downsample.0"), bn(p + "downsample.1")) if p + "downsample.0" in recs else None,
                    "se": _se_rows(*recs[p + "se.fc_1"][:2], *recs[p + "se.fc_2"][:2], device)
                    if p + "se.fc_1" in recs else None})
        self.segment = [from_record(*recs[name], device) for name in ("fc1", "fc2") if name in recs]
        self.eps = cfg["pooling_eps"]
        self.embed_dim = self.segment[-1].cout_real

    def _se_gate(self, z, se, lengths=None):
        """sigmoid(fc_2(relu(fc_1(mean over positions of z)))).  xvb_plane_mean puts one thread on 8 channels and spreads
        the positions over 8 warps, so a 32-channel layer would keep 4 lanes of a warp busy: the (B, P, C) planes are
        read as (B, P/k, k*C) instead, k consecutive positions side by side, and fc_1's copies of its weight (w1k) sum the
        k group means.  A masked batch (lengths: frames per utterance) takes k from F alone, so that k divides every
        utterance's own L * F positions, and averages each utterance's own rows."""
        b, _, f, c = z.hi.shape
        w1k, b1, w2, b2 = se
        p = z.hi.numel() // (b * c)
        k = 1
        while 2 * k in w1k and (p if lengths is None else f) % (2 * k) == 0:
            k *= 2
        zmean, _ = ops.plane_mean(ops.SplitPlanes(z.hi.view(b, p // k, k * c), z.lo.view(b, p // k, k * c), k * c),
                                  planes=False, lengths=lengths, rows_per_length=f // k)
        return ops.small_affine(ops.small_affine(zmean, w1k[k], b1, relu=True), w2, b2, sigmoid=True)

    def extract(self, feats, lengths=None):
        """feats (B, T, F) fp32 CUDA -> (B, embd_dim) fp32 CUDA, asynchronous on the current stream.  lengths (B,) host
        ints, 1 <= lengths[b] <= T: a masked batch as xvb_resnet_extract_lengths runs it (every length equal to T: the
        unmasked sequence)."""
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        feats = feats.contiguous()
        B, T, F = feats.shape
        dev, P = feats.device, ops.SplitPlanes
        levels = None    # (4, B) int32: the lengths after 0..3 stride-2 stages, ceil(L / 2) each
        if lengths is not None:
            lens = host_lengths(lengths, B)
            bad = np.flatnonzero((lens < 1) | (lens > T))
            if bad.size:
                raise ValueError("lengths[{}]={} outside [1, T={}]".format(bad[0], lens[bad[0]], T))
            if (lens != T).any():
                table = [lens]
                for _ in range(3):
                    table.append((table[-1] - 1) // 2 + 1)
                levels = torch.from_numpy(np.stack(table)).to(dev)
        at = lambda lv: None if levels is None else levels[lv]  # noqa: E731
        level = 0
        c0 = self.head_w.shape[0]
        x = P.empty((B, T, F, c0), dev)
        a = P.empty((B, T, F, c0), dev) if self.pre else None   # relu(bn1(x)) of the first pre-activation block
        s2, t2 = self.blocks[0]["bn1"] if self.pre else (None, None)
        ops.conv2d_head(feats, self.head_w, self.head_bn[0], self.head_bn[1], x, s2, t2, a, lengths=at(0))
        out = None
        for i, blk in enumerate(self.blocks):
            last = i + 1 == len(self.blocks)
            st, co = blk["stride"], blk["cout"]
            T, F = (T - 1) // st + 1, (F - 1) // st + 1
            lin, lout = at(level), at(level + 1 if st == 2 else level)
            h = P.empty((B, T, F, co), dev)
            if self.pre:     # h = relu(bn2(conv1(relu(bn1(x)))))  (resnet.py:87-98)
                ops.conv2d(a, blk["conv1"], co, 3, st, *blk["bn2"], relu=True, y=h, lengths=lin)
            else:            # h = relu(bn1(conv1(x)))  (resnet.py:70-75)
                ops.conv2d(x, blk["conv1"], co, 3, st, *blk["bn1"], relu=True, y=h, lengths=lin)
            ident = x
            if blk["ds"] is not None:   # downsample = conv1x1 (stride) + BN of the un-activated block input
                ident = P.empty((B, T, F, co), dev)
                ops.conv2d(x, blk["ds"][0], co, 1, st, *blk["ds"][1], y=ident, lengths=lin)
            nxt = None if last or not self.pre else self.blocks[i + 1]["bn1"]
            y = None if last else P.empty((B, T, F, co), dev)
            yf = torch.empty(B, T, F, co, dtype=torch.float32, device=dev) if last else None
            a = P.empty((B, T, F, co), dev) if nxt is not None else None
            s2, t2 = nxt if nxt is not None else (None, None)
            bn2 = (None, None) if self.pre else blk["bn2"]
            if blk["se"] is None:       # conv2 [+ bn2] + identity [-> relu] in one epilogue
                ops.conv2d(h, blk["conv2"], co, 3, 1, *bn2, res=ident, relu=not self.pre, y=y, y_f32=yf,
                           scale2=s2, shift2=t2, y2=a, lengths=lout)
            else:
                z = P.empty((B, T, F, co), dev)
                ops.conv2d(h, blk["conv2"], co, 3, 1, *bn2, y=z, lengths=lout)
                gate = self._se_gate(z, blk["se"], lout)
                ops.se_residual(z, gate, ident, relu=not self.pre, y=y, y_f32=yf, scale2=s2, shift2=t2, y2=a, lengths=lout)
            x, out = y, yf
            level += st == 2
        _, xp = ops.stats_pool_ex(out.view(B, T, F * out.shape[-1]), self.eps, 0, planes=True, lengths=at(level))
        for i, layer in enumerate(self.segment):
            if i + 1 == len(self.segment):
                emb = torch.empty(B, 1, layer.cout, dtype=torch.float32, device=dev)
                layer.run(xp, y_f32=emb)
            else:
                y, view = layer.planes(B, 1, dev)
                layer.run(xp, y=y)
                xp = view
        return emb.view(B, -1)[:, :self.embed_dim]

    def close(self):
        pass


class NativeResNetExtractor(ShardExtractor):
    """xvb_resnet_t: packed weights, workspace and the whole launch sequence of ResNetExtractor in the C library, on the
    device that is current when it is built (or loaded from an XVBR0001 file)."""

    PREFIX = "resnet"
    TAKES_LENGTHS = True

    def _create_args(self, m):
        from asv_subtools_b200._lib import int_array
        c = native_config(m)
        return (c["feat_dim"], int_array(c["layers"]), int_array(c["planes"]), 1 if c["pre_activation"] else 0,
                c["pooling_eps"])

    def _layers(self, m):
        for name, w, b, scale, shift, relu in _named_records(m):
            cout = (w if w is not None else scale).shape[0]
            cin, k = (w.shape[1], w.shape[2] if w.ndim == 4 else 1) if w is not None else (0, 0)
            yield name, (cout, cin, k), (w, b, scale, shift), (1 if relu else 0) | (2 if scale is not None else 0)


if __name__ == "__main__":
    print(ResNetXvector(80, 10, training=False))
