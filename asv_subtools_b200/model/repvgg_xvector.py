# -*- coding:utf-8 -*-
"""RepVGG / RepSPK x-vector (2-D) blueprint for the native path -- drop-in for pytorch/model/repvgg_xvector.py
(RepVggXvector.init :17-143, extract_embedding :181-208, auto_model :350-481) over pytorch/libs/nnet/repvgg.py
(RepVGGBlock :29-171, RepSPKBlock :173-294, RepVGG :297-376).

Same constructor signature and defaults, creation string and state_dict keys in both forms: the training form
(`repvgg.stageN.i.rbr_dense.{conv,bn}.*`, `rbr_1x1.*` or `rbr_dense_dilation.*`, `rbr_identity.*` where in == out and
stride == 1) and the deploy form of repvgg_model_convert (`rbr_reparam.{weight,bias}`), plus `fc1.*`, `fc2.*`.
Supported: RepVGG and RepSPK blocks, grouped stages (override_groups_map), BatchNorm with or without affine, per-stage
strides of 1 or 2 (stage0 at stride 1), stage widths that are multiples of 16, statistics pooling with stddev, fc1 on
or off, positions far / near_affine / near.  Other options raise; training-only keywords are accepted and ignored.

At inference every block is one convolution with a bias followed by ReLU (get_equivalent_kernel_bias, repvgg.py:112-152
and :226-275): the branches are folded at hand-over in float64 (groups expanded block-diagonally), cast to fp32, and
every tap whose (Cout, Cin) slab is exactly zero is dropped -- 8 of the 25 taps of a RepSPK block's 5x5 kernel.  stage0
(Cin = 1) runs on the head conv (xvb_conv2d_head_k), every other block on the tap-list conv (xvb_conv2d_taps) with the
bias and ReLU in its epilogue; pooling and fc1 / fc2 are the ResNet blueprint's (the reshape before pooling, :191, is
the same column permutation of the first segment layer).

The launch sequence runs in the native handle (NativeRepVGGExtractor over xvb_repvgg_*, csrc/repvgg_extractor.cu),
which also writes XVBV0001 model files for bin/xvb-extract.  Python hands it the folded blocks; the library prunes the
taps by the same rule (xvb_conv2d_kept_taps) and packs.  XVB_REPVGG_NATIVE=0 selects RepVGGExtractor, the Python driver
of the same kernels in the same order, whose embeddings are bit-identical."""
import ctypes as C
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.model.resnet_xvector import _assign, _segment_chain  # noqa: E402
from asv_subtools_b200.native import NativeExtractor  # noqa: E402
from asv_subtools_b200.nnet import ReluBatchNormTdnnLayer, StatisticsPooling, TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.framework import from_record  # noqa: E402

_GROUPWISE_LAYERS = range(2, 27, 2)


def auto_model(model_name):
    """The named configurations of repvgg_xvector.py:350-481: all at strides [1, 1, 2, 2, 2], base width 64 and
    BatchNorm (momentum 0.5, affine); gN = groups N on the even layers 2..26."""
    a, b, d = [2, 4, 14, 1], [4, 6, 16, 1], [8, 14, 24, 1]
    table = {"RepVGG_A0": (a, [0.75, 0.75, 0.75, 2.5]), "RepVGG_A1": (a, [1, 1, 1, 2.5]),
             "RepVGG_A2": (a, [1.5, 1.5, 1.5, 2.75]), "RepVGG_B0": (b, [1, 1, 1, 2.5]), "RepVGG_B1": (b, [2, 2, 2, 4]),
             "RepVGG_B2": (b, [2.5, 2.5, 2.5, 5]), "RepVGG_B3": (b, [3, 3, 3, 5]), "RepVGG_D2se": (d, [2.5, 2.5, 2.5, 5])}
    for base in ("RepVGG_B1", "RepVGG_B2", "RepVGG_B3"):
        for g in (2, 4):
            table["{}g{}".format(base, g)] = table[base] + ({layer: g for layer in _GROUPWISE_LAYERS},)
    entry = table[model_name]
    params = {"num_blocks": list(entry[0]), "strides": [1, 1, 2, 2, 2], "base_width": 64,
              "width_multiplier": list(entry[1]), "override_groups_map": entry[2] if len(entry) > 2 else None,
              "norm_layer_params": {"momentum": 0.5, "affine": True}}
    if model_name in ("RepVGG_B0", "RepVGG_D2se"):
        params["use_se"] = model_name == "RepVGG_D2se"
    return params


def _conv_bn(cin, cout, k, stride, padding, groups, norm, dilation=1):
    """conv_bn of repvgg.py:20-25 (keys conv.weight, bn.*)."""
    m = nn.Sequential()
    m.add_module("conv", nn.Conv2d(cin, cout, k, stride=stride, padding=padding, dilation=dilation, groups=groups,
                                   bias=False))
    m.add_module("bn", nn.BatchNorm2d(cout, **norm))
    return m


class RepVGGBlock(nn.Module):
    """Parameter container of repvgg.py:29-64: 3x3 conv-BN + 1x1 conv-BN [+ BN identity], or rbr_reparam (deploy)."""
    window = 3

    def __init__(self, in_channels, out_channels, stride=1, groups=1, deploy=False, norm_layer_params={}):
        super().__init__()
        self.in_channels, self.out_channels, self.stride, self.groups = in_channels, out_channels, stride, groups
        self.rbr_reparam = self.rbr_identity = self.rbr_dense = None
        if deploy:
            self.rbr_reparam = nn.Conv2d(in_channels, out_channels, 3, stride=stride, padding=1, groups=groups, bias=True)
            return
        if in_channels == out_channels and stride == 1:
            self.rbr_identity = nn.BatchNorm2d(in_channels, **norm_layer_params)
        self.rbr_dense = _conv_bn(in_channels, out_channels, 3, stride, 1, groups, norm_layer_params)
        self._add_second_branch(norm_layer_params)

    def _add_second_branch(self, norm):
        self.rbr_1x1 = _conv_bn(self.in_channels, self.out_channels, 1, self.stride, 0, self.groups, norm)

    def _second_branch(self):
        """(branch, where its kernel sits in the folded window: a slice pair)."""
        return self.rbr_1x1, (slice(1, 2), slice(1, 2))


class RepSPKBlock(RepVGGBlock):
    """Parameter container of repvgg.py:173-211: 3x3 conv-BN + dilation-2 3x3 conv-BN [+ BN identity], folded to 5x5."""
    window = 5

    def __init__(self, in_channels, out_channels, stride=1, groups=1, deploy=False, norm_layer_params={}):
        nn.Module.__init__(self)
        self.in_channels, self.out_channels, self.stride, self.groups = in_channels, out_channels, stride, groups
        self.rbr_reparam = self.rbr_identity = self.rbr_dense = None
        if deploy:
            self.rbr_reparam = nn.Conv2d(in_channels, out_channels, 5, stride=stride, padding=2, groups=groups, bias=True)
            return
        if in_channels == out_channels and stride == 1:
            self.rbr_identity = nn.BatchNorm2d(in_channels, **norm_layer_params)
        self.rbr_dense = _conv_bn(in_channels, out_channels, 3, stride, 1, groups, norm_layer_params)
        self.rbr_dense_dilation = _conv_bn(in_channels, out_channels, 3, stride, 2, groups, norm_layer_params, dilation=2)

    def _second_branch(self):
        return self.rbr_dense_dilation, (slice(0, 5, 2), slice(0, 5, 2))


def _bn_affine64(bn):
    """Eval BatchNorm as (t, beta - mean * t), t = gamma / sqrt(var + eps), in float64; affine=False: gamma 1, beta 0."""
    std = torch.sqrt(bn.running_var.detach().double().cpu() + bn.eps)
    gamma = bn.weight.detach().double().cpu() if bn.weight is not None else torch.ones_like(std)
    beta = bn.bias.detach().double().cpu() if bn.bias is not None else torch.zeros_like(std)
    t = gamma / std
    return t, beta - bn.running_mean.detach().double().cpu() * t


def _ungroup(w, groups):
    """(Cout, Cin / g, kh, kw) -> (Cout, Cin, kh, kw), block-diagonal over the g groups (Conv2d's rule)."""
    if groups == 1:
        return w
    co, ci = w.shape[0] // groups, w.shape[1]
    dense = w.new_zeros(w.shape[0], ci * groups, *w.shape[2:])
    for g in range(groups):
        dense[g * co:(g + 1) * co, g * ci:(g + 1) * ci] = w[g * co:(g + 1) * co]
    return dense


def fold_block(blk):
    """The block as one (Cout, Cin, k, k) kernel and a bias, float64 (get_equivalent_kernel_bias)."""
    k = blk.window
    if blk.rbr_reparam is not None:
        return _ungroup(blk.rbr_reparam.weight.detach().double().cpu(), blk.groups), blk.rbr_reparam.bias.detach().double().cpu()
    w = torch.zeros(blk.out_channels, blk.in_channels, k, k, dtype=torch.float64)
    t, bias = _bn_affine64(blk.rbr_dense.bn)
    w[:, :, k // 2 - 1:k // 2 + 2, k // 2 - 1:k // 2 + 2] += _ungroup(blk.rbr_dense.conv.weight.detach().double().cpu(),
                                                                      blk.groups) * t.view(-1, 1, 1, 1)
    branch, (sf, st) = blk._second_branch()
    t2, b2 = _bn_affine64(branch.bn)
    w[:, :, sf, st] += _ungroup(branch.conv.weight.detach().double().cpu(), blk.groups) * t2.view(-1, 1, 1, 1)
    bias = bias + b2
    if blk.rbr_identity is not None:
        ti, bi = _bn_affine64(blk.rbr_identity)
        idx = torch.arange(blk.in_channels)
        w[idx, idx, k // 2, k // 2] += ti
        bias = bias + bi
    return w, bias


def kept_taps(w):
    """Taps kf * k + kt whose (Cout, Cin) slab of the fp32 kernel w (Cout, Cin, k, k) is not all zero."""
    k = w.shape[-1]
    nz = (w.reshape(w.shape[0] * w.shape[1], k * k) != 0).any(0)
    taps = [j for j in range(k * k) if bool(nz[j])]
    return taps or [k * k // 2]


class RepVGG(nn.Module):
    """Parameter container of repvgg.py:297-361 (stage0 .. stage4; widths from base_width and width_multiplier)."""

    def __init__(self, head_inplanes, block="RepVGG", num_blocks=[2, 4, 14, 1], strides=[1, 1, 2, 2, 2], base_width=64,
                 width_multiplier=None, override_groups_map=None, deploy=False, use_se=False, norm_layer_params={}):
        super().__init__()
        if width_multiplier is None or len(width_multiplier) != 4 or len(num_blocks) != 4 or len(strides) != 5:
            raise ValueError("RepVGG needs 4 width multipliers, 4 block counts and 5 strides, got {}, {}, {}".format(
                width_multiplier, num_blocks, strides))
        if block == "RepVGG":
            used = RepVGGBlock
        elif block == "RepSPK":
            used = RepSPKBlock
        else:
            raise TypeError("Do not support {} block.".format(block))
        if use_se:
            raise NotImplementedError("use_se=True (SE blocks, e.g. RepVGG_D2se) is not on the native RepVGG path")
        if any(s not in (1, 2) for s in strides):
            raise NotImplementedError("strides={} are not on the native RepVGG path (1 or 2 per stage)".format(strides))
        if strides[0] != 1:
            raise NotImplementedError("strides[0]={}: stage0 runs on the head conv, which has stride 1 only".format(strides[0]))
        groups_map = dict(override_groups_map or {})
        if 0 in groups_map:
            raise ValueError("override_groups_map cannot regroup stage0 (layer 0)")
        wm = [w * (base_width / 64.) for w in width_multiplier]
        self.downsample_multiple = 1
        for s in strides:
            self.downsample_multiple *= s
        widths = [min(64, int(64 * wm[0]))] + [int(c * w) for c, w in zip((64, 128, 256, 512), wm)]
        if any(c % 16 for c in widths):
            raise ValueError("every stage width must be a multiple of 16 for the 2-D conv kernel, got {}".format(widths))
        self.stage0 = used(head_inplanes, widths[0], strides[0], 1, deploy, norm_layer_params)
        inp, layer = widths[0], 1
        for si in range(4):
            blocks = []
            for i in range(num_blocks[si]):
                blocks.append(used(inp, widths[si + 1], strides[si + 1] if i == 0 else 1, groups_map.get(layer, 1), deploy,
                                   norm_layer_params))
                inp, layer = widths[si + 1], layer + 1
            setattr(self, "stage{}".format(si + 1), nn.Sequential(*blocks))
        self.output_planes = inp

    def blocks(self):
        return [self.stage0] + [b for si in range(1, 5) for b in getattr(self, "stage{}".format(si))]

    def get_downsample_multiple(self):
        return self.downsample_multiple

    def get_output_planes(self):
        return self.output_planes


class RepVggXvector(TopVirtualNnet):
    """A repvgg vector framework."""

    def init(self, inputs_dim, num_targets, embd_dim=256, aug_dropout=0., tail_dropout=0., training=True,
             extracted_embedding="near", deploy=False, repvgg_config={}, pooling="statistics", pooling_params={}, fc1=False,
             fc1_params={}, fc2_params={}, margin_loss=False, margin_loss_params={}, use_step=False, step_params={},
             adacos=False, transfer_from="softmax_loss"):
        default_repvgg_config = {                                                              # :22-35
            "auto_model": False, "auto_model_name": "RepVGG_A1", "block": "RepSPK",
            "repvgg_params": {"num_blocks": [2, 4, 14, 1], "strides": [1, 1, 2, 2, 2], "base_width": 32,
                              "width_multiplier": [1, 1, 1, 2.5], "norm_layer_params": {"momentum": 0.5, "affine": True},
                              "override_groups_map": None, "use_se": False}}
        default_pooling_params = {"num_head": 1, "hidden_size": 64, "share": True, "affine_layers": 1, "context": [0],
                                  "stddev": True, "temperature": False, "fixed": True}          # :36-45
        default_fc_params = {"nonlinearity": 'relu', "nonlinearity_params": {"inplace": True}, "bn-relu": False,
                             "bn": True, "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        rc = _assign(default_repvgg_config, repvgg_config)
        rp = auto_model(rc["auto_model_name"]) if rc["auto_model"] else dict(rc["repvgg_params"])
        rp["deploy"], rp["block"] = deploy, rc["block"]
        pp = _assign(default_pooling_params, pooling_params)
        fc1_params = _assign(default_fc_params, fc1_params)
        fc2_params = _assign(default_fc_params, fc2_params)
        if pooling != "statistics":
            raise NotImplementedError("pooling={!r} is not on the native RepVGG path (statistics only)".format(pooling))
        if not pp["stddev"]:
            raise NotImplementedError("stddev=False is not on the native RepVGG path")
        self.inputs_dim = inputs_dim
        self.extracted_embedding = extracted_embedding
        self.use_step, self.step_params = use_step, step_params
        self.repvgg = RepVGG(1, **rp)
        dm = self.repvgg.get_downsample_multiple()
        self.out_freq = (inputs_dim + dm - 1) // dm                                           # :96-97
        self.stats = StatisticsPooling(self.out_freq * self.repvgg.get_output_planes(), stddev=True)
        self.fc1 = ReluBatchNormTdnnLayer(self.stats.get_output_dim(), embd_dim, **fc1_params) if fc1 else None
        self.fc2 = ReluBatchNormTdnnLayer(embd_dim if fc1 else self.stats.get_output_dim(), embd_dim, **fc2_params)
        self.embd_dim = embd_dim
        self.deploy = deploy
        self.transform_keys = ["repvgg", "stats", "fc1", "fc2", "loss"]
        if margin_loss and transfer_from == "softmax_loss":
            self.rename_transform_keys = {"loss.affine.weight": "loss.weight"}

    def build_extractor(self):
        if self.extracted_embedding == "far" and self.fc1 is None:
            raise ValueError("extracted_embedding='far' needs fc1=True (repvgg_xvector.py:194-196 asserts it)")
        if self.extracted_embedding not in ("far", "near_affine", "near"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        dev = self.device_for_extraction()
        if os.environ.get("XVB_REPVGG_NATIVE", "1") == "0":
            return RepVGGExtractor(self, dev)       # op-by-op twin of the native handle
        return NativeRepVGGExtractor(self, dev)


def _block_names(m):
    """The state_dict module path of every block, in m.repvgg.blocks() order."""
    r = m.repvgg
    return ["repvgg.stage0"] + ["repvgg.stage{}.{}".format(si, i) for si in range(1, 5)
                                for i in range(len(getattr(r, "stage{}".format(si))))]


def native_config(m):
    """The fields of xvb_repvgg_config_t for model m."""
    r = m.repvgg
    stages = [getattr(r, "stage{}".format(si)) for si in range(1, 5)]
    return {"feat_dim": m.inputs_dim, "ksize": r.stage0.window, "num_blocks": [len(s) for s in stages],
            "strides": [r.stage0.stride] + [s[0].stride for s in stages],
            "widths": [r.stage0.out_channels] + [s[0].out_channels for s in stages], "pooling_eps": float(m.stats.eps)}


def _named_records(m):
    """(name, w, bias, scale, shift, relu) records for xvb_repvgg_set_layer, named by block module path: every block
    as its fold_block kernel (Cout, Cin, k, k) and bias cast to fp32 -- the arrays RepVGGExtractor packs -- with its ReLU,
    then the segment layers of _segment_chain with their (Cout, Cin, 1) weight as (Cout, Cin), as the ResNet hands them
    over.  The library prunes the taps and packs."""
    f = lambda t: t.detach().float().cpu().numpy()  # noqa: E731
    out = []
    for name, blk in zip(_block_names(m), m.repvgg.blocks()):
        w, b = fold_block(blk)
        out.append((name, f(w), f(b), None, None, True))
    for name, w, b, scale, shift, relu in _segment_chain(m, m.repvgg.get_output_planes()):
        out.append((name, f(w)[:, :, 0], f(b) if b is not None else None, scale, shift, relu))
    return out


class NativeRepVGGExtractor(NativeExtractor):
    """xvb_repvgg_t: folded weights, workspace and the whole launch sequence of RepVGGExtractor in the C library, on the
    device that is current when it is built (or loaded from an XVBV0001 file)."""

    PREFIX = "repvgg"

    def _create_args(self, m):
        from asv_subtools_b200._lib import RepVGGConfig
        c = native_config(m)
        cfg = RepVGGConfig(feat_dim=c["feat_dim"], ksize=c["ksize"], pooling_eps=c["pooling_eps"])
        for field in ("num_blocks", "strides", "widths"):
            getattr(cfg, field)[:] = c[field]
        return (C.byref(cfg),)

    def _layers(self, m):
        for name, w, b, scale, shift, relu in _named_records(m):
            yield name, (w.shape[0], w.shape[1], w.shape[2] if w.ndim == 4 else 1), (w, b, scale, shift), \
                (1 if relu else 0) | (2 if scale is not None else 0)

    def _input(self, feats):
        """Any (B, T, F) CUDA float32 tensor, made contiguous as RepVGGExtractor.extract does."""
        if not (isinstance(feats, torch.Tensor) and feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 3):
            raise TypeError("feats must be a (B, T, F) CUDA float32 tensor")
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        return feats.contiguous()


class RepVGGExtractor:
    """Folded weights on one device + the launch sequence of RepVggXvector.extract_embedding (:181-208), driven from
    Python like ResNetExtractor: the head conv (stage0), one tap-list conv per block (bias and ReLU in the epilogue; the
    last one writes fp32), statistics pooling, the segment layers.  The weights are the records and configuration the
    native handle takes (_named_records, native_config)."""

    def __init__(self, m, device):
        recs = {r[0]: r[1:] for r in _named_records(m)}
        cfg = native_config(m)
        w, b = (torch.from_numpy(a) for a in recs["repvgg.stage0"][:2])
        self.head_w = w.to(device).contiguous()
        self.head_scale = torch.ones(w.shape[0], dtype=torch.float32, device=device)
        self.head_shift = b.to(device)
        self.feat_dim = cfg["feat_dim"]
        self.blocks = []
        for si, n in enumerate(cfg["num_blocks"]):
            for i in range(n):
                w, b = (torch.from_numpy(a) for a in recs["repvgg.stage{}.{}".format(si + 1, i)][:2])
                taps = kept_taps(w)
                self.blocks.append({"stride": cfg["strides"][si + 1] if i == 0 else 1, "cout": w.shape[0],
                                    "k": cfg["ksize"], "taps": taps, "w": ops.pack_conv2d_weight(w.to(device).contiguous(), taps),
                                    "scale": torch.ones(w.shape[0], dtype=torch.float32, device=device),
                                    "shift": b.to(device)})
        self.segment = [from_record(*recs[name], device) for name in ("fc1", "fc2") if name in recs]
        self.eps = cfg["pooling_eps"]
        self.embed_dim = self.segment[-1].cout_real

    def extract(self, feats):
        """feats (B, T, F) fp32 CUDA -> (B, embd_dim) fp32 CUDA, asynchronous on the current stream."""
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        feats = feats.contiguous()
        B, T, F = feats.shape
        dev, P = feats.device, ops.SplitPlanes
        x = P.empty((B, T, F, self.head_w.shape[0]), dev)
        ops.conv2d_head(feats, self.head_w, self.head_scale, self.head_shift, x)     # relu(conv + bias)
        out = None
        for i, blk in enumerate(self.blocks):
            last = i + 1 == len(self.blocks)
            st, co = blk["stride"], blk["cout"]
            T, F = (T - 1) // st + 1, (F - 1) // st + 1
            y = None if last else P.empty((B, T, F, co), dev)
            yf = torch.empty(B, T, F, co, dtype=torch.float32, device=dev) if last else None
            ops.conv2d(x, blk["w"], co, blk["k"], st, blk["scale"], blk["shift"], relu=True, y=y, y_f32=yf, taps=blk["taps"])
            x, out = y, yf
        _, xp = ops.stats_pool_ex(out.view(B, T, F * out.shape[-1]), self.eps, 0, planes=True)
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


if __name__ == "__main__":
    print(RepVggXvector(80, 10, training=False))
