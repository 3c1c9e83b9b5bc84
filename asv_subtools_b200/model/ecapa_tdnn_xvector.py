# -*- coding:utf-8 -*-
"""ECAPA-TDNN (SE-Res2Block + attentive statistics pooling) blueprint for the B200 path -- drop-in
for pytorch/model/ecapa_tdnn_xvector.py.

Same constructor signature, creation string and state_dict keys as the reference
(`layerN.conv_relu_bn1.affine.weight`, `layerN.res2net_block.blocks.i.affine.weight` (128,128,2d+1
with the masked taps), `layerN.se.se.1/3.weight`, `mfa.*`, `stats.attention.0/2/4.*`,
`bn_stats.*`, `fc2.*`; ecapa_tdnn_xvector.py:201-357) and the same `extract_embedding()` semantics
(:403-426).  Every contraction runs on the wgmma layer kernel; what the reference does with
chunk/cat/expand copies is expressed through channel-slice views instead:

  * Res2Net (:61-75): block i reads chunk i+1 of the 1024-channel tensor and, for i>=1, the previous
    block's output as a SECOND A source accumulated into the same fp32 accumulator
    (W.(sp + spx[i+1]) = W.sp + W.spx[i+1]) -- no add kernel, no chunk/cat copies;
  * SE (:97-111) = plane_mean -> two M=B GEMMs (ReLU, sigmoid epilogues) -> se_apply, which also
    writes the block output straight into its slot of the (B,T,3072) MFA input and the running sum
    x+x1(+x2) that feeds the next block (:405-409);
  * attentive pooling (:173-188): the (B,4608,T) concat is never built -- the time-constant
    [mean,std] part of the first conv becomes a per-utterance bias (a (B,3072)x(3072,128) GEMM),
    the softmax over T and the weighted moments are one streaming online-softmax pass;
  * bn_stats (:412) is folded into fc2's weights at build time.

pooling="mqmha" (MQMHASP, libs/nnet/pooling.py:589-698, the roadmap launcher's pooling) runs its two grouped attention
convs on the layer kernel's grouped mode (compact weights, each N tile streaming only its group's K slice), the
time-constant [mean_h | std_h] columns of the first as a per-utterance bias, and the pooling on the head-width map of
xvb_attn_head_stats_pool_mq.
"""
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.native import ShardExtractor  # noqa: E402
from asv_subtools_b200.nnet import ReluBatchNormTdnnLayer, TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402
from asv_subtools_b200.nnet.pooling import MQMHASP  # noqa: E402


def _merge(defaults, given):
    """The subset of utils.assign_params_dict (utils.py:319-356) the blueprint needs: recursive
    override of known keys."""
    out = dict(defaults)
    for k, v in (given or {}).items():
        if k in out and isinstance(out[k], dict) and isinstance(v, dict):
            out[k] = _merge(out[k], v)
        else:
            out[k] = v
    return out


class Res2NetBlock(nn.Module):
    def __init__(self, in_channels, out_channels, scale=8, kernel_size=3, dilation=1, bn_params={}):
        super().__init__()
        assert in_channels % scale == 0 and out_channels % scale == 0 and scale > 1
        width = in_channels // scale
        half = kernel_size // 2
        self.context = [i for i in range(-half * dilation, half * dilation + 1, dilation)]
        self.blocks = nn.ModuleList([ReluBatchNormTdnnLayer(width, out_channels // scale, self.context, **bn_params)
                                     for _ in range(scale - 1)])
        self.scale = scale
        self.width = width


class SE_Connect(nn.Module):
    def __init__(self, channels, bottleneck=128):
        super().__init__()
        self.se = nn.Sequential(nn.AdaptiveAvgPool1d(1), nn.Conv1d(channels, bottleneck, kernel_size=1), nn.ReLU(),
                                nn.Conv1d(bottleneck, channels, kernel_size=1), nn.Sigmoid())


class SE_Res2Block(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size=3, dilation=1, scale=8, bn_params={}):
        super().__init__()
        if in_channels != out_channels:
            raise NotImplementedError("B200 SE_Res2Block implements in_channels == out_channels (no shortcut conv)")
        width = int(math.floor(in_channels / scale))
        self.conv_relu_bn1 = ReluBatchNormTdnnLayer(in_channels, width * scale, **bn_params)
        self.res2net_block = Res2NetBlock(width * scale, width * scale, scale=scale, kernel_size=kernel_size,
                                          dilation=dilation, bn_params=bn_params)
        self.conv_relu_bn2 = ReluBatchNormTdnnLayer(in_channels, width * scale, **bn_params)
        self.se = SE_Connect(out_channels)
        self.shortcut = None


class AttentiveStatsPool(nn.Module):
    def __init__(self, in_dim, bottleneck_dim=128, time_attention=False, bn={}):
        super().__init__()
        if not time_attention:
            raise NotImplementedError("B200 AttentiveStatsPool implements time_attention=True (the c1024 recipe)")
        self.in_dim, self.time_attention = in_dim, time_attention
        self.attention = nn.Sequential(nn.Conv1d(in_dim * 3, bottleneck_dim, kernel_size=1), nn.ReLU(),
                                       nn.BatchNorm1d(bottleneck_dim, **bn), nn.Tanh(),
                                       nn.Conv1d(bottleneck_dim, in_dim, kernel_size=1), nn.Softmax(dim=2))


class ECAPA_TDNN(TopVirtualNnet):
    def init(self, inputs_dim, num_targets, aug_dropout=0., tail_dropout=0., training=True,
             extracted_embedding="near", mixup=False, mixup_alpha=1.0, pooling="ecpa-attentive", pooling_params={},
             ecapa_params={}, fc1=False, fc1_params={}, fc2_params={},
             margin_loss=True, margin_loss_params={}, use_step=False, step_params={}, transfer_from="softmax_loss"):
        default_ecapa = {"channels": 1024, "embd_dim": 192, "mfa_conv": 1536,
                         "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        default_pool = {"hidden_size": 128, "time_attention": True, "stddev": True}
        default_fc = {"nonlinearity": "relu", "nonlinearity_params": {"inplace": True}, "bn-relu": False, "bn": True,
                      "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        if pooling not in ("ecpa-attentive", "mqmha"):
            raise NotImplementedError("B200 ECAPA implements pooling='ecpa-attentive' (the reference default) and 'mqmha', "
                                      "not pooling={!r}".format(pooling))
        ecapa_params = _merge(default_ecapa, ecapa_params)
        pooling_params = _merge(default_pool, pooling_params)
        fc1_params = _merge(default_fc, fc1_params)
        fc2_params = _merge(default_fc, fc2_params)
        self.inputs_dim = inputs_dim
        self.use_step, self.step_params = use_step, step_params
        self.extracted_embedding = extracted_embedding
        self.embd_dim = ecapa_params["embd_dim"]
        channels, mfa_conv = ecapa_params["channels"], ecapa_params["mfa_conv"]
        self.layer1 = ReluBatchNormTdnnLayer(inputs_dim, channels, [-2, -1, 0, 1, 2], **ecapa_params)
        self.layer2 = SE_Res2Block(channels, channels, kernel_size=3, dilation=2, scale=8, bn_params=ecapa_params)
        self.layer3 = SE_Res2Block(channels, channels, kernel_size=3, dilation=3, scale=8, bn_params=ecapa_params)
        self.layer4 = SE_Res2Block(channels, channels, kernel_size=3, dilation=4, scale=8, bn_params=ecapa_params)
        self.mfa = ReluBatchNormTdnnLayer(channels * 3, mfa_conv, **ecapa_params)
        if pooling == "mqmha":          # :289-295; `stddev` was popped from pooling_params (:274), so MQMHASP keeps its default
            self.stats = MQMHASP(mfa_conv, **{k: v for k, v in pooling_params.items() if k != "stddev"})
            pooled = self.stats.get_output_dim()
        else:
            self.stats = AttentiveStatsPool(mfa_conv, pooling_params["hidden_size"], pooling_params["time_attention"])
            pooled = mfa_conv * 2
        self.bn_stats = nn.BatchNorm1d(pooled, **ecapa_params["bn_params"])
        self.fc1 = ReluBatchNormTdnnLayer(pooled, self.embd_dim, **fc1_params) if fc1 else None      # :286-287
        self.fc2 = ReluBatchNormTdnnLayer(self.embd_dim if fc1 else pooled, self.embd_dim, **fc2_params)   # :326-333
        self.transform_keys = ["layer1", "layer2", "layer3", "layer4", "stats", "mfa", "bn_stats", "fc1", "fc2", "loss"]
        if margin_loss and transfer_from == "softmax_loss":
            self.rename_transform_keys = {"loss.affine.weight": "loss.weight"}

    def build_extractor(self):
        if self.extracted_embedding == "far":
            assert self.fc1 is not None, "extracted_embedding='far' needs fc1 (ecapa_tdnn_xvector.py:415-416)"
        elif self.extracted_embedding not in ("near", "near_affine"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        dev = self.device_for_extraction()
        if os.environ.get("XVB_ECAPA_NATIVE", "1") == "0" or self.layer1.affine.output_dim not in NATIVE_CHANNELS:
            return EcapaExtractor(self, dev)       # op-by-op twin; also the path for other channel counts
        return NativeEcapaExtractor(self, dev)

    # the records and configuration the extractors below take (egrecho_ecapa_xvector.EcapaXvector has its own)
    def native_records(self):
        return _named_layers(self)

    def native_config(self):
        return native_config(self)


class _Layer(ops.PackedAffine):
    """One TDNN / 1x1-conv layer record of _named_layers (name, weight (Cout, Cin, tot), bias, context, scale, shift, relu)
    as an ops.PackedAffine, groups > 1 for a grouped 1x1 conv, with each launch marked for the profile.  Ungrouped
    one-tap layers keep the (N, K) fp32 matrix too: the segment-level ones run on CUDA cores (ops.small_affine)."""

    def __init__(self, rec, device, groups=1):
        _, w, bias, context, scale, shift, relu = rec
        super().__init__(w, device, context, bias, scale, shift, relu=relu, groups=groups)
        self.w_f32 = ops.to_device(w[:, :, 0], device) if groups == 1 and w.shape[2] == 1 and w.shape[1] % 4 == 0 else None

    def run(self, x, **kw):
        super().run(x, **kw)
        _mark("gemm K={}x{} N={}".format(len(self.context), x.channels, self.cout))

    def run_rows(self, x, sigmoid=False):
        """Segment-level form: x (B, K) fp32 -> (B, N) fp32 on CUDA cores (same kernel as the native extractor)."""
        y = ops.small_affine(x, self.w_f32, self.bias, self.scale, self.shift, relu=self.relu, sigmoid=sigmoid)
        _mark("rows K={} N={}".format(x.shape[1], self.cout))
        return y


# the block-diagonal expansion of a grouped weight, under the name the grouped-mode test imports
_block_diagonal = ops.block_diagonal


def _mqmha_attention(st):
    """The MQMHASP attention as extractor records (name, weight, bias, bn (scale, shift) | None, relu, groups):
    "att_x" = the first conv's x columns as stored (per head [x_h | mean_h | std_h], pooling.py:636-648), "att_gs" = its
    [mean_h | std_h] columns as ONE block-diagonal (Cout, 2C) matrix over the utterance's [mean | std] plus the conv's bias
    (time attention only: the time-constant part becomes a per-utterance bias), "att2" = the second conv.  The first
    conv is att[0], or `attention` itself where one affine layer is a bare conv (egrecho's MQMHASP); without a
    BatchNorm in the attention (egrecho's norm_type="") att_x has none."""
    f = lambda t: t.detach().float().cpu().numpy()  # noqa: E731
    att, H, cg = st.attention, st.num_head, st.head_width()
    first = att[0] if isinstance(att, nn.Sequential) else att
    w0, b0 = f(first.weight), f(first.bias)
    cout = w0.shape[0]
    xcols = np.ascontiguousarray(w0[:, :cg])
    two = st.affine_layers == 2
    bn = fold_batchnorm(att[2]) if two and isinstance(att[2], nn.BatchNorm1d) else None
    out = [("att_x", xcols, None if st.time_attention else b0, bn, two, H)]
    if st.time_attention:
        ns = 2 if st.stddev else 1
        gs = np.zeros((cout, ns * st.in_dim, 1), dtype=np.float32)
        rows = cout // H
        for h in range(H):
            r = slice(h * rows, (h + 1) * rows)
            for k in range(ns):        # k = 0: mean columns, 1: std columns
                gs[r, k * st.in_dim + h * cg:k * st.in_dim + (h + 1) * cg] = w0[r, (k + 1) * cg:(k + 2) * cg]
        out.append(("att_gs", gs, b0, None, False, 1))
    if two:
        out.append(("att2", f(att[4].weight), f(att[4].bias), None, False, H * st.num_q))
    return out


# channel counts the native extractor and the Res2Net chain kernel take: scale 8 x width 64 (C512) or 128 (C1024)
NATIVE_CHANNELS = (512, 1024)
CHAIN_WIDTHS = (64, 128)
_PROFILE = None  # list of (label, cuda event) when profiling (tools/bench_ecapa.py --profile)


def _mark(label):
    if _PROFILE is not None:
        ev = torch.cuda.Event(enable_timing=True)
        ev.record()
        _PROFILE.append((label, ev))


def _named_layers(m):
    """(name, weight (Cout,Cin,tot) ndarray, bias, context, scale, shift, relu) for xvb_ecapa_set_layer: the state_dict
    tensors as stored, eval BatchNorm folded; the attention conv split into its x / [mean|std] columns (:179) and
    bn_stats folded into fc2 (W' = W diag(s), b' = W t + b)."""
    f = lambda t: t.detach().float().cpu().numpy()  # noqa: E731

    def tdnn(name, layer):
        scale, shift = fold_batchnorm(layer.batchnorm)
        return (name, f(layer.affine.weight), f(layer.affine.bias) if layer.affine.bias is not None else None,
                list(layer.affine.context), scale, shift, layer.relu)

    out = [tdnn("layer1", m.layer1)]
    for li, blk in zip((2, 3, 4), (m.layer2, m.layer3, m.layer4)):
        p = "layer{}.".format(li)
        out.append(tdnn(p + "bn1", blk.conv_relu_bn1))
        out += [tdnn(p + "res{}".format(i), b) for i, b in enumerate(blk.res2net_block.blocks)]
        out.append(tdnn(p + "bn2", blk.conv_relu_bn2))
        out.append((p + "se1", f(blk.se.se[1].weight), f(blk.se.se[1].bias), [0], None, None, True))
        out.append((p + "se2", f(blk.se.se[3].weight), f(blk.se.se[3].bias), [0], None, None, False))
    out.append(tdnn("mfa", m.mfa))
    if isinstance(m.stats, MQMHASP):
        for name, w, b, bn, relu, _ in _mqmha_attention(m.stats):
            s, t = bn if bn is not None else (None, None)
            out.append((name, w, b, [0], s, t, relu))
        return out + _segment_layers(m)
    att, c = m.stats.attention, m.stats.in_dim
    w0 = f(att[0].weight)
    s, t = fold_batchnorm(att[2])
    out.append(("att_x", np.ascontiguousarray(w0[:, :c]), None, [0], s, t, True))
    out.append(("att_gs", np.ascontiguousarray(w0[:, c:]), f(att[0].bias), [0], None, None, False))
    out.append(("att2", f(att[4].weight), f(att[4].bias), [0], None, None, False))
    out += _segment_layers(m)
    return out


def _segment_layers(m):
    """[fc1 ->] [fc2] of ECAPA_TDNN.extract_embedding (:412-422) as (name, w, b, [0], scale, shift, relu) records: "far" =
    fc1.affine alone, "near_affine" = [fc1 full ->] fc2.affine, "near" = [fc1 full ->] fc2 full; bn_stats (eval BatchNorm on
    the pooled statistics, :412) is folded into whichever layer reads them: W' = W diag(s), b' = W t + b, in float64."""
    pos = m.extracted_embedding
    chain = ([("fc1", m.fc1, pos != "far")] if m.fc1 is not None else []) + \
            ([("fc2", m.fc2, pos == "near")] if pos != "far" else [])
    s, t = fold_batchnorm(m.bn_stats)
    out = []
    for i, (name, layer, full) in enumerate(chain):
        if full:
            w, b, scale, shift, relu = layer.export()
        else:
            w, b, scale, shift, relu = layer.affine.dense_weight(), layer.affine.bias.detach().float(), None, None, False
        w = w.double().cpu().numpy()[:, :, 0]
        b = b.double().cpu().numpy()
        if i == 0:
            b = w @ t.astype(np.float64) + b
            w = w * s.astype(np.float64)[None, :]
        out.append((name, w.astype(np.float32)[:, :, None], b.astype(np.float32), [0], scale, shift, relu))
    return out


def native_config(m):
    """{"create": the arguments of xvb_ecapa_create after the handle, "mqmha": those of xvb_ecapa_set_mqmha, or None for
    the attentive pooling, "chained": False (dense blocks, xvb_ecapa_set_chained), "attention": None (the default
    attentive pooling; else the arguments of xvb_ecapa_set_attention)} for model m."""
    st = m.stats
    mq = isinstance(st, MQMHASP)
    hidden = st.hidden_size * st.num_head * st.num_q if mq else st.attention[0].out_channels
    return {"create": (m.inputs_dim, m.layer1.affine.output_dim, st.in_dim, hidden, m.embd_dim),
            "mqmha": (st.num_head, st.num_q, st.hidden_size, int(st.share), st.affine_layers, int(st.time_attention),
                      int(st.stddev)) if mq else None,
            "chained": False, "attention": None}


class NativeEcapaExtractor(ShardExtractor):
    """xvb_ecapa_t: packed weights, workspace and the whole launch sequence in the C library, on the device that is
    current when it is built (or loaded from an XVBE0001 / XVBE0002 / XVBE0003 / XVBG0001 file), from the model's native_records()
    and native_config()."""

    PREFIX = "ecapa"

    def _create_args(self, m):
        return m.native_config()["create"]

    def _configure(self, m):
        cfg = m.native_config()
        if cfg["mqmha"] is not None:
            self._call("set_mqmha", self._h, *cfg["mqmha"])
        if cfg["chained"]:
            self._call("set_chained", self._h, 1)
        if cfg.get("attention") is not None:
            self._call("set_attention", self._h, *cfg["attention"])

    def _layers(self, m):
        from asv_subtools_b200._lib import int_array
        for name, w, b, ctx, scale, shift, relu in m.native_records():
            w = np.asarray(w, dtype=np.float32)
            w3 = w.reshape(w.shape[0], w.shape[1], -1)
            yield name, (w3.shape[0], w3.shape[1], int_array(ctx), len(ctx)), (w3, b, scale, shift), \
                (1 if relu else 0) | (2 if scale is not None else 0)


class EcapaExtractor:
    """Packed weights on one device + the launch sequence of ECAPA_TDNN.extract_embedding (:403-426), driven from
    Python op by op: the A/B and profiling twin of NativeEcapaExtractor (XVB_ECAPA_NATIVE=0, tools/bench_ecapa.py
    --profile), and the path for channel counts the handle does not take.  The weights are the records and configuration
    the handle takes (the model's native_records and native_config); the Res2Net stack, its dilation, scale and width come from the
    layerN.resI records, and the MQMHA attention convs are grouped by the handle's rule (att_x: heads, att2: heads x
    queries)."""

    def __init__(self, m, device):
        recs = {r[0]: r for r in m.native_records()}
        cfg = m.native_config()
        self.device = device
        self.feat_dim, self.channels, self.mfa_dim, _, self.embed_dim = cfg["create"]
        self.chained = cfg["chained"]
        # (global_context, floor) of the attentive pooling (xvb_ecapa_set_attention); the default is ECAPA_TDNN's
        self.global_context, self.floor = cfg.get("attention") or (1, 1e-5)
        self.ldf = (self.feat_dim + 7) // 8 * 8
        self.last_launches = 0
        mq = cfg["mqmha"]
        self.mq = None if mq is None else dict(zip(("heads", "q", "hidden", "share", "layers", "tatt", "stddev"), mq))
        # groups of the MQMHA attention convs as the state_dict stores them (pooling.py:665-698)
        groups = {} if mq is None else {"att_x": self.mq["heads"], "att2": self.mq["heads"] * self.mq["q"]}
        layer = lambda name: _Layer(recs[name], device, groups.get(name, 1))  # noqa: E731
        self.layer1 = layer("layer1")
        self.blocks = []
        self.chain = os.environ.get("XVB_ECAPA_RES2NET", "chain") != "gemm"   # one persistent kernel per Res2Net block
        for li in (2, 3, 4):
            p = "layer{}.".format(li)
            res = [layer(n) for n in recs if n.startswith(p + "res")]      # res0 .. res{scale - 2}, in order
            self.blocks.append({
                "bn1": layer(p + "bn1"),
                "res": res,
                "res_w_hi": torch.cat([r.w.hi for r in res], dim=0).contiguous(),
                "res_w_lo": torch.cat([r.w.lo for r in res], dim=0).contiguous(),
                "res_bias": torch.cat([r.bias for r in res]).contiguous(),
                "res_scale": torch.cat([r.scale for r in res]).contiguous(),
                "res_shift": torch.cat([r.shift for r in res]).contiguous(),
                "dilation": res[0].context[-1],
                "nscale": len(res) + 1,
                "width": res[0].cout,
                "bn2": layer(p + "bn2"),
                "se1": layer(p + "se1"),
                "se2": layer(p + "se2"),
            })
        self.mfa = layer("mfa")
        self.segment = [layer(name) for name in ("fc1", "fc2") if name in recs]
        if self.mq is not None:
            self.att = {name: layer(name) for name in ("att_x", "att_gs", "att2") if name in recs}
            return
        self.att_x, self.att2 = layer("att_x"), layer("att2")
        self.att_gs = layer("att_gs") if self.global_context else None

    def extract(self, feats):
        """feats (B,T,F) fp32 CUDA -> (B, embd_dim) fp32 CUDA (asynchronous on the current stream)."""
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        B, T, _ = feats.shape
        dev, C = feats.device, self.channels
        P = ops.SplitPlanes
        _mark("start")
        xin = ops.split_f32(feats, ld=self.ldf)
        _mark("split")
        X = P.empty((B, T, C), dev)
        self.layer1.run(xin, y=X)
        H, R, Z = P.empty((B, T, C), dev), P.empty((B, T, C), dev), P.empty((B, T, C), dev)
        N = P.empty((B, T, C), dev)
        CAT = P.empty((B, T, 3 * C), dev)
        cur = X
        for li, blk in enumerate(self.blocks):
            w = blk["width"]
            blk["bn1"].run(cur, y=H)
            if self.chain and w in CHAIN_WIDTHS:
                ops.res2net_block(H, blk["res_w_hi"], blk["res_w_lo"], blk["res_bias"], blk["res_scale"], blk["res_shift"],
                                  blk["dilation"], blk["nscale"], R, width=w)
                _mark("res2net chain kernel")
            else:
                ops.copy_planes(H.slice(0, w), R.slice(0, w))   # chunk 0 passes through (ecapa_tdnn_xvector.py:63-64)
                _mark("chunk0 copy")
                for i, layer in enumerate(blk["res"]):
                    layer.run(H.slice(w * (i + 1), w * (i + 2)), x2=R.slice(w * i, w * (i + 1)) if i >= 1 else None,
                              y=R.slice(w * (i + 1), w * (i + 2)))
            blk["bn2"].run(R, y=Z)
            zmean, _ = ops.plane_mean(Z, planes=False)
            _mark("plane_mean")
            gate = blk["se2"].run_rows(blk["se1"].run_rows(zmean), sigmoid=True)
            # dense: the running sum x + x1 (+ x2) into N for the next block; chained: the next block reads this slot
            slot = CAT.slice(C * li, C * (li + 1))
            nxt = li + 1 < len(self.blocks) and not self.chained
            ops.se_apply(Z, cur, gate.view(B, C), slot, N if nxt else None)
            _mark("se_apply")
            cur = slot if self.chained else N
        D = self.mfa_dim
        M = P.empty((B, T, D), dev)
        MF = torch.empty(B, T, D, dtype=torch.float32, device=dev)
        self.mfa.run(CAT, y=M, y_f32=MF)
        if self.mq is not None:
            return self._mqmha_tail(M, MF)
        ub = None
        if self.global_context:
            gstat = ops.stats_pool_ex(MF, 1e-5, 1)      # global mean | sqrt(var_unbiased + 1e-5)
            _mark("stats_pool(global)")
            ub = self.att_gs.run_rows(gstat).view(B, -1)
        A1 = P.empty((B, T, self.att_x.cout), dev)
        self.att_x.run(M, utt_bias=ub, tanh=True, y=A1)
        LOG = torch.empty(B, T, D, dtype=torch.float32, device=dev)
        self.att2.run(A1, y_f32=LOG)
        x = ops.attn_stats_pool(LOG, MF, self.floor)
        _mark("attn_stats_pool")
        for layer in self.segment:
            x = layer.run_rows(x)
        return x

    def _mqmha_tail(self, M, MF):
        """MQMHASP.forward (pooling.py:627-663) + the segment layers, in the native extractor's launch order."""
        mq, att = self.mq, self.att
        B, T, D = MF.shape
        dev = MF.device
        P = ops.SplitPlanes
        cg = D // mq["heads"]
        ub = None
        if mq["tatt"]:        # egrecho's compute_statistics: biased variance clamped at 1e-5
            gstat = ops.stats_pool_ex(MF, 1e-5, 0)
            _mark("stats_pool(global)")
            ub = att["att_gs"].run_rows(gstat[:, :att["att_gs"].w_f32.shape[1]].contiguous()).view(B, -1)
        nl = (1 if mq["share"] else cg) * mq["heads"] * mq["q"]
        LOG = torch.empty(B, T, (nl + 3) // 4 * 4, dtype=torch.float32, device=dev)
        if mq["layers"] == 2:
            A1 = P.empty((B, T, att["att_x"].cout), dev)
            att["att_x"].run(M, utt_bias=ub, tanh=True, y=A1)
            att["att2"].run(A1, y_f32=LOG)
        else:
            att["att_x"].run(M, utt_bias=ub, y_f32=LOG)
        pstat = ops.attn_head_stats_pool_mq(LOG[..., :nl], MF, mq["q"] * D, cg if mq["share"] else 1, cg, mq["q"], floor=1e-5)
        _mark("attn_head_stats_pool_mq")
        x = pstat[:, :(2 if mq["stddev"] else 1) * mq["q"] * D].contiguous()
        for layer in self.segment:
            x = layer.run_rows(x)
        return x

    def close(self):
        pass


# Test.
if __name__ == "__main__":
    print(ECAPA_TDNN(80, 10, training=False))
