# -*- coding:utf-8 -*-
"""egrecho's ECAPA-TDNN blueprint for the native path -- the backbone of subtools2/egrecho/models/ecapa/ (EcapaXvector,
ecapa_xvector.py:364-438; EcapaModel.extract_embedding, model.py:72-103) with the EcapaConfig defaults
(ecapa_config.py:10-50).

Creation string: EcapaXvector(inputs_dim, num_targets, channels=512, embd_dim=192, mfa_dim=1536, pooling_params=None,
embd_layer_num=1, post_norm=False, extracted_embedding="near"); num_targets (the classifier's classes) only matters in
training.  pooling_params takes MQMHASP's names over EcapaConfig's defaults (num_q=1, num_head=1, time_attention=True,
hidden_size=128, stddev=True; share=False, affine_layers=2, norm_type="bn" from the constructor).  The state_dict is
EcapaXvector's key for key (`layer1.linear.*`, `layerN.res2net_block.blocks.i.linear.*`, `layerN.se.linear1/2.*`,
`stats.attention.*`, `bn_stats.*`, `embd1.*`, `embd2.*`); an EcapaModel state_dict (`ecapa.*` + `classifier.*`, e.g.
torch.load(ckpt)["state_dict"] of a trained egrecho checkpoint) loads too: `ecapa.` is stripped and `classifier.*`
dropped.  A dict that carries none of the backbone keys is refused even with strict=False.

It runs on the ECAPA-TDNN extractors of ecapa_tdnn_xvector.py with two differences from ECAPA_TDNN:
  * the blocks are chained (x1 = layer2(x), x2 = layer3(x1), x3 = layer4(x2), :420-427) instead of densely summed, so
    each block reads the previous block's slot of the MFA input (xvb_ecapa_set_chained);
  * the head is bn_stats -> embd1 [-> embd2]: one DenseLayer (conv without bias, BatchNorm without affine when
    post_norm) as "fc2", or embd1 (conv, ReLU, BatchNorm) as "fc1" and embd2 as "fc2"; bn_stats is folded into the
    first of them in float64.  "far" is embd1's output and needs embd_layer_num=2, as in the reference.
extract_embedding applies EcapaModel's 4000-frame chunk rule (campplus_xvector.chunk_sizes).

build_extractor() returns NativeEcapaExtractor at 512 or 1024 channels, which also writes XVBG0001 model files for
bin/xvb-extract; XVB_ECAPA_NATIVE=0, or any other width, selects EcapaExtractor, its Python twin.  Not built:
GroupNorm attention (norm_type="ln") and utterances of different lengths in one batch."""
import os
import sys
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200.model import ecapa_tdnn_xvector as etx  # noqa: E402
from asv_subtools_b200.model.campplus_xvector import CamPPXvector, chunk_sizes  # noqa: E402,F401
from asv_subtools_b200.nnet import TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402

# EcapaConfig's pooling defaults (ecapa_config.py:10-16) over MQMHASP's constructor defaults (ecapa_xvector.py:75-86)
DEFAULT_POOLING = {"num_q": 1, "num_head": 1, "time_attention": True, "hidden_size": 128, "stddev": True,
                   "share": False, "affine_layers": 2, "norm_type": "bn"}
DILATIONS = (2, 3, 4)   # layer2 .. layer4, kernel size 3, scale 8
SCALE = 8
SE_BOTTLENECK = 128


def _unsupported(option, value):
    raise NotImplementedError("{}={!r} is not on the egrecho ECAPA-TDNN path".format(option, value))


class _TDNNBlock(nn.Module):
    """egrecho's TDNNBlock (conv with bias -> ReLU -> BatchNorm, zero padding (k - 1) / 2 * dilation) or, with
    dense=True, its DenseLayer (conv without bias -> BatchNorm without affine when `norm`, else nothing)."""

    def __init__(self, cin, cout, kernel_size=1, dilation=1, dense=False, norm=True):
        super().__init__()
        self.linear = nn.Conv1d(cin, cout, kernel_size, padding=(kernel_size - 1) // 2 * dilation, dilation=dilation,
                                bias=not dense)
        bn = nn.BatchNorm1d(cout, affine=not dense) if norm else nn.Identity()
        self.nonlinear = nn.Sequential(nn.Identity() if dense else nn.ReLU(), bn)
        self.dilation, self.relu = dilation, not dense

    def norm(self):
        bn = self.nonlinear[1]
        return bn if isinstance(bn, nn.BatchNorm1d) else None


class _Res2NetBlock(nn.Module):
    def __init__(self, channels, dilation):
        super().__init__()
        self.blocks = nn.ModuleList([_TDNNBlock(channels // SCALE, channels // SCALE, 3, dilation) for _ in range(SCALE - 1)])


class _SE(nn.Module):
    def __init__(self, channels):
        super().__init__()
        self.linear1 = nn.Linear(channels, SE_BOTTLENECK)
        self.linear2 = nn.Linear(SE_BOTTLENECK, channels)


class _SERes2Block(nn.Module):
    def __init__(self, channels, dilation):
        super().__init__()
        self.conv_relu_bn1 = _TDNNBlock(channels, channels)
        self.res2net_block = _Res2NetBlock(channels, dilation)
        self.conv_relu_bn2 = _TDNNBlock(channels, channels)
        self.se = _SE(channels)


class MQMHASP(nn.Module):
    """egrecho's MQMHASP (ecapa_xvector.py:68-200) with its parameter names, defaults and keys: `attention` is a
    Sequential (conv, ReLU, norm, Tanh, conv) with two affine layers and the bare grouped conv with one.  Its forward is
    that of libs/nnet/pooling.py's MQMHASP, which the ECAPA-TDNN extractors run; norm_type="" (no norm in the attention)
    is built, norm_type="ln" (GroupNorm) is not."""

    def __init__(self, in_dim, num_q=2, num_head=4, hidden_size=128, stddev=True, share=False, affine_layers=2,
                 time_attention=False, norm_type="bn"):
        super().__init__()
        if norm_type == "ln":
            _unsupported("norm_type", norm_type)
        if norm_type not in ("bn", ""):
            raise ValueError("Unsupport norm type:{}".format(norm_type))
        if affine_layers not in (1, 2):
            raise ValueError("Expected 1 or 2 affine layers, but got {}.".format(affine_layers))
        assert in_dim % num_head == 0
        self.stddev, self.share, self.time_attention, self.affine_layers = stddev, share, time_attention, affine_layers
        self.num_head, self.num_q, self.hidden_size, self.in_dim = max(1, num_head), max(1, num_q), hidden_size, in_dim
        head = in_dim // num_head
        idim = ((3 if stddev else 2) if time_attention else 1) * head * num_head
        odim = (1 if share else head) * num_head * num_q
        if affine_layers == 2:
            hidden = hidden_size * num_head * num_q
            self.attention = nn.Sequential(
                nn.Conv1d(idim, hidden, kernel_size=1, groups=num_head), nn.ReLU(),
                nn.BatchNorm1d(hidden) if norm_type == "bn" else nn.Identity(), nn.Tanh(),
                nn.Conv1d(hidden, odim, kernel_size=1, groups=num_head * num_q))
        else:
            self.attention = nn.Conv1d(idim, odim, kernel_size=1, groups=num_head)
        self.out_dim = in_dim * num_q * (2 if stddev else 1)

    def get_output_dim(self):
        return self.out_dim

    def head_width(self):
        return self.in_dim // self.num_head


BACKBONE_PREFIXES = ("layer1.", "layer2.", "layer3.", "layer4.", "mfa.", "stats.", "bn_stats.", "embd1.", "embd2.")


def backbone_state_dict(state_dict):
    """EcapaXvector's keys from an EcapaXvector or EcapaModel state_dict: `ecapa.` is stripped, `classifier.*` dropped.
    Raises when none of the backbone keys is there, and on a shortcut conv, which EcapaXvector never builds."""
    if any(k.startswith("ecapa.") for k in state_dict):
        state_dict = OrderedDict((k[6:] if k.startswith("ecapa.") else k, v) for k, v in state_dict.items()
                                 if not k.startswith("classifier."))
    if not any(k.startswith(BACKBONE_PREFIXES) for k in state_dict):
        raise KeyError("the state_dict carries none of the egrecho ECAPA-TDNN backbone keys (layer1.*, mfa.*, stats.*, "
                       "embd1.* or the same under ecapa.); a Lightning checkpoint keeps them under its 'state_dict' entry")
    if any(".shortcut." in k for k in state_dict):
        _unsupported("shortcut", "conv")
    return state_dict


class EcapaXvector(TopVirtualNnet):
    """egrecho's ECAPA-TDNN: layer1, three chained SE-Res2Net blocks, mfa, MQMHA pooling, bn_stats, embd1 [-> embd2]."""

    def init(self, inputs_dim, num_targets, channels=512, embd_dim=192, mfa_dim=1536, pooling_params=None,
             embd_layer_num=1, post_norm=False, extracted_embedding="near"):
        if embd_layer_num not in (1, 2):
            raise ValueError("embd_layer_num must be 1 or 2, got {!r}".format(embd_layer_num))
        if extracted_embedding not in ("near", "far"):
            raise TypeError("Expected far or near position, but got {}".format(extracted_embedding))
        pooling = dict(DEFAULT_POOLING, **(pooling_params or {}))
        unknown = sorted(set(pooling) - set(DEFAULT_POOLING))
        if unknown:
            raise TypeError("MQMHASP got unexpected pooling_params {}".format(unknown))
        self.inputs_dim, self.channels, self.embd_dim, self.mfa_dim = inputs_dim, channels, embd_dim, mfa_dim
        self.embd_layer_num, self.post_norm, self.extracted_embedding = embd_layer_num, post_norm, extracted_embedding
        self.layer1 = _TDNNBlock(inputs_dim, channels, kernel_size=5)
        self.layer2, self.layer3, self.layer4 = (_SERes2Block(channels, d) for d in DILATIONS)
        self.mfa = _TDNNBlock(channels * 3, mfa_dim)
        self.stats = MQMHASP(mfa_dim, **pooling)
        pooled = self.stats.get_output_dim()
        self.bn_stats = nn.BatchNorm1d(pooled)
        if embd_layer_num == 1:
            self.embd1 = _TDNNBlock(pooled, embd_dim, dense=True, norm=post_norm)
            self.embd2 = nn.Identity()
        else:
            self.embd1 = _TDNNBlock(pooled, embd_dim)
            self.embd2 = _TDNNBlock(embd_dim, embd_dim, dense=True, norm=post_norm)

    def load_state_dict(self, state_dict, strict=True, **kw):
        return super().load_state_dict(backbone_state_dict(state_dict), strict=strict, **kw)

    def native_records(self):
        return native_records(self)

    def native_config(self):
        return native_config(self)

    def build_extractor(self):
        if self.extracted_embedding == "far" and self.embd_layer_num == 1:
            raise RuntimeError("Request embd in far positon, but got one embd layer related to near.")
        dev = self.device_for_extraction()
        if os.environ.get("XVB_ECAPA_NATIVE", "1") == "0" or self.channels not in etx.NATIVE_CHANNELS:
            return etx.EcapaExtractor(self, dev)        # op-by-op twin; also the path for other channel counts
        return etx.NativeEcapaExtractor(self, dev)

    def _check(self, frames, feat_dim):
        if feat_dim != self.inputs_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.inputs_dim, feat_dim))

    # EcapaModel.extract_embedding's chunk rule is CamPPModel's: the same two methods, over this model's extractor
    extract_embedding = CamPPXvector.extract_embedding
    extract_embedding_batch = CamPPXvector.extract_embedding_batch


def native_config(m):
    """The ECAPA-TDNN handle's configuration of an EcapaXvector (ecapa_tdnn_xvector.native_config's form): always MQMHA
    pooling and the chained residual form."""
    st = m.stats
    return {"create": (m.inputs_dim, m.channels, m.mfa_dim, st.hidden_size * st.num_head * st.num_q, m.embd_dim),
            "mqmha": (st.num_head, st.num_q, st.hidden_size, int(st.share), st.affine_layers, int(st.time_attention),
                      int(st.stddev)),
            "chained": True}


def _f(t):
    return t.detach().float().cpu().numpy()


def _tdnn(name, blk):
    """A TDNNBlock as the handle's (name, w (Cout, Cin, span), bias, context, scale, shift, relu) record: a dilated
    kernel's taps spread over its span with zeros between them, as ECAPA_TDNN's state_dict stores them."""
    w = _f(blk.linear.weight)
    k, d = w.shape[2], blk.dilation
    half = (k - 1) // 2
    context = [d * (i - half) for i in range(k)]
    if d > 1:
        spread = np.zeros(w.shape[:2] + (d * (k - 1) + 1,), dtype=np.float32)
        spread[:, :, ::d] = w
        w = spread
    s, t = fold_batchnorm(blk.norm())
    return (name, w, _f(blk.linear.bias), context, s, t, True)


def head_records(m):
    """bn_stats -> embd1 [-> embd2] as "fc2" (one layer) or "fc1" [+ "fc2"] records; "far" stops after embd1.  bn_stats
    (eval BatchNorm on the pooled statistics) is folded into the first layer in float64: W' = W diag(s), b' = W t + b;
    a DenseLayer has no bias, so its record bias is exactly that fold."""
    if m.embd_layer_num == 1:
        chain = [("fc2", m.embd1)]
    else:
        chain = [("fc1", m.embd1)] + ([("fc2", m.embd2)] if m.extracted_embedding == "near" else [])
    s, t = fold_batchnorm(m.bn_stats)
    out = []
    for i, (name, blk) in enumerate(chain):
        w = blk.linear.weight.detach().double().cpu().numpy()[:, :, 0]
        b = np.zeros(w.shape[0]) if blk.linear.bias is None else blk.linear.bias.detach().double().cpu().numpy()
        if i == 0:
            b = w @ t.astype(np.float64) + b
            w = w * s.astype(np.float64)[None, :]
        scale, shift = fold_batchnorm(blk.norm())
        out.append((name, w.astype(np.float32)[:, :, None], b.astype(np.float32), [0], scale, shift, blk.relu))
    return out


def native_records(m):
    """(name, weight (Cout, Cin, span), bias, context, scale, shift, relu) records for xvb_ecapa_set_layer and
    EcapaExtractor, under the names ECAPA_TDNN's records have: layer1, layerN.bn1 / resI / bn2 / se1 / se2, mfa, the
    attention (ecapa_tdnn_xvector._mqmha_attention) and the head (head_records)."""
    out = [_tdnn("layer1", m.layer1)]
    for li, blk in zip((2, 3, 4), (m.layer2, m.layer3, m.layer4)):
        p = "layer{}.".format(li)
        out.append(_tdnn(p + "bn1", blk.conv_relu_bn1))
        out += [_tdnn(p + "res{}".format(i), b) for i, b in enumerate(blk.res2net_block.blocks)]
        out.append(_tdnn(p + "bn2", blk.conv_relu_bn2))
        for name, lin, relu in (("se1", blk.se.linear1, True), ("se2", blk.se.linear2, False)):
            out.append((p + name, _f(lin.weight)[:, :, None], _f(lin.bias), [0], None, None, relu))
    out.append(_tdnn("mfa", m.mfa))
    for name, w, b, bn, relu, _ in etx._mqmha_attention(m.stats):
        s, t = bn if bn is not None else (None, None)
        out.append((name, w, b, [0], s, t, relu))
    return out + head_records(m)
