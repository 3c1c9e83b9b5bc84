# -*- coding:utf-8 -*-
"""CAM++ x-vector blueprint for the native path -- the backbone of subtools2/egrecho/models/campplus/ (CamPP, campplus.py
:288-359; CamPPModel.extract_embedding, model.py:73-96) with the CamPPConfig defaults (campplus_config.py:11-37).

Creation string: CamPPXvector(inputs_dim, num_targets, embd_dim=512, init_channels=128, growth_rate=32, bn_size=4,
memory_efficient=True); num_targets (the classifier's classes) and memory_efficient (gradient checkpointing) only matter in
training.  The state_dict is CamPP's key for key (`head.*`, `xvector.*`), so a backbone state_dict loads with strict=True;
a CamPPModel state_dict (`cam.*` + `classifier.*`, e.g. torch.load(ckpt)["state_dict"] of a trained egrecho checkpoint)
loads too: `cam.` is stripped and `classifier.*` dropped.  A dict that carries none of the backbone keys is refused even
with strict=False, so that an unloaded model never writes embeddings.

At extraction (CamPPExtractor) the FCM head runs on the 2-D conv kernels (xvb_conv2d_head, xvb_conv2d with stride (2, 1)
and the BasicResBlock epilogue), the stride-2 `tdnn` on the layer kernel's im2col view over a time-padded copy of the head's
output, every dense layer as BN1 -> ReLU (xvb_bn_relu_planes) -> linear1 with BN2 folded in -> the per-segment
context-aware mask (xvb_cam_gate) -> linear_local -> y * m written into the layer's column slice of the block's
concatenation buffer (xvb_seg_gate_apply); transit3 carries out_nonlinear, xvb_stats_pool_ex takes [mean | unbiased std];
dense is xvb_small_affine.  extract_embedding applies CamPPModel's 4000-frame chunk rule (XvectorMixin.split_chunks with
even=False).  extract_embedding_batch(feats, lengths) takes a masked batch of chunks of different lengths: every layer
then stores exact zeros past each utterance's end at its own time resolution (xvb_cam_gate_lengths gives each utterance
the context of its own frames), and each row is the chunk extracted alone, bit for bit.

build_extractor() returns NativeCamPPExtractor: the same launch sequence in the C library (csrc/campplus_extractor.cu),
which also writes XVBP0001 model files for bin/xvb-extract.  XVB_CAMPP_NATIVE=0 selects CamPPExtractor, the Python driver
of the same kernels with the same embeddings bit for bit."""
import ctypes as C
import math
import os
import sys
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.native import NativeExtractor, host_lengths  # noqa: E402
from asv_subtools_b200.nnet import TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402

MAX_CHUNK = 4000      # CamPPModel.extract_embedding(max_chunk=4000)
MIN_FRAMES = 3        # T' = ceil(T / 2) >= 2 frames: the unbiased std of one frame is NaN
SEG_LEN = 100         # CAMLayer.seg_pooling's segment length
BLOCKS = ((12, 1), (24, 2), (16, 2))   # (layers, dilation) of the three CAMDenseTDNNBlocks, kernel size 3
M_CHANNELS = 32       # FCM's m_channels


def chunk_sizes(num_frames, max_chunk=MAX_CHUNK):
    """XvectorMixin.split_chunks(max_chunk, even=False) sizes (xvector.py:78-103 over get_chunksize): max_chunk-long
    chunks, then the last two re-split evenly, the first of them taking the odd frame (9000 -> [4000, 2500, 2500],
    4001 -> [2001, 2000])."""
    q, r = divmod(int(num_frames), max_chunk)
    n = q + (1 if r else 0)
    sizes = [max_chunk] * (n - 1) + [int(num_frames) - max_chunk * (n - 1)]
    if len(sizes) > 1:
        two = sizes.pop() + sizes.pop()
        sizes += [two - two // 2, two // 2]
    return sizes


def _bn_relu(channels):
    return nn.Sequential(OrderedDict([("batchnorm", nn.BatchNorm1d(channels)), ("relu", nn.ReLU())]))


class _BasicResBlock(nn.Module):
    """Post-activation residual block; stride (s, 1) strides the feature axis only."""

    def __init__(self, in_planes, planes, stride):
        super().__init__()
        self.stride = stride
        self.conv1 = nn.Conv2d(in_planes, planes, 3, stride=(stride, 1), padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, 3, stride=1, padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.shortcut = nn.Sequential()
        if stride != 1 or in_planes != planes:
            self.shortcut = nn.Sequential(nn.Conv2d(in_planes, planes, 1, stride=(stride, 1), bias=False), nn.BatchNorm2d(planes))


class _FCM(nn.Module):
    """The 2-D front end: conv1, layer1 / layer2 of two blocks each (first stride (2, 1)), conv2 stride (2, 1)."""

    def __init__(self, feat_dim, m=M_CHANNELS):
        super().__init__()
        self.conv1 = nn.Conv2d(1, m, 3, stride=1, padding=1, bias=False)
        self.bn1 = nn.BatchNorm2d(m)
        self.layer1 = nn.Sequential(_BasicResBlock(m, m, 2), _BasicResBlock(m, m, 1))
        self.layer2 = nn.Sequential(_BasicResBlock(m, m, 2), _BasicResBlock(m, m, 1))
        self.conv2 = nn.Conv2d(m, m, 3, stride=(2, 1), padding=1, bias=False)
        self.bn2 = nn.BatchNorm2d(m)
        self.out_channels = m * (feat_dim // 8)


class _TDNNBlock(nn.Module):
    """Conv1d -> BatchNorm -> ReLU (pre_norm) or, for `dense`, Conv1d -> (Identity, BatchNorm without affine)."""

    def __init__(self, cin, cout, kernel_size=1, stride=1, bias=True, dense=False):
        super().__init__()
        self.linear = nn.Conv1d(cin, cout, kernel_size, stride=stride, padding=(kernel_size - 1) // 2, bias=bias)
        if dense:
            self.nonlinear = nn.Sequential(nn.Identity(), nn.BatchNorm1d(cout, affine=False))
        else:
            self.nonlinear = nn.Sequential(nn.BatchNorm1d(cout), nn.ReLU())


class _CAMLayer(nn.Module):
    def __init__(self, bn_channels, out_channels, dilation):
        super().__init__()
        self.linear_local = nn.Conv1d(bn_channels, out_channels, 3, padding=dilation, dilation=dilation, bias=False)
        self.linear1 = nn.Conv1d(bn_channels, bn_channels // 2, 1)
        self.relu = nn.ReLU()
        self.linear2 = nn.Conv1d(bn_channels // 2, out_channels, 1)
        self.sigmoid = nn.Sigmoid()


class _DenseLayer(nn.Module):
    def __init__(self, cin, growth, bn_channels, dilation):
        super().__init__()
        self.dilation = dilation
        self.nonlinear1 = _bn_relu(cin)
        self.linear1 = nn.Conv1d(cin, bn_channels, 1, bias=False)
        self.nonlinear2 = _bn_relu(bn_channels)
        self.cam_layer = _CAMLayer(bn_channels, growth, dilation)


class _DenseBlock(nn.ModuleList):
    def __init__(self, layers, cin, growth, bn_channels, dilation):
        super().__init__()
        for i in range(layers):
            self.add_module("tdnnd%d" % (i + 1), _DenseLayer(cin + i * growth, growth, bn_channels, dilation))


class _TransitLayer(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.nonlinear = _bn_relu(cin)
        self.linear = nn.Conv1d(cin, cout, 1, bias=False)


def _unsupported(name, value, why):
    raise NotImplementedError("{}={!r} is not on the native CAM++ path: {}".format(name, value, why))


def backbone_state_dict(state_dict):
    """CamPP's keys from a CamPP or CamPPModel state_dict: `cam.` is stripped, `classifier.*` dropped.  Raises when none of
    the backbone keys is there."""
    if any(k.startswith("cam.") for k in state_dict):
        state_dict = OrderedDict((k[4:] if k.startswith("cam.") else k, v) for k, v in state_dict.items()
                                 if not k.startswith("classifier."))
    if not any(k.startswith("head.") or k.startswith("xvector.") for k in state_dict):
        raise KeyError("the state_dict carries none of the CAM++ backbone keys (head.*, xvector.* or cam.head.*, "
                       "cam.xvector.*); a Lightning checkpoint keeps them under its 'state_dict' entry")
    return state_dict


class CamPPXvector(TopVirtualNnet):
    """CAM++: FCM 2-D head, densely connected TDNN blocks with context-aware masking, statistics pooling, dense.

    `masked_chunks`, set by init: extract_embedding_batch takes lengths (a masked batch of single chunks) on this
    instance.  An instance that init did not build -- a blueprint that borrows these extraction methods (egrecho's
    EcapaXvector), or an object that was never constructed -- refuses lengths with NotImplementedError before it reads
    any configuration."""

    def init(self, inputs_dim, num_targets, embd_dim=512, init_channels=128, growth_rate=32, bn_size=4,
             memory_efficient=True):
        if inputs_dim % 8:
            raise ValueError("inputs_dim={} must be a multiple of 8: the FCM head halves F three times and reshapes to "
                             "32 * (F // 8) channels".format(inputs_dim))
        bn_channels = bn_size * growth_rate
        if growth_rate % 8:
            _unsupported("growth_rate", growth_rate, "each layer's column slice must start at a multiple of 8")
        if init_channels % 8:
            _unsupported("init_channels", init_channels, "the first block's width must be a multiple of 8")
        self.inputs_dim, self.embd_dim = inputs_dim, embd_dim
        self.masked_chunks = True
        self.growth_rate, self.bn_channels = growth_rate, bn_channels
        self.head = _FCM(inputs_dim)
        xv = OrderedDict([("tdnn", _TDNNBlock(self.head.out_channels, init_channels, 5, stride=2))])
        channels = init_channels
        self.widths = []
        for i, (layers, dilation) in enumerate(BLOCKS):
            xv["block%d" % (i + 1)] = _DenseBlock(layers, channels, growth_rate, bn_channels, dilation)
            channels += layers * growth_rate
            self.widths.append(channels)
            if i < 2 and (channels // 2) % 8:
                _unsupported("init_channels", init_channels, "transit{} gives {} channels, not a multiple of 8"
                             .format(i + 1, channels // 2))
            xv["transit%d" % (i + 1)] = _TransitLayer(channels, channels // 2)
            channels //= 2
        xv["out_nonlinear"] = _bn_relu(channels)
        xv["dense"] = _TDNNBlock(channels * 2, embd_dim, 1, bias=False, dense=True)
        self.xvector = nn.Sequential(xv)

    def load_state_dict(self, state_dict, strict=True, **kw):
        return super().load_state_dict(backbone_state_dict(state_dict), strict=strict, **kw)

    def build_extractor(self):
        dev = self.device_for_extraction()
        if os.environ.get("XVB_CAMPP_NATIVE", "1") == "0":
            return CamPPExtractor(self, dev)          # op-by-op twin of the native handle
        return NativeCamPPExtractor(self, dev)

    def _check(self, frames, feat_dim):
        if feat_dim != self.inputs_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.inputs_dim, feat_dim))
        if frames < MIN_FRAMES:
            raise ValueError("CAM++ needs at least {} frames (the unbiased std over ceil(T / 2) frames), got {}"
                             .format(MIN_FRAMES, frames))

    def extract_embedding(self, feats):
        """feats (T, F) float32 -> 1-D CPU float32 tensor with CamPPModel's 4000-frame chunk rule."""
        return self.extract_embedding_batch(torch.as_tensor(np.asarray(feats) if not isinstance(feats, torch.Tensor)
                                                            else feats)[None])[0].cpu()

    def chunk_sizes(self, num_frames):
        """The chunk lengths extract_embedding cuts a num_frames-long utterance into (CamPPModel's 4000-frame rule);
        pipeline/extract_embeddings.py --mixed-lengths cuts utterances with it before batching them."""
        return chunk_sizes(num_frames)

    def extract_embedding_batch(self, feats, lengths=None):
        """Equal-length utterances (B, T, F) float32 -> (B, embd_dim) CUDA tensor, the same arithmetic as B calls of
        extract_embedding(): each chunk position of chunk_sizes(T) runs as one batch, and the chunk embeddings are
        combined as sum_i size_i * emb_i / T in chunk order.

        lengths (B,) host ints: a masked batch of single chunks of different lengths padded to T <= 4000, row b being
        the embedding of feats[b, :lengths[b]] extracted alone (what is past it is never read).  ValueError for T > 4000
        (cut utterances with chunk_sizes first) and for a length outside [3, T], naming the first such entry."""
        if lengths is not None:
            if not getattr(self, "masked_chunks", False):
                raise NotImplementedError("{}: extract_embedding_batch(lengths=...) is for the TDNN x-vector, ResNet "
                                          "x-vector and CAM++ blueprints only".format(type(self).__name__))
            return self._extract_masked(feats, lengths)
        with torch.no_grad():
            x = torch.as_tensor(feats)
            if x.dtype != torch.float32:
                raise TypeError("extract_embedding_batch expects float32 features")
            B, T, Fd = x.shape
            self._check(T, Fd)
            x = x.to(self.device_for_extraction(), non_blocking=True)
            ex = self.extractor()
            acc, off = None, 0
            sizes = chunk_sizes(T)
            for s in sizes:
                e = ex.extract(x[:, off:off + s].contiguous())
                acc = e * s if acc is None else acc + s * e
                off += s
            return acc / sum(sizes)

    def _extract_masked(self, feats, lengths):
        with torch.no_grad():
            x = torch.as_tensor(feats)
            if x.dtype != torch.float32:
                raise TypeError("extract_embedding_batch expects float32 features")
            B, T, Fd = x.shape
            if Fd != self.inputs_dim:
                raise ValueError("expected feature dim {}, got {}".format(self.inputs_dim, Fd))
            if T > MAX_CHUNK:
                raise ValueError("extract_embedding_batch(lengths=...) takes one chunk per row, T <= {}, got T={}: cut the "
                                 "utterances with chunk_sizes first".format(MAX_CHUNK, T))
            lens = _checked_lengths(lengths, B, T)
            x = x.to(self.device_for_extraction(), non_blocking=True).contiguous()
            return self.extractor().extract(x, lens)


def _checked_lengths(lengths, b, t):
    """Host int32 (B,) lengths of a masked CAM++ batch; ValueError naming the first entry outside [MIN_FRAMES, t]."""
    lens = host_lengths(lengths, b)
    bad = np.flatnonzero((lens < MIN_FRAMES) | (lens > t))
    if bad.size:
        raise ValueError("lengths[{}]={} outside [{}, T={}]: a CAM++ chunk needs at least {} frames".format(
            bad[0], lens[bad[0]], MIN_FRAMES, t, MIN_FRAMES))
    return lens


def tdnn_im2col_weight(weight, channels, freq):
    """`tdnn`'s Conv1d weight (Cout, channels * freq, 5) in the reference's input order c * freq + f -> (Cout, 5 * freq *
    channels) with K index k * freq * channels + f * channels + c: the window of 5 consecutive frames of the (B, T, F'',
    C) head output as the layer kernel's im2col view reads it."""
    cout = weight.shape[0]
    w = weight.reshape(cout, channels, freq, -1)          # (o, c, f, k)
    return w.permute(0, 3, 2, 1).reshape(cout, -1)        # (o, k, f, c)


def _fold(w, bn, bias=None):
    """Weight (Cout, ...) and bias of conv -> eval BatchNorm as one affine: (scale * w, scale * bias + shift)."""
    s, t = fold_batchnorm(bn)
    s, t = torch.from_numpy(s).to(w.device), torch.from_numpy(t).to(w.device)
    b = t if bias is None else s * bias.detach().float() + t
    return w.detach().float() * s.view(-1, *([1] * (w.dim() - 1))), b


class CamPPExtractor:
    """Folded weights on one device + the launch sequence of CamPP.forward for one chunk per utterance (all utterances of
    a call have the same length, or a masked batch gives each its own), driven from Python over a workspace reused while
    the batch shape stays the same.  The weights are the records and configuration the native handle takes
    (native_records, native_config), each reshaped back from its (rows, cols) form."""

    TAKES_LENGTHS = True

    def __init__(self, m, device):
        from asv_subtools_b200._lib import RELU
        recs = {r[0]: r[1:] for r in native_records(m)}
        cfg = native_config(m)
        self.device, self.feat_dim, self.embed_dim = device, cfg["feat_dim"], cfg["embd_dim"]
        self.f8 = self.feat_dim // 8
        self.g, self.bn_ch = cfg["growth_rate"], cfg["bn_size"] * cfg["growth_rate"]

        def conv(name, cin):
            """(fp32 weight (Cout, Cin, k, k), scale, shift) of a bias-free Conv2d record with its folded BatchNorm."""
            w, _, sc, sh, _, _ = recs[name]
            k = math.isqrt(w.shape[1] // cin)
            return ops.to_device(w.reshape(w.shape[0], cin, k, k), device), ops.to_device(sc, device), ops.to_device(sh, device)

        def packed(name):
            w, sc, sh = conv(name, M_CHANNELS)
            return ops.pack_conv2d_weight(w), sc, sh

        self.conv1 = conv("head.conv1", 1)      # fp32 as stored: xvb_conv2d_head
        self.res_blocks = []
        for li in (1, 2):
            for i in range(2):
                p = "head.layer{}.{}.".format(li, i)
                sc = packed(p + "shortcut.0") if p + "shortcut.0" in recs else None
                self.res_blocks.append((2 if i == 0 else 1, packed(p + "conv1"), packed(p + "conv2"), sc))
        self.conv2 = packed("head.conv2")
        w, b = recs["xvector.tdnn.linear"][:2]
        self.tdnn = ops.PackedAffine(w, device, bias=b, relu=True)
        self.blocks, self.transits, self.widths = [], [], []
        for i, (layers, dilation) in enumerate(BLOCKS):
            L = []
            for li in range(layers):
                p = "xvector.block{}.tdnnd{}.".format(i + 1, li + 1)
                q = p + "cam_layer."
                s1, t1 = recs[p + "nonlinear1"][2:4]
                w1, b1 = recs[p + "linear1"][:2]
                local = recs[q + "linear_local"][0]
                L.append({"s1": ops.to_device(s1, device), "t1": ops.to_device(t1, device),
                          "lin1": ops.PackedAffine(w1, device, bias=b1, relu=True),
                          "local": ops.PackedAffine(local.reshape(local.shape[0], self.bn_ch, -1), device,
                                                    (-dilation, 0, dilation)),
                          "gate": tuple(ops.to_device(a.reshape(a.shape[0], -1), device)
                                        for name in ("linear1", "linear2") for a in recs[q + name][:2])})
            self.blocks.append(L)
            p = "xvector.transit{}.".format(i + 1)
            s, sh = recs[p + "nonlinear"][2:4]
            w, b, _, _, flags, _ = recs[p + "linear"]
            self.transits.append((ops.to_device(s, device), ops.to_device(sh, device),
                                  ops.PackedAffine(w, device, bias=b, relu=bool(flags & RELU))))
            self.widths.append(s.shape[0])
        w, _, ds, dt, _, _ = recs["xvector.dense.linear"]
        self.dense = (ops.to_device(w, device), ops.to_device(ds, device), ops.to_device(dt, device))
        self._ws_key, self._ws = None, None
        self.last_launches = 0

    def _workspace(self, B, T):
        if self._ws_key != (B, T):
            self._ws = None                 # release the old shape's buffers first
            P, dev, m = ops.SplitPlanes, self.device, M_CHANNELS
            T2 = (T + 1) // 2
            F, ws = self.feat_dim, {}
            ws["x0"] = P.empty((B, T, F, m), dev)
            for j, (stride, _, _, sc) in enumerate(self.res_blocks):
                F = (F + 1) // 2 if stride == 2 else F
                ws["a%d" % j], ws["o%d" % j] = P.empty((B, T, F, m), dev), P.empty((B, T, F, m), dev)
                ws["s%d" % j] = P.empty((B, T, F, m), dev) if sc is not None else None
            ws["c2"] = P.empty((B, T, self.f8, m), dev)
            row = self.f8 * m
            # 2 zero frames before and after every utterance: F.pad of the stride-2 conv, written once
            ws["pad"] = P(torch.zeros(B, T + 4, row, dtype=torch.bfloat16, device=dev),
                          torch.zeros(B, T + 4, row, dtype=torch.bfloat16, device=dev), row)
            ws["bufs"] = [P.empty((B, T2, w), dev) for w in self.widths]
            ws["pre"] = P.empty((B, T2, max(self.widths)), dev)
            ws["h"] = P.empty((B, T2, self.bn_ch), dev)
            ws["z"] = P.empty((B, T2, self.g), dev)
            ws["pool_in"] = torch.empty(B, T2, self.transits[-1][2].cout, dtype=torch.float32, device=dev)
            ws["gate"] = torch.empty(B, (T2 + SEG_LEN - 1) // SEG_LEN, self.g, dtype=torch.float32, device=dev)
            self._ws_key, self._ws = (B, T), ws
        return self._ws

    def extract(self, feats, lengths=None):
        """feats (B, T, F) fp32 CUDA (one chunk per utterance) -> (B, embd_dim) fp32 CUDA, asynchronous on the current
        stream.  lengths (B,) host ints, 3 <= lengths[b] <= T: a masked batch as xvb_campp_extract_lengths runs it, row b
        being feats[b, :lengths[b]] extracted alone (every length equal to T: the unmasked sequence).  Every workspace
        tensor then holds exact zeros past each utterance's length at its own resolution, except `pre`, whose only
        consumers are 1x1 layers that store zeros there themselves."""
        B, T, Fd = feats.shape
        if Fd != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, Fd))
        if T < MIN_FRAMES:
            raise ValueError("CAM++ needs at least {} frames, got {}".format(MIN_FRAMES, T))
        l1 = l2 = None    # a masked batch's lengths at the head's resolution and after the stride-2 tdnn, ceil(L / 2)
        if lengths is not None:
            lens = _checked_lengths(lengths, B, T)
            if (lens != T).any():
                table = torch.from_numpy(np.stack([lens, (lens + 1) // 2])).to(feats.device)
                l1, l2 = table[0], table[1]
        feats = feats.contiguous()
        ws = self._workspace(B, T)
        P, m = ops.SplitPlanes, M_CHANNELS
        ops.conv2d_head(feats, *self.conv1, ws["x0"], lengths=l1)
        n = 1
        x = ws["x0"]
        for j, (stride, c1, c2, sc) in enumerate(self.res_blocks):
            res = x
            if sc is not None:
                res = ws["s%d" % j]
                ops.conv2d(x, sc[0], m, 1, stride, sc[1], sc[2], y=res, stride_t=1, lengths=l1)
                n += 1
            ops.conv2d(x, c1[0], m, 3, stride, c1[1], c1[2], relu=True, y=ws["a%d" % j], stride_t=1, lengths=l1)
            ops.conv2d(ws["a%d" % j], c2[0], m, 3, 1, c2[1], c2[2], res=res, relu=True, y=ws["o%d" % j], lengths=l1)
            n += 2
            x = ws["o%d" % j]
        c = self.conv2
        ops.conv2d(x, c[0], m, 3, 2, c[1], c[2], relu=True, y=ws["c2"], stride_t=1, lengths=l1)
        # the head output into the time-padded copy: one row of T * F'' * C elements per utterance
        row = self.f8 * m
        pad, src = ws["pad"], ws["c2"]
        ops.copy_planes(P(src.hi.view(B, 1, T * row), src.lo.view(B, 1, T * row), T * row),
                        P(pad.hi.view(B, 1, -1)[..., 2 * row:(T + 2) * row], pad.lo.view(B, 1, -1)[..., 2 * row:(T + 2) * row],
                          T * row))
        n += 4
        # tdnn: Conv1d(k = 5, stride 2, padding 2) as a 1-tap layer over 5-frame windows that start every 2 frames
        T2 = (T + 1) // 2
        win = P(pad.hi.as_strided((B, T2, 2 * row), ((T + 4) * row, 2 * row, 1)),
                pad.lo.as_strided((B, T2, 2 * row), ((T + 4) * row, 2 * row, 1)), 5 * row)
        bufs, pre = ws["bufs"], ws["pre"]
        self.tdnn.run(win, y=bufs[0].slice(0, self.tdnn.cout), x_batch_stride=(T + 4) * row, lengths=l2)
        n += 1
        c0 = self.tdnn.cout
        h, z, gate = ws["h"], ws["z"], ws["gate"]
        for bi, layers in enumerate(self.blocks):
            buf = bufs[bi]
            for li, L in enumerate(layers):
                cin = c0 + li * self.g
                xin = buf.slice(0, cin)
                pv = pre.slice(0, cin)
                ops.bn_relu_planes(xin, L["s1"], L["t1"], pv)
                L["lin1"].run(pv, y=h, lengths=l2)
                ops.cam_gate(h, *L["gate"], seg_len=SEG_LEN, out=gate, lengths=l2)
                L["local"].run(h, y=z, lengths=l2)
                ops.seg_gate_apply(z, gate, SEG_LEN, buf.slice(cin, cin + self.g))
                n += 5
            s, t, lin = self.transits[bi]
            width = self.widths[bi]
            pv = pre.slice(0, width)
            ops.bn_relu_planes(buf if buf.channels == width else buf.slice(0, width), s, t, pv)
            n += 1
            if bi + 1 < len(self.blocks):
                lin.run(pv, y=bufs[bi + 1].slice(0, lin.cout), lengths=l2)
                n += 1
                c0 = lin.cout
            else:
                # out_nonlinear in the epilogue, then [mean | unbiased std] over T' (no eps) per utterance.  Not the fused
                # pooling epilogue: its time blocking follows the batch shape, so a batch would not reproduce
                # per-utterance calls bit for bit; the fp32 round trip costs ~80 MB of traffic at 128 x 300.
                lin.run(pv, y_f32=ws["pool_in"], lengths=l2)
                stats = ops.stats_pool_ex(ws["pool_in"], 0.0, 1, lengths=l2)
                n += 2
        wd, sd, td = self.dense
        emb = ops.small_affine(stats, wd, bn_scale=sd, bn_shift=td)
        self.last_launches = n + 1
        return emb

    def close(self):
        self._ws_key, self._ws = None, None


def native_config(m):
    """xvb_campp_config_t fields of a CamPPXvector."""
    return dict(feat_dim=m.inputs_dim, embd_dim=m.embd_dim, init_channels=m.xvector.tdnn.linear.weight.shape[0],
                growth_rate=m.growth_rate, bn_size=m.bn_channels // m.growth_rate)


def native_records(m):
    """(name, w, bias, scale, shift, flags, keys) records for xvb_campp_set_layer and CamPPExtractor, after the hand-over
    folds: every BatchNorm folded to scale / shift or into the preceding conv, the `tdnn` weight in the im2col column
    order, out_nonlinear folded into transit3.  `keys` are the state_dict entries the record carries."""
    from asv_subtools_b200._lib import BN, RELU
    f = lambda t: None if t is None else (t.detach().float().cpu().numpy() if isinstance(t, torch.Tensor) else t)  # noqa: E731
    out = []

    def keys_of(mod, name):
        return [name + "." + k for k in mod.state_dict()]

    def conv(name, c, bn, bn_name, flags):
        s, t = fold_batchnorm(bn)
        out.append((name, f(c.weight).reshape(c.weight.shape[0], -1), None, s, t, flags,
                    keys_of(c, name) + keys_of(bn, bn_name)))

    def bn_relu(name, bn):
        s, t = fold_batchnorm(bn)
        out.append((name, None, None, s, t, BN | RELU, keys_of(bn, name + ".batchnorm")))

    def folded(name, c, bn, bn_name, bias=None, extra=()):
        w, b = _fold(c.weight.detach().float().cpu(), bn, bias)
        out.append((name, f(w).reshape(w.shape[0], -1), f(b), None, None, RELU,
                    keys_of(c, name) + keys_of(bn, bn_name) + list(extra)))

    h = m.head
    conv("head.conv1", h.conv1, h.bn1, "head.bn1", BN | RELU)
    for li, layer in enumerate((h.layer1, h.layer2)):
        for i, blk in enumerate(layer):
            p = "head.layer{}.{}.".format(li + 1, i)
            conv(p + "conv1", blk.conv1, blk.bn1, p + "bn1", BN | RELU)
            conv(p + "conv2", blk.conv2, blk.bn2, p + "bn2", BN | RELU)
            if len(blk.shortcut):
                conv(p + "shortcut.0", blk.shortcut[0], blk.shortcut[1], p + "shortcut.1", BN)
    conv("head.conv2", h.conv2, h.bn2, "head.bn2", BN | RELU)
    xv = m.xvector
    lin = xv.tdnn.linear
    w, b = _fold(tdnn_im2col_weight(lin.weight.detach().float().cpu(), M_CHANNELS, m.inputs_dim // 8), xv.tdnn.nonlinear[0],
                 lin.bias.detach().float().cpu())
    out.append(("xvector.tdnn.linear", f(w), f(b), None, None, RELU,
                keys_of(lin, "xvector.tdnn.linear") + keys_of(xv.tdnn.nonlinear[0], "xvector.tdnn.nonlinear.0")))
    for bi in range(len(BLOCKS)):
        for li, layer in enumerate(getattr(xv, "block%d" % (bi + 1))):
            p = "xvector.block{}.tdnnd{}.".format(bi + 1, li + 1)
            bn_relu(p + "nonlinear1", layer.nonlinear1.batchnorm)
            folded(p + "linear1", layer.linear1, layer.nonlinear2.batchnorm, p + "nonlinear2.batchnorm")
            cam = layer.cam_layer
            q = p + "cam_layer."
            out.append((q + "linear_local", f(cam.linear_local.weight).reshape(cam.linear_local.weight.shape[0], -1), None, None,
                        None, 0, keys_of(cam.linear_local, q + "linear_local")))
            for name in ("linear1", "linear2"):
                c = getattr(cam, name)
                out.append((q + name, f(c.weight).reshape(c.weight.shape[0], -1), f(c.bias), None, None, 0, keys_of(c, q + name)))
        tr = getattr(xv, "transit%d" % (bi + 1))
        p = "xvector.transit{}.".format(bi + 1)
        bn_relu(p + "nonlinear", tr.nonlinear.batchnorm)
        if bi + 1 < len(BLOCKS):
            out.append((p + "linear", f(tr.linear.weight).reshape(tr.linear.weight.shape[0], -1), None, None, None, 0,
                        keys_of(tr.linear, p + "linear")))
        else:
            folded(p + "linear", tr.linear, xv.out_nonlinear.batchnorm, "xvector.out_nonlinear.batchnorm")
    ds, dt = fold_batchnorm(xv.dense.nonlinear[1])
    out.append(("xvector.dense.linear", f(xv.dense.linear.weight).reshape(m.embd_dim, -1), None, ds, dt, BN,
                keys_of(xv.dense.linear, "xvector.dense.linear") + keys_of(xv.dense.nonlinear[1], "xvector.dense.nonlinear.1")))
    return out


class NativeCamPPExtractor(NativeExtractor):
    """xvb_campp_t: packed weights, workspace and the whole launch sequence of CamPPExtractor in the C library, on the
    device that is current when it is built (or loaded from an XVBP0001 file)."""

    PREFIX = "campp"
    TAKES_LENGTHS = True

    def _create_args(self, m):
        from asv_subtools_b200._lib import CamPPConfig
        return (C.byref(CamPPConfig(**native_config(m))),)

    def _layers(self, m):
        for name, w, b, scale, shift, flags, _ in native_records(m):
            rows = (w if w is not None else scale).shape[0]
            yield name, (rows, w.shape[1] if w is not None else 0), (w, b, scale, shift), flags

    def _input(self, feats):
        if not (isinstance(feats, torch.Tensor) and feats.is_cuda and feats.dtype == torch.float32 and feats.dim() == 3):
            raise TypeError("feats must be a (B, T, F) CUDA float32 tensor")
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        return feats.contiguous()
