# -*- coding:utf-8 -*-
"""Factored (F-TDNN) x-vector blueprint for the B200 path -- drop-in for pytorch/model/factored_xvector.py
(Xvector.init :15-47, extract_embedding :99-122): same constructor keywords and state_dict keys
(layer01, layer02..09 = FTdnnBlock {factor, affine, bn}, layer10, embedding1/2).  Every contraction runs on
the wgmma layer kernel; the skip concatenations cat(x_2, x_4) / cat(x_4, x_6, x_8) are channel slices of two
wider buffers written in place, the bypass `out += 0.66 * identity` (components.py:208-210) is the existing
fused multiply-add kernel with a constant gate, and layer10 pools over time in its epilogue."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200.native import device_lengths  # noqa: E402
from asv_subtools_b200.nnet import FTdnnBlock, ReluBatchNormTdnnLayer, StatisticsPooling, TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import fold_batchnorm  # noqa: E402


class Xvector(TopVirtualNnet):
    """A factored x-vector framework."""

    def init(self, inputs_dim, num_targets, nonlinearity="relu", semi_orth=True, embd_dim=512, aug_dropout=0.2,
             training=False, extracted_embedding="far", jit_compile=False):
        if nonlinearity != "relu":
            raise NotImplementedError("B200 path implements the reference default nonlinearity='relu'")
        self.inputs_dim, self.embd_dim = inputs_dim, embd_dim
        self.semi_orth = semi_orth
        self.extracted_embedding = extracted_embedding
        self.layer01 = ReluBatchNormTdnnLayer(inputs_dim, 512, [-2, -1, 0, 1, 2], nonlinearity=nonlinearity)
        self.layer02 = FTdnnBlock(512, 1024, 256, 2, 0)
        self.layer03 = FTdnnBlock(1024, 1024, 256, 0, 0.66)
        self.layer04 = FTdnnBlock(1024, 1024, 256, 3, 0.66)
        self.layer05 = FTdnnBlock(1024, 1024, 256, 0, 0.66)
        self.layer06 = FTdnnBlock(1024, 1024, 256, 3, 0.66)
        self.layer07 = FTdnnBlock(2048, 1024, 256, 3, 0)
        self.layer08 = FTdnnBlock(1024, 1024, 256, 3, 0.66)
        self.layer09 = FTdnnBlock(3072, 1024, 256, 0, 0)
        self.layer10 = ReluBatchNormTdnnLayer(1024, 2048, nonlinearity=nonlinearity)
        self.stats = StatisticsPooling(2048, stddev=True)
        self.embedding1 = ReluBatchNormTdnnLayer(self.stats.get_output_dim(), embd_dim, nonlinearity=nonlinearity)
        self.embedding2 = ReluBatchNormTdnnLayer(embd_dim, embd_dim, nonlinearity=nonlinearity)
        self.transform_keys = ["layer01", "layer02", "layer03", "layer04", "layer05", "layer06", "layer07", "layer08",
                               "layer09", "layer10", "stats", "embedding1", "embedding2"]

    def build_extractor(self):
        if self.extracted_embedding not in ("far", "near"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        return FtdnnExtractor(self, self.device_for_extraction())


def _affine(affine, device, bn=None, relu=False):
    """A TdnnAffine with its weight as stored, [ReLU and] the eval BatchNorm bn folded in, as an ops.PackedAffine."""
    return ops.PackedAffine(affine.weight, device, affine.context, affine.bias, *fold_batchnorm(bn), relu=relu)


class FtdnnExtractor:
    """Packed weights on one device + the launch sequence of Xvector.extract_embedding (factored_xvector.py:99-122).
    Takes masked batches of utterances of different lengths (TAKES_LENGTHS)."""

    TAKES_LENGTHS = True

    def __init__(self, m, device):
        self.feat_dim, self.embed_dim = m.inputs_dim, m.embd_dim
        self.l01 = _affine(m.layer01.affine, device, m.layer01.batchnorm, m.layer01.relu)
        self.blocks = {}
        for i in range(2, 10):
            blk = getattr(m, "layer{:02d}".format(i))
            self.blocks[i] = (_affine(blk.factor, device), _affine(blk.affine, device, blk.bn, relu=True), blk.bypass_scale)
        self.l10 = _affine(m.layer10.affine, device, m.layer10.batchnorm, m.layer10.relu)
        self.eps = m.stats.eps
        self.far = m.extracted_embedding == "far"
        e1 = m.embedding1
        self.e1 = _affine(e1.affine, device) if self.far else _affine(e1.affine, device, e1.batchnorm, e1.relu)
        self.e2 = None if self.far else _affine(m.embedding2.affine, device)
        self.last_launches = 0

    def _block(self, i, x, out, tmp256, tmpo, lens=None):
        """FTdnnBlock i: x -> out (SplitPlanes views).  tmp256 / tmpo: scratch planes (B,T,256) / (B,T,1024).  lens: the
        device lengths of a masked batch; the bypass sum needs none, both of its inputs being zero past each end."""
        factor, affine, bypass = self.blocks[i]
        factor.run(x, y=tmp256, lengths=lens)
        if bypass == 0:
            affine.run(tmp256, y=out, lengths=lens)
        else:
            affine.run(tmp256, y=tmpo, lengths=lens)
            gate = self._gate(bypass, x.hi.shape[0], x.channels, x.hi.device)
            ops.se_apply(x, tmpo, gate, out)              # out = x * bypass + bn(relu(affine(factor(x))))

    def _gate(self, value, b, c, dev):
        key = (value, b, c)
        if getattr(self, "_gate_key", None) != key:
            self._gate_key, self._gate_t = key, torch.full((b, c), float(value), dtype=torch.float32, device=dev)
        return self._gate_t

    def extract(self, feats, lengths=None):
        """feats (B, T, F) fp32 CUDA -> (B, embed_dim) fp32 CUDA, asynchronous on the current stream.  lengths (B,) host
        ints, 1 <= lengths[b] <= T: a masked batch, row b being feats[b, :lengths[b]] extracted alone; layer10 then
        writes fp32 frames and the standalone pooling reduces each utterance's own (the fused pooling epilogue takes
        equal lengths only).  Every length equal to T runs the unmasked sequence."""
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        B, T, _ = feats.shape
        dev, P = feats.device, ops.SplitPlanes
        lens = None if lengths is None else device_lengths(lengths, B, T, dev)
        ld = (self.feat_dim + 7) // 8 * 8
        xin = ops.split_f32(feats, ld=ld) if lens is None else ops.split_frames(feats.contiguous(), ld=ld, lengths=lens)
        x1 = P.empty((B, T, 512), dev)
        self.l01.run(xin, y=x1, lengths=lens)
        t256, to = P.empty((B, T, 256), dev), P.empty((B, T, 1024), dev)
        cat7, cat9 = P.empty((B, T, 2048), dev), P.empty((B, T, 3072), dev)      # [x_2 | x_4], [x_4 | x_6 | x_8]
        x3, x5, x7, x9 = (P.empty((B, T, 1024), dev) for _ in range(4))
        x2, x4 = cat7.slice(0, 1024), cat7.slice(1024, 2048)
        self._block(2, x1, x2, t256, to, lens)
        self._block(3, x2, x3, t256, to, lens)
        self._block(4, x3, x4, t256, to, lens)
        ops.copy_planes(x4, cat9.slice(0, 1024))
        self._block(5, x3, x5, t256, to, lens)
        self._block(6, x5, cat9.slice(1024, 2048), t256, to, lens)
        self._block(7, cat7, x7, t256, to, lens)
        self._block(8, x7, cat9.slice(2048, 3072), t256, to, lens)
        self._block(9, cat9, x9, t256, to, lens)
        if lens is None:
            _, stats = ops.fused_pool_layer(x9, self.l10.w, self.l10.cout, self.l10.context, self.l10.bias, self.l10.scale,
                                            self.l10.shift, relu=self.l10.relu, eps=self.eps, planes=True)
        else:
            x10 = torch.empty(B, T, self.l10.cout, dtype=torch.float32, device=dev)
            self.l10.run(x9, y_f32=x10, lengths=lens)
            _, stats = ops.stats_pool_ex(x10, self.eps, 0, planes=True, lengths=lens)
        emb = torch.empty(B, 1, self.embed_dim, dtype=torch.float32, device=dev)
        if self.far:
            self.e1.run(stats, y_f32=emb)
        else:
            h = P.empty((B, 1, self.e1.cout), dev)
            self.e1.run(stats, y=h)
            self.e2.run(h, y_f32=emb)
        return emb.view(B, self.embed_dim)

    def close(self):
        pass


if __name__ == "__main__":
    print(Xvector(23, 1211))
