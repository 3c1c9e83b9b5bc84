"""torch-CPU restatement of the reference's CAM++ x-vector at extraction (subtools2/egrecho/models/campplus/campplus.py
CamPP.forward :355-359, model.py CamPPModel.extract_embedding :73-96 with XvectorMixin.split_chunks, models/architecture/
speaker/xvector.py:47-157), the golden cases of tests/golden/make_golden_campplus.py, and the chunk plan.

Written from the reference's arithmetic, in its operation order, over a backbone state_dict (`head.*`, `xvector.*`):
the FCM head (conv1 -> BN -> ReLU, two BasicResBlocks per layer whose first block strides the feature axis by 2, conv2
with stride (2, 1)), the reshape to (B, C * F / 8, T) with channel c * (F / 8) + f, the stride-2 `tdnn`, three densely
connected CAM blocks with their transit layers, out_nonlinear, [mean | unbiased std] and the dense layer (1x1 conv,
BatchNorm without affine).  The seeded state_dict rule is conformer_oracle's."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from conformer_oracle import seeded_state_dict  # noqa: E402,F401  (shared with the golden generator)

MAX_CHUNK = 4000          # CamPPModel.extract_embedding(max_chunk=4000), model.py:73
SEG_LEN = 100             # CAMLayer.seg_pooling(seg_len=100), campplus.py:164
BLOCKS = ((12, 1), (24, 2), (16, 2))   # (layers, dilation) of CamPP.__init__, campplus.py:327-329

DEFAULT = dict(inputs_dim=80, embd_dim=512, init_channels=128, growth_rate=32, bn_size=4)
SMALL = dict(inputs_dim=40, embd_dim=192, init_channels=64, growth_rate=32, bn_size=2)

# name -> (config, frame counts through CamPP.forward, frame counts through CamPPModel.extract_embedding, sd seed,
# feature seed)
CASES = {
    "default": (DEFAULT, (300, 200, 201, 37, 3), (4001, 9000), 31, 800),
    "small": (SMALL, (150, 4), (), 32, 850),
}
# T values whose split_chunks(max_chunk=4000, even=False) sizes the fixture records
SPLIT_T = (1, 3, 3999, 4000, 4001, 7999, 8000, 8001, 9000, 12000, 12001, 20000)


def utterances(n, frames, feat_dim, seed):
    """(n, frames, feat_dim) fp32 test features: oracle.nnet's synthetic frames plus a per-utterance offset of 2 N(0, 1)
    per dimension, so that utterances differ after pooling by more than the dense layer's BatchNorm shift."""
    from oracle import nnet as onn
    x = torch.from_numpy(onn.synthetic_feats(n, frames, feat_dim, seed))
    g = torch.Generator().manual_seed(seed)
    return (x + 2.0 * torch.randn(n, 1, feat_dim, generator=g)).contiguous()


def chunk_sizes(num_frames, max_chunk=MAX_CHUNK):
    """XvectorMixin.split_chunks(even=False) sizes: get_chunksize's max_chunk-long chunks and a shorter last one, then
    the last two chunks re-split evenly (the first of the two takes the odd frame)."""
    q, r = divmod(num_frames, max_chunk)
    n = q + (1 if r else 0)
    sizes = [max_chunk] * (n - 1) + [num_frames - max_chunk * (n - 1)]
    if len(sizes) > 1:
        two = sizes.pop() + sizes.pop()
        sizes += [two - two // 2, two // 2]
    return sizes


def _bn(x, sd, p, eps=1e-5):
    return F.batch_norm(x, sd[p + "running_mean"], sd[p + "running_var"], sd.get(p + "weight"), sd.get(p + "bias"),
                        False, 0.0, eps)


def _res_block(x, sd, p, stride):
    out = F.relu(_bn(F.conv2d(x, sd[p + "conv1.weight"], stride=(stride, 1), padding=1), sd, p + "bn1."))
    out = _bn(F.conv2d(out, sd[p + "conv2.weight"], padding=1), sd, p + "bn2.")
    if p + "shortcut.0.weight" in sd:
        out = out + _bn(F.conv2d(x, sd[p + "shortcut.0.weight"], stride=(stride, 1)), sd, p + "shortcut.1.")
    else:
        out = out + x
    return F.relu(out)


def seg_pooling(h, seg_len=SEG_LEN):
    """avg_pool1d(kernel = stride = seg_len, ceil_mode=True) repeated back over each segment and cut to T: the partial
    last segment is a mean over its valid frames."""
    seg = F.avg_pool1d(h, kernel_size=seg_len, stride=seg_len, ceil_mode=True)
    return seg.unsqueeze(-1).expand(*seg.shape, seg_len).reshape(h.shape[0], h.shape[1], -1)[..., :h.shape[-1]]


def forward(sd, feats):
    """CamPP.forward: feats (B, T, F) fp32 -> (B, embd_dim)."""
    x = feats.permute(0, 2, 1).unsqueeze(1)
    out = F.relu(_bn(F.conv2d(x, sd["head.conv1.weight"], padding=1), sd, "head.bn1."))
    for layer in (1, 2):
        for i, stride in enumerate((2, 1)):
            out = _res_block(out, sd, "head.layer{}.{}.".format(layer, i), stride)
    out = F.relu(_bn(F.conv2d(out, sd["head.conv2.weight"], stride=(2, 1), padding=1), sd, "head.bn2."))
    out = out.reshape(out.shape[0], out.shape[1] * out.shape[2], out.shape[3])
    x = F.conv1d(out, sd["xvector.tdnn.linear.weight"], sd["xvector.tdnn.linear.bias"], stride=2, padding=2)
    x = F.relu(_bn(x, sd, "xvector.tdnn.nonlinear.0."))
    for bi, (layers, d) in enumerate(BLOCKS):
        for li in range(layers):
            p = "xvector.block{}.tdnnd{}.".format(bi + 1, li + 1)
            h = F.conv1d(F.relu(_bn(x, sd, p + "nonlinear1.batchnorm.")), sd[p + "linear1.weight"])
            h = F.relu(_bn(h, sd, p + "nonlinear2.batchnorm."))
            y = F.conv1d(h, sd[p + "cam_layer.linear_local.weight"], padding=d, dilation=d)
            ctx = h.mean(-1, keepdim=True) + seg_pooling(h)
            ctx = F.relu(F.conv1d(ctx, sd[p + "cam_layer.linear1.weight"], sd[p + "cam_layer.linear1.bias"]))
            m = torch.sigmoid(F.conv1d(ctx, sd[p + "cam_layer.linear2.weight"], sd[p + "cam_layer.linear2.bias"]))
            x = torch.cat([x, y * m], dim=1)
        p = "xvector.transit{}.".format(bi + 1)
        x = F.conv1d(F.relu(_bn(x, sd, p + "nonlinear.batchnorm.")), sd[p + "linear.weight"])
    x = F.relu(_bn(x, sd, "xvector.out_nonlinear.batchnorm."))
    stats = torch.cat([x.mean(dim=-1), x.std(dim=-1, unbiased=True)], dim=-1)
    e = F.conv1d(stats.unsqueeze(2), sd["xvector.dense.linear.weight"])
    return _bn(e, sd, "xvector.dense.nonlinear.1.").squeeze(2)


def extract_embedding(sd, feats):
    """CamPPModel.extract_embedding: feats (B, T, F) -> (B, embd_dim), sum_i size_i * emb_i / sum_i size_i over the
    chunks of chunk_sizes(T), accumulated in chunk order."""
    sizes = chunk_sizes(feats.shape[1])
    acc, off = None, 0
    for s in sizes:
        e = forward(sd, feats[:, off:off + s])
        acc = e * s if acc is None else acc + s * e
        off += s
    return acc / sum(sizes)


def backbone_keys(sd):
    return {k: v for k, v in sd.items() if k.startswith("head.") or k.startswith("xvector.")}
