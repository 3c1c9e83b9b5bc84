# -*- coding:utf-8 -*-
"""Conformer x-vector blueprint for the native path -- drop-in for pytorch/model/transformer_xvector.py
(TransformerXvector.init :93-244, extract_embedding :321-346) with the Conformer encoder of
pytorch/libs/nnet/transformer/ (ConformerEncoder encoder.py:536-682, ConformerEncoderLayer encoder_layer.py:159-335).

Same file name, class name, constructor signature and defaults (transformer_params merged with unknown keys kept, as
assign_params_dict(support_unknow=True) does), creation string and state_dict keys for training=False; like the other
blueprints, the training-only loss is not built, so its keys are left to load_state_dict(strict=False).

Supported: transformer_type 'conformer' with input_layer 'conv2d' (4x subsampling) or 'conv2d2' (2x,
SVConv2dSubsampling2, subsampling.py:365-415); pos_enc_type 'rot_pos' (rotary_value either way),
'abs_pos' or 'no_pos'; attention norm 'softmax' or 'softmax_plus'; the convolution module with 'layer_norm' or
'batch_norm'; activation 'swish' or 'relu'; transform_out with a LayerNorm (ln_replace) or a BatchNorm; the
ecpa-attentive pooling with stddev; fc1 on or off (LayerNorm with or without affine); positions far / near_affine / near.
Every other option raises NotImplementedError naming it.

At extraction every contraction runs on the wgmma layer kernel with split-plane numerics: Q/K/V as
one GEMM over the concatenated weights, linear_out, the feed-forward linears (swish / ReLU in the epilogue), the
pointwise convs, the subsampling Linear (its input columns permuted from the reference's c * F'' + f to the f * C + c
order of the conv output, x * sqrt(d) applied after the bias as the epilogue's scale), transform_out, the pooling convs
and fc1 / fc2.  The second subsampling conv runs on the 2-D conv kernel without padding (xvb_conv2d_valid); the first
one, the residual + LayerNorm steps, the attention and the convolution module's middle run on the kernels of
csrc/conformer.cu (the 2x subsampling's first conv with feature stride 1, its second conv at stride 1).  The residual
stream stays fp32.

build_extractor() hands the weights to the native handle (NativeConformerExtractor over xvb_conformer_*, csrc/
conformer_extractor.cu), which runs the whole launch sequence in C++ and also writes XVBC0001 model files for
bin/xvb-extract.  XVB_CONFORMER_NATIVE=0 selects ConformerExtractor, the Python driver of the same kernels with the same
arguments in the same order, kept as the A/B and profiling twin; the two give bit-identical embeddings.

extract_embedding keeps the reference's maxChunk = 300 chunk rule (for_extract_embedding, framework.py:12-55): an
utterance is cut into num_split = ceil(T / 300) chunks, each chunk is extracted on its own and the embeddings are
averaged weighted by chunk length.  extract_embedding_batch applies the same rule to a batch of equal-length
utterances with two stack runs (all full chunks, then all last chunks).  extract_embedding_batch(feats, lengths) takes a
masked batch of single chunks of different lengths (cut by chunk_sizes first): the head conv, every frame-level linear,
the attention and the attentive pooling then run at each utterance's own length, and each row is its chunk extracted
alone, bit for bit."""
import copy
import ctypes as C
import math
import os
import sys

import numpy as np
import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from asv_subtools_b200 import ops  # noqa: E402
from asv_subtools_b200._lib import ACT_NONE, ACT_RELU, ACT_SWISH, ACT_TANH, BN, RELU, SWISH  # noqa: E402
from asv_subtools_b200.nnet import TopVirtualNnet  # noqa: E402
from asv_subtools_b200.nnet.components import TdnnAffine, fold_batchnorm  # noqa: E402
from asv_subtools_b200.native import NativeExtractor, host_lengths  # noqa: E402
from asv_subtools_b200.nnet.framework import for_extract_embedding  # noqa: E402

MAX_CHUNK = 300     # @for_extract_embedding(maxChunk=300) of transformer_xvector.py:321
MIN_FRAMES = 7      # the shortest input Conv2dSubsampling4 and SVConv2dSubsampling2 accept
TABLE_ROWS = 5000   # PositionalEncoding / RoPositionalEncoding max_len (embedding.py:41, :162)


def _assign(defaults, given, support_unknow=False):
    """utils.assign_params_dict: known keys override the defaults (recursively for sub-dicts); unknown keys are kept
    with support_unknow=True and dropped otherwise."""
    out = copy.deepcopy(defaults)
    for k, v in (given or {}).items():
        if k in out:
            out[k] = _assign(out[k], v, support_unknow) if isinstance(out[k], dict) and isinstance(v, dict) else v
        elif support_unknow:
            out[k] = v
    return out


def _unsupported(name, value):
    raise NotImplementedError("{}={!r} is not on the native Conformer path".format(name, value))


# ConformerEncoder's own defaults (encoder.py:538-581) under TransformerXvector's (transformer_xvector.py:98-127)
_ENCODER_DEFAULTS = {
    "attention_dim": 256, "attention_heads": 4, "linear_units": 2048, "mlp_head": False, "num_blocks": 6,
    "aux_layer_period": 3, "aux_layer_start": 1, "dropout_rate": 0.1, "layer_dropout": 0., "positional_dropout_rate": 0.1,
    "attention_dropout_rate": 0.0, "attention_conv_out": False, "attention_norm_args": {}, "input_layer": "conv2d",
    "pos_enc_type": "rel_pos", "rotary_value": True, "rope_abs_plus": False, "add_t5rel_bias": False, "att_type": "multi",
    "gau_units": 512, "gau_key": 64, "normalize_before": True, "norm_type": "layer_norm", "concat_after": False,
    "positionwise_layer_type": "linear", "positionwise_conv_kernel_size": 3, "activation_type": "swish",
    "activation_balancer": False, "static_chunk_size": 0, "left_chunk_size": -1, "use_dynamic_chunk": False,
    "use_dynamic_left_chunk": False, "macaron_style": True, "use_cnn_module": True, "cnn_module_kernel": 15,
    "causal": False, "cnn_module_norm": "batch_norm", "combiner_type": "norm", "re_scale": False, "convfnn_blocks": 0,
}
_ATT_NORM_DEFAULTS = {"scale_adapt": False, "norm_method": "softmax", "diag_mask": False, "g_sa": False, "train_len": 512}


def _check_encoder(p):
    """Raise for every encoder option the native path does not build."""
    a = p["attention_norm_args"]
    for name, ok in (("att_type", p["att_type"] == "multi"), ("input_layer", p["input_layer"] in ("conv2d", "conv2d2")),
                     ("pos_enc_type", p["pos_enc_type"] in ("rot_pos", "abs_pos", "no_pos")),
                     ("rope_abs_plus", not p["rope_abs_plus"]), ("add_t5rel_bias", not p["add_t5rel_bias"]),
                     ("attention_conv_out", not p["attention_conv_out"]), ("mlp_head", not p["mlp_head"]),
                     ("combiner_type", p["combiner_type"] == "norm"), ("convfnn_blocks", p["convfnn_blocks"] == 0),
                     ("macaron_style", p["macaron_style"]), ("use_cnn_module", p["use_cnn_module"]),
                     ("causal", not p["causal"]), ("normalize_before", p["normalize_before"]),
                     ("concat_after", not p["concat_after"]), ("norm_type", p["norm_type"] == "layer_norm"),
                     ("static_chunk_size", p["static_chunk_size"] == 0), ("use_dynamic_chunk", not p["use_dynamic_chunk"]),
                     ("use_dynamic_left_chunk", not p["use_dynamic_left_chunk"]),
                     ("activation_balancer", not p["activation_balancer"]), ("re_scale", not p["re_scale"]),
                     ("positionwise_layer_type", p["positionwise_layer_type"] == "linear"),
                     ("activation_type", p["activation_type"] in ("swish", "relu")),
                     ("cnn_module_norm", p["cnn_module_norm"] in ("layer_norm", "batch_norm")),
                     ("norm_method", a["norm_method"] in ("softmax", "softmax_plus")),
                     ("scale_adapt", not a["scale_adapt"]), ("g_sa", not a["g_sa"]), ("diag_mask", not a["diag_mask"])):
        if not ok:
            _unsupported(name, a.get(name, p.get(name)))
    d, h = p["attention_dim"], p["attention_heads"]
    if d % h or d // h not in (32, 64, 128):
        raise NotImplementedError("attention_dim / attention_heads = d_k must be 32, 64 or 128 on the native path (got {} / {})"
                                  .format(d, h))
    if d % 16 or p["linear_units"] % 8 or p["cnn_module_kernel"] % 2 == 0:
        raise ValueError("attention_dim must be a multiple of 16, linear_units of 8 and cnn_module_kernel odd")


class _Conv2dSubsampling4(nn.Module):
    """Parameter container of subsampling.py:100-116 (conv.0, conv.2, out.0; the positional encodings hold none)."""

    def __init__(self, idim, odim):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(1, odim, 3, 2), nn.ReLU(), nn.Conv2d(odim, odim, 3, 2), nn.ReLU())
        self.out = nn.Sequential(nn.Linear(odim * (((idim - 1) // 2 - 1) // 2), odim))


class _SVConv2dSubsampling2(nn.Module):
    """Parameter container of SVConv2dSubsampling2 (subsampling.py:365-389): Conv2d(1, C, 3, stride (2, 1)) (time 2,
    frequency 1), Conv2d(C, C, 3, 1), Linear(C * (F - 4), C); T' = (T - 1) // 2 - 2."""

    def __init__(self, idim, odim):
        super().__init__()
        self.conv = nn.Sequential(nn.Conv2d(1, odim, 3, (2, 1)), nn.ReLU(), nn.Conv2d(odim, odim, 3, 1), nn.ReLU())
        self.out = nn.Sequential(nn.Linear(odim * (idim - 4), odim))


def subsampled_shape(subsampling, frames, freq):
    """(T', F'') of the subsampling's output for a chunk of `frames` frames of `freq` bins: 4 = Conv2dSubsampling4, 2 =
    SVConv2dSubsampling2."""
    t1 = (frames - 1) // 2
    if subsampling == 4:
        return (t1 - 1) // 2, ((freq - 1) // 2 - 1) // 2
    return t1 - 2, freq - 4


class _AttentionNormalize(nn.Module):
    """attention.py:640-672: train_len = ln(train_len) is a parameter for softmax_plus only."""

    def __init__(self, norm_method, train_len):
        super().__init__()
        self.method = norm_method
        if norm_method == "softmax_plus":
            self.train_len = nn.Parameter(torch.tensor(math.log(train_len)))


class _SelfAttention(nn.Module):
    """MultiHeadedAttention / RoPESelfAttention parameters (attention.py:26-53, :255-267)."""

    def __init__(self, heads, dim, norm_args):
        super().__init__()
        self.d_k, self.h = dim // heads, heads
        self.att_norm = _AttentionNormalize(norm_args["norm_method"], norm_args["train_len"])
        self.linear_q = nn.Linear(dim, dim)
        self.linear_k = nn.Linear(dim, dim)
        self.linear_v = nn.Linear(dim, dim)
        self.linear_out = nn.Linear(dim, dim)


class _FeedForward(nn.Module):
    """PositionwiseFeedForward (positionwise_feed_forward.py:19-34)."""

    def __init__(self, dim, units):
        super().__init__()
        self.w_1 = nn.Linear(dim, units)
        self.w_2 = nn.Linear(units, dim)


class _ConvolutionModule(nn.Module):
    """ConvolutionModule (convolution.py:21-76)."""

    def __init__(self, channels, kernel_size, norm):
        super().__init__()
        self.pointwise_conv1 = nn.Conv1d(channels, 2 * channels, 1)
        self.depthwise_conv = nn.Conv1d(channels, channels, kernel_size, padding=kernel_size // 2, groups=channels)
        self.norm = nn.BatchNorm1d(channels) if norm == "batch_norm" else nn.LayerNorm(channels)
        self.pointwise_conv2 = nn.Conv1d(channels, channels, 1)


class _ConformerLayer(nn.Module):
    """ConformerEncoderLayer parameters in the reference's registration order (encoder_layer.py:173-197)."""

    def __init__(self, p):
        super().__init__()
        d = p["attention_dim"]
        self.self_attn = _SelfAttention(p["attention_heads"], d, p["attention_norm_args"])
        self.feed_forward = _FeedForward(d, p["linear_units"])
        self.feed_forward_macaron = _FeedForward(d, p["linear_units"])
        self.conv_module = _ConvolutionModule(d, p["cnn_module_kernel"], p["cnn_module_norm"])
        for name in ("norm_ff", "norm_mha", "norm_ff_macaron", "norm_conv", "norm_final"):
            setattr(self, name, nn.LayerNorm(d, eps=1e-5))


class _ConformerEncoder(nn.Module):
    """ConformerEncoder parameters: embed, after_norm (BaseEncoder.__init__), encoders."""

    def __init__(self, idim, p):
        super().__init__()
        self.p = p
        self.subsampling = 4 if p["input_layer"] == "conv2d" else 2
        self.embed = (_Conv2dSubsampling4 if self.subsampling == 4 else _SVConv2dSubsampling2)(idim, p["attention_dim"])
        self.after_norm = nn.LayerNorm(p["attention_dim"], eps=1e-5)
        self.encoders = nn.ModuleList([_ConformerLayer(p) for _ in range(p["num_blocks"])])


class _TdnnLayer(nn.Module):
    """ReluBatchNormTdnnLayer with a context-[0] TdnnAffine (components.py:337-461): affine -> activation -> LayerNorm
    (ln_replace, affine per bn_params) or BatchNorm1d.  Only the relu-bn order is built."""

    def __init__(self, input_dim, output_dim, **options):
        super().__init__()
        if options.get("bn-relu", False):
            _unsupported("bn-relu", True)
        nonlin = options.get("nonlinearity", "relu")
        if nonlin not in ("relu", "swish", "", None, False):
            _unsupported("nonlinearity", nonlin)
        self.act = {"relu": ACT_RELU, "swish": ACT_SWISH}.get(nonlin, ACT_NONE)
        self.affine = TdnnAffine(input_dim, output_dim, context=[0], bias=options.get("bias", True))
        self.batchnorm, self.ln = None, False
        if options.get("bn", True):
            bn_params = {"momentum": 0.1, "affine": True, "track_running_stats": True}
            bn_params.update(options.get("bn_params", {}))
            if options.get("ln_replace", False):
                self.ln = True
                self.batchnorm = nn.LayerNorm(output_dim, eps=1e-5, elementwise_affine=bn_params["affine"])
            else:
                self.batchnorm = nn.BatchNorm1d(output_dim, **bn_params)


class _AttentiveStatsPool(nn.Module):
    """transformer_xvector.py:27-51: attention = conv -> ReLU -> LayerNorm -> tanh -> conv; norm_stats LayerNorm."""

    def __init__(self, in_dim, hidden_size=128, time_attention=False, stddev=True):
        super().__init__()
        if time_attention:
            _unsupported("time_attention", True)
        if not stddev:
            _unsupported("stddev", False)
        self.output_dim = in_dim * 2
        self.attention = nn.Sequential(nn.Conv1d(in_dim, hidden_size, 1), nn.ReLU(), nn.LayerNorm(hidden_size, eps=1e-5),
                                       nn.Tanh(), nn.Conv1d(hidden_size, in_dim, 1))
        self.norm_stats = nn.LayerNorm(self.output_dim, eps=1e-5)

    def get_output_dim(self):
        return self.output_dim


class TransformerXvector(TopVirtualNnet):
    """A Conformer x-vector framework.

    `masked_chunks`, set by init: extract_embedding_batch takes lengths (a masked batch of single chunks) on this
    instance.  An object that init did not build refuses lengths with NotImplementedError before it reads any
    configuration."""

    def init(self, inputs_dim, num_targets, embd_dim=256, training=True,
             extracted_embedding="near", mixup=False, mixup_alpha=1.0, pooling="ecpa-attentive", pooling_params={},
             transformer_type="conformer", transformer_params={}, tansformer_out={}, fc1=False, fc1_params={}, fc2_params={},
             margin_loss=True, margin_loss_params={}, lsm_weight=0.0, use_step=False, step_params={},
             transfer_from="softmax_loss", wenet_transfer=False):
        default_transformer_params = {                                                          # :98-127
            "attention_dim": 256, "att_type": 'multi', "attention_heads": 4, "gau_key": 64, "gau_units": 512,
            "num_blocks": 6, "dropout_rate": 0.1, "layer_dropout": 0., "positionwise_layer_type": 'linear',
            "positional_dropout_rate": 0.1, "linear_units": 2048, "positionwise_conv_kernel_size": 3,
            "attention_dropout_rate": 0.0, "attention_norm_args": {"norm_method": "softmax", "train_len": 300.},
            "input_layer": "conv2d", "pos_enc_type": "abs_pos", "cnn_module_kernel": 15, "use_cnn_module": True,
            "cnn_module_norm": 'layer_norm', "static_chunk_size": 0, "left_chunk_size": -1, "use_dynamic_chunk": False,
            "use_dynamic_left_chunk": False, "combiner_type": "norm", "convfnn_blocks": 0}
        default_tansformer_out = {"out_dim": 1536, "nonlinearity": 'swish', "nonlinearity_params": {"inplace": True},
                                  "bn-relu": False, "bn": True, "ln_replace": True,
                                  "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        default_pooling_params = {"hidden_size": 128, "time_attention": False, "stddev": True}
        default_fc_params = {"nonlinearity": 'relu', "nonlinearity_params": {"inplace": True}, "bn-relu": False,
                             "bn": True, "ln_replace": True,
                             "bn_params": {"momentum": 0.5, "affine": True, "track_running_stats": True}}
        if transformer_type in ("transformer", "re_conformer"):
            _unsupported("transformer_type", transformer_type)
        if transformer_type != "conformer":
            raise ValueError("unknown transformer_type: " + transformer_type)
        if pooling != "ecpa-attentive":
            raise ValueError("Only supoort asp for conformer now.")
        tp = _assign(default_transformer_params, transformer_params, support_unknow=True)
        enc = _assign(_ENCODER_DEFAULTS, tp, support_unknow=True)
        enc["attention_norm_args"] = _assign(_ATT_NORM_DEFAULTS, enc["attention_norm_args"], support_unknow=True)
        _check_encoder(enc)
        to = _assign(default_tansformer_out, tansformer_out)
        pp = _assign(default_pooling_params, pooling_params)
        fc1_params = _assign(default_fc_params, fc1_params)
        fc2_params = _assign(default_fc_params, fc2_params)
        self.inputs_dim = inputs_dim
        self.masked_chunks = True
        self.extracted_embedding = extracted_embedding
        self.use_step, self.step_params = use_step, step_params
        self.embd_dim = embd_dim
        self.transformer = _ConformerEncoder(inputs_dim, enc)
        self.transform_out = _TdnnLayer(enc["attention_dim"], to["out_dim"], **to)
        self.stats = _AttentiveStatsPool(to["out_dim"], **pp)
        self.fc1 = _TdnnLayer(self.stats.get_output_dim(), embd_dim, **fc1_params) if fc1 else None
        self.fc2 = _TdnnLayer(embd_dim if fc1 else self.stats.get_output_dim(), embd_dim, **fc2_params)
        for name, d in (("transform_out.out_dim", to["out_dim"]), ("pooling_params.hidden_size", pp["hidden_size"]),
                        ("embd_dim", embd_dim)):
            if d % 8:
                raise ValueError("{}={} must be a multiple of 8 on the native Conformer path".format(name, d))
        self.transform_keys = ["transformer", "transform_out", "stats", "fc1", "fc2", "loss"]
        if margin_loss and transfer_from == "softmax_loss":
            self.rename_transform_keys = {"loss.affine.weight": "loss.weight"}
        self.wenet_transfer = wenet_transfer

    def build_extractor(self):
        if self.extracted_embedding == "far" and self.fc1 is None:
            raise ValueError("extracted_embedding='far' needs fc1=True (transformer_xvector.py:334-336 asserts it)")
        if self.extracted_embedding not in ("far", "near_affine", "near"):
            raise TypeError("Expected far or near position, but got {}".format(self.extracted_embedding))
        dev = self.device_for_extraction()
        if os.environ.get("XVB_CONFORMER_NATIVE", "1") == "0":
            return ConformerExtractor(self, dev)       # op-by-op twin of the native handle
        return NativeConformerExtractor(self, dev)

    @for_extract_embedding(maxChunk=MAX_CHUNK, isMatrix=True)
    def _extract_embedding_chunked(self, inputs):
        """inputs (1, frames, feat_dim) CUDA float32 -> (1, D)."""
        return self.extractor().extract(inputs)

    def extract_embedding(self, feats):
        """feats (T, F) float32 -> 1-D CPU float32 tensor, with the reference's maxChunk = 300 chunk rule (the
        framework's single-chunk host fast path does not apply: this model cuts every utterance above 300 frames)."""
        if int(feats.shape[0]) < MIN_FRAMES:
            raise ValueError("the Conformer needs at least {} frames, got {}".format(MIN_FRAMES, int(feats.shape[0])))
        return self._extract_embedding_chunked(feats)

    def chunk_sizes(self, num_frames):
        """The chunk lengths extract_embedding cuts a num_frames-long utterance into (the reference's maxChunk = 300
        rule, chunk_plan); pipeline/extract_embeddings.py --mixed-lengths cuts utterances with it before batching them."""
        return chunk_plan(num_frames)[0]

    def extract_embedding_batch(self, feats, lengths=None):
        """Equal-length utterances (B, T, F) float32 -> (B, D) CUDA tensor, the same arithmetic as B calls of
        extract_embedding(): the B * (num_split - 1) full chunks run as one batch, the B last chunks as another, and the
        chunk embeddings are recombined with the reference's length-weighted average.

        lengths (B,) host ints: a masked batch of single chunks of different lengths padded to T, row b being the
        embedding of feats[b, :lengths[b]] extracted as one chunk (what is past it is never read).  Rows are not cut
        again: the chunk rule itself gives chunks of up to 300 + num_split - 1 frames.  ValueError for a length outside
        [7, T], naming the first such entry, and for T' >= 5000 subsampled frames."""
        if lengths is not None:
            if not getattr(self, "masked_chunks", False):
                raise NotImplementedError("{}: extract_embedding_batch(lengths=...) is for the TDNN x-vector, ResNet "
                                          "x-vector, CAM++ and Conformer blueprints only".format(type(self).__name__))
            return self._extract_masked(feats, lengths)
        with torch.no_grad():
            x = torch.as_tensor(feats)
            if x.dtype != torch.float32:
                raise TypeError("extract_embedding_batch expects float32 features")
            B, T, Fd = x.shape
            if T < MIN_FRAMES:
                raise ValueError("the Conformer needs at least {} frames, got {}".format(MIN_FRAMES, T))
            x = x.to(self.device_for_extraction(), non_blocking=True).contiguous()
            lengths, offsets = chunk_plan(T)
            ex = self.extractor()
            last = ex.extract(x[:, offsets[-1]:].contiguous())
            if len(lengths) == 1:
                return (lengths[-1] * last) / T
            split, ns = lengths[0], len(lengths) - 1
            full = ex.extract(x[:, :split * ns].reshape(B * ns, split, Fd)).view(B, ns, -1)
            acc = split * full[:, 0]
            for i in range(1, ns):
                acc = acc + split * full[:, i]
            return (acc + lengths[-1] * last) / T

    def _extract_masked(self, feats, lengths):
        with torch.no_grad():
            x = torch.as_tensor(feats)
            if x.dtype != torch.float32:
                raise TypeError("extract_embedding_batch expects float32 features")
            B, T, Fd = x.shape
            if Fd != self.inputs_dim:
                raise ValueError("expected feature dim {}, got {}".format(self.inputs_dim, Fd))
            lens = _checked_lengths(lengths, B, T, self.transformer.subsampling)
            x = x.to(self.device_for_extraction(), non_blocking=True).contiguous()
            return self.extractor().extract(x, lens)


def _checked_lengths(lengths, b, t, subsampling):
    """Host int32 (B,) lengths of a masked Conformer batch padded to t frames; ValueError naming the first entry outside
    [MIN_FRAMES, t], or when t subsamples to TABLE_ROWS frames or more."""
    lens = host_lengths(lengths, b)
    bad = np.flatnonzero((lens < MIN_FRAMES) | (lens > t))
    if bad.size:
        raise ValueError("lengths[{}]={} outside [{}, T={}]: the Conformer needs at least {} frames".format(
            bad[0], lens[bad[0]], MIN_FRAMES, t, MIN_FRAMES))
    t2 = subsampled_shape(subsampling, t, MIN_FRAMES)[0]
    if t2 >= TABLE_ROWS:
        raise ValueError("a chunk of {} subsampled frames exceeds the positional tables' {}".format(t2, TABLE_ROWS))
    return lens


def chunk_plan(num_frames, max_chunk=MAX_CHUNK):
    """for_extract_embedding's split (framework.py:34-47): (chunk lengths, chunk offsets)."""
    num_split = (num_frames + max_chunk - 1) // max_chunk
    split = num_frames // num_split
    lengths = [split] * (num_split - 1) + [num_frames - split * (num_split - 1)]
    return lengths, [i * split for i in range(num_split)]


def sinusoid_table(dim, max_len=5000):
    """PositionalEncoding.pe (embedding.py:49-56), (max_len, dim)."""
    pe = torch.zeros(max_len, dim)
    position = torch.arange(0, max_len, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, dim, 2, dtype=torch.float32) * -(math.log(10000.0) / dim))
    pe[:, 0::2] = torch.sin(position * div_term)
    pe[:, 1::2] = torch.cos(position * div_term)
    return pe


def rotary_table(dk, max_len=5000):
    """RoPositionalEncoding.pe (embedding.py:162-176), (max_len, dk) = [sin | cos]: computed on the CPU exactly as the
    reference builds it."""
    abs_rope = sinusoid_table(dk, max_len)
    freq = torch.zeros_like(abs_rope)
    freq[:, 0:dk // 2] = abs_rope[:, 0::2]
    freq[:, dk // 2:] = abs_rope[:, 1::2]
    return freq


def subsampling_column_order(channels, freq):
    """Input column of the subsampling Linear for each column of the (B, T', F'', C) conv output flattened as f * C + c:
    the reference flattens (c, f) as c * F'' + f (subsampling.py:134-135)."""
    f, c = np.meshgrid(np.arange(freq), np.arange(channels), indexing="ij")
    return (c * freq + f).reshape(-1)


def softmax_plus_multiplier(frames, train_len):
    """AttentionNormalize.attention_normalize's factor (attention.py:719-726) with every score unmasked, in fp32:
    (ln(l) / train_len * 1 + 1) - 1 with l = frames."""
    mask = torch.ones((), dtype=torch.float32)
    l = torch.tensor(float(frames), dtype=torch.float32)
    return float(torch.log(l) / train_len.detach().float().cpu() * mask + 1 - mask)


def _lin(rec, device):
    """A Linear / kernel-size-1 conv record (name, w (Cout, Cin), bias, scale, shift, flags, ...) as an ops.PackedAffine:
    y = epi(W x + b) with the record's ReLU or swish, and its folded BatchNorm (or constant scale) as the epilogue's
    scale / shift."""
    w, b, scale, shift, flags = rec[1:6]
    return ops.PackedAffine(w, device, bias=b, scale=scale, shift=shift, relu=bool(flags & RELU), swish=bool(flags & SWISH))


class ConformerExtractor:
    """Folded weights on one device + the launch sequence of TransformerXvector.extract_embedding for one chunk per
    utterance (all utterances of a call have the same length, or a masked batch gives each its own), driven from Python.
    The weights and tables are the records and configuration the native handle takes (native_records, native_config)."""

    TAKES_LENGTHS = True

    def __init__(self, m, device):
        recs = {r[0]: r for r in native_records(m)}
        cfg = native_config(m)
        lin = lambda name: _lin(recs[name], device)  # noqa: E731
        norm = lambda name: (ops.to_device(recs[name][3], device), ops.to_device(recs[name][4], device))  # noqa: E731

        def tdnn(name):
            """(_lin with the record's activation [and folded BatchNorm], LayerNorm (gamma, beta) or None)."""
            return lin(name + ".affine"), norm(name + ".batchnorm") if name + ".batchnorm" in recs else None

        self.device, self.feat_dim = device, cfg["feat_dim"]
        self.D, self.H = cfg["D"], cfg["H"]
        self.dk = self.D // self.H
        self.pos = ("no_pos", "abs_pos", "rot_pos")[cfg["pos"]]
        self.rotary_value = self.pos == "rot_pos" and bool(cfg["rotary_value"])
        self.softmax_plus = bool(cfg["softmax_plus"])
        self.act = cfg["act"]
        self.subsampling = cfg["subsampling"]
        e = "transformer.embed."
        self.head_w = ops.to_device(recs[e + "conv.0"][1].reshape(self.D, 1, 3, 3), device)
        self.head_b = ops.to_device(recs[e + "conv.0"][2], device)
        self.conv2_w = ops.pack_conv2d_weight(ops.to_device(recs[e + "conv.2"][1].reshape(self.D, self.D, 3, 3), device))
        self.conv2_scale = torch.ones(self.D, dtype=torch.float32, device=device)
        self.conv2_shift = ops.to_device(recs[e + "conv.2"][2], device)
        self.embed_out = lin(e + "out.0")
        self.layers = []
        for i in range(cfg["blocks"]):
            q = "transformer.encoders.{}.".format(i)
            cm = q + "conv_module."
            L = {"ff_mac": (lin(q + "feed_forward_macaron.w_1"), lin(q + "feed_forward_macaron.w_2")),
                 "ff": (lin(q + "feed_forward.w_1"), lin(q + "feed_forward.w_2")),
                 "qkv": lin(q + "self_attn.linear_qkv"),
                 "out": lin(q + "self_attn.linear_out"),
                 "pw1": lin(cm + "pointwise_conv1"),
                 "pw2": lin(cm + "pointwise_conv2"),
                 "dw_w": ops.to_device(recs[cm + "depthwise_conv"][1], device),
                 "dw_b": ops.to_device(recs[cm + "depthwise_conv"][2], device),
                 "cm_norm": norm(cm + "norm") + (bool(recs[cm + "norm"][5] & BN),),
                 "att_norm": recs[q + "self_attn.att_norm"][1][0] if self.softmax_plus else None}
            # the multiplier table on the device, indexed by each utterance's T' in a masked batch
            L["mult_table"] = ops.to_device(L["att_norm"], device) if self.softmax_plus else None
            for name in ("norm_ff", "norm_mha", "norm_ff_macaron", "norm_conv", "norm_final"):
                L[name] = norm(q + name)
            self.layers.append(L)
        self.after_norm = norm("transformer.after_norm")
        # transform_out: affine -> activation -> LayerNorm (its own kernel) or BatchNorm (the epilogue)
        self.transform = tdnn("transform_out")
        self.att1 = lin("stats.attention.0")
        self.att_ln = norm("stats.attention.2")
        self.att2 = lin("stats.attention.4")
        self.norm_stats = norm("stats.norm_stats")
        self.segment = [tdnn(name) for name in ("fc1", "fc2") if name + ".affine" in recs]
        self.embed_dim = self.segment[-1][0].cout
        self._pos_table = recs["pos_table"][1] if "pos_table" in recs else None
        self._tables = {}
        self.last_launches = 0

    def _tables_for(self, t):
        if t not in self._tables:
            if t >= TABLE_ROWS:
                raise ValueError("a chunk of {} subsampled frames exceeds the positional tables' {}".format(t, TABLE_ROWS))
            table = ops.to_device(self._pos_table[:t], self.device) if self._pos_table is not None else None
            rope, absp = (table, None) if self.pos == "rot_pos" else (None, table)
            mults = [float(L["att_norm"][t]) if self.softmax_plus else 1.0 for L in self.layers]
            self._tables[t] = (rope, absp, mults)
        return self._tables[t]

    def extract(self, feats, lengths=None):
        """feats (B, T, F) fp32 CUDA (one chunk per utterance) -> (B, embd_dim) fp32 CUDA, asynchronous on the current
        stream.  lengths (B,) host ints, 7 <= lengths[b] <= T: a masked batch as xvb_conformer_extract_lengths runs it,
        row b being feats[b, :lengths[b]] extracted alone (every length equal to T: the unmasked sequence).  The head
        conv, every frame-level linear, the attention and the attentive pooling then take each utterance's length."""
        if feats.shape[2] != self.feat_dim:
            raise ValueError("expected feature dim {}, got {}".format(self.feat_dim, feats.shape[2]))
        feats = feats.contiguous()
        B, T, Fd = feats.shape
        l1 = l2 = None    # a masked batch's lengths L at the input and L' after the subsampling
        if lengths is not None:
            lens = _checked_lengths(lengths, B, T, self.subsampling)
            if (lens != T).any():
                sub = np.array([subsampled_shape(self.subsampling, int(v), Fd)[0] for v in lens], np.int32)
                table = torch.from_numpy(np.stack([lens, sub])).to(feats.device)
                l1, l2 = table[0], table[1]
        if T < MIN_FRAMES:
            raise ValueError("the Conformer needs at least {} frames, got {}".format(MIN_FRAMES, T))
        dev, P, D = feats.device, ops.SplitPlanes, self.D
        T1 = (T - 1) // 2
        F1 = (Fd - 1) // 2 if self.subsampling == 4 else Fd - 2
        T2, F2 = subsampled_shape(self.subsampling, T, Fd)
        rope, absp, mults = self._tables_for(T2)
        n = 0
        x1 = P.empty((B, T1, F1, D), dev)
        if self.subsampling == 4:
            ops.subsample_head(feats, self.head_w, self.head_b, x1, lengths=l1)
        else:       # SVConv2dSubsampling2: time stride 2, frequency stride 1, then a stride-1 valid conv
            ops.subsample_head(feats, self.head_w, self.head_b, x1, stride_f=1, lengths=l1)
        x2 = P.empty((B, T2, F2, D), dev)
        ops.conv2d(x1, self.conv2_w, D, 3, 2 if self.subsampling == 4 else 1, self.conv2_scale, self.conv2_shift, relu=True,
                   y=x2, valid=True)
        del x1
        r = torch.empty(B, T2, D, dtype=torch.float32, device=dev)
        self.embed_out.run(P(x2.hi.view(B, T2, F2 * D), x2.lo.view(B, T2, F2 * D), F2 * D), y_f32=r, lengths=l2)
        n += 3
        units = self.layers[0]["ff"][0].cout if self.layers else 0
        h = P.empty((B, T2, D), dev)
        hid = P.empty((B, T2, max(units, D)), dev)
        delta = torch.empty(B, T2, 2 * D, dtype=torch.float32, device=dev)
        qkv = torch.empty(B, T2, 3 * D, dtype=torch.float32, device=dev)
        d1 = delta[..., :D]
        hid_u = hid if units == hid.channels else hid.slice(0, units)
        hid_d = hid if D == hid.channels else hid.slice(0, D)

        def ffn(pair, out):
            pair[0].run(h, y=hid_u, lengths=l2)
            pair[1].run(hid_u, y_f32=out, lengths=l2)

        first = self.layers[0] if self.layers else None
        if first is not None:   # r [+ pe] -> r, norm_ff_macaron
            ops.layer_norm(r, *first["norm_ff_macaron"], table=absp, x_out=r, y=h)
            n += 1
        for i, L in enumerate(self.layers):
            ffn(L["ff_mac"], d1)
            ops.layer_norm(r, *L["norm_mha"], delta=d1, delta_scale=0.5, x_out=r, y=h)
            L["qkv"].run(h, y_f32=qkv, lengths=l2)
            if l2 is None:
                ops.rope_attention(qkv, self.H, self.dk, hid_d, rope=rope, rope_v=self.rotary_value, score_mult=mults[i])
            else:
                ops.rope_attention(qkv, self.H, self.dk, hid_d, rope=rope, rope_v=self.rotary_value, lengths=l2,
                                   mult_table=L["mult_table"])
            L["out"].run(hid_d, y_f32=d1, lengths=l2)
            ops.layer_norm(r, *L["norm_conv"], delta=d1, x_out=r, y=h)
            L["pw1"].run(h, y_f32=delta, lengths=l2)
            g, b, bn = L["cm_norm"]
            ops.conv_module(delta, L["dw_w"], L["dw_b"], g, b, hid_d, batch_norm=bn, act=self.act)
            L["pw2"].run(hid_d, y_f32=d1, lengths=l2)
            ops.layer_norm(r, *L["norm_ff"], delta=d1, x_out=r, y=h)
            ffn(L["ff"], d1)
            nxt = self.layers[i + 1]["norm_ff_macaron"] if i + 1 < len(self.layers) else self.after_norm
            ops.layer_norm(r, *L["norm_final"], delta=d1, delta_scale=0.5, x_out=r, second=nxt, y=h)
            n += 16
        del hid, delta, qkv
        # transform_out (+ its LayerNorm): x fp32 for the pooling sums, planes for the attention conv
        lin, ln = self.transform
        od = lin.cout
        xo = torch.empty(B, T2, od, dtype=torch.float32, device=dev)
        xp = P.empty((B, T2, od), dev)
        if ln is None:
            lin.run(h, y=xp, y_f32=xo, lengths=l2)
            n += 1
        else:
            lin.run(h, y_f32=xo, lengths=l2)
            ops.layer_norm(xo, *ln, x_out=None, y=xp, y_f32=xo)
            n += 2
        # AttentiveStatsPool
        a1 = torch.empty(B, T2, self.att1.cout, dtype=torch.float32, device=dev)
        self.att1.run(xp, y_f32=a1, lengths=l2)
        ap = P.empty((B, T2, self.att1.cout), dev)
        ops.layer_norm(a1, *self.att_ln, act=ACT_TANH, y=ap)
        logits = torch.empty(B, T2, od, dtype=torch.float32, device=dev)
        self.att2.run(ap, y_f32=logits, lengths=l2)
        stats = ops.attn_stats_pool(logits, xo, floor=1e-5, lengths=l2)
        z = P.empty((B, 1, 2 * od), dev)
        zf = torch.empty(B, 1, 2 * od, dtype=torch.float32, device=dev)
        ops.layer_norm(stats, *self.norm_stats, y=z, y_f32=zf)
        n += 5
        for j, (lin, ln) in enumerate(self.segment):
            last = j + 1 == len(self.segment)
            y = torch.empty(B, 1, lin.cout, dtype=torch.float32, device=dev)
            lin.run(z, y_f32=y)
            n += 1
            yp = None
            if ln is not None:
                yp = None if last else P.empty((B, 1, lin.cout), dev)
                ops.layer_norm(y, *ln, y=yp, y_f32=y)
                n += 1
            elif not last:
                yp = ops.split_f32(y)
                n += 1
            z, zf = yp, y
        self.last_launches = n
        return zf.view(B, -1)[:, :self.embed_dim]

    def close(self):
        pass


def _embed_out_weight(m):
    """The subsampling Linear's weight with its input columns permuted to the f * C + c order of the conv output, and
    the xscale sqrt(d) as the epilogue's scale (None for no_pos)."""
    enc = m.transformer
    d = enc.p["attention_dim"]
    f2 = subsampled_shape(enc.subsampling, MIN_FRAMES, m.inputs_dim)[1]
    w = enc.embed.out[0].weight.detach().float()[:, torch.from_numpy(subsampling_column_order(d, f2))]
    xscale = None if enc.p["pos_enc_type"] == "no_pos" else np.full(d, math.sqrt(d), np.float32)
    return w, xscale


def native_config(m):
    """xvb_conformer_config_t fields of a TransformerXvector."""
    p = m.transformer.p
    to = m.transform_out
    return dict(feat_dim=m.inputs_dim, subsampling=m.transformer.subsampling, D=p["attention_dim"], H=p["attention_heads"],
                linear_units=p["linear_units"], blocks=p["num_blocks"], conv_kernel=p["cnn_module_kernel"],
                pos={"no_pos": 0, "abs_pos": 1, "rot_pos": 2}[p["pos_enc_type"]], rotary_value=int(bool(p["rotary_value"])),
                softmax_plus=int(p["attention_norm_args"]["norm_method"] == "softmax_plus"),
                act=ACT_SWISH if p["activation_type"] == "swish" else ACT_RELU,
                cm_norm=int(p["cnn_module_norm"] == "batch_norm"), out_dim=to.affine.weight.shape[0],
                out_norm=0 if to.batchnorm is None else (2 if to.ln else 1),
                pool_hidden=m.stats.attention[0].weight.shape[0], fc1=int(m.fc1 is not None),
                position={"far": 0, "near_affine": 1, "near": 2}[m.extracted_embedding])


def native_records(m):
    """(name, w, bias, scale, shift, flags, keys) records and tables for xvb_conformer_set_layer and ConformerExtractor,
    after the hand-over transforms: the concatenated Q/K/V, the subsampling Linear's column permutation and xscale, the
    second subsampling conv transposed to (C, C, kf, kt), folded BatchNorms.  `keys` are the state_dict
    entries the record carries.  Tables: "pos_table" (rotary_table or sinusoid_table) and, for softmax_plus, each
    block's "self_attn.att_norm" = softmax_plus_multiplier for T' = 1 .. 4999 (index 0 unused, 0)."""
    from asv_subtools_b200._lib import BN, RELU, SWISH
    f = lambda t: None if t is None else t.detach().float().cpu().numpy()  # noqa: E731
    enc = m.transformer
    p = enc.p
    d, h = p["attention_dim"], p["attention_heads"]
    act = SWISH if p["activation_type"] == "swish" else RELU
    out = []

    def keys_of(mod, name):
        return [name + "." + k for k in mod.state_dict()]

    def lin(name, mod, flags=0, scale=None, shift=None, w=None):
        w = f(mod.weight).reshape(mod.weight.shape[0], -1) if w is None else w
        if scale is not None:
            flags |= BN
        out.append((name, w, f(mod.bias), scale, shift, flags, keys_of(mod, name)))

    def norm(name, mod):
        if isinstance(mod, nn.BatchNorm1d):
            s, t = fold_batchnorm(mod)
            out.append((name, None, None, s, t, BN, keys_of(mod, name)))
        else:
            out.append((name, None, None, f(mod.weight), f(mod.bias), 0, keys_of(mod, name)))

    def tdnn(name, layer, whole):
        a = layer.affine
        w = f(a.weight)[:, :, 0]
        flags = 0 if not whole else {ACT_RELU: RELU, ACT_SWISH: SWISH}.get(layer.act, 0)
        if whole and layer.batchnorm is not None and not layer.ln:
            s, t = fold_batchnorm(layer.batchnorm)
            out.append((name + ".affine", w, f(a.bias), s, t, flags | BN,
                        keys_of(a, name + ".affine") + keys_of(layer.batchnorm, name + ".batchnorm")))
            return
        out.append((name + ".affine", w, f(a.bias), None, None, flags, keys_of(a, name + ".affine")))
        if whole and layer.batchnorm is not None:
            norm(name + ".batchnorm", layer.batchnorm)

    e = "transformer.embed."
    conv0, conv2 = enc.embed.conv[0], enc.embed.conv[2]
    out.append((e + "conv.0", f(conv0.weight).reshape(d, 9), f(conv0.bias), None, None, 0, keys_of(conv0, e + "conv.0")))
    w2 = conv2.weight.detach().float().transpose(2, 3).reshape(d, 9 * d).cpu().numpy()
    out.append((e + "conv.2", w2, f(conv2.bias), None, None, 0, keys_of(conv2, e + "conv.2")))
    lw, xscale = _embed_out_weight(m)
    lin(e + "out.0", enc.embed.out[0], w=f(lw), scale=xscale, shift=None if xscale is None else np.zeros(d, np.float32))
    if p["pos_enc_type"] != "no_pos":
        table = rotary_table(d // h) if p["pos_enc_type"] == "rot_pos" else sinusoid_table(d)
        out.append(("pos_table", f(table), None, None, None, 0, []))
    softmax_plus = p["attention_norm_args"]["norm_method"] == "softmax_plus"
    for i, layer in enumerate(enc.encoders):
        q = "transformer.encoders.{}.".format(i)
        for ff in ("feed_forward_macaron", "feed_forward"):
            mod = getattr(layer, ff)
            lin(q + ff + ".w_1", mod.w_1, act)
            lin(q + ff + ".w_2", mod.w_2)
        a = layer.self_attn
        qkv = [a.linear_q, a.linear_k, a.linear_v]
        out.append((q + "self_attn.linear_qkv", f(torch.cat([x.weight for x in qkv], 0)), f(torch.cat([x.bias for x in qkv], 0)),
                    None, None, 0,
                    sum([keys_of(x, q + "self_attn." + n) for x, n in zip(qkv, ("linear_q", "linear_k", "linear_v"))], [])))
        lin(q + "self_attn.linear_out", a.linear_out)
        if softmax_plus:
            mult = np.zeros((1, TABLE_ROWS), np.float32)
            for t in range(1, TABLE_ROWS):
                mult[0, t] = softmax_plus_multiplier(t, a.att_norm.train_len)
            out.append((q + "self_attn.att_norm", mult, None, None, None, 0, keys_of(a.att_norm, q + "self_attn.att_norm")))
        cm = layer.conv_module
        lin(q + "conv_module.pointwise_conv1", cm.pointwise_conv1)
        out.append((q + "conv_module.depthwise_conv", f(cm.depthwise_conv.weight).reshape(d, -1), f(cm.depthwise_conv.bias),
                    None, None, 0, keys_of(cm.depthwise_conv, q + "conv_module.depthwise_conv")))
        norm(q + "conv_module.norm", cm.norm)
        lin(q + "conv_module.pointwise_conv2", cm.pointwise_conv2)
        for name in ("norm_ff", "norm_mha", "norm_ff_macaron", "norm_conv", "norm_final"):
            norm(q + name, getattr(layer, name))
    norm("transformer.after_norm", enc.after_norm)
    tdnn("transform_out", m.transform_out, True)
    att = m.stats.attention
    lin("stats.attention.0", att[0], RELU)
    norm("stats.attention.2", att[2])
    lin("stats.attention.4", att[4])
    norm("stats.norm_stats", m.stats.norm_stats)
    pos = m.extracted_embedding
    if pos == "far":
        tdnn("fc1", m.fc1, False)
    else:
        if m.fc1 is not None:
            tdnn("fc1", m.fc1, True)
        tdnn("fc2", m.fc2, pos == "near")
    return out


class NativeConformerExtractor(NativeExtractor):
    """xvb_conformer_t: packed weights, tables, workspace and the whole launch sequence of ConformerExtractor in the C
    library, on the device that is current when it is built (or loaded from an XVBC0001 file)."""

    PREFIX = "conformer"
    TAKES_LENGTHS = True

    def _create_args(self, m):
        from asv_subtools_b200._lib import ConformerConfig
        return (C.byref(ConformerConfig(**native_config(m))),)

    def _layers(self, m):
        for name, w, b, scale, shift, flags, _ in native_records(m):
            rows = w.shape[0] if w is not None else scale.shape[0] if scale is not None else _norm_width(m, name)
            yield name, (rows, w.shape[1] if w is not None else 0), (w, b, scale, shift), flags


def _norm_width(m, name):
    """Channel count of a LayerNorm record without affine (no array to read it from)."""
    mod = m
    for part in name.split("."):
        mod = mod[int(part)] if part.isdigit() else getattr(mod, part)
    return mod.normalized_shape[0]


if __name__ == "__main__":
    print(TransformerXvector(80, 10, training=False))
