"""Pooling layers mirroring pytorch/libs/nnet/pooling.py: StatisticsPooling (:15-76), LDEPooling (:130-162) and the attention poolings built
on AttentionAlphaComponent (:214-319) -- AttentiveStatisticsPooling (:322-368), MultiHeadAttentionPooling (:371-440),
GlobalMultiHeadAttentionPooling (:443-515), MultiResolutionMultiHeadAttentionPooling (:518-587) and MQMHASP (:589-698).  Parameter containers
under the reference's state_dict keys; the arithmetic lives in csrc/pooling.cu / csrc/ecapa.cu
(`xvb_attn_head_stats_pool`) and the wgmma layer kernel, driven by the owning model."""
import torch

from .. import ops
from .components import TdnnAffine


class StatisticsPooling(torch.nn.Module):
    def __init__(self, input_dim, stddev=True, unbiased=False, eps=1.0e-10):
        super().__init__()
        if not stddev or unbiased:
            raise NotImplementedError("B200 StatisticsPooling implements the mean+std, biased-variance case")
        self.input_dim, self.stddev, self.unbiased, self.eps = input_dim, stddev, unbiased, eps
        self.output_dim = 2 * input_dim

    def get_output_dim(self):
        return self.output_dim

    def forward(self, inputs):
        """inputs: (B, C, T) like the reference -> (B, 2C, 1)."""
        x = inputs.transpose(1, 2).contiguous().float()
        return ops.stats_pool(x, eps=self.eps).unsqueeze(2)


class LDEPooling(torch.nn.Module):
    """Learnable dictionary encoding (pooling.py:130-162): parameters `mu` (input_dim, c_num) and `s` (c_num,) under the
    reference's names; arithmetic in csrc/ecapa.cu (`xvb_lde_pool`: squared distances summed directly in fp32, softmax over
    the clusters, weighted residual mean over time).  c_num <= 64."""

    def __init__(self, input_dim, c_num=64, eps=1.0e-10):
        super().__init__()
        if c_num > 64:
            raise NotImplementedError("B200 LDEPooling holds at most 64 clusters (xvb_lde_pool)")
        self.input_dim, self.output_dim, self.eps = input_dim, input_dim * c_num, eps
        self.mu = torch.nn.Parameter(torch.randn(input_dim, c_num))
        self.s = torch.nn.Parameter(torch.ones(c_num))

    def get_output_dim(self):
        return self.output_dim

    def neg_beta(self):
        """-(s^2 + eps) per cluster, fp32 like the reference's forward (:155)."""
        return -(self.s.detach().float() ** 2 + self.eps)


class xivec_stdinit_softplus2_prec_pooling(torch.nn.Module):
    """Xi-vector pooling (pooling.py:165-212): a frame-wise precision network lin1_relu_bn -> lin2 -> softplus, Gaussian
    posterior inference against a learnt prior (prior_mean, prior_logprec): phi = sum over the T frames AND the prior of
    softmax(2 log precision) * value; `stddev=True` adds the posterior spread.  Same parameter names as the reference; the
    arithmetic runs on the layer kernel (lin1, lin2) and `xvb_attn_head_stats_pool_prior`."""

    def __init__(self, input_dim, hidden_size=256, context=[0], stddev=False, train_mean=True, train_prec=True):
        super().__init__()
        from .components import ReluBatchNormTdnnLayer
        self.input_dim, self.stddev = input_dim, stddev
        self.output_dim = 2 * input_dim if stddev else input_dim
        self.prior_mean = torch.nn.Parameter(torch.zeros(1, input_dim), requires_grad=train_mean)
        self.prior_logprec = torch.nn.Parameter(torch.zeros(1, input_dim), requires_grad=train_prec)
        self.lin1_relu_bn = ReluBatchNormTdnnLayer(input_dim, hidden_size, context)
        self.lin2 = TdnnAffine(hidden_size, input_dim, context=context)

    def get_output_dim(self):
        return self.output_dim


class AttentionAlphaComponent(torch.nn.Module):
    """alpha = softmax_T(last_affine(relu(first_affine(x)))) -- same constructor, same parameter / buffer names and
    shapes as the reference (pooling.py:226-298): grouped affines for split heads, `t` the per-head temperature
    (buffer when fixed, parameter otherwise)."""

    def __init__(self, input_dim, num_head=1, split_input=True, share=True, affine_layers=2, hidden_size=64, context=[0],
                 bias=True, temperature=False, fixed=True):
        super().__init__()
        assert num_head >= 1
        if num_head > 1:
            if split_input:
                assert input_dim % num_head == 0
            if temperature:
                if fixed:
                    self.register_buffer("t", torch.tensor([[[[max(1, (i // 2) * 5)]] for i in range(num_head)]]))
                else:
                    self.t = torch.nn.Parameter(torch.zeros(1, num_head, 1, 1))
        self.input_dim, self.num_head, self.split_input, self.share = input_dim, num_head, split_input, share
        self.temperature, self.fixed = temperature, fixed
        if affine_layers not in (1, 2):
            raise ValueError("Expected 1 or 2 affine layers, but got {}.".format(affine_layers))
        multi = num_head > 1
        # one logit per head when the weight is shared, else one per pooled channel of the head
        self.final_dim = 1 if share else (input_dim // num_head if split_input else input_dim)
        self.relu_affine = affine_layers == 2
        hidden = hidden_size * num_head
        if self.relu_affine:     # hidden layer: per-head blocks; its input is split too only for split heads
            self.first_affine = TdnnAffine(input_dim, hidden, context=context, bias=bias, groups=num_head if multi and split_input else 1)
        last_in = hidden if self.relu_affine else input_dim
        last_groups = num_head if multi and (self.relu_affine or split_input) else 1
        self.last_affine = TdnnAffine(last_in, self.final_dim * num_head, context=context, bias=bias, groups=last_groups)

    def head_temperatures(self):
        """(num_head,) divisors of the logits, or None: fixed buffer as stored, learnt as 1 + t^2 (:308-313)."""
        if not (self.num_head > 1 and self.temperature):
            return None
        t = self.t.detach().float().reshape(-1)
        return t if self.fixed else 1 + t ** 2


class _AttentionPooling(torch.nn.Module):
    """Shared shape logic: output channel o pools input channel o % C with the alpha of logit o // gdiv."""
    global_heads = False

    def _setup(self, input_dim, stddev, stddev_attention, num_head):
        if not stddev:
            raise NotImplementedError("stddev=False is not on the B200 path")
        self.input_dim, self.stddev, self.stddev_attention, self.num_head = input_dim, stddev, stddev_attention, num_head
        self.output_dim = 2 * input_dim

    def pooled_channels(self):
        return self.input_dim * (self.num_head if self.global_heads else 1)

    def logit_divisor(self):
        a = self.attention
        if not a.share:
            return 1                                              # one logit per pooled channel
        return self.input_dim if self.global_heads else self.input_dim // self.num_head

    def get_output_dim(self):
        return self.output_dim * (self.num_head if self.global_heads else 1)


class AttentiveStatisticsPooling(_AttentionPooling):
    def __init__(self, input_dim, affine_layers=2, hidden_size=64, context=[0], stddev=True, stddev_attention=True, eps=1.0e-10):
        super().__init__()
        self._setup(input_dim, stddev, stddev_attention, 1)
        self.eps = eps
        self.attention = AttentionAlphaComponent(input_dim, num_head=1, share=True, affine_layers=affine_layers,
                                                 hidden_size=hidden_size, context=context)


class MultiHeadAttentionPooling(_AttentionPooling):
    def __init__(self, input_dim, stddev=True, stddev_attention=True, num_head=4, share=True, affine_layers=1, **options):
        super().__init__()
        self._setup(input_dim, stddev, stddev_attention, num_head)
        self.eps = 1.0e-10
        if "split_input" in options:
            if not options["split_input"]:
                raise ValueError("split_input==False is not valid for this MultiHeadAttentionPooling.")
            options.pop("split_input")
        self.attention = AttentionAlphaComponent(input_dim, num_head=num_head, split_input=True, share=share,
                                                 affine_layers=affine_layers, bias=False, **options)


class GlobalMultiHeadAttentionPooling(_AttentionPooling):
    global_heads = True

    def __init__(self, input_dim, stddev=True, stddev_attention=True, num_head=4, share=True, affine_layers=2, **options):
        super().__init__()
        self._setup(input_dim, stddev, stddev_attention, num_head)
        self.eps = 1.0e-10
        if options.pop("split_input", False):
            raise ValueError("split_input==True is not valid for GlobalMultiHeadAttentionPooling.")
        if options.pop("temperature", False):
            raise ValueError("temperature==True is not valid for GlobalMultiHeadAttentionPooling.")
        self.attention = AttentionAlphaComponent(input_dim, num_head=num_head, split_input=False, share=share,
                                                 temperature=False, affine_layers=affine_layers, bias=True, **options)


class MultiResolutionMultiHeadAttentionPooling(_AttentionPooling):
    global_heads = True

    def __init__(self, input_dim, stddev=True, stddev_attention=True, num_head=4, share=True, affine_layers=2, **options):
        super().__init__()
        self._setup(input_dim, stddev, stddev_attention, num_head)
        self.eps = 1.0e-10
        if options.pop("split_input", False):
            raise ValueError("split_input==True is not valid for MultiResolutionMultiHeadAttentionPooling.")
        if "temperature" in options and not options.pop("temperature"):
            raise ValueError("temperature==False is not valid for MultiResolutionMultiHeadAttentionPooling.")
        self.attention = AttentionAlphaComponent(input_dim, num_head=num_head, split_input=False, temperature=True,
                                                 share=share, affine_layers=affine_layers, bias=True, **options)


class MQMHASP(torch.nn.Module):
    """Multi-query multi-head attention pooling (pooling.py:589-698): the input's C channels form num_head heads of
    Cg = C / num_head channels; the attention (grouped convs, groups = num_head then num_head * num_q) gives num_q alphas
    per head (one per channel of the head, or one shared with `share`); pooled channel (h*num_q + q)*Cg + c is channel
    h*Cg + c weighted by alpha (h, q[, c]), out = [mean | std] (stddev) or mean.  With `time_attention` the first conv
    also sees each head's utterance mean and std (biased, clamped at 1e-5).  Same constructor defaults, parameter names
    and shapes as the reference; the arithmetic runs in the owning ECAPA model's extractor."""

    def __init__(self, in_dim, num_q=2, num_head=4, hidden_size=128, stddev=True, share=True, affine_layers=2,
                 time_attention=False, norm_type="batch_norm", **kargs):
        super().__init__()
        if norm_type != "batch_norm":
            raise NotImplementedError("MQMHASP norm_type={!r} (GroupNorm in the attention) is not on the B200 path".format(norm_type))
        if affine_layers not in (1, 2):
            raise ValueError("Expected 1 or 2 affine layers, but got {}.".format(affine_layers))
        self.stddev, self.share, self.time_attention, self.affine_layers = stddev, share, time_attention, affine_layers
        self.num_head, self.num_q, self.hidden_size = max(1, num_head), max(1, num_q), hidden_size
        assert in_dim % num_head == 0
        self.in_dim = in_dim
        head = in_dim // num_head
        att_idim = ((3 if stddev else 2) if time_attention else 1) * head
        att_odim = (1 if share else head) * num_head * num_q
        if affine_layers == 2:
            hidden = hidden_size * num_head * num_q
            self.attention = torch.nn.Sequential(
                torch.nn.Conv1d(att_idim * num_head, hidden, kernel_size=1, groups=num_head), torch.nn.ReLU(),
                torch.nn.BatchNorm1d(hidden), torch.nn.Tanh(),
                torch.nn.Conv1d(hidden, att_odim, kernel_size=1, groups=num_head * num_q))
        else:
            self.attention = torch.nn.Sequential(torch.nn.Conv1d(att_idim * num_head, att_odim, kernel_size=1, groups=num_head))
        self.out_dim = in_dim * num_q * (2 if stddev else 1)

    def get_output_dim(self):
        return self.out_dim

    def head_width(self):
        return self.in_dim // self.num_head

    def num_logits(self):
        return (1 if self.share else self.head_width()) * self.num_head * self.num_q
