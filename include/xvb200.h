/*
 * xvb200.h -- C ABI of libxvb200.so, the H100 (sm_90a) x-vector extraction / back-end scoring
 * library that stands in for the hot path of Snowdar/asv-subtools.
 *
 * The reference has no native FFI for this path: its "kernels" are ATen calls issued from
 * Python (SURVEY.md section 2).  The entry points below are therefore what a ctypes stub in the
 * reference tree would bind to replace those calls; each one cites the reference code whose
 * arithmetic it takes over (paths relative to the reference root).  INTEGRATION.md shows the
 * stub.  Conventions:
 *
 *   - plain C, no C++/torch types; every pointer is a raw device pointer unless the name ends
 *     in _host; sizes are explicit; nothing is allocated behind the caller's back except by
 *     the xvb_extractor_* object, which owns its packed weights and workspace;
 *   - every function returns 0 on success or a negative XVB_E* code; xvb_last_error() gives
 *     the message (thread-local);
 *   - device functions are asynchronous on the caller-supplied cudaStream_t (passed as void*);
 *   - frame matrices are channel-contiguous "(B, T, C)" (the reference is (B, C, T); Kaldi
 *     features arrive as (T, F), so no transpose is needed on the way in);
 *   - "split planes": an fp32 tensor stored as two bf16 tensors hi = bf16(x), lo = bf16(x-hi)
 *     (same bytes as fp32).  The wgmma GEMM consumes them as x*w ~= hi*whi + lo*whi + hi*wlo
 *     with fp32 accumulation (|error| <= ~3 * 2^-18 |x w| per product), which is what
 *     keeps the stack within the 1e-4 parity budget at bf16 tensor-core rate.
 *
 * There is no CPU fallback anywhere in this library: on a machine without an sm_90 device
 * every compute entry point fails with XVB_ENODEVICE.
 */
#ifndef XVB200_H_
#define XVB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XVB_VERSION 100

/* error codes */
#define XVB_OK 0
#define XVB_EINVAL (-1)    /* bad argument (shape, alignment, null pointer) */
#define XVB_ECUDA (-2)     /* a CUDA runtime/driver call failed; see xvb_last_error() */
#define XVB_ENODEVICE (-3) /* no sm_90 GPU visible */
#define XVB_ESTATE (-4)    /* object used in the wrong state (e.g. extract before finalize) */

/* epilogue flags for xvb_tdnn_affine* (order is fixed: +bias -> ReLU -> swish -> BN affine -> tanh / sigmoid) */
#define XVB_RELU 1 /* components.py:410-416 (_relu_bn_forward): ReLU first ... */
#define XVB_BN 2   /* ... then eval-mode BatchNorm folded to y*scale[c] + shift[c] */
#define XVB_SIGMOID 4 /* ... then sigmoid (SE gate, ecapa_tdnn_xvector.py:97-106) */
#define XVB_TANH 8    /* ... then tanh (attention bottleneck, ecapa_tdnn_xvector.py:164-168) */
/* swish x * sigmoid(x), between ReLU and BN: the Conformer's feed-forward activation (transformer/
 * positionwise_feed_forward.py:31-34) and transform_out's swish before its norm (transformer_xvector.py:199).
 * xvb_tdnn_affine / xvb_tdnn_affine_ex layer epilogues only (not the fused pooling or histogram variants). */
#define XVB_SWISH 16

#define XVB_MAX_TAPS 16

int xvb_version(void);
const char* xvb_last_error(void);
/* 0 if the current device is sm_90 (H100); XVB_ENODEVICE otherwise. */
int xvb_device_check(void);

/* ---------------------------------------------------------------------------------------------
 * Frame-matrix staging
 * ------------------------------------------------------------------------------------------- */

/* fp32 (rows, C) with row pitch ldx  ->  split planes (rows, ldp); columns [C, ldp) are zeroed.
 * Replaces the torch.tensor(input)/unsqueeze/transpose staging of for_extract_embedding,
 * pytorch/libs/nnet/framework.py:28-33.  ldp % 8 == 0. */
int xvb_split_f32(const float* x, int64_t rows, int C, int64_t ldx, uint16_t* hi, uint16_t* lo, int64_t ldp,
                  void* stream);

/* Pack a TdnnAffine weight.  w: (Cout, Cin, tot_context) fp32 exactly as stored in the
 * reference state_dict, *including* the masked taps (pytorch/libs/nnet/components.py:62,
 * :78-83); only the taps listed in context[] are kept (the weight*mask of :133-138).
 * Output planes are K-major (Cout, ntaps*cin_p16) with cin_p16 = round_up(Cin,16) and
 * K index = tap*cin_p16 + c.  Size in elements: xvb_packed_weight_elems(). */
/* (B, T, C) fp32 frames -> split planes with `pad_front` / `pad_back` zero frames around every
 * utterance: planes are (B, pad_front + T + pad_back, ldp).  The zero frames are F.pad of
 * TdnnAffine.forward (components.py:117) made explicit, for the im2col view of xvb_tdnn_args_t. */
int xvb_split_frames(const float* x, int B, int T, int C, uint16_t* hi, uint16_t* lo, int64_t ldp, int pad_front,
                     int pad_back, void* stream);
/* xvb_split_frames over a masked batch: utterance b owns frames [0, lengths[b]) (DEVICE int32[B], 1 <= lengths[b] <= T);
 * the frames past them are written as zeros in both planes and never read.  XVB_EINVAL on a NULL lengths. */
int xvb_split_frames_lengths(const float* x, int B, int T, int C, uint16_t* hi, uint16_t* lo, int64_t ldp, int pad_front,
                             int pad_back, const int* lengths, void* stream);
int64_t xvb_packed_weight_elems(int Cout, int Cin, int ntaps);
int xvb_pack_tdnn_weight(const float* w, int Cout, int Cin, int tot_context, int left_context, const int* context_host,
                         int ntaps, uint16_t* w_hi, uint16_t* w_lo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * TDNN layer:  y[b,t,:] = epilogue( bias + sum_{c in context} W_c . x[b,t+c,:] ),  x = 0 outside
 * [0,T) -- TdnnAffine.forward (components.py:107-149) fused with ReLU/BatchNorm of
 * _BaseActivationBatchNorm (components.py:410-431).
 *
 * xvb_tdnn_affine: wgmma (bf16x3 split, fp32 accumulate in registers) GEMM with M = B*T frames,
 * K = ntaps*Cin, N = Cout; the context splice is done by TMA (3-D tensor map (C,T,B), time
 * coordinate offset per tap, out-of-bounds zero fill == F.pad).  Outputs: split planes
 * (y_hi,y_lo; may be NULL) and/or fp32 (y_f32; may be NULL); the TMA store clips ragged T / B /
 * Cout.  Requirements: ldx % 8 == 0, ldy % 8 == 0, ldyf % 4 == 0; pointers 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int xvb_tdnn_affine(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi,
                    const uint16_t* w_lo, const float* bias, const float* bn_scale, const float* bn_shift, int flags,
                    const int* context_host, int ntaps, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, float* y_f32,
                    int64_t ldyf, int B, int T, int Cin, int Cout, void* stream);

/* Extended form of the same kernel (everything xvb_tdnn_affine does, plus what ECAPA-TDNN and the
 * PLDA scorer need).  Zero-initialise the struct; unused pointers stay NULL.
 *   x2_*      : second A source with the same shape; computes W.(x + x2) by accumulating both
 *               sources into the same fp32 accumulator (Res2Net "sp + spx[i+1]",
 *               pytorch/model/ecapa_tdnn_xvector.py:66-71) -- no elementwise pass, no extra launch;
 *   row_bias  : per frame (B*T) additive term (PLDA row term);
 *   utt_bias  : per utterance x column (B, Cout) additive term, pitch ld_utt_bias (the
 *               time-constant [mean,std] part of AttentiveStatsPool's first conv, :173-180);
 *   both plane and fp32 outputs may be requested together. */
typedef struct xvb_tdnn_args {
  const uint16_t* x_hi; const uint16_t* x_lo; int64_t ldx;
  const uint16_t* x2_hi; const uint16_t* x2_lo; int64_t ldx2;
  const uint16_t* w_hi; const uint16_t* w_lo;
  const float* bias; const float* bn_scale; const float* bn_shift;
  const float* row_bias;
  const float* utt_bias; int64_t ld_utt_bias;
  int flags;
  const int* context_host; int ntaps;
  uint16_t* y_hi; uint16_t* y_lo; int64_t ldy;
  float* y_f32; int64_t ldyf;
  int B, T, Cin, Cout;
  /* Fused statistics pooling (no other output): the epilogue reduces each tile's frames per
   * utterance and writes [mean | centred sum of squares] partials, (num_blocks, B, 2*Cout) fp32 with
   * num_blocks = xvb_pool_partial_blocks(B, T, &frames_per_block); merge with xvb_pool_finalize. */
  float* pool_partial;
  /* 0: utterance b starts at row b*T of the x planes.  Otherwise the element distance between
   * utterances, and ldx may then be smaller than Cin: row t is the Cin-long window starting at
   * x[b*x_batch_stride + t*ldx] -- an im2col VIEW of consecutive context taps over a time-padded
   * frame matrix (ntaps = 1, Cin = taps*channels), so a [-2..2] layer over 80 channels streams 7
   * channel blocks of 64 instead of 5 x (64 + 16).  Requires x2_* == NULL. */
  int64_t x_batch_stride;
  /* 0 or 1: dense.  G > 1: grouped 1x1 convolution (Conv1d groups=G): output channels [g*Cout/G, (g+1)*Cout/G)
   * read only input channels [g*Cin/G, (g+1)*Cin/G) of x, and w is the COMPACT packing of the (Cout, Cin/G, 1)
   * weight (xvb_pack_tdnn_weight with Cin/G input channels), not its block-diagonal expansion.  Needs
   * xvb_tdnn_grouped_fits(Cin, Cout, G), one tap, and no x2, pool_partial, x_batch_stride or XVB_SWISH. */
  int groups;
  /* NULL, or a DEVICE int32[B] with 1 <= lengths[b] <= T: a masked batch of utterances of different lengths, utterance b
   * owning frames [0, lengths[b]).  The layer epilogue stores exact zeros (planes and fp32) for the frames past it, so
   * the next layer's context taps read the zero padding of F.pad (components.py:117).  The x planes must already hold
   * zeros past each utterance's end.  Not with pool_partial (pool a masked batch with xvb_stats_pool_lengths) or the
   * trial histogram. */
  const int* lengths;
} xvb_tdnn_args_t;
int xvb_tdnn_affine_ex(const xvb_tdnn_args_t* args, void* stream);
/* 1 when the grouped mode takes this shape: Cin/G a multiple of 64 and Cout/G a multiple of 32 (an N tile of
 * 128, 64 or 32 channels never straddles two groups); 0 otherwise -- such layers run as block-diagonal expansions. */
int xvb_tdnn_grouped_fits(int Cin, int Cout, int groups);
/* Time blocking the fused-pooling epilogue will use for a (B, T) batch. */
int xvb_pool_partial_blocks(int B, int T, int* frames_per_block);
/* Merge the fused-pooling partials into StatisticsPooling's output (mode as in xvb_stats_pool_ex):
 * Chan's parallel update over the time blocks, i.e. the two-pass result of pooling.py:58-67
 * without ever materialising the (B, T, C) tensor. */
int xvb_pool_finalize(const float* partial, int num_blocks, int frames_per_block, int B, int T, int C, float eps,
                      int mode, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* Same layer on CUDA cores in plain fp32 straight from the *unpacked* reference weight
 * (Cout, Cin, tot_context).  Slow; exists so the tensor-core path and the weight packer can
 * be cross-checked on the device and for shapes the wgmma path rejects. */
int xvb_tdnn_affine_simt(const float* x, int64_t ldx, const float* w, int tot_context, int left_context,
                         const float* bias, const float* bn_scale, const float* bn_shift, int flags,
                         const int* context_host, int ntaps, float* y, int64_t ldy, int B, int T, int Cin, int Cout,
                         void* stream);

/* ---------------------------------------------------------------------------------------------
 * Statistics pooling: StatisticsPooling.forward, no-lengths branch
 * (pytorch/libs/nnet/pooling.py:58-67): out[b, 0:C] = mean_t x, out[b, C:2C] =
 * sqrt(max(sum_t (x-mean)^2 / T, eps)).  x: (B, T, C) fp32 pitch ldx (ldx % 4 == 0, C % 4 == 0).
 * One HBM read of x.  out: (B, 2C) fp32; out_hi/out_lo (optional, pitch ldo % 8 == 0) receive
 * the same values as split planes for the following segment-level GEMM.
 * ------------------------------------------------------------------------------------------- */
int xvb_stats_pool(const float* x, int64_t ldx, int B, int T, int C, float eps, float* out, uint16_t* out_hi,
                   uint16_t* out_lo, int64_t ldo, void* stream);

/* mode 0 = xvb_stats_pool; mode 1 = the global context of ECAPA's AttentiveStatsPool
 * (pytorch/model/ecapa_tdnn_xvector.py:175-178): std = sqrt(unbiased_var + eps). */
int xvb_stats_pool_ex(const float* x, int64_t ldx, int B, int T, int C, float eps, int mode, float* out,
                      uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);
/* xvb_stats_pool_ex over a masked batch: utterance b pools its first lengths[b] frames (DEVICE int32[B],
 * 1 <= lengths[b] <= T); the frames past them are never read. */
int xvb_stats_pool_lengths(const float* x, int64_t ldx, int B, int T, int C, float eps, int mode, const int* lengths,
                           float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ECAPA-TDNN pieces that are not contractions (pytorch/model/ecapa_tdnn_xvector.py)
 * ------------------------------------------------------------------------------------------- */

/* Mean over time of a split-plane tensor (B,T,C) -> (B,C) fp32 and/or planes: the
 * AdaptiveAvgPool1d(1) of SE_Connect (:100).  C % 8 == 0. */
int xvb_plane_mean(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int B, int T, int C, float* out,
                   uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);
/* xvb_plane_mean over a masked batch: utterance b averages its first lengths[b] * rows_per_length rows (DEVICE
 * int32[B], 1 <= lengths[b] * rows_per_length <= T); the rows past them are never read.  A (B, T, F, C) position tensor
 * read as (B, T * F / k, k * C) rows takes rows_per_length = F / k (k dividing F). */
int xvb_plane_mean_lengths(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int B, int T, int C, const int* lengths,
                           int rows_per_length, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* Res2NetBlock.forward (pytorch/model/ecapa_tdnn_xvector.py:61-75) as ONE persistent kernel: chunk 0
 * of x passes through; step i = TDNN 128->128, context [-d,0,d], ReLU, BN on (x chunk i+1 [+ y chunk i]),
 * written to y chunk i+1.  A CTA owns whole utterances and walks them through all scale-1 steps, so the
 * serial chain needs no grid-wide synchronisation and no per-step launches.  x, y: split planes
 * (B,T,scale*128) with pitches ldx/ldy (distinct tensors).  w_hi/w_lo: the scale-1 packed weights
 * (xvb_pack_tdnn_weight, each (128, 3*128)) stacked along rows; bias/bn_scale/bn_shift: (scale-1, 128). */
int xvb_res2net_block(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi, const uint16_t* w_lo,
                      const float* bias, const float* bn_scale, const float* bn_shift, int dilation, int scale,
                      uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, int B, int T, void* stream);
/* The same block at Res2Net width `width` (channels per chunk), 64 or 128: x, y are (B,T,scale*width) with
 * ldx, ldy >= scale*width, the packed weights are each (width, 3*width) and the parameters (scale-1, width).
 * Any other width returns XVB_EINVAL with nothing launched.  xvb_res2net_block is width 128. */
int xvb_res2net_block_ex(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi, const uint16_t* w_lo,
                         const float* bias, const float* bn_scale, const float* bn_shift, int dilation, int scale,
                         uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, int B, int T, int width, void* stream);

/* Strided row copy (16-byte granularity): the pass-through of Res2Net's first chunk
 * (ecapa_tdnn_xvector.py:63-64) between two channel-slice views. */
int xvb_copy_rows(const void* src, int64_t src_pitch_bytes, void* dst, int64_t dst_pitch_bytes, int64_t rows,
                  int64_t row_bytes, void* stream);

/* out = z * gate[b,:] + in  and optionally next = in + out, all split planes (B,T,C): the SE
 * scaling + residual of SE_Res2Block.forward (:109-111, :149) fused with the running sums
 * x+x1, x+x1+x2 of ECAPA_TDNN.extract_embedding (:405-408).  gate: (B,C) fp32. */
int xvb_se_apply(const uint16_t* z_hi, const uint16_t* z_lo, int64_t ldz, const uint16_t* in_hi, const uint16_t* in_lo,
                 int64_t ldin, const float* gate, uint16_t* out_hi, uint16_t* out_lo, int64_t ldout, uint16_t* next_hi,
                 uint16_t* next_lo, int64_t ldnext, int B, int T, int C, void* stream);

/* AttentiveStatsPool.forward tail (:183-188): alpha = softmax_T(logits); mean = sum alpha x;
 * std = sqrt(max(sum alpha x^2 - mean^2, floor)); out (B,2C) = [mean | std].  One streaming pass
 * over logits and x (both (B,T,C) fp32) with an online softmax. */
int xvb_attn_stats_pool(const float* logits, int64_t ldl, const float* x, int64_t ldx, int B, int T, int C, float floor_,
                        float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* LDEPooling.forward (libs/nnet/pooling.py:130-162): x (B,T,C) fp32, dictionary mu (C,K) fp32 as the state_dict stores
 * it, neg_beta[k] = -(s_k^2 + eps); w[t,k] = softmax_k(neg_beta[k] * sum_c (x[t,c] - mu[c,k])^2) (distances summed directly
 * in fp32), out[b, c*K + k] = mean_t w[t,k] (x[t,c] - mu[c,k]); out (B, C*K) fp32, optionally also split planes.
 * w_scratch: (B*T, K) fp32.  K <= 64. */
int xvb_lde_pool(const float* x, int64_t ldx, int B, int T, int C, const float* mu, int K, const float* neg_beta,
                 float* w_scratch, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* Segment-level affine on CUDA cores, fp32 throughout: y[b,n] = epi(bias[n] + sum_k w[n,k] x[b,k]) for the few rows
 * (one per utterance) of the SE gate's two 1x1 convolutions (ecapa_tdnn_xvector.py:97-111), the time-constant half of
 * the attention's first conv (:179-181) and fc2 (:412-422).  x (B, >=K) fp32 pitch ldx, w (N, K) fp32 exactly as the
 * state_dict stores a kernel-size-1 conv weight; flags XVB_RELU | XVB_BN | XVB_SIGMOID | XVB_TANH applied in that
 * order after the bias; y fp32 (pitch ldy) and/or split planes (pitch ldplane).  K % 4 == 0. */
int xvb_small_affine(const float* x, int64_t ldx, const float* w, int B, int K, int N, const float* bias,
                     const float* bn_scale, const float* bn_shift, int flags, float* y, int64_t ldy, uint16_t* y_hi,
                     uint16_t* y_lo, int64_t ldplane, void* stream);

/* The attention poolings of libs/nnet/pooling.py with shared / per-head weights: AttentiveStatisticsPooling
 * (:322-368), MultiHeadAttentionPooling (:371-440), Global / MultiResolution multi-head (:443-587).  logits
 * (B,T,G) fp32 are the output of AttentionAlphaComponent's last affine (:300-319; temperature folded into its
 * weights); output channel o in [0,O) pools input channel o % C of x (B,T,C) with alpha = softmax_T(logits[:,:,o/gdiv]):
 * mean = sum alpha x, std = sqrt(max(sum alpha x^2 - mean^2, floor)) (unweighted_var = 1: the `stddev_attention=False`
 * branch, mean_T((x-mean)^2)).  out (B,2O) = [mean | std], optionally also as split planes. */
int xvb_attn_head_stats_pool(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T, int C,
                             int O, int gdiv, float floor_, int unweighted_var, float* out, uint16_t* out_hi,
                             uint16_t* out_lo, int64_t ldo, void* stream);
/* The xi-vector pooling (xivec_stdinit_softplus2_prec_pooling, pooling.py:165-212) on the same kernel: softplus2log = 1
 * turns the raw logit z (output of `lin2`) into a frame log-precision 2 log(softplus(z)) (:189-190); prior_logit / prior_x
 * (C each, may be NULL) add the prior as a (T+1)-th element of the softmax and of the weighted sums (:194-202).  out =
 * [phi | sqrt(max(sum w x^2 - phi^2, floor))]: the post-mean variant uses the first half. */
int xvb_attn_head_stats_pool_prior(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T, int C,
                                   int O, int gdiv, float floor_, int unweighted_var, const float* prior_logit,
                                   const float* prior_x, int softplus2log, float* out, uint16_t* out_hi, uint16_t* out_lo,
                                   int64_t ldo, void* stream);
/* xvb_attn_head_stats_pool_prior over a masked batch: utterance b reduces its first lengths[b] frames (DEVICE int32[B],
 * 1 <= lengths[b] <= T; the batch stride stays T rows of x and of the logits), so the softmax of the xi-vector form runs
 * over lengths[b] + 1 elements and the unweighted variance divides by lengths[b].  The frames past each end are never
 * read, and each row is bit-identical to a call on that utterance alone.  prior_logit / prior_x may be NULL (the plain
 * attention poolings).  XVB_EINVAL on a NULL lengths. */
int xvb_attn_head_stats_pool_lengths(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T,
                                     int C, int O, int gdiv, float floor_, int unweighted_var, const float* prior_logit,
                                     const float* prior_x, int softplus2log, const int* lengths, float* out, uint16_t* out_hi,
                                     uint16_t* out_lo, int64_t ldo, void* stream);
/* The same kernel with a head-width map, for multi-query multi-head attention pooling (MQMHASP, libs/nnet/pooling.py:589-
 * 698): x's C channels form C / head_width heads of head_width channels, each pooled `rep` times (once per query), so
 * output channel o pools x channel (o / (rep*head_width))*head_width + o % head_width with the alpha of logit o / gdiv.
 * head_width = C, rep = O / C is xvb_attn_head_stats_pool's map.  head_width % 4 == 0, O == rep * C. */
int xvb_attn_head_stats_pool_mq(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T, int C,
                                int O, int gdiv, int head_width, int rep, float floor_, int unweighted_var, float* out,
                                uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ResNet x-vector, 2-D (pytorch/model/resnet_xvector.py over pytorch/libs/nnet/resnet.py, BasicBlock)
 *
 * The reference convolves (B, 1, F, T): the conv "H" axis is the feature axis, "W" is time.  Position
 * tensors here are channel-contiguous (B, T, F, C) with row pitch C (dense); every conv pads by k/2
 * with zeros outside [0,F) x [0,T) of its own utterance and outputs ceil(F/s) x ceil(T/s) positions.
 * ------------------------------------------------------------------------------------------- */

/* Conv2d(Cin, Cout, k, stride s, padding k/2, bias=False) (resnet.py:12-20) on the wgmma kernel, split-plane
 * numerics as xvb_tdnn_affine_ex, with the block epilogues of BasicBlock (resnet.py:70-104):
 *   y  = [relu]( acc * scale[n] + shift[n]  [+ res] )      scale/shift: eval BatchNorm2d (NULL: none)
 *   y2 = relu( y * scale2[n] + shift2[n] )                 the next pre-activation block's bn1 + relu1
 * x: (B, T, F, Cin) planes; w: xvb_pack_tdnn_weight of the weight (Cout, Cin, k, k) viewed as (Cout, Cin, k*k)
 * with context 0..k*k-1 (tap = kf*k + kt); res, y, y2: (B, T', F', Cout) planes; y_f32 the same in fp32.
 * k in {1, 3}, s in {1, 2}, Cin % 16 == 0, Cout % 16 == 0, pointers 16-byte aligned.  Zero-initialise the struct;
 * unused pointers stay NULL; at least one of y, y_f32, y2 is required. */
typedef struct xvb_conv2d_args {
  const uint16_t* x_hi; const uint16_t* x_lo;
  const uint16_t* w_hi; const uint16_t* w_lo;
  int B, T, F, Cin, Cout, ksize, stride;
  const float* scale; const float* shift;
  const uint16_t* res_hi; const uint16_t* res_lo;
  int relu;
  uint16_t* y_hi; uint16_t* y_lo;
  float* y_f32;
  const float* scale2; const float* shift2;
  uint16_t* y2_hi; uint16_t* y2_lo;
  /* Time-axis stride: 0 means "same as stride" (every square-stride caller); 1 or 2 otherwise, with `stride` then the
   * feature-axis stride alone.  CAM++'s FCM head (subtools2/egrecho/models/campplus/campplus.py:60-80, :104-106) uses
   * stride (2, 1): feature 2, time 1, so T' = T and F' = ceil(F / 2). */
  int stride_t;
  /* NULL, or a DEVICE int32[B] with 1 <= lengths[b] <= T: a masked batch of utterances of different lengths, utterance b
   * owning input frames [0, lengths[b]).  Its output length follows the conv's own rule, L' = (L + 2 pad - k) / s_t + 1
   * (ceil(L / s_t) with pad = k / 2), and the epilogue stores exact zeros in y, y_f32 and y2 at every output frame
   * t >= L', so the next conv's taps read the utterance's own zero padding.  The x planes must already hold zeros at
   * the input frames t >= L.  Tiles are computed in full; only the stores differ.  Not with xvb_conv2d_valid. */
  const int* lengths;
} xvb_conv2d_args_t;
int xvb_conv2d(const xvb_conv2d_args_t* args, void* stream);

/* xvb_conv2d over a list of taps: only the taps in `taps` (host array, tap = kf*ksize + kt, strictly increasing,
 * 1 <= ntaps <= ksize*ksize) are computed; the others count as zero weights.  ksize in {1, 3, 5}, padding ksize/2,
 * output ceil(T/s) x ceil(F/s) as in xvb_conv2d.  w: xvb_pack_tdnn_weight of the weight viewed as (Cout, Cin, k*k)
 * with the tap list as context (packed tap j = taps[j]).  A re-parameterised RepSPK block (pytorch/libs/nnet/repvgg.py
 * RepSPKBlock) is a 5x5 kernel whose 8 off-pattern taps are zero: it runs with the other 17.  The dense list
 * 0..k*k-1 with ksize 1 or 3 gives xvb_conv2d's output bit for bit. */
int xvb_conv2d_taps(const xvb_conv2d_args_t* args, const int* taps, int ntaps, void* stream);

/* The head of ResNet._forward_impl (resnet.py:353-358): Conv2d(1, Cout, 3, 1, 1, bias=False) -> BatchNorm2d ->
 * ReLU on fp32 CUDA cores, straight from the (B, T, F) fp32 features (the unsqueeze of resnet_xvector.py:191 is
 * only a view).  w: (Cout, 1, 3, 3) fp32 as stored; y: (B, T, F, Cout) planes; y2 (optional) = relu(y * scale2 +
 * shift2), the first pre-activation block's bn1 + relu1.  Cout % 8 == 0. */
int xvb_conv2d_head(const float* x, int B, int T, int F, const float* w, int Cout, const float* bn_scale,
                    const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo, const float* scale2, const float* shift2,
                    uint16_t* y2_hi, uint16_t* y2_lo, void* stream);
/* xvb_conv2d_head over a masked batch (lengths: DEVICE int32[B], 1 <= lengths[b] <= T): the feature frames
 * t >= lengths[b] are read as zeros (never loaded), and y and y2 hold exact zeros there. */
int xvb_conv2d_head_lengths(const float* x, int B, int T, int F, const int* lengths, const float* w, int Cout,
                            const float* bn_scale, const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo,
                            const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream);

/* xvb_conv2d_head with a KxK window, ksize in {3, 5}, padding ksize/2: w is (Cout, 1, k, k) fp32.  ksize 3 is
 * xvb_conv2d_head.  A RepVGG / RepSPK stage0 block (Cin = 1) folds into this with bn_scale = 1 and bn_shift = its
 * bias. */
int xvb_conv2d_head_k(const float* x, int B, int T, int F, const float* w, int Cout, int ksize, const float* bn_scale,
                      const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo, const float* scale2, const float* shift2,
                      uint16_t* y2_hi, uint16_t* y2_lo, void* stream);

/* xvb_conv2d without padding: output (T - k) / s + 1 x (F - k) / s + 1, every tap inside the input (T, F >= k).
 * ksize in {1, 3}, stride in {1, 2}, everything else as xvb_conv2d (same kernel, same epilogue).  The second conv of
 * the Conformer's Conv2dSubsampling4 (pytorch/libs/nnet/transformer/subsampling.py:104-109: Conv2d(C, C, 3, 2) + ReLU)
 * with scale = 1, shift = its bias, relu = 1. */
int xvb_conv2d_valid(const xvb_conv2d_args_t* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Conformer x-vector (pytorch/model/transformer_xvector.py over pytorch/libs/nnet/transformer/): the pieces that are
 * not contractions.  Rows are channel-contiguous (B, T', C) frames of the subsampled sequence.
 * ------------------------------------------------------------------------------------------- */
#define XVB_ACT_NONE 0
#define XVB_ACT_RELU 1
#define XVB_ACT_SWISH 2 /* x * sigmoid(x) */
#define XVB_ACT_TANH 3

/* Conv2dSubsampling4's first conv (subsampling.py:104-106): Conv2d(1, C, 3, stride 2, no padding) + bias + ReLU in fp32
 * on CUDA cores.  The reference convolves (B, 1, T, F): x (B, T, F) fp32, w (C, 1, 3, 3) fp32 as stored (kt, kf);
 * y (B, T1, F1, C) planes with T1 = (T - 1) / 2, F1 = (F - 1) / 2.  T, F >= 3, C % 8 == 0. */
int xvb_subsample_head(const float* x, int B, int T, int F, const float* w, const float* bias, int C, uint16_t* y_hi,
                       uint16_t* y_lo, void* stream);
/* The same first conv with feature stride stride_f in {1, 2} (time stride 2): stride_f = 1 is SVConv2dSubsampling2's
 * Conv2d(1, C, 3, stride (2, 1)) (subsampling.py:365-415), F1 = F - 2; stride_f = 2 is xvb_subsample_head, bit for bit. */
int xvb_subsample_head_stride(const float* x, int B, int T, int F, const float* w, const float* bias, int C, int stride_f,
                              uint16_t* y_hi, uint16_t* y_lo, void* stream);

/* Residual update + LayerNorm over `rows` rows of C channels (C <= 8192), one pass:
 *   v     = x [+ table[row % table_rows]] [+ delta_scale * delta]     the residual adds of ConformerEncoderLayer
 *                                                                       (encoder_layer.py:248, :272, :293, :315) and
 *                                                                       PositionalEncoding's + pe (embedding.py:75)
 *   n1    = LN(v) [* gamma + beta]                                     eps as given (1e-5 everywhere in the model)
 *   x_out = second ? n1 : v                                            the new residual stream (may alias x)
 *   y     = act( second ? LN(n1) [* gamma2 + beta2] : n1 )             planes and/or fp32
 * second = 1 is norm_final followed by the next block's norm_ff_macaron (or after_norm).  gamma / beta NULL: a
 * LayerNorm without affine.  Zero-initialise the struct; unused pointers stay NULL. */
typedef struct xvb_layer_norm_args {
  int64_t rows; int C; float eps;
  const float* x; int64_t ldx;
  const float* delta; int64_t ld_delta; float delta_scale;
  const float* table; int table_rows;
  float* x_out; int64_t ld_x_out;
  const float* gamma; const float* beta;
  int second;
  const float* gamma2; const float* beta2;
  int act;
  uint16_t* y_hi; uint16_t* y_lo; int64_t ldy;
  float* y_f32; int64_t ldyf;
} xvb_layer_norm_args_t;
int xvb_layer_norm(const xvb_layer_norm_args_t* args, void* stream);

/* Multi-head self-attention over the fused Q/K/V projection, RoPESelfAttention / MultiHeadedAttention
 * (attention.py:120-154, :269-304) with AttentionNormalize (:640-728) at extraction (no mask):
 *   qkv (B, T, >= 3 H dk) fp32, row pitch ldq: [q | k | v], head h at columns h*dk of each;
 *   rope (T, dk) fp32 [sin | cos] (RoPositionalEncoding.pe[:T], embedding.py:162-192) or NULL: no rotation; when set,
 *     q and k are rotated as apply_rotary (:298-304), v too if rope_v;
 *   scores = (q . k / sqrt(dk)) * score_mult, softmax over keys: score_mult = 1 for softmax, (ln(T) / train_len + 1) - 1
 *     in fp32 for softmax_plus;
 *   y (B, T, H dk) planes = softmax . v, heads side by side (the input of linear_out).
 * dk in {32, 64, 128}; any T >= 1 (keys are tiled with an online softmax). */
int xvb_rope_attention(const float* qkv, int64_t ldq, int B, int T, int H, int dk, const float* rope, int rope_v,
                       float score_mult, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, void* stream);

/* ConvolutionModule.forward between its pointwise convs (convolution.py:110-125): x (B, T, >= 2C) fp32 = pointwise_conv1's
 * output; GLU a * sigmoid(b) over the two halves; depthwise Conv1d(C, C, K, padding K/2, groups C) with dw_w (C, K) and
 * dw_b (C), zero padding at the utterance's ends; norm 0: LayerNorm(C) with gamma norm_a, beta norm_b and eps; norm 1:
 * eval BatchNorm1d folded to y * norm_a + norm_b; then act; y (B, T, C) planes for pointwise_conv2.  K odd. */
int xvb_conv_module(const float* x, int64_t ldx, int B, int T, int C, const float* dw_w, const float* dw_b, int K,
                    const float* norm_a, const float* norm_b, int norm, float eps, int act, uint16_t* y_hi, uint16_t* y_lo,
                    int64_t ldy, void* stream);

/* y = [relu]( z * gate[b, c] + id ) over (B, P, C) planes (P positions per utterance): SEBlock_2D's scaling
 * (components.py:630-639) followed by BasicBlock's residual add (resnet.py:80-85 with relu, :100-104 without).
 * gate: (B, C) fp32 (the sigmoid output of the SE block); y planes and/or y_f32; y2 as in xvb_conv2d.  C % 8 == 0. */
int xvb_se_residual(const uint16_t* z_hi, const uint16_t* z_lo, const float* gate, const uint16_t* id_hi,
                    const uint16_t* id_lo, int B, int64_t P, int C, int relu, uint16_t* y_hi, uint16_t* y_lo, float* y_f32,
                    const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream);
/* xvb_se_residual over a masked batch of (B, T, F, C) planes (P = T * F): y, y_f32 and y2 hold exact zeros at the
 * positions of frames t >= lengths[b] (DEVICE int32[B], 1 <= lengths[b] <= T), whose z and identity are not read. */
int xvb_se_residual_lengths(const uint16_t* z_hi, const uint16_t* z_lo, const float* gate, const uint16_t* id_hi,
                            const uint16_t* id_lo, int B, int T, int F, int C, const int* lengths, int relu, uint16_t* y_hi,
                            uint16_t* y_lo, float* y_f32, const float* scale2, const float* shift2, uint16_t* y2_hi,
                            uint16_t* y2_lo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * CAM++ x-vector (subtools2/egrecho/models/campplus/campplus.py): the pieces of the densely connected D-TDNN layers that
 * are not contractions.  Frames are channel-contiguous (B, T', C) rows of the stride-2 `tdnn`'s output sequence.
 * ------------------------------------------------------------------------------------------- */

/* y = relu(x * scale[c] + shift[c]) over `rows` rows of C channels, split planes in and out, fp32 in between: the eval
 * BatchNorm1d + ReLU in front of every dense layer's linear1 (CAMDenseTDNNLayer.nonlinear1, :199, :212-213) and every
 * transit layer's 1x1 conv (TransitLayer, :262-271), which read the whole concatenation so far.  C % 8 == 0, pitches
 * ldx, ldy >= C and multiples of 8. */
int xvb_bn_relu_planes(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int64_t rows, int C, const float* scale,
                       const float* shift, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, void* stream);

/* CAMLayer's mask (:157-178) per segment: h (B, T, C) planes (pitch ldh) = the layer's bottleneck after BN2 + ReLU;
 * ctx[b, s] = mean_t h[b] + mean of h[b] over frames [s*seg_len, min(T, (s+1)*seg_len)) (avg_pool1d with ceil_mode: the
 * last segment divides by its valid frames); gate[b, s] = sigmoid(W2 relu(W1 ctx + b1) + b2), fp32 on CUDA cores, one CTA
 * per utterance.  w1 (R, C), w2 (G, R) fp32 as stored (linear1 / linear2 weights without the kernel axis).  gate: (B,
 * ceil(T / seg_len), G) fp32.  C % 8 == 0, C <= 2048. */
int xvb_cam_gate(const uint16_t* h_hi, const uint16_t* h_lo, int64_t ldh, int B, int T, int C, int seg_len, const float* w1,
                 const float* b1, int R, const float* w2, const float* b2, int G, float* gate, void* stream);

/* out = z * gate[b, t / seg_len, :] [+ in] over (B, T, C) planes: the kernel of xvb_se_apply with a gate row per
 * seg_len-frame segment (gate (B, ceil(T / seg_len), C) fp32, e.g. from xvb_cam_gate) and an optional `in` (NULL: no
 * add).  CAMLayer's y * m (:162) written straight into the layer's column slice of the block's concatenation buffer
 * (CAMDenseTDNNBlock.forward, :256-259); seg_len = T is xvb_se_apply without `next`.  C % 8 == 0, pitches % 8 == 0. */
int xvb_seg_gate_apply(const uint16_t* z_hi, const uint16_t* z_lo, int64_t ldz, const uint16_t* in_hi, const uint16_t* in_lo,
                       int64_t ldin, const float* gate, int seg_len, uint16_t* out_hi, uint16_t* out_lo, int64_t ldout, int B,
                       int T, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Feature-side front-end (SURVEY 8f rank 1) on a ragged batch: utterance u owns rows
 * offsets[u] .. offsets[u+1] of the (sum_T, F) fp32 matrix x.
 * ------------------------------------------------------------------------------------------- */

/* Energy VAD: TorchAsvExtractor::ComputeVadEnergy, runtime/extractor/torch_asv_extractor.cc:14-62
 * (column 0 = log-energy; threshold += mean_scale * mean(log-energy); a frame is voiced when at least
 * proportion_threshold of its +-frames_context neighbours exceed the threshold).  voiced: (sum_T)
 * bytes 0/1; voiced_counts: (U) number of voiced frames per utterance. */
int xvb_vad_energy(const float* x, const int32_t* offsets, int num_utts, int F, float energy_threshold,
                   float energy_mean_scale, int frames_context, float proportion_threshold, uint8_t* voiced,
                   int32_t* voiced_counts, void* stream);

/* Cepstral mean normalisation, no variance norm.  window <= 0: per-utterance mean
 * (torch_asv_extractor.cc:99-101).  window > 0: Kaldi apply-cmvn-sliding --center=true
 * --cmn-window=window as used by pytorch/pipeline/extract_xvectors_for_pytorch.sh:105-111. */
int xvb_cmn(const float* x, const int32_t* offsets, int num_utts, int F, int window, float* y, void* stream);

/* Keep the voiced frames of every utterance, order preserved (torch_asv_extractor.cc:103-107,
 * Kaldi select-voiced-frames).  out_offsets (U+1) = exclusive prefix sum of the voiced counts. */
int xvb_select_frames(const float* x, const int32_t* offsets, const uint8_t* voiced, const int32_t* out_offsets,
                      int num_utts, int F, float* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Back-end scoring
 * ------------------------------------------------------------------------------------------- */

/* y = (x - mean) / ||x - mean||_2 per row.  mean may be NULL.  Covers `submean` + `norm` of
 * score/process.sh:181-203 (ivector-subtract-global-mean, ivector-normalize-length
 * --scaleup=false). */
int xvb_center_length_norm(const float* x, const float* mean, float* y, int64_t rows, int D, void* stream);

/* Column mean of (rows, D): `getmean`, score/process.sh:169-179 (ivector-mean). */
int xvb_column_mean(const float* x, int64_t rows, int D, float* mean, void* stream);

/* Per-trial dot products: score/score.sh:82-97 (ivector-compute-dot-products).
 * scores[i] = <enroll[trial_e[i]], test[trial_t[i]]>. */
int xvb_cosine_trials(const float* enroll, const float* test, int D, const int32_t* trial_e, const int32_t* trial_t,
                      int64_t num_trials, float* scores, void* stream);

/* Per-speaker mean of embeddings: `mean` of score/process.sh:156-167 (ivector-mean ark:spk2utt).
 * CSR lists: speaker s owns rows members[offsets[s] .. offsets[s+1]) of x (N,D); out (S,D).
 * num_utts[s] = offsets[s+1]-offsets[s] is known to the caller. */
int xvb_speaker_mean(const float* x, int D, const int32_t* offsets, const int32_t* members, int num_spk, float* out,
                     void* stream);

/* Score normalisation (score/ScoreNormalization.py).  xvb_topn_mean_std: per row of a cohort score
 * matrix S (rows, ncoh), mean and unbiased std of the top_n largest entries (top_n <= 0: all) --
 * groupby().head(top_n) + .mean()/.std() of :151-166 (AS-norm) / :93-98 (S-norm).  xvb_snorm_trials:
 * out = 0.5*((s-mean_e[e])/std_e[e] + (s-mean_t[t])/std_t[t]) per listed trial (:101-104, :172-173). */
int xvb_topn_mean_std(const float* S, int64_t lds, int64_t rows, int ncoh, int top_n, float* mean, float* stdv,
                      void* stream);
/* The same with the divisor of the variance stated: ddof = 1 is pandas' .std() (ScoreNormalization.py:163-166),
 * ddof = 0 is np.std of subtools2/egrecho/score/asnorm.py:137-140 (`compute_cohort_stats`). */
int xvb_topn_mean_std_ddof(const float* S, int64_t lds, int64_t rows, int ncoh, int top_n, int ddof, float* mean,
                           float* stdv, void* stream);
int xvb_snorm_trials(const float* scores, const int32_t* trial_e, const int32_t* trial_t, int64_t num_trials,
                     const float* mean_e, const float* std_e, const float* mean_t, const float* std_t, float* out,
                     void* stream);

/* Per-trial bilinear scores with optional per-row / per-column terms:
 * scores[i] = <enroll[te[i]], test[tt[i]]> + row_term[te[i]] + col_term[tt[i]]  (terms may be NULL).
 * With enroll := E.(Lambda+Lambda^T) and the xvb_plda_terms() vectors this is PLDAScoring
 * (score/pyplda/gaussian-plda-scoring.py:23-29) for each listed trial (main loop :78-84). */
int xvb_bilinear_trials(const float* enroll, const float* test, int D, const int32_t* trial_e, const int32_t* trial_t,
                        int64_t num_trials, const float* row_term, const float* col_term, float* scores, void* stream);

/* y (rows, Dout) = x (rows, D) . M^T with M (Dout, D) row-major, Dout % 4 == 0: the small
 * projections of the back-end (PLDA's E.(Lambda+Lambda^T); `lda`/`whiten` transforms applied by
 * ivector-transform in score/process.sh:205-233).  Runs on the wgmma layer kernel. */
int xvb_project(const float* x, int64_t rows, int D, const float* M, int Dout, float* y, void* stream);

/* All-pairs score matrix S (Ne, Nt) = enroll . test^T (BASELINE config 4). */
int xvb_cosine_matrix(const float* enroll, int64_t Ne, const float* test, int64_t Nt, int D, float* S, int64_t lds,
                      void* stream);

/* Two-covariance PLDA, score/pyplda/gaussian-plda-scoring.py:23-29 in matrix form:
 * S[i,j] = e_i^T L2 t_j + row[i] + col[j],  L2 = Lambda + Lambda^T (D,D) fp32,
 * row = diag(E G E^T) + E c, col likewise (see xvb_plda_terms). */
int xvb_plda_terms(const float* x, int64_t rows, int D, const float* gamma, const float* c, float* term, void* stream);
int xvb_plda_matrix(const float* enroll, int64_t Ne, const float* test, int64_t Nt, int D, const float* L2,
                    const float* row, const float* col, float* S, int64_t lds, void* stream);

/* AS-norm with cross selection (score/ScoreNormalization.py:146-160, --cross-select true): the statistics of
 * the enroll side of trial (e, t) are taken over the cohort utterances that are the top_n of the TEST side and
 * vice versa.  xvb_topn_indices: idx (rows, top_n) int32 = cohort indices of every row's top_n scores, best
 * first (ncoh <= 16384); xvb_snorm_cross_trials: out[i] = 0.5 ((s - mu_e)/sd_e + (s - mu_t)/sd_t) with
 * mu_e, sd_e over enroll_cohort[e, top_test[t, :]] and mu_t, sd_t over test_cohort[t, top_enroll[e, :]],
 * std with ddof = 1 like pandas. */
int xvb_topn_indices(const float* S, int64_t lds, int64_t rows, int ncoh, int top_n, int32_t* idx, void* stream);
int xvb_snorm_cross_trials(const float* scores, const int32_t* trial_e, const int32_t* trial_t, int64_t num_trials,
                           const float* enroll_cohort, int64_t lde, const float* test_cohort, int64_t ldt,
                           const int32_t* top_enroll, const int32_t* top_test, int top_n, float* out, void* stream);

/* out (M, N) = a (M, K) . b (N, K)^T + row_bias[i] + col_bias[j] (biases may be NULL), fp32 row-major in
 * and out, N % 4 == 0: the general form behind xvb_project / xvb_cosine_matrix / xvb_plda_matrix. */
int xvb_matmul_nt(const float* a, int64_t M, const float* b, int64_t N, int K, const float* row_bias,
                  const float* col_bias, float* out, int64_t ldo, void* stream);

/* PLDA training on the GPU (score/pyplda/plda_base.py: PldaStats.add_samples :50-66, PldaEstimation
 * .get_stats_from_class_mean :262-287).  The D x D algebra (Cholesky, eigh, inverses) stays on the host in
 * float64; the O(N D^2) parts are Gram products X^T X, computed as xvb_matmul_nt(X^T, X^T) on transposed
 * operands these two kernels emit:
 *   xvb_center_rows_transposed: out[d][i] = sqrt_weight[spk[i]] * (x[i][d] - means[spk[i]][d])   (D, ldo >= N)
 *     -> offset_scatter = out . out^T  (the weighted within-class scatter, without the cancellation of
 *        sum x x^T - n m m^T);
 *   xvb_plda_em_rows: per class k, in the basis where within_var = I and between_var = diag(psi),
 *     what = n psi/(1 + n psi) * u;  what_T[d][k] = sqrt(w_k) what;  resid_T[d][k] = sqrt(w_k n_k) (u - what)
 *     -> the rank-one sums of one EM iteration are what_T . what_T^T and resid_T . resid_T^T. */
int xvb_center_rows_transposed(const float* x, const int32_t* spk, const float* means, const float* sqrt_weight,
                               int64_t N, int D, float* out, int64_t ldo, void* stream);
int xvb_plda_em_rows(const float* u, const float* n, const float* weight, const float* psi, int S, int D, float* what_T,
                     float* resid_T, int64_t ldo, void* stream);

/* Kaldi-style PLDA scoring in the diagonalised space, the arithmetic of ivector-plda-scoring as restated by the
 * reference's score/pyplda/plda_base.py (PLDA.transform_ivector :93-107, get_normalization_factor :151-158,
 * log_likelihood_ratio :109-136; called from score/score.sh:99-121 through the Kaldi binary):
 *   u = transform . x + offset                       -> xvb_matmul_nt with col_bias = offset
 *   u *= sqrt(D / sum_d u_d^2 / (psi_d + 1/n))       -> xvb_plda_normalize_rows (simple: sqrt(D)/||u||)
 *   LLR(i,j) = [t_j^2 | t_j] . [-1/(2 v_i) | m_i/v_i] + term_i + term_j,  m = n psi/(n psi+1) u, v = 1 + psi/(n psi+1)
 *     -> xvb_plda_llr_operands(side 0 = enroll with num_examples n, side 1 = test) writes the (rows, 2D) operand
 *        and the per-row term; the score matrix is xvb_matmul_nt(enroll_operand, test_operand, row, col), listed
 *        trials xvb_bilinear_trials. */
int xvb_plda_normalize_rows(float* u, const float* psi, const float* num_examples, int64_t rows, int D,
                            int simple_length_norm, void* stream);
int xvb_plda_llr_operands(const float* u, const float* psi, const float* num_examples, int64_t rows, int D, int side,
                          float* operand, float* term, void* stream);

/* Fused consumer for score matrices too large to store (BASELINE configs 4/5: 10^12 cosine trials,
 * 10^10 PLDA trials; SURVEY Appendix A "fused consumer"): every score
 *   s(i,j) = <enroll[i], test[j]> + row_term[i] + col_term[j]        (terms may be NULL)
 * is binned in the GEMM epilogue by trial class -- target when enroll_spk[i] == test_spk[j], the
 * trials file's third column (score/score.sh:82-97, computeEER.sh:21-22) -- and only the counters
 * leave the SM.  hist is (2, nbins) uint64 [nontarget | target] and is ACCUMULATED into (zero it
 * first; several calls / shards / GPUs add up).  Bins: w = (hi-lo)/(nbins-2);
 *   bin 0: s < lo;  bin k (1..nbins-2): lo+(k-1)w <= s < lo+kw;  bin nbins-1: s >= hi,
 * evaluated in fp32 as 1 + floor((s - lo) * ((nbins-2)/(hi-lo))).  4 <= nbins <= 2048.
 * symmetric != 0 (needs Ne == Nt, one set on both sides): only pairs j > i are counted, tiles
 * below the diagonal are skipped.  Row sharding for multi-GPU: this call walks the 256-row units
 * unit_first, unit_first + unit_stride, ... of enroll (rank r of W passes r, W). */
int xvb_trial_histogram(const float* enroll, int64_t Ne, const int32_t* enroll_spk, const float* test, int64_t Nt,
                        const int32_t* test_spk, int D, const float* row_term, const float* col_term, int symmetric,
                        int unit_first, int unit_stride, float lo, float hi, int nbins, unsigned long long* hist,
                        void* stream);

/* Speaker retrieval, task 2 of the CN-Celeb recipe (recipe/cnsrc/sr/run-cnsrc_sr.sh stage 4: all-pairs scores,
 * then trans_score_format.py's groupby('spk-id').nlargest(10, 'scores')): the k best test columns of every
 * enroll row, without storing the score matrix.  Order: higher score first; equal scores by lower column index
 * (nlargest(keep='first') over a score file in trials order, and xvb_topn_indices' rule).  1 <= k <= 256; at most
 * 2^31 - 1 columns in all.
 *
 * xvb_topk_merge: merges the columns of a score slab S (rows, ncols), pitch lds (a multiple of 4, S 16-byte aligned),
 * whose column j is column col0 + j of the full test set, into running per-row lists top_score (rows, k) fp32 /
 * top_idx (rows, k) int64, sorted best first.  Start the lists at (-inf, -1): a row that has seen fewer than k columns
 * keeps (-inf, -1) in its empty slots.  A column that does not beat a row's k-th entry is dropped without a sort.
 * A NaN score is never ranked: the row index is atomicMin'ed into *nan_row (device; set it to ~0 first).
 *
 * xvb_retrieve_topk: out (M, k) = the k best columns of a (M, K) . b (N, K)^T + row_bias[i] + col_bias[j] (biases may
 * be NULL).  Walks b in slabs of slab_cols rows (a positive multiple of 4): each slab is scored by xvb_matmul_nt into
 * `slab` (xvb_retrieve_topk_slab_bytes(M, slab_cols) bytes, 16-byte aligned, pitch slab_cols) and merged by
 * xvb_topk_merge, so the scores ranked are the bytes xvb_matmul_nt writes.  Any N: the last 1..3 test rows are scored
 * from a zero-padded copy and the padded columns are not merged.  Cosine: length-normalised rows, NULL biases.
 * Kaldi PLDA: the xvb_plda_llr_operands operands and terms (enroll side 0 -> a, row_bias; test side 1 -> b, col_bias).
 * The layer epilogue turns a NaN accumulator into -inf, so the operands and terms are checked first: a NaN or infinity
 * in a / row_bias or b / col_bias returns XVB_EINVAL naming the enroll or test row, as does a NaN that reaches a slab,
 * and like a bad argument writes nothing to out_score / out_idx.  The refusal covers non-finite inputs only: finite
 * operands whose products overflow fp32 make an infinite or NaN accumulator, which is stored as +inf or -inf and
 * ranked as such.  To know, the call synchronises `stream` once at the end. */
int xvb_topk_merge(const float* S, int64_t lds, int64_t rows, int64_t ncols, int64_t col0, int k, float* top_score,
                   int64_t* top_idx, uint64_t* nan_row, void* stream);
/* Bytes of the slab buffer xvb_retrieve_topk needs (M * slab_cols * 4), or XVB_EINVAL. */
int64_t xvb_retrieve_topk_slab_bytes(int64_t M, int64_t slab_cols);
int xvb_retrieve_topk(const float* a, int64_t M, const float* b, int64_t N, int K, const float* row_bias,
                      const float* col_bias, int k, float* slab, int64_t slab_cols, float* out_score, int64_t* out_idx,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor (x-vector TDNN family): owns packed weights + workspace on the current
 * device; replaces Xvector.extract_embedding (pytorch/model/xvector.py:77-98) for a whole batch
 * of equal-length utterances, and the model-loading role of runtime/ (torch_asv_model.cc:8-17).
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_extractor xvb_extractor_t;

int xvb_extractor_create(xvb_extractor_t** out, int feat_dim);
/* Append a frame-level layer (before pooling) / a segment-level layer (after pooling).
 * w_host: (Cout, Cin, tot_context) fp32 host; bias_host (Cout) or NULL; bn_scale_host/
 * bn_shift_host (Cout) or NULL (folded eval BatchNorm); flags: XVB_RELU | XVB_BN. */
int xvb_extractor_add_frame_layer(xvb_extractor_t* h, int Cout, const int* context_host, int ntaps,
                                  const float* w_host, const float* bias_host, const float* bn_scale_host,
                                  const float* bn_shift_host, int flags);
int xvb_extractor_add_segment_layer(xvb_extractor_t* h, int Cout, const float* w_host, const float* bias_host,
                                    const float* bn_scale_host, const float* bn_shift_host, int flags);
int xvb_extractor_finalize(xvb_extractor_t* h, float pooling_eps);
int xvb_extractor_embed_dim(const xvb_extractor_t* h);
/* feats (B, T, feat_dim) fp32 on the device -> emb (B, embed_dim) fp32 on the device. */
int xvb_extractor_extract(xvb_extractor_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* A batch of utterances of different lengths: feats (B, T, feat_dim) fp32 on the device, utterance b in its first
 * lengths_host[b] frames (HOST int32[B], 1 <= lengths_host[b] <= T; the frames past them are never read, whatever they
 * hold).  Row b of emb is the embedding of feats[b, :lengths_host[b]] extracted alone, up to the rounding of the
 * pooling merge order.  A batch with lengths below T pools with xvb_stats_pool_lengths after an fp32 last frame layer,
 * whatever xvb_extractor_set_fused_pooling says (the fused pooling epilogue takes equal lengths only).  The lengths are checked (XVB_EINVAL naming the first bad one) and copied into a device buffer
 * of the extractor on `stream`; the host array may be reused when the call returns.  With every length equal to T the
 * result equals xvb_extractor_extract bit for bit. */
int xvb_extractor_extract_lengths(xvb_extractor_t* h, const float* feats, const int32_t* lengths_host, int B, int T,
                                  float* emb, void* stream);
/* Same through host buffers (H2D of feats, D2H of emb inside; synchronises the stream). */
int xvb_extractor_extract_host(xvb_extractor_t* h, const float* feats_host, int B, int T, float* emb_host,
                               void* stream);
/* Pipelined host-buffer path: submit returns as soon as the work is queued (H2D on a private copy
 * stream into one of two device slots, the stack and the D2H on `stream`), so the host->device
 * copy of batch i+1 overlaps the kernels of batch i.  feats_host / emb_host must stay valid (and
 * should be pinned) until xvb_extractor_wait(h, slot) returns.  Typical loop:
 *   submit(batch0, slot0); for i>=1 { submit(batch_i, i&1); wait((i-1)&1); } wait(last). */
int xvb_extractor_submit_host(xvb_extractor_t* h, const float* feats_host, int B, int T, float* emb_host, int slot,
                              void* stream);
int xvb_extractor_wait(xvb_extractor_t* h, int slot);
/* A whole shard of N equal-length utterances -- the caller loop of the reference
 * (pytorch/pipeline/onestep/extract_embeddings.py:73-83, one utterance per iteration; sharded over `nj` jobs by
 * extract_xvectors_for_pytorch.sh:125-136) as ONE call: ceil(N / batch) batches through the stack.  One protocol for
 * the TDNN, ECAPA-TDNN and ResNet handles:
 *   _shard      : feats (N, T, feat_dim) and emb (N, embed_dim) on the device; asynchronous on `stream`;
 *   _shard_host : the same through host buffers (pinned, so that the copies overlap): batch k crosses the link on a
 *                 copy stream into device slot k % 4 while earlier batches run; returns when emb_host is complete.
 *                 Refused while a submit_host slot is in flight.
 * Batch k runs on lane k & 1: the handle itself and a twin on the same weights with its own workspace (made on first
 * use, kept until destroy), each on its own stream forked from `stream` and joined back into it.  There are two lanes
 * only when N > batch; XVB_LANES=0 in the environment (read on every call) and per-kernel profiling keep one lane,
 * on `stream`.  Launch plans (tensor maps, tile geometry) are cached per batch shape, so a batch costs its launches
 * only; last_launches after a shard call is the sum over its batches, xvb_scatter_rows launches included. */
int xvb_extractor_extract_shard(xvb_extractor_t* h, const float* feats, int64_t N, int T, int batch, float* emb,
                                void* stream);
int xvb_extractor_extract_shard_host(xvb_extractor_t* h, const float* feats_host, int64_t N, int T, int batch,
                                     float* emb_host, void* stream);
/* ---------------------------------------------------------------------------------------------
 * The embedding table of BASELINE configs[3] on every GPU of a node without a collective after extraction
 * (SURVEY 8e; replaces the `cat xvector.*.scp` of extract_xvectors_for_pytorch.sh:147-151 and the NCCL all-gather
 * of the plain path).  Each rank allocates its copy of the (world x n, D) table with xvb_ipc_alloc, exports it
 * (64-byte CUDA IPC handle, exchanged by the caller -- torch.distributed, MPI, a file), and maps its peers' copies
 * with xvb_ipc_open (NVLink peer access).  xvb_extractor_set_gather / xvb_ecapa_set_gather then make the shard calls
 * store every batch's embeddings into ALL copies at row0 + (row inside the shard) as soon as the batch's last layer
 * has produced them (xvb_scatter_rows on the batch's stream), overlapped with the following batches; the caller ends
 * the step with a barrier.  tables[k], k < ntables: base pointers valid in THIS process (own copy included);
 * ntables = 0 turns it off.  `emb` of the shard call still receives the rank's own rows.  Every batch of every shard
 * call stores, on one lane or two, with profiling on or off; each store is one launch in last_launches.
 * ------------------------------------------------------------------------------------------- */
#define XVB_MAX_PEERS 16
#define XVB_IPC_HANDLE_BYTES 64
int xvb_ipc_alloc(void** ptr, size_t bytes);
int xvb_ipc_free(void* ptr);
int xvb_ipc_export(void* ptr, void* handle64);
int xvb_ipc_open(const void* handle64, void** ptr);
int xvb_ipc_close(void* ptr);
int xvb_scatter_rows(const float* src, int64_t rows, int D, float* const* tables, int ntables, int64_t row0, int64_t ld,
                     void* stream);
int xvb_extractor_set_gather(xvb_extractor_t* h, float* const* tables, int ntables, int64_t row0, int64_t ld);

/* Per-kernel timing with CUDA events recorded on the launching stream around every kernel of
 * the next extract calls.  xvb_extractor_kernel_times() waits for the last call and returns the
 * number of kernels n (<= max_n) and their durations in ms, in launch order: split, frame layers,
 * stats pooling, segment layers.  After xvb_extractor_extract_shard the events of ALL its batches are kept: per batch
 * the same kernel intervals followed by the interval to the next batch's first event. */
int xvb_extractor_set_profiling(xvb_extractor_t* h, int enable);
int xvb_extractor_kernel_times(xvb_extractor_t* h, float* ms_host, int max_n);
/* Fused pooling (default on): the last frame layer's epilogue reduces over time itself and the
 * (B,T,C_last) fp32 tensor is never written.  Off: last layer -> fp32 -> xvb_stats_pool. */
int xvb_extractor_set_fused_pooling(xvb_extractor_t* h, int enable);
/* Number of kernels the last extract call launched (bench.py's gpu_launches). */
int xvb_extractor_last_launches(const xvb_extractor_t* h);
/* Device pointer/pitch of a frame layer's fp32 output from the last call (debug/tests; only
 * the last frame layer keeps fp32), or the pooled statistics (layer = -1). */
const float* xvb_extractor_debug_f32(const xvb_extractor_t* h, int which);
void xvb_extractor_destroy(xvb_extractor_t* h);

/* ---------------------------------------------------------------------------------------------
 * Kaldi-compatible fbank / MFCC from raw waveforms (the feature step of the reference's online
 * path: KaldiFeature, pytorch/libs/egs/kaldi_features.py:69-135 -> torchaudio.compliance.kaldi
 * fbank/mfcc; C++ runtime: runtime/kaldifeat/csrc/feature-fbank.cc).  snip_edges framing, no
 * dither (the launchers force dither = 0 for extraction), no VTLN, window rounded up to 2^k.
 * Field names and defaults are torchaudio's / Kaldi's.  num_ceps > 0 selects MFCC.
 * ------------------------------------------------------------------------------------------- */
#define XVB_WINDOW_POVEY 0
#define XVB_WINDOW_HAMMING 1
#define XVB_WINDOW_HANNING 2
#define XVB_WINDOW_RECTANGULAR 3
#define XVB_WINDOW_BLACKMAN 4
typedef struct {
  float sample_frequency, frame_length_ms, frame_shift_ms, preemphasis_coefficient, low_freq, high_freq,
      energy_floor, cepstral_lifter, blackman_coeff;
  int num_mel_bins, num_ceps, use_energy, raw_energy, remove_dc_offset, use_log_fbank, use_power, htk_compat,
      window_type;
} xvb_fbank_opts_t;
typedef struct xvb_fbank xvb_fbank_t;
void xvb_fbank_default_opts(xvb_fbank_opts_t* opts);
/* Builds window / twiddle / mel / DCT tables (double precision, stored fp32) on the current device. */
int xvb_fbank_create(xvb_fbank_t** out, const xvb_fbank_opts_t* opts);
int xvb_fbank_dim(const xvb_fbank_t* h);                            /* columns of the feature matrix */
int64_t xvb_fbank_num_frames(const xvb_fbank_t* h, int64_t num_samples); /* 1 + (n - window) / shift, or 0 */
/* wave: all utterances back to back (device, fp32, Kaldi i.e. int16-range scale if the model was
 * trained that way); sample_offsets (U+1) int64 and frame_offsets (U+1) int32 on the device, with
 * frame_offsets[u+1]-frame_offsets[u] = xvb_fbank_num_frames(len_u); feats (total_frames, dim). */
int xvb_fbank_compute(xvb_fbank_t* h, const float* wave, const int64_t* sample_offsets, const int32_t* frame_offsets,
                      int num_utts, int64_t total_frames, float* feats, void* stream);
void xvb_fbank_destroy(xvb_fbank_t* h);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor for ECAPA-TDNN (pytorch/model/ecapa_tdnn_xvector.py, ECAPA_TDNN.extract_embedding
 * :403-426; canonical c1024 parameters runEcapaXvector_online.py:221-263).  Layers are set by name with the
 * weights as the state_dict stores them (host fp32 (Cout, Cin, tot_context); eval BatchNorm folded to
 * scale/shift; flags XVB_RELU | XVB_BN):
 *   "layer1"; for L in 2..4: "layerL.bn1", "layerL.res0".."layerL.res6" (W -> W, [-d,0,d], W = channels / 8),
 *   "layerL.bn2", "layerL.se1" (ReLU), "layerL.se2"; "mfa"; "att_x" = the first attention conv's columns
 *   over x with its ReLU + BatchNorm, "att_gs" = its columns over [mean | std] plus its bias (:179),
 *   "att2"; "fc2" with bn_stats folded into the weight (and fc2's own BatchNorm for position "near").
 * channels must be 512 or 1024 (Res2Net scale 8 x width 64 or 128, the chain kernel's two instances: ECAPA C512
 * and C1024).
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_ecapa xvb_ecapa_t;
int xvb_ecapa_create(xvb_ecapa_t** out, int feat_dim, int channels, int mfa_dim, int att_hidden, int embed_dim);
/* Multi-query multi-head attention pooling (MQMHASP, libs/nnet/pooling.py:589-698) instead of the attentive one: call
 * between create and the first set_layer, with att_hidden = hidden * num_head * num_q.  Then "att_x" is the first
 * attention conv's x columns as stored, (Cout, mfa_dim / num_head, 1) with groups = num_head (its ReLU + BatchNorm when
 * affine_layers = 2; the logits themselves when 1); "att_gs" (time_attention only) its [mean_h | std_h] columns as a
 * block-diagonal (Cout, 2*mfa_dim) matrix over [mean | std] ((Cout, mfa_dim) over the mean without stddev) plus its
 * bias; "att2" (affine_layers = 2) the second conv, (logits, hidden, 1) with groups = num_head * num_q.  fc1 / fc2 read
 * the 2 * num_q * mfa_dim pooled statistics (num_q * mfa_dim without stddev). */
int xvb_ecapa_set_mqmha(xvb_ecapa_t* h, int num_head, int num_q, int hidden, int share, int affine_layers, int time_attention,
                        int stddev);
/* Residual form of the three SE-Res2Net blocks: 0 (the default) is ECAPA_TDNN's dense form, block 2 reading x + x1 and
 * block 3 x + x1 + x2; 1 is egrecho's EcapaXvector (subtools2/egrecho/models/ecapa/ecapa_xvector.py:420-427), each block
 * reading the previous block's output.  Call between create and the first set_layer; the layers are the same. */
int xvb_ecapa_set_chained(xvb_ecapa_t* h, int chained);
/* The attentive pooling of the default model: global_context = 1 with floor 1e-5 (the default) is ECAPA_TDNN's, attention
 * conv 1 reading [x | mean | std] ("att_x" + "att_gs") and the pooled std floored at variance 1e-5; global_context = 0 is
 * the AttentiveStatsPool of pytorch/model/ecapa-tdnn-xvector.py:120-134, alpha = softmax(att2(tanh(att_x(x)))) with
 * "att_x" the first conv with its own bias and no ReLU or BatchNorm, no "att_gs", and the std floored at `floor`
 * (1e-9 there).  Call between create and the first set_layer; not with xvb_ecapa_set_mqmha or xvb_ecapa_set_chained. */
int xvb_ecapa_set_attention(xvb_ecapa_t* h, int global_context, float floor);
int xvb_ecapa_set_layer(xvb_ecapa_t* h, const char* name, int Cout, int Cin, const int* context_host, int ntaps,
                        const float* w_host, const float* bias_host, const float* bn_scale_host,
                        const float* bn_shift_host, int flags);
int xvb_ecapa_finalize(xvb_ecapa_t* h);
int xvb_ecapa_embed_dim(const xvb_ecapa_t* h);
int xvb_ecapa_feat_dim(const xvb_ecapa_t* h);
/* feats (B, T, feat_dim) fp32 on the device -> emb (B, embed_dim) fp32 on the device; asynchronous. */
int xvb_ecapa_extract(xvb_ecapa_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* Same through host buffers (H2D of feats, D2H of emb inside; synchronises the stream). */
int xvb_ecapa_extract_host(xvb_ecapa_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream);
/* Whole shard of N equal-length utterances in `batch`-utterance batches (extract_embeddings.py:73-83's loop as one
 * call): device-resident and asynchronous, or through pinned host buffers with the copies overlapped; the protocol of
 * xvb_extractor_extract_shard[_host]. */
int xvb_ecapa_extract_shard(xvb_ecapa_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream);
/* the replicated-table form of the shard calls, see xvb_extractor_set_gather */
int xvb_ecapa_set_gather(xvb_ecapa_t* h, float* const* tables, int ntables, int64_t row0, int64_t ld);
int xvb_ecapa_extract_shard_host(xvb_ecapa_t* h, const float* feats_host, int64_t N, int T, int batch, float* emb_host,
                                 void* stream);
int xvb_ecapa_last_launches(const xvb_ecapa_t* h);
/* "XVBE0001" model files: the named layers as handed to xvb_ecapa_set_layer; "XVBE0002" for MQMHA models adds the
 * xvb_ecapa_set_mqmha record; "XVBG0001" for chained models (egrecho's, MQMHA pooling only) adds the residual form
 * after it; "XVBE0003" for an attention other than the default adds the xvb_ecapa_set_attention record to XVBE0001's
 * header.  All four load. */
int xvb_ecapa_save(const xvb_ecapa_t* h, const char* path);
int xvb_ecapa_load(xvb_ecapa_t** out, const char* path);
void xvb_ecapa_destroy(xvb_ecapa_t* h);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor for the 2-D ResNet x-vector (pytorch/model/resnet_xvector.py, extract_embedding :183-208,
 * BasicBlocks in either block order, optional SE, statistics pooling): the launch sequence of xvb_conv2d_head,
 * xvb_conv2d, xvb_plane_mean / xvb_small_affine / xvb_se_residual, xvb_stats_pool_ex and xvb_tdnn_affine_ex in
 * C++, with weights and workspace owned by the handle.  Bit-identical to the op-by-op Python driver of the same
 * kernels (ResNetExtractor, XVB_RESNET_NATIVE=0).
 *
 * Records are named by their state_dict module path: "resnet.conv1", "resnet.bn1", "resnet.layerL.i.{conv1,bn1,
 * conv2,bn2}", "resnet.layerL.0.downsample.{0,1}", "resnet.layerL.i.se.fc_{1,2}", "fc1", "fc2".  Convolutions:
 * w_host (Cout, Cin, k, k) as stored, ksize k in {1, 3}, no bias; BatchNorm: ksize 0, Cin 0, w_host NULL, the eval
 * BatchNorm folded to scale / shift; SE linears: ksize 1, w (Cout, Cin) with bias; segment layers "fc1" / "fc2": the
 * ones the extracted position uses, ksize 1, weight (Cout, Cin) with bias, scale / shift (XVB_BN) and XVB_RELU as
 * the layer applies them, the first one's input columns in the pooling order of (B, T', F', C) frames (column
 * f*C + c of each [mean | std] half).  The library pads the SE hidden width to a multiple of 4 and the segment rows
 * to a multiple of 8, and packs the convolutions itself.
 *
 * Workspace: grown to the largest (B, T) seen, then reused.  A call whose B*T*feat_dim exceeds 256*200*80
 * positions runs as consecutive groups of max(1, floor(256*200*80 / (T*feat_dim))) utterances, so the workspace of
 * one call stays within that budget (a single utterance longer than the budget is one group of its own).  At
 * B = 128, T = 200, feat_dim = 80 with planes 32..256 it is about 1.9 GB: seven (B, T', F', C) plane pairs of
 * 262 MB each, plus the last layer's fp32 output; the shard calls' second lane holds a second workspace.
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_resnet xvb_resnet_t;
/* layers, planes: four entries each (planes multiples of 16); pre_activation != 0: full_pre_activation blocks. */
int xvb_resnet_create(xvb_resnet_t** out, int feat_dim, const int* layers, const int* planes, int pre_activation,
                      float pooling_eps);
int xvb_resnet_set_layer(xvb_resnet_t* h, const char* name, int Cout, int Cin, int ksize, const float* w_host,
                         const float* bias_host, const float* scale_host, const float* shift_host, int flags);
/* Checks that every record the configuration needs is present with its shape (and nothing else), names the one
 * that is not, then packs the weights on the current device. */
int xvb_resnet_finalize(xvb_resnet_t* h);
int xvb_resnet_feat_dim(const xvb_resnet_t* h);
int xvb_resnet_embed_dim(const xvb_resnet_t* h);
/* Kernels launched by the last extract / shard call. */
int xvb_resnet_last_launches(const xvb_resnet_t* h);
/* feats (B, T, feat_dim) fp32 on the device -> emb (B, embed_dim) fp32 on the device; asynchronous. */
int xvb_resnet_extract(xvb_resnet_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* A batch of utterances of different lengths: feats (B, T, feat_dim) fp32 on the device, utterance b in its first
 * lengths_host[b] frames (HOST int32[B], 1 <= lengths_host[b] <= T; the frames past them are never read, whatever they
 * hold).  Row b of emb is the embedding of feats[b, :lengths_host[b]] extracted alone, up to the rounding of the
 * pooling merge order and of the SE mean's position grouping (chosen from F' alone in a masked batch).  Every conv,
 * SE scaling and the head conv store zeros past each utterance's length at their resolution (ceil(L / 2) per
 * stride-2 stage), and each utterance pools its own frames.  The lengths are checked (XVB_EINVAL naming the first bad
 * one) and copied, with the per-stage lengths, into the workspace on `stream`; the host array may be reused when the
 * call returns.  The position budget splits the call into groups as xvb_resnet_extract does.  With every length equal
 * to T the result equals xvb_resnet_extract bit for bit. */
int xvb_resnet_extract_lengths(xvb_resnet_t* h, const float* feats, const int32_t* lengths_host, int B, int T, float* emb,
                               void* stream);
/* Same through host buffers (H2D of feats, D2H of emb inside; synchronises the stream). */
int xvb_resnet_extract_host(xvb_resnet_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream);
/* Whole shard of N equal-length utterances in `batch`-utterance batches: the protocol of
 * xvb_extractor_extract_shard[_host]. */
int xvb_resnet_extract_shard(xvb_resnet_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream);
int xvb_resnet_extract_shard_host(xvb_resnet_t* h, const float* feats_host, int64_t N, int T, int batch,
                                  float* emb_host, void* stream);
/* "XVBR0001" model files: the create arguments, then the records as handed to xvb_resnet_set_layer (layout at
 * save_records in csrc/model_file.cpp). */
int xvb_resnet_save(const xvb_resnet_t* h, const char* path);
int xvb_resnet_load(xvb_resnet_t** out, const char* path);
void xvb_resnet_destroy(xvb_resnet_t* h);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor for the RepVGG / RepSPK x-vector (pytorch/model/repvgg_xvector.py, extract_embedding :181-208
 * over pytorch/libs/nnet/repvgg.py): the launch sequence of xvb_conv2d_head[_k], xvb_conv2d_taps, xvb_stats_pool_ex and
 * xvb_tdnn_affine_ex in C++, with weights and workspace owned by the handle.  Bit-identical to the op-by-op Python
 * driver of the same kernels (RepVGGExtractor, XVB_REPVGG_NATIVE=0).
 *
 * Every block is one convolution with a bias and ReLU.  Records are named by block module path and arrive folded:
 *   "repvgg.stage0", "repvgg.stageS.I"   Cout x Cin x k: w (Cout, Cin, k, k) the block's equivalent kernel (branches
 *                                        folded in float64, groups expanded block-diagonally, then cast to fp32), bias
 *                                        the folded bias, flags XVB_RELU; stage0 has Cin = 1.  Training-form and
 *                                        deploy-form checkpoints give the same records.
 *   "fc1", "fc2"                         as for xvb_resnet_set_layer: the ones the extracted position uses, ksize 1,
 *                                        the first one's input columns in the pooling order of (B, T', F', C) frames.
 * Finalize drops every tap whose (Cout, Cin) slab of a block's kernel is exactly zero (xvb_conv2d_kept_taps: 17 of the
 * 25 taps of a RepSPK block) and packs the rest.  stage0 runs on xvb_conv2d_head (k = 3) or xvb_conv2d_head_k (k = 5)
 * with scale 1 and shift = the bias, every other block on xvb_conv2d_taps with the same epilogue (the last block writes
 * fp32 only).
 *
 * Workspace: grown to the largest (B, T) seen, then reused: two ping-pong (B, T', F', C) plane pairs, the last block's
 * fp32 output, the pooled statistics and the segment layers.  A call whose B*T*feat_dim exceeds 256*200*80 positions
 * runs as consecutive groups of max(1, floor(256*200*80 / (T*feat_dim))) utterances.  The launcher's model (RepSPK,
 * base width 32) at B = 128, T = 200, feat_dim = 80 needs about 0.6 GB: 262 MB per plane pair at stage0 / stage1 widths
 * and 82 MB of fp32 for stage4's output.
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_repvgg_config {
  int feat_dim;
  int ksize;             /* 3: RepVGG blocks, 5: RepSPK blocks */
  int num_blocks[4];     /* blocks of stage1 .. stage4 (stage0 is one block) */
  int strides[5];        /* stage0 .. stage4, 1 or 2; stage0 1 (the head conv) */
  int widths[5];         /* output channels of stage0 .. stage4, multiples of 16 */
  float pooling_eps;
} xvb_repvgg_config_t;
typedef struct xvb_repvgg xvb_repvgg_t;
/* Refuses a configuration outside the bounds above, naming the field. */
int xvb_repvgg_create(xvb_repvgg_t** out, const xvb_repvgg_config_t* cfg);
int xvb_repvgg_set_layer(xvb_repvgg_t* h, const char* name, int Cout, int Cin, int ksize, const float* w_host,
                         const float* bias_host, const float* scale_host, const float* shift_host, int flags);
/* Checks that every record the configuration needs is present with its shape (and nothing else), names the one that
 * is not, then prunes the taps and packs the weights on the current device. */
int xvb_repvgg_finalize(xvb_repvgg_t* h);
int xvb_repvgg_feat_dim(const xvb_repvgg_t* h);
int xvb_repvgg_embed_dim(const xvb_repvgg_t* h);
/* Kernels launched by the last extract call. */
int xvb_repvgg_last_launches(const xvb_repvgg_t* h);
/* feats (B, T, feat_dim) fp32 on the device -> emb (B, embed_dim) fp32 on the device; asynchronous on `stream`. */
int xvb_repvgg_extract(xvb_repvgg_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* "XVBV0001" model files: the configuration, then the records as handed to xvb_repvgg_set_layer (layout at
 * save_records in csrc/model_file.cpp). */
int xvb_repvgg_save(const xvb_repvgg_t* h, const char* path);
int xvb_repvgg_load(xvb_repvgg_t** out, const char* path);
void xvb_repvgg_destroy(xvb_repvgg_t* h);
/* Host only, no GPU: the taps kf*k + kt of a (Cout, Cin, k, k) fp32 kernel whose (Cout, Cin) slab is not all zero, in
 * increasing order, or the centre tap alone when every slab is zero.  Writes them to taps[0..n) and returns n, or
 * XVB_EINVAL on a null pointer, a non-positive size or cap < n. */
int xvb_conv2d_kept_taps(const float* w, int Cout, int Cin, int k, int* taps, int cap);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor for the Conformer x-vector (pytorch/model/transformer_xvector.py, extract_embedding :321-346,
 * Conformer encoder with 4x (input_layer "conv2d") or 2x ("conv2d2") subsampling): the launch sequence of
 * xvb_subsample_head[_stride], xvb_conv2d_valid, xvb_tdnn_affine_ex, xvb_layer_norm, xvb_rope_attention,
 * xvb_conv_module, xvb_attn_stats_pool and xvb_split_f32 in C++, one chunk per utterance (the 300-frame chunk rule
 * stays with the caller).  Bit-identical to the op-by-op Python driver of the same kernels (ConformerExtractor,
 * XVB_CONFORMER_NATIVE=0).
 *
 * Records (rows x cols host fp32 w, optional bias / scale / shift of `rows` entries) are named by state_dict module path
 * and arrive after the hand-over transforms of the Python side:
 *   "transformer.embed.conv.0"     w (D, 9) as stored (kt, kf), bias
 *   "transformer.embed.conv.2"     w (D, 9 D) = the (D, D, kt, kf) weight transposed to (D, D, kf, kt), bias
 *   "transformer.embed.out.0"      w (D, D F'') with its columns in the f * D + c order of the conv output, bias;
 *                                  scale = sqrt(D), shift = 0 with XVB_BN unless pos is no_pos (the xscale)
 *   "transformer.encoders.i.{feed_forward_macaron,feed_forward}.{w_1,w_2}", ".self_attn.linear_qkv" (Q, K, V rows
 *   concatenated), ".self_attn.linear_out", ".conv_module.pointwise_conv{1,2}": w (Cout, Cin), bias, w_1 with the
 *   activation flag (XVB_RELU or XVB_SWISH)
 *   "transformer.encoders.i.conv_module.depthwise_conv"   w (D, K), bias
 *   LayerNorms (cols 0, scale = gamma, shift = beta, or neither without affine): "transformer.encoders.i.norm_{ff,mha,
 *   ff_macaron,conv,final}", "transformer.after_norm", ".conv_module.norm" (a BatchNorm there: folded, with XVB_BN),
 *   "stats.attention.2", "stats.norm_stats", and "transform_out.batchnorm" / "fc1.batchnorm" / "fc2.batchnorm" when that
 *   layer ends in a LayerNorm
 *   "transform_out.affine", "stats.attention.0" (XVB_RELU), "stats.attention.4", "fc1.affine", "fc2.affine":
 *   w (Cout, Cin), bias, a folded BatchNorm as scale / shift with XVB_BN, the activation flag; the segment layers are
 *   the ones the position uses (far: fc1.affine alone; near_affine: [fc1 ->] fc2.affine alone; near: [fc1 ->] fc2)
 * Tables, computed by the caller so that the library derives no transcendental value:
 *   "pos_table"                    rot_pos: (5000, D / H) rotary [sin | cos]; abs_pos: (5000, D) sinusoids
 *   "transformer.encoders.i.self_attn.att_norm"   softmax_plus only: (1, 5000), the score multiplier for T' = 0..4999
 *
 * Extraction takes one chunk of T >= 7 frames per utterance with T' < 5000 subsampled frames (else XVB_EINVAL).
 * Workspace: grown to the largest call seen, then reused.  A call whose B * T exceeds 128 * 300 frames runs as
 * consecutive groups of max(1, floor(128 * 300 / T)) utterances with the same results as one call.  At B = 128,
 * T = 300 it is about 1.3 GB with 4x subsampling and 3.6 GB with 2x, most of it the two subsampling conv outputs.
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_conformer_config {
  int feat_dim;
  int subsampling;        /* 4 (conv2d) or 2 (conv2d2) */
  int D, H, linear_units, blocks, conv_kernel;
  int pos;                /* 0 no_pos, 1 abs_pos, 2 rot_pos */
  int rotary_value;       /* rot_pos: rotate V too */
  int softmax_plus;       /* 0 softmax, 1 softmax_plus */
  int act;                /* XVB_ACT_SWISH or XVB_ACT_RELU */
  int cm_norm;            /* convolution module: 0 LayerNorm, 1 BatchNorm */
  int out_dim;            /* transform_out */
  int out_norm;           /* transform_out: 0 none, 1 BatchNorm (folded), 2 LayerNorm */
  int pool_hidden;        /* AttentiveStatsPool hidden size */
  int fc1;                /* the model has fc1 */
  int position;           /* 0 far, 1 near_affine, 2 near */
} xvb_conformer_config_t;
typedef struct xvb_conformer xvb_conformer_t;
int xvb_conformer_create(xvb_conformer_t** out, const xvb_conformer_config_t* cfg);
int xvb_conformer_set_layer(xvb_conformer_t* h, const char* name, int rows, int cols, const float* w_host,
                            const float* bias_host, const float* scale_host, const float* shift_host, int flags);
/* Checks that every record the configuration needs is present with its shape (and nothing else), names the one that
 * is not, then packs the weights on the current device. */
int xvb_conformer_finalize(xvb_conformer_t* h);
int xvb_conformer_feat_dim(const xvb_conformer_t* h);
int xvb_conformer_embed_dim(const xvb_conformer_t* h);
/* Kernels launched by the last extract call. */
int xvb_conformer_last_launches(const xvb_conformer_t* h);
/* feats (B, T, feat_dim) fp32 on the device, one chunk per utterance -> emb (B, embed_dim) fp32 on the device;
 * asynchronous on `stream`. */
int xvb_conformer_extract(xvb_conformer_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* "XVBC0001" model files: the configuration, then the records and tables as handed to xvb_conformer_set_layer
 * (layout at save_records in csrc/model_file.cpp). */
int xvb_conformer_save(const xvb_conformer_t* h, const char* path);
int xvb_conformer_load(xvb_conformer_t** out, const char* path);
void xvb_conformer_destroy(xvb_conformer_t* h);

/* ---------------------------------------------------------------------------------------------
 * Whole-model extractor for the CAM++ x-vector (subtools2/egrecho/models/campplus/campplus.py, CamPP.forward :355-359,
 * one chunk of CamPPModel.extract_embedding, model.py:73-96): the launch sequence of xvb_conv2d_head, xvb_conv2d,
 * xvb_copy_rows, xvb_tdnn_affine_ex, xvb_bn_relu_planes, xvb_cam_gate, xvb_seg_gate_apply, xvb_stats_pool_ex and
 * xvb_small_affine in C++, one chunk per utterance (the chunk rule stays with the caller, see xvb_campp_chunk_sizes).
 * Bit-identical to the op-by-op Python driver of the same kernels (CamPPExtractor, XVB_CAMPP_NATIVE=0).
 *
 * The block structure is fixed as in CamPP: an FCM head with 32 channels (conv1, layer1 and layer2 of two BasicResBlocks
 * each, the first striding the feature axis by 2, conv2 with stride (2, 1)); the stride-2 `tdnn` (k = 5); three
 * densely connected blocks of 12, 24 and 16 layers with dilations 1, 2 and 2, each followed by a transit layer that
 * halves the width; the context-aware mask over 100-frame segments.  bn = bn_size * growth_rate, c = the width after
 * transit3.
 *
 * Records (rows x cols host fp32 w, optional bias / scale / shift of `rows` entries) are named by state_dict module path
 * and arrive after the hand-over folds of the Python side; flags are exactly the ones listed:
 *   "head.conv1"                      w (32, 9) as stored; head.bn1 folded to scale / shift; XVB_BN | XVB_RELU
 *   "head.layerL.i.conv1", ".conv2"   w (32, 32 * 9) as stored; bn1 / bn2 as scale / shift; XVB_BN | XVB_RELU
 *   "head.layerL.0.shortcut.0"        w (32, 32); shortcut.1 as scale / shift; XVB_BN
 *   "head.conv2"                      w (32, 32 * 9); head.bn2 as scale / shift; XVB_BN | XVB_RELU
 *   "xvector.tdnn.linear"             w (init_channels, 5 * F'' * 32), F'' = feat_dim / 8, in the im2col order k * F'' * 32
 *                                     + f * 32 + c, with tdnn.nonlinear.0 folded into w and bias; XVB_RELU
 *   "xvector.blockB.tdnndL.nonlinear1"            cols 0, scale / shift; XVB_BN | XVB_RELU
 *   "xvector.blockB.tdnndL.linear1"               w (bn, cin) with nonlinear2 folded into w and bias; XVB_RELU
 *   "xvector.blockB.tdnndL.cam_layer.linear_local"  w (growth_rate, bn * 3) as stored (packed over the dilated span)
 *   "xvector.blockB.tdnndL.cam_layer.linear1", ".linear2"   w (bn / 2, bn) and (growth_rate, bn / 2), bias each
 *   "xvector.transitB.nonlinear"      cols 0, scale / shift; XVB_BN | XVB_RELU
 *   "xvector.transitB.linear"         w (width / 2, width); for transit3 out_nonlinear folded into w and bias, XVB_RELU
 *   "xvector.dense.linear"            w (embd_dim, 2 c); the affine-free BatchNorm as scale / shift; XVB_BN
 *
 * Extraction takes one chunk of T >= 3 frames per utterance (else XVB_EINVAL: the unbiased std over ceil(T / 2) frames
 * needs two).  Workspace: grown to the largest call seen, then reused; the pad frames of the time-padded head copy are
 * zeroed again whenever the (B, T) layout changes.  A call whose B * T exceeds 128 * 300 frames runs as consecutive
 * groups of max(1, floor(128 * 300 / T)) utterances with the same results as separate calls.  The workspace is about
 * 60 KB per input frame at feat_dim 80 with the default widths, most of it the FCM head's planes: about 2.3 GB at
 * B = 128, T = 300.
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_campp_config {
  int feat_dim;        /* inputs_dim, a multiple of 8 */
  int embd_dim, init_channels, growth_rate, bn_size;
} xvb_campp_config_t;
typedef struct xvb_campp xvb_campp_t;
int xvb_campp_create(xvb_campp_t** out, const xvb_campp_config_t* cfg);
int xvb_campp_set_layer(xvb_campp_t* h, const char* name, int rows, int cols, const float* w_host,
                        const float* bias_host, const float* scale_host, const float* shift_host, int flags);
/* Checks that every record the configuration needs is present with its shape and flags (and nothing else), names the
 * one that is not, then packs the weights on the current device. */
int xvb_campp_finalize(xvb_campp_t* h);
int xvb_campp_feat_dim(const xvb_campp_t* h);
int xvb_campp_embed_dim(const xvb_campp_t* h);
/* Kernels launched by the last extract call. */
int xvb_campp_last_launches(const xvb_campp_t* h);
/* feats (B, T, feat_dim) fp32 on the device, one chunk per utterance -> emb (B, embd_dim) fp32 on the device;
 * asynchronous on `stream`. */
int xvb_campp_extract(xvb_campp_t* h, const float* feats, int B, int T, float* emb, void* stream);
/* "XVBP0001" model files: the configuration, then the records as handed to xvb_campp_set_layer (layout at
 * save_records in csrc/model_file.cpp). */
int xvb_campp_save(const xvb_campp_t* h, const char* path);
int xvb_campp_load(xvb_campp_t** out, const char* path);
void xvb_campp_destroy(xvb_campp_t* h);
/* Host only, no GPU: the chunk sizes of egrecho's XvectorMixin.split_chunks(max_chunk, even=False) for a T-frame
 * utterance (max_chunk-long chunks, then the last two re-split evenly, the first taking the odd frame: 9000 at 4000 ->
 * 4000, 2500, 2500).  Writes them to sizes[0..n) and returns n, or XVB_EINVAL when T < 1, max_chunk < 1 or cap < n. */
int xvb_campp_chunk_sizes(int T, int max_chunk, int* sizes, int cap);

/* Load a finalized extractor from an .xvbm model file (written by xvb_extractor_save: the layers exactly as the
 * reference's state_dict stores them, eval BatchNorm folded) -- what torch::jit::load does for the reference's
 * runtime (runtime/extractor/torch_asv_model.cc:8-17). */
int xvb_extractor_load(xvb_extractor_t** out, const char* path);
/* Write a finalized extractor's layers, as they were added, and its pooling eps as an XVBM0001 file; XVB_EINVAL for a
 * draft. */
int xvb_extractor_save(const xvb_extractor_t* h, const char* path);
/* Feature dimension recorded in an .xvbm file (> 0), or a negative XVB_E* code.  Host only. */
int xvb_extractor_feat_dim(const char* path);

/* ---------------------------------------------------------------------------------------------
 * Kaldi ark/scp I/O on the host (no GPU needed): the byte formats of the reference's
 * pytorch/libs/support/kaldi_io.py -- read_key :148-163, _read_mat_binary :495-525 (FM/DM),
 * _read_compressed_mat :527-569 (CM), ascii matrices :478-493, write_vec_flt :367-399 (FV),
 * open_or_fd :43-73 (files, "-", "cmd |", "| cmd", "file:offset").
 * rspecifier: "ark:<src>" | "scp:<list>" | "<src>";  wspecifier: "ark:<dst>" | "ark,t:<dst>" |
 * "ark,scp:<ark file>,<scp file>".
 * ------------------------------------------------------------------------------------------- */
typedef struct xvb_ark_reader xvb_ark_reader_t;
typedef struct xvb_ark_writer xvb_ark_writer_t;
int xvb_ark_reader_open(xvb_ark_reader_t** out, const char* rspecifier);
/* Next matrix as fp32 row-major (DM is converted, CM decoded with the reference's fp32 steps).
 * Returns 1 (2 if the matrix was stored in double precision, which the reference's extractor rejects,
 * SURVEY Appendix B.1) and fills the outputs (owned by the reader, valid until the next call), 0 at the
 * end of the stream, a negative XVB_E* code on malformed input. */
int xvb_ark_reader_next(xvb_ark_reader_t* r, const char** key, int* rows, int* cols, const float** data);
void xvb_ark_reader_close(xvb_ark_reader_t* r);
int xvb_ark_writer_open(xvb_ark_writer_t** out, const char* wspecifier);
int xvb_ark_writer_put_vector(xvb_ark_writer_t* w, const char* key, const float* v, int dim);
/* Flushes and closes; fails if the stream or the pipe command failed. */
int xvb_ark_writer_close(xvb_ark_writer_t* w);

#ifdef __cplusplus
}
#endif
#endif /* XVB200_H_ */
