// Conformer x-vector pieces that are not contractions (pytorch/model/transformer_xvector.py over
// pytorch/libs/nnet/transformer/).  Every dense contraction of the model -- Q/K/V, linear_out, the feed-forward and
// pointwise convolutions, the subsampling Linear, transform_out, the pooling convs, fc1 / fc2 -- runs on the wgmma layer
// kernel (tdnn_gemm.cu) and the second subsampling conv on the 2-D conv kernel (conv2d.cu, xvb_conv2d_valid).  What is
// left is bandwidth- or latency-bound and runs here in fp32 on CUDA cores:
//   * the first subsampling conv, Conv2d(1, C, 3, stride 2, no padding) + ReLU (subsampling.py:104-109), or with
//     stride (2, 1) for SVConv2dSubsampling2 (subsampling.py:365-415);
//   * residual update + LayerNorm in one pass over the rows, with an optional second LayerNorm and activation
//     (encoder_layer.py:234-331, the after_norm of encoder.py:414-419, the ln_replace norms of components.py:372-376,
//     AttentiveStatsPool's LayerNorms, transformer_xvector.py:39-50);
//   * multi-head self-attention with rotary position encoding and softmax / softmax_plus (attention.py:255-304,
//     :640-728), keys tiled with an online softmax so any length works;
// The head conv and the attention also take a masked batch (lengths): utterance b then runs the unmasked code at its
// own length, and its rows past that length are written as exact zeros.
//   * the middle of the convolution module: GLU, depthwise conv, LayerNorm / eval BatchNorm, activation
//     (convolution.py:87-130).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace xvb {
namespace {

__device__ __forceinline__ float activate(float v, int act) {
  if (act == XVB_ACT_SWISH) return v / (1.f + expf(-v));   // torch.nn.SiLU
  if (act == XVB_ACT_TANH) return tanhf(v);
  if (act == XVB_ACT_RELU) return fmaxf(v, 0.f);
  return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ void store_plane(__nv_bfloat16* hi, __nv_bfloat16* lo, long long i, float v) {
  __nv_bfloat16 h, l;
  split_bf16(v, h, l);
  hi[i] = h;
  lo[i] = l;
}

// In-place LayerNorm of one row held in shared memory by one warp: v = (v - mean) / sqrt(var + eps) [* g + b], with the
// two-pass (centred) variance.
__device__ __forceinline__ void warp_layer_norm(float* v, int C, float eps, const float* g, const float* b, int lane) {
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += v[c];
  const float mean = warp_sum(s) / (float)C;
  float q = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float d = v[c] - mean;
    q = fmaf(d, d, q);
  }
  const float rstd = 1.f / sqrtf(warp_sum(q) / (float)C + eps);
  for (int c = lane; c < C; c += 32) {
    float y = (v[c] - mean) * rstd;
    if (g) y = fmaf(y, __ldg(g + c), __ldg(b + c));
    v[c] = y;
  }
  __syncwarp();
}

// ---- the subsampling's first conv: one thread per (output position, 8 channels) --------------------------------------
// Time stride 2, feature stride sf (2: Conv2dSubsampling4, 1: SVConv2dSubsampling2).  32-bit index arithmetic (the host
// checks total < 2^31), so decoding the flat index takes no emulated 64-bit division.  lengths (NULL: every utterance has
// T frames): the output rows t >= (lengths[b] - 1) / 2 of utterance b are written as zeros and load nothing, so no
// frame past its end is read; the rows before are computed as for T = lengths[b].  The launch bounds keep the 32
// registers that fit eight 256-thread CTAs per SM, which the lengths operand would otherwise push to 40.
__global__ void __launch_bounds__(256, 8)
subsample_head_kernel(const float* __restrict__ x, int T, int F, int sf, const float* __restrict__ w, const float* __restrict__ bias,
                      int C, int T1, int F1, const int* __restrict__ lengths, __nv_bfloat16* __restrict__ yh,
                      __nv_bfloat16* __restrict__ yl, unsigned total) {
  const unsigned groups = (unsigned)C / 8;
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int c0 = (int)(i % groups) * 8;
    const unsigned pos_u = i / groups;
    const long long pos = pos_u;
    const int f = (int)(pos_u % (unsigned)F1);
    const unsigned bt = pos_u / (unsigned)F1;
    const int t = (int)(bt % (unsigned)T1);
    const long long b = bt / (unsigned)T1;
    const bool live = !lengths || t < (__ldg(lengths + b) - 1) / 2;
    float in[9];
#pragma unroll
    for (int kt = 0; kt < 3; ++kt)
#pragma unroll
      for (int kf = 0; kf < 3; ++kf) in[kt * 3 + kf] = live ? __ldg(x + (b * T + 2 * t + kt) * F + sf * f + kf) : 0.f;
    float y[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float* wc = w + (c0 + k) * 9;   // (C, 1, kt, kf) as stored
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 9; ++j) s = fmaf(__ldg(wc + j), in[j], s);
      y[k] = fmaxf(s + __ldg(bias + c0 + k), 0.f);
    }
    uint4 h, l;
    pack8(y, h, l);
    if (!live) h = l = make_uint4(0u, 0u, 0u, 0u);
    *reinterpret_cast<uint4*>(yh + pos * C + c0) = h;
    *reinterpret_cast<uint4*>(yl + pos * C + c0) = l;
  }
}

// ---- residual + LayerNorm: one warp per row, the row staged in shared memory -------------------------------------
struct LnParams {
  long long rows;
  int C;
  float eps;
  const float* x; long long ldx;
  const float* delta; long long ld_delta; float delta_scale;
  const float* table; int table_rows;
  float* x_out; long long ld_x_out;
  const float* gamma; const float* beta;
  int second;
  const float* gamma2; const float* beta2;
  int act;
  __nv_bfloat16* y_hi; __nv_bfloat16* y_lo; long long ldy;
  float* y_f32; long long ldyf;
};

__global__ void layer_norm_kernel(const LnParams p) {
  extern __shared__ float ln_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* v = ln_smem + (size_t)warp * p.C;
  const int wpb = blockDim.x >> 5;
  for (long long row = (long long)blockIdx.x * wpb + warp; row < p.rows; row += (long long)gridDim.x * wpb) {
    const float* xr = p.x + row * p.ldx;
    const float* dr = p.delta ? p.delta + row * p.ld_delta : nullptr;
    const float* tr = p.table ? p.table + (row % p.table_rows) * (long long)p.C : nullptr;
    for (int c = lane; c < p.C; c += 32) {
      float a = xr[c];
      if (tr) a = __fadd_rn(a, __ldg(tr + c));                           // x * xscale + pe (embedding.py:75)
      if (dr) a = __fadd_rn(a, __fmul_rn(p.delta_scale, dr[c]));        // residual + ff_scale * x
      v[c] = a;
    }
    __syncwarp();
    if (p.second) {                                                     // norm_final, then the next norm
      warp_layer_norm(v, p.C, p.eps, p.gamma, p.beta, lane);
      if (p.x_out)
        for (int c = lane; c < p.C; c += 32) p.x_out[row * p.ld_x_out + c] = v[c];
      warp_layer_norm(v, p.C, p.eps, p.gamma2, p.beta2, lane);
    } else {
      if (p.x_out)
        for (int c = lane; c < p.C; c += 32) p.x_out[row * p.ld_x_out + c] = v[c];
      warp_layer_norm(v, p.C, p.eps, p.gamma, p.beta, lane);
    }
    for (int c = lane; c < p.C; c += 32) {
      const float y = activate(v[c], p.act);
      if (p.y_hi) store_plane(p.y_hi, p.y_lo, row * p.ldy + c, y);
      if (p.y_f32) p.y_f32[row * p.ldyf + c] = y;
    }
    __syncwarp();
  }
}

// ---- rotary multi-head self-attention ---------------------------------------------------------------------------------
// One CTA per (utterance, head, 8 queries), one warp per query.  Keys and values are staged 32 at a time (rotated as
// they are loaded); lane j scores key j of the tile, the running max / sum / output are rescaled per tile (online
// softmax), and lane l accumulates output dimensions l, l + 32, ...
// lengths (NULL: every utterance has T frames): utterance b attends over its keys [0, Tb) only, Tb = lengths[b], with the
// same tiles from key 0, so its rows are those of a call at T = Tb; its query rows past Tb are written as zeros, and a
// query block wholly past Tb loads nothing.  The score multiplier is mult_table[Tb] when mult_table is set, else mult.
// The batch stride stays T rows.
constexpr int kAttnQ = 8;
constexpr int kAttnK = 32;

__device__ __forceinline__ void rotate_pair(float& a, float& b, const float* rope, int dk, int i) {
  const float s = __ldg(rope + i), c = __ldg(rope + dk / 2 + i);
  const float a2 = __fsub_rn(__fmul_rn(a, c), __fmul_rn(b, s));       // x1 * cos - x2 * sin
  const float b2 = __fadd_rn(__fmul_rn(b, c), __fmul_rn(a, s));       // x2 * cos + x1 * sin
  a = a2;
  b = b2;
}

template <int DK>
__global__ void __launch_bounds__(256) rope_attention_kernel(const float* __restrict__ qkv, long long ldq, int T, int H,
                                                             const float* __restrict__ rope, int rope_v, float sqrt_dk,
                                                             float mult, const int* __restrict__ lengths,
                                                             const float* __restrict__ mult_table,
                                                             __nv_bfloat16* __restrict__ yh,
                                                             __nv_bfloat16* __restrict__ yl, long long ldy) {
  __shared__ float Qs[kAttnQ][DK];
  __shared__ float Ks[kAttnK][DK + 1];
  __shared__ float Vs[kAttnK][DK];
  const int nqb = (T + kAttnQ - 1) / kAttnQ;
  const int qb = blockIdx.x % nqb;
  const int h = (blockIdx.x / nqb) % H;
  const long long b = blockIdx.x / ((long long)nqb * H);
  const int D = H * DK;
  const float* base = qkv + b * T * ldq;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int Tb = lengths ? __ldg(lengths + b) : T;
  if (mult_table) mult = __ldg(mult_table + Tb);
  if (qb * kAttnQ >= Tb) {   // a query block wholly past the utterance's end (masked batches only): zero rows
    const int tq = qb * kAttnQ + warp;
    if (tq < T) {
      const long long off = (b * T + tq) * ldy + h * DK + lane;
#pragma unroll
      for (int i = 0; i < DK / 32; ++i) store_plane(yh, yl, off + 32 * i, 0.f);
    }
    return;
  }

  for (int i = threadIdx.x; i < kAttnQ * DK / 2; i += blockDim.x) {
    const int r = i / (DK / 2), j = i % (DK / 2), t = qb * kAttnQ + r;
    float a = 0.f, c = 0.f;
    if (t < Tb) {
      const float* q = base + t * ldq + h * DK;
      a = q[2 * j];
      c = q[2 * j + 1];
      if (rope) rotate_pair(a, c, rope + (long long)t * DK, DK, j);
    }
    Qs[r][2 * j] = a;
    Qs[r][2 * j + 1] = c;
  }

  float m = -INFINITY, l = 0.f, o[DK / 32];
#pragma unroll
  for (int i = 0; i < DK / 32; ++i) o[i] = 0.f;
  for (int k0 = 0; k0 < Tb; k0 += kAttnK) {
    __syncthreads();   // Q staged / the previous tile consumed
    for (int i = threadIdx.x; i < kAttnK * DK / 2; i += blockDim.x) {
      const int r = i / (DK / 2), j = i % (DK / 2), t = k0 + r;
      float ka = 0.f, kc = 0.f, va = 0.f, vc = 0.f;
      if (t < Tb) {
        const float* row = base + t * ldq + h * DK;
        ka = row[D + 2 * j];
        kc = row[D + 2 * j + 1];
        va = row[2 * D + 2 * j];
        vc = row[2 * D + 2 * j + 1];
        if (rope) {
          rotate_pair(ka, kc, rope + (long long)t * DK, DK, j);
          if (rope_v) rotate_pair(va, vc, rope + (long long)t * DK, DK, j);
        }
      }
      Ks[r][2 * j] = ka;
      Ks[r][2 * j + 1] = kc;
      Vs[r][2 * j] = va;
      Vs[r][2 * j + 1] = vc;
    }
    __syncthreads();
    const bool valid = k0 + lane < Tb;
    float s = -INFINITY;
    if (valid) {
      float d = 0.f;
#pragma unroll 16
      for (int j = 0; j < DK; ++j) d = fmaf(Qs[warp][j], Ks[lane][j], d);
      s = __fmul_rn(__fdiv_rn(d, sqrt_dk), mult);                      // scores / sqrt(d_k) [* ln(l) / train_len]
    }
    const float mnew = fmaxf(m, warp_max(s));
    const float pj = valid ? expf(s - mnew) : 0.f;
    const float corr = expf(m - mnew);
    l = fmaf(l, corr, warp_sum(pj));
#pragma unroll
    for (int i = 0; i < DK / 32; ++i) o[i] *= corr;
    const int nk = min(kAttnK, Tb - k0);
    for (int j = 0; j < nk; ++j) {
      const float pb = __shfl_sync(0xffffffffu, pj, j);
#pragma unroll
      for (int i = 0; i < DK / 32; ++i) o[i] = fmaf(pb, Vs[j][lane + 32 * i], o[i]);
    }
    m = mnew;
  }
  const int tq = qb * kAttnQ + warp;
  if (tq < T) {
    const float inv = 1.f / l;
    const bool live = tq < Tb;
    const long long off = (b * T + tq) * ldy + h * DK + lane;
#pragma unroll
    for (int i = 0; i < DK / 32; ++i) store_plane(yh, yl, off + 32 * i, live ? o[i] * inv : 0.f);
  }
}

// ---- convolution module middle: GLU -> depthwise conv -> norm -> activation ------------------------------------------
// One CTA per (utterance, 16 frames): the GLU of the frames the 16 outputs need (zero outside [0, T), the conv's zero
// padding) is staged in shared memory, the depthwise conv writes 16 rows, then one warp per row normalises.
constexpr int kConvRows = 16;

__global__ void __launch_bounds__(256) conv_module_kernel(const float* __restrict__ x, long long ldx, int T, int C,
                                                          const float* __restrict__ dw_w, const float* __restrict__ dw_b,
                                                          int K, const float* __restrict__ g, const float* __restrict__ bt,
                                                          int norm, float eps, int act, __nv_bfloat16* __restrict__ yh,
                                                          __nv_bfloat16* __restrict__ yl, long long ldy) {
  extern __shared__ float cm_smem[];
  const int pad = K / 2, span = kConvRows + K - 1;
  float* G = cm_smem;                   // (span, C)
  float* Y = cm_smem + (size_t)span * C;   // (kConvRows, C)
  const int nblk = (T + kConvRows - 1) / kConvRows;
  const long long b = blockIdx.x / nblk;
  const int t0 = (int)(blockIdx.x % nblk) * kConvRows;
  for (int i = threadIdx.x; i < span * C; i += blockDim.x) {
    const int r = i / C, c = i % C, t = t0 - pad + r;
    float v = 0.f;
    if (t >= 0 && t < T) {
      const float* row = x + (b * T + t) * ldx;
      v = row[c] * (1.f / (1.f + expf(-row[C + c])));                  // F.glu(x, dim=1): a * sigmoid(b)
    }
    G[i] = v;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kConvRows * C; i += blockDim.x) {
    const int r = i / C, c = i % C;
    float s = 0.f;
    for (int k = 0; k < K; ++k) s = fmaf(__ldg(dw_w + c * K + k), G[(r + k) * C + c], s);
    Y[i] = s + __ldg(dw_b + c);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = warp; r < kConvRows; r += blockDim.x >> 5) {
    const int t = t0 + r;
    if (t >= T) break;
    float* v = Y + (size_t)r * C;
    if (norm == 0) {
      warp_layer_norm(v, C, eps, g, bt, lane);
    } else {
      for (int c = lane; c < C; c += 32) v[c] = fmaf(v[c], __ldg(g + c), __ldg(bt + c));   // eval BatchNorm1d
    }
    const long long off = (b * T + t) * ldy;
    for (int c = lane; c < C; c += 32) store_plane(yh, yl, off + c, activate(v[c], act));
  }
}

int grid_cap(long long want) {
  const long long cap = (long long)sm_count() * 16;
  return (int)(want < 1 ? 1 : (want > cap ? cap : want));
}

}  // namespace
}  // namespace xvb

using namespace xvb;

static int subsample_head(const float* x, int B, int T, int F, const int* lengths, const float* w, const float* bias, int C,
                          int stride_f, uint16_t* y_hi, uint16_t* y_lo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x && w && bias && y_hi && y_lo, "xvb_subsample_head: null pointer");
  XVB_CHECK_ARG(stride_f == 1 || stride_f == 2, "xvb_subsample_head: feature stride must be 1 or 2 (got %d)", stride_f);
  XVB_CHECK_ARG(B > 0 && T >= 3 && F >= 3 && C > 0 && C % 8 == 0, "xvb_subsample_head: bad shape B=%d T=%d F=%d C=%d (T, F >= 3, C %% 8 == 0)",
                B, T, F, C);
  XVB_CHECK_ARG(((uintptr_t)y_hi | (uintptr_t)y_lo) % 16 == 0, "xvb_subsample_head: planes must be 16-byte aligned");
  const int T1 = (T - 3) / 2 + 1, F1 = (F - 3) / stride_f + 1;
  const long long total = (long long)B * T1 * F1 * (C / 8);
  XVB_CHECK_ARG(total < (1LL << 31), "xvb_subsample_head: %lld (position, 8-channel) items exceed one launch", total);
  subsample_head_kernel<<<grid_cap((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      x, T, F, stride_f, w, bias, C, T1, F1, lengths, reinterpret_cast<__nv_bfloat16*>(y_hi),
      reinterpret_cast<__nv_bfloat16*>(y_lo), (unsigned)total);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_subsample_head_stride(const float* x, int B, int T, int F, const float* w, const float* bias, int C,
                                         int stride_f, uint16_t* y_hi, uint16_t* y_lo, void* stream) {
  return subsample_head(x, B, T, F, nullptr, w, bias, C, stride_f, y_hi, y_lo, stream);
}

extern "C" int xvb_subsample_head_lengths(const float* x, int B, int T, int F, const int* lengths, const float* w,
                                          const float* bias, int C, int stride_f, uint16_t* y_hi, uint16_t* y_lo,
                                          void* stream) {
  XVB_CHECK_ARG(lengths, "xvb_subsample_head_lengths: null lengths");
  return subsample_head(x, B, T, F, lengths, w, bias, C, stride_f, y_hi, y_lo, stream);
}

extern "C" int xvb_subsample_head(const float* x, int B, int T, int F, const float* w, const float* bias, int C, uint16_t* y_hi,
                                  uint16_t* y_lo, void* stream) {
  return xvb_subsample_head_stride(x, B, T, F, w, bias, C, 2, y_hi, y_lo, stream);
}

extern "C" int xvb_layer_norm(const xvb_layer_norm_args_t* a, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(a && a->x, "xvb_layer_norm: null args or input");
  XVB_CHECK_ARG(a->rows > 0 && a->C > 0 && a->C <= 8192, "xvb_layer_norm: bad shape rows=%lld C=%d (C <= 8192)",
                (long long)a->rows, a->C);
  XVB_CHECK_ARG(a->ldx >= a->C && (!a->delta || a->ld_delta >= a->C) && (!a->x_out || a->ld_x_out >= a->C) &&
                    (!a->y_hi || a->ldy >= a->C) && (!a->y_f32 || a->ldyf >= a->C),
                "xvb_layer_norm: every row pitch must be >= C");
  XVB_CHECK_ARG(!a->table || a->table_rows > 0, "xvb_layer_norm: table needs table_rows > 0");
  XVB_CHECK_ARG((a->gamma != nullptr) == (a->beta != nullptr) && (a->gamma2 != nullptr) == (a->beta2 != nullptr),
                "xvb_layer_norm: gamma and beta must both be set or both NULL");
  XVB_CHECK_ARG((a->y_hi != nullptr) == (a->y_lo != nullptr), "xvb_layer_norm: y_hi/y_lo must both be set or both NULL");
  XVB_CHECK_ARG(a->y_hi || a->y_f32 || a->x_out, "xvb_layer_norm: no output requested");
  XVB_CHECK_ARG(a->act >= XVB_ACT_NONE && a->act <= XVB_ACT_TANH, "xvb_layer_norm: unknown activation %d", a->act);
  LnParams p{};
  p.rows = a->rows; p.C = a->C; p.eps = a->eps;
  p.x = a->x; p.ldx = a->ldx;
  p.delta = a->delta; p.ld_delta = a->ld_delta; p.delta_scale = a->delta_scale;
  p.table = a->table; p.table_rows = a->table_rows;
  p.x_out = a->x_out; p.ld_x_out = a->ld_x_out;
  p.gamma = a->gamma; p.beta = a->beta;
  p.second = a->second ? 1 : 0;
  p.gamma2 = a->gamma2; p.beta2 = a->beta2;
  p.act = a->act;
  p.y_hi = reinterpret_cast<__nv_bfloat16*>(a->y_hi); p.y_lo = reinterpret_cast<__nv_bfloat16*>(a->y_lo); p.ldy = a->ldy;
  p.y_f32 = a->y_f32; p.ldyf = a->ldyf;
  int warps = 8192 / a->C;   // the staged rows fit 32 KB of shared memory
  warps = warps < 1 ? 1 : (warps > 8 ? 8 : warps);
  const size_t smem = (size_t)warps * a->C * sizeof(float);
  layer_norm_kernel<<<grid_cap((a->rows + warps - 1) / warps), warps * 32, smem, (cudaStream_t)stream>>>(p);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

static int rope_attention(const float* qkv, int64_t ldq, int B, int T, int H, int dk, const float* rope, int rope_v,
                          float score_mult, const int* lengths, const float* mult_table, uint16_t* y_hi, uint16_t* y_lo,
                          int64_t ldy, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(qkv && y_hi && y_lo, "xvb_rope_attention: null pointer");
  XVB_CHECK_ARG(dk == 32 || dk == 64 || dk == 128, "xvb_rope_attention: d_k must be 32, 64 or 128 (got %d)", dk);
  XVB_CHECK_ARG(B > 0 && T > 0 && H > 0, "xvb_rope_attention: bad shape B=%d T=%d H=%d", B, T, H);
  XVB_CHECK_ARG(ldq >= 3LL * H * dk && ldy >= (int64_t)H * dk, "xvb_rope_attention: ldq must be >= 3*H*dk and ldy >= H*dk");
  XVB_CHECK_ARG(!rope_v || rope, "xvb_rope_attention: rotary value needs the rotary table");
  const long long grid = (long long)B * H * ((T + kAttnQ - 1) / kAttnQ);
  XVB_CHECK_ARG(grid < (1LL << 31), "xvb_rope_attention: too many CTAs");
  const float sq = sqrtf((float)dk);
  auto* yh = reinterpret_cast<__nv_bfloat16*>(y_hi);
  auto* yl = reinterpret_cast<__nv_bfloat16*>(y_lo);
  cudaStream_t s = (cudaStream_t)stream;
  if (dk == 32)
    rope_attention_kernel<32><<<(unsigned)grid, 256, 0, s>>>(qkv, ldq, T, H, rope, rope_v, sq, score_mult, lengths, mult_table,
                                                             yh, yl, ldy);
  else if (dk == 64)
    rope_attention_kernel<64><<<(unsigned)grid, 256, 0, s>>>(qkv, ldq, T, H, rope, rope_v, sq, score_mult, lengths, mult_table,
                                                             yh, yl, ldy);
  else
    rope_attention_kernel<128><<<(unsigned)grid, 256, 0, s>>>(qkv, ldq, T, H, rope, rope_v, sq, score_mult, lengths,
                                                              mult_table, yh, yl, ldy);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_rope_attention(const float* qkv, int64_t ldq, int B, int T, int H, int dk, const float* rope, int rope_v,
                                  float score_mult, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, void* stream) {
  return rope_attention(qkv, ldq, B, T, H, dk, rope, rope_v, score_mult, nullptr, nullptr, y_hi, y_lo, ldy, stream);
}

extern "C" int xvb_rope_attention_lengths(const float* qkv, int64_t ldq, int B, int T, int H, int dk, const float* rope,
                                          int rope_v, const int* lengths, const float* mult_table, int mult_rows,
                                          uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, void* stream) {
  XVB_CHECK_ARG(lengths, "xvb_rope_attention_lengths: null lengths");
  // lengths[b] <= T < mult_rows keeps every mult_table[lengths[b]] inside the table
  XVB_CHECK_ARG(!mult_table || (mult_rows > 0 && T < mult_rows),
                "xvb_rope_attention_lengths: T=%d needs a multiplier table of more than T rows (mult_rows=%d)", T, mult_rows);
  return rope_attention(qkv, ldq, B, T, H, dk, rope, rope_v, 1.0f, lengths, mult_table, y_hi, y_lo, ldy, stream);
}

extern "C" int xvb_conv_module(const float* x, int64_t ldx, int B, int T, int C, const float* dw_w, const float* dw_b, int K,
                               const float* norm_a, const float* norm_b, int norm, float eps, int act, uint16_t* y_hi,
                               uint16_t* y_lo, int64_t ldy, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x && dw_w && dw_b && norm_a && norm_b && y_hi && y_lo, "xvb_conv_module: null pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && K > 0 && K % 2 == 1, "xvb_conv_module: bad shape B=%d T=%d C=%d K=%d (K odd)", B, T,
                C, K);
  XVB_CHECK_ARG(ldx >= 2LL * C && ldy >= C, "xvb_conv_module: ldx must be >= 2C and ldy >= C");
  XVB_CHECK_ARG(norm == 0 || norm == 1, "xvb_conv_module: norm must be 0 (LayerNorm) or 1 (scale / shift)");
  XVB_CHECK_ARG(act >= XVB_ACT_NONE && act <= XVB_ACT_TANH, "xvb_conv_module: unknown activation %d", act);
  const size_t smem = (size_t)(2 * kConvRows + K - 1) * C * sizeof(float);
  constexpr int kMaxSmem = 200 * 1024;
  XVB_CHECK_ARG(smem <= (size_t)kMaxSmem, "xvb_conv_module: C=%d with K=%d needs %zu bytes of shared memory", C, K, smem);
  XVB_ENSURE_DYN_SMEM(conv_module_kernel, kMaxSmem);   // once per device, so the largest size any call may need
  const long long grid = (long long)B * ((T + kConvRows - 1) / kConvRows);
  XVB_CHECK_ARG(grid < (1LL << 31), "xvb_conv_module: too many CTAs");
  conv_module_kernel<<<(unsigned)grid, 256, smem, (cudaStream_t)stream>>>(
      x, ldx, T, C, dw_w, dw_b, K, norm_a, norm_b, norm, eps, act, reinterpret_cast<__nv_bfloat16*>(y_hi),
      reinterpret_cast<__nv_bfloat16*>(y_lo), ldy);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}
