// ECAPA-TDNN specific bandwidth-bound kernels (pytorch/model/ecapa_tdnn_xvector.py):
//   * plane_mean      : mean over time of a split-plane tensor (SE_Connect's AdaptiveAvgPool1d, :100)
//   * se_apply        : out = z * gate[b] + in  (+ next = in + out)   (SE_Connect :109-111, SE_Res2Block :149,
//                       and the dense residual sums x+x1, x+x1+x2 of ECAPA_TDNN.extract_embedding :405-408);
//                       with a gate per seg_len-frame segment and no `in`, CAM++'s context-aware mask y * m
//   * attn_stats_pool : softmax over time + weighted mean / std (AttentiveStatsPool.forward :183-188) as a
//                       single streaming pass with an online softmax (running max + rescaled sums)
// All the dense contractions of the model run on the wgmma layer kernel (tdnn_gemm.cu).
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace xvb {

// ---------------------------------------------------------------- mean over T of planes
// lengths != NULL: utterance b averages its first lengths[b] * rows_per_length rows (a masked batch).
constexpr int kPmWarps = 8;
__global__ void __launch_bounds__(kPmWarps * 32)
plane_mean_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl, long long ldx, int T_all, int C,
                  const int* __restrict__ lengths, int rows_per_length, float* __restrict__ out, __nv_bfloat16* __restrict__ oh,
                  __nv_bfloat16* __restrict__ ol, long long ldo) {
  const int b = blockIdx.y;
  const int T = lengths ? min(__ldg(lengths + b) * rows_per_length, T_all) : T_all;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 256 + lane * 8;
  const bool active = c < C;  // C % 8 == 0
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (active) {
    const long long base = (long long)b * T_all * ldx + c;
    for (int t = warp; t < T; t += kPmWarps) {
      const uint4 h = *reinterpret_cast<const uint4*>(xh + base + (long long)t * ldx);
      const uint4 l = *reinterpret_cast<const uint4*>(xl + base + (long long)t * ldx);
      float f[8];
      unpack8(h, l, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += f[k];
    }
  }
  __shared__ float sh[kPmWarps][32][8];
#pragma unroll
  for (int k = 0; k < 8; ++k) sh[warp][lane][k] = acc[k];
  __syncthreads();
  if (warp == 0 && active) {
    float m[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      float s = 0.f;
      for (int w = 0; w < kPmWarps; ++w) s += sh[w][lane][k];
      m[k] = s / (float)T;
    }
    if (out) {
      float* o = out + (long long)b * C + c;
      *reinterpret_cast<float4*>(o) = make_float4(m[0], m[1], m[2], m[3]);
      *reinterpret_cast<float4*>(o + 4) = make_float4(m[4], m[5], m[6], m[7]);
    }
    if (oh) {
      uint4 h, l;
      pack8(m, h, l);
      *reinterpret_cast<uint4*>(oh + (long long)b * ldo + c) = h;
      *reinterpret_cast<uint4*>(ol + (long long)b * ldo + c) = l;
    }
  }
}

// ---------------------------------------------------------------- strided row copy (channel-slice pass-through)
__global__ void copy_rows_kernel(const uint4* __restrict__ src, long long ld_src16, uint4* __restrict__ dst,
                                 long long ld_dst16, long long rows, int vec_per_row) {
  const long long total = rows * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / vec_per_row;
    const int c = (int)(i % vec_per_row);
    dst[r * ld_dst16 + c] = src[r * ld_src16 + c];
  }
}

// ---------------------------------------------------------------- SE gate + residual (+ running sum)
// gate[b, t / seg_len, :] scales frame t of utterance b (gate rows: nseg = ceil(T / seg_len) per utterance); seg_len = T
// is SE_Connect's one gate per utterance.  in NULL: out = z * gate (CAMLayer's y * m, campplus.py:157-162), no add.
__global__ void se_apply_kernel(const __nv_bfloat16* __restrict__ zh, const __nv_bfloat16* __restrict__ zl, long long ldz,
                                const __nv_bfloat16* __restrict__ ih, const __nv_bfloat16* __restrict__ il, long long ldi,
                                const float* __restrict__ gate, __nv_bfloat16* __restrict__ oh,
                                __nv_bfloat16* __restrict__ ol, long long ldo, __nv_bfloat16* __restrict__ nh,
                                __nv_bfloat16* __restrict__ nl, long long ldn, long long frames, int T, int C, int seg_len) {
  const int groups = C / 8;
  const int nseg = (T + seg_len - 1) / seg_len;
  const long long total = frames * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long fr = i / groups;
    const int c = (int)(i % groups) * 8;
    const long long b = fr / T;
    const long long row = b * nseg + (int)(fr - b * T) / seg_len;
    float z[8], x[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, o[8];
    unpack8(*reinterpret_cast<const uint4*>(zh + fr * ldz + c), *reinterpret_cast<const uint4*>(zl + fr * ldz + c), z);
    if (ih) unpack8(*reinterpret_cast<const uint4*>(ih + fr * ldi + c), *reinterpret_cast<const uint4*>(il + fr * ldi + c), x);
    const float4 g0 = *reinterpret_cast<const float4*>(gate + row * C + c);
    const float4 g1 = *reinterpret_cast<const float4*>(gate + row * C + c + 4);
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    // mul then add: the reference's two roundings (spelled out: the compiler would otherwise contract them into one FFMA)
    for (int k = 0; k < 8; ++k) o[k] = __fadd_rn(__fmul_rn(z[k], g[k]), x[k]);
    uint4 h, l;
    pack8(o, h, l);
    *reinterpret_cast<uint4*>(oh + fr * ldo + c) = h;
    *reinterpret_cast<uint4*>(ol + fr * ldo + c) = l;
    if (nh) {
#pragma unroll
      for (int k = 0; k < 8; ++k) o[k] += x[k];
      pack8(o, h, l);
      *reinterpret_cast<uint4*>(nh + fr * ldn + c) = h;
      *reinterpret_cast<uint4*>(nl + fr * ldn + c) = l;
    }
  }
}

int launch_se_apply(const uint16_t* z_hi, const uint16_t* z_lo, int64_t ldz, const uint16_t* in_hi, const uint16_t* in_lo,
                    int64_t ldin, const float* gate, int seg_len, uint16_t* out_hi, uint16_t* out_lo, int64_t ldout,
                    uint16_t* next_hi, uint16_t* next_lo, int64_t ldnext, int B, int T, int C, void* stream) {
  const long long frames = (long long)B * T;
  const long long total = frames * (C / 8);
  long long g = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 32;
  if (g > cap) g = cap;
  se_apply_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(z_hi), reinterpret_cast<const __nv_bfloat16*>(z_lo), ldz,
      reinterpret_cast<const __nv_bfloat16*>(in_hi), reinterpret_cast<const __nv_bfloat16*>(in_lo), ldin, gate,
      reinterpret_cast<__nv_bfloat16*>(out_hi), reinterpret_cast<__nv_bfloat16*>(out_lo), ldout,
      reinterpret_cast<__nv_bfloat16*>(next_hi), reinterpret_cast<__nv_bfloat16*>(next_lo), ldnext, frames, T, C, seg_len);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

// ---------------------------------------------------------------- attentive statistics pooling
constexpr int kApWarps = 8;
constexpr int kApRows = 4;

struct Online {  // per channel: running max and rescaled sums of e, e*x, e*x^2
  float m, s0, s1, s2;
};
__device__ __forceinline__ void online_add(Online& o, float l, float x) {
  const float mn = fmaxf(o.m, l);
  const float sc = expf(o.m - mn), e = expf(l - mn);
  o.s0 = fmaf(o.s0, sc, e);
  o.s1 = fmaf(o.s1, sc, e * x);
  o.s2 = fmaf(o.s2, sc, e * x * x);
  o.m = mn;
}
__device__ __forceinline__ void online_merge(Online& a, const Online& b) {
  const float mn = fmaxf(a.m, b.m);
  const float sa = expf(a.m - mn), sb = expf(b.m - mn);
  a.s0 = a.s0 * sa + b.s0 * sb;
  a.s1 = a.s1 * sa + b.s1 * sb;
  a.s2 = a.s2 * sa + b.s2 * sb;
  a.m = mn;
}

__global__ void __launch_bounds__(kApWarps * 32)
attn_stats_pool_kernel(const float* __restrict__ logits, long long ldl, const float* __restrict__ x, long long ldx, int T,
                       int C, float floor_, const int* __restrict__ lengths, float* __restrict__ out,
                       __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol, long long ldo) {
  const int b = blockIdx.y;
  // a masked batch reduces utterance b over its own frames [0, Tb) with the same walk, as a call at T = Tb would; the
  // batch stride stays T rows and the frames past Tb are never loaded
  const int Tb = lengths ? __ldg(lengths + b) : T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int c = blockIdx.x * 128 + lane * 4;
  const bool active = c < C;
  Online st[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) st[k] = {-INFINITY, 0.f, 0.f, 0.f};
  if (active) {
    const float* lb = logits + (long long)b * T * ldl + c;
    const float* xb = x + (long long)b * T * ldx + c;
    for (int t0 = warp; t0 < Tb; t0 += kApWarps * kApRows) {
      float4 lv[kApRows], xv[kApRows];
#pragma unroll
      for (int r = 0; r < kApRows; ++r) {
        const int t = t0 + r * kApWarps;
        if (t < Tb) {
          lv[r] = __ldcs(reinterpret_cast<const float4*>(lb + (long long)t * ldl));
          xv[r] = __ldcs(reinterpret_cast<const float4*>(xb + (long long)t * ldx));
        }
      }
#pragma unroll
      for (int r = 0; r < kApRows; ++r) {
        if (t0 + r * kApWarps < Tb) {
          online_add(st[0], lv[r].x, xv[r].x);
          online_add(st[1], lv[r].y, xv[r].y);
          online_add(st[2], lv[r].z, xv[r].z);
          online_add(st[3], lv[r].w, xv[r].w);
        }
      }
    }
  }
  __shared__ Online sh[kApWarps][32][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) sh[warp][lane][k] = st[k];
  __syncthreads();
  if (warp == 0 && active) {
    float mu[4], sd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      Online a = sh[0][lane][k];
      for (int w = 1; w < kApWarps; ++w)
        if (sh[w][lane][k].s0 > 0.f) online_merge(a, sh[w][lane][k]);
      mu[k] = a.s1 / a.s0;
      sd[k] = sqrtf(fmaxf(a.s2 / a.s0 - mu[k] * mu[k], floor_));   // residuals.clamp(min=1e-5), :186-187
    }
    float* ob = out + (long long)b * 2 * C;
    *reinterpret_cast<float4*>(ob + c) = make_float4(mu[0], mu[1], mu[2], mu[3]);
    *reinterpret_cast<float4*>(ob + C + c) = make_float4(sd[0], sd[1], sd[2], sd[3]);
    if (oh) {
      __nv_bfloat16 h[8], l[8];
#pragma unroll
      for (int k = 0; k < 4; ++k) { split_bf16(mu[k], h[k], l[k]); split_bf16(sd[k], h[4 + k], l[4 + k]); }
      __nv_bfloat16* ph = oh + (long long)b * ldo;
      __nv_bfloat16* pl = ol + (long long)b * ldo;
      *reinterpret_cast<uint2*>(ph + c) = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
      *reinterpret_cast<uint2*>(pl + c) = make_uint2(pack_bf16x2(l[0], l[1]), pack_bf16x2(l[2], l[3]));
      *reinterpret_cast<uint2*>(ph + C + c) = make_uint2(pack_bf16x2(h[4], h[5]), pack_bf16x2(h[6], h[7]));
      *reinterpret_cast<uint2*>(pl + C + c) = make_uint2(pack_bf16x2(l[4], l[5]), pack_bf16x2(l[6], l[7]));
    }
  }
}

// ---------------------------------------------------------------- LDE pooling (learnable dictionary encoding)
// LDEPooling.forward, libs/nnet/pooling.py:148-159:  r[t,c,k] = x[t,c] - mu[c,k];  w[t,k] = softmax_k(-(s_k^2 + eps) * sum_c r^2);
// e[c,k] = mean_t(w[t,k] * r[t,c,k]);  out (B, C*K), index c*K + k.  The squared distances are summed DIRECTLY in fp32
// (expanding |x - mu|^2 = |x|^2 - 2 x.mu + |mu|^2 on the tensor cores would lose ~1e-3 of the softmax weights to
// cancellation).  Two kernels: the weights (a block = 32 frames x all K clusters, x and mu staged through shared
// memory in channel chunks) and the weighted residual mean (a block = one utterance x 32 channels, w rows staged in
// shared memory in time chunks).  K <= 64, K % 4 == 0 (pad the dictionary with zero-weight columns: beta = +inf is
// not needed, the caller passes neg_beta = -inf for padded clusters so that their softmax weight is exactly 0).
constexpr int kLdeFr = 4;                      // frames per thread (weights kernel) / channels per thread (encode kernel)
constexpr int kLdeFrames = 32 * kLdeFr, kLdeChunk = 32, kLdeMaxK = 64;

// this thread's (up to 8) dictionary entries of one row: two 16-byte loads when the thread owns 8 consecutive ones
__device__ __forceinline__ void lde_row8(const float* row, int g, int kq, int K, float (&m)[8]) {
  if (kq == 8) {
    const float4 a = *reinterpret_cast<const float4*>(row + g * 8), b = *reinterpret_cast<const float4*>(row + g * 8 + 4);
    m[0] = a.x; m[1] = a.y; m[2] = a.z; m[3] = a.w; m[4] = b.x; m[5] = b.y; m[6] = b.z; m[7] = b.w;
  } else {
#pragma unroll
    for (int i = 0; i < 8; ++i) m[i] = (i < kq && g * kq + i < K) ? row[g * kq + i] : 0.f;
  }
}

__global__ void __launch_bounds__(256)
lde_weights_kernel(const float* __restrict__ x, long long ldx, long long rows, int C, const float* __restrict__ mu, int K,
                   const float* __restrict__ neg_beta, float* __restrict__ w) {
  __shared__ float xs[kLdeFrames][kLdeChunk + 1];
  __shared__ __align__(16) float ms[kLdeChunk][kLdeMaxK];
  const int fq = threadIdx.x >> 3, g = threadIdx.x & 7;      // frames fq*4 .. fq*4+3 of the tile, clusters g*kq .. +kq
  const int kq = (K + 7) >> 3;                               // clusters per thread (<= 8)
  const long long row0 = (long long)blockIdx.x * kLdeFrames;
  float d[kLdeFr][8];
#pragma unroll
  for (int r = 0; r < kLdeFr; ++r)
#pragma unroll
    for (int i = 0; i < 8; ++i) d[r][i] = 0.f;
  for (int c0 = 0; c0 < C; c0 += kLdeChunk) {
    const int cc = min(kLdeChunk, C - c0);
    for (int e = threadIdx.x; e < kLdeFrames * kLdeChunk; e += 256) {
      const int ff = e / kLdeChunk, c = e - ff * kLdeChunk;
      xs[ff][c] = (row0 + ff < rows && c < cc) ? __ldg(x + (row0 + ff) * ldx + c0 + c) : 0.f;
    }
    for (int e = threadIdx.x; e < kLdeChunk * kLdeMaxK; e += 256) {
      const int c = e / kLdeMaxK, k = e - c * kLdeMaxK;
      ms[c][k] = (c < cc && k < K) ? __ldg(mu + (long long)(c0 + c) * K + k) : 0.f;   // padded channels: x = mu = 0
    }
    __syncthreads();
    for (int c = 0; c < cc; ++c) {
      float m[8];
      lde_row8(ms[c], g, kq, K, m);
#pragma unroll
      for (int r = 0; r < kLdeFr; ++r) {
        const float xv = xs[fq * kLdeFr + r][c];
#pragma unroll
        for (int i = 0; i < 8; ++i) { const float q = xv - m[i]; d[r][i] = fmaf(q, q, d[r][i]); }   // absent clusters: unused
      }
    }
    __syncthreads();
  }
  float nb[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) nb[i] = (i < kq && g * kq + i < K) ? __ldg(neg_beta + g * kq + i) : 0.f;
#pragma unroll
  for (int r = 0; r < kLdeFr; ++r) {
    // softmax over the K clusters of this frame: the 8 threads of a frame are 8 consecutive lanes
    float l[8], mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      l[i] = (i < kq && g * kq + i < K) ? nb[i] * d[r][i] : -INFINITY;
      mx = fmaxf(mx, l[i]);
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) { l[i] = expf(l[i] - mx); sum += l[i]; }   // exp(-inf) = 0 for absent clusters
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const long long row = row0 + fq * kLdeFr + r;
    if (row < rows) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
        if (i < kq && g * kq + i < K) w[row * K + g * kq + i] = l[i] / sum;
    }
  }
}

__global__ void __launch_bounds__(256)
lde_encode_kernel(const float* __restrict__ x, long long ldx, int T, int C, const float* __restrict__ mu, int K,
                  const float* __restrict__ w, float* __restrict__ out, __nv_bfloat16* __restrict__ oh,
                  __nv_bfloat16* __restrict__ ol, long long ldo) {
  __shared__ __align__(16) float ws[64][kLdeMaxK];           // 64 frames of weights at a time
  const int b = blockIdx.y;
  const int cl = threadIdx.x & 31, g = threadIdx.x >> 5;      // channels blockIdx.x*128 + i*32 + cl, cluster group g
  const int kq = (K + 7) >> 3;
  float acc[kLdeFr][8], m[kLdeFr][8];
  int ch[kLdeFr];
#pragma unroll
  for (int r = 0; r < kLdeFr; ++r) {
    ch[r] = blockIdx.x * (32 * kLdeFr) + r * 32 + cl;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int k = g * kq + i;
      acc[r][i] = 0.f;
      m[r][i] = (i < kq && k < K && ch[r] < C) ? __ldg(mu + (long long)ch[r] * K + k) : 0.f;
    }
  }
  const float* xb = x + (long long)b * T * ldx;
  const float* wb = w + (long long)b * T * K;
  for (int t0 = 0; t0 < T; t0 += 64) {
    const int tn = min(64, T - t0);
    for (int e = threadIdx.x; e < tn * kLdeMaxK; e += 256) {
      const int t = e / kLdeMaxK, k = e - t * kLdeMaxK;
      ws[t][k] = k < K ? __ldg(wb + (long long)(t0 + t) * K + k) : 0.f;
    }
    __syncthreads();
    for (int t = 0; t < tn; ++t) {
      float wv[8];
      lde_row8(ws[t], g, kq, K, wv);
#pragma unroll
      for (int r = 0; r < kLdeFr; ++r) {
        const float xv = ch[r] < C ? __ldg(xb + (long long)(t0 + t) * ldx + ch[r]) : 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[r][i] = fmaf(wv[i], xv - m[r][i], acc[r][i]);   // absent clusters: weight 0
      }
    }
    __syncthreads();
  }
  const float inv = 1.f / (float)T;
#pragma unroll
  for (int r = 0; r < kLdeFr; ++r) {
    if (ch[r] >= C) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int k = g * kq + i;
      if (i < kq && k < K) {
        const float v = acc[r][i] * inv;
        const long long o = (long long)ch[r] * K + k;
        out[(long long)b * C * K + o] = v;
        if (oh) {
          __nv_bfloat16 h, l;
          split_bf16(v, h, l);
          oh[(long long)b * ldo + o] = h;
          ol[(long long)b * ldo + o] = l;
        }
      }
    }
  }
}

// ---------------------------------------------------------------- segment-level affine on CUDA cores
// y[b, n] = epi(bias[n] + sum_k W[n, k] x[b, k]) for a handful of rows b (one per utterance): the SE gate's two 1x1
// convolutions on the time-mean (ecapa_tdnn_xvector.py:97-111), the time-constant half of the attention's first conv
// (:179-181) and fc2 (:412-422).  As tensor-core GEMM launches these M = B-row products are latency-bound while
// holding whole SMs; here they are plain fp32 FMAs -- a warp owns a 4 x 4 (n x b) tile, its lanes stride over K with
// 16-byte loads, one butterfly at the end -- small enough to run next to the other lane's GEMM CTAs.
// epilogue order as everywhere: +bias -> ReLU -> BN(scale, shift) -> sigmoid | tanh; fp32 and/or split-plane output.
constexpr int kSaWarps = 8;

__global__ void __launch_bounds__(kSaWarps * 32)
small_affine_kernel(const float* __restrict__ x, long long ldx, const float* __restrict__ w, int B, int K, int N,
                    const float* __restrict__ bias, const float* __restrict__ scale, const float* __restrict__ shift, int flags,
                    float* __restrict__ y, long long ldy, __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl,
                    long long ldp) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * 2 + (warp & 1)) * 4;           // block: 2 n-tiles x 4 b-tiles
  const int b0 = (blockIdx.y * 4 + (warp >> 1)) * 4;
  if (n0 >= N || b0 >= B) return;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const float* wr[4];
  const float* xr[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    wr[i] = w + (long long)min(n0 + i, N - 1) * K;             // clamped rows are computed and dropped
    xr[i] = x + (long long)min(b0 + i, B - 1) * ldx;
  }
  for (int k = lane * 4; k < K; k += 128) {                    // K % 4 == 0
    float4 wv[4], xv[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      wv[i] = __ldg(reinterpret_cast<const float4*>(wr[i] + k));
      xv[i] = __ldg(reinterpret_cast<const float4*>(xr[i] + k));
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[i][j] = fmaf(wv[i].x, xv[j].x, acc[i][j]);
        acc[i][j] = fmaf(wv[i].y, xv[j].y, acc[i][j]);
        acc[i][j] = fmaf(wv[i].z, xv[j].z, acc[i][j]);
        acc[i][j] = fmaf(wv[i].w, xv[j].w, acc[i][j]);
      }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float v = acc[i][j];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      acc[i][j] = v;
    }
  if (lane < 16) {
    const int i = lane & 3, j = lane >> 2;                     // lane -> (n0 + i, b0 + j)
    const int n = n0 + i, b = b0 + j;
    if (n < N && b < B) {
      float v = 0.f;
#pragma unroll
      for (int ii = 0; ii < 4; ++ii)
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) v = (ii == i && jj == j) ? acc[ii][jj] : v;
      v += bias ? __ldg(bias + n) : 0.f;
      if (flags & XVB_RELU) v = fmaxf(v, 0.f);
      if (flags & XVB_BN) v = fmaf(v, __ldg(scale + n), __ldg(shift + n));
      if (flags & XVB_TANH) v = tanhf(v);
      if (flags & XVB_SIGMOID) v = 1.f / (1.f + expf(-v));
      if (y) y[(long long)b * ldy + n] = v;
      if (yh) {
        __nv_bfloat16 h, l;
        split_bf16(v, h, l);
        yh[(long long)b * ldp + n] = h;
        yl[(long long)b * ldp + n] = l;
      }
    }
  }
}

// ---------------------------------------------------------------- attention pooling with a head map
// The single-/multi-head attention poolings of libs/nnet/pooling.py (:322-587) differ only in WHICH logit weights
// WHICH channel: output channel o in [0, O) pools input channel c = o % C with the softmax over time of logit
// g = o / gdiv.  AttentiveStatisticsPooling: gdiv = C (one shared alpha); MultiHeadAttentionPooling share=True:
// gdiv = C / num_head, share=False: gdiv = 1; Global / MultiResolution multi-head: O = num_head * C, gdiv = C
// (share) or 1.  One streaming pass, online softmax; per-frame loads of x are 16-byte, logits are scalar
// (broadcast within the warp when heads are wide).  unweighted_var = 1: std of `stddev_attention=False`
// (:357-359): mean_T((x - mean)^2) around the attention-weighted mean.  MQMHASP (:589-698) splits C into heads of
// head_width channels and pools each head `rep` (= num_q) times: c = (o / (rep*head_width))*head_width + o % head_width.
struct OnlineU {
  float m, s0, s1, s2, u1, u2;
};

// xi-vector form (xivec_stdinit_softplus2_prec_pooling, pooling.py:165-212): the raw logit z becomes 2 log(softplus(z)) (a frame's
// log-precision, :189-190) and the softmax runs over T + 1 elements, the extra one being the prior (logit prior_logit[c], value
// prior_x[c], :194-202): it initialises the online-softmax state of warp 0.
// A masked batch (lengths != NULL, device int32[B]) reduces utterance b over frames [0, lengths[b]) only, with the batch
// stride still T rows: the frame walk (warp w takes frames w, w + 8, ...) is the same as a call on that utterance alone,
// so the row is bit-identical to it, and the frames past its end are never loaded.
template <int kRows>
__global__ void __launch_bounds__(kApWarps * 32)
attn_head_stats_pool_kernel(const float* __restrict__ logits, long long ldl, const float* __restrict__ x, long long ldx,
                            int T, int C, int O, int gdiv, int head_width, int rep, float floor_, int unweighted_var,
                            const float* __restrict__ prior_logit,
                            const float* __restrict__ prior_x, int softplus2log, const int* __restrict__ lengths,
                            float* __restrict__ out, __nv_bfloat16* __restrict__ oh, __nv_bfloat16* __restrict__ ol,
                            long long ldo) {
  const int b = blockIdx.y;
  const int Tb = lengths ? __ldg(lengths + b) : T;   // a masked batch reduces utterance b over its own frames only
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int o = blockIdx.x * 128 + lane * 4;
  const bool active = o < O;   // O % 4 == 0, C % 4 == 0: the four outputs read four consecutive input channels
  OnlineU st[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) st[k] = {-INFINITY, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (active) {
    const int c = (o / (rep * head_width)) * head_width + o % head_width;   // head_width = C, rep = O / C: o % C
    int g[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) g[k] = (o + k) / gdiv;
    if (prior_logit && warp == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float px = __ldg(prior_x + c + k);
        st[k] = {__ldg(prior_logit + c + k), 1.f, px, px * px, 0.f, 0.f};
      }
    }
    const float* lb = logits + (long long)b * T * ldl;
    const float* xb = x + (long long)b * T * ldx + c;
    const bool vec_logits = gdiv == 1 && (ldl & 3) == 0 && ((uintptr_t)lb & 15) == 0;   // per-channel logits: 16-byte loads
    for (int t0 = warp; t0 < Tb; t0 += kApWarps * kRows) {
      float4 xv[kRows], lv[kRows];                       // kRows frames in flight per thread before any is consumed
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const int t = t0 + r * kApWarps;
        if (t < Tb) {
          xv[r] = __ldcs(reinterpret_cast<const float4*>(xb + (long long)t * ldx));
          const float* lr = lb + (long long)t * ldl;
          if (vec_logits) lv[r] = __ldcs(reinterpret_cast<const float4*>(lr + o));
          else lv[r] = make_float4(__ldg(lr + g[0]), __ldg(lr + g[1]), __ldg(lr + g[2]), __ldg(lr + g[3]));
        }
      }
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        if (t0 + r * kApWarps >= Tb) continue;
        const float xs[4] = {xv[r].x, xv[r].y, xv[r].z, xv[r].w};
        const float ls[4] = {lv[r].x, lv[r].y, lv[r].z, lv[r].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          float l = ls[k];
          if (softplus2log) {
            l = 2.f * logf(l > 20.f ? l : log1pf(expf(l)));  // Softplus(beta=1, threshold=20), then 2 log
            if (l == -INFINITY) continue;                    // zero precision: weight exactly 0, like exp(-inf) in the softmax
          }
          OnlineU& s = st[k];
          const float mn = fmaxf(s.m, l);
          const float sc = expf(s.m - mn), e = expf(l - mn);
          s.s0 = fmaf(s.s0, sc, e);
          s.s1 = fmaf(s.s1, sc, e * xs[k]);
          s.s2 = fmaf(s.s2, sc, e * xs[k] * xs[k]);
          s.m = mn;
          s.u1 += xs[k];
          s.u2 = fmaf(xs[k], xs[k], s.u2);
        }
      }
    }
  }
  __shared__ OnlineU sh[kApWarps][32][4];
#pragma unroll
  for (int k = 0; k < 4; ++k) sh[warp][lane][k] = st[k];
  __syncthreads();
  if (warp == 0 && active) {
    float mu[4], sd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      OnlineU a = sh[0][lane][k];
      for (int w = 1; w < kApWarps; ++w) {
        const OnlineU& q = sh[w][lane][k];
        if (q.s0 > 0.f) {
          const float mn = fmaxf(a.m, q.m);
          const float sa = expf(a.m - mn), sb = expf(q.m - mn);
          a.s0 = a.s0 * sa + q.s0 * sb;
          a.s1 = a.s1 * sa + q.s1 * sb;
          a.s2 = a.s2 * sa + q.s2 * sb;
          a.m = mn;
          a.u1 += q.u1;
          a.u2 += q.u2;
        }
      }
      mu[k] = a.s1 / a.s0;
      const float var = unweighted_var ? (a.u2 - 2.f * mu[k] * a.u1) / (float)Tb + mu[k] * mu[k]
                                       : a.s2 / a.s0 - mu[k] * mu[k];
      sd[k] = sqrtf(fmaxf(var, floor_));
    }
    float* ob = out + (long long)b * 2 * O;
    *reinterpret_cast<float4*>(ob + o) = make_float4(mu[0], mu[1], mu[2], mu[3]);
    *reinterpret_cast<float4*>(ob + O + o) = make_float4(sd[0], sd[1], sd[2], sd[3]);
    if (oh) {
      __nv_bfloat16 h[8], l[8];
#pragma unroll
      for (int k = 0; k < 4; ++k) { split_bf16(mu[k], h[k], l[k]); split_bf16(sd[k], h[4 + k], l[4 + k]); }
      __nv_bfloat16* ph = oh + (long long)b * ldo;
      __nv_bfloat16* pl = ol + (long long)b * ldo;
      *reinterpret_cast<uint2*>(ph + o) = make_uint2(pack_bf16x2(h[0], h[1]), pack_bf16x2(h[2], h[3]));
      *reinterpret_cast<uint2*>(pl + o) = make_uint2(pack_bf16x2(l[0], l[1]), pack_bf16x2(l[2], l[3]));
      *reinterpret_cast<uint2*>(ph + O + o) = make_uint2(pack_bf16x2(h[4], h[5]), pack_bf16x2(h[6], h[7]));
      *reinterpret_cast<uint2*>(pl + O + o) = make_uint2(pack_bf16x2(l[4], l[5]), pack_bf16x2(l[6], l[7]));
    }
  }
}

static int launch_attn_head_stats_pool(const float* logits, int64_t ldl, const float* x, int64_t ldx, int B, int T, int C, int O,
                                      int gdiv, int head_width, int rep, float floor_, int unweighted_var, const float* prior_logit,
                                      const float* prior_x, int softplus2log, const int* lengths, float* out, uint16_t* out_hi,
                                      uint16_t* out_lo, int64_t ldo, void* stream) {
  dim3 grid((O + 127) / 128, B);
  // frames in flight per thread (XVB_ATTN_ROWS = 1, 2 or 4): 1 by default, since the extra registers of the unrolled
  // forms can cost more occupancy than they hide latency
  static const int rows_knob = getenv("XVB_ATTN_ROWS") ? atoi(getenv("XVB_ATTN_ROWS")) : 1;
  auto* kern = rows_knob == 1 ? attn_head_stats_pool_kernel<1> : rows_knob == 2 ? attn_head_stats_pool_kernel<2> : attn_head_stats_pool_kernel<4>;
  kern<<<grid, kApWarps * 32, 0, (cudaStream_t)stream>>>(
      logits, ldl, x, ldx, T, C, O, gdiv, head_width, rep, floor_, unweighted_var, prior_logit, prior_x, softplus2log, lengths,
      out,
      reinterpret_cast<__nv_bfloat16*>(out_hi), reinterpret_cast<__nv_bfloat16*>(out_lo), ldo);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

}  // namespace xvb

using namespace xvb;

extern "C" int xvb_lde_pool(const float* x, int64_t ldx, int B, int T, int C, const float* mu, int K, const float* neg_beta,
                            float* w_scratch, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x && mu && neg_beta && w_scratch && out && B > 0 && T > 0 && C > 0 && ldx >= C, "xvb_lde_pool: bad arguments");
  XVB_CHECK_ARG(K >= 1 && K <= kLdeMaxK, "xvb_lde_pool: %d clusters (1..%d)", K, kLdeMaxK);
  XVB_CHECK_ARG((out_hi != nullptr) == (out_lo != nullptr) && (!out_hi || ldo >= (int64_t)C * K), "xvb_lde_pool: bad plane output");
  XVB_CHECK_ARG(B <= 65535, "xvb_lde_pool: too many utterances for one launch");
  const long long rows = (long long)B * T;
  lde_weights_kernel<<<(unsigned)((rows + kLdeFrames - 1) / kLdeFrames), 256, 0, (cudaStream_t)stream>>>(x, ldx, rows, C, mu, K,
                                                                                                        neg_beta, w_scratch);
  XVB_LAUNCH_CHECK();
  dim3 grid((C + 32 * kLdeFr - 1) / (32 * kLdeFr), B);
  lde_encode_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, T, C, mu, K, w_scratch, out,
                                                           reinterpret_cast<__nv_bfloat16*>(out_hi),
                                                           reinterpret_cast<__nv_bfloat16*>(out_lo), ldo);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_small_affine(const float* x, int64_t ldx, const float* w, int B, int K, int N, const float* bias,
                                const float* bn_scale, const float* bn_shift, int flags, float* y, int64_t ldy,
                                uint16_t* y_hi, uint16_t* y_lo, int64_t ldplane, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x && w && (y || y_hi) && B > 0 && K > 0 && N > 0, "xvb_small_affine: bad arguments");
  XVB_CHECK_ARG(K % 4 == 0 && ldx % 4 == 0 && ldx >= K && ((uintptr_t)x | (uintptr_t)w) % 16 == 0,
                "xvb_small_affine: K and ldx must be multiples of 4, x and w 16-byte aligned");
  XVB_CHECK_ARG(!(flags & XVB_BN) || (bn_scale && bn_shift), "xvb_small_affine: XVB_BN without scale/shift");
  XVB_CHECK_ARG((y_hi != nullptr) == (y_lo != nullptr), "xvb_small_affine: y_hi/y_lo must both be set or both NULL");
  XVB_CHECK_ARG((!y || ldy >= N) && (!y_hi || ldplane >= N), "xvb_small_affine: output pitch smaller than N");
  dim3 grid((N + 7) / 8, (B + 15) / 16);
  XVB_CHECK_ARG(grid.y <= 65535, "xvb_small_affine: too many rows (%d) -- this is the segment-level kernel", B);
  small_affine_kernel<<<grid, kSaWarps * 32, 0, (cudaStream_t)stream>>>(
      x, ldx, w, B, K, N, bias, bn_scale, bn_shift, flags, y, ldy, reinterpret_cast<__nv_bfloat16*>(y_hi),
      reinterpret_cast<__nv_bfloat16*>(y_lo), ldplane);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

// The checks and launch of xvb_attn_head_stats_pool_prior and _lengths (lengths NULL: every utterance has T frames).
static int attn_head_stats_pool_run(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T, int C,
                                    int O, int gdiv, float floor_, int unweighted_var, const float* prior_logit,
                                    const float* prior_x, int softplus2log, const int* lengths, float* out, uint16_t* out_hi,
                                    uint16_t* out_lo, int64_t ldo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG((prior_logit != nullptr) == (prior_x != nullptr) && (!prior_logit || (O == C && !unweighted_var)),
                "xvb_attn_head_stats_pool: the prior element needs both arrays, O == C and weighted moments");
  XVB_CHECK_ARG(logits && x && out, "xvb_attn_head_stats_pool: null pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && C % 4 == 0 && O > 0 && O % C == 0 && ldx % 4 == 0 && ldx >= C && B <= 65535,
                "xvb_attn_head_stats_pool: need C%%4==0, O a multiple of C, ldx%%4==0");
  XVB_CHECK_ARG(gdiv > 0 && G > 0 && ldl >= G && (O - 1) / gdiv < G,
                "xvb_attn_head_stats_pool: the head map o / gdiv must stay inside the %d logits", G);
  XVB_CHECK_ARG((out_hi != nullptr) == (out_lo != nullptr), "xvb_attn_head_stats_pool: out_hi/out_lo must both be set or both NULL");
  if (out_hi) XVB_CHECK_ARG(ldo % 4 == 0 && ldo >= 2 * (int64_t)O, "xvb_attn_head_stats_pool: ldo too small / unaligned");
  return launch_attn_head_stats_pool(logits, ldl, x, ldx, B, T, C, O, gdiv, C, O / C, floor_, unweighted_var, prior_logit,
                                     prior_x, softplus2log, lengths, out, out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_attn_head_stats_pool(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T,
                                        int C, int O, int gdiv, float floor_, int unweighted_var, float* out,
                                        uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream) {
  return xvb_attn_head_stats_pool_prior(logits, ldl, G, x, ldx, B, T, C, O, gdiv, floor_, unweighted_var, nullptr, nullptr, 0, out,
                                        out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_attn_head_stats_pool_prior(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T,
                                              int C, int O, int gdiv, float floor_, int unweighted_var, const float* prior_logit,
                                              const float* prior_x, int softplus2log, float* out, uint16_t* out_hi,
                                              uint16_t* out_lo, int64_t ldo, void* stream) {
  return attn_head_stats_pool_run(logits, ldl, G, x, ldx, B, T, C, O, gdiv, floor_, unweighted_var, prior_logit, prior_x,
                                  softplus2log, nullptr, out, out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_attn_head_stats_pool_lengths(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B,
                                                int T, int C, int O, int gdiv, float floor_, int unweighted_var,
                                                const float* prior_logit, const float* prior_x, int softplus2log,
                                                const int* lengths, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo,
                                                void* stream) {
  XVB_CHECK_ARG(lengths, "xvb_attn_head_stats_pool_lengths: null lengths");
  return attn_head_stats_pool_run(logits, ldl, G, x, ldx, B, T, C, O, gdiv, floor_, unweighted_var, prior_logit, prior_x,
                                  softplus2log, lengths, out, out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_attn_head_stats_pool_mq(const float* logits, int64_t ldl, int G, const float* x, int64_t ldx, int B, int T,
                                           int C, int O, int gdiv, int head_width, int rep, float floor_, int unweighted_var,
                                           float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(logits && x && out, "xvb_attn_head_stats_pool_mq: null pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && ldx % 4 == 0 && ldx >= C && B <= 65535 && head_width > 0 && head_width % 4 == 0 &&
                C % head_width == 0 && rep > 0 && O == rep * C,
                "xvb_attn_head_stats_pool_mq: need head_width %% 4 == 0 dividing C, O == rep * C, ldx %% 4 == 0");
  XVB_CHECK_ARG(gdiv > 0 && G > 0 && ldl >= G && (O - 1) / gdiv < G,
                "xvb_attn_head_stats_pool_mq: the logit map o / gdiv must stay inside the %d logits", G);
  XVB_CHECK_ARG((out_hi != nullptr) == (out_lo != nullptr), "xvb_attn_head_stats_pool_mq: out_hi/out_lo must both be set or both NULL");
  if (out_hi) XVB_CHECK_ARG(ldo % 4 == 0 && ldo >= 2 * (int64_t)O, "xvb_attn_head_stats_pool_mq: ldo too small / unaligned");
  return launch_attn_head_stats_pool(logits, ldl, x, ldx, B, T, C, O, gdiv, head_width, rep, floor_, unweighted_var, nullptr,
                                     nullptr, 0, nullptr, out, out_hi, out_lo, ldo, stream);
}

namespace {

int plane_mean_run(const char* fn, const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int B, int T, int C,
                   const int* lengths, int rows_per_length, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo,
                   void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x_hi && x_lo && (out || out_hi), "%s: null pointer", fn);
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0 && ldx >= C && B <= 65535, "%s: need C%%8==0, ldx%%8==0", fn);
  XVB_CHECK_ARG((out_hi != nullptr) == (out_lo != nullptr), "%s: out_hi/out_lo must both be set or both NULL", fn);
  if (out_hi) XVB_CHECK_ARG(ldo % 8 == 0 && ldo >= C, "%s: ldo must be a multiple of 8 and >= C", fn);
  dim3 grid((C + 255) / 256, B);
  plane_mean_kernel<<<grid, kPmWarps * 32, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(x_hi), reinterpret_cast<const __nv_bfloat16*>(x_lo), ldx, T, C, lengths,
      rows_per_length, out, reinterpret_cast<__nv_bfloat16*>(out_hi), reinterpret_cast<__nv_bfloat16*>(out_lo), ldo);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

}  // namespace

extern "C" int xvb_plane_mean(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int B, int T, int C, float* out,
                              uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream) {
  return plane_mean_run("xvb_plane_mean", x_hi, x_lo, ldx, B, T, C, nullptr, 1, out, out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_plane_mean_lengths(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int B, int T, int C,
                                      const int* lengths, int rows_per_length, float* out, uint16_t* out_hi, uint16_t* out_lo,
                                      int64_t ldo, void* stream) {
  XVB_CHECK_ARG(lengths && rows_per_length > 0, "xvb_plane_mean_lengths: null lengths or rows_per_length=%d < 1",
                rows_per_length);
  return plane_mean_run("xvb_plane_mean_lengths", x_hi, x_lo, ldx, B, T, C, lengths, rows_per_length, out, out_hi, out_lo,
                        ldo, stream);
}

extern "C" int xvb_copy_rows(const void* src, int64_t src_pitch_bytes, void* dst, int64_t dst_pitch_bytes, int64_t rows,
                             int64_t row_bytes, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(src && dst && rows > 0 && row_bytes > 0, "xvb_copy_rows: bad arguments");
  XVB_CHECK_ARG(row_bytes % 16 == 0 && src_pitch_bytes % 16 == 0 && dst_pitch_bytes % 16 == 0 &&
                    ((uintptr_t)src | (uintptr_t)dst) % 16 == 0, "xvb_copy_rows: 16-byte granularity required");
  const long long total = rows * (row_bytes / 16);
  long long g = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  copy_rows_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint4*>(src), src_pitch_bytes / 16,
                                                                   reinterpret_cast<uint4*>(dst), dst_pitch_bytes / 16, rows,
                                                                   (int)(row_bytes / 16));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_se_apply(const uint16_t* z_hi, const uint16_t* z_lo, int64_t ldz, const uint16_t* in_hi,
                            const uint16_t* in_lo, int64_t ldin, const float* gate, uint16_t* out_hi, uint16_t* out_lo,
                            int64_t ldout, uint16_t* next_hi, uint16_t* next_lo, int64_t ldnext, int B, int T, int C,
                            void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(z_hi && z_lo && in_hi && in_lo && gate && out_hi && out_lo, "xvb_se_apply: null pointer");
  XVB_CHECK_ARG((next_hi != nullptr) == (next_lo != nullptr), "xvb_se_apply: next_hi/next_lo must both be set or both NULL");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && C % 8 == 0 && ldz % 8 == 0 && ldin % 8 == 0 && ldout % 8 == 0 &&
                    (!next_hi || ldnext % 8 == 0), "xvb_se_apply: C and all pitches must be multiples of 8");
  return launch_se_apply(z_hi, z_lo, ldz, in_hi, in_lo, ldin, gate, T, out_hi, out_lo, ldout, next_hi, next_lo, ldnext, B, T, C,
                         stream);
}

extern "C" int xvb_seg_gate_apply(const uint16_t* z_hi, const uint16_t* z_lo, int64_t ldz, const uint16_t* in_hi,
                                  const uint16_t* in_lo, int64_t ldin, const float* gate, int seg_len, uint16_t* out_hi,
                                  uint16_t* out_lo, int64_t ldout, int B, int T, int C, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(z_hi && z_lo && gate && out_hi && out_lo, "xvb_seg_gate_apply: null pointer");
  XVB_CHECK_ARG((in_hi != nullptr) == (in_lo != nullptr), "xvb_seg_gate_apply: in_hi/in_lo must both be set or both NULL");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && seg_len > 0 && C % 8 == 0 && ldz % 8 == 0 && ldout % 8 == 0 && (!in_hi || ldin % 8 == 0),
                "xvb_seg_gate_apply: need seg_len > 0, C and all pitches multiples of 8");
  XVB_CHECK_ARG(((uintptr_t)z_hi | (uintptr_t)z_lo | (uintptr_t)in_hi | (uintptr_t)in_lo | (uintptr_t)gate | (uintptr_t)out_hi |
                 (uintptr_t)out_lo) % 16 == 0, "xvb_seg_gate_apply: pointers must be 16-byte aligned");
  return launch_se_apply(z_hi, z_lo, ldz, in_hi, in_lo, ldin, gate, seg_len, out_hi, out_lo, ldout, nullptr, nullptr, 0, B, T, C,
                         stream);
}

static int attn_stats_pool(const float* logits, int64_t ldl, const float* x, int64_t ldx, int B, int T, int C, float floor_,
                           const int* lengths, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(logits && x && out, "xvb_attn_stats_pool: null pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && C > 0 && C % 4 == 0 && ldl % 4 == 0 && ldx % 4 == 0 && ldl >= C && ldx >= C && B <= 65535,
                "xvb_attn_stats_pool: need C%%4==0 and pitches %%4==0");
  XVB_CHECK_ARG((out_hi != nullptr) == (out_lo != nullptr), "xvb_attn_stats_pool: out_hi/out_lo must both be set or both NULL");
  if (out_hi) XVB_CHECK_ARG(ldo % 4 == 0 && ldo >= 2 * C, "xvb_attn_stats_pool: ldo too small / unaligned");
  dim3 grid((C + 127) / 128, B);
  attn_stats_pool_kernel<<<grid, kApWarps * 32, 0, (cudaStream_t)stream>>>(
      logits, ldl, x, ldx, T, C, floor_, lengths, out, reinterpret_cast<__nv_bfloat16*>(out_hi),
      reinterpret_cast<__nv_bfloat16*>(out_lo), ldo);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_attn_stats_pool(const float* logits, int64_t ldl, const float* x, int64_t ldx, int B, int T, int C,
                                   float floor_, float* out, uint16_t* out_hi, uint16_t* out_lo, int64_t ldo,
                                   void* stream) {
  return attn_stats_pool(logits, ldl, x, ldx, B, T, C, floor_, nullptr, out, out_hi, out_lo, ldo, stream);
}

extern "C" int xvb_attn_stats_pool_lengths(const float* logits, int64_t ldl, const float* x, int64_t ldx, int B, int T, int C,
                                           float floor_, const int* lengths, float* out, uint16_t* out_hi, uint16_t* out_lo,
                                           int64_t ldo, void* stream) {
  XVB_CHECK_ARG(lengths, "xvb_attn_stats_pool_lengths: null lengths");
  return attn_stats_pool(logits, ldl, x, ldx, B, T, C, floor_, lengths, out, out_hi, out_lo, ldo, stream);
}
