// 2-D convolution of the ResNet x-vector (pytorch/libs/nnet/resnet.py BasicBlock, pytorch/model/resnet_xvector.py)
// as an implicit-GEMM warpgroup-MMA kernel (sm_90a), plus the two bandwidth-bound pieces around it.
//
//   y[b,t,f,n] = epi( sum_{kf,kt} sum_c W[n, c, kf, kt] * x[b, t*s + kt - p, f*s + kf - p, c] )
//
// The reference feeds (1, 1, F, T) to Conv2d: "H" is the feature axis, "W" is time.  Here a frame tensor is a
// channel-contiguous (B, T, F, C) split-plane pair, and the kernel reads it through a 4-D tensor map (C, F, T, B):
//   * M = output positions, N = Cout, K = taps x Cin, tap-major (the xvb_pack_tdnn_weight layout of the weight
//     viewed as (Cout, Cin, k*k) with the kept taps as context); the taps are a list of (kf, kt) offsets, all k*k of a
//     dense window (xvb_conv2d) or any increasing subset of a k <= 5 window (xvb_conv2d_taps: a re-parameterised RepSPK
//     block is a 5x5 kernel with 8 taps that are always zero, which then cost nothing);
//   * an M tile is 128 positions = Bb utterances x Tb frames x Fb feature bins (powers of two, chosen on the host for
//     the fewest padded rows); tap (kf, kt) is only a coordinate offset, so TMA's out-of-bounds zero fill is exactly
//     the convolution's zero padding and never reads a neighbouring utterance;
//   * stride 2 uses the tensor map's element strides: the box traverses 2*Fb x 2*Tb input positions and lands Fb x Tb
//     of them, so no output is computed and thrown away; the two axes take their strides separately (CAM++'s FCM head
//     strides the feature axis only, stride (2, 1));
//   * Cin = 32 (the first stage) loads 64-channel boxes whose upper half TMA zero-fills; the MMA loop stops after the
//     real 32 channels, so the padding costs shared-memory traffic and no tensor-core work;
//   * numerics and pipeline are the TDNN layer's (tdnn_gemm.cu): bf16 hi/lo planes, three wgmma per K step into fp32
//     register accumulators, one TMA producer warp feeding an mbarrier operand ring, two consumer warpgroups;
//   * epilogue: y = acc * scale[n] + shift[n] (eval BatchNorm after the bias-free conv) [+ residual] [ReLU] -> planes
//     and/or fp32, and optionally a second output relu(y * scale2[n] + shift2[n]) (the next pre-activation block's
//     BN-ReLU, which cannot be folded into that block's conv because the zero padding comes after it);
//   * a masked batch (lengths: each utterance's input length) stores exact zeros at the frames past each utterance's
//     output length, so the next conv's taps read that utterance's own zero padding; the tiles are computed in full.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "ptx.cuh"

namespace xvb {
namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                      // bf16 elements = one 128-byte swizzle row
constexpr int kABytes = kBlockM * kBlockK * 2;   // 16 KB per plane per stage
constexpr int kNumConsumers = 256;
constexpr int kProducerWarp = kNumConsumers / 32;
constexpr int kNumThreads = kNumConsumers + 32;
constexpr int kMaxConvTaps = 25;                 // a 5x5 window

struct Conv2dParams {
  int B, T, F, Cin, To, Fo, Cout;
  int ks, stride, stride_t, pad;   // stride: feature axis; stride_t: time axis
  int ntaps;
  int8_t tap_f[kMaxConvTaps], tap_t[kMaxConvTaps];   // (kf, kt) of packed tap j
  int Fb, Tb, Bb, log2_fb, log2_tb;
  int num_f_blk, num_t_blk, num_n_blk, num_tiles;
  int cin_p16, num_cblk;
  int relu;
  const float* scale;
  const float* shift;
  const __nv_bfloat16* res_hi;
  const __nv_bfloat16* res_lo;
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
  float* y_f32;
  const float* scale2;
  const float* shift2;
  __nv_bfloat16* y2_hi;
  __nv_bfloat16* y2_lo;
  const int* lengths;   // NULL, or the input length of each utterance (xvb_conv2d_args_t.lengths)
};

template <int BLOCK_N>
struct ConvCfg {
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes > 6 ? 6 : (192 * 1024) / kStageBytes;
  static constexpr int kAccRegs = BLOCK_N / 2;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB shared memory of an sm_90 CTA");
  static_assert(kStages >= 2, "need at least a double-buffered operand pipeline");
};

// tile -> (first output position of the M tile, N block); N fastest so that CTAs running together share the A tile
__device__ __forceinline__ void decode_conv_tile(const Conv2dParams& p, int tile, int& b0, int& t0, int& f0, int& n_blk) {
  n_blk = tile % p.num_n_blk;
  int m = tile / p.num_n_blk;
  f0 = (m % p.num_f_blk) * p.Fb;
  m /= p.num_f_blk;
  t0 = (m % p.num_t_blk) * p.Tb;
  b0 = (m / p.num_t_blk) * p.Bb;
}

// A masked batch's output frames past an utterance's end: zeros in every output (y, y_f32, y2), this thread's column
// pairs c, c + 8, ... below c_end.  Out of line, so that the unmasked epilogue keeps its code and registers.
__device__ __noinline__ void conv_zero_row(const Conv2dParams& p, long long off, int c_begin, int c_end) {
  for (int c = c_begin; c < c_end; c += 8) {
    if (p.y_hi) {
      *reinterpret_cast<uint32_t*>(p.y_hi + off + c) = 0u;
      *reinterpret_cast<uint32_t*>(p.y_lo + off + c) = 0u;
    }
    if (p.y_f32) *reinterpret_cast<float2*>(p.y_f32 + off + c) = make_float2(0.f, 0.f);
    if (p.y2_hi) {
      *reinterpret_cast<uint32_t*>(p.y2_hi + off + c) = 0u;
      *reinterpret_cast<uint32_t*>(p.y2_lo + off + c) = 0u;
    }
  }
}

// Output frames of utterance b in a masked batch: the conv's own rule (conv2d_run's To) applied to its input length.
__device__ __noinline__ int conv_out_length(const Conv2dParams& p, int b) {
  return (__ldg(p.lengths + b) + 2 * p.pad - p.ks) / p.stride_t + 1;
}

template <int BLOCK_N>
__global__ void __launch_bounds__(kNumThreads, 1)
conv2d_bf16x3_kernel(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                     const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                     const __grid_constant__ Conv2dParams p) {
  using Cfg = ConvCfg<BLOCK_N>;
  constexpr int kStages = Cfg::kStages;
  constexpr int kBBytes = Cfg::kBBytes;
  constexpr int kStageBytes = Cfg::kStageBytes;

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
  uint64_t* empty_bar = full_bar + kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&map_x_hi);
    tma_prefetch_desc(&map_x_lo);
    tma_prefetch_desc(&map_w_hi);
    tma_prefetch_desc(&map_w_lo);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kNumConsumers / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("fence.proxy.async;" ::: "memory");   // operands may come from generic-proxy stores of the previous kernel

  const int num_kblk = p.ntaps * p.num_cblk;

  if (warp == kProducerWarp) {
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        int b0, t0, f0, n_blk;
        decode_conv_tile(p, tile, b0, t0, f0, n_blk);
        const int n0 = n_blk * BLOCK_N;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int fi = f0 * p.stride + p.tap_f[tap] - p.pad;
          const int ti = t0 * p.stride_t + p.tap_t[tap] - p.pad;
          for (int cb = 0; cb < p.num_cblk; ++cb) {
            mbar_wait(&empty_bar[stage], phase ^ 1);
            uint8_t* s = smem + stage * kStageBytes;
            mbar_expect_tx(&full_bar[stage], kStageBytes);
            tma_load_4d(s, &map_x_hi, &full_bar[stage], cb * kBlockK, fi, ti, b0);
            tma_load_4d(s + kABytes, &map_x_lo, &full_bar[stage], cb * kBlockK, fi, ti, b0);
            tma_load_2d(s + 2 * kABytes, &map_w_hi, &full_bar[stage], tap * p.cin_p16 + cb * kBlockK, n0);
            tma_load_2d(s + 2 * kABytes + kBBytes, &map_w_lo, &full_bar[stage], tap * p.cin_p16 + cb * kBlockK, n0);
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ================================ consumers: wgmma + epilogue ================================
  const int wg = warp >> 2;
  const int q4 = lane & 3;
  const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // this thread's rows: row0 and row0 + 8
  const float relu_floor = p.relu ? 0.f : -INFINITY;
  float acc[Cfg::kAccRegs];
#pragma unroll
  for (int i = 0; i < Cfg::kAccRegs; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;

  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    int prev_stage = -1;
    uint32_t scale_d = 0;
    for (int kb = 0; kb < num_kblk; ++kb) {
      const int cb = kb % p.num_cblk;
      int nsteps = (p.Cin - cb * kBlockK + 15) >> 4;
      nsteps = nsteps > 4 ? 4 : nsteps;
      mbar_wait(&full_bar[stage], phase);
      const uint32_t sa = smem_u32(smem + stage * kStageBytes);
      const uint64_t m_off = (uint64_t)((wg * 64 * 128) >> 4);
      const uint64_t da_hi = make_sw128_desc(sa) + m_off, da_lo = make_sw128_desc(sa + kABytes) + m_off;
      const uint64_t db_hi = make_sw128_desc(sa + 2 * kABytes), db_lo = make_sw128_desc(sa + 2 * kABytes + kBBytes);
      wgmma_fence();
      for (int s = 0; s < nsteps; ++s) {
        const uint64_t koff = (uint64_t)(s * 32 >> 4);
        wgmma_bf16<BLOCK_N>(acc, da_lo + koff, db_hi + koff, scale_d);
        wgmma_bf16<BLOCK_N>(acc, da_hi + koff, db_lo + koff, 1);
        wgmma_bf16<BLOCK_N>(acc, da_hi + koff, db_hi + koff, 1);
        scale_d = 1;
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    // ---- epilogue: BN -> [+ residual] -> [ReLU] -> planes / fp32 [, relu(BN2) planes]
    int b0, t0, f0, n_blk;
    decode_conv_tile(p, tile, b0, t0, f0, n_blk);
    const int n0 = n_blk * BLOCK_N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      const int f = f0 + (row & (p.Fb - 1));
      const int t = t0 + ((row >> p.log2_fb) & (p.Tb - 1));
      const int b = b0 + (row >> (p.log2_fb + p.log2_tb));
      if (f >= p.Fo || t >= p.To || b >= p.B) continue;
      const long long off = (((long long)b * p.To + t) * p.Fo + f) * p.Cout;
      if (p.lengths && t >= conv_out_length(p, b)) {   // masked batch, frame past the utterance's end
        conv_zero_row(p, off, n0 + 2 * q4, min(n0 + BLOCK_N, p.Cout));
        continue;
      }
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        const int c = n0 + 8 * i + 2 * q4;   // Cout % 16 == 0: c and c + 1 both exist or neither
        if (c >= p.Cout) break;
        float x[2] = {acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]};
        if (p.scale) {
          x[0] = fmaf(x[0], __ldg(p.scale + c), __ldg(p.shift + c));
          x[1] = fmaf(x[1], __ldg(p.scale + c + 1), __ldg(p.shift + c + 1));
        }
        if (p.res_hi) {
          const uint32_t rh = *reinterpret_cast<const uint32_t*>(p.res_hi + off + c);
          const uint32_t rl = *reinterpret_cast<const uint32_t*>(p.res_lo + off + c);
          x[0] += __uint_as_float(rh << 16) + __uint_as_float(rl << 16);
          x[1] += __uint_as_float(rh & 0xffff0000u) + __uint_as_float(rl & 0xffff0000u);
        }
        x[0] = fmaxf(x[0], relu_floor);
        x[1] = fmaxf(x[1], relu_floor);
        if (p.y_hi) {
          __nv_bfloat16 h0, l0, h1, l1;
          split_bf16(x[0], h0, l0);
          split_bf16(x[1], h1, l1);
          *reinterpret_cast<uint32_t*>(p.y_hi + off + c) = pack_bf16x2(h0, h1);
          *reinterpret_cast<uint32_t*>(p.y_lo + off + c) = pack_bf16x2(l0, l1);
        }
        if (p.y_f32) *reinterpret_cast<float2*>(p.y_f32 + off + c) = make_float2(x[0], x[1]);
        if (p.y2_hi) {
          const float u0 = fmaxf(fmaf(x[0], __ldg(p.scale2 + c), __ldg(p.shift2 + c)), 0.f);
          const float u1 = fmaxf(fmaf(x[1], __ldg(p.scale2 + c + 1), __ldg(p.shift2 + c + 1)), 0.f);
          __nv_bfloat16 h0, l0, h1, l1;
          split_bf16(u0, h0, l0);
          split_bf16(u1, h1, l1);
          *reinterpret_cast<uint32_t*>(p.y2_hi + off + c) = pack_bf16x2(h0, h1);
          *reinterpret_cast<uint32_t*>(p.y2_lo + off + c) = pack_bf16x2(l0, l1);
        }
      }
    }
  }
}

// Head conv (Cin = 1, KxK with K = 3 or 5, stride 1, padding K/2) on CUDA cores, fp32: its input rows (one value per
// position) break TMA's 16-byte rule and it is ~0.1 % of the MACs.  One thread per (position, 8 output channels);
// fused BN + ReLU, the split to planes and the optional second output relu(y * scale2 + shift2).  A masked batch
// (lengths != NULL) reads the frames t >= lengths[b] as zeros and stores zeros there.
template <int K>
__global__ void head_conv_kernel(const float* __restrict__ x, const int* __restrict__ lengths, int B, int T, int F,
                                 const float* __restrict__ w, int Cout,
                                 const float* __restrict__ scale, const float* __restrict__ shift,
                                 __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl,
                                 const float* __restrict__ scale2, const float* __restrict__ shift2,
                                 __nv_bfloat16* __restrict__ y2h, __nv_bfloat16* __restrict__ y2l) {
  const int groups = Cout / 8;
  const long long total = (long long)B * T * F * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % groups) * 8;
    const long long pos = i / groups;
    const int f = (int)(pos % F);
    const long long bt = pos / F;
    const int t = (int)(bt % T);
    const long long b = bt / T;
    const int L = lengths ? __ldg(lengths + b) : T;
    uint4 h, l;
    if (t >= L) {
      h = l = make_uint4(0u, 0u, 0u, 0u);
      *reinterpret_cast<uint4*>(yh + pos * Cout + c0) = h;
      *reinterpret_cast<uint4*>(yl + pos * Cout + c0) = l;
      if (y2h) {
        *reinterpret_cast<uint4*>(y2h + pos * Cout + c0) = h;
        *reinterpret_cast<uint4*>(y2l + pos * Cout + c0) = l;
      }
      continue;
    }
    float in[K * K];
#pragma unroll
    for (int kf = 0; kf < K; ++kf)
#pragma unroll
      for (int kt = 0; kt < K; ++kt) {
        const int ff = f + kf - K / 2, tt = t + kt - K / 2;
        in[kf * K + kt] = (ff >= 0 && ff < F && tt >= 0 && tt < L) ? __ldg(x + (b * T + tt) * F + ff) : 0.f;
      }
    float y[8], y2[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float* wc = w + (c0 + k) * (K * K);
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < K * K; ++j) s = fmaf(__ldg(wc + j), in[j], s);
      y[k] = fmaxf(fmaf(s, __ldg(scale + c0 + k), __ldg(shift + c0 + k)), 0.f);
      if (y2h) y2[k] = fmaxf(fmaf(y[k], __ldg(scale2 + c0 + k), __ldg(shift2 + c0 + k)), 0.f);
    }
    pack8(y, h, l);
    *reinterpret_cast<uint4*>(yh + pos * Cout + c0) = h;
    *reinterpret_cast<uint4*>(yl + pos * Cout + c0) = l;
    if (y2h) {
      pack8(y2, h, l);
      *reinterpret_cast<uint4*>(y2h + pos * Cout + c0) = h;
      *reinterpret_cast<uint4*>(y2l + pos * Cout + c0) = l;
    }
  }
}

// y = [relu]( z * gate[b, c] + identity ) over (B, P, C) planes -> planes and/or fp32 [, relu(y * scale2 + shift2) planes]:
// SEBlock_2D's scaling (components.py:630-639) with the residual add of BasicBlock (resnet.py:70-104).  A masked batch
// (lengths != NULL, P = T * F positions per utterance) stores zeros at the positions of frames t >= lengths[b].
__global__ void se_residual_kernel(const __nv_bfloat16* __restrict__ zh, const __nv_bfloat16* __restrict__ zl,
                                   const float* __restrict__ gate, const __nv_bfloat16* __restrict__ ih,
                                   const __nv_bfloat16* __restrict__ il, long long P, int C, const int* __restrict__ lengths,
                                   int F, int relu,
                                   __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, float* __restrict__ yf,
                                   const float* __restrict__ scale2, const float* __restrict__ shift2,
                                   __nv_bfloat16* __restrict__ y2h, __nv_bfloat16* __restrict__ y2l, long long total) {
  const int groups = C / 8;
  const float floor_v = relu ? 0.f : -INFINITY;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long pos = i / groups;
    const int c = (int)(i % groups) * 8;
    const long long b = pos / P;
    const long long e = pos * C + c;
    uint4 h, l;
    if (lengths && pos - b * P >= (long long)__ldg(lengths + b) * F) {
      h = l = make_uint4(0u, 0u, 0u, 0u);
      if (yh) {
        *reinterpret_cast<uint4*>(yh + e) = h;
        *reinterpret_cast<uint4*>(yl + e) = l;
      }
      if (yf) {
        *reinterpret_cast<float4*>(yf + e) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(yf + e + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      if (y2h) {
        *reinterpret_cast<uint4*>(y2h + e) = h;
        *reinterpret_cast<uint4*>(y2l + e) = l;
      }
      continue;
    }
    float z[8], x[8], y[8];
    unpack8(*reinterpret_cast<const uint4*>(zh + e), *reinterpret_cast<const uint4*>(zl + e), z);
    unpack8(*reinterpret_cast<const uint4*>(ih + e), *reinterpret_cast<const uint4*>(il + e), x);
    const float4 g0 = *reinterpret_cast<const float4*>(gate + b * C + c);
    const float4 g1 = *reinterpret_cast<const float4*>(gate + b * C + c + 4);
    const float g[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) y[k] = fmaxf(__fadd_rn(__fmul_rn(z[k], g[k]), x[k]), floor_v);   // the reference's two roundings
    if (yh) {
      pack8(y, h, l);
      *reinterpret_cast<uint4*>(yh + e) = h;
      *reinterpret_cast<uint4*>(yl + e) = l;
    }
    if (yf) {
      *reinterpret_cast<float4*>(yf + e) = make_float4(y[0], y[1], y[2], y[3]);
      *reinterpret_cast<float4*>(yf + e + 4) = make_float4(y[4], y[5], y[6], y[7]);
    }
    if (y2h) {
#pragma unroll
      for (int k = 0; k < 8; ++k) y[k] = fmaxf(fmaf(y[k], __ldg(scale2 + c + k), __ldg(shift2 + c + k)), 0.f);
      pack8(y, h, l);
      *reinterpret_cast<uint4*>(y2h + e) = h;
      *reinterpret_cast<uint4*>(y2l + e) = l;
    }
  }
}

int grid_for(long long total, int block) {
  long long g = (total + block - 1) / block;
  const long long cap = (long long)sm_count() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// (Fb, Tb, Bb) powers of two with Fb*Tb*Bb = 128 and the fewest padded output rows; ties go to the fewest utterances
// per tile, then the widest Fb (spatially compact tiles: the 9 taps of one tile overlap in L2).  stride_f / stride_t:
// the feature / time strides, which scale the TMA box along their axis.
void choose_conv_tile(int B, int To, int Fo, int stride_f, int stride_t, int* Fb, int* Tb, int* Bb) {
  long long best = -1;
  for (int lb = 0; lb <= 7; ++lb) {
    for (int lf = 7 - lb; lf >= 0; --lf) {
      const int bb = 1 << lb, fb = 1 << lf, tb = 128 / (bb * fb);
      if (fb * stride_f > 256 || tb * stride_t > 256) continue;   // TMA box dimensions <= 256
      const long long rows = (long long)((Fo + fb - 1) / fb) * fb * ((To + tb - 1) / tb) * tb * ((B + bb - 1) / bb) * bb;
      if (best < 0 || rows < best) { best = rows; *Fb = fb; *Tb = tb; *Bb = bb; }
    }
  }
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// 4-D bf16 map of a (B, T, F, C) position tensor with element strides (the strided traversal of stride-2 convs, which
// make_tensor_map does not expose)
int make_position_map(CUtensorMap* m, const void* base, const cuuint64_t* dims, const cuuint64_t* strides,
                      const cuuint32_t* box, const cuuint32_t* estr) {
  static PFN_encodeTiled enc = [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    return (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess) ? reinterpret_cast<PFN_encodeTiled>(f) : nullptr;
  }();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return XVB_ECUDA; }
  const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled(position map C=%llu F=%llu T=%llu B=%llu) failed: %d", (unsigned long long)dims[0],
              (unsigned long long)dims[1], (unsigned long long)dims[2], (unsigned long long)dims[3], (int)r);
    return XVB_ECUDA;
  }
  return XVB_OK;
}

template <int BLOCK_N>
int launch_conv(const CUtensorMap* mx, Conv2dParams& p, const void* w_hi, const void* w_lo, cudaStream_t stream) {
  using Cfg = ConvCfg<BLOCK_N>;
  CUtensorMap mw_hi, mw_lo;   // packed (Cout, k*k*Cin) weight, K contiguous; box 64 x BLOCK_N
  const unsigned long long K = (unsigned long long)p.ntaps * p.cin_p16;
  const unsigned long long wd[2] = {K, (unsigned long long)p.Cout};
  const unsigned long long ws[1] = {K * 2};
  const unsigned wb[2] = {(unsigned)kBlockK, (unsigned)BLOCK_N};
  int rc;
  if ((rc = make_tensor_map(&mw_hi, w_hi, 2, 2, wd, ws, wb, 128))) return rc;
  if ((rc = make_tensor_map(&mw_lo, w_lo, 2, 2, wd, ws, wb, 128))) return rc;
  p.num_n_blk = (p.Cout + BLOCK_N - 1) / BLOCK_N;
  const long long tiles = (long long)p.num_f_blk * p.num_t_blk * ((p.B + p.Bb - 1) / p.Bb) * p.num_n_blk;
  XVB_CHECK_ARG(tiles < (1ll << 31), "xvb_conv2d: too many tiles for one launch");
  p.num_tiles = (int)tiles;
  const int sms = sm_count();
  XVB_ENSURE_DYN_SMEM(conv2d_bf16x3_kernel<BLOCK_N>, Cfg::kSmemBytes);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(p.num_tiles < sms ? p.num_tiles : sms);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  XVB_CUDA(cudaLaunchKernelEx(&cfg, conv2d_bf16x3_kernel<BLOCK_N>, mx[0], mx[1], mw_hi, mw_lo, p));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

// Checks shared by xvb_conv2d, xvb_conv2d_taps and xvb_conv2d_valid (the window size and the tap list are checked by
// each), then the launch.  taps: strictly increasing kf * ksize + kt, in the packed weight's order.  pad: zero padding
// on each side (ksize / 2, or 0 for xvb_conv2d_valid); the output is (T + 2 pad - k) / s + 1 x (F + 2 pad - k) / s + 1.
int conv2d_run(const char* fn, const xvb_conv2d_args_t* a, const int* taps, int ntaps, int pad, void* stream) {
  XVB_CHECK_ARG(a->x_hi && a->x_lo && a->w_hi && a->w_lo, "%s: null operand pointer", fn);
  XVB_CHECK_ARG(a->B > 0 && a->T > 0 && a->F > 0 && a->Cin > 0 && a->Cout > 0,
                "%s: bad shape B=%d T=%d F=%d Cin=%d Cout=%d", fn, a->B, a->T, a->F, a->Cin, a->Cout);
  XVB_CHECK_ARG(a->Cin % 16 == 0 && a->Cout % 16 == 0, "%s: Cin=%d and Cout=%d must be multiples of 16", fn, a->Cin, a->Cout);
  XVB_CHECK_ARG((a->y_hi != nullptr) == (a->y_lo != nullptr) && (a->res_hi != nullptr) == (a->res_lo != nullptr) &&
                    (a->y2_hi != nullptr) == (a->y2_lo != nullptr),
                "%s: hi/lo plane pointers must both be set or both NULL", fn);
  XVB_CHECK_ARG(a->y_hi || a->y_f32 || a->y2_hi, "%s: no output requested", fn);
  XVB_CHECK_ARG((a->scale != nullptr) == (a->shift != nullptr), "%s: scale and shift must both be set or both NULL", fn);
  XVB_CHECK_ARG(!a->y2_hi || (a->scale2 && a->shift2), "%s: the second output needs scale2 and shift2", fn);
  XVB_CHECK_ARG(((uintptr_t)a->x_hi | (uintptr_t)a->x_lo | (uintptr_t)a->w_hi | (uintptr_t)a->w_lo | (uintptr_t)a->res_hi |
                 (uintptr_t)a->res_lo | (uintptr_t)a->y_hi | (uintptr_t)a->y_lo | (uintptr_t)a->y_f32 | (uintptr_t)a->y2_hi |
                 (uintptr_t)a->y2_lo) % 16 == 0,
                "%s: pointers must be 16-byte aligned", fn);
  int rc;
  Conv2dParams p{};
  p.B = a->B; p.T = a->T; p.F = a->F; p.Cin = a->Cin; p.Cout = a->Cout;
  XVB_CHECK_ARG(a->T + 2 * pad >= a->ksize && a->F + 2 * pad >= a->ksize, "%s: T=%d, F=%d shorter than the %dx%d window", fn,
                a->T, a->F, a->ksize, a->ksize);
  XVB_CHECK_ARG(a->stride_t >= 0 && a->stride_t <= 2, "%s: stride_t must be 0 (same as stride), 1 or 2 (got %d)", fn,
                a->stride_t);
  p.ks = a->ksize; p.stride = a->stride; p.stride_t = a->stride_t ? a->stride_t : a->stride; p.pad = pad;
  p.ntaps = ntaps;
  for (int j = 0; j < ntaps; ++j) {
    p.tap_f[j] = (int8_t)(taps[j] / a->ksize);
    p.tap_t[j] = (int8_t)(taps[j] % a->ksize);
  }
  p.To = (a->T + 2 * pad - a->ksize) / p.stride_t + 1;   // with pad = k / 2: ceil(T / s) for odd k
  p.Fo = (a->F + 2 * pad - a->ksize) / a->stride + 1;
  choose_conv_tile(p.B, p.To, p.Fo, p.stride, p.stride_t, &p.Fb, &p.Tb, &p.Bb);
  p.log2_fb = 0;
  while ((1 << p.log2_fb) < p.Fb) ++p.log2_fb;
  p.log2_tb = 0;
  while ((1 << p.log2_tb) < p.Tb) ++p.log2_tb;
  p.num_f_blk = (p.Fo + p.Fb - 1) / p.Fb;
  p.num_t_blk = (p.To + p.Tb - 1) / p.Tb;
  p.cin_p16 = p.Cin;
  p.num_cblk = (p.Cin + kBlockK - 1) / kBlockK;
  p.relu = a->relu ? 1 : 0;
  p.scale = a->scale; p.shift = a->shift;
  p.res_hi = reinterpret_cast<const __nv_bfloat16*>(a->res_hi);
  p.res_lo = reinterpret_cast<const __nv_bfloat16*>(a->res_lo);
  p.y_hi = reinterpret_cast<__nv_bfloat16*>(a->y_hi);
  p.y_lo = reinterpret_cast<__nv_bfloat16*>(a->y_lo);
  p.y_f32 = a->y_f32;
  p.scale2 = a->scale2; p.shift2 = a->shift2;
  p.y2_hi = reinterpret_cast<__nv_bfloat16*>(a->y2_hi);
  p.y2_lo = reinterpret_cast<__nv_bfloat16*>(a->y2_lo);
  p.lengths = a->lengths;

  // input (B, T, F, Cin) planes as a 4-D tensor map (C, F, T, B); box 64 channels x Fb x Tb x Bb output positions
  CUtensorMap mx[2];
  const cuuint64_t C = (cuuint64_t)p.Cin;
  const cuuint64_t dims[4] = {C, (cuuint64_t)p.F, (cuuint64_t)p.T, (cuuint64_t)p.B};
  const cuuint64_t strides[3] = {C * 2, C * 2 * p.F, C * 2 * p.F * p.T};
  const cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(p.Fb * p.stride), (cuuint32_t)(p.Tb * p.stride_t), (cuuint32_t)p.Bb};
  const cuuint32_t estr[4] = {1u, (cuuint32_t)p.stride, (cuuint32_t)p.stride_t, 1u};
  if ((rc = make_position_map(&mx[0], a->x_hi, dims, strides, box, estr))) return rc;
  if ((rc = make_position_map(&mx[1], a->x_lo, dims, strides, box, estr))) return rc;

  const long long m_tiles = (long long)p.num_f_blk * p.num_t_blk * ((p.B + p.Bb - 1) / p.Bb);
  const int sms = sm_count();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (p.Cout >= 128 && m_tiles * ((p.Cout + 127) / 128) >= sms) return launch_conv<128>(mx, p, a->w_hi, a->w_lo, s);
  if (p.Cout >= 64 && m_tiles * ((p.Cout + 63) / 64) >= sms / 2) return launch_conv<64>(mx, p, a->w_hi, a->w_lo, s);
  return launch_conv<32>(mx, p, a->w_hi, a->w_lo, s);
}

int conv2d_head_run(const char* fn, const float* x, const int* lengths, int B, int T, int F, const float* w, int Cout, int ksize,
                    const float* bn_scale, const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo, const float* scale2,
                    const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream) {
  XVB_CHECK_ARG(x && w && bn_scale && bn_shift && y_hi && y_lo, "%s: null pointer", fn);
  XVB_CHECK_ARG(B > 0 && T > 0 && F > 0 && Cout > 0 && Cout % 8 == 0, "%s: bad shape B=%d T=%d F=%d Cout=%d", fn, B, T, F, Cout);
  XVB_CHECK_ARG(ksize == 3 || ksize == 5, "%s: ksize must be 3 or 5 (got %d)", fn, ksize);
  XVB_CHECK_ARG((y2_hi != nullptr) == (y2_lo != nullptr) && (!y2_hi || (scale2 && shift2)),
                "%s: the second output needs both planes, scale2 and shift2", fn);
  XVB_CHECK_ARG(((uintptr_t)y_hi | (uintptr_t)y_lo | (uintptr_t)y2_hi | (uintptr_t)y2_lo) % 16 == 0,
                "%s: planes must be 16-byte aligned", fn);
  const long long total = (long long)B * T * F * (Cout / 8);
  auto kernel = ksize == 5 ? head_conv_kernel<5> : head_conv_kernel<3>;
  kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      x, lengths, B, T, F, w, Cout, bn_scale, bn_shift, reinterpret_cast<__nv_bfloat16*>(y_hi), reinterpret_cast<__nv_bfloat16*>(y_lo),
      scale2, shift2, reinterpret_cast<__nv_bfloat16*>(y2_hi), reinterpret_cast<__nv_bfloat16*>(y2_lo));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

}  // namespace
}  // namespace xvb

using namespace xvb;

extern "C" int xvb_conv2d(const xvb_conv2d_args_t* a, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(a, "xvb_conv2d: null args");
  XVB_CHECK_ARG((a->ksize == 3 || a->ksize == 1) && (a->stride == 1 || a->stride == 2),
                "xvb_conv2d: ksize must be 1 or 3 and stride 1 or 2 (got %d, %d)", a->ksize, a->stride);
  int dense[9];
  for (int j = 0; j < a->ksize * a->ksize; ++j) dense[j] = j;
  return conv2d_run("xvb_conv2d", a, dense, a->ksize * a->ksize, a->ksize / 2, stream);
}

extern "C" int xvb_conv2d_taps(const xvb_conv2d_args_t* a, const int* taps, int ntaps, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(a, "xvb_conv2d_taps: null args");
  XVB_CHECK_ARG((a->ksize == 1 || a->ksize == 3 || a->ksize == 5) && (a->stride == 1 || a->stride == 2),
                "xvb_conv2d_taps: ksize must be 1, 3 or 5 and stride 1 or 2 (got %d, %d)", a->ksize, a->stride);
  XVB_CHECK_ARG(taps, "xvb_conv2d_taps: null tap list");
  XVB_CHECK_ARG(ntaps >= 1 && ntaps <= a->ksize * a->ksize, "xvb_conv2d_taps: ntaps=%d outside [1, %d] for ksize %d", ntaps,
                a->ksize * a->ksize, a->ksize);
  for (int j = 0; j < ntaps; ++j) {
    XVB_CHECK_ARG(taps[j] >= 0 && taps[j] < a->ksize * a->ksize, "xvb_conv2d_taps: tap %d = %d outside [0, %d)", j, taps[j],
                  a->ksize * a->ksize);
    XVB_CHECK_ARG(j == 0 || taps[j] > taps[j - 1], "xvb_conv2d_taps: taps must be strictly increasing (tap %d = %d after %d)",
                  j, taps[j], taps[j - 1]);
  }
  return conv2d_run("xvb_conv2d_taps", a, taps, ntaps, a->ksize / 2, stream);
}

// No padding: every tap of every written output lies inside the input, and the outputs a padded conv would add at the
// far edges are neither computed into the output nor written (the epilogue clips at To x Fo).  The kernel is xvb_conv2d's.
extern "C" int xvb_conv2d_valid(const xvb_conv2d_args_t* a, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(a, "xvb_conv2d_valid: null args");
  XVB_CHECK_ARG(!a->lengths, "xvb_conv2d_valid: lengths are not supported (a masked batch needs the padded convs)");
  XVB_CHECK_ARG((a->ksize == 3 || a->ksize == 1) && (a->stride == 1 || a->stride == 2),
                "xvb_conv2d_valid: ksize must be 1 or 3 and stride 1 or 2 (got %d, %d)", a->ksize, a->stride);
  int dense[9];
  for (int j = 0; j < a->ksize * a->ksize; ++j) dense[j] = j;
  return conv2d_run("xvb_conv2d_valid", a, dense, a->ksize * a->ksize, 0, stream);
}

extern "C" int xvb_conv2d_head(const float* x, int B, int T, int F, const float* w, int Cout, const float* bn_scale,
                               const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo, const float* scale2,
                               const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  return conv2d_head_run("xvb_conv2d_head", x, nullptr, B, T, F, w, Cout, 3, bn_scale, bn_shift, y_hi, y_lo, scale2, shift2, y2_hi,
                         y2_lo, stream);
}

extern "C" int xvb_conv2d_head_k(const float* x, int B, int T, int F, const float* w, int Cout, int ksize,
                                 const float* bn_scale, const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo,
                                 const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  return conv2d_head_run("xvb_conv2d_head_k", x, nullptr, B, T, F, w, Cout, ksize, bn_scale, bn_shift, y_hi, y_lo, scale2, shift2,
                         y2_hi, y2_lo, stream);
}

namespace xvb {
namespace {

int se_residual_run(const char* fn, const uint16_t* z_hi, const uint16_t* z_lo, const float* gate, const uint16_t* id_hi,
                    const uint16_t* id_lo, int B, int64_t P, int C, const int* lengths, int F, int relu, uint16_t* y_hi,
                    uint16_t* y_lo, float* y_f32, const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo,
                    void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(z_hi && z_lo && gate && id_hi && id_lo, "%s: null pointer", fn);
  XVB_CHECK_ARG(B > 0 && P > 0 && C > 0 && C % 8 == 0, "%s: bad shape B=%d P=%lld C=%d", fn, B, (long long)P, C);
  XVB_CHECK_ARG((y_hi != nullptr) == (y_lo != nullptr) && (y2_hi != nullptr) == (y2_lo != nullptr) && (!y2_hi || (scale2 && shift2)),
                "%s: hi/lo planes must both be set or both NULL; the second output needs scale2 and shift2", fn);
  XVB_CHECK_ARG(y_hi || y_f32 || y2_hi, "%s: no output requested", fn);
  XVB_CHECK_ARG(((uintptr_t)z_hi | (uintptr_t)z_lo | (uintptr_t)gate | (uintptr_t)id_hi | (uintptr_t)id_lo | (uintptr_t)y_hi |
                 (uintptr_t)y_lo | (uintptr_t)y_f32 | (uintptr_t)y2_hi | (uintptr_t)y2_lo) % 16 == 0,
                "%s: pointers must be 16-byte aligned", fn);
  const long long total = (long long)B * P * (C / 8);
  se_residual_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(z_hi), reinterpret_cast<const __nv_bfloat16*>(z_lo), gate,
      reinterpret_cast<const __nv_bfloat16*>(id_hi), reinterpret_cast<const __nv_bfloat16*>(id_lo), (long long)P, C, lengths, F,
      relu ? 1 : 0, reinterpret_cast<__nv_bfloat16*>(y_hi), reinterpret_cast<__nv_bfloat16*>(y_lo), y_f32, scale2, shift2,
      reinterpret_cast<__nv_bfloat16*>(y2_hi), reinterpret_cast<__nv_bfloat16*>(y2_lo), total);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

}  // namespace
}  // namespace xvb

extern "C" int xvb_conv2d_head_lengths(const float* x, int B, int T, int F, const int* lengths, const float* w, int Cout,
                                       const float* bn_scale, const float* bn_shift, uint16_t* y_hi, uint16_t* y_lo,
                                       const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(lengths, "xvb_conv2d_head_lengths: null lengths");
  return conv2d_head_run("xvb_conv2d_head_lengths", x, lengths, B, T, F, w, Cout, 3, bn_scale, bn_shift, y_hi, y_lo, scale2,
                         shift2, y2_hi, y2_lo, stream);
}

extern "C" int xvb_se_residual(const uint16_t* z_hi, const uint16_t* z_lo, const float* gate, const uint16_t* id_hi,
                               const uint16_t* id_lo, int B, int64_t P, int C, int relu, uint16_t* y_hi, uint16_t* y_lo,
                               float* y_f32, const float* scale2, const float* shift2, uint16_t* y2_hi, uint16_t* y2_lo,
                               void* stream) {
  return se_residual_run("xvb_se_residual", z_hi, z_lo, gate, id_hi, id_lo, B, P, C, nullptr, 1, relu, y_hi, y_lo, y_f32,
                         scale2, shift2, y2_hi, y2_lo, stream);
}

extern "C" int xvb_se_residual_lengths(const uint16_t* z_hi, const uint16_t* z_lo, const float* gate, const uint16_t* id_hi,
                                       const uint16_t* id_lo, int B, int T, int F, int C, const int* lengths, int relu,
                                       uint16_t* y_hi, uint16_t* y_lo, float* y_f32, const float* scale2, const float* shift2,
                                       uint16_t* y2_hi, uint16_t* y2_lo, void* stream) {
  XVB_CHECK_ARG(lengths && T > 0 && F > 0, "xvb_se_residual_lengths: null lengths or bad shape T=%d F=%d", T, F);
  return se_residual_run("xvb_se_residual_lengths", z_hi, z_lo, gate, id_hi, id_lo, B, (int64_t)T * F, C, lengths, F, relu,
                         y_hi, y_lo, y_f32, scale2, shift2, y2_hi, y2_lo, stream);
}
