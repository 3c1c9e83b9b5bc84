// CAM++ x-vector pieces that are not contractions (subtools2/egrecho/models/campplus/campplus.py):
//   * bn_relu_planes : relu(x * scale[c] + shift[c]) over split planes -- the BN1 -> ReLU pre-activation of every dense
//                      layer (CAMDenseTDNNLayer.nonlinear1, :199, :212-213) and transit layer (TransitLayer.nonlinear,
//                      :265-270), which cannot fold into the following 1x1 conv because the ReLU sits between them;
//   * cam_gate       : CAMLayer's context-aware mask (:157-178) up to the sigmoid: the per-segment context
//                      mean_T(h) + seg_avg(h), then linear1 + ReLU and linear2 + sigmoid in fp32 on CUDA cores, one CTA per
//                      utterance.  The mask is constant over each seg_len-frame segment, so it is stored per segment and
//                      applied by xvb_seg_gate_apply (ecapa.cu), outside the layer kernel.  A masked batch (lengths) gives
//                      each utterance the context of its own frames and zero gate rows past its last segment.
// The contractions (linear1, linear_local, the transits, tdnn and dense) run on the wgmma layer kernel / xvb_small_affine.
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"

namespace xvb {
namespace {

__global__ void bn_relu_planes_kernel(const __nv_bfloat16* __restrict__ xh, const __nv_bfloat16* __restrict__ xl, long long ldx,
                                      const float* __restrict__ scale, const float* __restrict__ shift,
                                      __nv_bfloat16* __restrict__ yh, __nv_bfloat16* __restrict__ yl, long long ldy,
                                      long long rows, int C) {
  const int groups = C / 8;
  const long long total = rows * groups;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / groups;
    const int c = (int)(i % groups) * 8;
    float v[8];
    unpack8(*reinterpret_cast<const uint4*>(xh + r * ldx + c), *reinterpret_cast<const uint4*>(xl + r * ldx + c), v);
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(scale + c)), s1 = __ldg(reinterpret_cast<const float4*>(scale + c + 4));
    const float4 t0 = __ldg(reinterpret_cast<const float4*>(shift + c)), t1 = __ldg(reinterpret_cast<const float4*>(shift + c + 4));
    const float s[8] = {s0.x, s0.y, s0.z, s0.w, s1.x, s1.y, s1.z, s1.w};
    const float t[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaxf(fmaf(v[k], s[k], t[k]), 0.f);
    uint4 h, l;
    pack8(v, h, l);
    *reinterpret_cast<uint4*>(yh + r * ldy + c) = h;
    *reinterpret_cast<uint4*>(yl + r * ldy + c) = l;
  }
}

constexpr int kGateThreads = 256;

// One CTA per utterance.  Shared memory: ctx (nseg, C) segment sums -> contexts, hid (nseg, R), partial (rows, C).
// Threads own 8 channels x one frame lane: C / 8 channel groups, kGateThreads / (C / 8) frame lanes.  lengths (NULL: every
// utterance has T frames): utterance b reduces its own L frames exactly as an unmasked call at T = L does, and writes
// zero gate rows for the segments past its last one; T is then only the batch stride and the gate's segment count.
__global__ void __launch_bounds__(kGateThreads)
cam_gate_kernel(const __nv_bfloat16* __restrict__ hh, const __nv_bfloat16* __restrict__ hl, long long ldh, int T, int C,
                int seg_len, const float* __restrict__ w1, const float* __restrict__ b1, int R, const float* __restrict__ w2,
                const float* __restrict__ b2, int G, const int* __restrict__ lengths, float* __restrict__ gate) {
  extern __shared__ float sm[];
  const int b = blockIdx.x;
  const int L = lengths ? __ldg(lengths + b) : T;
  const int nseg_all = (T + seg_len - 1) / seg_len;   // gate rows per utterance
  const int nseg = (L + seg_len - 1) / seg_len;       // this utterance's segments
  const int groups = C / 8;
  const int lanes = kGateThreads / groups;
  float* ctx = sm;                           // nseg * C
  float* hid = ctx + (size_t)nseg * C;       // nseg * R
  float* part = hid + (size_t)nseg * R;      // lanes * C
  const int cg = threadIdx.x % groups, lane = threadIdx.x / groups;
  const bool active = lane < lanes;
  const long long base = (long long)b * T * ldh + cg * 8;
  // 1. segment sums: every lane adds its frames of the segment, then the lanes are reduced in a fixed order
  for (int s = 0; s < nseg; ++s) {
    const int t1 = min(L, (s + 1) * seg_len);
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    if (active) {
      for (int t = s * seg_len + lane; t < t1; t += lanes) {
        float v[8];
        unpack8(*reinterpret_cast<const uint4*>(hh + base + (long long)t * ldh),
                *reinterpret_cast<const uint4*>(hl + base + (long long)t * ldh), v);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += v[k];
      }
#pragma unroll
      for (int k = 0; k < 8; ++k) part[lane * C + cg * 8 + k] = acc[k];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kGateThreads) {
      float sum = 0.f;
      for (int l = 0; l < lanes; ++l) sum += part[l * C + c];
      ctx[s * C + c] = sum;
    }
    __syncthreads();
  }
  // 2. context = mean over all L frames + mean over the segment's valid frames (avg_pool1d ceil_mode: the last segment
  //    divides by its own length)
  for (int c = threadIdx.x; c < C; c += kGateThreads) {
    float total = 0.f;
    for (int s = 0; s < nseg; ++s) total += ctx[s * C + c];
    const float mean = total / (float)L;
    for (int s = 0; s < nseg; ++s) {
      const int n = min(L, (s + 1) * seg_len) - s * seg_len;
      ctx[s * C + c] = mean + ctx[s * C + c] / (float)n;
    }
  }
  __syncthreads();
  // 3. hid = relu(W1 ctx + b1), (nseg, R)
  for (int i = threadIdx.x; i < nseg * R; i += kGateThreads) {
    const int s = i / R, r = i % R;
    const float* w = w1 + (size_t)r * C;
    const float* x = ctx + (size_t)s * C;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(__ldg(w + c), x[c], acc);
    hid[i] = fmaxf(acc + __ldg(b1 + r), 0.f);
  }
  __syncthreads();
  // 4. gate = sigmoid(W2 hid + b2), (nseg, G); rows past the utterance's segments are zeros, which the gate's
  //    consumer multiplies by the zero frames there
  for (int i = threadIdx.x; i < nseg * G; i += kGateThreads) {
    const int s = i / G, g = i % G;
    const float* w = w2 + (size_t)g * R;
    const float* x = hid + (size_t)s * R;
    float acc = 0.f;
    for (int r = 0; r < R; ++r) acc = fmaf(__ldg(w + r), x[r], acc);
    gate[((size_t)b * nseg_all + s) * G + g] = 1.f / (1.f + expf(-(acc + __ldg(b2 + g))));
  }
  for (int i = nseg * G + threadIdx.x; i < nseg_all * G; i += kGateThreads) gate[(size_t)b * nseg_all * G + i] = 0.f;
}

size_t cam_gate_smem(int T, int C, int seg_len, int R) {
  const size_t nseg = (size_t)(T + seg_len - 1) / seg_len;
  return (nseg * C + nseg * R + (size_t)(kGateThreads / (C / 8)) * C) * sizeof(float);
}

}  // namespace
}  // namespace xvb

using namespace xvb;

extern "C" int xvb_bn_relu_planes(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, int64_t rows, int C,
                                  const float* scale, const float* shift, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy,
                                  void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(x_hi && x_lo && scale && shift && y_hi && y_lo, "xvb_bn_relu_planes: null pointer");
  XVB_CHECK_ARG(rows > 0 && C > 0 && C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
                "xvb_bn_relu_planes: need C %% 8 == 0 and pitches >= C, multiples of 8 (C=%d ldx=%lld ldy=%lld)", C,
                (long long)ldx, (long long)ldy);
  XVB_CHECK_ARG(((uintptr_t)x_hi | (uintptr_t)x_lo | (uintptr_t)scale | (uintptr_t)shift | (uintptr_t)y_hi | (uintptr_t)y_lo) % 16 == 0,
                "xvb_bn_relu_planes: pointers must be 16-byte aligned");
  const long long total = rows * (C / 8);
  long long g = (total + 255) / 256;
  const long long cap = (long long)sm_count() * 32;
  if (g > cap) g = cap;
  bn_relu_planes_kernel<<<(unsigned)g, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const __nv_bfloat16*>(x_hi), reinterpret_cast<const __nv_bfloat16*>(x_lo), ldx, scale, shift,
      reinterpret_cast<__nv_bfloat16*>(y_hi), reinterpret_cast<__nv_bfloat16*>(y_lo), ldy, rows, C);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

static int cam_gate(const char* fn, const uint16_t* h_hi, const uint16_t* h_lo, int64_t ldh, int B, int T, int C, int seg_len,
                    const float* w1, const float* b1, int R, const float* w2, const float* b2, int G, const int* lengths,
                    float* gate, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(h_hi && h_lo && w1 && b1 && w2 && b2 && gate, "%s: null pointer", fn);
  XVB_CHECK_ARG(B > 0 && T > 0 && seg_len > 0 && R > 0 && G > 0 && C > 0 && C % 8 == 0 && C / 8 <= kGateThreads && ldh % 8 == 0 &&
                    ldh >= C,
                "%s: need C %% 8 == 0, 8 <= C <= %d, ldh %% 8 == 0 (C=%d ldh=%lld)", fn, 8 * kGateThreads, C, (long long)ldh);
  XVB_CHECK_ARG(((uintptr_t)h_hi | (uintptr_t)h_lo) % 16 == 0, "%s: planes must be 16-byte aligned", fn);
  const size_t smem = cam_gate_smem(T, C, seg_len, R);
  XVB_CHECK_ARG(smem <= 227 * 1024, "%s: %d segments of %d channels exceed the shared memory of one CTA", fn,
                (T + seg_len - 1) / seg_len, C);
  if (smem > 48 * 1024) XVB_ENSURE_DYN_SMEM(cam_gate_kernel, 227 * 1024);
  cam_gate_kernel<<<B, kGateThreads, smem, (cudaStream_t)stream>>>(reinterpret_cast<const __nv_bfloat16*>(h_hi),
                                                                   reinterpret_cast<const __nv_bfloat16*>(h_lo), ldh, T, C,
                                                                   seg_len, w1, b1, R, w2, b2, G, lengths, gate);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int xvb_cam_gate(const uint16_t* h_hi, const uint16_t* h_lo, int64_t ldh, int B, int T, int C, int seg_len,
                            const float* w1, const float* b1, int R, const float* w2, const float* b2, int G, float* gate,
                            void* stream) {
  return cam_gate("xvb_cam_gate", h_hi, h_lo, ldh, B, T, C, seg_len, w1, b1, R, w2, b2, G, nullptr, gate, stream);
}

extern "C" int xvb_cam_gate_lengths(const uint16_t* h_hi, const uint16_t* h_lo, int64_t ldh, int B, int T, int C, int seg_len,
                                    const float* w1, const float* b1, int R, const float* w2, const float* b2, int G,
                                    const int* lengths, float* gate, void* stream) {
  XVB_CHECK_ARG(lengths, "xvb_cam_gate_lengths: null lengths");
  return cam_gate("xvb_cam_gate_lengths", h_hi, h_lo, ldh, B, T, C, seg_len, w1, b1, R, w2, b2, G, lengths, gate, stream);
}
