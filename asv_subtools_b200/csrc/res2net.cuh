// The Res2Net chain kernel of res2net.cu, templated on the Res2Net width kW.  Each width is instantiated in a
// translation unit of its own -- width 128 in res2net.cu, width 64 in res2net_w64.cu -- so that every object file
// holds one instance of the kernel and its SASS can be checked on its own.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "common.cuh"
#include "ptx.cuh"

namespace xvb {

// The kernel is templated on the Res2Net width kW (channels per chunk = tile N): 128 for ECAPA C1024, 64 for C512.
// The A tile is always 128 frames x 64 channels; a tap of one source is kW / 64 such channel boxes.
constexpr int kRABytes = 128 * 64 * 2;             // one plane of a 128-row x 64-channel A tile
constexpr int kRConsumers = 256;                   // two warpgroups, 64 frames each
constexpr int kRThreads = kRConsumers + 32;        // + the TMA producer warp

template <int kW>
struct Res2Cfg;
template <>
struct Res2Cfg<128> {
  static constexpr int kStages = 3, kCtas = 1;     // 3 x 64 KB stages, one CTA per SM
};
template <>
struct Res2Cfg<64> {
  static constexpr int kStages = 4, kCtas = 1;     // 4 x 48 KB stages: measured ahead of 3 x 1 and 2 x 2 (DESIGN section 4)
};

template <int kW>
struct Res2Tile {
  static constexpr int kStages = Res2Cfg<kW>::kStages;
  static constexpr int kBBytes = kW * 64 * 2;                        // one plane of the kW x 64 weight tile
  static constexpr int kStageBytes = 2 * kRABytes + 2 * kBBytes;     // 64 KB at width 128, 48 KB at 64
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + 256;
  static constexpr int kBoxes = kW / 64;                             // 64-channel boxes per tap
  static constexpr int kVec = kW / 8;                                // 16-byte vectors per chunk row
  static constexpr int kVecShift = kW == 128 ? 4 : 3;
  static_assert(kW == 64 || kW == 128, "Res2Net chain: width 64 or 128");
  static_assert(kVec == 1 << kVecShift, "kVecShift");
};

struct Res2Params {
  int B, T, C;            // C = scale * width channels of the block input / output
  int num_steps;          // scale - 1 (= 7)
  int dilation;
  int num_m;              // ceil(T / 128)
  const float* bias;      // [num_steps][width]
  const float* scale;
  const float* shift;
  const __nv_bfloat16* x_hi;   // block input planes (B,T,ldx): chunk 0 is passed through
  const __nv_bfloat16* x_lo;
  __nv_bfloat16* y_hi;         // block output planes (B,T,ldy)
  __nv_bfloat16* y_lo;
  long long ldx, ldy;
};

template <int kW>
__global__ void __launch_bounds__(kRThreads, Res2Cfg<kW>::kCtas)
res2net_chain_kernel(const __grid_constant__ CUtensorMap map_x_hi, const __grid_constant__ CUtensorMap map_x_lo,
                     const __grid_constant__ CUtensorMap map_yin_hi, const __grid_constant__ CUtensorMap map_yin_lo,
                     const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                     const __grid_constant__ Res2Params p) {
  using Tile = Res2Tile<kW>;
  constexpr int kRStages = Tile::kStages, kRStageBytes = Tile::kStageBytes, kRBBytes = Tile::kBBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kRStages * kRStageBytes);
  uint64_t* empty_bar = full_bar + kRStages;
  uint64_t* step_bar = empty_bar + kRStages;      // completes once per step: that step's outputs are in global memory

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int producer_warp = kRConsumers / 32;
  if (warp == producer_warp && lane == 0) {
    tma_prefetch_desc(&map_x_hi); tma_prefetch_desc(&map_x_lo);
    tma_prefetch_desc(&map_yin_hi); tma_prefetch_desc(&map_yin_lo);
    tma_prefetch_desc(&map_w_hi); tma_prefetch_desc(&map_w_lo);
    for (int i = 0; i < kRStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kRConsumers / 32); }
    mbar_init(step_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int d = p.dilation;

  if (warp == producer_warp) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0, steps_done = 0;   // number of completed step_bar phases this thread has consumed
      for (int b = blockIdx.x; b < p.B; b += gridDim.x) {
        for (int st = 0; st < p.num_steps; ++st) {
          for (int m = 0; m < p.num_m; ++m) {
            const int t0 = m * 128;
            for (int src = 0; src < (st == 0 ? 1 : 2); ++src) {
              if (src == 1 && m == 0) {
                // outputs of step st-1 (all tiles of this utterance) must have landed before we read them back
                mbar_wait(step_bar, steps_done & 1);
                ++steps_done;
                asm volatile("fence.proxy.async;" ::: "memory");
              }
              const CUtensorMap* mh = src == 0 ? &map_x_hi : &map_yin_hi;
              const CUtensorMap* ml = src == 0 ? &map_x_lo : &map_yin_lo;
              const int cbase = src == 0 ? (st + 1) * kW : st * kW;   // chunk st+1 of x, chunk st of y
              for (int tap = 0; tap < 3; ++tap) {
                const int tt = t0 + (tap - 1) * d;
                for (int cb = 0; cb < Tile::kBoxes; ++cb) {
                  mbar_wait(&empty_bar[stage], phase ^ 1);
                  uint8_t* s = smem + stage * kRStageBytes;
                  mbar_expect_tx(&full_bar[stage], kRStageBytes);
                  tma_load_3d(s, mh, &full_bar[stage], cbase + cb * 64, tt, b);
                  tma_load_3d(s + kRABytes, ml, &full_bar[stage], cbase + cb * 64, tt, b);
                  const int kw = tap * kW + cb * 64;
                  tma_load_2d(s + 2 * kRABytes, &map_w_hi, &full_bar[stage], kw, st * kW);
                  tma_load_2d(s + 2 * kRABytes + kRBBytes, &map_w_lo, &full_bar[stage], kw, st * kW);
                  if (++stage == kRStages) { stage = 0; phase ^= 1; }
                }
              }
            }
          }
        }
        // the consumers also release the last step of an utterance; consume that phase too so the parity
        // bookkeeping stays in step
        mbar_wait(step_bar, steps_done & 1);
        ++steps_done;
      }
    }
    return;
  }

  // ================================ consumers: wgmma + epilogue ================================
  const int wg = warp >> 2, q4 = lane & 3;
  const int row0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // this thread's frames: t0 + row0 and t0 + row0 + 8
  const int etid = threadIdx.x;
  float acc[kW / 2];
#pragma unroll
  for (int i = 0; i < kW / 2; ++i) acc[i] = 0.f;
  int stage = 0;
  uint32_t phase = 0;
  for (int b = blockIdx.x; b < p.B; b += gridDim.x) {
    // chunk 0 passes through (ecapa_tdnn_xvector.py:63-64): 16-byte vectors, kW / 8 per row and plane
    for (int i = etid; i < p.T * Tile::kVec * 2; i += kRConsumers) {
      const int plane = i / (p.T * Tile::kVec), r = (i % (p.T * Tile::kVec)) >> Tile::kVecShift, v = i & (Tile::kVec - 1);
      const __nv_bfloat16* src = (plane ? p.x_lo : p.x_hi) + ((long long)b * p.T + r) * p.ldx + v * 8;
      __nv_bfloat16* dst = (plane ? p.y_lo : p.y_hi) + ((long long)b * p.T + r) * p.ldy + v * 8;
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
    }
    for (int st = 0; st < p.num_steps; ++st) {
      const int nkb = (st == 0 ? 1 : 2) * 3 * Tile::kBoxes;
      for (int m = 0; m < p.num_m; ++m) {
        int prev_stage = -1;
        for (int kb = 0; kb < nkb; ++kb) {
          mbar_wait(&full_bar[stage], phase);
          const uint32_t sa = smem_u32(smem + stage * kRStageBytes);
          const uint64_t m_off = (uint64_t)((wg * 64 * 128) >> 4);
          const uint64_t da_hi = make_sw128_desc(sa) + m_off, da_lo = make_sw128_desc(sa + kRABytes) + m_off;
          const uint64_t db_hi = make_sw128_desc(sa + 2 * kRABytes);
          const uint64_t db_lo = make_sw128_desc(sa + 2 * kRABytes + kRBBytes);
          wgmma_fence();
#pragma unroll
          for (int s = 0; s < 4; ++s) {
            const uint64_t koff = (uint64_t)(s * 32 >> 4);
            wgmma_bf16<kW>(acc, da_lo + koff, db_hi + koff, (kb | s) ? 1u : 0u);
            wgmma_bf16<kW>(acc, da_hi + koff, db_lo + koff, 1);
            wgmma_bf16<kW>(acc, da_hi + koff, db_hi + koff, 1);
          }
          wgmma_commit();
          wgmma_wait<1>();
          if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == kRStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_operands(acc);
        if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        // epilogue: +bias -> ReLU -> BN -> split -> output chunk st+1
        const int t0 = m * 128;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int t = t0 + row0 + 8 * h;
          if (t >= p.T) continue;
          __nv_bfloat16* yh = p.y_hi + ((long long)b * p.T + t) * p.ldy + (st + 1) * kW;
          __nv_bfloat16* yl = p.y_lo + ((long long)b * p.T + t) * p.ldy + (st + 1) * kW;
#pragma unroll
          for (int i = 0; i < kW / 8; ++i) {
            const int c = 8 * i + 2 * q4;
            const int pc = st * kW + c;
            const float f0 = fmaf(fmaxf(acc[4 * i + 2 * h] + __ldg(p.bias + pc), 0.f), __ldg(p.scale + pc), __ldg(p.shift + pc));
            const float f1 = fmaf(fmaxf(acc[4 * i + 2 * h + 1] + __ldg(p.bias + pc + 1), 0.f), __ldg(p.scale + pc + 1),
                                  __ldg(p.shift + pc + 1));
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(f0, h0, l0);
            split_bf16(f1, h1, l1);
            *reinterpret_cast<uint32_t*>(yh + c) = pack_bf16x2(h0, h1);
            *reinterpret_cast<uint32_t*>(yl + c) = pack_bf16x2(l0, l1);
          }
        }
      }
      // step finished: make this step's stores visible to the producer's TMA reads, then release it
      __threadfence_block();
      asm volatile("fence.proxy.async;" ::: "memory");
      asm volatile("bar.sync 1, 256;" ::: "memory");
      if (etid == 0) mbar_arrive(step_bar);
    }
  }
}


template <int kW>
int launch_chain(const Res2Params& p, const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi,
                        const uint16_t* w_lo, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, int scale, cudaStream_t stream) {
  using Tile = Res2Tile<kW>;
  const int B = p.B, T = p.T, C = p.C;
  int rc;
  CUtensorMap mx_hi, mx_lo, myi_hi, myi_lo, mw_hi, mw_lo;
  const unsigned long long dx[3] = {(unsigned long long)C, (unsigned long long)T, (unsigned long long)B};
  const unsigned long long sx[2] = {(unsigned long long)ldx * 2, (unsigned long long)ldx * 2 * T};
  const unsigned long long sy[2] = {(unsigned long long)ldy * 2, (unsigned long long)ldy * 2 * T};
  const unsigned box_a[3] = {64u, 128u, 1u};
  if ((rc = make_tensor_map(&mx_hi, x_hi, 2, 3, dx, sx, box_a, 128))) return rc;
  if ((rc = make_tensor_map(&mx_lo, x_lo, 2, 3, dx, sx, box_a, 128))) return rc;
  if ((rc = make_tensor_map(&myi_hi, y_hi, 2, 3, dx, sy, box_a, 128))) return rc;
  if ((rc = make_tensor_map(&myi_lo, y_lo, 2, 3, dx, sy, box_a, 128))) return rc;
  const unsigned long long dw[2] = {(unsigned long long)3 * kW, (unsigned long long)(scale - 1) * kW};
  const unsigned long long sw[1] = {(unsigned long long)3 * kW * 2};
  const unsigned box_w[2] = {64u, (unsigned)kW};
  if ((rc = make_tensor_map(&mw_hi, w_hi, 2, 2, dw, sw, box_w, 128))) return rc;
  if ((rc = make_tensor_map(&mw_lo, w_lo, 2, 2, dw, sw, box_w, 128))) return rc;
  XVB_ENSURE_DYN_SMEM((res2net_chain_kernel<kW>), Tile::kSmemBytes);
  // a CTA owns utterances b = blockIdx.x, blockIdx.x + grid, ...: one round is every CTA slot of the machine
  const int slots = sm_count() * Res2Cfg<kW>::kCtas;
  const int grid = B < slots ? B : slots;
  res2net_chain_kernel<kW><<<grid, kRThreads, Tile::kSmemBytes, stream>>>(mx_hi, mx_lo, myi_hi, myi_lo, mw_hi, mw_lo, p);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

// explicitly instantiated in res2net.cu (128) and res2net_w64.cu (64)
extern template int launch_chain<128>(const Res2Params&, const uint16_t*, const uint16_t*, int64_t, const uint16_t*,
                                      const uint16_t*, uint16_t*, uint16_t*, int64_t, int, cudaStream_t);
extern template int launch_chain<64>(const Res2Params&, const uint16_t*, const uint16_t*, int64_t, const uint16_t*,
                                     const uint16_t*, uint16_t*, uint16_t*, int64_t, int, cudaStream_t);

}  // namespace xvb
