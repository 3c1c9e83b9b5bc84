// TDNN affine layer as a warpgroup-MMA GEMM (sm_90a).
//
//   y[b,t,n] = epi( bias[n] + sum_{tap} sum_{c} W[n, tap, c] * x[b, t + ctx[tap], c] )
//
// Restates TdnnAffine.forward + ReLU + eval-BatchNorm of the reference
// (pytorch/libs/nnet/components.py:107-149, :410-431) as ONE kernel:
//   * M = B*T frames, N = Cout, K = ntaps*Cin -- only the taps in `context` (the reference's
//     conv1d also multiplies the masked taps, components.py:133-138);
//   * the context splice is never materialised: the A tile of tap `c` is fetched by TMA from the
//     (C, T, B) frame matrix at time coordinate t0 + c; TMA's out-of-bounds zero fill *is*
//     F.pad(..., value=0) (components.py:117) and can never cross an utterance boundary;
//   * fp32-grade accuracy at bf16 tensor rate: operands are bf16 "split planes" (hi, lo) and each
//     K step issues hi*hi + lo*hi + hi*lo into the same fp32 accumulator;
//   * warp-specialised persistent CTAs: one producer warp drives TMA through an mbarrier ring of
//     operand stages, two consumer warpgroups issue wgmma with the accumulators in registers and run
//     the epilogue (+bias -> ReLU -> BN -> split -> shared memory -> TMA store for plane-only layers, st.global
//     otherwise) while the producer already loads the next tile's operands.  The 128-wide layer and fused-pooling instances run the two warpgroups
//     ping-pong: each one owns every other tile of the CTA whole (128 accumulator rows), so one
//     warpgroup's epilogue runs under the other's MMAs.  The other instances split each tile
//     between the two warpgroups (64 accumulator rows each).
// Variants of the same kernel (template flags): kPool -- swapped operands, the epilogue pools over time
// instead of storing (fused statistics pooling); kHist -- the epilogue bins scores into a trial histogram
// (scoring.cu); runtime: a second A source (W.(a+b)), split-K slices for the segment layers, an im2col
// view of the first layer (x_batch_stride).
//
// An M tile is 128 rows = Bb utterances x Tb consecutive frames (Tb*Bb = 128, chosen on the host
// to minimise padding: T=200 -> Tb=8, Bb=16 has none).
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <stdlib.h>

#include <mutex>

#include "common.cuh"
#include "ptx.cuh"

namespace xvb {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                      // bf16 elements = one 128-byte swizzle row
constexpr int kABytes = kBlockM * kBlockK * 2;   // 16 KB per plane per stage
constexpr int kNumConsumers = 256;               // two consumer warpgroups
constexpr int kProducerWarp = kNumConsumers / 32;
constexpr int kSlabBytes = 16384;                // trial histogram: 2 x hist_bins u32 counters
// Staged layer epilogue (outputs leave through shared memory and TMA stores): each consumer warpgroup owns one piece of
// 64 rows x 64 channels x both planes, swizzled like the operand tiles, and the bias, scale and shift of its 64 columns.
// The two ping-pong warpgroups can be in their epilogues at once, so they share nothing.  The fused pooling epilogue
// stages a tile's partials in the same 16 KB per warpgroup.  The histogram's slab is the first 16 KB of the region: no
// instance has both.
constexpr int kStagePlaneBytes = 64 * kBlockK * 2;
constexpr int kStageOutBytes = 2 * kStagePlaneBytes;
constexpr int kCoefBytes = 3 * kBlockK * 4;
constexpr int kEpiBytes = 2 * (kStageOutBytes + kCoefBytes);
static_assert(kEpiBytes >= kSlabBytes, "the histogram slab lives in the epilogue region");

// The instances whose two consumer warpgroups run ping-pong (see the kernel).  Each of their consumer threads holds a
// whole 128 x 128 tile's share of accumulators (128 registers), more than fits in the 168 registers a thread of a
// 288-thread CTA may use.  So they run a whole producer warpgroup (384 threads) that gives its registers to the consumers
// with setmaxnreg: 40 for the producer, 232 for each consumer, 64512 in all as at launch (168 x 384).
template <int BLOCK_N, bool kHist, bool kSwish>
__host__ __device__ constexpr bool ping_pong() { return BLOCK_N == 128 && !kHist && !kSwish; }
template <int BLOCK_N, bool kHist, bool kSwish>
__host__ __device__ constexpr int gemm_threads() { return kNumConsumers + (ping_pong<BLOCK_N, kHist, kSwish>() ? 128 : 32); }
constexpr uint32_t kProducerRegs = 40, kConsumerRegs = 232;

struct TdnnGemmParams {
  int B, T, Cin, Cout;
  int Tb, Bb, num_t_blk, num_b_blk, num_n_blk, num_tiles;
  int ntaps, cin_p16, num_cblk;
  int ctx[XVB_MAX_TAPS];
  int flags;
  const float* bias;
  const float* scale;
  const float* shift;
  const float* row_bias;  // per-frame additive term (PLDA row term), may be NULL
  const float* utt_bias;  // per-utterance x column additive term (B, ld_utt), may be NULL
  long long ld_utt;
  int log2_tb;            // Tb is a power of two
  float* pool_partial;    // fused statistics pooling: per (time block, utterance, channel) [mean | M2] partials
  int num_src;            // 1, or 2: a second A source accumulated with the same weights (W.(x + x2))
  // M-unit sharding (a unit = one 128-row block; two for the trial histogram, whose callers count in
  // 256-row units): this launch walks units unit_first + k * unit_stride
  int unit_first, unit_stride;
  // fused trial histogram (scoring.cu: xvb_trial_histogram): the scores never leave the SM
  unsigned long long* hist;   // (2, hist_bins) u64 counters [nontarget | target], accumulated; NULL = off
  const int* row_label;       // speaker id per row / per column
  const int* col_label;
  float hist_lo, hist_inv_w;  // bin = 1 + floor((s - lo) * inv_w); bin 0: s < lo; bin nbins-1: at or above hi
  int hist_bins;
  int hist_sym;               // count only column index > row index (all pairs of one set, each once)
  int hist_group, num_units;  // tile raster of the score-matrix mode (decode_tile)
  // split-K for the segment-level layers (M = B rows, K in the thousands: too few tiles to fill the
  // machine otherwise): slice s of a tile covers channel blocks [s*kb_per_slice, (s+1)*kb_per_slice)
  // and stores its fp32 partial at "time" s of a (B, k_slices, Cout) buffer; segment_reduce_kernel sums
  // the slices in order (deterministic) and applies the epilogue.  ntaps == 1, one source only.
  int k_slices, kb_per_slice;
  // grouped convolution (groups > 1): N block n0 belongs to group n0 / group_ng and streams only that group's
  // group_kg input channels, starting at frame channel (n0 / group_ng) * group_kg; 0 = dense
  int group_ng, group_kg;
  int out_T;              // time extent of the fp32 output (k_slices for split-K partials, else T)
  // masked batch of utterances of different lengths: utterance b owns frames [0, lengths[b]); the layer epilogue stores
  // zeros for the frames past it (what the next layer's taps must read, F.pad).  NULL: every utterance is T frames long.
  const int* lengths;
  // the layer epilogue stages its output tiles in shared memory and stores them with TMA (map_y_hi / map_y_lo): planes
  // only, no fp32 output, split-K, row or utterance term
  int tma_store;
#ifdef XVB_TILE_TIMELINE
  unsigned long long* timeline;   // per CTA: kTimelineHead words, then kTimelineRec per tile of its list
  int timeline_tiles;             // tiles per CTA the buffer has room for
  int timeline_general;           // keep the fused pooling epilogue on its general path
#endif
  __nv_bfloat16* y_hi;
  __nv_bfloat16* y_lo;
  long long ldy;
  float* y_f32;
  long long ldyf;
};

// The instances with the staged layer epilogue: it moves 64-channel boxes, so the 32-wide ones keep the direct stores.
template <int BLOCK_N, bool kPool, bool kHist>
__host__ __device__ constexpr bool staged_epilogue() { return !kPool && !kHist && BLOCK_N % kBlockK == 0; }

// One CTA per 128 x BLOCK_N tile; operand stages as deep as 192 KB of shared memory allows.  Behind them the staged
// layer and fused pooling instances have the epilogue region; the others keep the 16 KB slab alone, and with it the
// shared memory they leave to a kernel of another stream.
template <int BLOCK_N, bool kPool, bool kHist>
struct GemmCfg {
  static constexpr int kTailBytes = (staged_epilogue<BLOCK_N, kPool, kHist>() || kPool) ? kEpiBytes : kSlabBytes;
  static constexpr int kBBytes = BLOCK_N * kBlockK * 2;          // one plane of the weight tile
  static constexpr int kStageBytes = 2 * kABytes + 2 * kBBytes;
  static constexpr int kStages = (192 * 1024) / kStageBytes > 6 ? 6 : (192 * 1024) / kStageBytes;
  static constexpr int kAccRegs = BLOCK_N / 2;                   // per consumer thread
  static constexpr int kSmemBytes = kStages * kStageBytes + kTailBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 232448, "exceeds the 227 KB shared memory of an sm_90 CTA");
  static_assert(kStages >= 2, "need at least a double-buffered operand pipeline");
};

// kPool: fused statistics pooling.  The MMA operands swap roles -- the weight tile is the M side
// (128 output channels = accumulator rows), the frame tile the N side (128 frames = accumulator
// columns) -- so pooling over time becomes a reduction along a thread's own columns plus at most
// two quad shuffles, with no (B,T,C) output at all.
// Tile index -> (M unit, N block).  Layers: N fastest, so the CTAs running together share the frame
// (A) tile and walk the small, L2-resident weight matrix.  Score matrices (kHist): both operands are
// huge, so tiles are rastered in bands of `hist_group` M units x all N blocks, M fastest -- the CTAs in
// flight cover hist_group rows x a few columns and each test (B) tile leaves HBM once per band
// instead of once per M unit.  Returns false for tiles that do not exist / lie below the diagonal.
template <bool kHist>
__device__ __forceinline__ bool decode_tile(const TdnnGemmParams& p, int tile, int& m_unit, int& n_blk, int& slice) {
  slice = 0;
  if constexpr (!kHist) {
    if (p.k_slices > 1) { slice = tile % p.k_slices; tile /= p.k_slices; }
    m_unit = p.unit_first + (tile / p.num_n_blk) * p.unit_stride;
    n_blk = tile % p.num_n_blk;
    return true;
  } else {
    const int per_band = p.num_n_blk * p.hist_group;
    const int band = tile / per_band, r = tile - band * per_band;
    n_blk = r / p.hist_group;
    const int mi = band * p.hist_group + (r - n_blk * p.hist_group);   // 128-row half of a 256-row unit
    m_unit = 2 * (p.unit_first + (mi >> 1) * p.unit_stride) + (mi & 1);
    return mi < 2 * p.num_units && !(p.hist_sym && n_blk < m_unit);
  }
}

// Chan et al. merge of two (count, mean, M2) summaries.
__device__ __forceinline__ void chan_merge(float& n, float& mean, float& m2, float nb, float meanb, float m2b) {
  const float tot = n + nb;
  if (tot > 0.f) {
    const float d = meanb - mean, wb = nb / tot;
    mean = fmaf(d, wb, mean);
    m2 += m2b + d * d * n * wb;
  }
  n = tot;
}

// The layer epilogue is unrolled over all of a thread's accumulators, so whatever it inlines is repeated 64 times
// (BLOCK_N = 128).  tanh and sigmoid, which the x-vector layers never use, stay out of line: inlined, their bodies
// made the epilogue code larger than the instruction cache, and every tile's epilogue fetched its code from L2.
__device__ __noinline__ float epi_tanh(float v) { return tanhf(v); }
__device__ __noinline__ float epi_sigmoid(float v) { return 1.f / (1.f + expf(-v)); }

// A masked batch's rows past an utterance's end store zeros: this thread's column pairs c, c + 8, ... below c_end.  Out
// of line for the same reason, and because unmasked layers never take it.
__device__ __noinline__ void epi_zero_row(const TdnnGemmParams& p, long long grow, long long frow, int c_begin, int c_end) {
  for (int c = c_begin; c < c_end; c += 8) {
    const bool has1 = c + 1 < p.Cout;
    if (p.y_hi) {
      if (has1) {
        *reinterpret_cast<uint32_t*>(p.y_hi + grow * p.ldy + c) = 0u;
        *reinterpret_cast<uint32_t*>(p.y_lo + grow * p.ldy + c) = 0u;
      } else {
        p.y_hi[grow * p.ldy + c] = __float2bfloat16(0.f);
        p.y_lo[grow * p.ldy + c] = __float2bfloat16(0.f);
      }
    }
    if (p.y_f32) {
      float* df = p.y_f32 + frow * p.ldyf + c;
      if (has1) *reinterpret_cast<float2*>(df) = make_float2(0.f, 0.f);
      else *df = 0.f;
    }
  }
}

// Per-tile timeline of the consumer warpgroups, for tools/tile_timeline.py.  Compiled in only with -DXVB_TILE_TIMELINE
// (`make timeline` builds libxvb200_timeline.so next to the library the package loads); the default build contains none
// of it.  One thread per warpgroup writes clock64 stamps per tile into the buffer given to xvb_tile_timeline_set: main
// loop start, first operands there, last MMA issued, MMAs retired, epilogue end, and the clocks spent waiting on the full
// barriers.  The CTA's head holds %globaltimer and clock64 at its start and at each warpgroup's end, which gives the
// clock's rate.  Plain stores: a printf or any other call would serialise the MMAs (C7510).
#ifdef XVB_TILE_TIMELINE
#define XVB_TL(...) __VA_ARGS__   // host side: the plan's timeline fields
constexpr int kTimelineHead = 8, kTimelineRec = 12;
static unsigned long long* g_timeline = nullptr;
static int g_timeline_tiles = 0;
static bool g_timeline_direct = false;
__device__ __forceinline__ unsigned long long global_timer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// keep the fused pooling epilogue on its general path (tile_timeline.py --direct-stores)
__device__ __forceinline__ bool timeline_general(const TdnnGemmParams& p) { return p.timeline_general; }
struct TileClock {
  unsigned long long* cta;   // this CTA's part of the buffer, or NULL
  long long start = 0, first = 0, issued = 0, retired = 0, wait = 0, w0 = 0, t = 0;
  long long ep[4] = {0, 0, 0, 0};   // epilogue sub-phases: TMA read wait, coefficients + barrier, arithmetic, store issue
  __device__ __forceinline__ explicit TileClock(const TdnnGemmParams& p)
      : cta(p.timeline ? p.timeline + (size_t)blockIdx.x * (kTimelineHead + (size_t)kTimelineRec * p.timeline_tiles)
                       : nullptr) {
    if (cta && threadIdx.x == 0) { cta[0] = global_timer(); cta[1] = (unsigned long long)clock64(); }
  }
  __device__ __forceinline__ void tile_start() { start = clock64(); wait = 0; ep[0] = ep[1] = ep[2] = ep[3] = 0; }
  __device__ __forceinline__ void wait_begin() { w0 = clock64(); }
  __device__ __forceinline__ void wait_end(bool first_stage) {
    const long long w1 = clock64();
    wait += w1 - w0;
    first = first_stage ? w1 : first;
  }
  __device__ __forceinline__ void mmas_issued() { issued = clock64(); }
  __device__ __forceinline__ void mmas_retired() { retired = clock64(); t = retired; }
  __device__ __forceinline__ void mark(int ph) { const long long now = clock64(); ep[ph] += now - t; t = now; }
  __device__ __forceinline__ void flush(const TdnnGemmParams& p, int tj, int wg) const {
    if (cta && (threadIdx.x & 127) == 0 && tj < p.timeline_tiles) {
      unsigned long long* r = cta + kTimelineHead + (size_t)kTimelineRec * tj;
      r[0] = (unsigned long long)start; r[1] = (unsigned long long)first; r[2] = (unsigned long long)issued;
      r[3] = (unsigned long long)retired; r[4] = (unsigned long long)clock64(); r[5] = (unsigned long long)wait;
      r[6] = (unsigned long long)wg; r[7] = 1ull;
      for (int ph = 0; ph < 4; ++ph) r[8 + ph] = (unsigned long long)ep[ph];
    }
  }
  __device__ __forceinline__ void end(int wg) const {
    if (cta && (threadIdx.x & 127) == 0) { cta[2 + 2 * wg] = global_timer(); cta[3 + 2 * wg] = (unsigned long long)clock64(); }
  }
};
#else
#define XVB_TL(...)
__device__ __forceinline__ bool timeline_general(const TdnnGemmParams&) { return false; }
struct TileClock {
  __device__ __forceinline__ explicit TileClock(const TdnnGemmParams&) {}
  __device__ __forceinline__ void tile_start() {}
  __device__ __forceinline__ void wait_begin() {}
  __device__ __forceinline__ void wait_end(bool) {}
  __device__ __forceinline__ void mmas_issued() {}
  __device__ __forceinline__ void mmas_retired() {}
  __device__ __forceinline__ void mark(int) {}
  __device__ __forceinline__ void flush(const TdnnGemmParams&, int, int) const {}
  __device__ __forceinline__ void end(int) const {}
};
#endif

// A position in the ring of operand stages.  Full and empty barriers are waited on by phase parity.
template <int kStages>
struct RingPos {
  int stage = 0;
  uint32_t phase = 0;
  __device__ __forceinline__ void next() { if (++stage == kStages) { stage = 0; phase ^= 1; } }
  __device__ __forceinline__ void skip(int n) {
    stage += n;
    phase ^= (uint32_t)(stage / kStages) & 1u;
    stage %= kStages;
  }
  // the stage before `stage`, whose MMAs retire next.  Derived rather than carried: the ping-pong main loop has no
  // register to spare.
  __device__ __forceinline__ int before() const { return stage == 0 ? kStages - 1 : stage - 1; }
};

// The epilogue switches of p.flags.
struct EpiFlags {
  bool bn, act_sigmoid, act_tanh;
  float relu_floor;   // branch-free ReLU switch
  __device__ __forceinline__ explicit EpiFlags(int flags)
      : bn((flags & XVB_BN) != 0), act_sigmoid((flags & XVB_SIGMOID) != 0), act_tanh((flags & XVB_TANH) != 0),
        relu_floor((flags & XVB_RELU) != 0 ? 0.f : -INFINITY) {}
  // The layer epilogues' chain after the pre-activation sum: ReLU -> swish -> BN -> tanh / sigmoid.
  template <bool kSwish>
  __device__ __forceinline__ float activate(float v, float scale, float shift) const {
    v = fmaxf(v, relu_floor);
    if constexpr (kSwish) v = v / (1.f + expf(-v));
    if (bn) v = fmaf(v, scale, shift);
    if (act_tanh) v = epi_tanh(v);
    if (act_sigmoid) v = epi_sigmoid(v);
    return v;
  }
};

// Fused pooling: one output channel's bias, scale and shift, and the value it pools, BN(ReLU(acc + bias)).
struct PoolChannel {
  bool valid;
  float bias, scale, shift;
  __device__ __forceinline__ PoolChannel(const TdnnGemmParams& p, int c, bool bn)
      : valid(c < p.Cout), bias((valid && p.bias) ? __ldg(p.bias + c) : 0.f), scale((valid && bn) ? __ldg(p.scale + c) : 1.f),
        shift((valid && bn) ? __ldg(p.shift + c) : 0.f) {}
  __device__ __forceinline__ float operator()(float acc, float relu_floor) const {
    return fmaf(fmaxf(acc + bias, relu_floor), scale, shift);
  }
};

// Fused trial histogram (scoring.cu): score -> bin -> shared-memory counter of its class (same / different speaker).
// The 16 KB slab holds 2 x hist_bins u32 counters; out-of-window scores (the vast majority in a zoomed pass) are counted
// branch-free in registers.
struct TrialHistogram {
  uint32_t slab;
  uint32_t below[2] = {0u, 0u}, above[2] = {0u, 0u};
  uint32_t tiles = 0;
  __device__ __forceinline__ explicit TrialHistogram(const uint8_t* slab_base) : slab(smem_u32(slab_base)) {}
  __device__ __forceinline__ void clear(const TdnnGemmParams& p) const {
    for (int e = threadIdx.x; e < 2 * p.hist_bins; e += kNumConsumers)
      asm volatile("st.shared.u32 [%0], %1;" ::"r"(slab + e * 4), "r"(0u) : "memory");
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
  template <int BLOCK_N>
  __device__ __forceinline__ void count(const TdnnGemmParams& p, const float (&acc)[BLOCK_N / 2], int b0, int t0, int n0,
                                        int row0) {
    const int q4 = threadIdx.x & 3;
    const float top = (float)(p.hist_bins - 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = row0 + 8 * h;
      const int b = b0 + (row >> p.log2_tb), t = t0 + (row & (p.Tb - 1));
      const bool valid = (b < p.B) && (t < p.T);
      const float rbias = (p.row_bias && valid) ? __ldg(p.row_bias + (long long)b * p.T + t) : 0.f;
      const int lab_r = valid ? __ldg(p.row_label + b) : -1;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int c = n0 + 8 * i + 2 * q4 + e;
          const bool in = c < p.Cout;
          const uint32_t ok = (valid && in && (!p.hist_sym || c > b)) ? 1u : 0u;
          const float sc = acc[4 * i + 2 * h + e] + ((in && p.bias) ? __ldg(p.bias + c) : 0.f) + rbias;
          const float x = (sc - p.hist_lo) * p.hist_inv_w;
          const uint32_t cls = (in && __ldg(p.col_label + c) == lab_r) ? 1u : 0u;
          const uint32_t bl = x < 0.f ? ok : 0u;
          const uint32_t ab = !(x < top) ? ok : 0u;          // also catches NaN
          below[0] += bl & (cls ^ 1u); below[1] += bl & cls;
          above[0] += ab & (cls ^ 1u); above[1] += ab & cls;
          if (ok & ~(bl | ab))
            asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(slab + ((int)cls * p.hist_bins + 1 + (int)x) * 4), "r"(1u) : "memory");
        }
      }
    }
    if ((++tiles & 0x3fffu) == 0) flush(p);   // u32 counters: <= 2^14 tiles x 2^14 scores between flushes
  }
  // adds the slab and the register counts to p.hist and clears them
  __device__ __forceinline__ void flush(const TdnnGemmParams& p) {
    asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      if (below[c]) asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(slab + (c * p.hist_bins) * 4), "r"(below[c]) : "memory");
      if (above[c]) asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(slab + (c * p.hist_bins + p.hist_bins - 1) * 4), "r"(above[c]) : "memory");
      below[c] = 0u; above[c] = 0u;
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
    for (int e = threadIdx.x; e < 2 * p.hist_bins; e += kNumConsumers) {
      uint32_t c;
      asm volatile("ld.shared.u32 %0, [%1];" : "=r"(c) : "r"(slab + e * 4) : "memory");
      if (c) {
        atomicAdd(p.hist + e, (unsigned long long)c);
        asm volatile("st.shared.u32 [%0], %1;" ::"r"(slab + e * 4), "r"(0u) : "memory");
      }
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");
  }
};

// The roles of one instance of the layer kernel: the TMA producer, the consumers' main loop and their epilogues.
//
// kSwish: the layer epilogue applies x * sigmoid(x) after the ReLU (XVB_SWISH).  A template flag rather than a runtime
// one, so that the instantiations without it compile to the same code as before the flag existed.
//
// Every function is force-inlined: a call would serialise every wgmma of the kernel (C7510).
template <int BLOCK_N, bool kPool, bool kHist, bool kSwish>
struct LayerKernel {
  // the staged epilogue moves 64-channel boxes; the 32-wide instances keep the direct stores
  static constexpr bool kStaged = staged_epilogue<BLOCK_N, kPool, kHist>();
  using Cfg = GemmCfg<BLOCK_N, kPool, kHist>;
  static constexpr int kStages = Cfg::kStages;
  static constexpr int kBBytes = Cfg::kBBytes;
  static constexpr int kStageBytes = Cfg::kStageBytes;
  static constexpr int kAccRegs = Cfg::kAccRegs;
  static_assert(!kPool || BLOCK_N == kBlockM, "fused pooling: 128 channels x 128 frames per tile");
  static constexpr bool kPingPong = ping_pong<BLOCK_N, kHist, kSwish>();
  static constexpr int kHalves = kPingPong ? 2 : 1;                          // 64-row accumulator halves per consumer thread
  static constexpr int kReleaseWarps = kPingPong ? 4 : kNumConsumers / 32;   // warps that consume (and release) one stage
  using Acc = float[kHalves][kAccRegs];
  using Ring = RingPos<kStages>;

  // The epilogues take the halves one after the other through the same code on acc[0] (a rolled loop): unrolled over
  // both, the ping-pong instances' code was twice as large, more than the instruction cache holds.
  static __device__ __forceinline__ void half_down(Acc& acc) {
#pragma unroll
    for (int i = 0; i < kAccRegs; ++i) acc[0][i] = acc[kHalves - 1][i];
  }

  // ================================ TMA producer (one thread) ================================
  static __device__ __forceinline__ void produce(const TdnnGemmParams& p, uint8_t* smem, uint64_t* full_bar,
                                                 uint64_t* empty_bar, const CUtensorMap* map_a_hi,
                                                 const CUtensorMap* map_a_lo, const CUtensorMap* map_a2_hi,
                                                 const CUtensorMap* map_a2_lo, const CUtensorMap* map_w_hi,
                                                 const CUtensorMap* map_w_lo) {
    Ring ring;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      int m_unit, n_blk, slice;
      if (!decode_tile<kHist>(p, tile, m_unit, n_blk, slice)) continue;   // e.g. entirely on or below the diagonal
      const int cb_begin = slice * p.kb_per_slice;                        // (0, num_cblk) unless split-K
      const int cb_end = p.k_slices > 1 ? min(p.num_cblk, cb_begin + p.kb_per_slice) : p.num_cblk;
      const int b0 = (m_unit / p.num_t_blk) * p.Bb, t0 = (m_unit % p.num_t_blk) * p.Tb;  // may be fully out of
      const int n0 = n_blk * BLOCK_N;                                                    // range: TMA zero-fills
      const int a_c0 = p.group_ng ? (n0 / p.group_ng) * p.group_kg : 0;                  // grouped: this group's K slice
      for (int src = 0; src < p.num_src; ++src) {
        const CUtensorMap* ma_hi = src == 0 ? map_a_hi : map_a2_hi;
        const CUtensorMap* ma_lo = src == 0 ? map_a_lo : map_a2_lo;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const int tt = t0 + p.ctx[tap];
          for (int cb = cb_begin; cb < cb_end; ++cb) {
            mbar_wait(&empty_bar[ring.stage], ring.phase ^ 1);
            uint8_t* s = smem + ring.stage * kStageBytes;
            const int kw = tap * p.cin_p16 + cb * kBlockK;
            mbar_expect_tx(&full_bar[ring.stage], kStageBytes);
            tma_load_3d(s, ma_hi, &full_bar[ring.stage], a_c0 + cb * kBlockK, tt, b0);
            tma_load_3d(s + kABytes, ma_lo, &full_bar[ring.stage], a_c0 + cb * kBlockK, tt, b0);
            tma_load_2d(s + 2 * kABytes, map_w_hi, &full_bar[ring.stage], kw, n0);
            tma_load_2d(s + 2 * kABytes + kBBytes, map_w_lo, &full_bar[ring.stage], kw, n0);
            ring.next();
          }
        }
      }
    }
  }

  // ================================ consumer main loop ================================
  // One tile's K blocks [kb_begin, kb_end), one (64 channels of one tap and source) per operand stage from `ring` on.
  // Returns with the accumulators retired and the last stage released.  Ping-pong: once this tile's MMAs are issued, the
  // warpgroup of the CTA's next tile (if any) may start its main loop (named barrier 3 - wg).
  static __device__ __forceinline__ void main_loop(const TdnnGemmParams& p, Acc& acc, uint8_t* smem, uint64_t* full_bar,
                                                   uint64_t* empty_bar, Ring& ring, int kb_begin, int kb_end, int tile,
                                                   int wg, TileClock& clk) {
    const int lane = threadIdx.x & 31;
    const int row_base = kPingPong ? 0 : 64 * wg;   // first accumulator row of this warpgroup's (first) half
    // The tile's first MMA (which overwrites the accumulators) is derived from kb, not carried, as is ring.before().
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      clk.wait_begin();
      mbar_wait(&full_bar[ring.stage], ring.phase);
      clk.wait_end(kb == kb_begin);
      const uint32_t sa = smem_u32(smem + ring.stage * kStageBytes);
      const uint64_t dx_hi = make_sw128_desc(sa), dx_lo = make_sw128_desc(sa + kABytes);
      const uint64_t dw_hi = make_sw128_desc(sa + 2 * kABytes), dw_lo = make_sw128_desc(sa + 2 * kABytes + kBBytes);
      // M side: 64 rows per half (8 KB each into the 128-row tile); N side: the whole other tile
      const uint64_t da_hi = kPool ? dw_hi : dx_hi, da_lo = kPool ? dw_lo : dx_lo;
      const uint64_t db_hi = kPool ? dx_hi : dw_hi, db_lo = kPool ? dx_lo : dw_lo;
      // Every stage issues all four K steps, also the last channel block of a Cin that is not a multiple of 64: the
      // frame maps' channel extent is Cin (the im2col view's too), so TMA fills the channels past it with zeros and the
      // extra products add exact zeros.  The trip count has to be a compile-time constant: with a runtime one (or a
      // branch between the fence and the commit) ptxas serialises every wgmma of the kernel (C7520), each one waiting
      // for the previous one to finish.
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < kBlockK / 16; ++s) {
        const uint64_t koff = (uint64_t)(s * 32 >> 4);   // 16 bf16 = 32 bytes along K inside the swizzle row
#pragma unroll
        for (int hh = 0; hh < kHalves; ++hh) {
          const uint64_t m_off = (uint64_t)((row_base + 64 * hh) * 128 >> 4);
          wgmma_bf16<BLOCK_N>(acc[hh], da_lo + m_off + koff, db_hi + koff, s == 0 ? (uint32_t)(kb != kb_begin) : 1u);
          wgmma_bf16<BLOCK_N>(acc[hh], da_hi + m_off + koff, db_lo + koff, 1);
          wgmma_bf16<BLOCK_N>(acc[hh], da_hi + m_off + koff, db_hi + koff, 1);
        }
      }
      wgmma_commit();
      wgmma_wait<1>();                               // the previous stage's MMAs have retired: release it
      if (kb != kb_begin && lane == 0) mbar_arrive(&empty_bar[ring.before()]);
      ring.next();
    }
    // the next tile's warpgroup may start its main loop
    if (kPingPong && tile + gridDim.x < p.num_tiles) asm volatile("bar.arrive %0, 256;" ::"r"(3 - wg) : "memory");
    clk.mmas_issued();
    wgmma_wait<0>();
    clk.mmas_retired();
#pragma unroll
    for (int hh = 0; hh < kHalves; ++hh) wgmma_fence_operands(acc[hh]);
    if (kb_end > kb_begin && lane == 0) mbar_arrive(&empty_bar[ring.before()]);
  }

  // ================================ fused statistics pooling epilogue ================================
  // Rows = channels, columns = the tile's 128 frames.  Time block g of the tile is columns [g*Tb, (g+1)*Tb) = utterance
  // b0+g, frames t0.. ; the first nv of them exist.
  //
  // Full 8-frame time blocks (Tb == 8 and all 8 frames exist; uniform per tile) stage the tile's partials in the
  // warpgroup's 16 KB, [utterance][mean | M2][128 channels] fp32, and one thread stores them with one TMA store through
  // the (Cout, 2, B, time block) map of pool_partial, whose extents clip the channels past Cout and the utterances past
  // B.  The previous tile's store has read the buffer: its thread waited for that before the turn barrier of this
  // tile's main loop.
  static __device__ __forceinline__ bool pool_full_blocks(const TdnnGemmParams& p, int nv) {
    return p.tma_store && p.Tb == 8 && nv == 8 && !timeline_general(p);
  }

  static __device__ __forceinline__ void pool_epilogue(const TdnnGemmParams& p, Acc& acc, uint8_t* slab_base, int b0,
                                                       int t0, int tblk, int n0, int row0, int wg, const EpiFlags& f,
                                                       const CUtensorMap* map_pool, TileClock& clk) {
    int nv = p.T - t0;
    nv = nv < 0 ? 0 : (nv > p.Tb ? p.Tb : nv);
#pragma unroll 1
    for (int hh = 0; hh < kHalves; ++hh) {
      if (hh > 0) half_down(acc);
      // opaque per half: hoisted out of the rolled loop, the store addresses and validity masks derived from them
      // stayed live through both halves and spilled
      int b0h = b0, nvh = nv;
      asm volatile("" : "+r"(b0h), "+r"(nvh));
      if (pool_full_blocks(p, nvh)) {
        pool_full_block_half(p, acc[0], slab_base, hh, n0 + row0 + 64 * hh, f);
        clk.mark(2);
        continue;
      }
      pool_general_half(p, acc[0], b0h, nvh, tblk, n0 + row0 + 64 * hh, f);
    }
    clk.mark(2);
    if (pool_full_blocks(p, nv)) {
      fence_proxy_async();                             // the staged partials become visible to the TMA unit
      asm volatile("bar.sync %0, 128;" ::"r"(4 + wg) : "memory");
      clk.mark(1);
      if ((threadIdx.x & 127) == 0) {
        tma_store_4d(map_pool, smem_u32(slab_base) + wg * kStageOutBytes, n0, 0, b0, tblk);
        tma_store_commit();
      }
      clk.mark(3);
    }
  }

  // Full 8-frame time blocks: block i of the tile is exactly the 8-column chunk i, and every Chan merge in it has known
  // counts, so the divisions fold.  With chan_merge's names:
  //   pair into the empty summary: n = 0, nb = tot = 2, wb = 1: d = pm - 0 = pm, mean = fmaf(pm, 1, 0) = pm + 0 (a -0
  //     becomes +0), m2 = 0 + (pm2 + pm * pm * 0 * 1) = pm2, since pm2 >= 0 and the product is +0 on finite data;
  //   lanes q4 ^ 1: n = nb = 2, tot = 4, wb = 0.5: mean = fmaf(d, 0.5, mean), m2 += m2b + d * d * 2 * 0.5;
  //   lanes q4 ^ 2: n = nb = 4, tot = 8, wb = 0.5: mean = fmaf(d, 0.5, mean), m2 += m2b + d * d * 4 * 0.5.
  // Every operation that rounds is kept, in chan_merge's order (the two multiplications by powers of two as well: they
  // are exact except where d * d * n overflows, and there they give what chan_merge gives), so the partials are
  // bit-identical to the general path's on finite data.  No summary carries from one chunk to the next, so the 16
  // chunks of a row are independent chains that the compiler interleaves.  `ch0`: this thread's first output channel.
  static __device__ __forceinline__ void pool_full_block_half(const TdnnGemmParams& p, const float (&a)[kAccRegs],
                                                              uint8_t* slab_base, int hh, int ch0, const EpiFlags& f) {
    const int q4 = threadIdx.x & 3;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const PoolChannel ch(p, ch0 + 8 * h, f.bn);
      int tid = threadIdx.x;                          // opaque, as b0h: derived per use, not kept live
      asm volatile("" : "+r"(tid));
      const uint32_t dst0 = smem_u32(slab_base) + (tid >> 7) * kStageOutBytes +
                            4 * (16 * ((tid >> 5) & 3) + ((tid & 31) >> 2) + 64 * hh + 8 * h);
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        const float x0 = ch(a[4 * i + 2 * h], f.relu_floor);
        const float x1 = ch(a[4 * i + 2 * h + 1], f.relu_floor);
        float mean = 0.5f * (x0 + x1) + 0.f;
        float m2 = 0.5f * (x0 - x1) * (x0 - x1);
        float d = __shfl_xor_sync(0xffffffffu, mean, 1) - mean;
        float m2b = __shfl_xor_sync(0xffffffffu, m2, 1);
        mean = fmaf(d, 0.5f, mean);
        m2 += m2b + d * d * 2.f * 0.5f;
        d = __shfl_xor_sync(0xffffffffu, mean, 2) - mean;
        m2b = __shfl_xor_sync(0xffffffffu, m2, 2);
        mean = fmaf(d, 0.5f, mean);
        m2 += m2b + d * d * 4.f * 0.5f;
        if (q4 == 0) {
          st_shared_f32(dst0 + 2 * 4 * BLOCK_N * i, mean);
          st_shared_f32(dst0 + 2 * 4 * BLOCK_N * i + 4 * BLOCK_N, m2);
        }
      }
    }
  }

  // General path (masked, ragged or Tb != 8): Chan merges within each thread and across the quad, direct stores.
  static __device__ __forceinline__ void pool_general_half(const TdnnGemmParams& p, const float (&a)[kAccRegs], int b0h,
                                                           int nvh, int tblk, int ch0, const EpiFlags& f) {
    const int q4 = threadIdx.x & 3;
    const int gl = p.Tb < 8 ? p.Tb : 8;              // columns of one group inside one 8-column chunk
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int cch = ch0 + 8 * h;                   // this thread's output channel
      const PoolChannel ch(p, cch, f.bn);
      auto emit = [&](int col, float mean, float m2) {
        const int bb = b0h + (col >> p.log2_tb);
        if (ch.valid && bb < p.B) {
          float* dst = p.pool_partial + ((long long)tblk * p.B + bb) * (2LL * p.Cout) + cch;
          dst[0] = mean;
          dst[p.Cout] = m2;
        }
      };
      float rn = 0.f, rmean = 0.f, rm2 = 0.f;
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        const int col = 8 * i + 2 * q4;
        const float x0 = ch(a[4 * i + 2 * h], f.relu_floor);
        const float x1 = ch(a[4 * i + 2 * h + 1], f.relu_floor);
        if (p.Tb == 1) {
          if (nvh > 0) { emit(col, x0, 0.f); emit(col + 1, x1, 0.f); }
          continue;
        }
        const int j = col & (p.Tb - 1);              // frame offset of x0 inside its time block
        const bool v0 = j < nvh, v1 = j + 1 < nvh;
        const float pn = (float)v0 + (float)v1;
        const float pm = v1 ? 0.5f * (x0 + x1) : (v0 ? x0 : 0.f);
        const float pm2 = v1 ? 0.5f * (x0 - x1) * (x0 - x1) : 0.f;
        chan_merge(rn, rmean, rm2, pn, pm, pm2);
        if (((col - 2 * q4 + 8) & (p.Tb - 1)) == 0) {  // a time block ends in this chunk (warp-uniform)
          if (gl >= 4) chan_merge(rn, rmean, rm2, __shfl_xor_sync(0xffffffffu, rn, 1),
                                  __shfl_xor_sync(0xffffffffu, rmean, 1), __shfl_xor_sync(0xffffffffu, rm2, 1));
          if (gl >= 8) chan_merge(rn, rmean, rm2, __shfl_xor_sync(0xffffffffu, rn, 2),
                                  __shfl_xor_sync(0xffffffffu, rmean, 2), __shfl_xor_sync(0xffffffffu, rm2, 2));
          if (((2 * q4) & (gl - 1)) == 0 && rn > 0.f) emit(col & ~(p.Tb - 1), rmean, rm2);
          rn = 0.f; rmean = 0.f; rm2 = 0.f;
        }
      }
    }
  }

  // ================================ layer epilogues ================================
  // +bias (+ row / utterance terms) -> ReLU -> swish -> BN -> tanh / sigmoid -> fp32 and/or split planes.
  //
  // Staged (p.tma_store, one uniform branch per tile): a 64-row half leaves in pieces of 64 channels.  Per piece the
  // warpgroup puts the 64 columns' bias, scale and shift into shared memory once, every thread applies the same
  // arithmetic in the same order as the direct path and writes its packed hi and lo pairs into the warpgroup's staging
  // buffer, and one thread stores the two planes with TMA.  The buffer has the 128-byte swizzle of the store maps
  // (16-byte chunk index ^ row & 7): a warp's eight rows fall into eight different chunks, so its stores do not
  // conflict.  The maps' extents (Cout, T, B) clip the rows past T or B and the channels past Cout, so there are no
  // tail branches; rows past an utterance's length are staged as zeros.
  static __device__ __forceinline__ void layer_epilogue_staged(const TdnnGemmParams& p, Acc& acc, uint8_t* slab_base,
                                                               int b0, int t0, int n0, const EpiFlags& f,
                                                               const CUtensorMap* map_y_hi, const CUtensorMap* map_y_lo,
                                                               TileClock& clk) {
    // Everything below derives from an opaque copy of the thread index, per tile: hoisted out of the tile loop, these
    // addresses stayed live through the main loop, which has no register to spare, and spilled more.
    int tid = threadIdx.x;
    asm volatile("" : "+r"(tid));
    const int wgo = tid >> 7, wtid = tid & 127, q4o = tid & 3;
    const int prow = 16 * ((tid >> 5) & 3) + ((tid & 31) >> 2);   // this thread's first row of a 64-row piece
    const uint32_t stg = smem_u32(slab_base) + wgo * kStageOutBytes;
    const uint32_t coefs = smem_u32(slab_base) + 2 * kStageOutBytes + wgo * kCoefBytes;
    const int ebar = 4 + wgo;                         // named barrier of this warpgroup's epilogue
    const uint32_t coef = coefs + 8 * q4o;            // this thread's column pair of the first 8 columns
    // this thread's 4 bytes of 16-byte chunk 0 of its first row (the second is 8 rows on, with the same row & 7):
    // chunk i of the row is at my ^ (i << 4), the swizzle being an XOR on those three address bits
    const uint32_t my = stg + (uint32_t)prow * 128u + ((uint32_t)(prow & 7) << 4) + 4u * q4o;
#pragma unroll 1
    for (int hh = 0; hh < kHalves; ++hh) {
      if (hh > 0) half_down(acc);
      const int hrow = (kPingPong ? 0 : 64 * wgo) + 64 * hh;   // the half's first row of the tile: a box of the store maps
      uint32_t keep[2];                               // 0 for a masked batch's rows past the utterance's end
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int row = hrow + prow + 8 * r;
        const int b = b0 + (row >> p.log2_tb), t = t0 + (row & (p.Tb - 1));
        keep[r] = (p.lengths && b < p.B && t >= __ldg(p.lengths + b)) ? 0u : 0xffffffffu;
      }
#pragma unroll
      for (int cr = 0; cr < BLOCK_N / kBlockK; ++cr) {
        const int c0 = n0 + kBlockK * cr;
        if (c0 >= p.Cout) break;
        if (wtid == 0) tma_store_wait_read<0>();      // the previous piece has left the staging buffer
        clk.mark(0);
        if (wtid < kBlockK) {
          const int c = c0 + wtid;
          const bool in = c < p.Cout;
          st_shared_f32(coefs + 4 * wtid, (in && p.bias) ? __ldg(p.bias + c) : 0.f);
          st_shared_f32(coefs + 4 * (kBlockK + wtid), (in && f.bn) ? __ldg(p.scale + c) : 1.f);
          st_shared_f32(coefs + 4 * (2 * kBlockK + wtid), (in && f.bn) ? __ldg(p.shift + c) : 0.f);
        }
        asm volatile("bar.sync %0, 128;" ::"r"(ebar) : "memory");
        clk.mark(1);
#pragma unroll
        for (int i = 0; i < kBlockK / 8; ++i) {
          const float2 bias_c = ld_shared_f2(coef + 32 * i), scale_c = ld_shared_f2(coef + 32 * i + 4 * kBlockK),
                       shift_c = ld_shared_f2(coef + 32 * i + 8 * kBlockK);
          const float bias_e[2] = {bias_c.x, bias_c.y}, scale_e[2] = {scale_c.x, scale_c.y},
                      shift_e[2] = {shift_c.x, shift_c.y};
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float x[2] = {acc[0][4 * (8 * cr + i) + 2 * r], acc[0][4 * (8 * cr + i) + 2 * r + 1]};
#pragma unroll
            for (int e = 0; e < 2; ++e)   // + 0.f: the direct path adds its (absent) row term here, which turns a -0 sum into +0
              x[e] = f.activate<kSwish>(x[e] + bias_e[e] + 0.f, scale_e[e], shift_e[e]);
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(x[0], h0, l0);
            split_bf16(x[1], h1, l1);
            const uint32_t at = (my ^ ((uint32_t)i << 4)) + 1024u * r;
            st_shared_u32(at, pack_bf16x2(h0, h1) & keep[r]);
            st_shared_u32(at + kStagePlaneBytes, pack_bf16x2(l0, l1) & keep[r]);
          }
        }
        clk.mark(2);
        fence_proxy_async();                          // the staged piece becomes visible to the TMA unit
        asm volatile("bar.sync %0, 128;" ::"r"(ebar) : "memory");
        if (wtid == 0) {
          const int hb = b0 + (hrow >> p.log2_tb), ht = t0 + (hrow & (p.Tb - 1));
          tma_store_3d(map_y_hi, stg, c0, ht, hb);
          tma_store_3d(map_y_lo, stg + kStagePlaneBytes, c0, ht, hb);
          tma_store_commit();
        }
        clk.mark(3);
      }
    }
  }

  // Direct stores.  Column pairs outer, rows inner: a thread's two rows of a half share its columns, so bias, scale and
  // shift are loaded once per column and half.
  static __device__ __forceinline__ void layer_epilogue_direct(const TdnnGemmParams& p, Acc& acc, int b0, int t0, int n0,
                                                               int slice, int row0, const EpiFlags& f) {
    const int q4 = threadIdx.x & 3;
#pragma unroll 1
    for (int hh = 0; hh < kHalves; ++hh) {
      if (hh > 0) half_down(acc);
      constexpr int kRows = 2;
      bool live[kRows];                               // row exists and is not masked
      float rbias[kRows];
      const float* ub[kRows];
      long long grow[kRows], frow[kRows];
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const int row = row0 + 64 * hh + 8 * r;
        const int b = b0 + (row >> p.log2_tb), t = t0 + (row & (p.Tb - 1));
        live[r] = b < p.B && t < p.T;
        grow[r] = (long long)b * p.T + t;
        frow[r] = (long long)b * p.out_T + t + slice;   // split-K: partial of slice s at "time" s
        if (live[r] && p.lengths && t >= __ldg(p.lengths + b)) {   // masked batch, frame past the utterance's end: zeros
          epi_zero_row(p, grow[r], frow[r], n0 + 2 * q4, min(n0 + BLOCK_N, p.Cout));
          live[r] = false;
        }
        rbias[r] = (live[r] && p.row_bias) ? __ldg(p.row_bias + grow[r]) : 0.f;
        ub[r] = (live[r] && p.utt_bias) ? p.utt_bias + (long long)b * p.ld_utt : nullptr;
      }
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        const int c = n0 + 8 * i + 2 * q4;
        if (c >= p.Cout) break;
        const bool has1 = c + 1 < p.Cout;
        float bias_c[2], scale_c[2], shift_c[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool in = e == 0 || has1;
          bias_c[e] = (in && p.bias) ? __ldg(p.bias + c + e) : 0.f;
          scale_c[e] = (in && f.bn) ? __ldg(p.scale + c + e) : 1.f;
          shift_c[e] = (in && f.bn) ? __ldg(p.shift + c + e) : 0.f;
        }
#pragma unroll
        for (int r = 0; r < kRows; ++r) {
          if (!live[r]) continue;
          float x[2] = {acc[0][4 * i + 2 * r], acc[0][4 * i + 2 * r + 1]};
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            if (e == 1 && !has1) break;
            float v = x[e] + bias_c[e] + rbias[r];
            if (ub[r]) v += __ldg(ub[r] + c + e);
            x[e] = f.activate<kSwish>(v, scale_c[e], shift_c[e]);
          }
          if (p.y_hi) {
            __nv_bfloat16 h0, l0, h1, l1;
            split_bf16(x[0], h0, l0);
            split_bf16(x[1], h1, l1);
            __nv_bfloat16* dh = p.y_hi + grow[r] * p.ldy + c;
            __nv_bfloat16* dl = p.y_lo + grow[r] * p.ldy + c;
            if (has1) {
              *reinterpret_cast<uint32_t*>(dh) = pack_bf16x2(h0, h1);
              *reinterpret_cast<uint32_t*>(dl) = pack_bf16x2(l0, l1);
            } else {
              *dh = h0;
              *dl = l0;
            }
          }
          if (p.y_f32) {
            float* df = p.y_f32 + frow[r] * p.ldyf + c;
            if (has1) *reinterpret_cast<float2*>(df) = make_float2(x[0], x[1]);
            else *df = x[0];
          }
        }
      }
    }
  }
};

// Ping-pong (the 128-wide layer and fused-pooling instances): tile j of the CTA's list (blockIdx.x + j * gridDim.x)
// belongs to warpgroup j & 1, which computes all 128 of its rows as two m64 halves.  Each warpgroup finds its place in
// the operand ring from a running count of the K blocks of all the CTA's tiles, the other warpgroup's included.  Both
// wait on the ring's full barriers by phase parity, which only tells the phase being waited for from the one before it:
// a warpgroup that started waiting on its next tile's first stage while the producer was still more than one lap of
// the ring behind would take an older load of that stage for its own.  So the main loops take turns on named barriers
// 2 + wg ("warpgroup wg may start its main loop"): a warpgroup starts one only after the other has issued the previous
// tile's MMAs, and the epilogue of that tile then runs under the other's main loop.
template <int BLOCK_N, bool kPool, bool kHist, bool kSwish = false>
__global__ void __launch_bounds__(gemm_threads<BLOCK_N, kHist, kSwish>(), 1)
tdnn_gemm_bf16x3_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                        const __grid_constant__ CUtensorMap map_a2_hi, const __grid_constant__ CUtensorMap map_a2_lo,
                        const __grid_constant__ CUtensorMap map_w_hi, const __grid_constant__ CUtensorMap map_w_lo,
                        const __grid_constant__ CUtensorMap map_y_hi, const __grid_constant__ CUtensorMap map_y_lo,
                        const __grid_constant__ TdnnGemmParams p) {
  using K = LayerKernel<BLOCK_N, kPool, kHist, kSwish>;

  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* slab_base = smem + K::kStages * K::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(slab_base + K::Cfg::kTailBytes);
  uint64_t* empty_bar = full_bar + K::kStages;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&map_a_hi);
    tma_prefetch_desc(&map_a_lo);
    tma_prefetch_desc(&map_w_hi);
    tma_prefetch_desc(&map_w_lo);
    if ((K::kStaged || kPool) && p.tma_store) {
      tma_prefetch_desc(&map_y_hi);
      tma_prefetch_desc(&map_y_lo);
    }
    for (int i = 0; i < K::kStages; ++i) {
      mbar_init(&full_bar[i], 1);                      // producer arrival + all TMA bytes
      mbar_init(&empty_bar[i], K::kReleaseWarps);      // one arrival per consumer warp of the stage's warpgroup(s)
    }
    fence_barrier_init();
  }
  __syncthreads();
  // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) may overlap the
  // tail of the previous kernel in the stream; its results are needed from here on.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // the previous kernel may have written our operands with ordinary (generic-proxy) stores -- the staging
  // / pooling kernels do -- while we read them through TMA (async proxy): order the two proxies explicitly,
  // a kernel boundary would have done it for us
  asm volatile("fence.proxy.async;" ::: "memory");

  if (warp >= kProducerWarp) {
    if constexpr (K::kPingPong) setmaxnreg_dec<kProducerRegs>();   // the whole producer warpgroup
    if (warp == kProducerWarp && lane == 0)
      K::produce(p, smem, full_bar, empty_bar, &map_a_hi, &map_a_lo, &map_a2_hi, &map_a2_lo, &map_w_hi, &map_w_lo);
    return;
  }

  // ================================ consumers: wgmma + epilogue ================================
  if constexpr (K::kPingPong) setmaxnreg_inc<kConsumerRegs>();
  const int wg = warp >> 2;                          // split tiles: accumulator rows 64*wg .. 64*wg+63
  // this thread's rows: row0 + 64 * hh + 8 * h for half hh < kHalves and h < 2
  const int row0 = (K::kPingPong ? 0 : 64 * wg) + 16 * (warp & 3) + (lane >> 2);
  const EpiFlags f(p.flags);
  typename K::Acc acc;
#pragma unroll
  for (int hh = 0; hh < K::kHalves; ++hh)
#pragma unroll
    for (int i = 0; i < K::kAccRegs; ++i) acc[hh][i] = 0.f;
  typename K::Ring ring;
  TrialHistogram hist(slab_base);
  if constexpr (kHist) hist.clear(p);
  TileClock clk(p);
  const int num_kblk = p.num_src * p.ntaps * p.num_cblk;

  int tj = 0;                                        // index of the tile in the CTA's list
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, ++tj) {
    int m_unit, n_blk, slice;
    if (!decode_tile<kHist>(p, tile, m_unit, n_blk, slice)) continue;
    int kb_begin = 0, kb_end = num_kblk;
    if (p.k_slices > 1) {
      kb_begin = slice * p.kb_per_slice;
      kb_end = min(num_kblk, kb_begin + p.kb_per_slice);
    }
    if constexpr (K::kPingPong) {
      if ((tj & 1) != wg) {                          // the other warpgroup's tile: skip its stages in the ring
        ring.skip(kb_end - kb_begin);
        continue;
      }
      if (tj > 0) {
        // fused pooling: the warpgroup's previous TMA store has read the staging buffer, for all its threads past here
        if (kPool && (threadIdx.x & 127) == 0) tma_store_wait_read<0>();
        asm volatile("bar.sync %0, 256;" ::"r"(2 + wg) : "memory");   // the other's main loop is issued
      }
    }
    clk.tile_start();
    K::main_loop(p, acc, smem, full_bar, empty_bar, ring, kb_begin, kb_end, tile, wg, clk);

    const int b0 = (m_unit / p.num_t_blk) * p.Bb, t0 = (m_unit % p.num_t_blk) * p.Tb;
    const int n0 = n_blk * BLOCK_N;
    if constexpr (kHist) {
      hist.count<BLOCK_N>(p, acc[0], b0, t0, n0, row0);
      continue;
    } else if constexpr (kPool) {
      K::pool_epilogue(p, acc, slab_base, b0, t0, m_unit % p.num_t_blk, n0, row0, wg, f, &map_y_hi, clk);
    } else if (K::kStaged && p.tma_store) {
      K::layer_epilogue_staged(p, acc, slab_base, b0, t0, n0, f, &map_y_hi, &map_y_lo, clk);
    } else {
      K::layer_epilogue_direct(p, acc, b0, t0, n0, slice, row0, f);
    }
    clk.flush(p, tj, wg);
  }
  if constexpr (kHist) hist.flush(p);
  if constexpr (K::kStaged || kPool) {
    if (p.tma_store && (threadIdx.x & 127) == 0) tma_store_wait_done<0>();   // this thread's stores have landed
  }
  clk.end(wg);
}

// Split-K tail: y[b,c] = epi(sum_s part[b,s,c]) with the slices added in index order (deterministic),
// same epilogue order as the GEMM's: +bias -> ReLU -> BN -> tanh/sigmoid -> fp32 and/or split planes (a layer with
// XVB_SWISH never takes the split-K path).
__global__ void segment_reduce_kernel(const float* __restrict__ part, int S, int B, int Cout, const float* __restrict__ bias,
                                      const float* __restrict__ scale, const float* __restrict__ shift, int flags,
                                      float* __restrict__ y_f32, long long ldyf, __nv_bfloat16* __restrict__ y_hi,
                                      __nv_bfloat16* __restrict__ y_lo, long long ldy) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)B * Cout) return;
  const int b = (int)(idx / Cout), c = (int)(idx - (long long)b * Cout);
  const float* src = part + (long long)b * S * Cout + c;
  float x = src[0];
  for (int s = 1; s < S; ++s) x += src[(long long)s * Cout];
  x += bias ? bias[c] : 0.f;
  if (flags & XVB_RELU) x = fmaxf(x, 0.f);
  if (flags & XVB_BN) x = fmaf(x, scale[c], shift[c]);
  if (flags & XVB_TANH) x = tanhf(x);
  if (flags & XVB_SIGMOID) x = 1.f / (1.f + expf(-x));
  if (y_f32) y_f32[(long long)b * ldyf + c] = x;
  if (y_hi) {
    __nv_bfloat16 h, l;
    split_bf16(x, h, l);
    y_hi[(long long)b * ldy + c] = h;
    y_lo[(long long)b * ldy + c] = l;
  }
}

// ------------------------------------------------------------------------------------------------
// Host side: tensor maps + launch
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

// Generic tiled tensor map (exported for pooling.cu).  esize 2 -> bf16, 4 -> fp32; swizzle_bytes 0/64/128.
int make_tensor_map(CUtensorMap* m, const void* base, int esize, int rank, const unsigned long long* dims,
                    const unsigned long long* strides_bytes, const unsigned* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return XVB_ECUDA; }
  cuuint64_t d[5], st[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) st[i] = strides_bytes[i];
  const CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                               : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(m, esize == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, rank,
                   const_cast<void*>(base), d, st, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(rank %d) failed: %d", rank, (int)r); return XVB_ECUDA; }
  return XVB_OK;
}

// (C, T, B) bf16 frame matrix with row pitch ld; box = 64 channels x Tb frames x Bb utterances.
static int make_frame_map(CUtensorMap* m, const void* base, int C, int T, int B, long long ld, int Tb, int Bb,
                          long long batch_stride = 0) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return XVB_ECUDA; }
  cuuint64_t dims[3] = {(cuuint64_t)C, (cuuint64_t)T, (cuuint64_t)B};
  cuuint64_t strides[2] = {(cuuint64_t)ld * 2, batch_stride ? (cuuint64_t)batch_stride * 2 : (cuuint64_t)ld * 2 * (cuuint64_t)T};
  cuuint32_t box[3] = {(cuuint32_t)kBlockK, (cuuint32_t)Tb, (cuuint32_t)Bb};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(frame map C=%d T=%d B=%d ld=%lld) failed: %d", C, T, B, ld, (int)r); return XVB_ECUDA; }
  return XVB_OK;
}

// Store map of the staged layer epilogue: the (Cout, T, B) bf16 output plane with row pitch ld; box = 64 channels x the 64
// rows of one accumulator half (Tb frames x 64 / Tb utterances, or 64 frames of one utterance).  The extents clip the box.
static int make_store_map(CUtensorMap* m, const void* base, int Cout, int T, int B, long long ld, int Tb) {
  const int box_t = Tb < 64 ? Tb : 64;
  const unsigned long long dims[3] = {(unsigned long long)Cout, (unsigned long long)T, (unsigned long long)B};
  const unsigned long long strides[2] = {(unsigned long long)ld * 2, (unsigned long long)ld * 2 * (unsigned long long)T};
  const unsigned box[3] = {(unsigned)kBlockK, (unsigned)box_t, (unsigned)(64 / box_t)};
  return make_tensor_map(m, base, 2, 3, dims, strides, box, 128);
}

// Store map of the fused pooling's partials, pool_partial as (Cout, 2, B, time blocks) fp32 ([mean | M2] per time block
// and utterance); box = 128 channels x both x the 16 utterances of a tile with 8-frame time blocks x one time block.
static int make_partial_map(CUtensorMap* m, const float* base, int Cout, int B, int nblk) {
  const unsigned long long dims[4] = {(unsigned long long)Cout, 2ull, (unsigned long long)B, (unsigned long long)nblk};
  const unsigned long long strides[3] = {4ull * Cout, 8ull * Cout, 8ull * Cout * (unsigned long long)B};
  const unsigned box[4] = {(unsigned)kBlockM, 2u, 16u, 1u};
  return make_tensor_map(m, base, 4, 4, dims, strides, box, 0);
}

// (K, Cout) bf16 packed weight, K contiguous; box = 64 x block_n.
static int make_weight_map(CUtensorMap* m, const void* base, long long K, int Cout, int block_n) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) { set_error("cuTensorMapEncodeTiled entry point not available"); return XVB_ECUDA; }
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)Cout};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)block_n};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weight map K=%lld Cout=%d) failed: %d", K, Cout, (int)r); return XVB_ECUDA; }
  return XVB_OK;
}

// Pick the (Tb, Bb) factorisation of the 128-row M tile with the fewest padded rows.
static void choose_m_tile(int B, int T, int* Tb_out, int* Bb_out, int max_tb = 128) {
  if (T == 1) {   // segment-level layers: one row per utterance.  (Also what split-K's "slice as time" store
    *Tb_out = 1;  // relies on: a box taller than one frame would spill zeros into the next slices' rows.)
    *Bb_out = 128;
    return;
  }
  long long best = -1;
  int bt = max_tb;
  for (int Tb = max_tb; Tb >= 1; Tb >>= 1) {
    const int Bb = 128 / Tb;
    const long long rows = (long long)((T + Tb - 1) / Tb) * Tb * ((B + Bb - 1) / Bb) * Bb;
    if (best < 0 || rows < best) { best = rows; bt = Tb; }
  }
  *Tb_out = bt;
  *Bb_out = 128 / bt;
}

// ------------------------------------------------------------------------------------------------
// Plan / launch split.  Everything that depends only on shapes and pointers -- tile geometry, the six
// tensor maps (cuTensorMapEncodeTiled is a ~1 us driver call each), the kernel instantiation, the grid --
// is decided once in a GemmPlan; launching a plan is one cudaLaunchKernelEx (+ the split-K reduce).  The
// extractor objects keep their plans per (B, T), so a batch costs launches only.
// ------------------------------------------------------------------------------------------------
struct GemmPlan {
  CUtensorMap ma_hi, ma_lo, ma2_hi, ma2_lo, mw_hi, mw_lo, my_hi, my_lo;
  TdnnGemmParams p;
  int (*launch)(const GemmPlan&, const TdnnGemmParams&, cudaStream_t) = nullptr;   // nullptr: this shard owns no rows
  int grid = 0;
  int pdl = 1;
  // split-K tail (segment_reduce_kernel); the GEMM itself then writes fp32 partials into `scratch`
  bool reduce = false;
  const float* r_bias = nullptr; const float* r_scale = nullptr; const float* r_shift = nullptr;
  int r_flags = 0;
  float* r_y_f32 = nullptr; long long r_ldyf = 0;
  __nv_bfloat16* r_y_hi = nullptr; __nv_bfloat16* r_y_lo = nullptr; long long r_ldy = 0;
};

template <int BLOCK_N, bool kPool, bool kHist, bool kSwish>
static int launch_inst(const GemmPlan& pl, const TdnnGemmParams& p, cudaStream_t stream) {
  using Cfg = GemmCfg<BLOCK_N, kPool, kHist>;
  XVB_ENSURE_DYN_SMEM((tdnn_gemm_bf16x3_kernel<BLOCK_N, kPool, kHist, kSwish>), Cfg::kSmemBytes);
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(pl.grid);
  cfg.blockDim = dim3(gemm_threads<BLOCK_N, kHist, kSwish>());
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pl.pdl ? 1 : 0;
  XVB_CUDA(cudaLaunchKernelEx(&cfg, tdnn_gemm_bf16x3_kernel<BLOCK_N, kPool, kHist, kSwish>, pl.ma_hi, pl.ma_lo, pl.ma2_hi,
                              pl.ma2_lo, pl.mw_hi, pl.mw_lo, pl.my_hi, pl.my_lo, p));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

template <int BLOCK_N, bool kPool = false, bool kHist = false, bool kSwish = false>
static int prepare_gemm(GemmPlan& pl, const void* w_hi, const void* w_lo) {
  TdnnGemmParams& p = pl.p;
  const long long K = (long long)p.ntaps * p.cin_p16;
  int rc = make_weight_map(&pl.mw_hi, w_hi, K, p.Cout, BLOCK_N);
  if (rc) return rc;
  rc = make_weight_map(&pl.mw_lo, w_lo, K, p.Cout, BLOCK_N);
  if (rc) return rc;
  p.num_n_blk = (p.Cout + BLOCK_N - 1) / BLOCK_N;
  // Plane-only layers (every frame layer of the extractors) take the staged epilogue.  The direct stores stay for fp32
  // outputs, split-K partials, row and utterance terms, and for the 32-wide instances.  They also stay when Cout % 8 != 0:
  // the store maps' Cout extent does not clip inside a 16-byte chunk, so the last chunk of every row would be written
  // whole, up to 7 channels past Cout (in a channel slice of a wider buffer, another tensor's channels).
  p.tma_store = staged_epilogue<BLOCK_N, kPool, kHist>() && p.y_hi && !p.y_f32 && p.k_slices == 1 && !p.row_bias && !p.utt_bias &&
                p.Cout % 8 == 0;
  // Fused pooling: the full 8-frame time blocks' partials leave through one TMA store per tile (the kernel's map_y_hi).
  if (kPool) p.tma_store = p.Tb == 8;
  XVB_TL(if (g_timeline_direct) p.tma_store = 0;)
  if (kPool && p.tma_store) {
    if ((rc = make_partial_map(&pl.my_hi, p.pool_partial, p.Cout, p.B, p.num_t_blk))) return rc;
    pl.my_lo = pl.mw_lo;   // unused
  } else if (p.tma_store) {
    if ((rc = make_store_map(&pl.my_hi, p.y_hi, p.Cout, p.T, p.B, p.ldy, p.Tb))) return rc;
    if ((rc = make_store_map(&pl.my_lo, p.y_lo, p.Cout, p.T, p.B, p.ldy, p.Tb))) return rc;
  } else {
    pl.my_hi = pl.mw_hi; pl.my_lo = pl.mw_lo;  // unused
  }
  const int all_m_units = kHist ? (p.num_t_blk * p.num_b_blk + 1) / 2 : p.num_t_blk * p.num_b_blk;  // see unit_first
  if (p.unit_first >= all_m_units) { pl.launch = nullptr; return XVB_OK; }  // this shard owns no rows
  const int num_m_units = (all_m_units - p.unit_first + p.unit_stride - 1) / p.unit_stride;
  p.num_units = num_m_units;
  p.hist_group = 8;
  const long long tiles = kHist ? (long long)((2 * num_m_units + p.hist_group - 1) / p.hist_group) * p.hist_group * p.num_n_blk
                                : (long long)num_m_units * p.num_n_blk * (p.k_slices > 1 ? p.k_slices : 1);
  XVB_CHECK_ARG(tiles < (1ll << 31), "xvb_tdnn_affine: %d x %d tiles exceed one launch", num_m_units, p.num_n_blk);
  p.num_tiles = (int)tiles;
  p.out_T = p.k_slices > 1 ? p.k_slices : p.T;
  const int sms = sm_count();  // one CTA per SM
  pl.grid = p.num_tiles < sms ? p.num_tiles : sms;
  static const int pdl = getenv("XVB_PDL") ? atoi(getenv("XVB_PDL")) : 1;
  pl.pdl = pdl;
  pl.launch = &launch_inst<BLOCK_N, kPool, kHist, kSwish>;
  return XVB_OK;
}

// Split-K for segment-level layers (T == 1: M = B rows, tdnn6 has K = 3000): the slice count depends
// on K only, so a sub-batch reproduces the full batch's rows bit for bit.  Returns the number of slices (1 = off).
static int splitk_slices(const xvb_tdnn_args_t& a, bool has_hist, int* kb_per_slice) {
  const int num_cblk = (a.Cin + kBlockK - 1) / kBlockK;
  *kb_per_slice = num_cblk;
  const int splitk = getenv("XVB_SPLITK") ? atoi(getenv("XVB_SPLITK")) : 1;   // read per plan: tests flip it
  if (!(splitk && a.T == 1 && a.ntaps == 1 && !a.x2_hi && !a.pool_partial && !has_hist && !a.row_bias && !a.utt_bias &&
        !(a.flags & XVB_SWISH) && a.groups <= 1 &&
        a.B <= 1024 && num_cblk >= 24 && a.Cout % 4 == 0))
    return 1;
  int S = num_cblk / 6;
  S = S > 8 ? 8 : S;
  *kb_per_slice = (num_cblk + S - 1) / S;
  return (num_cblk + *kb_per_slice - 1) / *kb_per_slice;   // every slice owns >= 1 channel block
}

}  // namespace xvb

using namespace xvb;

size_t xvb::gemm_plan_scratch_bytes(const xvb_tdnn_args_t& a, const TrialHist* th) {
  int kb;
  const int S = splitk_slices(a, th != nullptr, &kb);
  return S > 1 ? (size_t)a.B * S * a.Cout * sizeof(float) : 0;
}

int xvb::gemm_plan_build(GemmPlan** out, const xvb_tdnn_args_t& a, const TrialHist* th, void* scratch) {
  int rc = require_sm90();
  if (rc) return rc;
  *out = nullptr;
  const int B = a.B, T = a.T, Cin = a.Cin, Cout = a.Cout, ntaps = a.ntaps;
  XVB_CHECK_ARG(a.x_hi && a.x_lo && a.w_hi && a.w_lo, "xvb_tdnn_affine: null operand pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && Cin > 0 && Cout > 0, "xvb_tdnn_affine: bad shape B=%d T=%d Cin=%d Cout=%d", B, T, Cin, Cout);
  XVB_CHECK_ARG(ntaps >= 1 && ntaps <= XVB_MAX_TAPS && a.context_host, "xvb_tdnn_affine: ntaps=%d out of range", ntaps);
  if (a.x_batch_stride)   // im2col view: overlapping rows
    XVB_CHECK_ARG(a.ldx % 8 == 0 && a.x_batch_stride % 8 == 0 && !a.x2_hi && ntaps == 1 &&
                  a.x_batch_stride >= (long long)(T - 1) * a.ldx + Cin,
                  "xvb_tdnn_affine: x_batch_stride=%lld needs ntaps==1, no second source, 8-element alignment and room for T windows",
                  (long long)a.x_batch_stride);
  else
    XVB_CHECK_ARG(a.ldx % 8 == 0 && a.ldx >= Cin, "xvb_tdnn_affine: ldx=%lld must be a multiple of 8 and >= Cin", (long long)a.ldx);
  XVB_CHECK_ARG((a.x2_hi != nullptr) == (a.x2_lo != nullptr), "xvb_tdnn_affine: x2_hi/x2_lo must both be set or both NULL");
  if (a.x2_hi) XVB_CHECK_ARG(a.ldx2 % 8 == 0 && a.ldx2 >= Cin, "xvb_tdnn_affine: ldx2=%lld must be a multiple of 8 and >= Cin", (long long)a.ldx2);
  XVB_CHECK_ARG((a.y_hi != nullptr) == (a.y_lo != nullptr), "xvb_tdnn_affine: y_hi/y_lo must both be set or both NULL");
  XVB_CHECK_ARG(a.y_hi || a.y_f32 || a.pool_partial || th, "xvb_tdnn_affine: no output requested");
  XVB_CHECK_ARG(!(a.flags & XVB_SWISH) || !(a.pool_partial || th), "xvb_tdnn_affine: XVB_SWISH is a layer-epilogue flag only");
  XVB_CHECK_ARG(!(a.lengths && (th || a.pool_partial)), "xvb_tdnn_affine: lengths apply to the layer epilogue only");
  if (a.pool_partial) XVB_CHECK_ARG(!a.y_hi && !a.y_f32 && Cout % 4 == 0 && (uintptr_t)a.pool_partial % 16 == 0,
                                    "xvb_tdnn_affine: pool_partial excludes other outputs and needs Cout%%4==0");
  if (a.y_hi) XVB_CHECK_ARG(a.ldy % 8 == 0 && a.ldy >= Cout, "xvb_tdnn_affine: plane output needs ldy%%8==0 and ldy>=Cout");
  if (a.y_f32) XVB_CHECK_ARG(a.ldyf % 4 == 0 && a.ldyf >= Cout, "xvb_tdnn_affine: fp32 output needs ldyf%%4==0 and ldyf>=Cout");
  XVB_CHECK_ARG(!(a.flags & XVB_BN) || (a.bn_scale && a.bn_shift), "xvb_tdnn_affine: XVB_BN without scale/shift");
  if (a.utt_bias) XVB_CHECK_ARG(a.ld_utt_bias % 4 == 0 && a.ld_utt_bias >= Cout && Cout % 4 == 0 && (uintptr_t)a.utt_bias % 16 == 0,
                                "xvb_tdnn_affine: utt_bias needs ld%%4==0, Cout%%4==0, 16-byte alignment");
  XVB_CHECK_ARG(((uintptr_t)a.x_hi | (uintptr_t)a.x_lo | (uintptr_t)a.x2_hi | (uintptr_t)a.x2_lo | (uintptr_t)a.w_hi |
                 (uintptr_t)a.w_lo | (uintptr_t)a.y_hi | (uintptr_t)a.y_lo | (uintptr_t)a.y_f32) % 16 == 0,
                "xvb_tdnn_affine: pointers must be 16-byte aligned");
  for (int i = 1; i < ntaps; ++i)
    XVB_CHECK_ARG(a.context_host[i] > a.context_host[i - 1], "xvb_tdnn_affine: context must be strictly increasing (components.py:34-36)");
  const int G = a.groups > 1 ? a.groups : 1;
  if (G > 1)
    XVB_CHECK_ARG(xvb_tdnn_grouped_fits(Cin, Cout, G) && ntaps == 1 && !a.x2_hi && !a.pool_partial && !th && !a.x_batch_stride &&
                  !(a.flags & XVB_SWISH),
                  "xvb_tdnn_affine: groups=%d needs Cin/groups %% 64 == 0, Cout/groups %% 32 == 0, one tap and no second source, "
                  "fused pooling, histogram, im2col view or XVB_SWISH (Cin=%d Cout=%d ntaps=%d)", G, Cin, Cout, ntaps);

  GemmPlan* plp = new GemmPlan();
  struct Guard { GemmPlan* p; ~Guard() { delete p; } } guard{plp};
  GemmPlan& pl = *plp;
  TdnnGemmParams& p = pl.p;
  p = TdnnGemmParams{};
  p.B = B; p.T = T; p.Cin = Cin; p.Cout = Cout;
  choose_m_tile(B, T, &p.Tb, &p.Bb);
  p.num_t_blk = (T + p.Tb - 1) / p.Tb;
  p.num_b_blk = (B + p.Bb - 1) / p.Bb;
  p.ntaps = ntaps;
  p.cin_p16 = (int)round_up(Cin / G, 16);        // weight K per tap: the group's slice (compact packing) when grouped
  p.num_cblk = (Cin / G + kBlockK - 1) / kBlockK;
  if (G > 1) { p.group_ng = Cout / G; p.group_kg = Cin / G; }
  for (int i = 0; i < ntaps; ++i) p.ctx[i] = a.context_host[i];
  p.flags = a.flags;
  p.bias = a.bias; p.scale = a.bn_scale; p.shift = a.bn_shift; p.row_bias = a.row_bias;
  p.utt_bias = a.utt_bias; p.ld_utt = a.ld_utt_bias;
  p.pool_partial = a.pool_partial;
  p.lengths = a.lengths;
  p.num_src = a.x2_hi ? 2 : 1;
  p.unit_first = 0; p.unit_stride = 1;
  if (th) {
    p.hist = th->hist; p.row_label = th->row_label; p.col_label = th->col_label;
    p.hist_lo = th->lo; p.hist_inv_w = th->inv_w; p.hist_bins = th->nbins; p.hist_sym = th->symmetric;
    p.unit_first = th->unit_first; p.unit_stride = th->unit_stride;
  }
  p.log2_tb = 0;
  while ((1 << p.log2_tb) < p.Tb) ++p.log2_tb;
  p.y_hi = reinterpret_cast<__nv_bfloat16*>(a.y_hi);
  p.y_lo = reinterpret_cast<__nv_bfloat16*>(a.y_lo);
  p.ldy = a.ldy; p.y_f32 = a.y_f32; p.ldyf = a.ldyf;

  XVB_TL(p.timeline = g_timeline; p.timeline_tiles = g_timeline_tiles; p.timeline_general = g_timeline_direct;)
  p.k_slices = splitk_slices(a, th != nullptr, &p.kb_per_slice);
  if (p.k_slices > 1) {
    XVB_CHECK_ARG(scratch, "xvb_tdnn_affine: split-K plan needs %zu bytes of scratch", gemm_plan_scratch_bytes(a, th));
    pl.reduce = true;
    pl.r_bias = a.bias; pl.r_scale = a.bn_scale; pl.r_shift = a.bn_shift; pl.r_flags = a.flags;
    pl.r_y_f32 = a.y_f32; pl.r_ldyf = a.ldyf;
    pl.r_y_hi = reinterpret_cast<__nv_bfloat16*>(a.y_hi); pl.r_y_lo = reinterpret_cast<__nv_bfloat16*>(a.y_lo); pl.r_ldy = a.ldy;
    p.y_hi = nullptr; p.y_lo = nullptr;
    p.y_f32 = static_cast<float*>(scratch); p.ldyf = Cout;
    p.bias = nullptr; p.scale = nullptr; p.shift = nullptr; p.flags = 0;
  }

  if ((rc = make_frame_map(&pl.ma_hi, a.x_hi, Cin, T, B, a.ldx, p.Tb, p.Bb, a.x_batch_stride))) return rc;
  if ((rc = make_frame_map(&pl.ma_lo, a.x_lo, Cin, T, B, a.ldx, p.Tb, p.Bb, a.x_batch_stride))) return rc;
  if (a.x2_hi) {
    if ((rc = make_frame_map(&pl.ma2_hi, a.x2_hi, Cin, T, B, a.ldx2, p.Tb, p.Bb))) return rc;
    if ((rc = make_frame_map(&pl.ma2_lo, a.x2_lo, Cin, T, B, a.ldx2, p.Tb, p.Bb))) return rc;
  } else {
    pl.ma2_hi = pl.ma_hi; pl.ma2_lo = pl.ma_lo;  // unused
  }

  // Wide N tiles when there are enough M tiles to fill the machine, narrow ones for the segment-level
  // layers (M = B rows) so that more SMs get a tile.
  const long long m_tiles = (long long)p.num_t_blk * p.num_b_blk * p.k_slices;   // independent work items along M (and K slices)
  const int sms = sm_count();
  const void* w_hi = a.w_hi;
  const void* w_lo = a.w_lo;
  auto dispatch = [&]() -> int {
    if (a.pool_partial)  // fused pooling always runs on the swapped kernel (any shape: TMA zero-fills)
      return prepare_gemm<128, true>(pl, w_hi, w_lo);
    if (th)              // the diagonal test of the symmetric mode assumes 128-row blocks x 128-column tiles
      return prepare_gemm<128, false, true>(pl, w_hi, w_lo);
    if (G > 1) {         // an N tile must not straddle two groups: the widest tile that divides the group's outputs
      const int ng = Cout / G;
      if (ng % 128 == 0) return prepare_gemm<128>(pl, w_hi, w_lo);
      if (ng % 64 == 0) return prepare_gemm<64>(pl, w_hi, w_lo);
      return prepare_gemm<32>(pl, w_hi, w_lo);
    }
    if (a.flags & XVB_SWISH) {
      if (Cout >= 128 && m_tiles * ((Cout + 127) / 128) >= sms) return prepare_gemm<128, false, false, true>(pl, w_hi, w_lo);
      if (Cout >= 64 && m_tiles * ((Cout + 63) / 64) >= sms / 2) return prepare_gemm<64, false, false, true>(pl, w_hi, w_lo);
      return prepare_gemm<32, false, false, true>(pl, w_hi, w_lo);
    }
    if (Cout >= 128 && m_tiles * ((Cout + 127) / 128) >= sms) return prepare_gemm<128>(pl, w_hi, w_lo);
    if (Cout >= 64 && m_tiles * ((Cout + 63) / 64) >= sms / 2) return prepare_gemm<64>(pl, w_hi, w_lo);
    return prepare_gemm<32>(pl, w_hi, w_lo);
  };
  if ((rc = dispatch())) return rc;
  guard.p = nullptr;
  *out = plp;
  return XVB_OK;
}

void xvb::gemm_plan_destroy(GemmPlan* pl) { delete pl; }

// Launch a plan.  `y_f32_override` (optional) redirects the fp32 output of this launch to another buffer of the
// same shape and pitch (the extractors' last layer writes straight into the caller's embedding matrix): for a
// split-K plan it is the reduce kernel's output, otherwise the GEMM's.
int xvb::gemm_plan_launch(const GemmPlan* plp, void* stream, float* y_f32_override) {
  const GemmPlan& pl = *plp;
  if (!pl.launch) return XVB_OK;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  int rc;
  if (!pl.reduce && y_f32_override && y_f32_override != pl.p.y_f32) {
    XVB_CHECK_ARG(pl.p.y_f32 && !pl.p.hist && !pl.p.pool_partial && (uintptr_t)y_f32_override % 16 == 0,
                  "gemm_plan_launch: this plan has no fp32 output to redirect");
    TdnnGemmParams p = pl.p;
    p.y_f32 = y_f32_override;
    return pl.launch(pl, p, s);
  }
  if ((rc = pl.launch(pl, pl.p, s))) return rc;
  if (!pl.reduce) return XVB_OK;
  float* yf = y_f32_override ? y_f32_override : pl.r_y_f32;
  const long long n = (long long)pl.p.B * pl.p.Cout;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3((unsigned)((n + 255) / 256));
  cfg.blockDim = dim3(256);
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  XVB_CUDA(cudaLaunchKernelEx(&cfg, segment_reduce_kernel, (const float*)pl.p.y_f32, pl.p.k_slices, pl.p.B, pl.p.Cout, pl.r_bias,
                              pl.r_scale, pl.r_shift, pl.r_flags, yf, pl.r_ldyf, pl.r_y_hi, pl.r_y_lo, pl.r_ldy));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

int xvb::tdnn_affine_impl(const xvb_tdnn_args_t& a, void* stream, const TrialHist* th) {
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  TempBuf partial(s);
  int rc;
  XVB_CHECK_ARG(a.B > 0 && a.Cin > 0 && a.Cout > 0, "xvb_tdnn_affine: bad shape B=%d Cin=%d Cout=%d", a.B, a.Cin, a.Cout);
  const size_t need = gemm_plan_scratch_bytes(a, th);
  if (need && (rc = partial.alloc(need))) return rc;
  GemmPlan* pl = nullptr;
  if ((rc = gemm_plan_build(&pl, a, th, partial.p))) return rc;
  rc = gemm_plan_launch(pl, stream, nullptr);
  gemm_plan_destroy(pl);
  return rc;
}

#ifdef XVB_TILE_TIMELINE
// Timeline build only: plans built from now on stamp into `buf` (device memory, gridDim x (8 + 8 x tiles_per_cta) u64,
// zeroed by the caller; NULL switches it off).  direct_stores != 0 keeps such plans on the direct-store layer epilogue
// and on the general path of the fused pooling epilogue, so that the old and new epilogues can be set side by side.
extern "C" void xvb_tile_timeline_set(unsigned long long* buf, int tiles_per_cta, int direct_stores) {
  g_timeline = buf;
  g_timeline_tiles = tiles_per_cta;
  g_timeline_direct = direct_stores != 0;
}
#endif

extern "C" int xvb_tdnn_grouped_fits(int Cin, int Cout, int groups) {
  return groups > 1 && Cin > 0 && Cout > 0 && Cin % groups == 0 && Cout % groups == 0 && (Cin / groups) % kBlockK == 0 &&
         (Cout / groups) % 32 == 0;
}

extern "C" int xvb_pool_partial_blocks(int B, int T, int* frames_per_block) {
  int Tb, Bb;
  choose_m_tile(B, T, &Tb, &Bb);
  if (frames_per_block) *frames_per_block = Tb;
  return (T + Tb - 1) / Tb;
}

extern "C" int xvb_tdnn_affine_ex(const xvb_tdnn_args_t* args, void* stream) {
  XVB_CHECK_ARG(args, "xvb_tdnn_affine_ex: null args");
  return tdnn_affine_impl(*args, stream);
}

extern "C" int xvb_tdnn_affine(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi,
                               const uint16_t* w_lo, const float* bias, const float* bn_scale, const float* bn_shift,
                               int flags, const int* context_host, int ntaps, uint16_t* y_hi, uint16_t* y_lo,
                               int64_t ldy, float* y_f32, int64_t ldyf, int B, int T, int Cin, int Cout,
                               void* stream) {
  xvb_tdnn_args_t a{};
  a.x_hi = x_hi; a.x_lo = x_lo; a.ldx = ldx; a.w_hi = w_hi; a.w_lo = w_lo;
  a.bias = bias; a.bn_scale = bn_scale; a.bn_shift = bn_shift; a.flags = flags;
  a.context_host = context_host; a.ntaps = ntaps;
  a.y_hi = y_hi; a.y_lo = y_lo; a.ldy = ldy; a.y_f32 = y_f32; a.ldyf = ldyf;
  a.B = B; a.T = T; a.Cin = Cin; a.Cout = Cout;
  return tdnn_affine_impl(a, stream);
}
