// Speaker retrieval (recipe/cnsrc/sr/run-cnsrc_sr.sh stage 4): the k best test utterances of every enrolled speaker.
// The reference scores every (speaker, test utterance) pair into a text file and ranks it with pandas
// (trans_score_format.py: groupby('spk-id').nlargest(10, 'scores')).  Here the score matrix is produced slab by slab
// by xvb_matmul_nt into one reused buffer, and topk_merge_kernel folds each slab into a running per-row list, so
// neither the M x N matrix nor a score file ever exists.
//
// Order: higher score first; equal scores by lower column index -- nlargest(keep='first') over a score file in
// trials order (getTrials.sh 1 lists the speakers of one test utterance together), and topn_index_kernel's rule.
//
// topk_merge_kernel: one CTA of 256 threads per row.  The row's list (k <= 256 pairs) and a candidate buffer share
// one 4096-pair shared-memory array.  Each round reads 2048 columns (two coalesced float4 per thread) and compares
// them with the list's k-th entry; a column that does not beat it is dropped right there.  Survivors are appended
// with one warp ballot and one shared atomic per warp.  When the next round could overflow the array, the list and
// the candidates are bitonic-sorted together (size padded to a power of two with empty slots) and the first k kept.
// After the first few rounds the k-th score is high, almost every column is dropped, and the kernel streams the
// slab at memory speed.  Empty slots are (-inf, index 0xffffffff) in shared memory and sort after every real column,
// including a real -inf score; they leave the kernel as (-inf, -1).
#include <cuda_runtime.h>

#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace xvb {

constexpr int kMergeThreads = 256;
constexpr int kMergeVec = 8;                              // columns per thread per round: two float4
constexpr int kMergeRound = kMergeThreads * kMergeVec;    // 2048 columns per round
constexpr int kMergeCap = 4096;                           // list + candidates, in (score, index) pairs
constexpr uint32_t kEmpty = 0xffffffffu;
static_assert(kMergeCap - 256 - kMergeRound >= 0, "a round must fit after the largest list");

__device__ __forceinline__ bool ranks_before(float a, uint32_t ia, float b, uint32_t ib) {
  return a > b || (a == b && ia < ib);
}

// Bitonic sort of ss/si[0, P) into ranking order; [n, P) is filled with empty slots first.
__device__ void merge_sort(float* ss, uint32_t* si, int n) {
  int P = 1;
  while (P < n) P <<= 1;
  for (int t = n + threadIdx.x; t < P; t += blockDim.x) { ss[t] = -INFINITY; si[t] = kEmpty; }
  __syncthreads();
  for (int kk = 2; kk <= P; kk <<= 1) {
    for (int j = kk >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const float a = ss[i], b = ss[ixj];
          const uint32_t ia = si[i], ib = si[ixj];
          const bool a_first = ranks_before(a, ia, b, ib);
          if (((i & kk) == 0) ? !a_first : a_first) { ss[i] = b; ss[ixj] = a; si[i] = ib; si[ixj] = ia; }
        }
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(kMergeThreads) topk_merge_kernel(const float* __restrict__ S, long long lds, int ncols,
                                                                    long long col0, int k, float* __restrict__ top_s,
                                                                    long long* __restrict__ top_i,
                                                                    unsigned long long* __restrict__ nan_row) {
  __shared__ float ss[kMergeCap];
  __shared__ uint32_t si[kMergeCap];
  __shared__ int count;
  const long long row = blockIdx.x;
  const float* src = S + row * lds;
  float* ls = top_s + row * k;
  long long* li = top_i + row * k;
  for (int t = threadIdx.x; t < k; t += blockDim.x) {
    ss[t] = ls[t];
    si[t] = li[t] < 0 ? kEmpty : (uint32_t)li[t];
  }
  if (threadIdx.x == 0) count = 0;
  __syncthreads();
  float thr = ss[k - 1];
  uint32_t thr_i = si[k - 1];
  const int lane = threadIdx.x & 31;
  const uint32_t below = (1u << lane) - 1u;
  bool saw_nan = false;
  for (int base = 0; base < ncols; base += kMergeRound) {
    float v[kMergeVec];
    int col[kMergeVec / 4];
#pragma unroll
    for (int j = 0; j < kMergeVec / 4; ++j) {
      col[j] = base + (j * kMergeThreads + (int)threadIdx.x) * 4;
      float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
      if (col[j] < ncols) f = __ldcs(reinterpret_cast<const float4*>(src + col[j]));   // lds % 4 == 0: in the row
      v[4 * j] = f.x; v[4 * j + 1] = f.y; v[4 * j + 2] = f.z; v[4 * j + 3] = f.w;
    }
    bool keep[kMergeVec];
    bool any = false;
#pragma unroll
    for (int e = 0; e < kMergeVec; ++e) {
      const int c = col[e / 4] + (e & 3);
      const bool valid = c < ncols;
      saw_nan |= valid && isnan(v[e]);
      keep[e] = valid && ranks_before(v[e], (uint32_t)(col0 + c), thr, thr_i);
      any |= keep[e];
    }
    if (__any_sync(0xffffffffu, any)) {
#pragma unroll
      for (int e = 0; e < kMergeVec; ++e) {
        const unsigned m = __ballot_sync(0xffffffffu, keep[e]);
        if (!m) continue;
        const int leader = __ffs(m) - 1;
        int pos = 0;
        if (lane == leader) pos = atomicAdd(&count, __popc(m));
        pos = __shfl_sync(0xffffffffu, pos, leader);
        if (keep[e]) {
          const int o = k + pos + __popc(m & below);
          ss[o] = v[e];
          si[o] = (uint32_t)(col0 + col[e / 4] + (e & 3));
        }
      }
    }
    __syncthreads();
    const int n = count;
    // Every thread must have read `count` before any warp appends to it in the next round: the merge decision below
    // has to be the same in the whole CTA, or its barriers would pair with the next round's.
    __syncthreads();
    if (n > kMergeCap - k - kMergeRound || (n > 0 && base + kMergeRound >= ncols)) {
      merge_sort(ss, si, k + n);
      thr = ss[k - 1];
      thr_i = si[k - 1];
      if (threadIdx.x == 0) count = 0;
      __syncthreads();
    }
  }
  for (int t = threadIdx.x; t < k; t += blockDim.x) {
    ls[t] = ss[t];
    li[t] = si[t] == kEmpty ? -1ll : (long long)si[t];
  }
  if (__syncthreads_or(saw_nan) && threadIdx.x == 0) atomicMin(nan_row, (unsigned long long)row);
}

// *bad = the lowest row of x (rows, K) or term (rows) holding a NaN or an infinity (atomicMin; *bad starts at ~0).
__global__ void nonfinite_rows_kernel(const float* __restrict__ x, long long rows, int K, const float* __restrict__ term,
                                      unsigned long long* __restrict__ bad) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long first = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  for (long long t = first; t < rows * K; t += stride)
    if (!isfinite(x[t])) atomicMin(bad, (unsigned long long)(t / K));
  if (term)
    for (long long t = first; t < rows; t += stride)
      if (!isfinite(term[t])) atomicMin(bad, (unsigned long long)t);
}

__global__ void topk_init_kernel(float* __restrict__ s, long long* __restrict__ i, long long n) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
    s[t] = -INFINITY;
    i[t] = -1;
  }
}

}  // namespace xvb

using namespace xvb;

extern "C" int xvb_topk_merge(const float* S, int64_t lds, int64_t rows, int64_t ncols, int64_t col0, int k, float* top_score,
                              int64_t* top_idx, uint64_t* nan_row, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(S && top_score && top_idx && nan_row && rows > 0 && ncols > 0 && col0 >= 0, "xvb_topk_merge: bad arguments");
  XVB_CHECK_ARG(k >= 1 && k <= 256, "xvb_topk_merge: k=%d outside [1, 256]", k);
  XVB_CHECK_ARG(lds % 4 == 0 && lds >= ncols && (uintptr_t)S % 16 == 0,
                "xvb_topk_merge: lds must be a multiple of 4 and >= ncols, S 16-byte aligned");
  XVB_CHECK_ARG(rows < (1ll << 31) && col0 + ncols <= INT32_MAX, "xvb_topk_merge: more than 2^31 - 1 rows or columns");
  topk_merge_kernel<<<(unsigned)rows, kMergeThreads, 0, (cudaStream_t)stream>>>(
      S, lds, (int)ncols, col0, k, top_score, reinterpret_cast<long long*>(top_idx),
      reinterpret_cast<unsigned long long*>(nan_row));
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" int64_t xvb_retrieve_topk_slab_bytes(int64_t M, int64_t slab_cols) {
  XVB_CHECK_ARG(M > 0 && M < (1ll << 31) && slab_cols >= 4 && slab_cols % 4 == 0 && slab_cols <= INT32_MAX - 3 &&
                    M <= (1ll << 60) / 4 / slab_cols,
                "xvb_retrieve_topk_slab_bytes: M=%lld, slab_cols=%lld (a positive multiple of 4)", (long long)M,
                (long long)slab_cols);
  return M * slab_cols * (int64_t)sizeof(float);
}

extern "C" int xvb_retrieve_topk(const float* a, int64_t M, const float* b, int64_t N, int K, const float* row_bias,
                                 const float* col_bias, int k, float* slab, int64_t slab_cols, float* out_score,
                                 int64_t* out_idx, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(a && b && slab && out_score && out_idx && M > 0 && N > 0 && K > 0, "xvb_retrieve_topk: bad arguments");
  XVB_CHECK_ARG(k >= 1 && k <= 256, "xvb_retrieve_topk: k=%d outside [1, 256]", k);
  XVB_CHECK_ARG(M < (1ll << 31) && N <= INT32_MAX, "xvb_retrieve_topk: more than 2^31 - 1 enroll or test rows");
  XVB_CHECK_ARG(xvb_retrieve_topk_slab_bytes(M, slab_cols) > 0 && (uintptr_t)slab % 16 == 0,
                "xvb_retrieve_topk: slab_cols=%lld must be a positive multiple of 4 and the slab 16-byte aligned",
                (long long)slab_cols);
  cudaStream_t s = (cudaStream_t)stream;
  // The running lists live in scratch until every slab is merged and checked for NaN: a refused call writes nothing.
  TempBuf lists(s), pad(s);
  const long long nk = (long long)M * k;
  // flags[0]: first row with a NaN score; flags[1] / [2]: first enroll / test row with a non-finite operand or term
  if ((rc = lists.alloc(3 * sizeof(unsigned long long) + (size_t)nk * (sizeof(long long) + sizeof(float))))) return rc;
  unsigned long long* flags = (unsigned long long*)lists.p;
  long long* list_i = (long long*)(flags + 3);
  float* list_s = (float*)(list_i + nk);
  const unsigned grid = (unsigned)sm_count() * 8;
  topk_init_kernel<<<(unsigned)std::min<long long>((nk + 255) / 256, grid), 256, 0, s>>>(list_s, list_i, nk);
  XVB_LAUNCH_CHECK();
  XVB_CUDA(cudaMemsetAsync(flags, 0xff, 3 * sizeof(unsigned long long), s));
  // The layer epilogue applies its ReLU switch branch-free, as fmaxf(x, -inf), which turns a NaN accumulator into
  // -inf: a NaN or infinite operand would be ranked as -inf instead of refused.  So the operands are checked here.
  nonfinite_rows_kernel<<<grid, 256, 0, s>>>(a, M, K, row_bias, flags + 1);
  XVB_LAUNCH_CHECK();
  nonfinite_rows_kernel<<<grid, 256, 0, s>>>(b, N, K, col_bias, flags + 2);
  XVB_LAUNCH_CHECK();
  // xvb_matmul_nt takes N % 4 == 0: the last 1..3 test rows (and their column terms) are scored from a zero-padded copy.
  float* pad_b = nullptr;
  float* pad_col = nullptr;
  if (N % 4) {
    if ((rc = pad.alloc((size_t)(4 * K + 4) * sizeof(float)))) return rc;
    pad_b = (float*)pad.p;
    pad_col = pad_b + 4 * (size_t)K;
    const int64_t r0 = N & ~3ll;
    XVB_CUDA(cudaMemsetAsync(pad_b, 0, (size_t)(4 * K + 4) * sizeof(float), s));
    XVB_CUDA(cudaMemcpyAsync(pad_b, b + r0 * K, (size_t)(N - r0) * K * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (col_bias) XVB_CUDA(cudaMemcpyAsync(pad_col, col_bias + r0, (size_t)(N - r0) * sizeof(float), cudaMemcpyDeviceToDevice, s));
  }
  for (int64_t c0 = 0; c0 < N; c0 += slab_cols) {
    const int64_t n = std::min<int64_t>(slab_cols, N - c0);
    const int64_t n4 = n & ~3ll;
    if (n4 && (rc = xvb_matmul_nt(a, M, b + c0 * K, n4, K, row_bias, col_bias ? col_bias + c0 : nullptr, slab, slab_cols, s)))
      return rc;
    if (n4 < n && (rc = xvb_matmul_nt(a, M, pad_b, 4, K, row_bias, col_bias ? pad_col : nullptr, slab + n4, slab_cols, s)))
      return rc;
    if ((rc = xvb_topk_merge(slab, slab_cols, M, n, c0, k, list_s, (int64_t*)list_i, (uint64_t*)flags, s))) return rc;
  }
  unsigned long long first[3];
  XVB_CUDA(cudaMemcpyAsync(first, flags, sizeof(first), cudaMemcpyDeviceToHost, s));
  XVB_CUDA(cudaStreamSynchronize(s));
  XVB_CHECK_ARG(first[1] == ~0ull, "xvb_retrieve_topk: NaN or infinity in enroll row %llu (a or row_bias)", first[1]);
  XVB_CHECK_ARG(first[2] == ~0ull, "xvb_retrieve_topk: NaN or infinity in test row %llu (b or col_bias)", first[2]);
  XVB_CHECK_ARG(first[0] == ~0ull, "xvb_retrieve_topk: NaN score in row %llu", first[0]);
  XVB_CUDA(cudaMemcpyAsync(out_score, list_s, (size_t)nk * sizeof(float), cudaMemcpyDeviceToDevice, s));
  XVB_CUDA(cudaMemcpyAsync(out_idx, list_i, (size_t)nk * sizeof(long long), cudaMemcpyDeviceToDevice, s));
  return XVB_OK;
}
