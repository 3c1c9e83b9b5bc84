// Device side of the ResNet, Conformer and CAM++ native extractors' shared plumbing: the packed split-bf16 planes, the
// arena that owns a model's device weights, the grow-only workspace and the group loop of an extract call.  The record
// store and the model-file codec are host code in records.h.
#pragma once
#include <vector>

#include "common.cuh"
#include "records.h"

namespace xvb {

struct Planes { uint16_t* hi = nullptr; uint16_t* lo = nullptr; };

// Every device allocation of one model's weights, freed with it.  `fn` prefixes pack's upload error.
struct Weights {
  explicit Weights(const char* fn) : fn(fn) {}
  ~Weights() { for (void* p : dev) cudaFree(p); }
  const char* fn;
  std::vector<void*> dev;

  template <typename T>
  int alloc(T** p, size_t n) {
    XVB_CUDA(cudaMalloc((void**)p, (n ? n : 1) * sizeof(T)));
    dev.push_back(*p);
    return XVB_OK;
  }
  int upload(float** d, const std::vector<float>& v) {
    if (v.empty()) { *d = nullptr; return XVB_OK; }
    int rc = alloc(d, v.size());
    if (rc) return rc;
    XVB_CUDA(cudaMemcpy(*d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
    return XVB_OK;
  }
  // (Cout, Cin, tot) fp32 host -> packed planes of the taps ctx[0..n) (ops.pack_tdnn_weight / pack_conv2d_weight)
  int pack(Planes* c, const std::vector<float>& w, int Cout, int Cin, int tot, const int* ctx, int n) {
    float* w_dev = nullptr;
    XVB_CUDA(cudaMalloc((void**)&w_dev, w.size() * sizeof(float)));
    cudaError_t e = cudaMemcpy(w_dev, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice);
    const int left = ctx[0] < 0 ? ctx[0] : 0;
    const size_t pn = (size_t)xvb_packed_weight_elems(Cout, Cin, n);
    int rc = e != cudaSuccess ? XVB_ECUDA : XVB_OK;
    if (!rc) rc = alloc(&c->hi, pn);
    if (!rc) rc = alloc(&c->lo, pn);
    if (!rc) rc = xvb_pack_tdnn_weight(w_dev, Cout, Cin, tot, left, ctx, n, c->hi, c->lo, nullptr);
    if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = XVB_ECUDA;
    if (rc == XVB_ECUDA && e != cudaSuccess) set_error("%s: weight upload failed: %s", fn, cudaGetErrorString(e));
    cudaFree(w_dev);
    return rc;
  }
};

// taps 0 .. n-1 of a weight packed over its whole span
constexpr int kTaps[9] = {0, 1, 2, 3, 4, 5, 6, 7, 8};

// N enum-indexed buffers, each grown to the largest call seen: fp32, or the hi and lo bf16 planes where planes[i].
template <int N>
struct Workspace {
  static_assert(N <= 64, "reserve reports reallocations as a 64-bit mask");
  size_t cap[N] = {0};
  void* buf[N][2] = {{nullptr}};   // [0]: fp32 or the hi plane, [1]: the lo plane

  ~Workspace() { free(); }
  // Grows buffer i to need[i] elements; bit i of *grown is set when buffer i was reallocated (its contents are lost).
  int reserve(const size_t (&need)[N], const bool (&planes)[N], uint64_t* grown) {
    *grown = 0;
    for (int i = 0; i < N; ++i) {
      if (need[i] <= cap[i]) continue;
      release(i);
      *grown |= 1ull << i;
      const size_t bytes = need[i] * (planes[i] ? sizeof(uint16_t) : sizeof(float));
      XVB_CUDA(cudaMalloc(&buf[i][0], bytes));
      if (planes[i]) XVB_CUDA(cudaMalloc(&buf[i][1], bytes));
      cap[i] = need[i];
    }
    return XVB_OK;
  }
  Planes planes(int i) const { return {(uint16_t*)buf[i][0], (uint16_t*)buf[i][1]}; }
  float* f32(int i) const { return (float*)buf[i][0]; }
  void release(int i) {
    cudaFree(buf[i][0]); cudaFree(buf[i][1]);
    buf[i][0] = buf[i][1] = nullptr;
    cap[i] = 0;
  }
  void free() { for (int i = 0; i < N; ++i) release(i); }
};

// One extract call as groups of floor(budget / per_utt) utterances (at least one): run(first, count) per group.
template <typename Run>
int for_groups(int B, long long per_utt, long long budget, Run run) {
  int g = (int)(budget / per_utt);
  if (g < 1) g = 1;
  for (int i = 0; i < B; i += g) {
    int rc = run(i, B - i < g ? B - i : g);
    if (rc) return rc;
  }
  return XVB_OK;
}

}  // namespace xvb
