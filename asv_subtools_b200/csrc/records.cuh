// Device side of the native extractors' shared plumbing: the handle base, the packed split-bf16 planes and the arena
// that owns a model's device weights (every family), the packed affine layer and its layer-kernel arguments (every
// family), the grow-only workspace, the segment level of the 2-D families, the group loop of an extract call and the lengths check of a masked
// one.  The host records and the model-file codecs are host code in records.h.
#pragma once
#include <stdlib.h>

#include <memory>
#include <type_traits>
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
  // n host floats, or nothing (*d = NULL) when v is NULL or n is 0
  int upload(float** d, const float* v, size_t n) {
    if (!v || !n) { *d = nullptr; return XVB_OK; }
    int rc = alloc(d, n);
    if (rc) return rc;
    XVB_CUDA(cudaMemcpy(*d, v, n * sizeof(float), cudaMemcpyHostToDevice));
    return XVB_OK;
  }
  int upload(float** d, const std::vector<float>& v) { return upload(d, v.data(), v.size()); }
  // (Cout, Cin, tot) fp32 host -> newly allocated packed planes of the taps ctx[0..n).
  int pack(Planes* c, const std::vector<float>& w, int Cout, int Cin, int tot, const int* ctx, int n) {
    const size_t pn = (size_t)xvb_packed_weight_elems(Cout, Cin, n);
    int rc;
    if ((rc = alloc(&c->hi, pn)) || (rc = alloc(&c->lo, pn))) return rc;
    return pack_into(*c, w, Cout, Cin, tot, ctx, n);
  }
  // (Cout, Cin, tot) fp32 host -> the packed planes of the taps ctx[0..n) at c (ops.pack_tdnn_weight /
  // pack_conv2d_weight), xvb_packed_weight_elems(Cout, Cin, n) elements each.
  // xvb_pack_tdnn_weight takes at most XVB_MAX_TAPS taps per call: a longer list is packed in pieces of that many taps
  // (the last one shorter), each piece's rows then copied into its K range of every output row, as pack_conv2d_weight
  // concatenates the pieces along K.  Up to XVB_MAX_TAPS taps it is the one call straight into the planes.
  int pack_into(Planes c, const std::vector<float>& w, int Cout, int Cin, int tot, const int* ctx, int n) {
    float* w_dev = nullptr;
    XVB_CUDA(cudaMalloc((void**)&w_dev, w.size() * sizeof(float)));
    cudaError_t e = cudaMemcpy(w_dev, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice);
    const int left = ctx[0] < 0 ? ctx[0] : 0;
    const size_t pn = (size_t)xvb_packed_weight_elems(Cout, Cin, n);
    int rc = e != cudaSuccess ? XVB_ECUDA : XVB_OK;
    if (!rc && n <= XVB_MAX_TAPS) rc = xvb_pack_tdnn_weight(w_dev, Cout, Cin, tot, left, ctx, n, c.hi, c.lo, nullptr);
    Planes piece;
    if (!rc && n > XVB_MAX_TAPS) {
      const size_t tap = pn / ((size_t)Cout * n);   // packed elements of one tap in one output row (Cin padded to 16)
      const size_t bytes = (size_t)xvb_packed_weight_elems(Cout, Cin, XVB_MAX_TAPS) * sizeof(uint16_t);
      if (cudaMalloc((void**)&piece.hi, bytes) != cudaSuccess || cudaMalloc((void**)&piece.lo, bytes) != cudaSuccess) {
        set_error("%s: cudaMalloc of a packing piece failed", fn);
        rc = XVB_ECUDA;
      }
      for (int i = 0; i < n && !rc; i += XVB_MAX_TAPS) {
        const int m = n - i < XVB_MAX_TAPS ? n - i : XVB_MAX_TAPS;
        rc = xvb_pack_tdnn_weight(w_dev, Cout, Cin, tot, left, ctx + i, m, piece.hi, piece.lo, nullptr);
        const size_t dpitch = (size_t)n * tap * sizeof(uint16_t), spitch = (size_t)m * tap * sizeof(uint16_t);
        for (int p = 0; p < 2 && !rc; ++p) {
          uint16_t* dst = (p ? c.lo : c.hi) + (size_t)i * tap;
          const cudaError_t ce = cudaMemcpy2D(dst, dpitch, p ? piece.lo : piece.hi, spitch, spitch, (size_t)Cout,
                                              cudaMemcpyDeviceToDevice);
          if (ce != cudaSuccess) { set_error("%s: joining the packed pieces failed: %s", fn, cudaGetErrorString(ce)); rc = XVB_ECUDA; }
        }
      }
    }
    if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = XVB_ECUDA;
    if (rc == XVB_ECUDA && e != cudaSuccess) set_error("%s: weight upload failed: %s", fn, cudaGetErrorString(e));
    cudaFree(piece.hi); cudaFree(piece.lo);
    cudaFree(w_dev);
    return rc;
  }
};

// One affine layer on the wgmma layer kernel, in every family: its shape (Cout, Cin, the taps of ctx, the epilogue
// flags), packed weight, bias, scale and shift.  Cin and groups are what the kernel is called with: a compact grouped
// layer keeps its whole input width and its G groups, a block-diagonal expansion its whole input width and 1.
struct Affine : TapShape {
  Planes w;
  float* bias = nullptr;
  float* scale = nullptr;
  float* shift = nullptr;
  int groups = 1;
};

// L on the device: w (Cout, Cin / groups, tot) fp32 host over the taps ctx[0..ntaps) packed, and b, s, t uploaded (each
// empty when the layer has none).
inline int pack_affine(Weights& dev, Affine* L, const std::vector<float>& w, int Cout, int Cin, const int* ctx, int ntaps,
                       const std::vector<float>& b, const std::vector<float>& s, const std::vector<float>& t, int flags,
                       int groups = 1) {
  L->Cout = Cout; L->Cin = Cin; L->ntaps = ntaps; L->flags = flags; L->groups = groups;
  for (int i = 0; i < ntaps; ++i) L->ctx[i] = ctx[i];
  int rc;
  if ((rc = dev.pack(&L->w, w, Cout, Cin / groups, L->tot(), ctx, ntaps)) || (rc = dev.upload(&L->bias, b)) ||
      (rc = dev.upload(&L->scale, s)) || (rc = dev.upload(&L->shift, t)))
    return rc;
  return XVB_OK;
}
inline int pack_tap(Weights& dev, const TapRec& r, Affine* L) {
  return pack_affine(dev, L, r.w, r.Cout, r.Cin, r.ctx, r.ntaps, r.b, r.s, r.t, r.flags);
}

// The layer-kernel arguments of L over the planes x (row pitch ldx) at (B, T): input, weight, parameters, flags, taps,
// Cin, Cout and groups.  The caller sets what is its own: the outputs, and any utt_bias, x2, lengths, pool_partial,
// x_batch_stride or im2col view.
inline xvb_tdnn_args_t affine_args(const Affine& L, Planes x, int64_t ldx, int B, int T) {
  xvb_tdnn_args_t a{};
  a.x_hi = x.hi; a.x_lo = x.lo; a.ldx = ldx;
  a.w_hi = L.w.hi; a.w_lo = L.w.lo;
  a.bias = L.bias; a.bn_scale = L.scale; a.bn_shift = L.shift;
  a.flags = L.flags;
  a.context_host = L.ctx; a.ntaps = L.ntaps;
  a.B = B; a.T = T; a.Cin = L.Cin; a.Cout = L.Cout;
  a.groups = L.groups;
  return a;
}

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
  int* i32(int i) const { return (int*)buf[i][0]; }
  void release(int i) {
    cudaFree(buf[i][0]); cudaFree(buf[i][1]);
    buf[i][0] = buf[i][1] = nullptr;
    cap[i] = 0;
  }
  void free() { for (int i = 0; i < N; ++i) release(i); }
};

// The first layer of the TDNN and ECAPA-TDNN as an im2col view: a window of ntaps consecutive frames is one long row
// of planes padded with pad_front / pad_back zero frames around every utterance (7 channel blocks instead of 10 for
// [-2..2] x 80).  A model fixes it at finalize; each lane keeps a copy and turns it off for good if the driver refuses
// the overlapping tensor map.
struct Im2col {
  bool on = false;
  int pad_front = 0, pad_back = 0;
};

// Consecutive taps around 0, and feat_dim % 16 == 0 so that the plane pitch is the packed tap pitch.  XVB_IM2COL=0
// turns the view off; it is read for every model, not once per process, since tests flip it between models.
inline Im2col im2col_choice(const int* ctx, int ntaps, int feat_dim) {
  bool consecutive = ntaps > 1 && ctx[0] <= 0 && ctx[ntaps - 1] >= 0;
  for (int i = 1; i < ntaps; ++i) consecutive = consecutive && ctx[i] == ctx[i - 1] + 1;
  const int knob = getenv("XVB_IM2COL") ? atoi(getenv("XVB_IM2COL")) : 1;
  if (!knob || !consecutive || feat_dim % 16 != 0) return Im2col{};
  return Im2col{true, -ctx[0], ctx[ntaps - 1]};
}

// The segment level of the 2-D families (ResNet, RepVGG): statistics pooling of the last conv's fp32 (B, T', F' * C)
// output with planes out, then [fc1 ->] fc2 on the wgmma layer kernel at T = 1, each as ops.PackedAffine runs it.
struct SegTail {
  std::vector<Affine> seg;   // output rows padded to a multiple of 8
  int E = 0;     // the embedding dim, the last layer's real rows
  int mid = 0;   // the first layer's padded rows when there are two layers, else 0

  // Takes "fc1" / "fc2", as many as the extracted position hands over, the first one over `cin` pooled columns: each
  // record (Cout, Cin, 1) with a bias, scale / shift as XVB_BN and XVB_RELU as the layer applies them.  Pads the rows to
  // a multiple of 8 with zeros (the padded outputs are exact zeros) and packs them.  fn: the caller's name.
  int build(RecordStore& recs, Weights& dev, const char* fn, int cin) {
    for (const char* n : {"fc1", "fc2"}) {
      const Rec* s = recs.find(n);
      if (!s) continue;
      const int shape[3] = {s->shape[0], cin, 1};
      int rc = recs.take(fn, n, shape, &s);
      if (rc) return rc;
      E = s->shape[0];
      const int Cout = (E + 7) / 8 * 8;
      std::vector<float> w(s->w), b(s->b), sc(s->s), sh(s->t);
      w.resize((size_t)Cout * cin, 0.f);
      if (!b.empty()) b.resize(Cout, 0.f);
      if (!sc.empty()) { sc.resize(Cout, 0.f); sh.resize(Cout, 0.f); }
      const int flags = (s->flags & XVB_RELU) | (s->s.empty() ? 0 : XVB_BN);
      if ((rc = pack_affine(dev, &seg.emplace_back(), w, Cout, cin, kTaps, 1, b, sc, sh, flags))) return rc;
      cin = E;
    }
    XVB_CHECK_ARG(!seg.empty(), "%s: record 'fc1' or 'fc2' is missing (no segment layer)", fn);
    mid = seg.size() > 1 ? seg[0].Cout : 0;
    return XVB_OK;
  }
  int out_rows() const { return seg.back().Cout; }

  // last: the (B, T, pc) fp32 output of the last conv -> emb (B, E).  Buffers per utterance: pooled planes and
  // pooled_f32 of 2 * pc, mid planes of `mid` and out of out_rows() (used when the last layer is padded).  lengths:
  // NULL, or a masked batch's frame counts at the last conv's resolution (device int32[B]), each pooling its own.
  int run(const float* last, int pc, int B, int T, float eps, Planes pooled, float* pooled_f32, Planes mid_planes,
          float* out, float* emb, void* stream, const int* lengths = nullptr) const {
    int rc;
    if ((rc = stats_pool(last, pc, B, T, pc, eps, 0, lengths, pooled_f32, pooled.hi, pooled.lo, 2 * pc, stream))) return rc;
    Planes x = pooled;
    int64_t ldx = 2 * pc;
    for (size_t j = 0; j < seg.size(); ++j) {
      const Affine& s = seg[j];
      xvb_tdnn_args_t a = affine_args(s, x, ldx, B, 1);
      if (j + 1 == seg.size()) { a.y_f32 = s.Cout == E ? emb : out; a.ldyf = s.Cout; }
      else { a.y_hi = mid_planes.hi; a.y_lo = mid_planes.lo; a.ldy = s.Cout; }
      if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
      x = mid_planes; ldx = s.Cout;
    }
    const Affine& s = seg.back();
    if (s.Cout != E)
      XVB_CUDA(cudaMemcpy2DAsync(emb, (size_t)E * sizeof(float), out, (size_t)s.Cout * sizeof(float), (size_t)E * sizeof(float),
                                 (size_t)B, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return XVB_OK;
  }
};

// The part of a native extractor handle that is not workspace or per-lane state.  From create until finalize succeeds
// the handle is a draft: set_layer / add_*_layer write `draft`, the model that `m` owns, so that getters read drafts and
// finalized handles alike.  Once finalized, the model is immutable and shared by the handle and its second shard lane.
template <typename Model>
struct Handle {
  std::shared_ptr<const Model> m;
  Model* draft = nullptr;
  int last_launches = 0;

  Handle() { auto d = std::make_shared<Model>(); draft = d.get(); m = std::move(d); }
  explicit Handle(std::shared_ptr<const Model> model) : m(std::move(model)) {}   // a lane on a finalized model
};

template <typename Model> bool finalized(const Handle<Model>* h) { return h && !h->draft; }
template <typename Model> bool is_draft(const Handle<Model>* h) { return h && h->draft; }

// The finalize of every family (fn: its name): build(fresh, records) makes a new model from the draft's configuration
// and records, and only a model built without error is published, the records moved into it for save and the getters.
// A failed build is discarded with its device weights and the draft keeps its records, so that the caller can add what
// was missing and finalize again.
template <typename Model, typename Build>
int publish_built(Handle<Model>* h, Build build, const char* fn) {
  XVB_CHECK_ARG(is_draft(h), "%s: null or finalized model", fn);
  auto fresh = std::make_shared<Model>();
  fresh->cfg = h->draft->cfg;
  if constexpr (std::is_same_v<decltype(h->draft->recs), RecordStore>) h->draft->recs.used.clear();
  int rc = build(fresh.get(), h->draft->recs);
  if (rc) return rc;
  fresh->recs = std::move(h->draft->recs);
  h->m = std::move(fresh);
  h->draft = nullptr;
  return XVB_OK;
}

// The host lengths of a masked call: each in [min_len, T], or XVB_EINVAL naming the first that is not (fn: the caller's
// name).  *all_T: every utterance is T frames long, so that there is nothing to mask.
inline int check_lengths(const char* fn, const int32_t* lengths_host, int B, int T, bool* all_T, int min_len = 1) {
  *all_T = true;
  for (int b = 0; b < B; ++b) {
    XVB_CHECK_ARG(lengths_host[b] >= min_len && lengths_host[b] <= T, "%s: lengths[%d]=%d outside [%d, T=%d]", fn, b,
                  (int)lengths_host[b], min_len, T);
    *all_T = *all_T && lengths_host[b] == T;
  }
  return XVB_OK;
}

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
