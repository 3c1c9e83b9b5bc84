// Whole-model extractor for the TDNN x-vector family: frame-level TDNN layers -> statistics
// pooling -> segment-level affine layers.  Owns packed weights and workspace on the current device.
// Stands in for Xvector.extract_embedding (pytorch/model/xvector.py:77-98) on a whole batch of
// equal-length utterances and for the "load weights, run extraction without Python" role of the
// reference's C++ runtime (runtime/bin/extractor_main.cc, runtime/speaker/torch_asv_model.cc).
// With xvb_extractor_set_attention_pooling the pooling is an attention tail instead (the snowdar x-vector's attentive,
// multi-head and multi-resolution poolings and the xi-vector): the launch sequence of nnet/framework.py's
// AttentionPoolingExtractor, kernel for kernel, so that the embeddings are that sequence's bit for bit.
#include <cuda_runtime.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <memory>
#include <tuple>
#include <vector>

#include "records.cuh"
#include "shard.cuh"

// The model types are local to this file: each family has its own Model.
namespace {

using namespace xvb;

// B * T frames per group of an attention model's extract call: larger calls run as consecutive groups (xvb200.h)
constexpr long long kAttnFrameBudget = 256LL * 300;

struct Config {
  int feat_dim = 0, ldf = 0;
  // the pooling: 0 statistics, else XVB_POOL_ATTENTION / _XI_POSTMEAN / _XI_POSTDIST with its pooled channels O, logit
  // divisor, unweighted variance and (xi-vector) prior, as xvb_extractor_set_attention_pooling took them
  int pool_kind = 0, pooled = 0, gdiv = 1, unweighted = 0;
  std::vector<float> prior_logprec, prior_mean;
  bool attention() const { return pool_kind != 0; }
  bool xi() const { return pool_kind == XVB_POOL_XI_POSTMEAN || pool_kind == XVB_POOL_XI_POSTDIST; }
  // columns of the pooled statistics (and their planes' pitch), and the first segment layer's input width
  int stats_width(int c_last) const { return attention() ? 2 * pooled : 2 * c_last; }
  int segment_in(int c_last) const { return pool_kind == XVB_POOL_XI_POSTMEAN ? pooled : stats_width(c_last); }
};

// as handed over, in order; attention: an attention model's [first affine,] last affine
struct Layers { std::vector<TapRec> frame, attention, segment; };

// The layers and what finalize fixes; shared read-only by a handle and its second shard lane once finalized.
struct Model {
  Config cfg;
  Layers recs;
  float pooling_eps = 1e-10f;
  // recs on the device, built at finalize; an attention model's last frame layer, attention and segment layers with
  // their output rows zero-padded to a multiple of 8, as the Python sequence packs them (ops.PackedAffine pad_to=8)
  std::vector<Affine> frame, attention, segment;
  int max_c = 0, max_seg_c = 0;
  int embed = 0;   // the embedding dim: the last segment layer's own rows
  float *prior_logprec = nullptr, *prior_mean = nullptr;   // the xi-vector's prior on the device
  Im2col im2col;   // the first layer as an im2col view (records.cuh)
  Weights dev{"xvb_extractor_finalize"};
};

// Everything one (B, T) batch shape needs besides launches: a GemmPlan per layer (tensor maps over the
// extractor's own workspace, tile geometry, kernel instantiation) and the split-K scratch those plans own.
struct StepPlan {
  std::vector<GemmPlan*> frame, attention, segment;
  std::vector<void*> scratch;
  int pool_blocks = 0, pool_tb = 0;
  ~StepPlan() {
    for (GemmPlan* g : frame) gemm_plan_destroy(g);
    for (GemmPlan* g : attention) gemm_plan_destroy(g);
    for (GemmPlan* g : segment) gemm_plan_destroy(g);
    for (void* q : scratch) cudaFree(q);
  }
};

}  // namespace

using namespace xvb;

struct xvb_extractor : Handle<Model> {
  // workspace, each buffer grown to the largest call seen: the input planes (B, pad_front + T + pad_back, ldf), the
  // ping-pong activations (B, T, max_c), the last frame layer's fp32 output (B, T, C_last), the pooled statistics
  // (B, 2 C_last) in fp32, the nominal target of the last segment layer's plan (B, D), the pooled statistics as planes,
  // the segment ping-pong (B, max_seg_c), the partials of the fused pooling epilogue (time blocks, B, 2 C_last) and the
  // per-utterance frame counts of a masked call (xvb_extractor_extract_lengths); an attention model's fp32 logits
  // (B, T, G) (its last frame layer and first attention affine write their planes into the ping-pong activations)
  enum { kIn, kAct0, kAct1, kLast, kStats, kEmb, kStatsPlanes, kSeg0, kSeg1, kPoolPartial, kLengths, kLogits, kBufs };
  Workspace<kBufs> ws;
  bool fused_pooling = true;
  Im2col im2col;   // this lane's copy of the model's choice
  // launch plans per batch shape (B, T, masked); they hold workspace addresses, so a reserve that reallocates clears them
  std::map<std::tuple<int, int, bool>, StepPlan*> plans;
  // optional per-kernel CUDA-event timing on the launching stream (bench.py roofline)
  bool profiling = false;
  bool in_shard = false;
  std::vector<cudaEvent_t> events;
  int events_used = 0;
  cudaStream_t events_stream = nullptr;
  Shard<xvb_extractor> shard;

  xvb_extractor() = default;
  explicit xvb_extractor(std::shared_ptr<const Model> model) : Handle(std::move(model)), im2col(m->im2col) {}
  ~xvb_extractor() {
    drop_plans();
    for (cudaEvent_t e : events) cudaEventDestroy(e);
  }

  void drop_plans() {
    for (auto& kv : plans) delete kv.second;
    plans.clear();
  }

  int mark(cudaStream_t s) {
    if (!profiling) return XVB_OK;
    if (events_used == (int)events.size()) {
      cudaEvent_t e;
      XVB_CUDA(cudaEventCreate(&e));
      events.push_back(e);
    }
    XVB_CUDA(cudaEventRecord(events[events_used++], s));
    return XVB_OK;
  }
};

using H = xvb_extractor;

template <>
struct xvb::ShardFamily<xvb_extractor> {
  static int extract(xvb_extractor* h, const float* feats, int B, int T, float* emb, void* stream) {
    return xvb_extractor_extract(h, feats, B, T, emb, stream);
  }
  static xvb_extractor* twin(const xvb_extractor* h) {
    xvb_extractor* c = new xvb_extractor(h->m);
    c->fused_pooling = h->fused_pooling;
    return c;
  }
  static int feat_dim(const xvb_extractor* h) { return h->m->cfg.feat_dim; }
  static int embed_dim(const xvb_extractor* h) { return h->m->embed; }
};

static int add_layer(std::vector<TapRec>& dst, int Cin, int Cout, const int* ctx, int ntaps, const float* w_host,
                     const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(ntaps >= 1 && ntaps <= XVB_MAX_TAPS && ctx && w_host, "add layer: bad taps/weights");
  XVB_CHECK_ARG(!(flags & XVB_BN) || (scale_host && shift_host), "add layer: XVB_BN without scale/shift");
  for (int i = 1; i < ntaps; ++i) XVB_CHECK_ARG(ctx[i] > ctx[i - 1], "add layer: context must be strictly increasing");
  dst.push_back(tap_record("", Cout, Cin, ctx, ntaps, w_host, bias_host, scale_host, shift_host, flags));
  return XVB_OK;
}

extern "C" int xvb_extractor_create(xvb_extractor_t** out, int feat_dim) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && feat_dim > 0, "xvb_extractor_create: bad arguments");
  xvb_extractor* h = new xvb_extractor();
  h->draft->cfg.feat_dim = feat_dim;
  h->draft->cfg.ldf = (int)round_up(feat_dim, 8);
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_extractor_add_frame_layer(xvb_extractor_t* h, int Cout, const int* context_host, int ntaps,
                                             const float* w_host, const float* bias_host, const float* bn_scale_host,
                                             const float* bn_shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h), "xvb_extractor_add_frame_layer: null or finalized extractor");
  Layers& r = h->draft->recs;
  XVB_CHECK_ARG(r.segment.empty(), "xvb_extractor_add_frame_layer: frame layers must precede segment layers");
  const int Cin = r.frame.empty() ? h->draft->cfg.feat_dim : r.frame.back().Cout;
  return add_layer(r.frame, Cin, Cout, context_host, ntaps, w_host, bias_host, bn_scale_host, bn_shift_host, flags);
}

extern "C" int xvb_extractor_set_attention_pooling(xvb_extractor_t* h, int kind, int pooled, int gdiv, int unweighted_var,
                                                   const float* prior_logprec_host, const float* prior_mean_host) {
  const char* fn = "xvb_extractor_set_attention_pooling";
  XVB_CHECK_ARG(is_draft(h) && h->draft->recs.frame.empty() && !h->draft->cfg.attention(),
                "%s: call it once on a draft extractor, before its first layer", fn);
  const bool xi = kind == XVB_POOL_XI_POSTMEAN || kind == XVB_POOL_XI_POSTDIST;
  XVB_CHECK_ARG(kind == XVB_POOL_ATTENTION || xi,
                "%s: kind %d is not XVB_POOL_ATTENTION, XVB_POOL_XI_POSTMEAN or XVB_POOL_XI_POSTDIST (LDE pooling has no "
                "native form)", fn, kind);
  XVB_CHECK_ARG(pooled > 0 && gdiv > 0 && pooled % gdiv == 0, "%s: pooled=%d must be a positive multiple of gdiv=%d", fn,
                pooled, gdiv);
  XVB_CHECK_ARG((prior_logprec_host && prior_mean_host) == xi && (prior_logprec_host != nullptr) == (prior_mean_host != nullptr),
                "%s: the xi-vector takes prior_logprec and prior_mean, the attention poolings neither", fn);
  XVB_CHECK_ARG(!xi || (gdiv == 1 && !unweighted_var), "%s: the xi-vector pools with gdiv 1 and weighted moments", fn);
  Config& c = h->draft->cfg;
  c.pool_kind = kind; c.pooled = pooled; c.gdiv = gdiv; c.unweighted = unweighted_var != 0;
  if (xi) {
    c.prior_logprec.assign(prior_logprec_host, prior_logprec_host + pooled);
    c.prior_mean.assign(prior_mean_host, prior_mean_host + pooled);
  }
  return XVB_OK;
}

extern "C" int xvb_extractor_add_attention_layer(xvb_extractor_t* h, int Cout, const int* context_host, int ntaps,
                                                 const float* w_host, const float* bias_host, const float* bn_scale_host,
                                                 const float* bn_shift_host, int flags) {
  const char* fn = "xvb_extractor_add_attention_layer";
  XVB_CHECK_ARG(is_draft(h) && h->draft->cfg.attention(), "%s: needs a draft extractor with an attention pooling", fn);
  Layers& r = h->draft->recs;
  XVB_CHECK_ARG(!r.frame.empty() && r.segment.empty(), "%s: attention layers go after the frame and before the segment layers", fn);
  XVB_CHECK_ARG(r.attention.size() < 2, "%s: an attention pooling has at most two affines (the first and the last)", fn);
  const int Cin = r.attention.empty() ? r.frame.back().Cout : r.attention.back().Cout;
  return add_layer(r.attention, Cin, Cout, context_host, ntaps, w_host, bias_host, bn_scale_host, bn_shift_host, flags);
}

extern "C" int xvb_extractor_add_segment_layer(xvb_extractor_t* h, int Cout, const float* w_host, const float* bias_host,
                                               const float* bn_scale_host, const float* bn_shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && !h->draft->recs.frame.empty(), "xvb_extractor_add_segment_layer: need frame layers first");
  Layers& r = h->draft->recs;
  const int Cin = r.segment.empty() ? h->draft->cfg.segment_in(r.frame.back().Cout) : r.segment.back().Cout;
  const int ctx0 = 0;
  return add_layer(r.segment, Cin, Cout, &ctx0, 1, w_host, bias_host, bn_scale_host, bn_shift_host, flags);
}

extern "C" int xvb_extractor_finalize(xvb_extractor_t* h, float pooling_eps) {
  XVB_CHECK_ARG(is_draft(h) && !h->draft->recs.frame.empty() && !h->draft->recs.segment.empty(),
                "xvb_extractor_finalize: need >=1 frame and >=1 segment layer");
  auto build = [&](Model* m, const Layers& r) -> int {
    for (size_t i = 0; i + 1 < r.frame.size(); ++i) {
      XVB_CHECK_ARG(r.frame[i].Cout % 8 == 0, "frame layer %d: Cout=%d must be a multiple of 8", (int)i, r.frame[i].Cout);
      if (r.frame[i].Cout > m->max_c) m->max_c = r.frame[i].Cout;
    }
    XVB_CHECK_ARG(r.frame.back().Cout % 4 == 0, "last frame layer: Cout=%d must be a multiple of 4", r.frame.back().Cout);
    for (size_t i = 0; i + 1 < r.segment.size(); ++i) {
      XVB_CHECK_ARG(r.segment[i].Cout % 8 == 0, "segment layer %d: Cout must be a multiple of 8", (int)i);
      if (r.segment[i].Cout > m->max_seg_c) m->max_seg_c = r.segment[i].Cout;
    }
    XVB_CHECK_ARG(r.segment.back().Cout % 4 == 0, "last segment layer: Cout must be a multiple of 4");
    const Config& c = m->cfg;
    const int cl = r.frame.back().Cout;
    if (c.attention()) {
      XVB_CHECK_ARG(!r.attention.empty(), "xvb_extractor_finalize: the attention pooling needs its last affine "
                    "(xvb_extractor_add_attention_layer)");
      XVB_CHECK_ARG(r.attention.back().Cout == c.pooled / c.gdiv,
                    "xvb_extractor_finalize: the last attention affine has %d outputs, the pooling takes pooled / gdiv = %d "
                    "logits", r.attention.back().Cout, c.pooled / c.gdiv);
      XVB_CHECK_ARG(c.pooled % cl == 0 && (!c.xi() || c.pooled == cl),
                    "xvb_extractor_finalize: pooled=%d must be a multiple of the last frame layer's %d channels (equal for "
                    "the xi-vector)", c.pooled, cl);
    }
    // an attention model packs its layers as the Python sequence does: output rows zero-padded to a multiple of 8
    auto pack = [&](const TapRec& rec, std::vector<Affine>& dst) {
      if (!c.attention() || rec.Cout % 8 == 0) return pack_tap(m->dev, rec, &dst.emplace_back());
      TapRec p = rec;
      p.Cout = (int)round_up(rec.Cout, 8);
      p.w.resize((size_t)p.Cout * p.Cin * p.tot(), 0.f);
      if (!p.b.empty()) p.b.resize(p.Cout, 0.f);
      if (!p.s.empty()) { p.s.resize(p.Cout, 0.f); p.t.resize(p.Cout, 0.f); }
      return pack_tap(m->dev, p, &dst.emplace_back());
    };
    int rc = XVB_OK;
    for (const TapRec& rec : r.frame) if (!rc) rc = pack(rec, m->frame);
    for (const TapRec& rec : r.attention) if (!rc) rc = pack(rec, m->attention);
    for (const TapRec& rec : r.segment) if (!rc) rc = pack(rec, m->segment);
    if (!rc && c.xi() && !(rc = m->dev.upload(&m->prior_logprec, c.prior_logprec))) rc = m->dev.upload(&m->prior_mean, c.prior_mean);
    if (rc) return rc;
    if (c.attention()) {   // the last frame layer and a first attention affine write planes into the ping-pong too
      m->max_c = std::max(m->max_c, m->frame.back().Cout);
      if (m->attention.size() > 1) m->max_c = std::max(m->max_c, m->attention[0].Cout);
    }
    m->embed = r.segment.back().Cout;
    m->pooling_eps = pooling_eps;
    // the Python sequence stages the first layer's input as plain planes: no im2col view for an attention model
    m->im2col = c.attention() ? Im2col{} : im2col_choice(r.frame[0].ctx, r.frame[0].ntaps, m->cfg.feat_dim);
    return XVB_OK;
  };
  const int rc = publish_built(h, build, "xvb_extractor_finalize");
  if (rc == XVB_OK) h->im2col = h->m->im2col;
  return rc;
}

extern "C" int xvb_extractor_embed_dim(const xvb_extractor_t* h) {
  return (h && !h->m->recs.segment.empty()) ? h->m->recs.segment.back().Cout : XVB_ESTATE;
}

extern "C" int xvb_extractor_save(const xvb_extractor_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_extractor_save: extractor not finalized");
  const Model* m = h->m.get();
  const struct { int32_t feat_dim; float pooling_eps; int32_t n_frame, n_segment; } head = {
      m->cfg.feat_dim, m->pooling_eps, (int32_t)m->recs.frame.size(), (int32_t)m->recs.segment.size()};
  std::vector<const TapRec*> layers;
  for (const auto* v : {&m->recs.frame, &m->recs.attention, &m->recs.segment})
    for (const TapRec& r : *v) layers.push_back(&r);
  if (!m->cfg.attention())
    return save_tap_file("xvb_extractor_save", path, "XVBM0001", &head, sizeof head, layers, false);
  const Config& c = m->cfg;
  const AttnPoolRecord pool = {c.pool_kind, c.pooled, c.gdiv, c.unweighted, (int32_t)m->recs.attention.size()};
  std::vector<char> block(sizeof head + sizeof pool);
  memcpy(block.data(), &head, sizeof head);
  memcpy(block.data() + sizeof head, &pool, sizeof pool);
  for (const std::vector<float>* v : {&c.prior_logprec, &c.prior_mean})
    block.insert(block.end(), (const char*)v->data(), (const char*)(v->data() + v->size()));
  return save_tap_file("xvb_extractor_save", path, "XVBM0002", block.data(), block.size(), layers, false);
}

// Grows the workspace to what one (B, T, masked) call needs.  Any reallocation drops the launch plans, which hold the
// old addresses.  Without growth this is host arithmetic only.
static int reserve(H* h, int B, int T, bool masked) {
  const Model* m = h->m.get();
  const bool att = m->cfg.attention();
  const size_t b = (size_t)B, f = (size_t)B * T, cl = (size_t)m->frame.back().Cout;
  const size_t sw = (size_t)m->cfg.stats_width((int)cl);
  const size_t pool = h->fused_pooling && !masked && !att ? (size_t)xvb_pool_partial_blocks(B, T, nullptr) * b * 2 * cl : 0;
  const size_t need[H::kBufs] = {(f + b * (h->im2col.pad_front + h->im2col.pad_back)) * m->cfg.ldf,
                                 f * m->max_c, f * m->max_c, f * cl, b * sw, b * m->segment.back().Cout, b * sw,
                                 b * m->max_seg_c, b * m->max_seg_c, pool, masked ? b : 0,
                                 att ? f * m->attention.back().Cout : 0};
  const bool planes[H::kBufs] = {true, true, true, false, false, false, true, true, true, false, false, false};
  uint64_t grown;
  const int rc = h->ws.reserve(need, planes, &grown);
  if (grown) h->drop_plans();
  return rc;
}

// Build the launch plan of one batch shape (see StepPlan).  On failure nothing is cached.
// A masked plan (utterances of different lengths) passes the extractor's device lengths to every frame layer, whose
// epilogue then zeroes the frames past each utterance's end, and always keeps the last layer's fp32 output for the
// length-aware standalone pooling (the fused pooling epilogue takes equal lengths only); the segment layers see one row
// per utterance either way.
static int build_step_plan(H* h, int B, int T, bool masked, StepPlan** out) {
  const Model* m = h->m.get();
  StepPlan* sp = new StepPlan();
  struct Guard { StepPlan* p; ~Guard() { delete p; } } guard{sp};
  int rc;
  sp->pool_blocks = xvb_pool_partial_blocks(B, T, &sp->pool_tb);
  Planes x = h->ws.planes(H::kIn);
  int64_t ldx = m->cfg.ldf;
  auto add = [&](std::vector<GemmPlan*>& dst, const xvb_tdnn_args_t& a) -> int {
    void* scratch = nullptr;
    const size_t need = gemm_plan_scratch_bytes(a);
    if (need) {
      XVB_CUDA(cudaMalloc(&scratch, need));
      sp->scratch.push_back(scratch);
    }
    GemmPlan* g = nullptr;
    int r = gemm_plan_build(&g, a, nullptr, scratch);
    if (r) return r;
    dst.push_back(g);
    return XVB_OK;
  };
  const bool att = m->cfg.attention();
  const int* lens = masked ? h->ws.i32(H::kLengths) : nullptr;
  for (size_t i = 0; i < m->frame.size(); ++i) {
    const Affine& L = m->frame[i];
    const bool last = i + 1 == m->frame.size();
    const Planes y = last && !att ? Planes{} : h->ws.planes(H::kAct0 + (i & 1));
    xvb_tdnn_args_t a = affine_args(L, x, ldx, B, T);
    a.y_hi = y.hi; a.y_lo = y.lo; a.ldy = L.Cout;
    a.lengths = lens;
    if (i == 0 && h->im2col.on) {   // window of ntaps consecutive frames = one long row of the padded planes
      a.context_host = kTaps; a.ntaps = 1; a.Cin = L.ntaps * L.Cin;
      a.x_batch_stride = (int64_t)(T + h->im2col.pad_front + h->im2col.pad_back) * ldx;
    }
    if (last && h->fused_pooling && !masked && !att) {
      a.pool_partial = h->ws.f32(H::kPoolPartial);
    } else if (last) {
      a.y_f32 = h->ws.f32(H::kLast); a.ldyf = L.Cout;
    }
    rc = add(sp->frame, a);
    if (rc && i == 0 && h->im2col.on) return -1000;   // overlapping tensor map refused: caller falls back for good
    if (rc) return rc;
    x = y; ldx = L.Cout;
  }
  // the attention affines over the last frame layer's planes: [first ->] last, whose fp32 logits the pooling takes
  for (size_t i = 0; i < m->attention.size(); ++i) {
    const Affine& L = m->attention[i];
    xvb_tdnn_args_t a = affine_args(L, x, ldx, B, T);
    a.lengths = lens;
    if (i + 1 == m->attention.size()) {
      a.y_f32 = h->ws.f32(H::kLogits); a.ldyf = L.Cout;
    } else {   // the ping-pong buffer the last frame layer did not write
      x = h->ws.planes(H::kAct0 + (m->frame.size() & 1)); ldx = L.Cout;
      a.y_hi = x.hi; a.y_lo = x.lo; a.ldy = L.Cout;
    }
    if ((rc = add(sp->attention, a))) return rc;
  }
  x = h->ws.planes(H::kStatsPlanes); ldx = m->cfg.stats_width(m->frame.back().Cout);
  for (size_t i = 0; i < m->segment.size(); ++i) {
    const Affine& L = m->segment[i];
    const bool last = i + 1 == m->segment.size();
    const Planes y = last ? Planes{} : h->ws.planes(H::kSeg0 + (i & 1));
    xvb_tdnn_args_t a = affine_args(L, x, ldx, B, 1);
    a.y_hi = y.hi; a.y_lo = y.lo; a.ldy = L.Cout;
    if (last) { a.y_f32 = h->ws.f32(H::kEmb); a.ldyf = L.Cout; }   // redirected to the caller's matrix at launch
    if ((rc = add(sp->segment, a))) return rc;
    x = y; ldx = L.Cout;
  }
  guard.p = nullptr;
  *out = sp;
  return XVB_OK;
}

// One batch through the stack.  masked: the workspace's lengths already hold the B utterance lengths (stream-ordered on
// `stream`).
static int extract_batch(H* h, const float* feats, int B, int T, bool masked, float* emb, void* stream) {
  int rc = reserve(h, B, T, masked);
  if (rc) return rc;
  const Model* m = h->m.get();
  const long before = g_launches;
  cudaStream_t cs = (cudaStream_t)stream;
  if (!h->in_shard) h->events_used = 0;   // a shard call keeps the events of all its batches
  h->events_stream = cs;
  StepPlan* sp = nullptr;
  const auto key = std::make_tuple(B, T, masked);
  auto it = h->plans.find(key);
  if (it != h->plans.end()) {
    sp = it->second;
  } else {
    rc = build_step_plan(h, B, T, masked, &sp);
    if (rc == -1000) {        // the driver refused the overlapping (im2col) tensor map: plain first layer from now on
      h->im2col = Im2col{};
      h->drop_plans();
      return extract_batch(h, feats, B, T, masked, emb, stream);
    }
    if (rc) return rc;
    h->plans[key] = sp;
  }
  if ((rc = h->mark(cs))) return rc;
  // 1. stage the frame matrix as split planes (framework.py:28-33 staging); for the im2col first layer with
  //    the zero frames of F.pad (components.py:117) written out around every utterance; a masked batch also writes
  //    zeros for every frame past an utterance's end, so no layer ever reads what the caller left there
  const int* lens = masked ? h->ws.i32(H::kLengths) : nullptr;
  const Planes in = h->ws.planes(H::kIn);
  if (h->im2col.on || masked)
    rc = split_frames(feats, B, T, m->cfg.feat_dim, in.hi, in.lo, m->cfg.ldf, h->im2col.pad_front, h->im2col.pad_back, lens, stream);
  else
    rc = xvb_split_f32(feats, (int64_t)B * T, m->cfg.feat_dim, m->cfg.feat_dim, in.hi, in.lo, m->cfg.ldf, stream);
  if (rc) return rc;
  if ((rc = h->mark(cs))) return rc;
  // 2. frame-level TDNN stack (xvector.py:85-89)
  for (GemmPlan* g : sp->frame) {
    if ((rc = gemm_plan_launch(g, stream))) return rc;
    if ((rc = h->mark(cs))) return rc;
  }
  // 3. statistics pooling (xvector.py:90, pooling.py:58-67), or the attention tail of AttentionPoolingExtractor.extract:
  //    [first affine ->] last affine to fp32 logits (masked like the frame layers), then the head-map pooling of the
  //    last frame layer's fp32 output, with the xi-vector's prior element and 2 log softplus logits
  const Config& c = m->cfg;
  const int cl = m->frame.back().Cout;
  float* stats = h->ws.f32(H::kStats);
  const Planes pooled = h->ws.planes(H::kStatsPlanes);
  if (c.attention()) {
    for (GemmPlan* g : sp->attention) {
      if ((rc = gemm_plan_launch(g, stream))) return rc;
      if ((rc = h->mark(cs))) return rc;
    }
    const int C = m->recs.frame.back().Cout, G = m->recs.attention.back().Cout, ldl = m->attention.back().Cout;
    const float* plp = c.xi() ? m->prior_logprec : nullptr;
    const float* pm = c.xi() ? m->prior_mean : nullptr;
    if (masked)
      rc = xvb_attn_head_stats_pool_lengths(h->ws.f32(H::kLogits), ldl, G, h->ws.f32(H::kLast), cl, B, T, C, c.pooled, c.gdiv,
                                            m->pooling_eps, c.unweighted, plp, pm, c.xi(), lens, stats, pooled.hi, pooled.lo,
                                            2 * c.pooled, stream);
    else
      rc = xvb_attn_head_stats_pool_prior(h->ws.f32(H::kLogits), ldl, G, h->ws.f32(H::kLast), cl, B, T, C, c.pooled, c.gdiv,
                                          m->pooling_eps, c.unweighted, plp, pm, c.xi(), stats, pooled.hi, pooled.lo,
                                          2 * c.pooled, stream);
  } else if (h->fused_pooling && !masked) {
    rc = xvb_pool_finalize(h->ws.f32(H::kPoolPartial), sp->pool_blocks, sp->pool_tb, B, T, cl, m->pooling_eps, 0, stats,
                           pooled.hi, pooled.lo, 2 * cl, stream);
  } else {
    rc = stats_pool(h->ws.f32(H::kLast), cl, B, T, cl, m->pooling_eps, 0, lens, stats, pooled.hi, pooled.lo, 2 * cl, stream);
  }
  if (rc) return rc;
  if ((rc = h->mark(cs))) return rc;
  // 4. segment-level layers (xvector.py:92-96); the last one writes the caller's embedding matrix, or (rows padded to a
  //    multiple of 8) its own buffer, whose first `embed` columns are then copied there
  const bool direct = m->segment.back().Cout == m->embed;
  for (size_t i = 0; i < sp->segment.size(); ++i) {
    const bool last = i + 1 == sp->segment.size();
    if ((rc = gemm_plan_launch(sp->segment[i], stream, last && direct ? emb : nullptr))) return rc;
    if ((rc = h->mark(cs))) return rc;
  }
  if (!direct)
    XVB_CUDA(cudaMemcpy2DAsync(emb, (size_t)m->embed * sizeof(float), h->ws.f32(H::kEmb), (size_t)m->segment.back().Cout * sizeof(float),
                               (size_t)m->embed * sizeof(float), (size_t)B, cudaMemcpyDeviceToDevice, cs));
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

// An attention model's extract call: consecutive groups of at most kAttnFrameBudget frames (at least one utterance),
// each run as its own call would run it: masked when lengths_host is given and some length of the group is below T.
// The lengths were checked by the caller.
static int extract_attention(H* h, const float* feats, const int32_t* lengths_host, int B, int T, float* emb, void* stream) {
  const long before = g_launches;
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->embed;
  const int rc = for_groups(B, T, kAttnFrameBudget, [&](int i, int b) -> int {
    bool masked = false;
    for (int j = 0; lengths_host && j < b; ++j) masked = masked || lengths_host[i + j] != T;
    if (masked) {
      int r = reserve(h, b, T, true);   // first, so that the lengths land in the buffer the plans read
      if (r) return r;
      // stream-ordered: the previous group's kernels on `stream` have read the old lengths before these land
      XVB_CUDA(cudaMemcpyAsync(h->ws.i32(H::kLengths), lengths_host + i, (size_t)b * sizeof(int32_t), cudaMemcpyHostToDevice,
                               (cudaStream_t)stream));
    }
    return extract_batch(h, feats + i * per_utt, b, T, masked, emb + i * E, stream);
  });
  h->last_launches = (int)(g_launches - before);
  return rc;
}

extern "C" int xvb_extractor_extract(xvb_extractor_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_extractor_extract: extractor not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_extractor_extract: bad arguments");
  if (h->m->cfg.attention()) return extract_attention(h, feats, nullptr, B, T, emb, stream);
  return extract_batch(h, feats, B, T, false, emb, stream);
}

extern "C" int xvb_extractor_extract_lengths(xvb_extractor_t* h, const float* feats, const int32_t* lengths_host, int B, int T,
                                             float* emb, void* stream) {
  const char* fn = "xvb_extractor_extract_lengths";
  XVB_CHECK_ARG(finalized(h), "%s: extractor not finalized", fn);
  XVB_CHECK_ARG(feats && lengths_host && emb && B > 0 && T > 0, "%s: bad arguments", fn);
  bool all_T;
  int rc = check_lengths(fn, lengths_host, B, T, &all_T);
  if (rc) return rc;
  if (h->m->cfg.attention()) return extract_attention(h, feats, all_T ? nullptr : lengths_host, B, T, emb, stream);
  if (all_T) return extract_batch(h, feats, B, T, false, emb, stream);   // nothing to mask: the unmasked call itself
  if ((rc = reserve(h, B, T, true))) return rc;   // first, so that the lengths land in the buffer the plans read
  // stream-ordered: the previous call's kernels on `stream` have read the old lengths before these land
  XVB_CUDA(cudaMemcpyAsync(h->ws.i32(H::kLengths), lengths_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice,
                           (cudaStream_t)stream));
  return extract_batch(h, feats, B, T, true, emb, stream);
}

extern "C" int xvb_extractor_set_gather(xvb_extractor_t* h, float* const* tables, int ntables, int64_t row0, int64_t ld) {
  XVB_CHECK_ARG(finalized(h), "xvb_extractor_set_gather: bad arguments");
  return h->shard.set_gather(tables, ntables, row0, ld, h->m->embed, "xvb_extractor_set_gather");
}

// The caller loop of the reference (extract_embeddings.py:73-83: one utterance per iteration) for a whole shard of N
// equal-length utterances (shard.cuh).  With per-kernel profiling on, the batches run back to back on `stream` itself
// and the events of all of them are kept.
extern "C" int xvb_extractor_extract_shard(xvb_extractor_t* h, const float* feats, int64_t N, int T, int batch, float* emb,
                                           void* stream) {
  XVB_CHECK_ARG(h, "xvb_extractor_extract_shard: bad arguments");
  h->events_used = 0;
  h->in_shard = true;
  const int rc = Shard<H>::device(h, feats, N, T, batch, emb, stream, h->profiling, "xvb_extractor_extract_shard");
  h->in_shard = false;
  return rc;
}

extern "C" int xvb_extractor_extract_host(xvb_extractor_t* h, const float* feats_host, int B, int T, float* emb_host,
                                          void* stream) {
  return Shard<H>::extract_host(h, feats_host, B, T, emb_host, stream, "xvb_extractor_extract_host");
}

extern "C" int xvb_extractor_submit_host(xvb_extractor_t* h, const float* feats_host, int B, int T, float* emb_host,
                                         int slot, void* stream) {
  return Shard<H>::submit(h, feats_host, B, T, emb_host, slot, stream, "xvb_extractor_submit_host");
}

extern "C" int xvb_extractor_wait(xvb_extractor_t* h, int slot) {
  XVB_CHECK_ARG(h && (slot == 0 || slot == 1), "xvb_extractor_wait: bad arguments");
  return h->shard.wait(slot);
}

extern "C" int xvb_extractor_extract_shard_host(xvb_extractor_t* h, const float* feats_host, int64_t N, int T, int batch,
                                                float* emb_host, void* stream) {
  return Shard<H>::host(h, feats_host, N, T, batch, emb_host, stream, h && h->profiling, "xvb_extractor_extract_shard_host");
}

extern "C" int xvb_extractor_set_fused_pooling(xvb_extractor_t* h, int enable) {
  XVB_CHECK_ARG(h, "xvb_extractor_set_fused_pooling: null extractor");
  if (h->fused_pooling != (enable != 0)) h->drop_plans();
  h->fused_pooling = enable != 0;
  if (h->shard.lane1) return xvb_extractor_set_fused_pooling(h->shard.lane1.get(), enable);
  return XVB_OK;
}

extern "C" int xvb_extractor_set_profiling(xvb_extractor_t* h, int enable) {
  XVB_CHECK_ARG(h, "xvb_extractor_set_profiling: null extractor");
  h->profiling = enable != 0;
  h->events_used = 0;
  return XVB_OK;
}

extern "C" int xvb_extractor_kernel_times(xvb_extractor_t* h, float* ms_host, int max_n) {
  XVB_CHECK_ARG(h && ms_host, "xvb_extractor_kernel_times: null argument");
  if (h->events_used < 2) return 0;
  XVB_CUDA(cudaEventSynchronize(h->events[h->events_used - 1]));
  int n = h->events_used - 1;
  if (n > max_n) n = max_n;
  for (int i = 0; i < n; ++i) XVB_CUDA(cudaEventElapsedTime(&ms_host[i], h->events[i], h->events[i + 1]));
  return n;
}

extern "C" int xvb_extractor_last_launches(const xvb_extractor_t* h) { return h ? h->last_launches : XVB_ESTATE; }

extern "C" const float* xvb_extractor_debug_f32(const xvb_extractor_t* h, int which) {
  if (!h) return nullptr;
  return h->ws.f32(which < 0 ? H::kStats : H::kLast);
}

extern "C" void xvb_extractor_destroy(xvb_extractor_t* h) { delete h; }
