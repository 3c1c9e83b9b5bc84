// Whole-model extractor for ECAPA-TDNN (pytorch/model/ecapa_tdnn_xvector.py, ECAPA_TDNN.extract_embedding
// :403-426): packed weights + workspace on the current device and the launch sequence, in C++, so that the
// model needs no Python at run time (the role of the reference's TorchScript runtime, runtime/extractor/
// torch_asv_model.cc) and the ~55 launches of a batch are issued back to back with programmatic dependent
// launch.  Same kernels and the same order as the Python orchestration it replaces
// (asv_subtools_b200/model/ecapa_tdnn_xvector.py keeps that as XVB_ECAPA_NATIVE=0 for A/B runs):
//
//   split -> layer1 -> 3 x [ 1x1 TDNN-ReLU-BN -> Res2Net chain kernel -> 1x1 TDNN-ReLU-BN -> plane mean ->
//   SE gate (two M = B GEMMs, ReLU / sigmoid) -> z*gate + in (+ running sum x + x1 (+ x2)) into its slot of
//   the (B,T,3C) MFA input ] -> mfa -> global mean/std (unbiased var + 1e-5) -> per-utterance bias of the
//   first attention conv -> attention conv 1 (ReLU, BN, tanh; time-constant columns as utt_bias) ->
//   attention conv 2 -> online-softmax weighted moments -> fc2 (bn_stats folded in; own BN for "near").
//
// Layers are handed over by NAME with the weights as the state_dict stores them (host fp32, eval BatchNorm
// folded to scale/shift by the caller); the two derived layers of the attention conv ("att_x": its columns
// over x, "att_gs": its columns over [mean | std] plus the bias) and "fc2" (bn_stats folded into its weight)
// are prepared by the caller -- see EcapaExtractor.save() / the Python blueprint.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "records.cuh"
#include "shard.cuh"

// The model types are local to this file: each family has its own Model.
namespace {

using namespace xvb;

struct ELayer {
  int Cin = 0, Cout = 0, ntaps = 0, flags = 0, tot = 0;
  int ctx[XVB_MAX_TAPS] = {0};
  Planes w;
  float* bias = nullptr;
  float* scale = nullptr;
  float* shift = nullptr;
  float* w_f32 = nullptr;   // (Cout, Cin) fp32 as stored, kept for one-tap layers: the segment-level ones run on CUDA cores
  // grouped 1x1 conv (the MQMHA attention convs): Cin is the per-group width; packed compactly for the layer kernel's
  // grouped mode, or as the block-diagonal expansion (expanded) when the shape does not fit that mode
  int groups = 1;
  bool expanded = false;
  // host copies for save()
  std::vector<float> hw, hb, hs, ht;
};

// split planes with their row pitch
struct View {
  uint16_t* hi = nullptr;
  uint16_t* lo = nullptr;
  int64_t ld = 0;
  View slice(int c0) const { return View{hi + c0, lo + c0, ld}; }
};

// The layers and what finalize fixes; shared read-only by a handle and its second shard lane once finalized.
struct Model {
  int feat_dim = 0, ldf = 0, C = 0, D = 0, H = 0, E = 0, scale = 8, se_dim = 0;
  int dilation[3] = {2, 3, 4};
  std::map<std::string, ELayer> layers;
  std::vector<std::string> order;   // insertion order, for save()
  // stacked Res2Net parameters per block
  Planes res_w[3];
  float* res_bias[3] = {nullptr, nullptr, nullptr};
  float* res_scale[3] = {nullptr, nullptr, nullptr};
  float* res_shift[3] = {nullptr, nullptr, nullptr};
  int fc1_dim = 0;
  // multi-query multi-head attention pooling (xvb_ecapa_set_mqmha); mq == 0: ECAPA's own attentive pooling
  int mq = 0, mq_heads = 1, mq_q = 1, mq_hidden = 0, mq_share = 0, mq_layers = 2, mq_tatt = 1, mq_stddev = 1;
  // widths derived from the pooling: att_x outputs AX, the logits NL (row pitch ldlog), the pooled statistics P of the
  // P2-wide [mean | std] buffer (default model: AX = H, NL = D, P = P2 = 2D)
  int AX = 0, NL = 0, ldlog = 0, P = 0, P2 = 0;
  Im2col im2col;   // layer1 as an im2col view (records.cuh)
  Weights dev{"xvb_ecapa_set_layer"};
};

}  // namespace

using namespace xvb;

struct xvb_ecapa : Handle<Model> {
  // workspace, each buffer grown to the largest call seen: the plane buffers up to kPp, then the fp32 ones
  enum { kIn, kX, kH, kR, kZ, kN, kCat, kM, kA1, kGp, kS1, kZm, kPp, kMF, kLog, kGate, kUb, kZmean, kGstat, kPstat, kS1f,
         kF1, kBufs };
  Workspace<kBufs> ws;
  // the workspace's buffers as reserve last left them: planes with their row pitch, and fp32
  View in, X, Hh, R, Z, N, CAT, M, A1, gp, s1, zm, pp;
  float *MF = nullptr, *LOG = nullptr, *gate = nullptr, *ub = nullptr, *zmean = nullptr, *gstat = nullptr, *pstat = nullptr;
  float* s1f = nullptr;   // (B, se_dim) fp32: hidden vector of the SE gate
  float* f1 = nullptr;    // (B, fc1_dim) fp32: output of fc1 when the model has one
  Im2col im2col;   // this lane's copy of the model's choice
  Shard<xvb_ecapa> shard;

  xvb_ecapa() = default;
  explicit xvb_ecapa(std::shared_ptr<const Model> model) : Handle(std::move(model)), im2col(m->im2col) {}
};

template <>
struct xvb::ShardFamily<xvb_ecapa> {
  static int extract(xvb_ecapa* h, const float* feats, int B, int T, float* emb, void* stream) {
    return xvb_ecapa_extract(h, feats, B, T, emb, stream);
  }
  static xvb_ecapa* twin(const xvb_ecapa* h) { return new xvb_ecapa(h->m); }
  static int feat_dim(const xvb_ecapa* h) { return h->m->feat_dim; }
  static int embed_dim(const xvb_ecapa* h) { return h->m->E; }
};

extern "C" int xvb_ecapa_create(xvb_ecapa_t** out, int feat_dim, int channels, int mfa_dim, int att_hidden, int embed_dim) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && feat_dim > 0 && channels > 0 && mfa_dim > 0 && att_hidden > 0 && embed_dim > 0, "xvb_ecapa_create: bad arguments");
  XVB_CHECK_ARG(channels == 8 * 64 || channels == 8 * 128,
                "xvb_ecapa_create: the Res2Net chain kernel is built for scale 8 x width 64 or 128 (channels = 512 or 1024), got %d",
                channels);
  XVB_CHECK_ARG(mfa_dim % 8 == 0 && att_hidden % 8 == 0 && embed_dim % 4 == 0, "xvb_ecapa_create: mfa_dim/att_hidden must be multiples of 8, embed_dim of 4");
  xvb_ecapa* h = new xvb_ecapa();
  Model* m = h->draft;
  m->feat_dim = feat_dim; m->ldf = (int)round_up(feat_dim, 8);
  m->C = channels; m->D = mfa_dim; m->H = att_hidden; m->E = embed_dim;
  m->AX = att_hidden; m->NL = mfa_dim; m->ldlog = mfa_dim; m->P = 2 * mfa_dim; m->P2 = 2 * mfa_dim;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_ecapa_set_mqmha(xvb_ecapa_t* h, int num_head, int num_q, int hidden, int share, int affine_layers,
                                   int time_attention, int stddev) {
  XVB_CHECK_ARG(is_draft(h) && h->draft->layers.empty(), "xvb_ecapa_set_mqmha: call it between xvb_ecapa_create and the first set_layer");
  Model* m = h->draft;
  XVB_CHECK_ARG(num_head >= 1 && num_q >= 1 && hidden >= 1 && (affine_layers == 1 || affine_layers == 2) && m->D % num_head == 0 &&
                (m->D / num_head) % 4 == 0 && hidden * num_head * num_q == m->H,
                "xvb_ecapa_set_mqmha: need %d channels in heads of a multiple of 4, 1 or 2 affine layers and att_hidden = "
                "hidden * num_head * num_q (= %d)", m->D, m->H);
  const int cg = m->D / num_head, hq = num_head * num_q;
  m->mq = 1; m->mq_heads = num_head; m->mq_q = num_q; m->mq_hidden = hidden; m->mq_share = share ? 1 : 0;
  m->mq_layers = affine_layers; m->mq_tatt = time_attention ? 1 : 0; m->mq_stddev = stddev ? 1 : 0;
  m->NL = hq * (share ? 1 : cg);
  m->ldlog = (int)round_up(m->NL, 4);
  m->AX = affine_layers == 2 ? m->H : m->NL;
  XVB_CHECK_ARG(!time_attention || m->AX % 4 == 0, "xvb_ecapa_set_mqmha: the time-constant columns of the first attention conv "
                "become a per-utterance bias, which needs a multiple of 4 outputs (got %d)", m->AX);
  m->P2 = 2 * num_q * m->D;
  m->P = stddev ? m->P2 : num_q * m->D;
  return XVB_OK;
}

// Groups of a layer as the state_dict stores it: the MQMHA attention convs are grouped (pooling.py:665-698)
static int layer_groups(const Model* m, const std::string& n) {
  if (!m->mq) return 1;
  if (n == "att_x") return m->mq_heads;
  if (n == "att2") return m->mq_heads * m->mq_q;
  return 1;
}

extern "C" int xvb_ecapa_set_layer(xvb_ecapa_t* h, const char* name, int Cout, int Cin, const int* context_host, int ntaps,
                                   const float* w_host, const float* bias_host, const float* bn_scale_host,
                                   const float* bn_shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && w_host && context_host, "xvb_ecapa_set_layer: bad arguments or finalized model");
  Model* m = h->draft;
  XVB_CHECK_ARG(Cout > 0 && Cin > 0 && ntaps >= 1 && ntaps <= XVB_MAX_TAPS, "xvb_ecapa_set_layer(%s): bad shape", name);
  XVB_CHECK_ARG(!(flags & XVB_BN) || (bn_scale_host && bn_shift_host), "xvb_ecapa_set_layer(%s): XVB_BN without scale/shift", name);
  XVB_CHECK_ARG(m->layers.find(name) == m->layers.end(), "xvb_ecapa_set_layer: layer '%s' set twice", name);
  ELayer L;
  L.Cin = Cin; L.Cout = Cout; L.ntaps = ntaps; L.flags = flags;
  for (int i = 0; i < ntaps; ++i) L.ctx[i] = context_host[i];
  const int left = L.ctx[0] < 0 ? L.ctx[0] : 0, right = L.ctx[ntaps - 1] > 0 ? L.ctx[ntaps - 1] : 0;
  L.tot = right - left + 1;
  const size_t wn = (size_t)Cout * Cin * L.tot;
  L.hw.assign(w_host, w_host + wn);
  if (bias_host) L.hb.assign(bias_host, bias_host + Cout);
  if (flags & XVB_BN) { L.hs.assign(bn_scale_host, bn_scale_host + Cout); L.ht.assign(bn_shift_host, bn_shift_host + Cout); }
  L.groups = layer_groups(m, name);
  XVB_CHECK_ARG(L.groups == 1 || (ntaps == 1 && L.tot == 1 && Cout % L.groups == 0),
                "xvb_ecapa_set_layer(%s): a grouped layer is a 1x1 conv with Cout divisible by its %d groups", name, L.groups);
  // a grouped shape the layer kernel's grouped mode does not take runs as its block-diagonal expansion
  L.expanded = L.groups > 1 && !xvb_tdnn_grouped_fits(Cin * L.groups, Cout, L.groups);
  std::vector<float> dense;
  int cin_pack = Cin;
  if (L.expanded) {
    const int G = L.groups, co = Cout / G;
    cin_pack = Cin * G;
    dense.assign((size_t)Cout * cin_pack, 0.f);
    for (int n = 0; n < Cout; ++n)
      memcpy(&dense[(size_t)n * cin_pack + (size_t)(n / co) * Cin], w_host + (size_t)n * Cin, Cin * sizeof(float));
  }
  int rc;
  if ((rc = m->dev.pack(&L.w, L.expanded ? dense : L.hw, Cout, cin_pack, L.tot, L.ctx, ntaps))) return rc;
  // one tap: (Cout, Cin, 1) is the (N, K) matrix xvb_small_affine takes
  if (L.tot == 1 && Cin % 4 == 0 && L.groups == 1 && (rc = m->dev.upload(&L.w_f32, L.hw))) return rc;
  if ((rc = m->dev.upload(&L.bias, L.hb)) || (rc = m->dev.upload(&L.scale, L.hs)) || (rc = m->dev.upload(&L.shift, L.ht))) return rc;
  m->layers[name] = L;
  m->order.push_back(name);
  return XVB_OK;
}

static const ELayer* find(const Model* m, const std::string& n) {
  auto it = m->layers.find(n);
  return it == m->layers.end() ? nullptr : &it->second;
}

extern "C" int xvb_ecapa_finalize(xvb_ecapa_t* h) {
  XVB_CHECK_ARG(is_draft(h), "xvb_ecapa_finalize: null or finalized model");
  Model* m = h->draft;
  const int C = m->C, W = C / m->scale;
  auto need = [&](const std::string& n, int cin, int cout, int ntaps) -> int {
    const ELayer* L = find(m, n);
    XVB_CHECK_ARG(L, "xvb_ecapa_finalize: layer '%s' is missing", n.c_str());
    XVB_CHECK_ARG(L->Cin == cin && L->Cout == cout && L->ntaps == ntaps, "xvb_ecapa_finalize: layer '%s' is %d->%d x%d taps, expected %d->%d x%d",
                  n.c_str(), L->Cin, L->Cout, L->ntaps, cin, cout, ntaps);
    return XVB_OK;
  };
  int rc;
  rc = need("layer1", m->feat_dim, C, find(m, "layer1") ? find(m, "layer1")->ntaps : 5);
  if (rc) return rc;
  for (int b = 0; b < 3; ++b) {
    const std::string p = "layer" + std::to_string(b + 2) + ".";
    if ((rc = need(p + "bn1", C, C, 1)) || (rc = need(p + "bn2", C, C, 1))) return rc;
    const ELayer* se1 = find(m, p + "se1");
    XVB_CHECK_ARG(se1 && se1->Cin == C, "xvb_ecapa_finalize: layer '%sse1' is missing", p.c_str());
    if (b == 0) m->se_dim = se1->Cout;
    XVB_CHECK_ARG(se1->Cout == m->se_dim && m->se_dim % 8 == 0, "xvb_ecapa_finalize: SE bottleneck must be a multiple of 8 and equal in all blocks");
    rc = need(p + "se2", m->se_dim, C, 1);
    if (rc) return rc;
    // stack the scale-1 Res2Net layers: packed weights along rows, parameters back to back
    const size_t pw = (size_t)xvb_packed_weight_elems(W, W, 3);
    if ((rc = m->dev.alloc(&m->res_w[b].hi, pw * (m->scale - 1))) || (rc = m->dev.alloc(&m->res_w[b].lo, pw * (m->scale - 1))) ||
        (rc = m->dev.alloc(&m->res_bias[b], (size_t)W * (m->scale - 1))) || (rc = m->dev.alloc(&m->res_scale[b], (size_t)W * (m->scale - 1))) ||
        (rc = m->dev.alloc(&m->res_shift[b], (size_t)W * (m->scale - 1))))
      return rc;
    for (int i = 0; i < m->scale - 1; ++i) {
      const std::string n = p + "res" + std::to_string(i);
      if ((rc = need(n, W, W, 3))) return rc;
      const ELayer* L = find(m, n);
      XVB_CHECK_ARG(L->ctx[0] == -L->ctx[2] && L->ctx[1] == 0 && L->bias && L->scale && L->shift && (L->flags & XVB_RELU),
                    "xvb_ecapa_finalize: '%s' must be a [-d,0,d] TDNN-ReLU-BN layer with bias", n.c_str());
      if (i == 0) m->dilation[b] = L->ctx[2];
      XVB_CHECK_ARG(L->ctx[2] == m->dilation[b], "xvb_ecapa_finalize: '%s' has another dilation than its block", n.c_str());
      XVB_CUDA(cudaMemcpy(m->res_w[b].hi + pw * i, L->w.hi, pw * 2, cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(m->res_w[b].lo + pw * i, L->w.lo, pw * 2, cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(m->res_bias[b] + (size_t)W * i, L->bias, W * sizeof(float), cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(m->res_scale[b] + (size_t)W * i, L->scale, W * sizeof(float), cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(m->res_shift[b] + (size_t)W * i, L->shift, W * sizeof(float), cudaMemcpyDeviceToDevice));
    }
  }
  rc = need("mfa", 3 * C, m->D, 1);
  if (rc) return rc;
  if (!m->mq) {
    if ((rc = need("att_x", m->D, m->H, 1)) || (rc = need("att_gs", 2 * m->D, m->H, 1)) || (rc = need("att2", m->H, m->D, 1)))
      return rc;
  } else {   // per-group input widths: att_x reads a head's Cg channels of x, att2 one query's hidden units
    rc = need("att_x", m->D / m->mq_heads, m->AX, 1);
    if (rc) return rc;
    if (m->mq_layers == 2 && (rc = need("att2", m->mq_hidden, m->NL, 1))) return rc;
    XVB_CHECK_ARG(m->mq_layers == 2 || !find(m, "att2"), "xvb_ecapa_finalize: one-layer attention has no 'att2'");
    if (m->mq_tatt && (rc = need("att_gs", (m->mq_stddev ? 2 : 1) * m->D, m->AX, 1))) return rc;
    XVB_CHECK_ARG(m->mq_tatt || !find(m, "att_gs"), "xvb_ecapa_finalize: 'att_gs' without time attention");
  }
  // segment level (ecapa_tdnn_xvector.py:412-422): [fc1 ->] [fc2]; "far" hands over fc1 alone, fc1=False fc2 alone
  if (const ELayer* fc1 = find(m, "fc1")) {
    XVB_CHECK_ARG(fc1->Cin == m->P && fc1->ntaps == 1 && fc1->w_f32, "xvb_ecapa_finalize: 'fc1' must be a one-tap layer over the %d pooled statistics", m->P);
    if (find(m, "fc2")) {
      rc = need("fc2", fc1->Cout, m->E, 1);
      if (rc) return rc;
    } else {
      XVB_CHECK_ARG(fc1->Cout == m->E, "xvb_ecapa_finalize: 'fc1' alone must produce the %d-d embedding", m->E);
    }
    m->fc1_dim = fc1->Cout;
  } else {
    rc = need("fc2", m->P, m->E, 1);
    if (rc) return rc;
  }
  const ELayer* L0 = find(m, "layer1");
  m->im2col = h->im2col = im2col_choice(L0->ctx, L0->ntaps, m->feat_dim);
  h->draft = nullptr;
  return XVB_OK;
}

extern "C" int xvb_ecapa_embed_dim(const xvb_ecapa_t* h) { return h ? h->m->E : XVB_EINVAL; }
extern "C" int xvb_ecapa_feat_dim(const xvb_ecapa_t* h) { return h ? h->m->feat_dim : XVB_EINVAL; }
extern "C" int xvb_ecapa_last_launches(const xvb_ecapa_t* h) { return h ? h->last_launches : 0; }

static int reserve(xvb_ecapa* h, int B, int T) {
  using H = xvb_ecapa;
  const Model* m = h->m.get();
  const size_t b = (size_t)B, f = (size_t)B * T, C = (size_t)m->C, D = (size_t)m->D;
  const size_t need[H::kBufs] = {(f + b * (h->im2col.pad_front + h->im2col.pad_back)) * m->ldf, f * C, f * C, f * C, f * C,
                                 f * C, f * 3 * C, f * D, f * m->H, b * 2 * D, b * m->se_dim, b * C, b * m->P2,
                                 f * D, f * m->ldlog, b * C, b * m->AX, b * C, b * 2 * D, b * m->P2, b * m->se_dim,
                                 b * m->fc1_dim};
  bool planes[H::kBufs];
  for (int i = 0; i < H::kBufs; ++i) planes[i] = i <= H::kPp;
  uint64_t grown;
  const int rc = h->ws.reserve(need, planes, &grown);
  if (rc) return rc;
  auto view = [&](int i, int64_t ld) { const Planes p = h->ws.planes(i); return View{p.hi, p.lo, ld}; };
  h->in = view(H::kIn, m->ldf); h->X = view(H::kX, C); h->Hh = view(H::kH, C); h->R = view(H::kR, C);
  h->Z = view(H::kZ, C); h->N = view(H::kN, C); h->CAT = view(H::kCat, 3 * C); h->M = view(H::kM, D);
  h->A1 = view(H::kA1, m->H); h->gp = view(H::kGp, 2 * D); h->s1 = view(H::kS1, m->se_dim); h->zm = view(H::kZm, C);
  h->pp = view(H::kPp, m->P2);
  h->MF = h->ws.f32(H::kMF); h->LOG = h->ws.f32(H::kLog); h->gate = h->ws.f32(H::kGate); h->ub = h->ws.f32(H::kUb);
  h->zmean = h->ws.f32(H::kZmean); h->gstat = h->ws.f32(H::kGstat); h->pstat = h->ws.f32(H::kPstat);
  h->s1f = h->ws.f32(H::kS1f); h->f1 = h->ws.f32(H::kF1);
  return XVB_OK;
}

namespace {
struct Run {   // one layer launch: fill only what differs from the defaults
  const ELayer* L;
  View x, y;
  float* y_f32 = nullptr;
  int64_t ldyf = 0;
  const float* utt_bias = nullptr;
  int64_t ld_utt = 0;
  int extra_flags = 0;
  int B, T;
  int im2col_taps = 0;          // > 0: one-tap view, Cin = taps * L->Cin, rows overlap (x_batch_stride)
  int64_t x_batch_stride = 0;
};
// segment-level layer (one row per utterance) on CUDA cores: fp32 in, fp32 out
int small_layer(const ELayer* L, const float* x, int64_t ldx, int B, float* y, int64_t ldy, int extra_flags, void* stream) {
  return xvb_small_affine(x, ldx, L->w_f32, B, L->Cin, L->Cout, L->bias, L->scale, L->shift, L->flags | extra_flags, y, ldy,
                          nullptr, nullptr, 0, stream);
}
bool small_ok(const ELayer* L) {
  static const int knob = getenv("XVB_ECAPA_SMALL") ? atoi(getenv("XVB_ECAPA_SMALL")) : 1;
  return knob && L->w_f32 != nullptr;
}
int launch(const Run& r, void* stream) {
  xvb_tdnn_args_t a{};
  a.x_hi = r.x.hi; a.x_lo = r.x.lo; a.ldx = r.x.ld;
  a.w_hi = r.L->w.hi; a.w_lo = r.L->w.lo;
  a.bias = r.L->bias; a.bn_scale = r.L->scale; a.bn_shift = r.L->shift;
  a.flags = r.L->flags | r.extra_flags;
  a.utt_bias = r.utt_bias; a.ld_utt_bias = r.ld_utt;
  a.context_host = r.L->ctx; a.ntaps = r.L->ntaps;
  const int ctx0 = 0;
  if (r.im2col_taps > 0) { a.context_host = &ctx0; a.ntaps = 1; a.x_batch_stride = r.x_batch_stride; }
  a.y_hi = r.y.hi; a.y_lo = r.y.lo; a.ldy = r.y.ld;
  a.y_f32 = r.y_f32; a.ldyf = r.ldyf;
  a.B = r.B; a.T = r.T; a.Cin = r.im2col_taps > 0 ? r.im2col_taps * r.L->Cin : r.L->Cin * r.L->groups; a.Cout = r.L->Cout;
  a.groups = r.L->expanded ? 1 : r.L->groups;
  return xvb_tdnn_affine_ex(&a, stream);
}
}  // namespace

// MQMHASP.forward (libs/nnet/pooling.py:627-663) over the mfa output (M planes, MF fp32) into pstat / pp:
// time attention: biased mean | sqrt(clamp(var, 1e-5)) of every channel (egrecho's compute_statistics) -> the
// per-utterance bias of the first attention conv (its [mean_h | std_h] columns, block-diagonal over the heads) ->
// grouped conv over x (ReLU -> BN -> tanh) -> grouped conv to the logits -> softmax over T and weighted moments with
// the head-width map: pooled channel (h*Q + q)*Cg + c is x channel h*Cg + c under the alpha of logit (h*Q + q)[*Cg + c].
static int mqmha_pool(xvb_ecapa* h, int B, int T, void* stream) {
  const Model* m = h->m.get();
  const int D = m->D, cg = D / m->mq_heads;
  const ELayer* ax = find(m, "att_x");
  int rc;
  if (m->mq_tatt) {
    if ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 0, h->gstat, h->gp.hi, h->gp.lo, 2 * D, stream))) return rc;
    const ELayer* gs = find(m, "att_gs");
    if (small_ok(gs)) {
      if ((rc = small_layer(gs, h->gstat, 2 * D, B, h->ub, m->AX, 0, stream))) return rc;
    } else {
      Run r{}; r.B = B; r.T = 1; r.L = gs; r.x = h->gp; r.y_f32 = h->ub; r.ldyf = m->AX;
      if ((rc = launch(r, stream))) return rc;
    }
  }
  Run r{}; r.B = B; r.T = T; r.L = ax; r.x = h->M;
  if (m->mq_tatt) { r.utt_bias = h->ub; r.ld_utt = m->AX; }
  if (m->mq_layers == 2) { r.y = h->A1; r.extra_flags = XVB_TANH; }
  else { r.y_f32 = h->LOG; r.ldyf = m->ldlog; }
  if ((rc = launch(r, stream))) return rc;
  if (m->mq_layers == 2) {
    r = Run{}; r.B = B; r.T = T; r.L = find(m, "att2"); r.x = h->A1; r.y_f32 = h->LOG; r.ldyf = m->ldlog;
    if ((rc = launch(r, stream))) return rc;
  }
  return xvb_attn_head_stats_pool_mq(h->LOG, m->ldlog, m->NL, h->MF, D, B, T, D, m->mq_q * D, m->mq_share ? cg : 1, cg, m->mq_q,
                                     1e-5f, 0, h->pstat, h->pp.hi, h->pp.lo, m->P2, stream);
}

extern "C" int xvb_ecapa_extract(xvb_ecapa_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_ecapa_extract: model not finalized");
  const Model* m = h->m.get();
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_ecapa_extract: bad arguments");
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const long before = g_launches;
  const int C = m->C, D = m->D;
  auto L = [&](const std::string& n) { return find(m, n); };
  const Im2col& im = h->im2col;
  if (im.on)
    rc = xvb_split_frames(feats, B, T, m->feat_dim, h->in.hi, h->in.lo, m->ldf, im.pad_front, im.pad_back, stream);
  else
    rc = xvb_split_f32(feats, (int64_t)B * T, m->feat_dim, m->feat_dim, h->in.hi, h->in.lo, m->ldf, stream);
  if (rc) return rc;
  Run r{};
  r.B = B; r.T = T;
  r.L = L("layer1"); r.x = h->in; r.y = h->X;
  if (im.on) { r.im2col_taps = r.L->ntaps; r.x_batch_stride = (int64_t)(T + im.pad_front + im.pad_back) * m->ldf; }
  rc = launch(r, stream);
  if (rc && im.on) {   // overlapping tensor map refused by the driver: plain path from now on
    h->im2col = Im2col{};
    return xvb_ecapa_extract(h, feats, B, T, emb, stream);
  }
  if (rc) return rc;
  View cur = h->X;
  for (int b = 0; b < 3; ++b) {
    const std::string p = "layer" + std::to_string(b + 2) + ".";
    r = Run{}; r.B = B; r.T = T; r.L = L(p + "bn1"); r.x = cur; r.y = h->Hh;
    if ((rc = launch(r, stream))) return rc;
    if ((rc = xvb_res2net_block_ex(h->Hh.hi, h->Hh.lo, C, m->res_w[b].hi, m->res_w[b].lo, m->res_bias[b], m->res_scale[b],
                                   m->res_shift[b], m->dilation[b], m->scale, h->R.hi, h->R.lo, C, B, T, C / m->scale, stream)))
      return rc;
    r = Run{}; r.B = B; r.T = T; r.L = L(p + "bn2"); r.x = h->R; r.y = h->Z;
    if ((rc = launch(r, stream))) return rc;
    if ((rc = xvb_plane_mean(h->Z.hi, h->Z.lo, C, B, T, C, h->zmean, h->zm.hi, h->zm.lo, C, stream))) return rc;
    if (small_ok(L(p + "se1")) && small_ok(L(p + "se2"))) {
      rc = small_layer(L(p + "se1"), h->zmean, C, B, h->s1f, m->se_dim, 0, stream);
      if (rc) return rc;
      rc = small_layer(L(p + "se2"), h->s1f, m->se_dim, B, h->gate, C, XVB_SIGMOID, stream);
      if (rc) return rc;
    } else {
      r = Run{}; r.B = B; r.T = 1; r.L = L(p + "se1"); r.x = h->zm; r.y = h->s1;
      if ((rc = launch(r, stream))) return rc;
      r = Run{}; r.B = B; r.T = 1; r.L = L(p + "se2"); r.x = h->s1; r.y_f32 = h->gate; r.ldyf = C; r.extra_flags = XVB_SIGMOID;
      if ((rc = launch(r, stream))) return rc;
    }
    const bool last = b == 2;
    const View slot = h->CAT.slice(C * b);
    if ((rc = xvb_se_apply(h->Z.hi, h->Z.lo, C, cur.hi, cur.lo, cur.ld, h->gate, slot.hi, slot.lo, slot.ld,
                           last ? nullptr : h->N.hi, last ? nullptr : h->N.lo, C, B, T, C, stream)))
      return rc;
    cur = h->N;
  }
  r = Run{}; r.B = B; r.T = T; r.L = L("mfa"); r.x = h->CAT; r.y = h->M; r.y_f32 = h->MF; r.ldyf = D;
  if ((rc = launch(r, stream))) return rc;
  if (m->mq) {
    if ((rc = mqmha_pool(h, B, T, stream))) return rc;
  } else {
  if ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 1, h->gstat, h->gp.hi, h->gp.lo, 2 * D, stream))) return rc;
  if (small_ok(L("att_gs"))) {
    rc = small_layer(L("att_gs"), h->gstat, 2 * D, B, h->ub, m->H, 0, stream);
      if (rc) return rc;
  } else {
    r = Run{}; r.B = B; r.T = 1; r.L = L("att_gs"); r.x = h->gp; r.y_f32 = h->ub; r.ldyf = m->H;
    if ((rc = launch(r, stream))) return rc;
  }
  r = Run{}; r.B = B; r.T = T; r.L = L("att_x"); r.x = h->M; r.y = h->A1; r.utt_bias = h->ub; r.ld_utt = m->H; r.extra_flags = XVB_TANH;
  if ((rc = launch(r, stream))) return rc;
  r = Run{}; r.B = B; r.T = T; r.L = L("att2"); r.x = h->A1; r.y_f32 = h->LOG; r.ldyf = D;
  if ((rc = launch(r, stream))) return rc;
  if ((rc = xvb_attn_stats_pool(h->LOG, D, h->MF, D, B, T, D, 1e-5f, h->pstat, h->pp.hi, h->pp.lo, 2 * D, stream))) return rc;
  }
  if (const ELayer* fc1 = L("fc1")) {              // fc1 [-> fc2] on CUDA cores (fp32)
    const ELayer* fc2 = L("fc2");
    rc = small_layer(fc1, h->pstat, m->P2, B, fc2 ? h->f1 : emb, fc1->Cout, 0, stream);
    if (rc) return rc;
    if (fc2) {
      XVB_CHECK_ARG(fc2->w_f32, "xvb_ecapa_extract: 'fc2' after 'fc1' needs an input width that is a multiple of 4");
      rc = small_layer(fc2, h->f1, fc1->Cout, B, emb, m->E, 0, stream);
      if (rc) return rc;
    }
  } else if (small_ok(L("fc2"))) {
    rc = small_layer(L("fc2"), h->pstat, m->P2, B, emb, m->E, 0, stream);
      if (rc) return rc;
  } else {
    r = Run{}; r.B = B; r.T = 1; r.L = L("fc2"); r.x = h->pp; r.y_f32 = emb; r.ldyf = m->E;   // reads the first P of P2 columns
    if ((rc = launch(r, stream))) return rc;
  }
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

extern "C" int xvb_ecapa_extract_host(xvb_ecapa_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream) {
  return Shard<xvb_ecapa>::extract_host(h, feats_host, B, T, emb_host, stream, "xvb_ecapa_extract_host");
}

// A whole shard of N equal-length utterances in `batch`-utterance batches (the reference's caller loop,
// extract_embeddings.py:73-83), device-resident / through pinned host buffers with the copies overlapped (shard.cuh).
extern "C" int xvb_ecapa_set_gather(xvb_ecapa_t* h, float* const* tables, int ntables, int64_t row0, int64_t ld) {
  XVB_CHECK_ARG(finalized(h), "xvb_ecapa_set_gather: bad arguments");
  return h->shard.set_gather(tables, ntables, row0, ld, h->m->E, "xvb_ecapa_set_gather");
}

extern "C" int xvb_ecapa_extract_shard(xvb_ecapa_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream) {
  return Shard<xvb_ecapa>::device(h, feats, N, T, batch, emb, stream, false, "xvb_ecapa_extract_shard");
}

extern "C" int xvb_ecapa_extract_shard_host(xvb_ecapa_t* h, const float* feats_host, int64_t N, int T, int batch, float* emb_host,
                                            void* stream) {
  return Shard<xvb_ecapa>::host(h, feats_host, N, T, batch, emb_host, stream, false, "xvb_ecapa_extract_shard_host");
}

// ---- .xvbm files for ECAPA ("XVBE0001"): dims, then named layer records -------------------------------------
// "XVBE0002" (MQMHA pooling): the same with the pooling record {num_head, num_q, hidden, share, affine_layers,
// time_attention, stddev} after the dims; layers of grouped convs are stored as the state_dict holds them.
extern "C" int xvb_ecapa_save(const xvb_ecapa_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_ecapa_save: model not finalized");
  const Model* m = h->m.get();
  FILE* f = fopen(path, "wb");
  XVB_CHECK_ARG(f, "xvb_ecapa_save: cannot open '%s'", path);
  bool ok = fwrite(m->mq ? "XVBE0002" : "XVBE0001", 1, 8, f) == 8;
  const int32_t hd[6] = {m->feat_dim, m->C, m->D, m->H, m->E, (int32_t)m->order.size()};
  ok = ok && fwrite(hd, 4, 6, f) == 6;
  if (m->mq) {
    const int32_t pr[7] = {m->mq_heads, m->mq_q, m->mq_hidden, m->mq_share, m->mq_layers, m->mq_tatt, m->mq_stddev};
    ok = ok && fwrite(pr, 4, 7, f) == 7;
  }
  for (const std::string& n : m->order) {
    const ELayer& L = m->layers.at(n);
    const int32_t nl = (int32_t)n.size();
    const int32_t rec[7] = {L.Cout, L.Cin, L.ntaps, L.tot, L.flags, (int32_t)!L.hb.empty(), (int32_t)!L.hs.empty()};
    ok = ok && fwrite(&nl, 4, 1, f) == 1 && fwrite(n.data(), 1, n.size(), f) == n.size() && fwrite(rec, 4, 7, f) == 7 &&
         fwrite(L.ctx, 4, L.ntaps, f) == (size_t)L.ntaps && fwrite(L.hw.data(), 4, L.hw.size(), f) == L.hw.size();
    if (!L.hb.empty()) ok = ok && fwrite(L.hb.data(), 4, L.hb.size(), f) == L.hb.size();
    if (!L.hs.empty()) ok = ok && fwrite(L.hs.data(), 4, L.hs.size(), f) == L.hs.size() && fwrite(L.ht.data(), 4, L.ht.size(), f) == L.ht.size();
  }
  ok = fclose(f) == 0 && ok;
  XVB_CHECK_ARG(ok, "xvb_ecapa_save: write to '%s' failed", path);
  return XVB_OK;
}

extern "C" int xvb_ecapa_load(xvb_ecapa_t** out, const char* path) {
  XVB_CHECK_ARG(out && path, "xvb_ecapa_load: null argument");
  FILE* f = fopen(path, "rb");
  XVB_CHECK_ARG(f, "xvb_ecapa_load: cannot open '%s'", path);
  auto rd = [&](void* p, size_t n) { return fread(p, 1, n, f) == n; };
  char magic[8];
  int32_t hd[6];
  xvb_ecapa_t* h = nullptr;
  int rc = XVB_EINVAL;
  do {
    int32_t pr[7];
    const bool ok_magic = rd(magic, 8) && (memcmp(magic, "XVBE0001", 8) == 0 || memcmp(magic, "XVBE0002", 8) == 0);
    const bool mq = ok_magic && magic[7] == '2';
    if (!ok_magic || !rd(hd, sizeof hd) || hd[5] < 1 || hd[5] > 256 || (mq && !rd(pr, sizeof pr))) {
      set_error("xvb_ecapa_load: '%s' is not an XVBE0001 / XVBE0002 file", path);
      break;
    }
    if ((rc = xvb_ecapa_create(&h, hd[0], hd[1], hd[2], hd[3], hd[4]))) break;
    if (mq && (rc = xvb_ecapa_set_mqmha(h, pr[0], pr[1], pr[2], pr[3], pr[4], pr[5], pr[6]))) break;
    std::vector<float> w, b, s, t;
    for (int i = 0; i < hd[5] && rc == XVB_OK; ++i) {
      int32_t nl = 0, rec[7], ctx[XVB_MAX_TAPS];
      char name[128];
      bool ok = rd(&nl, 4) && nl > 0 && nl < 127 && rd(name, (size_t)nl) && rd(rec, sizeof rec) && rec[0] > 0 && rec[1] > 0 &&
                rec[2] >= 1 && rec[2] <= XVB_MAX_TAPS && rec[3] >= rec[2] && rec[3] < 4096 && rd(ctx, 4 * (size_t)rec[2]);
      if (ok) {
        name[nl] = 0;
        w.resize((size_t)rec[0] * rec[1] * rec[3]);
        ok = rd(w.data(), w.size() * 4);
        if (ok && rec[5]) { b.resize(rec[0]); ok = rd(b.data(), b.size() * 4); }
        if (ok && rec[6]) { s.resize(rec[0]); t.resize(rec[0]); ok = rd(s.data(), s.size() * 4) && rd(t.data(), t.size() * 4); }
      }
      if (!ok) { set_error("xvb_ecapa_load: '%s' is truncated or corrupt at layer %d", path, i); rc = XVB_EINVAL; break; }
      rc = xvb_ecapa_set_layer(h, name, rec[0], rec[1], ctx, rec[2], w.data(), rec[5] ? b.data() : nullptr,
                               rec[6] ? s.data() : nullptr, rec[6] ? t.data() : nullptr, rec[4]);
    }
    if (rc == XVB_OK) rc = xvb_ecapa_finalize(h);
  } while (0);
  fclose(f);
  if (rc != XVB_OK) { if (h) xvb_ecapa_destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}

extern "C" void xvb_ecapa_destroy(xvb_ecapa_t* h) { delete h; }
