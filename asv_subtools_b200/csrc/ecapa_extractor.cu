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
// egrecho's EcapaXvector (subtools2/egrecho/models/ecapa/ecapa_xvector.py:420-427) chains its blocks instead
// (xvb_ecapa_set_chained): block b + 1 reads block b's output straight from its slot of the MFA input, at row pitch
// 3C, as the input of its first 1x1 layer and as its residual, and no running sum is written.
//
// The launcher model of runEcapaXvector.py (pytorch/model/ecapa-tdnn-xvector.py) pools without global context
// (xvb_ecapa_set_attention(h, 0, 1e-9f)): attention conv 1 reads x alone, with its own bias, and no ReLU or BN before the
// tanh, so the global mean/std pass and "att_gs" are left out, and the weighted std is floored at the given variance.
//
// Layers are handed over by NAME with the weights as the state_dict stores them (host fp32, eval BatchNorm
// folded to scale/shift by the caller); the two derived layers of the attention conv ("att_x": its columns
// over x, "att_gs": its columns over [mean | std] plus the bias) and "fc2" (bn_stats folded into its weight)
// are prepared by the caller -- see the Python blueprint.  The handle keeps the layers as handed over and builds the
// model from them at finalize; xvb_ecapa_save writes them back (the XVBE0001 / XVBE0002 / XVBG0001 layouts are in
// model_file.cpp, with XVBE0003 for the attention without global context).
#include <cuda_runtime.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "records.cuh"
#include "shard.cuh"

// The model types are local to this file: each family has its own Model.
namespace {

using namespace xvb;

struct ELayer : Affine {
  float* w_f32 = nullptr;   // (Cout, Cin) fp32 as stored, kept for one-tap layers: the segment-level ones run on CUDA cores
};

// One SE-Res2Net block ("layer2." .. "layer4."): its 1x1 convs and SE gate, and its scale - 1 Res2Net convs ("res0" ..)
// stacked for the chain kernel, packed weights along rows and parameters back to back.
struct Block {
  ELayer bn1, bn2, se1, se2;
  Planes res_w;
  float* res_bias = nullptr;
  float* res_scale = nullptr;
  float* res_shift = nullptr;
  int dilation = 0;
};

// split planes with their row pitch
struct View {
  uint16_t* hi = nullptr;
  uint16_t* lo = nullptr;
  int64_t ld = 0;
  View slice(int c0) const { return View{hi + c0, lo + c0, ld}; }
};

struct Config {
  int feat_dim = 0, ldf = 0, C = 0, D = 0, H = 0, E = 0, scale = 8;
  // multi-query multi-head attention pooling (xvb_ecapa_set_mqmha); mq == 0: ECAPA's own attentive pooling
  int mq = 0, mq_heads = 1, mq_q = 1, mq_hidden = 0, mq_share = 0, mq_layers = 2, mq_tatt = 1, mq_stddev = 1;
  // residual form (xvb_ecapa_set_chained): 0 dense, block b + 1 reads x + x1 (+ x2); 1 chained, it reads block b's output
  int chained = 0;
  // attentive pooling (xvb_ecapa_set_attention): global context (1: [x | mean | std] into the first attention conv) and the
  // variance floor of the pooled std
  int gctx = 1;
  float floor = 1e-5f;
  bool attention_set = false;   // xvb_ecapa_set_attention was called (it excludes set_mqmha and set_chained)
  // widths derived from the pooling: att_x outputs AX, the logits NL (row pitch ldlog), the pooled statistics P of the
  // P2-wide [mean | std] buffer (default model: AX = H, NL = D, P = P2 = 2D)
  int AX = 0, NL = 0, ldlog = 0, P = 0, P2 = 0;
};

// The layers and what finalize fixes; shared read-only by a handle and its second shard lane once finalized.
struct Model {
  Config cfg;
  std::vector<TapRec> recs;   // as handed over, in order
  // built at finalize, by role; a layer that the configuration does without has Cout 0
  ELayer layer1;
  Block blocks[3];
  ELayer mfa, att_x, att_gs, att2, fc1, fc2;
  int se_dim = 0, fc1_dim = 0;
  Im2col im2col;   // layer1 as an im2col view (records.cuh)
  Weights dev{"xvb_ecapa_finalize"};
};

}  // namespace

using namespace xvb;

struct xvb_ecapa : Handle<Model> {
  // workspace, each buffer grown to the largest call seen: the plane buffers up to kA1, then the fp32 ones
  enum { kIn, kX, kH, kR, kZ, kN, kCat, kM, kA1, kMF, kLog, kGate, kUb, kZmean, kGstat, kPstat, kS1f, kF1, kBufs };
  Workspace<kBufs> ws;
  // the workspace's buffers as reserve last left them: planes with their row pitch, and fp32
  View in, X, Hh, R, Z, N, CAT, M, A1;
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
  static int feat_dim(const xvb_ecapa* h) { return h->m->cfg.feat_dim; }
  static int embed_dim(const xvb_ecapa* h) { return h->m->cfg.E; }
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
  m->cfg.feat_dim = feat_dim; m->cfg.ldf = (int)round_up(feat_dim, 8);
  m->cfg.C = channels; m->cfg.D = mfa_dim; m->cfg.H = att_hidden; m->cfg.E = embed_dim;
  m->cfg.AX = att_hidden; m->cfg.NL = mfa_dim; m->cfg.ldlog = mfa_dim; m->cfg.P = 2 * mfa_dim; m->cfg.P2 = 2 * mfa_dim;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_ecapa_set_mqmha(xvb_ecapa_t* h, int num_head, int num_q, int hidden, int share, int affine_layers,
                                   int time_attention, int stddev) {
  XVB_CHECK_ARG(is_draft(h) && h->draft->recs.empty(), "xvb_ecapa_set_mqmha: call it between xvb_ecapa_create and the first set_layer");
  Model* m = h->draft;
  XVB_CHECK_ARG(!m->cfg.attention_set, "xvb_ecapa_set_mqmha: the model's attentive pooling is set by xvb_ecapa_set_attention");
  XVB_CHECK_ARG(num_head >= 1 && num_q >= 1 && hidden >= 1 && (affine_layers == 1 || affine_layers == 2) && m->cfg.D % num_head == 0 &&
                (m->cfg.D / num_head) % 4 == 0 && hidden * num_head * num_q == m->cfg.H,
                "xvb_ecapa_set_mqmha: need %d channels in heads of a multiple of 4, 1 or 2 affine layers and att_hidden = "
                "hidden * num_head * num_q (= %d)", m->cfg.D, m->cfg.H);
  const int cg = m->cfg.D / num_head, hq = num_head * num_q;
  m->cfg.mq = 1; m->cfg.mq_heads = num_head; m->cfg.mq_q = num_q; m->cfg.mq_hidden = hidden; m->cfg.mq_share = share ? 1 : 0;
  m->cfg.mq_layers = affine_layers; m->cfg.mq_tatt = time_attention ? 1 : 0; m->cfg.mq_stddev = stddev ? 1 : 0;
  m->cfg.NL = hq * (share ? 1 : cg);
  m->cfg.ldlog = (int)round_up(m->cfg.NL, 4);
  m->cfg.AX = affine_layers == 2 ? m->cfg.H : m->cfg.NL;
  XVB_CHECK_ARG(!time_attention || m->cfg.AX % 4 == 0, "xvb_ecapa_set_mqmha: the time-constant columns of the first attention conv "
                "become a per-utterance bias, which needs a multiple of 4 outputs (got %d)", m->cfg.AX);
  m->cfg.P2 = 2 * num_q * m->cfg.D;
  m->cfg.P = stddev ? m->cfg.P2 : num_q * m->cfg.D;
  return XVB_OK;
}

extern "C" int xvb_ecapa_set_chained(xvb_ecapa_t* h, int chained) {
  XVB_CHECK_ARG(is_draft(h) && h->draft->recs.empty(), "xvb_ecapa_set_chained: call it between xvb_ecapa_create and the first set_layer");
  XVB_CHECK_ARG(chained == 0 || chained == 1, "xvb_ecapa_set_chained: chained must be 0 or 1, got %d", chained);
  XVB_CHECK_ARG(!h->draft->cfg.attention_set, "xvb_ecapa_set_chained: the chained form has MQMHA pooling, not xvb_ecapa_set_attention's");
  h->draft->cfg.chained = chained;
  return XVB_OK;
}

extern "C" int xvb_ecapa_set_attention(xvb_ecapa_t* h, int global_context, float floor) {
  XVB_CHECK_ARG(is_draft(h) && h->draft->recs.empty(), "xvb_ecapa_set_attention: call it between xvb_ecapa_create and the first set_layer");
  Config& c = h->draft->cfg;
  XVB_CHECK_ARG(!c.mq && !c.chained, "xvb_ecapa_set_attention: not with xvb_ecapa_set_mqmha or xvb_ecapa_set_chained, which have "
                "their own attention and residual forms");
  XVB_CHECK_ARG(global_context == 0 || global_context == 1, "xvb_ecapa_set_attention: global_context must be 0 or 1, got %d",
                global_context);
  XVB_CHECK_ARG(floor > 0.f && floor < 1.f, "xvb_ecapa_set_attention: the variance floor must lie in (0, 1), got %g", (double)floor);
  c.gctx = global_context; c.floor = floor; c.attention_set = true;
  return XVB_OK;
}

// Groups of a layer as the state_dict stores it: the MQMHA attention convs are grouped (pooling.py:665-698)
static int layer_groups(const Config& c, const std::string& n) {
  if (!c.mq) return 1;
  if (n == "att_x") return c.mq_heads;
  if (n == "att2") return c.mq_heads * c.mq_q;
  return 1;
}

static const TapRec* find(const std::vector<TapRec>& recs, const std::string& n) {
  for (const TapRec& r : recs)
    if (r.name == n) return &r;
  return nullptr;
}

extern "C" int xvb_ecapa_set_layer(xvb_ecapa_t* h, const char* name, int Cout, int Cin, const int* context_host, int ntaps,
                                   const float* w_host, const float* bias_host, const float* bn_scale_host,
                                   const float* bn_shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && w_host && context_host, "xvb_ecapa_set_layer: bad arguments or finalized model");
  Model* m = h->draft;
  XVB_CHECK_ARG(Cout > 0 && Cin > 0 && ntaps >= 1 && ntaps <= XVB_MAX_TAPS, "xvb_ecapa_set_layer(%s): bad shape", name);
  XVB_CHECK_ARG(!(flags & XVB_BN) || (bn_scale_host && bn_shift_host), "xvb_ecapa_set_layer(%s): XVB_BN without scale/shift", name);
  XVB_CHECK_ARG(!find(m->recs, name), "xvb_ecapa_set_layer: layer '%s' set twice", name);
  TapRec r = tap_record(name, Cout, Cin, context_host, ntaps, w_host, bias_host, bn_scale_host, bn_shift_host, flags);
  const int groups = layer_groups(m->cfg, name);
  XVB_CHECK_ARG(groups == 1 || (ntaps == 1 && r.tot() == 1 && Cout % groups == 0),
                "xvb_ecapa_set_layer(%s): a grouped layer is a 1x1 conv with Cout divisible by its %d groups", name, groups);
  m->recs.push_back(std::move(r));
  return XVB_OK;
}

// r on the device as L.  A grouped layer (the MQMHA attention convs, r.Cin the per-group width) is packed compactly for
// the layer kernel's grouped mode, or as its block-diagonal expansion when the shape does not fit that mode.
static int build_layer(Model* m, const TapRec& r, ELayer* L) {
  const int G = layer_groups(m->cfg, r.name), cin = r.Cin * G;
  int rc;
  if (G > 1 && !xvb_tdnn_grouped_fits(cin, r.Cout, G)) {
    const int co = r.Cout / G;
    std::vector<float> dense((size_t)r.Cout * cin, 0.f);
    for (int n = 0; n < r.Cout; ++n)
      memcpy(&dense[(size_t)n * cin + (size_t)(n / co) * r.Cin], &r.w[(size_t)n * r.Cin], r.Cin * sizeof(float));
    rc = pack_affine(m->dev, L, dense, r.Cout, cin, r.ctx, r.ntaps, r.b, r.s, r.t, r.flags);
  } else {
    rc = pack_affine(m->dev, L, r.w, r.Cout, cin, r.ctx, r.ntaps, r.b, r.s, r.t, r.flags, G);
  }
  if (rc) return rc;
  // one tap: (Cout, Cin, 1) is the (N, K) matrix xvb_small_affine takes
  if (r.tot() == 1 && r.Cin % 4 == 0 && G == 1 && (rc = m->dev.upload(&L->w_f32, r.w))) return rc;
  return XVB_OK;
}

// The model of the draft's configuration and layers, each layer built into its role.
static int build(Model* m, const std::vector<TapRec>& recs) {
  const Config& c = m->cfg;
  const int C = c.C, W = C / c.scale;
  // *out: the layer n, which must have this shape
  auto need = [&](const std::string& n, int cin, int cout, int ntaps, const TapRec** out) -> int {
    const TapRec* L = *out = find(recs, n);
    XVB_CHECK_ARG(L, "xvb_ecapa_finalize: layer '%s' is missing", n.c_str());
    XVB_CHECK_ARG(L->Cin == cin && L->Cout == cout && L->ntaps == ntaps, "xvb_ecapa_finalize: layer '%s' is %d->%d x%d taps, expected %d->%d x%d",
                  n.c_str(), L->Cin, L->Cout, L->ntaps, cin, cout, ntaps);
    return XVB_OK;
  };
  auto take = [&](const std::string& n, int cin, int cout, int ntaps, ELayer* L) -> int {
    const TapRec* r;
    const int rc = need(n, cin, cout, ntaps, &r);
    return rc ? rc : build_layer(m, *r, L);
  };
  const TapRec* r = find(recs, "layer1");
  int rc = take("layer1", c.feat_dim, C, r ? r->ntaps : 5, &m->layer1);
  if (rc) return rc;
  for (int b = 0; b < 3; ++b) {
    Block& k = m->blocks[b];
    const std::string p = "layer" + std::to_string(b + 2) + ".";
    if ((rc = take(p + "bn1", C, C, 1, &k.bn1)) || (rc = take(p + "bn2", C, C, 1, &k.bn2))) return rc;
    const TapRec* se1 = find(recs, p + "se1");
    XVB_CHECK_ARG(se1 && se1->Cin == C, "xvb_ecapa_finalize: layer '%sse1' is missing", p.c_str());
    if (b == 0) m->se_dim = se1->Cout;
    XVB_CHECK_ARG(se1->Cout == m->se_dim && m->se_dim % 8 == 0, "xvb_ecapa_finalize: SE bottleneck must be a multiple of 8 and equal in all blocks");
    if ((rc = build_layer(m, *se1, &k.se1)) || (rc = take(p + "se2", m->se_dim, C, 1, &k.se2))) return rc;
    // the scale-1 Res2Net layers, each packed straight into its slot of the block's stack
    const size_t pw = (size_t)xvb_packed_weight_elems(W, W, 3);
    if ((rc = m->dev.alloc(&k.res_w.hi, pw * (c.scale - 1))) || (rc = m->dev.alloc(&k.res_w.lo, pw * (c.scale - 1))) ||
        (rc = m->dev.alloc(&k.res_bias, (size_t)W * (c.scale - 1))) || (rc = m->dev.alloc(&k.res_scale, (size_t)W * (c.scale - 1))) ||
        (rc = m->dev.alloc(&k.res_shift, (size_t)W * (c.scale - 1))))
      return rc;
    for (int i = 0; i < c.scale - 1; ++i) {
      const std::string n = p + "res" + std::to_string(i);
      if ((rc = need(n, W, W, 3, &r))) return rc;
      XVB_CHECK_ARG(r->ctx[0] == -r->ctx[2] && r->ctx[1] == 0 && !r->b.empty() && !r->s.empty() && (r->flags & XVB_RELU),
                    "xvb_ecapa_finalize: '%s' must be a [-d,0,d] TDNN-ReLU-BN layer with bias", n.c_str());
      if (i == 0) k.dilation = r->ctx[2];
      XVB_CHECK_ARG(r->ctx[2] == k.dilation, "xvb_ecapa_finalize: '%s' has another dilation than its block", n.c_str());
      if ((rc = m->dev.pack_into(Planes{k.res_w.hi + pw * i, k.res_w.lo + pw * i}, r->w, W, W, r->tot(), r->ctx, 3))) return rc;
      XVB_CUDA(cudaMemcpy(k.res_bias + (size_t)W * i, r->b.data(), W * sizeof(float), cudaMemcpyHostToDevice));
      XVB_CUDA(cudaMemcpy(k.res_scale + (size_t)W * i, r->s.data(), W * sizeof(float), cudaMemcpyHostToDevice));
      XVB_CUDA(cudaMemcpy(k.res_shift + (size_t)W * i, r->t.data(), W * sizeof(float), cudaMemcpyHostToDevice));
    }
  }
  rc = take("mfa", 3 * C, c.D, 1, &m->mfa);
  if (rc) return rc;
  if (!c.mq) {
    if ((rc = take("att_x", c.D, c.H, 1, &m->att_x)) || (c.gctx && (rc = take("att_gs", 2 * c.D, c.H, 1, &m->att_gs))) ||
        (rc = take("att2", c.H, c.D, 1, &m->att2)))
      return rc;
    XVB_CHECK_ARG(c.gctx || !find(recs, "att_gs"), "xvb_ecapa_finalize: 'att_gs' in an attention without global context");
  } else {   // per-group input widths: att_x reads a head's Cg channels of x, att2 one query's hidden units
    rc = take("att_x", c.D / c.mq_heads, c.AX, 1, &m->att_x);
    if (rc) return rc;
    if (c.mq_layers == 2 && (rc = take("att2", c.mq_hidden, c.NL, 1, &m->att2))) return rc;
    XVB_CHECK_ARG(c.mq_layers == 2 || !find(recs, "att2"), "xvb_ecapa_finalize: one-layer attention has no 'att2'");
    if (c.mq_tatt && (rc = take("att_gs", (c.mq_stddev ? 2 : 1) * c.D, c.AX, 1, &m->att_gs))) return rc;
    XVB_CHECK_ARG(c.mq_tatt || !find(recs, "att_gs"), "xvb_ecapa_finalize: 'att_gs' without time attention");
  }
  // segment level (ecapa_tdnn_xvector.py:412-422): [fc1 ->] [fc2]; "far" hands over fc1 alone, fc1=False fc2 alone
  if (const TapRec* fc1 = find(recs, "fc1")) {
    if ((rc = build_layer(m, *fc1, &m->fc1))) return rc;
    XVB_CHECK_ARG(fc1->Cin == c.P && fc1->ntaps == 1 && m->fc1.w_f32, "xvb_ecapa_finalize: 'fc1' must be a one-tap layer over the %d pooled statistics", c.P);
    if (find(recs, "fc2")) {
      rc = take("fc2", fc1->Cout, c.E, 1, &m->fc2);
      if (rc) return rc;
    } else {
      XVB_CHECK_ARG(fc1->Cout == c.E, "xvb_ecapa_finalize: 'fc1' alone must produce the %d-d embedding", c.E);
    }
    m->fc1_dim = fc1->Cout;
  } else {
    rc = take("fc2", c.P, c.E, 1, &m->fc2);
    if (rc) return rc;
  }
  m->im2col = im2col_choice(m->layer1.ctx, m->layer1.ntaps, c.feat_dim);
  return XVB_OK;
}

extern "C" int xvb_ecapa_finalize(xvb_ecapa_t* h) {
  const int rc = publish_built(h, build, "xvb_ecapa_finalize");
  if (rc == XVB_OK) h->im2col = h->m->im2col;
  return rc;
}

extern "C" int xvb_ecapa_embed_dim(const xvb_ecapa_t* h) { return h ? h->m->cfg.E : XVB_EINVAL; }
extern "C" int xvb_ecapa_feat_dim(const xvb_ecapa_t* h) { return h ? h->m->cfg.feat_dim : XVB_EINVAL; }
extern "C" int xvb_ecapa_last_launches(const xvb_ecapa_t* h) { return h ? h->last_launches : 0; }

static int reserve(xvb_ecapa* h, int B, int T) {
  using H = xvb_ecapa;
  const Model* m = h->m.get();
  const size_t b = (size_t)B, f = (size_t)B * T, C = (size_t)m->cfg.C, D = (size_t)m->cfg.D;
  const size_t need[H::kBufs] = {(f + b * (h->im2col.pad_front + h->im2col.pad_back)) * m->cfg.ldf, f * C, f * C, f * C, f * C,
                                 f * C, f * 3 * C, f * D, f * m->cfg.H, f * D, f * m->cfg.ldlog, b * C, b * m->cfg.AX, b * C,
                                 b * 2 * D, b * m->cfg.P2, b * m->se_dim, b * m->fc1_dim};
  bool planes[H::kBufs];
  for (int i = 0; i < H::kBufs; ++i) planes[i] = i <= H::kA1;
  uint64_t grown;
  const int rc = h->ws.reserve(need, planes, &grown);
  if (rc) return rc;
  auto view = [&](int i, int64_t ld) { const Planes p = h->ws.planes(i); return View{p.hi, p.lo, ld}; };
  h->in = view(H::kIn, m->cfg.ldf); h->X = view(H::kX, C); h->Hh = view(H::kH, C); h->R = view(H::kR, C);
  h->Z = view(H::kZ, C); h->N = view(H::kN, C); h->CAT = view(H::kCat, 3 * C); h->M = view(H::kM, D);
  h->A1 = view(H::kA1, m->cfg.H);
  h->MF = h->ws.f32(H::kMF); h->LOG = h->ws.f32(H::kLog); h->gate = h->ws.f32(H::kGate); h->ub = h->ws.f32(H::kUb);
  h->zmean = h->ws.f32(H::kZmean); h->gstat = h->ws.f32(H::kGstat); h->pstat = h->ws.f32(H::kPstat);
  h->s1f = h->ws.f32(H::kS1f); h->f1 = h->ws.f32(H::kF1);
  return XVB_OK;
}

namespace {
// The layer-kernel arguments of L over x at (B, T) into the planes y and / or the fp32 yf (row pitch ldyf)
xvb_tdnn_args_t layer_args(const ELayer& L, const View& x, int B, int T, const View& y, float* yf = nullptr, int64_t ldyf = 0) {
  xvb_tdnn_args_t a = affine_args(L, Planes{x.hi, x.lo}, x.ld, B, T);
  a.y_hi = y.hi; a.y_lo = y.lo; a.ldy = y.ld;
  a.y_f32 = yf; a.ldyf = ldyf;
  return a;
}
// segment-level layer (one row per utterance) on CUDA cores: fp32 in, fp32 out
int small_layer(const ELayer* L, const float* x, int64_t ldx, int B, float* y, int64_t ldy, int extra_flags, void* stream) {
  return xvb_small_affine(x, ldx, L->w_f32, B, L->Cin, L->Cout, L->bias, L->scale, L->shift, L->flags | extra_flags, y, ldy,
                          nullptr, nullptr, 0, stream);
}
}  // namespace

// MQMHASP.forward (libs/nnet/pooling.py:627-663) over the mfa output (M planes, MF fp32) into pstat / pp:
// time attention: biased mean | sqrt(clamp(var, 1e-5)) of every channel (egrecho's compute_statistics) -> the
// per-utterance bias of the first attention conv (its [mean_h | std_h] columns, block-diagonal over the heads) ->
// grouped conv over x (ReLU -> BN -> tanh) -> grouped conv to the logits -> softmax over T and weighted moments with
// the head-width map: pooled channel (h*Q + q)*Cg + c is x channel h*Cg + c under the alpha of logit (h*Q + q)[*Cg + c].
static int mqmha_pool(xvb_ecapa* h, int B, int T, void* stream) {
  const Model* m = h->m.get();
  const int D = m->cfg.D, cg = D / m->cfg.mq_heads;
  int rc;
  if (m->cfg.mq_tatt) {
    if ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 0, h->gstat, nullptr, nullptr, 0, stream))) return rc;
    if ((rc = small_layer(&m->att_gs, h->gstat, 2 * D, B, h->ub, m->cfg.AX, 0, stream))) return rc;
  }
  const bool two = m->cfg.mq_layers == 2;
  xvb_tdnn_args_t a = two ? layer_args(m->att_x, h->M, B, T, h->A1)
                          : layer_args(m->att_x, h->M, B, T, View{}, h->LOG, m->cfg.ldlog);
  if (two) a.flags |= XVB_TANH;
  if (m->cfg.mq_tatt) { a.utt_bias = h->ub; a.ld_utt_bias = m->cfg.AX; }
  if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
  if (two) {
    a = layer_args(m->att2, h->A1, B, T, View{}, h->LOG, m->cfg.ldlog);
    if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
  }
  return xvb_attn_head_stats_pool_mq(h->LOG, m->cfg.ldlog, m->cfg.NL, h->MF, D, B, T, D, m->cfg.mq_q * D, m->cfg.mq_share ? cg : 1, cg, m->cfg.mq_q,
                                     1e-5f, 0, h->pstat, nullptr, nullptr, 0, stream);
}

extern "C" int xvb_ecapa_extract(xvb_ecapa_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_ecapa_extract: model not finalized");
  const Model* m = h->m.get();
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_ecapa_extract: bad arguments");
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const long before = g_launches;
  const int C = m->cfg.C, D = m->cfg.D;
  const Im2col& im = h->im2col;
  if (im.on)
    rc = xvb_split_frames(feats, B, T, m->cfg.feat_dim, h->in.hi, h->in.lo, m->cfg.ldf, im.pad_front, im.pad_back, stream);
  else
    rc = xvb_split_f32(feats, (int64_t)B * T, m->cfg.feat_dim, m->cfg.feat_dim, h->in.hi, h->in.lo, m->cfg.ldf, stream);
  if (rc) return rc;
  xvb_tdnn_args_t a = layer_args(m->layer1, h->in, B, T, h->X);
  if (im.on) {   // window of ntaps consecutive frames = one long row of the padded planes
    a.context_host = kTaps; a.ntaps = 1; a.Cin = m->layer1.ntaps * m->layer1.Cin;
    a.x_batch_stride = (int64_t)(T + im.pad_front + im.pad_back) * m->cfg.ldf;
  }
  rc = xvb_tdnn_affine_ex(&a, stream);
  if (rc && im.on) {   // overlapping tensor map refused by the driver: plain path from now on
    h->im2col = Im2col{};
    return xvb_ecapa_extract(h, feats, B, T, emb, stream);
  }
  if (rc) return rc;
  View cur = h->X;
  for (int b = 0; b < 3; ++b) {
    const Block& k = m->blocks[b];
    a = layer_args(k.bn1, cur, B, T, h->Hh);
    if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
    if ((rc = xvb_res2net_block_ex(h->Hh.hi, h->Hh.lo, C, k.res_w.hi, k.res_w.lo, k.res_bias, k.res_scale, k.res_shift,
                                   k.dilation, m->cfg.scale, h->R.hi, h->R.lo, C, B, T, C / m->cfg.scale, stream)))
      return rc;
    a = layer_args(k.bn2, h->R, B, T, h->Z);
    if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
    if ((rc = xvb_plane_mean(h->Z.hi, h->Z.lo, C, B, T, C, h->zmean, nullptr, nullptr, 0, stream)) ||
        (rc = small_layer(&k.se1, h->zmean, C, B, h->s1f, m->se_dim, 0, stream)) ||
        (rc = small_layer(&k.se2, h->s1f, m->se_dim, B, h->gate, C, XVB_SIGMOID, stream)))
      return rc;
    // dense: the running sum x + x1 (+ x2) goes to N for the next block; chained: the next block reads this slot
    const bool next = b < 2 && !m->cfg.chained;
    const View slot = h->CAT.slice(C * b);
    if ((rc = xvb_se_apply(h->Z.hi, h->Z.lo, C, cur.hi, cur.lo, cur.ld, h->gate, slot.hi, slot.lo, slot.ld,
                           next ? h->N.hi : nullptr, next ? h->N.lo : nullptr, C, B, T, C, stream)))
      return rc;
    cur = m->cfg.chained ? slot : h->N;
  }
  a = layer_args(m->mfa, h->CAT, B, T, h->M, h->MF, D);
  if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
  if (m->cfg.mq) {
    if ((rc = mqmha_pool(h, B, T, stream))) return rc;
  } else {
  // global context: the time-constant [mean | std] columns of attention conv 1 become the per-utterance bias
  if (m->cfg.gctx && ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 1, h->gstat, nullptr, nullptr, 0, stream)) ||
                      (rc = small_layer(&m->att_gs, h->gstat, 2 * D, B, h->ub, m->cfg.H, 0, stream))))
    return rc;
  a = layer_args(m->att_x, h->M, B, T, h->A1);
  a.flags |= XVB_TANH;
  if (m->cfg.gctx) { a.utt_bias = h->ub; a.ld_utt_bias = m->cfg.H; }
  if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
  a = layer_args(m->att2, h->A1, B, T, View{}, h->LOG, D);
  if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
  if ((rc = xvb_attn_stats_pool(h->LOG, D, h->MF, D, B, T, D, m->cfg.floor, h->pstat, nullptr, nullptr, 0, stream))) return rc;
  }
  if (m->fc1.Cout) {              // fc1 [-> fc2] on CUDA cores (fp32)
    const ELayer* fc1 = &m->fc1;
    const ELayer* fc2 = m->fc2.Cout ? &m->fc2 : nullptr;
    rc = small_layer(fc1, h->pstat, m->cfg.P2, B, fc2 ? h->f1 : emb, fc1->Cout, 0, stream);
    if (rc) return rc;
    if (fc2) {
      XVB_CHECK_ARG(fc2->w_f32, "xvb_ecapa_extract: 'fc2' after 'fc1' needs an input width that is a multiple of 4");
      rc = small_layer(fc2, h->f1, fc1->Cout, B, emb, m->cfg.E, 0, stream);
      if (rc) return rc;
    }
  } else if ((rc = small_layer(&m->fc2, h->pstat, m->cfg.P2, B, emb, m->cfg.E, 0, stream))) {
    return rc;
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
  return h->shard.set_gather(tables, ntables, row0, ld, h->m->cfg.E, "xvb_ecapa_set_gather");
}

extern "C" int xvb_ecapa_extract_shard(xvb_ecapa_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream) {
  return Shard<xvb_ecapa>::device(h, feats, N, T, batch, emb, stream, false, "xvb_ecapa_extract_shard");
}

extern "C" int xvb_ecapa_extract_shard_host(xvb_ecapa_t* h, const float* feats_host, int64_t N, int T, int batch, float* emb_host,
                                            void* stream) {
  return Shard<xvb_ecapa>::host(h, feats_host, N, T, batch, emb_host, stream, false, "xvb_ecapa_extract_shard_host");
}

extern "C" int xvb_ecapa_save(const xvb_ecapa_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_ecapa_save: model not finalized");
  const Config& c = h->m->cfg;
  XVB_CHECK_ARG(c.mq || !c.chained, "xvb_ecapa_save: an XVBG0001 file holds a chained model with MQMHA pooling");
  std::vector<const TapRec*> layers;
  for (const TapRec& r : h->m->recs) layers.push_back(&r);
  if (c.gctx != 1 || c.floor != 1e-5f) {   // XVBE0003: XVBE0001's header, then the attention of xvb_ecapa_set_attention
    int32_t fbits;
    memcpy(&fbits, &c.floor, sizeof fbits);
    const int32_t head3[8] = {c.feat_dim, c.C, c.D, c.H, c.E, (int32_t)h->m->recs.size(), c.gctx, fbits};
    return save_tap_file("xvb_ecapa_save", path, "XVBE0003", head3, sizeof head3, layers, true);
  }
  const int32_t head[14] = {c.feat_dim, c.C, c.D, c.H, c.E, (int32_t)h->m->recs.size(),   // then XVBE0002's pooling
                            c.mq_heads, c.mq_q, c.mq_hidden, c.mq_share, c.mq_layers, c.mq_tatt, c.mq_stddev,
                            c.chained};                                                   // then XVBG0001's residual form
  const char* magic = c.chained ? "XVBG0001" : c.mq ? "XVBE0002" : "XVBE0001";
  return save_tap_file("xvb_ecapa_save", path, magic, head, (c.chained ? 14 : c.mq ? 13 : 6) * sizeof(int32_t), layers, true);
}

extern "C" void xvb_ecapa_destroy(xvb_ecapa_t* h) { delete h; }
