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
#include <string>
#include <vector>

#include "common.cuh"

namespace xvb {

struct ELayer {
  int Cin = 0, Cout = 0, ntaps = 0, flags = 0, tot = 0;
  int ctx[XVB_MAX_TAPS] = {0};
  uint16_t* w_hi = nullptr;
  uint16_t* w_lo = nullptr;
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

struct Planes {
  uint16_t* hi = nullptr;
  uint16_t* lo = nullptr;
  int64_t ld = 0;
  Planes slice(int c0) const { return Planes{hi + c0, lo + c0, ld}; }
};

template <typename T>
static int ealloc(T** p, size_t n) {
  XVB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
  return XVB_OK;
}

}  // namespace xvb

using namespace xvb;

struct xvb_ecapa {
  int feat_dim = 0, ldf = 0, C = 0, D = 0, H = 0, E = 0, scale = 8, se_dim = 0;
  int dilation[3] = {2, 3, 4};
  bool finalized = false;
  std::map<std::string, ELayer> layers;
  std::vector<std::string> order;   // insertion order, for save()
  // stacked Res2Net parameters per block
  uint16_t* res_w_hi[3] = {nullptr, nullptr, nullptr};
  uint16_t* res_w_lo[3] = {nullptr, nullptr, nullptr};
  float* res_bias[3] = {nullptr, nullptr, nullptr};
  float* res_scale[3] = {nullptr, nullptr, nullptr};
  float* res_shift[3] = {nullptr, nullptr, nullptr};
  // workspace
  long long cap_frames = 0;
  int cap_B = 0;
  std::vector<void*> ws;
  Planes in, X, Hh, R, Z, N, CAT, M, A1, gp, s1, zm, pp;
  float *MF = nullptr, *LOG = nullptr, *gate = nullptr, *ub = nullptr, *zmean = nullptr, *gstat = nullptr, *pstat = nullptr;
  float* s1f = nullptr;   // (B, se_dim) fp32: hidden vector of the SE gate
  float* f1 = nullptr;    // (B, fc1_dim) fp32: output of fc1 when the model has one
  int fc1_dim = 0;
  // multi-query multi-head attention pooling (xvb_ecapa_set_mqmha); mq == 0: ECAPA's own attentive pooling
  int mq = 0, mq_heads = 1, mq_q = 1, mq_hidden = 0, mq_share = 0, mq_layers = 2, mq_tatt = 1, mq_stddev = 1;
  // widths derived from the pooling: att_x outputs AX, the logits NL (row pitch ldlog), the pooled statistics P of the
  // P2-wide [mean | std] buffer (default model: AX = H, NL = D, P = P2 = 2D)
  int AX = 0, NL = 0, ldlog = 0, P = 0, P2 = 0;
  int last_launches = 0;
  float* h_feats = nullptr; float* h_emb = nullptr;   // device staging of xvb_ecapa_extract_host
  size_t h_feats_cap = 0, h_emb_cap = 0;
  // two-slot pipeline of xvb_ecapa_extract_shard_host
  static constexpr int kSlots = 4;    // two device slots per lane: the copy engine runs ahead of both lanes
  float* p_feats[kSlots] = {nullptr, nullptr, nullptr, nullptr}; float* p_emb[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  size_t p_feats_cap[kSlots] = {0, 0, 0, 0}, p_emb_cap[kSlots] = {0, 0, 0, 0};
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_h2d[kSlots] = {nullptr, nullptr, nullptr, nullptr}, ev_done[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  // layer1 as an im2col view over time-padded planes (see extractor.cu): consecutive taps, feat_dim % 16 == 0
  bool im2col_first = false;
  int pad_front = 0, pad_back = 0;
  // two-lane shard pipeline (see extractor.cu): `lane1` shares the weights, owns its workspace; batches alternate
  // between the lanes on two streams so that one batch's bandwidth kernels (plane mean, SE apply, the two pooling
  // passes, staging) run next to the other batch's GEMM CTAs
  xvb_ecapa* lane1 = nullptr;
  bool is_lane = false;
  // replicated embedding table (peer.cu): every batch's rows go to all these copies as soon as they exist
  float* gather_tables[XVB_MAX_PEERS] = {nullptr};
  int gather_n = 0;
  int64_t gather_row0 = 0, gather_ld = 0;
  cudaStream_t lane_stream[2] = {nullptr, nullptr};
  cudaEvent_t ev_lane_start = nullptr, ev_lane_done[2] = {nullptr, nullptr};

  void free_ws() {
    for (void* p : ws) cudaFree(p);
    ws.clear();
    cap_frames = 0; cap_B = 0;
  }
  int planes(Planes* p, size_t rows, int64_t ld) {
    int rc = ealloc(&p->hi, rows * ld);
    if (rc) return rc;
    ws.push_back(p->hi);
    rc = ealloc(&p->lo, rows * ld);
    if (rc) return rc;
    ws.push_back(p->lo);
    p->ld = ld;
    return XVB_OK;
  }
  int f32(float** p, size_t n) {
    int rc = ealloc(p, n);
    if (rc) return rc;
    ws.push_back(*p);
    return XVB_OK;
  }
};

extern "C" int xvb_ecapa_create(xvb_ecapa_t** out, int feat_dim, int channels, int mfa_dim, int att_hidden, int embed_dim) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && feat_dim > 0 && channels > 0 && mfa_dim > 0 && att_hidden > 0 && embed_dim > 0, "xvb_ecapa_create: bad arguments");
  XVB_CHECK_ARG(channels % 64 == 0 && channels / 8 == 128, "xvb_ecapa_create: the Res2Net chain kernel is built for scale 8 x width 128 (channels = 1024), got %d", channels);
  XVB_CHECK_ARG(mfa_dim % 8 == 0 && att_hidden % 8 == 0 && embed_dim % 4 == 0, "xvb_ecapa_create: mfa_dim/att_hidden must be multiples of 8, embed_dim of 4");
  xvb_ecapa* h = new xvb_ecapa();
  h->feat_dim = feat_dim; h->ldf = (int)round_up(feat_dim, 8);
  h->C = channels; h->D = mfa_dim; h->H = att_hidden; h->E = embed_dim;
  h->AX = att_hidden; h->NL = mfa_dim; h->ldlog = mfa_dim; h->P = 2 * mfa_dim; h->P2 = 2 * mfa_dim;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_ecapa_set_mqmha(xvb_ecapa_t* h, int num_head, int num_q, int hidden, int share, int affine_layers,
                                   int time_attention, int stddev) {
  XVB_CHECK_ARG(h && !h->finalized && h->layers.empty(), "xvb_ecapa_set_mqmha: call it between xvb_ecapa_create and the first set_layer");
  XVB_CHECK_ARG(num_head >= 1 && num_q >= 1 && hidden >= 1 && (affine_layers == 1 || affine_layers == 2) && h->D % num_head == 0 &&
                (h->D / num_head) % 4 == 0 && hidden * num_head * num_q == h->H,
                "xvb_ecapa_set_mqmha: need %d channels in heads of a multiple of 4, 1 or 2 affine layers and att_hidden = "
                "hidden * num_head * num_q (= %d)", h->D, h->H);
  const int cg = h->D / num_head, hq = num_head * num_q;
  h->mq = 1; h->mq_heads = num_head; h->mq_q = num_q; h->mq_hidden = hidden; h->mq_share = share ? 1 : 0;
  h->mq_layers = affine_layers; h->mq_tatt = time_attention ? 1 : 0; h->mq_stddev = stddev ? 1 : 0;
  h->NL = hq * (share ? 1 : cg);
  h->ldlog = (int)round_up(h->NL, 4);
  h->AX = affine_layers == 2 ? h->H : h->NL;
  XVB_CHECK_ARG(!time_attention || h->AX % 4 == 0, "xvb_ecapa_set_mqmha: the time-constant columns of the first attention conv "
                "become a per-utterance bias, which needs a multiple of 4 outputs (got %d)", h->AX);
  h->P2 = 2 * num_q * h->D;
  h->P = stddev ? h->P2 : num_q * h->D;
  return XVB_OK;
}

// Groups of a layer as the state_dict stores it: the MQMHA attention convs are grouped (pooling.py:665-698)
static int layer_groups(const xvb_ecapa* h, const std::string& n) {
  if (!h->mq) return 1;
  if (n == "att_x") return h->mq_heads;
  if (n == "att2") return h->mq_heads * h->mq_q;
  return 1;
}

extern "C" int xvb_ecapa_set_layer(xvb_ecapa_t* h, const char* name, int Cout, int Cin, const int* context_host, int ntaps,
                                   const float* w_host, const float* bias_host, const float* bn_scale_host,
                                   const float* bn_shift_host, int flags) {
  XVB_CHECK_ARG(h && !h->finalized && name && w_host && context_host, "xvb_ecapa_set_layer: bad arguments or finalized model");
  XVB_CHECK_ARG(Cout > 0 && Cin > 0 && ntaps >= 1 && ntaps <= XVB_MAX_TAPS, "xvb_ecapa_set_layer(%s): bad shape", name);
  XVB_CHECK_ARG(!(flags & XVB_BN) || (bn_scale_host && bn_shift_host), "xvb_ecapa_set_layer(%s): XVB_BN without scale/shift", name);
  XVB_CHECK_ARG(h->layers.find(name) == h->layers.end(), "xvb_ecapa_set_layer: layer '%s' set twice", name);
  ELayer L;
  L.Cin = Cin; L.Cout = Cout; L.ntaps = ntaps; L.flags = flags;
  for (int i = 0; i < ntaps; ++i) L.ctx[i] = context_host[i];
  const int left = L.ctx[0] < 0 ? L.ctx[0] : 0, right = L.ctx[ntaps - 1] > 0 ? L.ctx[ntaps - 1] : 0;
  L.tot = right - left + 1;
  const size_t wn = (size_t)Cout * Cin * L.tot;
  L.hw.assign(w_host, w_host + wn);
  if (bias_host) L.hb.assign(bias_host, bias_host + Cout);
  if (flags & XVB_BN) { L.hs.assign(bn_scale_host, bn_scale_host + Cout); L.ht.assign(bn_shift_host, bn_shift_host + Cout); }
  L.groups = layer_groups(h, name);
  XVB_CHECK_ARG(L.groups == 1 || (ntaps == 1 && L.tot == 1 && Cout % L.groups == 0),
                "xvb_ecapa_set_layer(%s): a grouped layer is a 1x1 conv with Cout divisible by its %d groups", name, L.groups);
  // a grouped shape the layer kernel's grouped mode does not take runs as its block-diagonal expansion
  L.expanded = L.groups > 1 && !xvb_tdnn_grouped_fits(Cin * L.groups, Cout, L.groups);
  std::vector<float> dense;
  const float* w_pack = w_host;
  int cin_pack = Cin;
  if (L.expanded) {
    const int G = L.groups, co = Cout / G;
    cin_pack = Cin * G;
    dense.assign((size_t)Cout * cin_pack, 0.f);
    for (int n = 0; n < Cout; ++n)
      memcpy(&dense[(size_t)n * cin_pack + (size_t)(n / co) * Cin], w_host + (size_t)n * Cin, Cin * sizeof(float));
    w_pack = dense.data();
  }
  const size_t wpn = (size_t)Cout * cin_pack * L.tot;
  float* w_dev = nullptr;
  int rc = ealloc(&w_dev, wpn);
  if (rc) return rc;
  XVB_CUDA(cudaMemcpy(w_dev, w_pack, wpn * sizeof(float), cudaMemcpyHostToDevice));
  const size_t pn = (size_t)xvb_packed_weight_elems(Cout, cin_pack, ntaps);
  if ((rc = ealloc(&L.w_hi, pn)) || (rc = ealloc(&L.w_lo, pn))) return rc;
  rc = xvb_pack_tdnn_weight(w_dev, Cout, cin_pack, L.tot, left, L.ctx, ntaps, L.w_hi, L.w_lo, nullptr);
  if (rc) return rc;
  XVB_CUDA(cudaDeviceSynchronize());
  if (L.tot == 1 && Cin % 4 == 0 && L.groups == 1) L.w_f32 = w_dev;   // one tap: (Cout, Cin, 1) is the (N, K) matrix xvb_small_affine takes
  else cudaFree(w_dev);
  auto up = [&](float** d, const std::vector<float>& v) -> int {
    if (v.empty()) return XVB_OK;
    int r = ealloc(d, v.size());
    if (r) return r;
    XVB_CUDA(cudaMemcpy(*d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice));
    return XVB_OK;
  };
  if ((rc = up(&L.bias, L.hb)) || (rc = up(&L.scale, L.hs)) || (rc = up(&L.shift, L.ht))) return rc;
  h->layers[name] = L;
  h->order.push_back(name);
  return XVB_OK;
}

static const ELayer* find(const xvb_ecapa* h, const std::string& n) {
  auto it = h->layers.find(n);
  return it == h->layers.end() ? nullptr : &it->second;
}

extern "C" int xvb_ecapa_finalize(xvb_ecapa_t* h) {
  XVB_CHECK_ARG(h && !h->finalized, "xvb_ecapa_finalize: null or finalized model");
  const int C = h->C, W = C / h->scale;
  auto need = [&](const std::string& n, int cin, int cout, int ntaps) -> int {
    const ELayer* L = find(h, n);
    XVB_CHECK_ARG(L, "xvb_ecapa_finalize: layer '%s' is missing", n.c_str());
    XVB_CHECK_ARG(L->Cin == cin && L->Cout == cout && L->ntaps == ntaps, "xvb_ecapa_finalize: layer '%s' is %d->%d x%d taps, expected %d->%d x%d",
                  n.c_str(), L->Cin, L->Cout, L->ntaps, cin, cout, ntaps);
    return XVB_OK;
  };
  int rc;
  rc = need("layer1", h->feat_dim, C, find(h, "layer1") ? find(h, "layer1")->ntaps : 5);
  if (rc) return rc;
  for (int b = 0; b < 3; ++b) {
    const std::string p = "layer" + std::to_string(b + 2) + ".";
    if ((rc = need(p + "bn1", C, C, 1)) || (rc = need(p + "bn2", C, C, 1))) return rc;
    const ELayer* se1 = find(h, p + "se1");
    XVB_CHECK_ARG(se1 && se1->Cin == C, "xvb_ecapa_finalize: layer '%sse1' is missing", p.c_str());
    if (b == 0) h->se_dim = se1->Cout;
    XVB_CHECK_ARG(se1->Cout == h->se_dim && h->se_dim % 8 == 0, "xvb_ecapa_finalize: SE bottleneck must be a multiple of 8 and equal in all blocks");
    rc = need(p + "se2", h->se_dim, C, 1);
    if (rc) return rc;
    // stack the scale-1 Res2Net layers: packed weights along rows, parameters back to back
    const size_t pw = (size_t)xvb_packed_weight_elems(W, W, 3);
    if ((rc = ealloc(&h->res_w_hi[b], pw * (h->scale - 1))) || (rc = ealloc(&h->res_w_lo[b], pw * (h->scale - 1))) ||
        (rc = ealloc(&h->res_bias[b], (size_t)W * (h->scale - 1))) || (rc = ealloc(&h->res_scale[b], (size_t)W * (h->scale - 1))) ||
        (rc = ealloc(&h->res_shift[b], (size_t)W * (h->scale - 1))))
      return rc;
    for (int i = 0; i < h->scale - 1; ++i) {
      const std::string n = p + "res" + std::to_string(i);
      if ((rc = need(n, W, W, 3))) return rc;
      const ELayer* L = find(h, n);
      XVB_CHECK_ARG(L->ctx[0] == -L->ctx[2] && L->ctx[1] == 0 && L->bias && L->scale && L->shift && (L->flags & XVB_RELU),
                    "xvb_ecapa_finalize: '%s' must be a [-d,0,d] TDNN-ReLU-BN layer with bias", n.c_str());
      if (i == 0) h->dilation[b] = L->ctx[2];
      XVB_CHECK_ARG(L->ctx[2] == h->dilation[b], "xvb_ecapa_finalize: '%s' has another dilation than its block", n.c_str());
      XVB_CUDA(cudaMemcpy(h->res_w_hi[b] + pw * i, L->w_hi, pw * 2, cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(h->res_w_lo[b] + pw * i, L->w_lo, pw * 2, cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(h->res_bias[b] + (size_t)W * i, L->bias, W * sizeof(float), cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(h->res_scale[b] + (size_t)W * i, L->scale, W * sizeof(float), cudaMemcpyDeviceToDevice));
      XVB_CUDA(cudaMemcpy(h->res_shift[b] + (size_t)W * i, L->shift, W * sizeof(float), cudaMemcpyDeviceToDevice));
    }
  }
  rc = need("mfa", 3 * C, h->D, 1);
  if (rc) return rc;
  if (!h->mq) {
    if ((rc = need("att_x", h->D, h->H, 1)) || (rc = need("att_gs", 2 * h->D, h->H, 1)) || (rc = need("att2", h->H, h->D, 1)))
      return rc;
  } else {   // per-group input widths: att_x reads a head's Cg channels of x, att2 one query's hidden units
    rc = need("att_x", h->D / h->mq_heads, h->AX, 1);
    if (rc) return rc;
    if (h->mq_layers == 2 && (rc = need("att2", h->mq_hidden, h->NL, 1))) return rc;
    XVB_CHECK_ARG(h->mq_layers == 2 || !find(h, "att2"), "xvb_ecapa_finalize: one-layer attention has no 'att2'");
    if (h->mq_tatt && (rc = need("att_gs", (h->mq_stddev ? 2 : 1) * h->D, h->AX, 1))) return rc;
    XVB_CHECK_ARG(h->mq_tatt || !find(h, "att_gs"), "xvb_ecapa_finalize: 'att_gs' without time attention");
  }
  // segment level (ecapa_tdnn_xvector.py:412-422): [fc1 ->] [fc2]; "far" hands over fc1 alone, fc1=False fc2 alone
  if (const ELayer* fc1 = find(h, "fc1")) {
    XVB_CHECK_ARG(fc1->Cin == h->P && fc1->ntaps == 1 && fc1->w_f32, "xvb_ecapa_finalize: 'fc1' must be a one-tap layer over the %d pooled statistics", h->P);
    if (find(h, "fc2")) {
      rc = need("fc2", fc1->Cout, h->E, 1);
      if (rc) return rc;
    } else {
      XVB_CHECK_ARG(fc1->Cout == h->E, "xvb_ecapa_finalize: 'fc1' alone must produce the %d-d embedding", h->E);
    }
    h->fc1_dim = fc1->Cout;
  } else {
    rc = need("fc2", h->P, h->E, 1);
    if (rc) return rc;
  }
  {
    const ELayer* L0 = find(h, "layer1");
    bool consecutive = L0->ntaps > 1 && L0->ctx[0] <= 0 && L0->ctx[L0->ntaps - 1] >= 0;
    for (int i = 1; i < L0->ntaps; ++i) consecutive = consecutive && L0->ctx[i] == L0->ctx[i - 1] + 1;
    const int knob = getenv("XVB_IM2COL") ? atoi(getenv("XVB_IM2COL")) : 1;
    h->im2col_first = knob && consecutive && h->feat_dim % 16 == 0;
    h->pad_front = h->im2col_first ? -L0->ctx[0] : 0;
    h->pad_back = h->im2col_first ? L0->ctx[L0->ntaps - 1] : 0;
  }
  h->finalized = true;
  return XVB_OK;
}

extern "C" int xvb_ecapa_embed_dim(const xvb_ecapa_t* h) { return h ? h->E : XVB_EINVAL; }
extern "C" int xvb_ecapa_feat_dim(const xvb_ecapa_t* h) { return h ? h->feat_dim : XVB_EINVAL; }
extern "C" int xvb_ecapa_last_launches(const xvb_ecapa_t* h) { return h ? h->last_launches : 0; }

static int reserve(xvb_ecapa* h, int B, int T) {
  const long long frames = (long long)B * T;
  if (frames <= h->cap_frames && B <= h->cap_B) return XVB_OK;
  const size_t nf = (size_t)(frames > h->cap_frames ? frames : h->cap_frames);
  const size_t nb = (size_t)(B > h->cap_B ? B : h->cap_B);
  h->free_ws();
  const int C = h->C, D = h->D;
  int rc;
  if ((rc = h->planes(&h->in, nf + nb * (size_t)(h->pad_front + h->pad_back), h->ldf)) || (rc = h->planes(&h->X, nf, C)) || (rc = h->planes(&h->Hh, nf, C)) ||
      (rc = h->planes(&h->R, nf, C)) || (rc = h->planes(&h->Z, nf, C)) || (rc = h->planes(&h->N, nf, C)) ||
      (rc = h->planes(&h->CAT, nf, 3 * C)) || (rc = h->planes(&h->M, nf, D)) || (rc = h->planes(&h->A1, nf, h->H)) ||
      (rc = h->planes(&h->gp, nb, 2 * D)) || (rc = h->planes(&h->s1, nb, h->se_dim)) || (rc = h->planes(&h->zm, nb, C)) ||
      (rc = h->planes(&h->pp, nb, h->P2)) || (rc = h->f32(&h->MF, nf * D)) || (rc = h->f32(&h->LOG, nf * h->ldlog)) ||
      (rc = h->f32(&h->gate, nb * C)) || (rc = h->f32(&h->ub, nb * h->AX)) || (rc = h->f32(&h->zmean, nb * C)) ||
      (rc = h->f32(&h->gstat, nb * 2 * D)) || (rc = h->f32(&h->pstat, nb * h->P2)) || (rc = h->f32(&h->s1f, nb * (size_t)h->se_dim)) ||
      (h->fc1_dim && (rc = h->f32(&h->f1, nb * (size_t)h->fc1_dim))))
    return rc;
  h->cap_frames = (long long)nf;
  h->cap_B = (int)nb;
  return XVB_OK;
}

namespace {
struct Run {   // one layer launch: fill only what differs from the defaults
  const ELayer* L;
  Planes x, y;
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
  a.w_hi = r.L->w_hi; a.w_lo = r.L->w_lo;
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
  const int D = h->D, cg = D / h->mq_heads;
  const ELayer* ax = find(h, "att_x");
  int rc;
  if (h->mq_tatt) {
    if ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 0, h->gstat, h->gp.hi, h->gp.lo, 2 * D, stream))) return rc;
    const ELayer* gs = find(h, "att_gs");
    if (small_ok(gs)) {
      if ((rc = small_layer(gs, h->gstat, 2 * D, B, h->ub, h->AX, 0, stream))) return rc;
    } else {
      Run r{}; r.B = B; r.T = 1; r.L = gs; r.x = h->gp; r.y_f32 = h->ub; r.ldyf = h->AX;
      if ((rc = launch(r, stream))) return rc;
    }
  }
  Run r{}; r.B = B; r.T = T; r.L = ax; r.x = h->M;
  if (h->mq_tatt) { r.utt_bias = h->ub; r.ld_utt = h->AX; }
  if (h->mq_layers == 2) { r.y = h->A1; r.extra_flags = XVB_TANH; }
  else { r.y_f32 = h->LOG; r.ldyf = h->ldlog; }
  if ((rc = launch(r, stream))) return rc;
  if (h->mq_layers == 2) {
    r = Run{}; r.B = B; r.T = T; r.L = find(h, "att2"); r.x = h->A1; r.y_f32 = h->LOG; r.ldyf = h->ldlog;
    if ((rc = launch(r, stream))) return rc;
  }
  return xvb_attn_head_stats_pool_mq(h->LOG, h->ldlog, h->NL, h->MF, D, B, T, D, h->mq_q * D, h->mq_share ? cg : 1, cg, h->mq_q,
                                     1e-5f, 0, h->pstat, h->pp.hi, h->pp.lo, h->P2, stream);
}

extern "C" int xvb_ecapa_extract(xvb_ecapa_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(h && h->finalized, "xvb_ecapa_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_ecapa_extract: bad arguments");
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const long before = g_launches;
  const int C = h->C, D = h->D;
  auto L = [&](const std::string& n) { return find(h, n); };
  if (h->im2col_first)
    rc = xvb_split_frames(feats, B, T, h->feat_dim, h->in.hi, h->in.lo, h->ldf, h->pad_front, h->pad_back, stream);
  else
    rc = xvb_split_f32(feats, (int64_t)B * T, h->feat_dim, h->feat_dim, h->in.hi, h->in.lo, h->ldf, stream);
  if (rc) return rc;
  Run r{};
  r.B = B; r.T = T;
  r.L = L("layer1"); r.x = h->in; r.y = h->X;
  if (h->im2col_first) { r.im2col_taps = r.L->ntaps; r.x_batch_stride = (int64_t)(T + h->pad_front + h->pad_back) * h->ldf; }
  rc = launch(r, stream);
  if (rc && h->im2col_first) {   // overlapping tensor map refused by the driver: plain path from now on
    h->im2col_first = false;
    h->pad_front = h->pad_back = 0;
    return xvb_ecapa_extract(h, feats, B, T, emb, stream);
  }
  if (rc) return rc;
  Planes cur = h->X;
  for (int b = 0; b < 3; ++b) {
    const std::string p = "layer" + std::to_string(b + 2) + ".";
    r = Run{}; r.B = B; r.T = T; r.L = L(p + "bn1"); r.x = cur; r.y = h->Hh;
    if ((rc = launch(r, stream))) return rc;
    if ((rc = xvb_res2net_block(h->Hh.hi, h->Hh.lo, C, h->res_w_hi[b], h->res_w_lo[b], h->res_bias[b], h->res_scale[b],
                                h->res_shift[b], h->dilation[b], h->scale, h->R.hi, h->R.lo, C, B, T, stream)))
      return rc;
    r = Run{}; r.B = B; r.T = T; r.L = L(p + "bn2"); r.x = h->R; r.y = h->Z;
    if ((rc = launch(r, stream))) return rc;
    if ((rc = xvb_plane_mean(h->Z.hi, h->Z.lo, C, B, T, C, h->zmean, h->zm.hi, h->zm.lo, C, stream))) return rc;
    if (small_ok(L(p + "se1")) && small_ok(L(p + "se2"))) {
      rc = small_layer(L(p + "se1"), h->zmean, C, B, h->s1f, h->se_dim, 0, stream);
      if (rc) return rc;
      rc = small_layer(L(p + "se2"), h->s1f, h->se_dim, B, h->gate, C, XVB_SIGMOID, stream);
      if (rc) return rc;
    } else {
      r = Run{}; r.B = B; r.T = 1; r.L = L(p + "se1"); r.x = h->zm; r.y = h->s1;
      if ((rc = launch(r, stream))) return rc;
      r = Run{}; r.B = B; r.T = 1; r.L = L(p + "se2"); r.x = h->s1; r.y_f32 = h->gate; r.ldyf = C; r.extra_flags = XVB_SIGMOID;
      if ((rc = launch(r, stream))) return rc;
    }
    const bool last = b == 2;
    const Planes slot = h->CAT.slice(C * b);
    if ((rc = xvb_se_apply(h->Z.hi, h->Z.lo, C, cur.hi, cur.lo, cur.ld, h->gate, slot.hi, slot.lo, slot.ld,
                           last ? nullptr : h->N.hi, last ? nullptr : h->N.lo, C, B, T, C, stream)))
      return rc;
    cur = h->N;
  }
  r = Run{}; r.B = B; r.T = T; r.L = L("mfa"); r.x = h->CAT; r.y = h->M; r.y_f32 = h->MF; r.ldyf = D;
  if ((rc = launch(r, stream))) return rc;
  if (h->mq) {
    if ((rc = mqmha_pool(h, B, T, stream))) return rc;
  } else {
  if ((rc = xvb_stats_pool_ex(h->MF, D, B, T, D, 1e-5f, 1, h->gstat, h->gp.hi, h->gp.lo, 2 * D, stream))) return rc;
  if (small_ok(L("att_gs"))) {
    rc = small_layer(L("att_gs"), h->gstat, 2 * D, B, h->ub, h->H, 0, stream);
      if (rc) return rc;
  } else {
    r = Run{}; r.B = B; r.T = 1; r.L = L("att_gs"); r.x = h->gp; r.y_f32 = h->ub; r.ldyf = h->H;
    if ((rc = launch(r, stream))) return rc;
  }
  r = Run{}; r.B = B; r.T = T; r.L = L("att_x"); r.x = h->M; r.y = h->A1; r.utt_bias = h->ub; r.ld_utt = h->H; r.extra_flags = XVB_TANH;
  if ((rc = launch(r, stream))) return rc;
  r = Run{}; r.B = B; r.T = T; r.L = L("att2"); r.x = h->A1; r.y_f32 = h->LOG; r.ldyf = D;
  if ((rc = launch(r, stream))) return rc;
  if ((rc = xvb_attn_stats_pool(h->LOG, D, h->MF, D, B, T, D, 1e-5f, h->pstat, h->pp.hi, h->pp.lo, 2 * D, stream))) return rc;
  }
  if (const ELayer* fc1 = L("fc1")) {              // fc1 [-> fc2] on CUDA cores (fp32)
    const ELayer* fc2 = L("fc2");
    rc = small_layer(fc1, h->pstat, h->P2, B, fc2 ? h->f1 : emb, fc1->Cout, 0, stream);
    if (rc) return rc;
    if (fc2) {
      XVB_CHECK_ARG(fc2->w_f32, "xvb_ecapa_extract: 'fc2' after 'fc1' needs an input width that is a multiple of 4");
      rc = small_layer(fc2, h->f1, fc1->Cout, B, emb, h->E, 0, stream);
      if (rc) return rc;
    }
  } else if (small_ok(L("fc2"))) {
    rc = small_layer(L("fc2"), h->pstat, h->P2, B, emb, h->E, 0, stream);
      if (rc) return rc;
  } else {
    r = Run{}; r.B = B; r.T = 1; r.L = L("fc2"); r.x = h->pp; r.y_f32 = emb; r.ldyf = h->E;   // reads the first P of P2 columns
    if ((rc = launch(r, stream))) return rc;
  }
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

extern "C" int xvb_ecapa_extract_host(xvb_ecapa_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats_host && emb_host && B > 0 && T > 0, "xvb_ecapa_extract_host: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t nf = (size_t)B * T * h->feat_dim, ne = (size_t)B * h->E;
  if (nf > h->h_feats_cap) {
    cudaFree(h->h_feats);
    int rc = ealloc(&h->h_feats, nf);
    if (rc) return rc;
    h->h_feats_cap = nf;
  }
  if (ne > h->h_emb_cap) {
    cudaFree(h->h_emb);
    int rc = ealloc(&h->h_emb, ne);
    if (rc) return rc;
    h->h_emb_cap = ne;
  }
  XVB_CUDA(cudaMemcpyAsync(h->h_feats, feats_host, nf * sizeof(float), cudaMemcpyHostToDevice, s));
  int rc = xvb_ecapa_extract(h, h->h_feats, B, T, h->h_emb, stream);
  if (rc) return rc;
  XVB_CUDA(cudaMemcpyAsync(emb_host, h->h_emb, ne * sizeof(float), cudaMemcpyDeviceToHost, s));
  XVB_CUDA(cudaStreamSynchronize(s));
  return XVB_OK;
}

// A whole shard of N equal-length utterances in `batch`-utterance batches (the reference's caller loop,
// extract_embeddings.py:73-83), device-resident / through pinned host buffers with the copies overlapped
// (same protocol as xvb_extractor_extract_shard[_host]).
extern "C" int xvb_ecapa_set_gather(xvb_ecapa_t* h, float* const* tables, int ntables, int64_t row0, int64_t ld) {
  XVB_CHECK_ARG(h && h->finalized && ntables >= 0 && ntables <= XVB_MAX_PEERS, "xvb_ecapa_set_gather: bad arguments");
  XVB_CHECK_ARG(ntables == 0 || (tables && row0 >= 0 && ld >= h->E && ld % 4 == 0),
                "xvb_ecapa_set_gather: need tables, row0 >= 0, ld >= embed_dim and ld %% 4 == 0");
  for (int k = 0; k < ntables; ++k) h->gather_tables[k] = tables[k];
  h->gather_n = ntables; h->gather_row0 = row0; h->gather_ld = ld;
  return XVB_OK;
}

static bool ecapa_lanes_enabled() {
  static const int knob = getenv("XVB_LANES") ? atoi(getenv("XVB_LANES")) : 1;
  return knob != 0;
}

static int ecapa_ensure_lanes(xvb_ecapa* h) {
  if (h->lane1) return XVB_OK;
  for (int i = 0; i < 2; ++i) {
    XVB_CUDA(cudaStreamCreateWithFlags(&h->lane_stream[i], cudaStreamNonBlocking));
    XVB_CUDA(cudaEventCreateWithFlags(&h->ev_lane_done[i], cudaEventDisableTiming));
  }
  XVB_CUDA(cudaEventCreateWithFlags(&h->ev_lane_start, cudaEventDisableTiming));
  xvb_ecapa* c = new xvb_ecapa();
  c->feat_dim = h->feat_dim; c->ldf = h->ldf; c->C = h->C; c->D = h->D; c->H = h->H; c->E = h->E; c->scale = h->scale;
  c->se_dim = h->se_dim; c->fc1_dim = h->fc1_dim; c->finalized = true;
  c->mq = h->mq; c->mq_heads = h->mq_heads; c->mq_q = h->mq_q; c->mq_hidden = h->mq_hidden; c->mq_share = h->mq_share;
  c->mq_layers = h->mq_layers; c->mq_tatt = h->mq_tatt; c->mq_stddev = h->mq_stddev;
  c->AX = h->AX; c->NL = h->NL; c->ldlog = h->ldlog; c->P = h->P; c->P2 = h->P2;
  for (int b = 0; b < 3; ++b) {
    c->dilation[b] = h->dilation[b];
    c->res_w_hi[b] = h->res_w_hi[b]; c->res_w_lo[b] = h->res_w_lo[b]; c->res_bias[b] = h->res_bias[b];
    c->res_scale[b] = h->res_scale[b]; c->res_shift[b] = h->res_shift[b];
  }
  for (const auto& kv : h->layers) {            // device pointers + shapes only: the twin never saves, so no host copies
    ELayer L;
    L.Cin = kv.second.Cin; L.Cout = kv.second.Cout; L.ntaps = kv.second.ntaps; L.flags = kv.second.flags; L.tot = kv.second.tot;
    for (int i = 0; i < XVB_MAX_TAPS; ++i) L.ctx[i] = kv.second.ctx[i];
    L.w_hi = kv.second.w_hi; L.w_lo = kv.second.w_lo; L.bias = kv.second.bias; L.scale = kv.second.scale; L.shift = kv.second.shift;
    L.w_f32 = kv.second.w_f32;
    L.groups = kv.second.groups; L.expanded = kv.second.expanded;
    c->layers[kv.first] = L;
  }
  c->im2col_first = h->im2col_first; c->pad_front = h->pad_front; c->pad_back = h->pad_back;
  c->is_lane = true;
  h->lane1 = c;
  return XVB_OK;
}
static int ecapa_lanes_fork(xvb_ecapa* h, cudaStream_t s) {
  XVB_CUDA(cudaEventRecord(h->ev_lane_start, s));
  for (int i = 0; i < 2; ++i) XVB_CUDA(cudaStreamWaitEvent(h->lane_stream[i], h->ev_lane_start, 0));
  return XVB_OK;
}
static int ecapa_lanes_join(xvb_ecapa* h, cudaStream_t s) {
  for (int i = 0; i < 2; ++i) {
    XVB_CUDA(cudaEventRecord(h->ev_lane_done[i], h->lane_stream[i]));
    XVB_CUDA(cudaStreamWaitEvent(s, h->ev_lane_done[i], 0));
  }
  return XVB_OK;
}

extern "C" int xvb_ecapa_extract_shard(xvb_ecapa_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats && emb && N > 0 && T > 0 && batch > 0, "xvb_ecapa_extract_shard: bad arguments");
  int launches = 0;
  if (ecapa_lanes_enabled() && N > batch) {
    int rc = ecapa_ensure_lanes(h);
    if (rc) return rc;
    if ((rc = ecapa_lanes_fork(h, (cudaStream_t)stream))) return rc;
    int k = 0;
    for (int64_t i = 0; i < N; i += batch, ++k) {
      const int b = (int)(N - i < batch ? N - i : batch);
      xvb_ecapa* lane = (k & 1) ? h->lane1 : h;
      if ((rc = xvb_ecapa_extract(lane, feats + (size_t)i * T * h->feat_dim, b, T, emb + (size_t)i * h->E, h->lane_stream[k & 1]))) return rc;
      launches += lane->last_launches;
      if (h->gather_n && (rc = xvb_scatter_rows(emb + (size_t)i * h->E, b, h->E, h->gather_tables, h->gather_n, h->gather_row0 + i,
                                                h->gather_ld, h->lane_stream[k & 1]))) return rc;
    }
    if ((rc = ecapa_lanes_join(h, (cudaStream_t)stream))) return rc;
    h->last_launches = launches;
    return XVB_OK;
  }
  for (int64_t i = 0; i < N; i += batch) {
    const int b = (int)(N - i < batch ? N - i : batch);
    int rc = xvb_ecapa_extract(h, feats + (size_t)i * T * h->feat_dim, b, T, emb + (size_t)i * h->E, stream);
    if (!rc && h->gather_n)
      rc = xvb_scatter_rows(emb + (size_t)i * h->E, b, h->E, h->gather_tables, h->gather_n, h->gather_row0 + i, h->gather_ld, stream);
    if (rc) return rc;
    launches += h->last_launches;
  }
  h->last_launches = launches;
  return XVB_OK;
}

extern "C" int xvb_ecapa_extract_shard_host(xvb_ecapa_t* h, const float* feats_host, int64_t N, int T, int batch, float* emb_host,
                                            void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats_host && emb_host && N > 0 && T > 0 && batch > 0, "xvb_ecapa_extract_shard_host: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  if (!h->copy_stream) {
    XVB_CUDA(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < xvb_ecapa::kSlots; ++i) {
      XVB_CUDA(cudaEventCreateWithFlags(&h->ev_h2d[i], cudaEventDisableTiming));
      XVB_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
    }
  }
  constexpr int S = xvb_ecapa::kSlots;
  const int bmax = (int)(N < batch ? N : batch);
  const size_t nf = (size_t)bmax * T * h->feat_dim, ne = (size_t)bmax * h->E;
  int rc;
  for (int slot = 0; slot < S; ++slot) {
    if (nf > h->p_feats_cap[slot]) {
      cudaFree(h->p_feats[slot]); h->p_feats[slot] = nullptr; h->p_feats_cap[slot] = 0;
      if ((rc = ealloc(&h->p_feats[slot], nf))) return rc;
      h->p_feats_cap[slot] = nf;
    }
    if (ne > h->p_emb_cap[slot]) {
      cudaFree(h->p_emb[slot]); h->p_emb[slot] = nullptr; h->p_emb_cap[slot] = 0;
      if ((rc = ealloc(&h->p_emb[slot], ne))) return rc;
      h->p_emb_cap[slot] = ne;
    }
  }
  const bool lanes = ecapa_lanes_enabled() && N > batch;
  if (lanes) {
    if ((rc = ecapa_ensure_lanes(h))) return rc;
    if ((rc = ecapa_lanes_fork(h, s))) return rc;
  }
  int launches = 0, k = 0;
  for (int64_t i = 0; i < N; i += batch, ++k) {
    const int b = (int)(N - i < batch ? N - i : batch);
    const int slot = k % S;
    xvb_ecapa* lane = (lanes && (k & 1)) ? h->lane1 : h;
    cudaStream_t ls = lanes ? h->lane_stream[k & 1] : s;
    if (k >= S) XVB_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[slot], 0));
    XVB_CUDA(cudaMemcpyAsync(h->p_feats[slot], feats_host + (size_t)i * T * h->feat_dim, (size_t)b * T * h->feat_dim * sizeof(float),
                             cudaMemcpyHostToDevice, h->copy_stream));
    XVB_CUDA(cudaEventRecord(h->ev_h2d[slot], h->copy_stream));
    XVB_CUDA(cudaStreamWaitEvent(ls, h->ev_h2d[slot], 0));
    if ((rc = xvb_ecapa_extract(lane, h->p_feats[slot], b, T, h->p_emb[slot], ls))) return rc;
    if (h->gather_n && (rc = xvb_scatter_rows(h->p_emb[slot], b, h->E, h->gather_tables, h->gather_n, h->gather_row0 + i, h->gather_ld, ls)))
      return rc;
    XVB_CUDA(cudaMemcpyAsync(emb_host + (size_t)i * h->E, h->p_emb[slot], (size_t)b * h->E * sizeof(float), cudaMemcpyDeviceToHost, ls));
    XVB_CUDA(cudaEventRecord(h->ev_done[slot], ls));
    launches += lane->last_launches;
  }
  if (lanes && (rc = ecapa_lanes_join(h, s))) return rc;
  XVB_CUDA(cudaStreamSynchronize(s));
  h->last_launches = launches;
  return XVB_OK;
}

// ---- .xvbm files for ECAPA ("XVBE0001"): dims, then named layer records -------------------------------------
// "XVBE0002" (MQMHA pooling): the same with the pooling record {num_head, num_q, hidden, share, affine_layers,
// time_attention, stddev} after the dims; layers of grouped convs are stored as the state_dict holds them.
extern "C" int xvb_ecapa_save(const xvb_ecapa_t* h, const char* path) {
  XVB_CHECK_ARG(h && h->finalized && path, "xvb_ecapa_save: model not finalized");
  FILE* f = fopen(path, "wb");
  XVB_CHECK_ARG(f, "xvb_ecapa_save: cannot open '%s'", path);
  bool ok = fwrite(h->mq ? "XVBE0002" : "XVBE0001", 1, 8, f) == 8;
  const int32_t hd[6] = {h->feat_dim, h->C, h->D, h->H, h->E, (int32_t)h->order.size()};
  ok = ok && fwrite(hd, 4, 6, f) == 6;
  if (h->mq) {
    const int32_t pr[7] = {h->mq_heads, h->mq_q, h->mq_hidden, h->mq_share, h->mq_layers, h->mq_tatt, h->mq_stddev};
    ok = ok && fwrite(pr, 4, 7, f) == 7;
  }
  for (const std::string& n : h->order) {
    const ELayer& L = h->layers.at(n);
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

extern "C" void xvb_ecapa_destroy(xvb_ecapa_t* h) {
  if (!h) return;
  if (h->lane1) xvb_ecapa_destroy(h->lane1);
  for (int i = 0; i < 2; ++i) {
    if (h->lane_stream[i]) cudaStreamDestroy(h->lane_stream[i]);
    if (h->ev_lane_done[i]) cudaEventDestroy(h->ev_lane_done[i]);
  }
  if (h->ev_lane_start) cudaEventDestroy(h->ev_lane_start);
  h->free_ws();
  cudaFree(h->h_feats); cudaFree(h->h_emb);
  for (int i = 0; i < xvb_ecapa::kSlots; ++i) {
    cudaFree(h->p_feats[i]); cudaFree(h->p_emb[i]);
    if (h->ev_h2d[i]) cudaEventDestroy(h->ev_h2d[i]);
    if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]);
  }
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  if (!h->is_lane) {
    for (auto& kv : h->layers) {
      ELayer& L = kv.second;
      cudaFree(L.w_hi); cudaFree(L.w_lo); cudaFree(L.bias); cudaFree(L.scale); cudaFree(L.shift); cudaFree(L.w_f32);
    }
    for (int b = 0; b < 3; ++b) {
      cudaFree(h->res_w_hi[b]); cudaFree(h->res_w_lo[b]); cudaFree(h->res_bias[b]); cudaFree(h->res_scale[b]); cudaFree(h->res_shift[b]);
    }
  }
  delete h;
}
