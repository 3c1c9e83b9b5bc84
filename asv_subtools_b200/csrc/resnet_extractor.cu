// Whole-model extractor for the 2-D ResNet x-vector (pytorch/model/resnet_xvector.py, ResNetXvector.extract_embedding
// :183-208 over pytorch/libs/nnet/resnet.py, BasicBlock): packed weights + workspace on the current device and the
// launch sequence, in C++, so that a ResNet model needs no Python at run time (bin/xvb-extract, the role of the
// reference's runtime/).  Same kernels, same C entry points, same arguments and the same order as the Python
// orchestration it replaces (ResNetExtractor in asv_subtools_b200/model/resnet_xvector.py, kept as
// XVB_RESNET_NATIVE=0), so the embeddings are bit-identical to it:
//
//   head conv (+ BN, ReLU [, first block's bn1-relu]) -> per block: conv1 [-> 1x1 stride-2 downsample] -> conv2 with
//   BN / residual / ReLU / next block's bn1-relu in its epilogue, or with SE: conv2 -> plane mean -> two small affines
//   (ReLU, sigmoid) -> SE scaling + residual -> statistics pooling (planes out) -> segment layers.
//
// Records are handed over by their state_dict module path with the weights as stored (host fp32), eval BatchNorm
// folded to (scale, shift) by the caller; the segment layers arrive as the Python hands them to _PackedAffine (fc1 /
// fc2 export(), the first one's input columns already permuted to the (B, T', F', C) pooling order).  This file only
// packs and pads: conv weights through xvb_pack_tdnn_weight, the SE hidden width zero-padded to a multiple of 4 with
// fc_1 replicated k times (divided by k) for the k-grouped plane mean, segment rows padded to a multiple of 8.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <set>
#include <string>
#include <vector>

#include "common.cuh"

namespace {

using namespace xvb;

// One B*T*F position budget per extract call: larger calls run as consecutive groups of utterances (see xvb200.h).
constexpr long long kPositionBudget = 256LL * 200 * 80;
constexpr int kSeMaxK = 9;   // k = 1, 2, ..., 256 for the k-grouped SE mean

struct Rec {   // one named record exactly as handed over (host copies, for xvb_resnet_save)
  int Cout = 0, Cin = 0, ksize = 0, flags = 0;
  std::vector<float> w, b, s, t;
};

struct Conv { uint16_t* hi = nullptr; uint16_t* lo = nullptr; };
struct Bn { float* s = nullptr; float* t = nullptr; };
struct Se {
  int C = 0, Hp = 0, kmax = 1;           // hidden width padded to a multiple of 4; k = 1 .. kmax (powers of two)
  float* w1k[kSeMaxK] = {nullptr};       // index log2(k): (Hp, k*C) = [w1 / k, ..., w1 / k]
  float* b1 = nullptr; float* w2 = nullptr; float* b2 = nullptr;
};
struct Block {
  int stride = 1, cin = 0, cout = 0;
  Conv conv1, conv2, ds;
  Bn bn1, bn2, dsbn;
  bool has_ds = false, has_se = false;
  Se se;
};
struct Seg {   // one segment layer on the wgmma layer kernel (T = 1), output rows padded to a multiple of 8
  Conv w;
  float* bias = nullptr; float* scale = nullptr; float* shift = nullptr;
  int Cin = 0, Cout = 0, Cout_real = 0, flags = 0;
};

struct Model {   // shared by a handle and its second shard lane
  int feat_dim = 0, layers[4] = {0}, planes[4] = {0}, pre = 0;
  float eps = 0.f;
  std::map<std::string, Rec> recs;
  std::vector<std::string> order;   // insertion order, for save()
  float* head_w = nullptr;
  Bn head_bn;
  std::vector<Block> blocks;
  std::vector<Seg> seg;
  int F4 = 0, C4 = 0, E = 0, Cmax = 0, Hmax = 0, seg_mid = 0;
  std::vector<void*> dev;           // every device allocation of the weights

  template <typename T>
  int alloc(T** p, size_t n) {
    XVB_CUDA(cudaMalloc((void**)p, n * sizeof(T)));
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
  // (Cout, Cin, taps) fp32 host -> packed planes, taps 0..ntaps-1 (what ops.pack_tdnn_weight does)
  int pack(Conv* c, const std::vector<float>& w, int Cout, int Cin, int ntaps) {
    float* w_dev = nullptr;
    XVB_CUDA(cudaMalloc((void**)&w_dev, w.size() * sizeof(float)));
    cudaError_t e = cudaMemcpy(w_dev, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice);
    int ctx[XVB_MAX_TAPS];
    for (int i = 0; i < ntaps; ++i) ctx[i] = i;
    const size_t pn = (size_t)xvb_packed_weight_elems(Cout, Cin, ntaps);
    int rc = e != cudaSuccess ? XVB_ECUDA : XVB_OK;
    if (!rc) rc = alloc(&c->hi, pn);
    if (!rc) rc = alloc(&c->lo, pn);
    if (!rc) rc = xvb_pack_tdnn_weight(w_dev, Cout, Cin, ntaps, 0, ctx, ntaps, c->hi, c->lo, nullptr);
    if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = XVB_ECUDA;
    if (rc == XVB_ECUDA && e != cudaSuccess) set_error("xvb_resnet_finalize: weight upload failed: %s", cudaGetErrorString(e));
    cudaFree(w_dev);
    return rc;
  }
  ~Model() { for (void* p : dev) cudaFree(p); }
};

struct Planes { uint16_t* hi = nullptr; uint16_t* lo = nullptr; };

}  // namespace

struct xvb_resnet {
  Model* m = nullptr;
  bool owns_model = true, finalized = false;
  // workspace, grown to the largest (B, T) seen: seven rotating (B, T', F', C) plane buffers for the roles block
  // input / activated input / h / identity / z / output / next activated input, the fp32 last-layer output, then the
  // per-utterance buffers (pooled statistics, SE mean / hidden / gate, segment layers)
  static constexpr int kBufs = 7;
  size_t cap_planes = 0, cap_last = 0;
  int cap_B = 0;
  std::vector<void*> ws;
  Planes buf[kBufs], pooled, seg_mid;
  float *last = nullptr, *pooled_f32 = nullptr, *se_mean = nullptr, *se_hidden = nullptr, *se_gate = nullptr, *seg_out = nullptr;
  int last_launches = 0;
  float* h_feats = nullptr; float* h_emb = nullptr;   // device staging of xvb_resnet_extract_host
  size_t h_feats_cap = 0, h_emb_cap = 0;
  // pipeline of xvb_resnet_extract_shard_host: two device slots per lane, the copy engine runs ahead of both lanes
  static constexpr int kSlots = 4;
  float* p_feats[kSlots] = {nullptr, nullptr, nullptr, nullptr}; float* p_emb[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  size_t p_feats_cap[kSlots] = {0, 0, 0, 0}, p_emb_cap[kSlots] = {0, 0, 0, 0};
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_h2d[kSlots] = {nullptr, nullptr, nullptr, nullptr}, ev_done[kSlots] = {nullptr, nullptr, nullptr, nullptr};
  // two-lane shard pipeline: `lane1` shares the weights and owns its workspace; batches alternate between two streams
  xvb_resnet* lane1 = nullptr;
  cudaStream_t lane_stream[2] = {nullptr, nullptr};
  cudaEvent_t ev_lane_start = nullptr, ev_lane_done[2] = {nullptr, nullptr};

  void free_ws() {
    for (void* p : ws) cudaFree(p);
    ws.clear();
    cap_planes = cap_last = 0;
    cap_B = 0;
  }
  template <typename T>
  int alloc(T** p, size_t n) {
    XVB_CUDA(cudaMalloc((void**)p, (n ? n : 1) * sizeof(T)));
    ws.push_back(*p);
    return XVB_OK;
  }
  int planes(Planes* p, size_t n) {
    int rc = alloc(&p->hi, n);
    return rc ? rc : alloc(&p->lo, n);
  }
};

namespace {

int log2i(int k) { int l = 0; while ((1 << l) < k) ++l; return l; }

// Position-buffer sizes (elements) of one (B, T) call: the largest (B, T', F', C) tensor and the last layer's output.
void shapes(const Model* m, int B, int T, size_t* planes, size_t* last) {
  long long t = T, f = m->feat_dim;
  size_t mx = (size_t)B * t * f * m->planes[0];
  for (const Block& b : m->blocks) {
    t = (t - 1) / b.stride + 1;
    f = (f - 1) / b.stride + 1;
    const size_t n = (size_t)B * t * f * b.cout;
    if (n > mx) mx = n;
  }
  *planes = mx;
  *last = (size_t)B * t * f * m->C4;
}

int reserve(xvb_resnet* h, int B, int T) {
  size_t np, nl;
  shapes(h->m, B, T, &np, &nl);
  if (np <= h->cap_planes && nl <= h->cap_last && B <= h->cap_B) return XVB_OK;
  np = np > h->cap_planes ? np : h->cap_planes;
  nl = nl > h->cap_last ? nl : h->cap_last;
  const size_t nb = (size_t)(B > h->cap_B ? B : h->cap_B);
  h->free_ws();
  const Model* m = h->m;
  const size_t pooled = (size_t)2 * m->F4 * m->C4, mean = m->Cmax > 256 ? m->Cmax : 256;
  const size_t out = (size_t)m->seg.back().Cout;
  int rc = XVB_OK;
  for (int i = 0; i < xvb_resnet::kBufs && !rc; ++i) rc = h->planes(&h->buf[i], np);
  if (rc || (rc = h->alloc(&h->last, nl)) || (rc = h->planes(&h->pooled, nb * pooled)) || (rc = h->alloc(&h->pooled_f32, nb * pooled)) ||
      (rc = h->alloc(&h->se_mean, nb * mean)) || (rc = h->alloc(&h->se_hidden, nb * (size_t)(m->Hmax ? m->Hmax : 4))) ||
      (rc = h->alloc(&h->se_gate, nb * (size_t)m->Cmax)) || (rc = h->planes(&h->seg_mid, nb * (size_t)(m->seg_mid ? m->seg_mid : 8))) ||
      (rc = h->alloc(&h->seg_out, nb * out))) {
    h->free_ws();
    return rc;
  }
  h->cap_planes = np; h->cap_last = nl; h->cap_B = (int)nb;
  return XVB_OK;
}

int conv(const Planes& x, const Conv& w, int B, int T, int F, int Cin, int Cout, int k, int stride, const Bn& bn,
         const Planes* res, int relu, const Planes* y, float* y_f32, const Bn& bn2, const Planes* y2, void* stream) {
  xvb_conv2d_args_t a{};
  a.x_hi = x.hi; a.x_lo = x.lo;
  a.w_hi = w.hi; a.w_lo = w.lo;
  a.B = B; a.T = T; a.F = F; a.Cin = Cin; a.Cout = Cout; a.ksize = k; a.stride = stride;
  a.scale = bn.s; a.shift = bn.t;
  if (res) { a.res_hi = res->hi; a.res_lo = res->lo; }
  a.relu = relu;
  if (y) { a.y_hi = y->hi; a.y_lo = y->lo; }
  a.y_f32 = y_f32;
  a.scale2 = bn2.s; a.shift2 = bn2.t;
  if (y2) { a.y2_hi = y2->hi; a.y2_lo = y2->lo; }
  return xvb_conv2d(&a, stream);
}

// sigmoid(fc_2(relu(fc_1(mean over the P positions of z)))) as ResNetExtractor._se_gate: the (B, P, C) planes read as
// (B, P/k, k*C) with the largest k in the table (2k too) that divides P.
int se_gate(xvb_resnet* h, const Se& se, const Planes& z, int B, long long P, void* stream) {
  int k = 1;
  while (2 * k <= se.kmax && P % (2 * k) == 0) k *= 2;
  const int kc = k * se.C;
  int rc = xvb_plane_mean(z.hi, z.lo, kc, B, (int)(P / k), kc, h->se_mean, nullptr, nullptr, kc, stream);
  if (!rc) rc = xvb_small_affine(h->se_mean, kc, se.w1k[log2i(k)], B, kc, se.Hp, se.b1, nullptr, nullptr, XVB_RELU,
                                 h->se_hidden, se.Hp, nullptr, nullptr, 0, stream);
  if (!rc) rc = xvb_small_affine(h->se_hidden, se.Hp, se.w2, B, se.Hp, se.C, se.b2, nullptr, nullptr, XVB_SIGMOID,
                                 h->se_gate, se.C, nullptr, nullptr, 0, stream);
  return rc;
}

// One group of utterances (B * T * F within the budget, or a single utterance): ResNetExtractor.extract.
int extract_group(xvb_resnet* h, const float* feats, int B, int T, float* emb, void* stream) {
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const Model* m = h->m;
  const bool pre = m->pre != 0;
  int Tl = T, Fl = m->feat_dim;
  int xi = 0, ai = pre ? 1 : -1;
  const Bn none;
  {
    const Bn first = pre ? m->blocks[0].bn1 : none;
    const Planes* a = pre ? &h->buf[ai] : nullptr;
    rc = xvb_conv2d_head(feats, B, T, Fl, m->head_w, m->planes[0], m->head_bn.s, m->head_bn.t, h->buf[xi].hi, h->buf[xi].lo,
                         first.s, first.t, a ? a->hi : nullptr, a ? a->lo : nullptr, stream);
    if (rc) return rc;
  }
  const int nb = (int)m->blocks.size();
  for (int i = 0; i < nb; ++i) {
    const Block& blk = m->blocks[i];
    const bool last = i + 1 == nb;
    const int st = blk.stride, co = blk.cout, Tn = (Tl - 1) / st + 1, Fn = (Fl - 1) / st + 1;
    unsigned used = (1u << xi) | (ai >= 0 ? 1u << ai : 0u);
    auto take = [&]() { int j = 0; while (used & (1u << j)) ++j; used |= 1u << j; return j; };
    const int hh = take();
    // pre-activation: h = relu(bn2(conv1(relu(bn1(x))))); post-activation: h = relu(bn1(conv1(x)))
    if ((rc = conv(pre ? h->buf[ai] : h->buf[xi], blk.conv1, B, Tl, Fl, blk.cin, co, 3, st, pre ? blk.bn2 : blk.bn1, nullptr, 1,
                   &h->buf[hh], nullptr, none, nullptr, stream)))
      return rc;
    int id = xi;
    if (blk.has_ds) {   // conv1x1 (stride) + BN of the un-activated block input
      id = take();
      if ((rc = conv(h->buf[xi], blk.ds, B, Tl, Fl, blk.cin, co, 1, st, blk.dsbn, nullptr, 0, &h->buf[id], nullptr, none, nullptr, stream)))
        return rc;
    }
    const Bn nxt = (!last && pre) ? m->blocks[i + 1].bn1 : none;
    const int yi = last ? -1 : take();
    const int an = nxt.s ? take() : -1;
    const Planes* y = yi >= 0 ? &h->buf[yi] : nullptr;
    const Planes* y2 = an >= 0 ? &h->buf[an] : nullptr;
    float* yf = last ? h->last : nullptr;
    const Bn bn2 = pre ? none : blk.bn2;
    if (!blk.has_se) {   // conv2 [+ bn2] + identity [-> relu] in one epilogue
      if ((rc = conv(h->buf[hh], blk.conv2, B, Tn, Fn, co, co, 3, 1, bn2, &h->buf[id], pre ? 0 : 1, y, yf, nxt, y2, stream))) return rc;
    } else {
      const int zi = take();
      if ((rc = conv(h->buf[hh], blk.conv2, B, Tn, Fn, co, co, 3, 1, bn2, nullptr, 0, &h->buf[zi], nullptr, none, nullptr, stream)))
        return rc;
      const long long P = (long long)Tn * Fn;
      if ((rc = se_gate(h, blk.se, h->buf[zi], B, P, stream))) return rc;
      if ((rc = xvb_se_residual(h->buf[zi].hi, h->buf[zi].lo, h->se_gate, h->buf[id].hi, h->buf[id].lo, B, P, co, pre ? 0 : 1,
                                y ? y->hi : nullptr, y ? y->lo : nullptr, yf, nxt.s, nxt.t, y2 ? y2->hi : nullptr,
                                y2 ? y2->lo : nullptr, stream)))
        return rc;
    }
    xi = yi; ai = an; Tl = Tn; Fl = Fn;
  }
  const int pc = Fl * m->C4;
  if ((rc = xvb_stats_pool_ex(h->last, pc, B, Tl, pc, m->eps, 0, h->pooled_f32, h->pooled.hi, h->pooled.lo, 2 * pc, stream))) return rc;
  Planes x = h->pooled;
  int64_t ldx = 2 * pc;
  const int ctx0 = 0;
  for (size_t j = 0; j < m->seg.size(); ++j) {
    const Seg& s = m->seg[j];
    const bool fin = j + 1 == m->seg.size();
    xvb_tdnn_args_t a{};
    a.x_hi = x.hi; a.x_lo = x.lo; a.ldx = ldx;
    a.w_hi = s.w.hi; a.w_lo = s.w.lo;
    a.bias = s.bias; a.bn_scale = s.scale; a.bn_shift = s.shift;
    a.flags = s.flags;
    a.context_host = &ctx0; a.ntaps = 1;
    if (fin) { a.y_f32 = s.Cout == m->E ? emb : h->seg_out; a.ldyf = s.Cout; }
    else { a.y_hi = h->seg_mid.hi; a.y_lo = h->seg_mid.lo; a.ldy = s.Cout; }
    a.B = B; a.T = 1; a.Cin = s.Cin; a.Cout = s.Cout;
    if ((rc = xvb_tdnn_affine_ex(&a, stream))) return rc;
    x = h->seg_mid; ldx = s.Cout;
  }
  const Seg& s = m->seg.back();
  if (s.Cout != m->E)
    XVB_CUDA(cudaMemcpy2DAsync(emb, (size_t)m->E * sizeof(float), h->seg_out, (size_t)s.Cout * sizeof(float), (size_t)m->E * sizeof(float),
                               (size_t)B, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return XVB_OK;
}

const Rec* find(const Model* m, const std::string& n) {
  auto it = m->recs.find(n);
  return it == m->recs.end() ? nullptr : &it->second;
}

}  // namespace

extern "C" int xvb_resnet_create(xvb_resnet_t** out, int feat_dim, const int* layers, const int* planes, int pre_activation,
                                 float pooling_eps) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && layers && planes && feat_dim > 0 && feat_dim <= 4096 && isfinite(pooling_eps) && pooling_eps >= 0.f,
                "xvb_resnet_create: bad arguments");
  for (int i = 0; i < 4; ++i) {
    XVB_CHECK_ARG(layers[i] >= 1 && layers[i] <= 64, "xvb_resnet_create: layers[%d] = %d, need 1..64 blocks", i, layers[i]);
    XVB_CHECK_ARG(planes[i] >= 16 && planes[i] <= 4096 && planes[i] % 16 == 0,
                  "xvb_resnet_create: planes[%d] = %d, need a multiple of 16 for the 2-D conv kernel", i, planes[i]);
  }
  xvb_resnet* h = new xvb_resnet();
  h->m = new Model();
  h->m->feat_dim = feat_dim;
  for (int i = 0; i < 4; ++i) { h->m->layers[i] = layers[i]; h->m->planes[i] = planes[i]; }
  h->m->pre = pre_activation ? 1 : 0;
  h->m->eps = pooling_eps;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_resnet_set_layer(xvb_resnet_t* h, const char* name, int Cout, int Cin, int ksize, const float* w_host,
                                    const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(h && !h->finalized && name && strlen(name) > 0 && strlen(name) < 127, "xvb_resnet_set_layer: bad arguments or finalized model");
  XVB_CHECK_ARG(Cout > 0 && Cout <= 65536 && Cin >= 0 && Cin <= (1 << 20) && (ksize == 0 || ksize == 1 || ksize == 3),
                "xvb_resnet_set_layer(%s): bad shape %d x %d x k%d", name, Cout, Cin, ksize);
  XVB_CHECK_ARG((ksize > 0) == (w_host != nullptr) && (ksize == 0 || Cin > 0),
                "xvb_resnet_set_layer(%s): a weight needs ksize 1 or 3 and Cin > 0, a BatchNorm record ksize 0 and no weight", name);
  XVB_CHECK_ARG((scale_host == nullptr) == (shift_host == nullptr), "xvb_resnet_set_layer(%s): scale and shift go together", name);
  XVB_CHECK_ARG(!(flags & XVB_BN) || scale_host, "xvb_resnet_set_layer(%s): XVB_BN without scale/shift", name);
  XVB_CHECK_ARG(h->m->recs.find(name) == h->m->recs.end(), "xvb_resnet_set_layer: record '%s' set twice", name);
  Rec r;
  r.Cout = Cout; r.Cin = Cin; r.ksize = ksize; r.flags = flags;
  if (w_host) r.w.assign(w_host, w_host + (size_t)Cout * Cin * ksize * ksize);
  if (bias_host) r.b.assign(bias_host, bias_host + Cout);
  if (scale_host) { r.s.assign(scale_host, scale_host + Cout); r.t.assign(shift_host, shift_host + Cout); }
  h->m->recs[name] = std::move(r);
  h->m->order.push_back(name);
  return XVB_OK;
}

extern "C" int xvb_resnet_finalize(xvb_resnet_t* h) {
  XVB_CHECK_ARG(h && !h->finalized && h->m, "xvb_resnet_finalize: null or finalized model");
  Model* m = h->m;
  std::set<std::string> used;
  // a record the configuration needs: present, with the expected shape
  auto need = [&](const std::string& n, int cout, int cin, int k, const Rec** out) -> int {
    const Rec* r = find(m, n);
    XVB_CHECK_ARG(r, "xvb_resnet_finalize: record '%s' is missing", n.c_str());
    XVB_CHECK_ARG(r->Cout == cout && r->Cin == cin && r->ksize == k, "xvb_resnet_finalize: record '%s' is %d x %d x k%d, expected %d x %d x k%d",
                  n.c_str(), r->Cout, r->Cin, r->ksize, cout, cin, k);
    used.insert(n);
    *out = r;
    return XVB_OK;
  };
  auto bn = [&](const std::string& n, int c, Bn* out) -> int {
    const Rec* r;
    int rc = need(n, c, 0, 0, &r);
    if (rc) return rc;
    XVB_CHECK_ARG(!r->s.empty(), "xvb_resnet_finalize: BatchNorm record '%s' has no scale/shift", n.c_str());
    if ((rc = m->upload(&out->s, r->s)) || (rc = m->upload(&out->t, r->t))) return rc;
    return XVB_OK;
  };
  auto conv_rec = [&](const std::string& n, int cout, int cin, int k, Conv* out) -> int {
    const Rec* r;
    int rc = need(n, cout, cin, k, &r);
    return rc ? rc : m->pack(out, r->w, cout, cin, k * k);
  };
  int rc;
  const Rec* r;
  if ((rc = need("resnet.conv1", m->planes[0], 1, 3, &r)) || (rc = m->upload(&m->head_w, r->w)) || (rc = bn("resnet.bn1", m->planes[0], &m->head_bn)))
    return rc;
  const bool use_se = find(m, "resnet.layer1.0.se.fc_1") != nullptr;
  int inp = m->planes[0], f = m->feat_dim;
  m->Cmax = 0; m->Hmax = 0;
  for (int li = 0; li < 4; ++li) {
    const int p = m->planes[li];
    if (li) f = (f - 1) / 2 + 1;
    for (int i = 0; i < m->layers[li]; ++i) {
      const std::string pre = "resnet.layer" + std::to_string(li + 1) + "." + std::to_string(i) + ".";
      Block b;
      b.stride = (li > 0 && i == 0) ? 2 : 1;
      b.cin = i == 0 ? inp : p;
      b.cout = p;
      if ((rc = conv_rec(pre + "conv1", p, b.cin, 3, &b.conv1)) || (rc = conv_rec(pre + "conv2", p, p, 3, &b.conv2)) ||
          (rc = bn(pre + "bn1", m->pre ? b.cin : p, &b.bn1)) || (rc = bn(pre + "bn2", p, &b.bn2)))
        return rc;
      b.has_ds = i == 0 && (li > 0 || inp != p);   // resnet.py:324-328
      if (b.has_ds && ((rc = conv_rec(pre + "downsample.0", p, inp, 1, &b.ds)) || (rc = bn(pre + "downsample.1", p, &b.dsbn)))) return rc;
      b.has_se = use_se;
      if (use_se) {
        const Rec* r1 = find(m, pre + "se.fc_1");
        XVB_CHECK_ARG(r1, "xvb_resnet_finalize: record '%sse.fc_1' is missing (the first block has SE)", pre.c_str());
        const int hid = r1->Cout;
        const Rec* r2;
        if ((rc = need(pre + "se.fc_1", hid, p, 1, &r1)) || (rc = need(pre + "se.fc_2", p, hid, 1, &r2))) return rc;
        XVB_CHECK_ARG(!r1->b.empty() && !r2->b.empty(), "xvb_resnet_finalize: the SE linears of '%s' need their biases", pre.c_str());
        Se& se = b.se;
        se.C = p;
        se.Hp = (hid + 3) / 4 * 4;   // padded hidden units are relu(0) = 0 and meet zero columns of fc_2
        std::vector<float> w1((size_t)se.Hp * p, 0.f), b1(se.Hp, 0.f), w2((size_t)p * se.Hp, 0.f);
        for (int u = 0; u < hid; ++u) {
          for (int c = 0; c < p; ++c) w1[(size_t)u * p + c] = r1->w[(size_t)u * p + c];
          b1[u] = r1->b[u];
        }
        for (int c = 0; c < p; ++c)
          for (int u = 0; u < hid; ++u) w2[(size_t)c * se.Hp + u] = r2->w[(size_t)c * hid + u];
        se.kmax = 1;
        for (int k = 1, l = 0; k * p <= 256 && l < kSeMaxK; k *= 2, ++l) {   // fc_1 of the mean of k-position groups
          std::vector<float> wk((size_t)se.Hp * k * p);
          for (int u = 0; u < se.Hp; ++u)
            for (int j = 0; j < k; ++j)
              for (int c = 0; c < p; ++c) wk[((size_t)u * k + j) * p + c] = w1[(size_t)u * p + c] / (float)k;
          if ((rc = m->upload(&se.w1k[l], wk))) return rc;
          se.kmax = k;
        }
        if (!se.w1k[0] && (rc = m->upload(&se.w1k[0], w1))) return rc;   // C > 256: the plain mean only
        if ((rc = m->upload(&se.b1, b1)) || (rc = m->upload(&se.w2, w2)) || (rc = m->upload(&se.b2, r2->b))) return rc;
        if (se.Hp > m->Hmax) m->Hmax = se.Hp;
      }
      if (p > m->Cmax) m->Cmax = p;
      m->blocks.push_back(b);
    }
    inp = p;
  }
  m->F4 = f;
  m->C4 = m->planes[3];
  // segment level (resnet_xvector.py:194-206): [fc1 ->] [fc2], as many as the extracted position hands over
  int cin = 2 * m->F4 * m->C4;
  for (const char* n : {"fc1", "fc2"}) {
    const Rec* s = find(m, n);
    if (!s) continue;
    rc = need(n, s->Cout, cin, 1, &s);
    if (rc) return rc;
    Seg g;
    g.Cin = cin; g.Cout_real = s->Cout; g.Cout = (s->Cout + 7) / 8 * 8;
    g.flags = (s->flags & XVB_RELU) | (s->s.empty() ? 0 : XVB_BN);
    std::vector<float> w(s->w), b(s->b), sc(s->s), sh(s->t);
    w.resize((size_t)g.Cout * cin, 0.f);   // padded output rows come out as exact zeros
    if (!b.empty()) b.resize(g.Cout, 0.f);
    if (!sc.empty()) { sc.resize(g.Cout, 0.f); sh.resize(g.Cout, 0.f); }
    if ((rc = m->pack(&g.w, w, g.Cout, cin, 1)) || (rc = m->upload(&g.bias, b)) || (rc = m->upload(&g.scale, sc)) ||
        (rc = m->upload(&g.shift, sh)))
      return rc;
    m->seg.push_back(g);
    cin = s->Cout;
  }
  XVB_CHECK_ARG(!m->seg.empty(), "xvb_resnet_finalize: record 'fc1' or 'fc2' is missing (no segment layer)");
  m->E = m->seg.back().Cout_real;
  m->seg_mid = m->seg.size() > 1 ? m->seg[0].Cout : 0;
  for (const std::string& n : m->order)
    XVB_CHECK_ARG(used.count(n), "xvb_resnet_finalize: record '%s' is not part of this configuration", n.c_str());
  h->finalized = true;
  return XVB_OK;
}

extern "C" int xvb_resnet_feat_dim(const xvb_resnet_t* h) { return h && h->m ? h->m->feat_dim : XVB_EINVAL; }
extern "C" int xvb_resnet_embed_dim(const xvb_resnet_t* h) { return h && h->finalized ? h->m->E : XVB_EINVAL; }
extern "C" int xvb_resnet_last_launches(const xvb_resnet_t* h) { return h ? h->last_launches : 0; }

extern "C" int xvb_resnet_extract(xvb_resnet_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(h && h->finalized, "xvb_resnet_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_resnet_extract: bad arguments");
  const long before = g_launches;
  const long long per_utt = (long long)T * h->m->feat_dim;
  int g = (int)(kPositionBudget / per_utt);
  if (g < 1) g = 1;
  for (int i = 0; i < B; i += g) {
    const int b = B - i < g ? B - i : g;
    int rc = extract_group(h, feats + (size_t)i * per_utt, b, T, emb + (size_t)i * h->m->E, stream);
    if (rc) return rc;
  }
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

extern "C" int xvb_resnet_extract_host(xvb_resnet_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats_host && emb_host && B > 0 && T > 0, "xvb_resnet_extract_host: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t nf = (size_t)B * T * h->m->feat_dim, ne = (size_t)B * h->m->E;
  int rc;
  if (nf > h->h_feats_cap) {
    cudaFree(h->h_feats); h->h_feats = nullptr; h->h_feats_cap = 0;
    XVB_CUDA(cudaMalloc((void**)&h->h_feats, nf * sizeof(float)));
    h->h_feats_cap = nf;
  }
  if (ne > h->h_emb_cap) {
    cudaFree(h->h_emb); h->h_emb = nullptr; h->h_emb_cap = 0;
    XVB_CUDA(cudaMalloc((void**)&h->h_emb, ne * sizeof(float)));
    h->h_emb_cap = ne;
  }
  XVB_CUDA(cudaMemcpyAsync(h->h_feats, feats_host, nf * sizeof(float), cudaMemcpyHostToDevice, s));
  if ((rc = xvb_resnet_extract(h, h->h_feats, B, T, h->h_emb, stream))) return rc;
  XVB_CUDA(cudaMemcpyAsync(emb_host, h->h_emb, ne * sizeof(float), cudaMemcpyDeviceToHost, s));
  XVB_CUDA(cudaStreamSynchronize(s));
  return XVB_OK;
}

// ---- whole shards: the protocol of xvb_ecapa_extract_shard[_host] ------------------------------------------------
namespace {

// Two lanes unless XVB_LANES=0 (read per call, so one process can compare both).
bool lanes_enabled() {
  const char* v = getenv("XVB_LANES");
  return v ? atoi(v) != 0 : true;
}

int ensure_lanes(xvb_resnet* h) {
  if (h->lane1) return XVB_OK;
  for (int i = 0; i < 2; ++i) {
    XVB_CUDA(cudaStreamCreateWithFlags(&h->lane_stream[i], cudaStreamNonBlocking));
    XVB_CUDA(cudaEventCreateWithFlags(&h->ev_lane_done[i], cudaEventDisableTiming));
  }
  XVB_CUDA(cudaEventCreateWithFlags(&h->ev_lane_start, cudaEventDisableTiming));
  xvb_resnet* c = new xvb_resnet();
  c->m = h->m;
  c->owns_model = false;
  c->finalized = true;
  h->lane1 = c;
  return XVB_OK;
}
int lanes_fork(xvb_resnet* h, cudaStream_t s) {
  XVB_CUDA(cudaEventRecord(h->ev_lane_start, s));
  for (int i = 0; i < 2; ++i) XVB_CUDA(cudaStreamWaitEvent(h->lane_stream[i], h->ev_lane_start, 0));
  return XVB_OK;
}
int lanes_join(xvb_resnet* h, cudaStream_t s) {
  for (int i = 0; i < 2; ++i) {
    XVB_CUDA(cudaEventRecord(h->ev_lane_done[i], h->lane_stream[i]));
    XVB_CUDA(cudaStreamWaitEvent(s, h->ev_lane_done[i], 0));
  }
  return XVB_OK;
}

}  // namespace

extern "C" int xvb_resnet_extract_shard(xvb_resnet_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats && emb && N > 0 && T > 0 && batch > 0, "xvb_resnet_extract_shard: bad arguments");
  const size_t F = (size_t)h->m->feat_dim, E = (size_t)h->m->E;
  const bool lanes = lanes_enabled() && N > batch;
  int rc, launches = 0, k = 0;
  if (lanes && ((rc = ensure_lanes(h)) || (rc = lanes_fork(h, (cudaStream_t)stream)))) return rc;
  for (int64_t i = 0; i < N; i += batch, ++k) {
    const int b = (int)(N - i < batch ? N - i : batch);
    xvb_resnet* lane = (lanes && (k & 1)) ? h->lane1 : h;
    void* ls = lanes ? (void*)h->lane_stream[k & 1] : stream;
    if ((rc = xvb_resnet_extract(lane, feats + (size_t)i * T * F, b, T, emb + (size_t)i * E, ls))) return rc;
    launches += lane->last_launches;
  }
  if (lanes && (rc = lanes_join(h, (cudaStream_t)stream))) return rc;
  h->last_launches = launches;
  return XVB_OK;
}

extern "C" int xvb_resnet_extract_shard_host(xvb_resnet_t* h, const float* feats_host, int64_t N, int T, int batch,
                                             float* emb_host, void* stream) {
  XVB_CHECK_ARG(h && h->finalized && feats_host && emb_host && N > 0 && T > 0 && batch > 0, "xvb_resnet_extract_shard_host: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  constexpr int S = xvb_resnet::kSlots;
  if (!h->copy_stream) {
    XVB_CUDA(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < S; ++i) {
      XVB_CUDA(cudaEventCreateWithFlags(&h->ev_h2d[i], cudaEventDisableTiming));
      XVB_CUDA(cudaEventCreateWithFlags(&h->ev_done[i], cudaEventDisableTiming));
    }
  }
  const size_t F = (size_t)h->m->feat_dim, E = (size_t)h->m->E;
  const int bmax = (int)(N < batch ? N : batch);
  const size_t nf = (size_t)bmax * T * F, ne = (size_t)bmax * E;
  int rc;
  for (int slot = 0; slot < S; ++slot) {
    if (nf > h->p_feats_cap[slot]) {
      cudaFree(h->p_feats[slot]); h->p_feats[slot] = nullptr; h->p_feats_cap[slot] = 0;
      XVB_CUDA(cudaMalloc((void**)&h->p_feats[slot], nf * sizeof(float)));
      h->p_feats_cap[slot] = nf;
    }
    if (ne > h->p_emb_cap[slot]) {
      cudaFree(h->p_emb[slot]); h->p_emb[slot] = nullptr; h->p_emb_cap[slot] = 0;
      XVB_CUDA(cudaMalloc((void**)&h->p_emb[slot], ne * sizeof(float)));
      h->p_emb_cap[slot] = ne;
    }
  }
  const bool lanes = lanes_enabled() && N > batch;
  if (lanes && ((rc = ensure_lanes(h)) || (rc = lanes_fork(h, s)))) return rc;
  int launches = 0, k = 0;
  for (int64_t i = 0; i < N; i += batch, ++k) {
    const int b = (int)(N - i < batch ? N - i : batch);
    const int slot = k % S;
    xvb_resnet* lane = (lanes && (k & 1)) ? h->lane1 : h;
    cudaStream_t ls = lanes ? h->lane_stream[k & 1] : s;
    if (k >= S) XVB_CUDA(cudaStreamWaitEvent(h->copy_stream, h->ev_done[slot], 0));
    XVB_CUDA(cudaMemcpyAsync(h->p_feats[slot], feats_host + (size_t)i * T * F, (size_t)b * T * F * sizeof(float),
                             cudaMemcpyHostToDevice, h->copy_stream));
    XVB_CUDA(cudaEventRecord(h->ev_h2d[slot], h->copy_stream));
    XVB_CUDA(cudaStreamWaitEvent(ls, h->ev_h2d[slot], 0));
    if ((rc = xvb_resnet_extract(lane, h->p_feats[slot], b, T, h->p_emb[slot], ls))) return rc;
    XVB_CUDA(cudaMemcpyAsync(emb_host + (size_t)i * E, h->p_emb[slot], (size_t)b * E * sizeof(float), cudaMemcpyDeviceToHost, ls));
    XVB_CUDA(cudaEventRecord(h->ev_done[slot], ls));
    launches += lane->last_launches;
  }
  if (lanes && (rc = lanes_join(h, s))) return rc;
  XVB_CUDA(cudaStreamSynchronize(s));
  h->last_launches = launches;
  return XVB_OK;
}

// ---- "XVBR0001" model files: the create arguments, then the named records as handed over -------------------------
extern "C" int xvb_resnet_save(const xvb_resnet_t* h, const char* path) {
  XVB_CHECK_ARG(h && h->finalized && path, "xvb_resnet_save: model not finalized");
  const Model* m = h->m;
  FILE* f = fopen(path, "wb");
  XVB_CHECK_ARG(f, "xvb_resnet_save: cannot open '%s'", path);
  bool ok = fwrite("XVBR0001", 1, 8, f) == 8;
  const int32_t hd[10] = {m->feat_dim, m->layers[0], m->layers[1], m->layers[2], m->layers[3],
                          m->planes[0], m->planes[1], m->planes[2], m->planes[3], m->pre};
  const int32_t nrec = (int32_t)m->order.size();
  ok = ok && fwrite(hd, 4, 10, f) == 10 && fwrite(&m->eps, 4, 1, f) == 1 && fwrite(&nrec, 4, 1, f) == 1;
  for (const std::string& n : m->order) {
    const Rec& r = m->recs.at(n);
    const int32_t nl = (int32_t)n.size();
    const int32_t rec[7] = {r.Cout, r.Cin, r.ksize, r.flags, (int32_t)!r.w.empty(), (int32_t)!r.b.empty(), (int32_t)!r.s.empty()};
    ok = ok && fwrite(&nl, 4, 1, f) == 1 && fwrite(n.data(), 1, n.size(), f) == n.size() && fwrite(rec, 4, 7, f) == 7 &&
         fwrite(r.w.data(), 4, r.w.size(), f) == r.w.size() && fwrite(r.b.data(), 4, r.b.size(), f) == r.b.size() &&
         fwrite(r.s.data(), 4, r.s.size(), f) == r.s.size() && fwrite(r.t.data(), 4, r.t.size(), f) == r.t.size();
  }
  ok = fclose(f) == 0 && ok;
  XVB_CHECK_ARG(ok, "xvb_resnet_save: write to '%s' failed", path);
  return XVB_OK;
}

extern "C" int xvb_resnet_load(xvb_resnet_t** out, const char* path) {
  XVB_CHECK_ARG(out && path, "xvb_resnet_load: null argument");
  FILE* f = fopen(path, "rb");
  XVB_CHECK_ARG(f, "xvb_resnet_load: cannot open '%s'", path);
  auto rd = [&](void* p, size_t n) { return fread(p, 1, n, f) == n; };
  char magic[8];
  int32_t hd[10], nrec = 0;
  float eps = 0.f;
  xvb_resnet_t* h = nullptr;
  int rc = XVB_EINVAL;
  do {
    if (!rd(magic, 8) || memcmp(magic, "XVBR0001", 8) != 0 || !rd(hd, sizeof hd) || !rd(&eps, 4) || !rd(&nrec, 4) || nrec < 1 ||
        nrec > 4096) {
      set_error("xvb_resnet_load: '%s' is not an XVBR0001 file", path);
      break;
    }
    if ((rc = xvb_resnet_create(&h, hd[0], hd + 1, hd + 5, hd[9], eps))) break;
    std::vector<float> w, b, s, t;
    for (int i = 0; i < nrec && rc == XVB_OK; ++i) {
      int32_t nl = 0, rec[7];
      char name[128];
      bool ok = rd(&nl, 4) && nl > 0 && nl < 127 && rd(name, (size_t)nl) && rd(rec, sizeof rec) && rec[0] > 0 && rec[0] <= 65536 &&
                rec[1] >= 0 && rec[1] <= (1 << 20) && (rec[2] == 0 || rec[2] == 1 || rec[2] == 3) && rec[4] == (rec[2] > 0) &&
                (int64_t)rec[0] * rec[1] * rec[2] * rec[2] <= (int64_t)1 << 28;
      if (ok) {
        name[nl] = 0;
        w.resize(rec[4] ? (size_t)rec[0] * rec[1] * rec[2] * rec[2] : 0);
        ok = rd(w.data(), w.size() * 4);
        if (ok && rec[5]) { b.resize(rec[0]); ok = rd(b.data(), b.size() * 4); }
        if (ok && rec[6]) { s.resize(rec[0]); t.resize(rec[0]); ok = rd(s.data(), s.size() * 4) && rd(t.data(), t.size() * 4); }
      }
      if (!ok) { set_error("xvb_resnet_load: '%s' is truncated or corrupt at record %d", path, i); rc = XVB_EINVAL; break; }
      rc = xvb_resnet_set_layer(h, name, rec[0], rec[1], rec[2], rec[4] ? w.data() : nullptr, rec[5] ? b.data() : nullptr,
                                rec[6] ? s.data() : nullptr, rec[6] ? t.data() : nullptr, rec[3]);
    }
    if (rc == XVB_OK) rc = xvb_resnet_finalize(h);
  } while (0);
  fclose(f);
  if (rc != XVB_OK) { if (h) xvb_resnet_destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}

extern "C" void xvb_resnet_destroy(xvb_resnet_t* h) {
  if (!h) return;
  if (h->lane1) xvb_resnet_destroy(h->lane1);
  for (int i = 0; i < 2; ++i) {
    if (h->lane_stream[i]) cudaStreamDestroy(h->lane_stream[i]);
    if (h->ev_lane_done[i]) cudaEventDestroy(h->ev_lane_done[i]);
  }
  if (h->ev_lane_start) cudaEventDestroy(h->ev_lane_start);
  h->free_ws();
  cudaFree(h->h_feats); cudaFree(h->h_emb);
  for (int i = 0; i < xvb_resnet::kSlots; ++i) {
    cudaFree(h->p_feats[i]); cudaFree(h->p_emb[i]);
    if (h->ev_h2d[i]) cudaEventDestroy(h->ev_h2d[i]);
    if (h->ev_done[i]) cudaEventDestroy(h->ev_done[i]);
  }
  if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
  if (h->owns_model) delete h->m;
  delete h;
}
