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
// folded to (scale, shift) by the caller; the segment layers arrive as the Python hands them to ops.PackedAffine (fc1
// / fc2 export(), the first one's input columns already permuted to the (B, T', F', C) pooling order).  This file only
// packs and pads: conv weights through xvb_pack_tdnn_weight, the SE hidden width zero-padded to a multiple of 4 with
// fc_1 replicated k times (divided by k) for the k-grouped plane mean, segment rows padded to a multiple of 8.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <memory>
#include <string>
#include <vector>

#include "records.cuh"
#include "shard.cuh"

namespace {

using namespace xvb;

// One B*T*F position budget per extract call: larger calls run as consecutive groups of utterances (see xvb200.h).
constexpr long long kPositionBudget = 256LL * 200 * 80;
constexpr int kSeMaxK = 9;   // k = 1, 2, ..., 256 for the k-grouped SE mean
struct Config {   // the create arguments, laid out as the configuration block of a model file
  int32_t feat_dim = 0, layers[4] = {0}, planes[4] = {0}, pre = 0;
  float eps = 0.f;   // pooling_eps
};
static_assert(sizeof(Config) == 10 * sizeof(int32_t) + sizeof(float), "the XVBR0001 configuration block");
const RecordFormat kFile = {"XVBR0001", sizeof(Config), 3, 4096};
struct Bn { float* s = nullptr; float* t = nullptr; };
struct Se {
  int C = 0, Hp = 0, kmax = 1;           // hidden width padded to a multiple of 4; k = 1 .. kmax (powers of two)
  float* w1k[kSeMaxK] = {nullptr};       // index log2(k): (Hp, k*C) = [w1 / k, ..., w1 / k]
  float* b1 = nullptr; float* w2 = nullptr; float* b2 = nullptr;
};
struct Block {
  int stride = 1, cin = 0, cout = 0;
  Planes conv1, conv2, ds;
  Bn bn1, bn2, dsbn;
  bool has_ds = false, has_se = false;
  Se se;
};
struct Model {
  Config cfg;
  RecordStore recs{kFile.nshape};
  float* head_w = nullptr;
  Bn head_bn;
  std::vector<Block> blocks;
  SegTail tail;
  int F4 = 0, C4 = 0, Cmax = 0, Hmax = 0;
  Weights dev{"xvb_resnet_finalize"};
};

}  // namespace

struct xvb_resnet : Handle<Model> {
  // workspace, each buffer grown to the largest call seen: seven rotating (B, T', F', C) plane buffers for the roles
  // block input / activated input / h / identity / z / output / next activated input, picked by index, the fp32
  // last-layer output, then the per-utterance buffers (pooled statistics, SE mean / hidden / gate, segment layers) and
  // a masked call's lengths at the four time resolutions (int32 (kLevels, B), level l = after l stride-2 stages)
  static constexpr int kRotating = 7;
  static constexpr int kLevels = 4;
  enum { kRot0, kLast = kRot0 + kRotating, kPooled, kPooledF32, kSeMean, kSeHidden, kSeGate, kSegMid, kSegOut, kLengths, kBufs };
  Workspace<kBufs> ws;
  Shard<xvb_resnet> shard;

  using Handle::Handle;
};

using H = xvb_resnet;

template <>
struct xvb::ShardFamily<xvb_resnet> {
  static int extract(xvb_resnet* h, const float* feats, int B, int T, float* emb, void* stream) {
    return xvb_resnet_extract(h, feats, B, T, emb, stream);
  }
  static xvb_resnet* twin(const xvb_resnet* h) { return new xvb_resnet(h->m); }
  static int feat_dim(const xvb_resnet* h) { return h->m->cfg.feat_dim; }
  static int embed_dim(const xvb_resnet* h) { return h->m->tail.E; }
};

namespace {

int log2i(int k) { int l = 0; while ((1 << l) < k) ++l; return l; }

// Position-buffer sizes (elements) of one (B, T) call: the largest (B, T', F', C) tensor and the last layer's output.
void shapes(const Model* m, int B, int T, size_t* planes, size_t* last) {
  long long t = T, f = m->cfg.feat_dim;
  size_t mx = (size_t)B * t * f * m->cfg.planes[0];
  for (const Block& b : m->blocks) {
    t = (t - 1) / b.stride + 1;
    f = (f - 1) / b.stride + 1;
    const size_t n = (size_t)B * t * f * b.cout;
    if (n > mx) mx = n;
  }
  *planes = mx;
  *last = (size_t)B * t * f * m->C4;
}

int reserve(H* h, int B, int T) {
  const Model* m = h->m.get();
  size_t need[H::kBufs], np;
  shapes(m, B, T, &np, &need[H::kLast]);
  for (int i = 0; i < H::kRotating; ++i) need[H::kRot0 + i] = np;
  const size_t b = (size_t)B;
  need[H::kPooled] = need[H::kPooledF32] = b * 2 * m->F4 * m->C4;
  need[H::kSeMean] = b * (m->Cmax > 256 ? m->Cmax : 256);
  need[H::kSeHidden] = b * (m->Hmax ? m->Hmax : 4);
  need[H::kSeGate] = b * m->Cmax;
  need[H::kSegMid] = b * (m->tail.mid ? m->tail.mid : 8);
  need[H::kSegOut] = b * m->tail.out_rows();
  need[H::kLengths] = 0;   // sized by xvb_resnet_extract_lengths for the whole call, before its groups run
  bool planes[H::kBufs];
  for (int i = 0; i < H::kBufs; ++i) planes[i] = i < H::kLast || i == H::kPooled || i == H::kSegMid;
  uint64_t grown;
  return h->ws.reserve(need, planes, &grown);
}

int conv(const Planes& x, const Planes& w, int B, int T, int F, int Cin, int Cout, int k, int stride, const Bn& bn,
         const Planes* res, int relu, const Planes* y, float* y_f32, const Bn& bn2, const Planes* y2, const int* lens,
         void* stream) {
  xvb_conv2d_args_t a{};
  a.lengths = lens;
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

// sigmoid(fc_2(relu(fc_1(mean over the T * F positions of z)))) as ResNetExtractor._se_gate: the (B, T*F, C) planes
// read as (B, T*F/k, k*C) with the largest k in the table (2k too) that divides T * F.  A masked batch (lens: frames
// per utterance) takes the largest such k dividing F, so that k divides every utterance's own positions.
int se_gate(xvb_resnet* h, const Se& se, const Planes& z, int B, int T, int F, const int* lens, void* stream) {
  const long long P = (long long)T * F;
  int k = 1;
  while (2 * k <= se.kmax && (lens ? F : P) % (2 * k) == 0) k *= 2;
  const int kc = k * se.C;
  float* mean = h->ws.f32(H::kSeMean);
  float* hidden = h->ws.f32(H::kSeHidden);
  int rc = lens ? xvb_plane_mean_lengths(z.hi, z.lo, kc, B, (int)(P / k), kc, lens, F / k, mean, nullptr, nullptr, kc, stream)
                : xvb_plane_mean(z.hi, z.lo, kc, B, (int)(P / k), kc, mean, nullptr, nullptr, kc, stream);
  if (!rc) rc = xvb_small_affine(mean, kc, se.w1k[log2i(k)], B, kc, se.Hp, se.b1, nullptr, nullptr, XVB_RELU,
                                 hidden, se.Hp, nullptr, nullptr, 0, stream);
  if (!rc) rc = xvb_small_affine(hidden, se.Hp, se.w2, B, se.Hp, se.C, se.b2, nullptr, nullptr, XVB_SIGMOID,
                                 h->ws.f32(H::kSeGate), se.C, nullptr, nullptr, 0, stream);
  return rc;
}

// One group of utterances (B * T * F within the budget, or a single utterance): ResNetExtractor.extract.  A masked
// group passes lens, its lengths at level 0 of the workspace's (kLevels, ld) table; NULL otherwise.
int extract_group(xvb_resnet* h, const float* feats, int B, int T, const int* lens, int ld, float* emb, void* stream) {
  int rc = reserve(h, B, T);
  if (rc) return rc;
  Planes buf[H::kRotating];
  for (int i = 0; i < H::kRotating; ++i) buf[i] = h->ws.planes(H::kRot0 + i);
  const Model* m = h->m.get();
  const bool pre = m->cfg.pre != 0;
  int Tl = T, Fl = m->cfg.feat_dim;
  int xi = 0, ai = pre ? 1 : -1;
  const Bn none;
  int level = 0;
  auto at = [&](int l) { return lens ? lens + (size_t)l * ld : nullptr; };
  {
    const Bn first = pre ? m->blocks[0].bn1 : none;
    const Planes* a = pre ? &buf[ai] : nullptr;
    rc = lens ? xvb_conv2d_head_lengths(feats, B, T, Fl, lens, m->head_w, m->cfg.planes[0], m->head_bn.s, m->head_bn.t, buf[xi].hi,
                                        buf[xi].lo, first.s, first.t, a ? a->hi : nullptr, a ? a->lo : nullptr, stream)
              : xvb_conv2d_head(feats, B, T, Fl, m->head_w, m->cfg.planes[0], m->head_bn.s, m->head_bn.t, buf[xi].hi, buf[xi].lo,
                                first.s, first.t, a ? a->hi : nullptr, a ? a->lo : nullptr, stream);
    if (rc) return rc;
  }
  const int nb = (int)m->blocks.size();
  for (int i = 0; i < nb; ++i) {
    const Block& blk = m->blocks[i];
    const bool last = i + 1 == nb;
    const int st = blk.stride, co = blk.cout, Tn = (Tl - 1) / st + 1, Fn = (Fl - 1) / st + 1;
    const int* lin = at(level);   // lengths of the block input and of its output
    const int* lout = at(st == 2 ? level + 1 : level);
    unsigned used = (1u << xi) | (ai >= 0 ? 1u << ai : 0u);
    auto take = [&]() { int j = 0; while (used & (1u << j)) ++j; used |= 1u << j; return j; };
    const int hh = take();
    // pre-activation: h = relu(bn2(conv1(relu(bn1(x))))); post-activation: h = relu(bn1(conv1(x)))
    if ((rc = conv(pre ? buf[ai] : buf[xi], blk.conv1, B, Tl, Fl, blk.cin, co, 3, st, pre ? blk.bn2 : blk.bn1, nullptr, 1,
                   &buf[hh], nullptr, none, nullptr, lin, stream)))
      return rc;
    int id = xi;
    if (blk.has_ds) {   // conv1x1 (stride) + BN of the un-activated block input
      id = take();
      if ((rc = conv(buf[xi], blk.ds, B, Tl, Fl, blk.cin, co, 1, st, blk.dsbn, nullptr, 0, &buf[id], nullptr, none, nullptr, lin,
                     stream)))
        return rc;
    }
    const Bn nxt = (!last && pre) ? m->blocks[i + 1].bn1 : none;
    const int yi = last ? -1 : take();
    const int an = nxt.s ? take() : -1;
    const Planes* y = yi >= 0 ? &buf[yi] : nullptr;
    const Planes* y2 = an >= 0 ? &buf[an] : nullptr;
    float* yf = last ? h->ws.f32(H::kLast) : nullptr;
    const Bn bn2 = pre ? none : blk.bn2;
    if (!blk.has_se) {   // conv2 [+ bn2] + identity [-> relu] in one epilogue
      if ((rc = conv(buf[hh], blk.conv2, B, Tn, Fn, co, co, 3, 1, bn2, &buf[id], pre ? 0 : 1, y, yf, nxt, y2, lout, stream)))
        return rc;
    } else {
      const int zi = take();
      if ((rc = conv(buf[hh], blk.conv2, B, Tn, Fn, co, co, 3, 1, bn2, nullptr, 0, &buf[zi], nullptr, none, nullptr, lout,
                     stream)))
        return rc;
      if ((rc = se_gate(h, blk.se, buf[zi], B, Tn, Fn, lout, stream))) return rc;
      const float* gate = h->ws.f32(H::kSeGate);
      Planes yp, y2p;
      if (y) yp = *y;
      if (y2) y2p = *y2;
      rc = lout ? xvb_se_residual_lengths(buf[zi].hi, buf[zi].lo, gate, buf[id].hi, buf[id].lo, B, Tn, Fn, co, lout, pre ? 0 : 1,
                                          yp.hi, yp.lo, yf, nxt.s, nxt.t, y2p.hi, y2p.lo, stream)
                : xvb_se_residual(buf[zi].hi, buf[zi].lo, gate, buf[id].hi, buf[id].lo, B, (long long)Tn * Fn, co, pre ? 0 : 1,
                                  yp.hi, yp.lo, yf, nxt.s, nxt.t, y2p.hi, y2p.lo, stream);
      if (rc) return rc;
    }
    xi = yi; ai = an; Tl = Tn; Fl = Fn;
    if (st == 2) ++level;
  }
  return m->tail.run(h->ws.f32(H::kLast), Fl * m->C4, B, Tl, m->cfg.eps, h->ws.planes(H::kPooled), h->ws.f32(H::kPooledF32),
                     h->ws.planes(H::kSegMid), h->ws.f32(H::kSegOut), emb, stream, at(level));
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
  Config& c = h->draft->cfg;
  c.feat_dim = feat_dim;
  for (int i = 0; i < 4; ++i) { c.layers[i] = layers[i]; c.planes[i] = planes[i]; }
  c.pre = pre_activation ? 1 : 0;
  c.eps = pooling_eps;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_resnet_set_layer(xvb_resnet_t* h, const char* name, int Cout, int Cin, int ksize, const float* w_host,
                                    const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && strlen(name) > 0 && strlen(name) < 127, "xvb_resnet_set_layer: bad arguments or finalized model");
  XVB_CHECK_ARG(ksize == 0 || ksize == 1 || ksize == 3, "xvb_resnet_set_layer(%s): bad shape %d x %d x k%d", name, Cout, Cin, ksize);
  const char* fn = "xvb_resnet_set_layer";
  const int shape[3] = {Cout, Cin, ksize};
  int rc = h->draft->recs.check(fn, name, shape, w_host, scale_host, shift_host);
  if (rc) return rc;
  XVB_CHECK_ARG(!(flags & XVB_BN) || scale_host, "xvb_resnet_set_layer(%s): XVB_BN without scale/shift", name);
  return h->draft->recs.add(fn, name, shape, w_host, bias_host, scale_host, shift_host, flags);
}

static int build(Model* m, RecordStore& recs) {
  // a record the configuration needs: present, with the expected shape
  auto need = [&](const std::string& n, int cout, int cin, int k, const Rec** out) -> int {
    const int shape[3] = {cout, cin, k};
    return recs.take("xvb_resnet_finalize", n, shape, out);
  };
  auto bn = [&](const std::string& n, int c, Bn* out) -> int {
    const Rec* r;
    int rc = need(n, c, 0, 0, &r);
    if (rc) return rc;
    XVB_CHECK_ARG(!r->s.empty(), "xvb_resnet_finalize: BatchNorm record '%s' has no scale/shift", n.c_str());
    if ((rc = m->dev.upload(&out->s, r->s)) || (rc = m->dev.upload(&out->t, r->t))) return rc;
    return XVB_OK;
  };
  auto conv_rec = [&](const std::string& n, int cout, int cin, int k, Planes* out) -> int {
    const Rec* r;
    int rc = need(n, cout, cin, k, &r);
    return rc ? rc : m->dev.pack(out, r->w, cout, cin, k * k, kTaps, k * k);
  };
  int rc;
  const Rec* r;
  if ((rc = need("resnet.conv1", m->cfg.planes[0], 1, 3, &r)) || (rc = m->dev.upload(&m->head_w, r->w)) || (rc = bn("resnet.bn1", m->cfg.planes[0], &m->head_bn)))
    return rc;
  const bool use_se = recs.find("resnet.layer1.0.se.fc_1") != nullptr;
  int inp = m->cfg.planes[0], f = m->cfg.feat_dim;
  m->Cmax = 0; m->Hmax = 0;
  for (int li = 0; li < 4; ++li) {
    const int p = m->cfg.planes[li];
    if (li) f = (f - 1) / 2 + 1;
    for (int i = 0; i < m->cfg.layers[li]; ++i) {
      const std::string pre = "resnet.layer" + std::to_string(li + 1) + "." + std::to_string(i) + ".";
      Block b;
      b.stride = (li > 0 && i == 0) ? 2 : 1;
      b.cin = i == 0 ? inp : p;
      b.cout = p;
      if ((rc = conv_rec(pre + "conv1", p, b.cin, 3, &b.conv1)) || (rc = conv_rec(pre + "conv2", p, p, 3, &b.conv2)) ||
          (rc = bn(pre + "bn1", m->cfg.pre ? b.cin : p, &b.bn1)) || (rc = bn(pre + "bn2", p, &b.bn2)))
        return rc;
      b.has_ds = i == 0 && (li > 0 || inp != p);   // resnet.py:324-328
      if (b.has_ds && ((rc = conv_rec(pre + "downsample.0", p, inp, 1, &b.ds)) || (rc = bn(pre + "downsample.1", p, &b.dsbn)))) return rc;
      b.has_se = use_se;
      if (use_se) {
        const Rec* r1 = recs.find(pre + "se.fc_1");
        XVB_CHECK_ARG(r1, "xvb_resnet_finalize: record '%sse.fc_1' is missing (the first block has SE)", pre.c_str());
        const int hid = r1->shape[0];
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
          if ((rc = m->dev.upload(&se.w1k[l], wk))) return rc;
          se.kmax = k;
        }
        if (!se.w1k[0] && (rc = m->dev.upload(&se.w1k[0], w1))) return rc;   // C > 256: the plain mean only
        if ((rc = m->dev.upload(&se.b1, b1)) || (rc = m->dev.upload(&se.w2, w2)) || (rc = m->dev.upload(&se.b2, r2->b))) return rc;
        if (se.Hp > m->Hmax) m->Hmax = se.Hp;
      }
      if (p > m->Cmax) m->Cmax = p;
      m->blocks.push_back(b);
    }
    inp = p;
  }
  m->F4 = f;
  m->C4 = m->cfg.planes[3];
  // segment level (resnet_xvector.py:194-206): [fc1 ->] [fc2], as many as the extracted position hands over
  if ((rc = m->tail.build(recs, m->dev, "xvb_resnet_finalize", 2 * m->F4 * m->C4))) return rc;
  return recs.check_all_used("xvb_resnet_finalize");
}

extern "C" int xvb_resnet_finalize(xvb_resnet_t* h) { return publish_built(h, build, "xvb_resnet_finalize"); }

extern "C" int xvb_resnet_feat_dim(const xvb_resnet_t* h) { return h ? h->m->cfg.feat_dim : XVB_EINVAL; }
extern "C" int xvb_resnet_embed_dim(const xvb_resnet_t* h) { return finalized(h) ? h->m->tail.E : XVB_EINVAL; }
extern "C" int xvb_resnet_last_launches(const xvb_resnet_t* h) { return h ? h->last_launches : 0; }

extern "C" int xvb_resnet_extract(xvb_resnet_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_resnet_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_resnet_extract: bad arguments");
  const long before = g_launches;
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->tail.E;
  int rc = for_groups(B, (long long)per_utt, kPositionBudget,
                      [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, nullptr, 0, emb + i * E, stream); });
  if (rc) return rc;
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

extern "C" int xvb_resnet_extract_lengths(xvb_resnet_t* h, const float* feats, const int32_t* lengths_host, int B, int T,
                                          float* emb, void* stream) {
  const char* fn = "xvb_resnet_extract_lengths";
  XVB_CHECK_ARG(finalized(h), "%s: model not finalized", fn);
  XVB_CHECK_ARG(feats && lengths_host && emb && B > 0 && T > 0, "%s: bad arguments", fn);
  bool all_T;
  int rc = check_lengths(fn, lengths_host, B, T, &all_T);
  if (rc) return rc;
  if (all_T) return xvb_resnet_extract(h, feats, B, T, emb, stream);   // nothing to mask: the unmasked call itself
  // level l + 1 = ceil(level l / 2): every stride-2 conv's output length, (L + 2 * pad - k) / 2 + 1 for k = 3 and 1
  std::vector<int32_t> table((size_t)H::kLevels * B);
  for (int b = 0; b < B; ++b) {
    table[b] = lengths_host[b];
    for (int l = 1; l < H::kLevels; ++l) table[(size_t)l * B + b] = (table[(size_t)(l - 1) * B + b] - 1) / 2 + 1;
  }
  size_t need[H::kBufs] = {0};
  bool planes[H::kBufs] = {false};
  need[H::kLengths] = table.size();
  uint64_t grown;
  if ((rc = h->ws.reserve(need, planes, &grown))) return rc;
  int* lens = h->ws.i32(H::kLengths);
  // stream-ordered: the previous call's kernels on `stream` have read the old table before this one lands
  XVB_CUDA(cudaMemcpyAsync(lens, table.data(), table.size() * sizeof(int32_t), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  const long before = g_launches;
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->tail.E;
  rc = for_groups(B, (long long)per_utt, kPositionBudget,
                  [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, lens + i, B, emb + i * E, stream); });
  if (rc) return rc;
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

extern "C" int xvb_resnet_extract_host(xvb_resnet_t* h, const float* feats_host, int B, int T, float* emb_host, void* stream) {
  return Shard<H>::extract_host(h, feats_host, B, T, emb_host, stream, "xvb_resnet_extract_host");
}

// ---- whole shards: the protocol of shard.cuh ---------------------------------------------------------------------
extern "C" int xvb_resnet_extract_shard(xvb_resnet_t* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream) {
  return Shard<H>::device(h, feats, N, T, batch, emb, stream, false, "xvb_resnet_extract_shard");
}

extern "C" int xvb_resnet_extract_shard_host(xvb_resnet_t* h, const float* feats_host, int64_t N, int T, int batch,
                                             float* emb_host, void* stream) {
  return Shard<H>::host(h, feats_host, N, T, batch, emb_host, stream, false, "xvb_resnet_extract_shard_host");
}

// ---- "XVBR0001" model files: the create arguments, then the named records as handed over (save_records) -----------
extern "C" int xvb_resnet_save(const xvb_resnet_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_resnet_save: model not finalized");
  return save_records("xvb_resnet_save", path, kFile, &h->m->cfg, h->m->recs);
}

extern "C" int xvb_resnet_load(xvb_resnet_t** out, const char* path) {
  return load_records(
      "xvb_resnet_load", path, kFile, (void**)out,
      [](void** h, const void* cfg) {
        const Config* c = (const Config*)cfg;
        return xvb_resnet_create((xvb_resnet_t**)h, c->feat_dim, c->layers, c->planes, c->pre, c->eps);
      },
      [](void* h, const char* name, const int* shape, const float* w, const float* b, const float* s, const float* t, int flags) {
        return xvb_resnet_set_layer((xvb_resnet_t*)h, name, shape[0], shape[1], shape[2], w, b, s, t, flags);
      },
      [](void* h) { return xvb_resnet_finalize((xvb_resnet_t*)h); }, [](void* h) { xvb_resnet_destroy((xvb_resnet_t*)h); });
}

extern "C" void xvb_resnet_destroy(xvb_resnet_t* h) { delete h; }
