// Whole-model extractor for the RepVGG / RepSPK x-vector (pytorch/model/repvgg_xvector.py, RepVggXvector
// .extract_embedding :181-208 over pytorch/libs/nnet/repvgg.py): packed weights, workspace and the launch sequence in
// C++, so that a RepVGG model needs no Python at run time (bin/xvb-extract).  Same kernels, same C entry points, same
// arguments and the same order as the Python driver it replaces (RepVGGExtractor in
// asv_subtools_b200/model/repvgg_xvector.py, kept as XVB_REPVGG_NATIVE=0), so the embeddings are bit-identical to it:
//
//   stage0 on the head conv (scale 1, shift = bias, ReLU) -> per block: the tap-list conv with the same epilogue (the
//   last block fp32 only) -> statistics pooling (planes out) -> segment layers.
//
// Records arrive folded by the Python side (fold_block, see xvb200.h); this file prunes the all-zero taps with the
// rule of kept_taps and packs.  No residual path, so two ping-pong plane buffers carry the whole stack.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "records.cuh"

namespace {

using namespace xvb;

// One B*T*F position budget per extract call: larger calls run as consecutive groups of utterances (see xvb200.h).
constexpr long long kPositionBudget = 256LL * 200 * 80;
// the configuration block of a model file is the config struct, 16 int32s and the f32 pooling eps
static_assert(sizeof(xvb_repvgg_config_t) == 16 * sizeof(int32_t) + sizeof(float), "the XVBV0001 configuration block");
const RecordFormat kFile = {"XVBV0001", sizeof(xvb_repvgg_config_t), 3, 4096};

struct Block {   // one folded block on the tap-list conv: relu(conv(x) * 1 + bias)
  int stride = 1, cin = 0, cout = 0;
  std::vector<int> taps;
  Planes w;
  float* bias = nullptr;
};

struct Model {
  xvb_repvgg_config_t cfg{};
  RecordStore recs{kFile.nshape};
  float* head_w = nullptr; float* head_b = nullptr;
  float* ones = nullptr;   // the epilogue scale of every conv, widest stage's length
  std::vector<Block> blocks;
  SegTail tail;
  int F4 = 0, C4 = 0;
  Weights dev{"xvb_repvgg_finalize"};
};

// kept_taps: taps whose (Cout, Cin) slab is not all zero, else the centre tap
std::vector<int> kept_taps(const float* w, int Cout, int Cin, int k) {
  const int kk = k * k;
  std::vector<int> taps;
  for (int j = 0; j < kk; ++j) {
    bool nz = false;
    for (size_t r = 0; r < (size_t)Cout * Cin && !nz; ++r) nz = w[r * kk + j] != 0.f;
    if (nz) taps.push_back(j);
  }
  if (taps.empty()) taps.push_back(kk / 2);
  return taps;
}

}  // namespace

struct xvb_repvgg : Handle<Model> {
  enum { kX0, kX1, kLast, kPooled, kPooledF32, kSegMid, kSegOut, kBufs };
  Workspace<kBufs> ws;
};

namespace {

using H = xvb_repvgg;

int reserve(H* h, int B, int T) {
  const Model* m = h->m.get();
  long long t = T, f = m->cfg.feat_dim;
  size_t mx = (size_t)B * t * f * m->cfg.widths[0];
  for (const Block& b : m->blocks) {
    t = (t - 1) / b.stride + 1;
    f = (f - 1) / b.stride + 1;
    const size_t n = (size_t)B * t * f * b.cout;
    if (n > mx) mx = n;
  }
  size_t need[H::kBufs] = {0};
  need[H::kX0] = need[H::kX1] = mx;
  need[H::kLast] = (size_t)B * t * f * m->C4;
  need[H::kPooled] = need[H::kPooledF32] = (size_t)B * 2 * m->F4 * m->C4;
  need[H::kSegMid] = (size_t)B * (m->tail.mid ? m->tail.mid : 8);
  need[H::kSegOut] = (size_t)B * m->tail.out_rows();
  const bool planes[H::kBufs] = {true, true, false, true, false, true, false};
  uint64_t grown;
  return h->ws.reserve(need, planes, &grown);
}

// One group of utterances (B * T * F within the budget, or a single utterance): RepVGGExtractor.extract.
int extract_group(H* h, const float* feats, int B, int T, float* emb, void* stream) {
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const Model* m = h->m.get();
  const xvb_repvgg_config_t& c = m->cfg;
  int Tl = T, Fl = c.feat_dim;
  Planes x = h->ws.planes(H::kX0), y = h->ws.planes(H::kX1);
  rc = c.ksize == 3 ? xvb_conv2d_head(feats, B, T, Fl, m->head_w, c.widths[0], m->ones, m->head_b, x.hi, x.lo, nullptr, nullptr,
                                      nullptr, nullptr, stream)
                    : xvb_conv2d_head_k(feats, B, T, Fl, m->head_w, c.widths[0], c.ksize, m->ones, m->head_b, x.hi, x.lo, nullptr,
                                        nullptr, nullptr, nullptr, stream);
  if (rc) return rc;
  float* last = h->ws.f32(H::kLast);
  const int nb = (int)m->blocks.size();
  for (int i = 0; i < nb; ++i) {
    const Block& b = m->blocks[i];
    const bool fin = i + 1 == nb;
    xvb_conv2d_args_t a{};
    a.x_hi = x.hi; a.x_lo = x.lo;
    a.w_hi = b.w.hi; a.w_lo = b.w.lo;
    a.B = B; a.T = Tl; a.F = Fl; a.Cin = b.cin; a.Cout = b.cout; a.ksize = c.ksize; a.stride = b.stride;
    a.scale = m->ones; a.shift = b.bias;
    a.relu = 1;
    if (fin) a.y_f32 = last;
    else { a.y_hi = y.hi; a.y_lo = y.lo; }
    if ((rc = xvb_conv2d_taps(&a, b.taps.data(), (int)b.taps.size(), stream))) return rc;
    Tl = (Tl - 1) / b.stride + 1;
    Fl = (Fl - 1) / b.stride + 1;
    const Planes t = x; x = y; y = t;
  }
  return m->tail.run(last, Fl * m->C4, B, Tl, c.pooling_eps, h->ws.planes(H::kPooled), h->ws.f32(H::kPooledF32),
                     h->ws.planes(H::kSegMid), h->ws.f32(H::kSegOut), emb, stream);
}

}  // namespace

extern "C" int xvb_conv2d_kept_taps(const float* w, int Cout, int Cin, int k, int* taps, int cap) {
  XVB_CHECK_ARG(w && taps && Cout > 0 && Cin > 0 && k > 0 && k <= 64,
                "xvb_conv2d_kept_taps: bad arguments (Cout %d, Cin %d, k %d)", Cout, Cin, k);
  const std::vector<int> kept = kept_taps(w, Cout, Cin, k);
  XVB_CHECK_ARG(cap >= (int)kept.size(), "xvb_conv2d_kept_taps: %d taps do not fit in %d entries", (int)kept.size(), cap);
  for (size_t i = 0; i < kept.size(); ++i) taps[i] = kept[i];
  return (int)kept.size();
}

extern "C" int xvb_repvgg_create(xvb_repvgg_t** out, const xvb_repvgg_config_t* cfg) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && cfg, "xvb_repvgg_create: null argument");
  const xvb_repvgg_config_t& c = *cfg;
  XVB_CHECK_ARG(c.feat_dim > 0 && c.feat_dim <= 4096, "xvb_repvgg_create: feat_dim %d, need 1..4096", c.feat_dim);
  XVB_CHECK_ARG(c.ksize == 3 || c.ksize == 5, "xvb_repvgg_create: ksize %d, need 3 (RepVGG) or 5 (RepSPK)", c.ksize);
  XVB_CHECK_ARG(isfinite(c.pooling_eps) && c.pooling_eps >= 0.f, "xvb_repvgg_create: pooling_eps must be finite and >= 0");
  XVB_CHECK_ARG(c.strides[0] == 1, "xvb_repvgg_create: strides[0] = %d, stage0 runs on the head conv at stride 1", c.strides[0]);
  for (int i = 0; i < 5; ++i) {
    XVB_CHECK_ARG(c.strides[i] == 1 || c.strides[i] == 2, "xvb_repvgg_create: strides[%d] = %d, need 1 or 2", i, c.strides[i]);
    XVB_CHECK_ARG(c.widths[i] >= 16 && c.widths[i] <= 4096 && c.widths[i] % 16 == 0,
                  "xvb_repvgg_create: widths[%d] = %d, need a multiple of 16 for the 2-D conv kernel", i, c.widths[i]);
  }
  for (int i = 0; i < 4; ++i)
    XVB_CHECK_ARG(c.num_blocks[i] >= 1 && c.num_blocks[i] <= 64, "xvb_repvgg_create: num_blocks[%d] = %d, need 1..64", i,
                  c.num_blocks[i]);
  xvb_repvgg* h = new xvb_repvgg();
  h->draft->cfg = c;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_repvgg_set_layer(xvb_repvgg_t* h, const char* name, int Cout, int Cin, int ksize, const float* w_host,
                                    const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && strlen(name) > 0 && strlen(name) < 127, "xvb_repvgg_set_layer: bad arguments or finalized model");
  XVB_CHECK_ARG(ksize == 1 || ksize == 3 || ksize == 5, "xvb_repvgg_set_layer(%s): bad shape %d x %d x k%d", name, Cout, Cin, ksize);
  const char* fn = "xvb_repvgg_set_layer";
  const int shape[3] = {Cout, Cin, ksize};
  int rc = h->draft->recs.check(fn, name, shape, w_host, scale_host, shift_host);
  if (rc) return rc;
  XVB_CHECK_ARG((flags & ~(XVB_RELU | XVB_BN)) == 0, "xvb_repvgg_set_layer(%s): flags %d", name, flags);
  XVB_CHECK_ARG(!(flags & XVB_BN) || scale_host, "xvb_repvgg_set_layer(%s): XVB_BN without scale/shift", name);
  return h->draft->recs.add(fn, name, shape, w_host, bias_host, scale_host, shift_host, flags);
}

static int build(Model* m, RecordStore& recs) {
  const xvb_repvgg_config_t& c = m->cfg;
  const int k = c.ksize;
  // a folded block: (cout, cin, k) with its bias, no scale / shift, flags XVB_RELU
  auto block = [&](const std::string& n, int cout, int cin, const Rec** out) -> int {
    const int shape[3] = {cout, cin, k};
    int rc = recs.take("xvb_repvgg_finalize", n, shape, out);
    if (rc) return rc;
    const Rec* r = *out;
    XVB_CHECK_ARG(!r->b.empty() && r->s.empty() && r->flags == XVB_RELU,
                  "xvb_repvgg_finalize: block record '%s' needs a bias, no scale / shift and flags XVB_RELU (has flags %d)",
                  n.c_str(), r->flags);
    return XVB_OK;
  };
  int rc;
  const Rec* r;
  int cmax = c.widths[0];
  for (int i = 1; i < 5; ++i) cmax = c.widths[i] > cmax ? c.widths[i] : cmax;
  if ((rc = block("repvgg.stage0", c.widths[0], 1, &r)) || (rc = m->dev.upload(&m->head_w, r->w)) ||
      (rc = m->dev.upload(&m->head_b, r->b)) || (rc = m->dev.upload(&m->ones, std::vector<float>(cmax, 1.f))))
    return rc;
  int inp = c.widths[0], f = c.feat_dim;
  for (int si = 1; si <= 4; ++si) {
    for (int i = 0; i < c.num_blocks[si - 1]; ++i) {
      const std::string n = "repvgg.stage" + std::to_string(si) + "." + std::to_string(i);
      Block b;
      b.stride = i == 0 ? c.strides[si] : 1;
      b.cin = inp;
      b.cout = c.widths[si];
      if ((rc = block(n, b.cout, b.cin, &r))) return rc;
      b.taps = kept_taps(r->w.data(), b.cout, b.cin, k);
      if ((rc = m->dev.pack(&b.w, r->w, b.cout, b.cin, k * k, b.taps.data(), (int)b.taps.size())) ||
          (rc = m->dev.upload(&b.bias, r->b)))
        return rc;
      f = (f - 1) / b.stride + 1;
      m->blocks.push_back(std::move(b));
      inp = c.widths[si];
    }
  }
  m->F4 = f;
  m->C4 = inp;
  // segment level (repvgg_xvector.py:192-206): [fc1 ->] [fc2], as many as the extracted position hands over
  if ((rc = m->tail.build(recs, m->dev, "xvb_repvgg_finalize", 2 * m->F4 * m->C4))) return rc;
  return recs.check_all_used("xvb_repvgg_finalize");
}

extern "C" int xvb_repvgg_finalize(xvb_repvgg_t* h) { return publish_built(h, build, "xvb_repvgg_finalize"); }

extern "C" int xvb_repvgg_feat_dim(const xvb_repvgg_t* h) { return h ? h->m->cfg.feat_dim : XVB_EINVAL; }
extern "C" int xvb_repvgg_embed_dim(const xvb_repvgg_t* h) { return finalized(h) ? h->m->tail.E : XVB_EINVAL; }
extern "C" int xvb_repvgg_last_launches(const xvb_repvgg_t* h) { return h ? h->last_launches : 0; }

extern "C" int xvb_repvgg_extract(xvb_repvgg_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_repvgg_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0 && T > 0, "xvb_repvgg_extract: bad arguments");
  const long before = g_launches;
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->tail.E;
  int rc = for_groups(B, (long long)per_utt, kPositionBudget,
                      [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, emb + i * E, stream); });
  if (rc) return rc;
  h->last_launches = (int)(g_launches - before);
  return XVB_OK;
}

// ---- "XVBV0001" model files: the configuration, then the records as handed over (save_records) ------------------
extern "C" int xvb_repvgg_save(const xvb_repvgg_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_repvgg_save: model not finalized");
  return save_records("xvb_repvgg_save", path, kFile, &h->m->cfg, h->m->recs);
}

extern "C" int xvb_repvgg_load(xvb_repvgg_t** out, const char* path) {
  return load_records(
      "xvb_repvgg_load", path, kFile, (void**)out,
      [](void** h, const void* cfg) { return xvb_repvgg_create((xvb_repvgg_t**)h, (const xvb_repvgg_config_t*)cfg); },
      [](void* h, const char* name, const int* shape, const float* w, const float* b, const float* s, const float* t, int flags) {
        return xvb_repvgg_set_layer((xvb_repvgg_t*)h, name, shape[0], shape[1], shape[2], w, b, s, t, flags);
      },
      [](void* h) { return xvb_repvgg_finalize((xvb_repvgg_t*)h); }, [](void* h) { xvb_repvgg_destroy((xvb_repvgg_t*)h); });
}

extern "C" void xvb_repvgg_destroy(xvb_repvgg_t* h) { delete h; }
