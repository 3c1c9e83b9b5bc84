// Whole-model extractor for the Conformer x-vector (pytorch/model/transformer_xvector.py, TransformerXvector
// .extract_embedding :321-346 over pytorch/libs/nnet/transformer/, 4x or 2x subsampling): packed weights, handed-over
// tables, workspace and the launch sequence in C++, so that a Conformer model needs no Python at run time
// (bin/xvb-extract, the role of the reference's runtime/).  Same kernels, same C entry points, same arguments and the
// same order as the Python driver it replaces (ConformerExtractor in asv_subtools_b200/model/transformer_xvector.py,
// kept as XVB_CONFORMER_NATIVE=0), so the embeddings are bit-identical to it:
//
//   subsampling head conv -> valid conv -> Linear (x xscale) -> [+ pe] norm_ff_macaron -> per block: macaron FFN,
//   norm_mha, Q/K/V, attention, linear_out, norm_conv, pointwise_conv1, conv module middle, pointwise_conv2, norm_ff,
//   FFN, norm_final + the next norm -> transform_out [+ LayerNorm] -> AttentiveStatsPool -> segment layers.
//
// Records arrive by state_dict module path after the Python side's hand-over transforms (see xvb200.h); this file only
// packs them.  The positional table and the softmax_plus score multipliers are handed over too, so nothing here
// computes a transcendental value the driver takes from torch.
//
// A masked batch (xvb_conformer_extract_lengths) runs the same sequence with each utterance's lengths: the head conv,
// every frame-level linear, the attention and the attentive pooling run masked; the valid conv, the convolution module
// and the LayerNorms need no mask (see extract_group).
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

constexpr long long kFrameBudget = 128LL * 300;   // B * T frames per group of one extract call (see xvb200.h)
constexpr int kTableRows = 5000;                   // PositionalEncoding max_len (embedding.py:41)
constexpr int kMinFrames = 7;
// the configuration block of a model file is the config struct, 17 int32s in declaration order
static_assert(sizeof(xvb_conformer_config_t) == 17 * sizeof(int32_t), "the XVBC0001 configuration block");
const RecordFormat kFile = {"XVBC0001", sizeof(xvb_conformer_config_t), 2, 65536};

struct Ln { float* g = nullptr; float* b = nullptr; };
struct Layer {
  Affine ff_mac1, ff_mac2, ff1, ff2, qkv, out, pw1, pw2;
  float* dw_w = nullptr; float* dw_b = nullptr;
  Ln cm_norm, norm_ff, norm_mha, norm_ff_macaron, norm_conv, norm_final;
  std::vector<float> mult;   // softmax_plus score multiplier per T' (host; passed by value to the kernel)
  float* mult_dev = nullptr;  // the same table on the device, indexed by each utterance's T' in a masked batch
};
struct Seg { Affine lin; bool ln = false; Ln norm; };

struct Model {
  xvb_conformer_config_t cfg{};
  RecordStore recs{kFile.nshape};
  float* head_w = nullptr; float* head_b = nullptr;
  Planes conv2_w;
  float* conv2_scale = nullptr; float* conv2_shift = nullptr;
  Affine embed_out;
  float* table = nullptr;
  std::vector<Layer> layers;
  Ln after_norm;
  Affine transform, att1, att2;
  bool transform_ln = false;
  Ln transform_norm, att_ln, norm_stats;
  std::vector<Seg> seg;
  int E = 0, dk = 0, F2 = 0;
  Weights dev{"xvb_conformer_finalize"};
};

// Subsampled sizes of one chunk of T frames: (T1, F1) after the head conv, (T2, F2) after the valid conv.
void sub_shape(const xvb_conformer_config_t& c, int T, int* T1, int* F1, int* T2, int* F2) {
  *T1 = (T - 1) / 2;
  if (c.subsampling == 4) {
    *F1 = (c.feat_dim - 1) / 2;
    *T2 = (*T1 - 1) / 2;
    *F2 = (*F1 - 1) / 2;
  } else {
    *F1 = c.feat_dim - 2;
    *T2 = *T1 - 2;
    *F2 = *F1 - 2;
  }
}

}  // namespace

struct xvb_conformer : Handle<Model> {
  enum { kX1, kX2, kR, kH, kHid, kDelta, kQkv, kXo, kXp, kA1, kAp, kLogits, kStats, kZ, kZf, kSegY, kSegP, kLengths, kBufs };
  Workspace<kBufs> ws;
};

namespace {

const bool kPlanes[xvb_conformer::kBufs] = {true, true, false, true, true, false, false, false, true, false, true, false,
                                            false, true, false, false, true, false};

int reserve(xvb_conformer* h, int B, int T) {
  const xvb_conformer_config_t& c = h->m->cfg;
  int T1, F1, T2, F2;
  sub_shape(c, T, &T1, &F1, &T2, &F2);
  const size_t b = (size_t)B, D = (size_t)c.D, r2 = b * T2, od = (size_t)c.out_dim;
  const size_t units = (size_t)c.linear_units > D ? (size_t)c.linear_units : D;
  size_t seg = 8;
  for (const Seg& s : h->m->seg) seg = (size_t)s.lin.Cout > seg ? (size_t)s.lin.Cout : seg;
  const size_t need[xvb_conformer::kBufs] = {
      b * T1 * F1 * D, b * T2 * F2 * D, r2 * D, r2 * D, r2 * units, r2 * 2 * D, r2 * 3 * D, r2 * od, r2 * od,
      r2 * c.pool_hidden, r2 * c.pool_hidden, r2 * od, b * 2 * od, b * 2 * od, b * 2 * od, b * seg, b * seg,
      0};   // kLengths: sized by xvb_conformer_extract_lengths for the whole call, before its groups run
  uint64_t grown;
  return h->ws.reserve(need, kPlanes, &grown);
}

// ops.PackedAffine.run: x planes (B, T, l.Cin) with row pitch ldx -> y planes (pitch ldy) and / or yf (pitch ldyf);
// lens: NULL, or a masked batch's frame counts (the rows past them store zeros)
int lin(const Affine& l, Planes x, int64_t ldx, int B, int T, const Planes* y, int64_t ldy, float* yf, int64_t ldyf,
        const int* lens, void* stream) {
  xvb_tdnn_args_t a = affine_args(l, x, ldx, B, T);
  if (y) { a.y_hi = y->hi; a.y_lo = y->lo; a.ldy = ldy; }
  a.y_f32 = yf; a.ldyf = ldyf;
  a.lengths = lens;
  return xvb_tdnn_affine_ex(&a, stream);
}

struct LnCall {   // ops.layer_norm's arguments
  long long rows; int C;
  const float* x; int64_t ldx;
  const float* delta = nullptr; int64_t ld_delta = 0; float delta_scale = 0.f;
  const float* table = nullptr; int table_rows = 0;
  float* x_out = nullptr; int64_t ld_x_out = 0;
  Ln n; bool second = false; Ln n2; int act = XVB_ACT_NONE;
  const Planes* y = nullptr; int64_t ldy = 0;
  float* yf = nullptr; int64_t ldyf = 0;
};

int layer_norm(const LnCall& c, void* stream) {
  xvb_layer_norm_args_t a{};
  a.rows = c.rows; a.C = c.C; a.eps = 1e-5f; a.x = c.x; a.ldx = c.ldx;
  if (c.delta) { a.delta = c.delta; a.ld_delta = c.ld_delta; a.delta_scale = c.delta_scale; }
  if (c.table) { a.table = c.table; a.table_rows = c.table_rows; }
  if (c.x_out) { a.x_out = c.x_out; a.ld_x_out = c.ld_x_out; }
  a.gamma = c.n.g; a.beta = c.n.b;
  if (c.second) { a.second = 1; a.gamma2 = c.n2.g; a.beta2 = c.n2.b; }
  a.act = c.act;
  if (c.y) { a.y_hi = c.y->hi; a.y_lo = c.y->lo; a.ldy = c.ldy; }
  if (c.yf) { a.y_f32 = c.yf; a.ldyf = c.ldyf; }
  return xvb_layer_norm(&a, stream);
}

// One group of utterances: ConformerExtractor.extract.  *n counts the launches as the driver does.  A masked group passes
// lens, its frame counts L in row 0 of the workspace's (2, ld) table and their subsampled lengths L' in row 1; NULL
// otherwise.  Masked, the head conv zeroes its rows t1 >= (L - 1) / 2, and every frame-level linear, the attention and the
// pooling take L'.  Three kernels need no mask: the valid conv's rows t' < L' read only head rows below (L - 1) / 2; the
// convolution module reads pointwise_conv1's exact zeros past L' (GLU(0, 0) = 0), which is the zero padding an
// utterance alone gets; and the LayerNorms work row by row, their rows past L' staying finite and read by nothing that
// crosses frames.  So each row is its utterance extracted alone.
int extract_group(xvb_conformer* h, const float* feats, int B, int T, const int* lens, int ld, float* emb, int* n,
                  void* stream) {
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const Model* m = h->m.get();
  const xvb_conformer_config_t& c = m->cfg;
  const int D = c.D;
  int T1, F1, T2, F2;
  sub_shape(c, T, &T1, &F1, &T2, &F2);
  const long long rows = (long long)B * T2;
  const Planes x1 = h->ws.planes(xvb_conformer::kX1), x2 = h->ws.planes(xvb_conformer::kX2);
  const int* lens2 = lens ? lens + ld : nullptr;   // L', after the subsampling
  if (lens)
    rc = xvb_subsample_head_lengths(feats, B, T, c.feat_dim, lens, m->head_w, m->head_b, D, c.subsampling == 4 ? 2 : 1, x1.hi,
                                    x1.lo, stream);
  else if (c.subsampling == 4)
    rc = xvb_subsample_head(feats, B, T, c.feat_dim, m->head_w, m->head_b, D, x1.hi, x1.lo, stream);
  else
    rc = xvb_subsample_head_stride(feats, B, T, c.feat_dim, m->head_w, m->head_b, D, 1, x1.hi, x1.lo, stream);
  if (rc) return rc;
  {
    xvb_conv2d_args_t a{};
    a.x_hi = x1.hi; a.x_lo = x1.lo;
    a.w_hi = m->conv2_w.hi; a.w_lo = m->conv2_w.lo;
    a.B = B; a.T = T1; a.F = F1; a.Cin = D; a.Cout = D; a.ksize = 3; a.stride = c.subsampling == 4 ? 2 : 1;
    a.scale = m->conv2_scale; a.shift = m->conv2_shift;
    a.relu = 1;
    a.y_hi = x2.hi; a.y_lo = x2.lo;
    if ((rc = xvb_conv2d_valid(&a, stream)) != XVB_OK) return rc;
  }
  float* r = h->ws.f32(xvb_conformer::kR);
  if ((rc = lin(m->embed_out, x2, (int64_t)F2 * D, B, T2, nullptr, 0, r, D, lens2, stream)) != XVB_OK) return rc;
  *n += 3;
  const int units = c.linear_units;
  const int hid_ld = units > D ? units : D;
  const Planes hh = h->ws.planes(xvb_conformer::kH), hid = h->ws.planes(xvb_conformer::kHid);
  float* delta = h->ws.f32(xvb_conformer::kDelta);
  float* qkv = h->ws.f32(xvb_conformer::kQkv);
  float* d1 = delta;   // delta[..., :D], pitch 2D
  const float* rope = c.pos == 2 ? m->table : nullptr;
  const float* absp = c.pos == 1 ? m->table : nullptr;
  auto ffn = [&](const Affine& a, const Affine& b) -> int {
    int e = lin(a, hh, D, B, T2, &hid, hid_ld, nullptr, 0, lens2, stream);
    return e ? e : lin(b, hid, hid_ld, B, T2, nullptr, 0, d1, 2 * D, lens2, stream);
  };
  {
    LnCall l{rows, D, r, D};
    l.table = absp; l.table_rows = T2;
    l.x_out = r; l.ld_x_out = D;
    l.n = m->layers[0].norm_ff_macaron;
    l.y = &hh; l.ldy = D;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    *n += 1;
  }
  const int nl = (int)m->layers.size();
  for (int i = 0; i < nl; ++i) {
    const Layer& L = m->layers[i];
    if ((rc = ffn(L.ff_mac1, L.ff_mac2)) != XVB_OK) return rc;
    LnCall l{rows, D, r, D};
    l.delta = d1; l.ld_delta = 2 * D; l.delta_scale = 0.5f;
    l.x_out = r; l.ld_x_out = D;
    l.n = L.norm_mha;
    l.y = &hh; l.ldy = D;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    if ((rc = lin(L.qkv, hh, D, B, T2, nullptr, 0, qkv, 3 * D, lens2, stream)) != XVB_OK) return rc;
    const int rope_v = c.rotary_value && rope ? 1 : 0;
    if (lens2)
      rc = xvb_rope_attention_lengths(qkv, 3 * D, B, T2, c.H, m->dk, rope, rope_v, lens2, c.softmax_plus ? L.mult_dev : nullptr,
                                      kTableRows, hid.hi, hid.lo, hid_ld, stream);
    else
      rc = xvb_rope_attention(qkv, 3 * D, B, T2, c.H, m->dk, rope, rope_v, c.softmax_plus ? L.mult[T2] : 1.0f, hid.hi, hid.lo,
                              hid_ld, stream);
    if (rc) return rc;
    if ((rc = lin(L.out, hid, hid_ld, B, T2, nullptr, 0, d1, 2 * D, lens2, stream)) != XVB_OK) return rc;
    l.delta_scale = 1.0f;
    l.n = L.norm_conv;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    if ((rc = lin(L.pw1, hh, D, B, T2, nullptr, 0, delta, 2 * D, lens2, stream)) != XVB_OK) return rc;
    if ((rc = xvb_conv_module(delta, 2 * D, B, T2, D, L.dw_w, L.dw_b, c.conv_kernel, L.cm_norm.g, L.cm_norm.b, c.cm_norm,
                              1e-5f, c.act, hid.hi, hid.lo, hid_ld, stream)))
      return rc;
    if ((rc = lin(L.pw2, hid, hid_ld, B, T2, nullptr, 0, d1, 2 * D, lens2, stream)) != XVB_OK) return rc;
    l.n = L.norm_ff;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    if ((rc = ffn(L.ff1, L.ff2)) != XVB_OK) return rc;
    l.delta_scale = 0.5f;
    l.n = L.norm_final;
    l.second = true;
    l.n2 = i + 1 < nl ? m->layers[i + 1].norm_ff_macaron : m->after_norm;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    *n += 16;
  }
  // transform_out (+ its LayerNorm): x fp32 for the pooling sums, planes for the attention conv
  const int od = c.out_dim, hd = c.pool_hidden;
  float* xo = h->ws.f32(xvb_conformer::kXo);
  const Planes xp = h->ws.planes(xvb_conformer::kXp);
  if (!m->transform_ln) {
    if ((rc = lin(m->transform, hh, D, B, T2, &xp, od, xo, od, lens2, stream)) != XVB_OK) return rc;
    *n += 1;
  } else {
    if ((rc = lin(m->transform, hh, D, B, T2, nullptr, 0, xo, od, lens2, stream)) != XVB_OK) return rc;
    LnCall l{rows, od, xo, od};
    l.n = m->transform_norm;
    l.y = &xp; l.ldy = od;
    l.yf = xo; l.ldyf = od;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
    *n += 2;
  }
  // AttentiveStatsPool
  float* a1 = h->ws.f32(xvb_conformer::kA1);
  if ((rc = lin(m->att1, xp, od, B, T2, nullptr, 0, a1, hd, lens2, stream)) != XVB_OK) return rc;
  const Planes ap = h->ws.planes(xvb_conformer::kAp);
  {
    LnCall l{rows, hd, a1, hd};
    l.n = m->att_ln;
    l.act = XVB_ACT_TANH;
    l.y = &ap; l.ldy = hd;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
  }
  float* logits = h->ws.f32(xvb_conformer::kLogits);
  if ((rc = lin(m->att2, ap, hd, B, T2, nullptr, 0, logits, od, lens2, stream)) != XVB_OK) return rc;
  float* stats = h->ws.f32(xvb_conformer::kStats);
  rc = lens2 ? xvb_attn_stats_pool_lengths(logits, od, xo, od, B, T2, od, 1e-5f, lens2, stats, nullptr, nullptr, 2 * od, stream)
             : xvb_attn_stats_pool(logits, od, xo, od, B, T2, od, 1e-5f, stats, nullptr, nullptr, 2 * od, stream);
  if (rc) return rc;
  Planes z = h->ws.planes(xvb_conformer::kZ);
  float* zf = h->ws.f32(xvb_conformer::kZf);
  {
    LnCall l{B, 2 * od, stats, 2 * od};
    l.n = m->norm_stats;
    l.y = &z; l.ldy = 2 * od;
    l.yf = zf; l.ldyf = 2 * od;
    if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
  }
  *n += 5;
  int zc = 2 * od;
  const int ns = (int)m->seg.size();
  for (int j = 0; j < ns; ++j) {
    const Seg& s = m->seg[j];
    const bool last = j + 1 == ns;
    const int co = s.lin.Cout;
    float* y = last ? emb : h->ws.f32(xvb_conformer::kSegY);
    if ((rc = lin(s.lin, z, zc, B, 1, nullptr, 0, y, co, nullptr, stream)) != XVB_OK) return rc;
    *n += 1;
    const Planes yp = h->ws.planes(xvb_conformer::kSegP);
    if (s.ln) {
      LnCall l{B, co, y, co};
      l.n = s.norm;
      if (!last) { l.y = &yp; l.ldy = co; }
      l.yf = y; l.ldyf = co;
      if ((rc = layer_norm(l, stream)) != XVB_OK) return rc;
      *n += 1;
    } else if (!last) {
      if ((rc = xvb_split_f32(y, B, co, co, yp.hi, yp.lo, co, stream)) != XVB_OK) return rc;
      *n += 1;
    }
    z = yp;
    zc = co;
  }
  return XVB_OK;
}

}  // namespace

extern "C" int xvb_conformer_create(xvb_conformer_t** out, const xvb_conformer_config_t* cfg) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && cfg, "xvb_conformer_create: null argument");
  const xvb_conformer_config_t& c = *cfg;
  XVB_CHECK_ARG(c.subsampling == 4 || c.subsampling == 2, "xvb_conformer_create: subsampling must be 4 or 2 (got %d)", c.subsampling);
  XVB_CHECK_ARG(c.feat_dim >= (c.subsampling == 4 ? 7 : 5) && c.feat_dim <= 4096, "xvb_conformer_create: feat_dim %d is out of range",
                c.feat_dim);
  XVB_CHECK_ARG(c.D >= 16 && c.D <= 4096 && c.D % 16 == 0 && c.H > 0 && c.D % c.H == 0 &&
                    (c.D / c.H == 32 || c.D / c.H == 64 || c.D / c.H == 128),
                "xvb_conformer_create: attention_dim %d / heads %d: D %% 16 == 0 and d_k in {32, 64, 128}", c.D, c.H);
  XVB_CHECK_ARG(c.linear_units > 0 && c.linear_units % 8 == 0 && c.linear_units <= 65536 && c.blocks >= 1 && c.blocks <= 256 &&
                    c.conv_kernel > 0 && c.conv_kernel % 2 == 1 && c.conv_kernel <= 255,
                "xvb_conformer_create: linear_units %d (multiple of 8), blocks %d (>= 1), conv kernel %d (odd)", c.linear_units,
                c.blocks, c.conv_kernel);
  XVB_CHECK_ARG(c.pos >= 0 && c.pos <= 2 && (c.rotary_value == 0 || c.rotary_value == 1) && (c.softmax_plus == 0 || c.softmax_plus == 1) &&
                    (c.act == XVB_ACT_SWISH || c.act == XVB_ACT_RELU) && (c.cm_norm == 0 || c.cm_norm == 1),
                "xvb_conformer_create: bad pos / rotary_value / softmax_plus / act / cm_norm");
  XVB_CHECK_ARG(c.out_dim > 0 && c.out_dim % 8 == 0 && c.out_dim <= 4096 && c.out_norm >= 0 && c.out_norm <= 2 && c.pool_hidden > 0 &&
                    c.pool_hidden % 8 == 0 && c.pool_hidden <= 8192 && (c.fc1 == 0 || c.fc1 == 1) && c.position >= 0 && c.position <= 2 &&
                    (c.position != 0 || c.fc1),
                "xvb_conformer_create: bad transform_out / pooling / fc1 / position (far needs fc1)");
  xvb_conformer* h = new xvb_conformer();
  h->draft->cfg = c;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_conformer_set_layer(xvb_conformer_t* h, const char* name, int rows, int cols, const float* w_host,
                                       const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && strlen(name) > 0 && strlen(name) < 127,
                "xvb_conformer_set_layer: bad arguments or finalized model");
  const char* fn = "xvb_conformer_set_layer";
  const int shape[2] = {rows, cols};
  int rc = h->draft->recs.check(fn, name, shape, w_host, scale_host, shift_host);
  if (rc) return rc;
  XVB_CHECK_ARG(!(flags & XVB_BN) || scale_host, "xvb_conformer_set_layer(%s): XVB_BN without scale/shift", name);
  XVB_CHECK_ARG((flags & ~(XVB_RELU | XVB_BN | XVB_SWISH)) == 0, "xvb_conformer_set_layer(%s): flags %d", name, flags);
  return h->draft->recs.add(fn, name, shape, w_host, bias_host, scale_host, shift_host, flags);
}

static int build(Model* m, RecordStore& recs) {
  const xvb_conformer_config_t& c = m->cfg;
  const int D = c.D;
  auto need = [&](const std::string& n, int rows, int cols, const Rec** out) -> int {
    const int shape[2] = {rows, cols};
    return recs.take("xvb_conformer_finalize", n, shape, out);
  };
  // a Linear: weight and bias; the folded BatchNorm / xscale and the activation as flagged
  auto linear = [&](const std::string& n, int cout, int cin, Affine* l) -> int {
    const Rec* r;
    int rc = need(n, cout, cin, &r);
    if (rc) return rc;
    XVB_CHECK_ARG(!r->b.empty(), "xvb_conformer_finalize: record '%s' needs its bias", n.c_str());
    XVB_CHECK_ARG(r->s.empty() || (r->flags & XVB_BN), "xvb_conformer_finalize: record '%s' has scale/shift without XVB_BN", n.c_str());
    return pack_affine(m->dev, l, r->w, cout, cin, kTaps, 1, r->b, r->s, r->t, r->flags);
  };
  auto plain = [&](const std::string& n, int cout, int cin, Affine* l) -> int {
    int rc = linear(n, cout, cin, l);
    if (rc) return rc;
    XVB_CHECK_ARG(l->flags == 0, "xvb_conformer_finalize: record '%s' must be a plain affine (flags %d)", n.c_str(), l->flags);
    return XVB_OK;
  };
  // a LayerNorm: gamma / beta as scale / shift, or neither; `affine` demands them
  auto norm = [&](const std::string& n, int C, bool affine, Ln* l) -> int {
    const Rec* r;
    int rc = need(n, C, 0, &r);
    if (rc) return rc;
    XVB_CHECK_ARG(r->b.empty() && !(r->flags & ~XVB_BN) && (!affine || !r->s.empty()),
                  "xvb_conformer_finalize: record '%s' is not a LayerNorm", n.c_str());
    if ((rc = m->dev.upload(&l->g, r->s)) || (rc = m->dev.upload(&l->b, r->t)) != XVB_OK) return rc;
    return XVB_OK;
  };
  int rc;
  const Rec* r;
  const std::string e = "transformer.embed.";
  int T1_, F1_, T2_;
  sub_shape(c, kMinFrames, &T1_, &F1_, &T2_, &m->F2);   // F'' depends on feat_dim alone
  m->dk = D / c.H;
  if ((rc = need(e + "conv.0", D, 9, &r)) != XVB_OK) return rc;
  XVB_CHECK_ARG(!r->b.empty() && r->s.empty() && r->flags == 0, "xvb_conformer_finalize: record '%sconv.0' needs a bias only", e.c_str());
  if ((rc = m->dev.upload(&m->head_w, r->w)) || (rc = m->dev.upload(&m->head_b, r->b)) != XVB_OK) return rc;
  if ((rc = need(e + "conv.2", D, 9 * D, &r)) != XVB_OK) return rc;
  XVB_CHECK_ARG(!r->b.empty() && r->s.empty() && r->flags == 0, "xvb_conformer_finalize: record '%sconv.2' needs a bias only", e.c_str());
  if ((rc = m->dev.pack(&m->conv2_w, r->w, D, D, 9, kTaps, 9)) || (rc = m->dev.upload(&m->conv2_scale, std::vector<float>(D, 1.f))) ||
      (rc = m->dev.upload(&m->conv2_shift, r->b)))
    return rc;
  if ((rc = linear(e + "out.0", D, m->F2 * D, &m->embed_out)) != XVB_OK) return rc;
  XVB_CHECK_ARG((m->embed_out.flags == XVB_BN) == (c.pos != 0) && (m->embed_out.flags & ~XVB_BN) == 0,
                "xvb_conformer_finalize: record '%sout.0' must carry the xscale (XVB_BN) exactly when there is a positional encoding",
                e.c_str());
  if (c.pos) {
    const int width = c.pos == 2 ? m->dk : D;
    if ((rc = need("pos_table", kTableRows, width, &r)) || (rc = m->dev.upload(&m->table, r->w)) != XVB_OK) return rc;
  }
  const int act_flag = c.act == XVB_ACT_SWISH ? XVB_SWISH : XVB_RELU;
  for (int i = 0; i < c.blocks; ++i) {
    const std::string p = "transformer.encoders." + std::to_string(i) + ".";
    Layer L;
    if ((rc = linear(p + "feed_forward_macaron.w_1", c.linear_units, D, &L.ff_mac1)) ||
        (rc = plain(p + "feed_forward_macaron.w_2", D, c.linear_units, &L.ff_mac2)) ||
        (rc = linear(p + "feed_forward.w_1", c.linear_units, D, &L.ff1)) || (rc = plain(p + "feed_forward.w_2", D, c.linear_units, &L.ff2)) ||
        (rc = plain(p + "self_attn.linear_qkv", 3 * D, D, &L.qkv)) || (rc = plain(p + "self_attn.linear_out", D, D, &L.out)) ||
        (rc = plain(p + "conv_module.pointwise_conv1", 2 * D, D, &L.pw1)) || (rc = plain(p + "conv_module.pointwise_conv2", D, D, &L.pw2)))
      return rc;
    XVB_CHECK_ARG(L.ff_mac1.flags == act_flag && L.ff1.flags == act_flag,
                  "xvb_conformer_finalize: the feed-forward w_1 records of block %d must carry the configured activation", i);
    if ((rc = need(p + "conv_module.depthwise_conv", D, c.conv_kernel, &r)) != XVB_OK) return rc;
    XVB_CHECK_ARG(!r->b.empty(), "xvb_conformer_finalize: record '%sconv_module.depthwise_conv' needs its bias", p.c_str());
    if ((rc = m->dev.upload(&L.dw_w, r->w)) || (rc = m->dev.upload(&L.dw_b, r->b)) != XVB_OK) return rc;
    if ((rc = norm(p + "conv_module.norm", D, true, &L.cm_norm)) != XVB_OK) return rc;
    XVB_CHECK_ARG(((recs.find(p + "conv_module.norm")->flags & XVB_BN) != 0) == (c.cm_norm == 1),
                  "xvb_conformer_finalize: record '%sconv_module.norm' does not match the configured norm", p.c_str());
    if ((rc = norm(p + "norm_ff", D, false, &L.norm_ff)) || (rc = norm(p + "norm_mha", D, false, &L.norm_mha)) ||
        (rc = norm(p + "norm_ff_macaron", D, false, &L.norm_ff_macaron)) || (rc = norm(p + "norm_conv", D, false, &L.norm_conv)) ||
        (rc = norm(p + "norm_final", D, false, &L.norm_final)))
      return rc;
    if (c.softmax_plus) {
      if ((rc = need(p + "self_attn.att_norm", 1, kTableRows, &r)) != XVB_OK) return rc;
      L.mult = r->w;
      if ((rc = m->dev.upload(&L.mult_dev, L.mult)) != XVB_OK) return rc;
    }
    m->layers.push_back(std::move(L));
  }
  if ((rc = norm("transformer.after_norm", D, false, &m->after_norm)) != XVB_OK) return rc;
  const int od = c.out_dim;
  if ((rc = linear("transform_out.affine", od, D, &m->transform)) != XVB_OK) return rc;
  XVB_CHECK_ARG((m->transform.flags & (XVB_RELU | XVB_SWISH)) != (XVB_RELU | XVB_SWISH) &&
                    ((m->transform.flags & XVB_BN) != 0) == (c.out_norm == 1),
                "xvb_conformer_finalize: record 'transform_out.affine' does not match the configured norm");
  m->transform_ln = c.out_norm == 2;
  if (m->transform_ln && (rc = norm("transform_out.batchnorm", od, false, &m->transform_norm))) return rc;
  if ((rc = linear("stats.attention.0", c.pool_hidden, od, &m->att1)) || (rc = norm("stats.attention.2", c.pool_hidden, false, &m->att_ln)) ||
      (rc = plain("stats.attention.4", od, c.pool_hidden, &m->att2)) || (rc = norm("stats.norm_stats", 2 * od, false, &m->norm_stats)))
    return rc;
  XVB_CHECK_ARG(m->att1.flags == XVB_RELU, "xvb_conformer_finalize: record 'stats.attention.0' must carry XVB_RELU only");
  // segment layers (transformer_xvector.py:331-346): far = fc1.affine; otherwise [fc1 whole ->] fc2 whole / fc2.affine
  int cin = 2 * od;
  struct Want { const char* name; bool whole; };
  std::vector<Want> chain;
  if (c.position == 0) chain.push_back({"fc1", false});
  else {
    if (c.fc1) chain.push_back({"fc1", true});
    chain.push_back({"fc2", c.position == 2});
  }
  for (const Want& w : chain) {
    const std::string a = std::string(w.name) + ".affine", b = std::string(w.name) + ".batchnorm";
    const Rec* ra = recs.find(a);
    XVB_CHECK_ARG(ra, "xvb_conformer_finalize: record '%s' is missing", a.c_str());
    Seg s;
    if ((rc = w.whole ? linear(a, ra->shape[0], cin, &s.lin) : plain(a, ra->shape[0], cin, &s.lin)) != XVB_OK) return rc;
    XVB_CHECK_ARG(s.lin.Cout % 8 == 0, "xvb_conformer_finalize: record '%s' has %d rows, need a multiple of 8", a.c_str(), s.lin.Cout);
    s.ln = w.whole && recs.find(b) != nullptr;
    if (s.ln && (rc = norm(b, s.lin.Cout, false, &s.norm))) return rc;
    XVB_CHECK_ARG(!(s.ln && (s.lin.flags & XVB_BN)), "xvb_conformer_finalize: '%s' has both a LayerNorm and a folded BatchNorm", w.name);
    m->seg.push_back(s);
    cin = s.lin.Cout;
  }
  m->E = m->seg.back().lin.Cout;
  return recs.check_all_used("xvb_conformer_finalize");
}

extern "C" int xvb_conformer_finalize(xvb_conformer_t* h) { return publish_built(h, build, "xvb_conformer_finalize"); }

extern "C" int xvb_conformer_feat_dim(const xvb_conformer_t* h) { return h ? h->m->cfg.feat_dim : XVB_EINVAL; }
extern "C" int xvb_conformer_embed_dim(const xvb_conformer_t* h) { return finalized(h) ? h->m->E : XVB_EINVAL; }
extern "C" int xvb_conformer_last_launches(const xvb_conformer_t* h) { return h ? h->last_launches : 0; }

extern "C" int xvb_conformer_extract(xvb_conformer_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_conformer_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0, "xvb_conformer_extract: bad arguments");
  XVB_CHECK_ARG(T >= kMinFrames, "xvb_conformer_extract: the Conformer needs at least %d frames, got %d", kMinFrames, T);
  int T1, F1, T2, F2;
  sub_shape(h->m->cfg, T, &T1, &F1, &T2, &F2);
  XVB_CHECK_ARG(T2 < kTableRows, "xvb_conformer_extract: a chunk of %d subsampled frames exceeds the positional tables' %d", T2,
                kTableRows);
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->E;
  int n = 0;
  int rc = for_groups(B, T, kFrameBudget,
                      [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, nullptr, 0, emb + i * E, &n, stream); });
  if (rc) return rc;
  h->last_launches = n;
  return XVB_OK;
}

extern "C" int xvb_conformer_extract_lengths(xvb_conformer_t* h, const float* feats, const int32_t* lengths_host, int B, int T,
                                             float* emb, void* stream) {
  const char* fn = "xvb_conformer_extract_lengths";
  XVB_CHECK_ARG(finalized(h), "%s: model not finalized", fn);
  XVB_CHECK_ARG(feats && lengths_host && emb && B > 0 && T > 0, "%s: bad arguments", fn);
  bool all_T;
  int rc = check_lengths(fn, lengths_host, B, T, &all_T, kMinFrames);
  if (rc) return rc;
  int T1, F1, T2, F2;
  sub_shape(h->m->cfg, T, &T1, &F1, &T2, &F2);   // the longest utterance's T' bounds every other one
  XVB_CHECK_ARG(T2 < kTableRows, "%s: a chunk of %d subsampled frames exceeds the positional tables' %d", fn, T2, kTableRows);
  if (all_T) return xvb_conformer_extract(h, feats, B, T, emb, stream);   // nothing to mask: the unmasked call itself
  // row 0: L, the head conv's input length; row 1: L', the utterance's length after the subsampling
  std::vector<int32_t> table((size_t)2 * B);
  for (int b = 0; b < B; ++b) {
    table[b] = lengths_host[b];
    sub_shape(h->m->cfg, lengths_host[b], &T1, &F1, &table[(size_t)B + b], &F2);
  }
  size_t need[xvb_conformer::kBufs] = {0};
  uint64_t grown;
  need[xvb_conformer::kLengths] = table.size();
  if ((rc = h->ws.reserve(need, kPlanes, &grown))) return rc;
  int* lens = h->ws.i32(xvb_conformer::kLengths);
  // stream-ordered: the previous call's kernels on `stream` have read the old table before this one lands
  XVB_CUDA(cudaMemcpyAsync(lens, table.data(), table.size() * sizeof(int32_t), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->E;
  int n = 0;
  rc = for_groups(B, T, kFrameBudget,
                  [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, lens + i, B, emb + i * E, &n, stream); });
  if (rc) return rc;
  h->last_launches = n;
  return XVB_OK;
}

// ---- "XVBC0001" model files: the configuration, then the records and tables as handed over (save_records) ---------
extern "C" int xvb_conformer_save(const xvb_conformer_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_conformer_save: model not finalized");
  return save_records("xvb_conformer_save", path, kFile, &h->m->cfg, h->m->recs);
}

extern "C" int xvb_conformer_load(xvb_conformer_t** out, const char* path) {
  return load_records(
      "xvb_conformer_load", path, kFile, (void**)out,
      [](void** h, const void* cfg) { return xvb_conformer_create((xvb_conformer_t**)h, (const xvb_conformer_config_t*)cfg); },
      [](void* h, const char* name, const int* shape, const float* w, const float* b, const float* s, const float* t, int flags) {
        return xvb_conformer_set_layer((xvb_conformer_t*)h, name, shape[0], shape[1], w, b, s, t, flags);
      },
      [](void* h) { return xvb_conformer_finalize((xvb_conformer_t*)h); },
      [](void* h) { xvb_conformer_destroy((xvb_conformer_t*)h); });
}

extern "C" void xvb_conformer_destroy(xvb_conformer_t* h) { delete h; }
