// Whole-model extractor for the CAM++ x-vector (subtools2/egrecho/models/campplus/campplus.py, CamPP.forward :355-359,
// one chunk of CamPPModel.extract_embedding, model.py:73-96): packed weights, workspace and the launch sequence in C++,
// so that a CAM++ model needs no Python at run time (bin/xvb-extract).  Same kernels, same C entry points, same
// arguments and the same order as the Python driver it replaces (CamPPExtractor in
// asv_subtools_b200/model/campplus_xvector.py, kept as XVB_CAMPP_NATIVE=0), so the embeddings are bit-identical to it:
//
//   FCM head: conv1 -> 4 BasicResBlocks (shortcut, conv1, conv2 + residual) -> conv2 -> copy into the time-padded
//   frame matrix -> stride-2 tdnn (im2col view) -> per dense layer: BN1 -> ReLU, linear1 (+ BN2, ReLU), CAM gate,
//   linear_local, y * m into the layer's column slice -> per transit: BN -> ReLU, 1x1 conv (transit3 with
//   out_nonlinear, fp32) -> [mean | unbiased std] -> dense.
//
// Records arrive by state_dict module path after the Python side's folds and permutations (see xvb200.h); this file
// only packs them.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "records.cuh"

namespace {

using namespace xvb;

constexpr long long kFrameBudget = 128LL * 300;   // B * T frames per group of one extract call (see xvb200.h)
constexpr int kMinFrames = 3;
constexpr int kM = 32;                             // FCM m_channels
constexpr int kSegLen = 100;                       // CAMLayer's segment length
constexpr int kBlocks = 3;
constexpr int kLayers[kBlocks] = {12, 24, 16};
constexpr int kDilation[kBlocks] = {1, 2, 2};
constexpr int kResBlocks = 4;                      // layer1.0, layer1.1, layer2.0, layer2.1
// the configuration block of a model file is the config struct, 5 int32s in declaration order
static_assert(sizeof(xvb_campp_config_t) == 5 * sizeof(int32_t), "the XVBP0001 configuration block");
const RecordFormat kFile = {"XVBP0001", sizeof(xvb_campp_config_t), 2, 65536};

struct Conv {   // a bias-free Conv2d with its eval BatchNorm as the epilogue's scale / shift
  Planes w;
  float* scale = nullptr; float* shift = nullptr;
};

struct Dense {   // one CAMDenseTDNNLayer
  float* s1 = nullptr; float* t1 = nullptr;
  Affine lin1, local;
  float* gw1 = nullptr; float* gb1 = nullptr; float* gw2 = nullptr; float* gb2 = nullptr;
};

struct Transit { float* s = nullptr; float* t = nullptr; Affine lin; };

struct ResBlk { int stride = 1; bool has_sc = false; Conv c1, c2, sc; };

struct Model {
  xvb_campp_config_t cfg{};
  RecordStore recs{kFile.nshape};
  float* conv1_w = nullptr; float* conv1_s = nullptr; float* conv1_t = nullptr;
  ResBlk res[kResBlocks];
  Conv conv2;
  Affine tdnn;
  std::vector<Dense> layers[kBlocks];
  Transit transit[kBlocks];
  float* dense_w = nullptr; float* dense_s = nullptr; float* dense_t = nullptr;
  int f8 = 0, bn = 0, widths[kBlocks] = {0}, maxw = 0, c3 = 0;
  Weights dev{"xvb_campp_finalize"};
};

// Feature-axis size after each residual block: layerL.0 strides it by 2 (ceil), layerL.1 keeps it.
int res_freq(int F, int j) {
  for (int i = 0; i <= j; ++i) F = (i % 2 == 0) ? (F + 1) / 2 : F;
  return F;
}

}  // namespace

struct xvb_campp : Handle<Model> {
  enum { kX0, kA0, kO0 = kA0 + kResBlocks, kS0 = kO0 + kResBlocks, kC2 = kS0 + kResBlocks, kPad, kBuf0, kPre = kBuf0 + kBlocks,
         kH, kZ, kPool, kGate, kStats, kLengths, kBufs };
  Workspace<kBufs> ws;
  int pad_B = -1, pad_T = -1;          // the (B, T) layout whose pad frames are zero
};

namespace {

using H = xvb_campp;

int reserve(H* h, int B, int T) {
  const Model* m = h->m.get();
  const size_t b = (size_t)B, t = (size_t)T, t2 = (size_t)(T + 1) / 2, row = (size_t)m->f8 * kM;
  const size_t nseg = (t2 + kSegLen - 1) / kSegLen;
  size_t need[H::kBufs] = {0};
  need[H::kX0] = b * t * m->cfg.feat_dim * kM;
  for (int j = 0; j < kResBlocks; ++j) {
    const size_t n = b * t * res_freq(m->cfg.feat_dim, j) * kM;
    need[H::kA0 + j] = need[H::kO0 + j] = n;
    need[H::kS0 + j] = m->res[j].has_sc ? n : 0;
  }
  need[H::kC2] = b * t * row;
  need[H::kPad] = b * (t + 4) * row;
  for (int i = 0; i < kBlocks; ++i) need[H::kBuf0 + i] = b * t2 * m->widths[i];
  need[H::kPre] = b * t2 * m->maxw;
  need[H::kH] = b * t2 * m->bn;
  need[H::kZ] = b * t2 * m->cfg.growth_rate;
  need[H::kPool] = b * t2 * m->c3;
  need[H::kGate] = b * nseg * m->cfg.growth_rate;
  need[H::kStats] = b * 2 * m->c3;
  need[H::kLengths] = 0;   // sized by xvb_campp_extract_lengths for the whole call, before its groups run
  bool planes[H::kBufs];
  for (int i = 0; i < H::kBufs; ++i) planes[i] = i != H::kPool && i != H::kGate && i != H::kStats && i != H::kLengths;
  uint64_t grown;
  const int rc = h->ws.reserve(need, planes, &grown);
  if (grown >> H::kPad & 1) h->pad_B = h->pad_T = -1;
  return rc;
}

Planes offset(Planes p, size_t n) { return {p.hi + n, p.lo + n}; }

// ops.PackedAffine.run: x planes (B, T, l.Cin) with row pitch ldx -> y planes (pitch ldy) or yf (pitch ldyf); a nonzero
// x_batch_stride makes x an im2col view (xvb_tdnn_args_t); lens: NULL, or a masked batch's output lengths
int lin(const Affine& l, Planes x, int64_t ldx, int B, int T, const Planes* y, int64_t ldy, float* yf, int64_t ldyf,
        int64_t x_batch_stride, const int* lens, void* stream) {
  xvb_tdnn_args_t a = affine_args(l, x, ldx, B, T);
  if (y) { a.y_hi = y->hi; a.y_lo = y->lo; a.ldy = ldy; }
  a.y_f32 = yf; a.ldyf = ldyf;
  a.x_batch_stride = x_batch_stride;
  a.lengths = lens;
  return xvb_tdnn_affine_ex(&a, stream);
}

// ops.conv2d: x (B, T, F, 32) planes -> y (B, T, F', 32) with F' = ceil(F / stride); stride_t 0 or 1 as the driver passes it
// (the time axis is never strided, so a masked batch's lens are the input's and the output's frame counts)
int conv(const Conv& c, Planes x, int B, int T, int F, int ksize, int stride, int stride_t, const Planes* res, bool relu, Planes y,
         const int* lens, void* stream) {
  xvb_conv2d_args_t a{};
  a.lengths = lens;
  a.x_hi = x.hi; a.x_lo = x.lo;
  a.w_hi = c.w.hi; a.w_lo = c.w.lo;
  a.B = B; a.T = T; a.F = F; a.Cin = kM; a.Cout = kM; a.ksize = ksize; a.stride = stride; a.stride_t = stride_t;
  a.scale = c.scale; a.shift = c.shift;
  if (res) { a.res_hi = res->hi; a.res_lo = res->lo; }
  a.relu = relu ? 1 : 0;
  a.y_hi = y.hi; a.y_lo = y.lo;
  return xvb_conv2d(&a, stream);
}

// One group of utterances: CamPPExtractor.extract.  *n counts the launches as the driver does.  A masked group passes
// lens, its frame counts in row 0 of the workspace's (2, ld) table and their ceil(L / 2) after the stride-2 tdnn in row 1;
// NULL otherwise.  Every tensor of a masked group then holds exact zeros past each utterance's length at its own time
// resolution, except `pre`, whose only consumers are 1x1 layers that store zeros there themselves.
int extract_group(H* h, const float* feats, int B, int T, const int* lens, int ld, float* emb, int* n, void* stream) {
  int rc = reserve(h, B, T);
  if (rc) return rc;
  const Model* m = h->m.get();
  const xvb_campp_config_t& c = m->cfg;
  const int g = c.growth_rate, T2 = (T + 1) / 2, row = m->f8 * kM;
  const long long rows = (long long)B * T2;
  // the time-padded copy of the head output: 2 zero frames before and after every utterance.  The copy below writes
  // only the T middle frames, so the pad frames of a layout stay zero until another layout's copy lands on them.
  const Planes pad = h->ws.planes(H::kPad);
  if (h->pad_B != B || h->pad_T != T) {
    const size_t pitch = (size_t)(T + 4) * row * sizeof(uint16_t), width = (size_t)2 * row * sizeof(uint16_t);
    for (uint16_t* p : {pad.hi, pad.lo}) {
      XVB_CUDA(cudaMemset2DAsync(p, pitch, 0, width, B, (cudaStream_t)stream));
      XVB_CUDA(cudaMemset2DAsync(p + (size_t)(T + 2) * row, pitch, 0, width, B, (cudaStream_t)stream));
    }
    h->pad_B = B; h->pad_T = T;
  }
  const int* lens2 = lens ? lens + ld : nullptr;   // after the stride-2 tdnn
  Planes x = h->ws.planes(H::kX0);
  rc = lens ? xvb_conv2d_head_lengths(feats, B, T, c.feat_dim, lens, m->conv1_w, kM, m->conv1_s, m->conv1_t, x.hi, x.lo, nullptr,
                                      nullptr, nullptr, nullptr, stream)
            : xvb_conv2d_head(feats, B, T, c.feat_dim, m->conv1_w, kM, m->conv1_s, m->conv1_t, x.hi, x.lo, nullptr, nullptr,
                              nullptr, nullptr, stream);
  if (rc) return rc;
  *n += 1;
  int F = c.feat_dim;
  for (int j = 0; j < kResBlocks; ++j) {
    const ResBlk& r = m->res[j];
    const int Fo = res_freq(c.feat_dim, j);
    Planes res = x;
    if (r.has_sc) {
      res = h->ws.planes(H::kS0 + j);
      if ((rc = conv(r.sc, x, B, T, F, 1, r.stride, 1, nullptr, false, res, lens, stream))) return rc;
      *n += 1;
    }
    const Planes a = h->ws.planes(H::kA0 + j), o = h->ws.planes(H::kO0 + j);
    if ((rc = conv(r.c1, x, B, T, F, 3, r.stride, 1, nullptr, true, a, lens, stream)) ||
        (rc = conv(r.c2, a, B, T, Fo, 3, 1, 0, &res, true, o, lens, stream)))
      return rc;
    *n += 2;
    x = o;
    F = Fo;
  }
  const Planes c2 = h->ws.planes(H::kC2);
  if ((rc = conv(m->conv2, x, B, T, F, 3, 2, 1, nullptr, true, c2, lens, stream))) return rc;
  // the head output into the time-padded copy: one row of T * F'' * C elements per utterance
  const int64_t tb = (int64_t)T * row * sizeof(uint16_t), pb = (int64_t)(T + 4) * row * sizeof(uint16_t);
  if ((rc = xvb_copy_rows(c2.hi, tb, pad.hi + 2 * row, pb, B, tb, stream)) ||
      (rc = xvb_copy_rows(c2.lo, tb, pad.lo + 2 * row, pb, B, tb, stream)))
    return rc;
  *n += 4;   // conv2 and the copy, counted as CamPPExtractor counts them
  // tdnn: Conv1d(k = 5, stride 2, padding 2) as a 1-tap layer over 5-frame windows that start every 2 frames
  Planes bufs[kBlocks];
  for (int i = 0; i < kBlocks; ++i) bufs[i] = h->ws.planes(H::kBuf0 + i);
  if ((rc = lin(m->tdnn, pad, 2 * row, B, T2, &bufs[0], m->widths[0], nullptr, 0, (int64_t)(T + 4) * row, lens2, stream)))
    return rc;
  *n += 1;
  const Planes pre = h->ws.planes(H::kPre), hh = h->ws.planes(H::kH), z = h->ws.planes(H::kZ);
  float* gate = h->ws.f32(H::kGate);
  int c0 = m->tdnn.Cout;
  float* stats = h->ws.f32(H::kStats);
  for (int bi = 0; bi < kBlocks; ++bi) {
    const Planes buf = bufs[bi];
    const int width = m->widths[bi];
    for (int li = 0; li < kLayers[bi]; ++li) {
      const Dense& L = m->layers[bi][li];
      const int cin = c0 + li * g;
      Planes out = offset(buf, cin);
      if ((rc = xvb_bn_relu_planes(buf.hi, buf.lo, width, rows, cin, L.s1, L.t1, pre.hi, pre.lo, m->maxw, stream)) ||
          (rc = lin(L.lin1, pre, m->maxw, B, T2, &hh, m->bn, nullptr, 0, 0, lens2, stream)) ||
          (rc = lens2 ? xvb_cam_gate_lengths(hh.hi, hh.lo, m->bn, B, T2, m->bn, kSegLen, L.gw1, L.gb1, m->bn / 2, L.gw2, L.gb2, g,
                                             lens2, gate, stream)
                      : xvb_cam_gate(hh.hi, hh.lo, m->bn, B, T2, m->bn, kSegLen, L.gw1, L.gb1, m->bn / 2, L.gw2, L.gb2, g, gate,
                                     stream)) ||
          (rc = lin(L.local, hh, m->bn, B, T2, &z, g, nullptr, 0, 0, lens2, stream)) ||
          (rc = xvb_seg_gate_apply(z.hi, z.lo, g, nullptr, nullptr, 0, gate, kSegLen, out.hi, out.lo, width, B, T2, g, stream)))
        return rc;
      *n += 5;
    }
    const Transit& tr = m->transit[bi];
    if ((rc = xvb_bn_relu_planes(buf.hi, buf.lo, width, rows, width, tr.s, tr.t, pre.hi, pre.lo, m->maxw, stream))) return rc;
    *n += 1;
    if (bi + 1 < kBlocks) {
      if ((rc = lin(tr.lin, pre, m->maxw, B, T2, &bufs[bi + 1], m->widths[bi + 1], nullptr, 0, 0, lens2, stream))) return rc;
      *n += 1;
      c0 = tr.lin.Cout;
    } else {
      // out_nonlinear in the epilogue, then [mean | unbiased std] over T' (no eps) per utterance
      float* pool = h->ws.f32(H::kPool);
      if ((rc = lin(tr.lin, pre, m->maxw, B, T2, nullptr, 0, pool, m->c3, 0, lens2, stream)) ||
          (rc = lens2 ? xvb_stats_pool_lengths(pool, m->c3, B, T2, m->c3, 0.0f, 1, lens2, stats, nullptr, nullptr, 2 * m->c3, stream)
                      : xvb_stats_pool_ex(pool, m->c3, B, T2, m->c3, 0.0f, 1, stats, nullptr, nullptr, 2 * m->c3, stream)))
        return rc;
      *n += 2;
    }
  }
  if ((rc = xvb_small_affine(stats, 2 * m->c3, m->dense_w, B, 2 * m->c3, c.embd_dim, nullptr, m->dense_s, m->dense_t, XVB_BN, emb,
                             c.embd_dim, nullptr, nullptr, 0, stream)))
    return rc;
  *n += 1;
  return XVB_OK;
}

}  // namespace

extern "C" int xvb_campp_create(xvb_campp_t** out, const xvb_campp_config_t* cfg) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && cfg, "xvb_campp_create: null argument");
  const xvb_campp_config_t& c = *cfg;
  XVB_CHECK_ARG(c.feat_dim >= 8 && c.feat_dim <= 4096 && c.feat_dim % 8 == 0,
                "xvb_campp_create: feat_dim %d must be a multiple of 8 in [8, 4096]", c.feat_dim);
  XVB_CHECK_ARG(c.growth_rate > 0 && c.growth_rate % 8 == 0 && c.growth_rate <= 1024 && c.bn_size >= 1 &&
                    c.bn_size * c.growth_rate <= 2048,
                "xvb_campp_create: growth_rate %d (a multiple of 8), bn_size %d (bn_size * growth_rate <= 2048)", c.growth_rate,
                c.bn_size);
  XVB_CHECK_ARG(c.init_channels > 0 && c.init_channels % 8 == 0 && c.init_channels <= 8192 && c.embd_dim > 0 && c.embd_dim <= 8192,
                "xvb_campp_create: init_channels %d (a multiple of 8), embd_dim %d", c.init_channels, c.embd_dim);
  int ch = c.init_channels;
  for (int i = 0; i < kBlocks; ++i) {
    ch += kLayers[i] * c.growth_rate;
    XVB_CHECK_ARG(i == kBlocks - 1 || (ch / 2) % 8 == 0, "xvb_campp_create: transit%d gives %d channels, not a multiple of 8",
                  i + 1, ch / 2);
    ch /= 2;
  }
  xvb_campp* h = new xvb_campp();
  h->draft->cfg = c;
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_campp_set_layer(xvb_campp_t* h, const char* name, int rows, int cols, const float* w_host,
                                   const float* bias_host, const float* scale_host, const float* shift_host, int flags) {
  XVB_CHECK_ARG(is_draft(h) && name && strlen(name) > 0 && strlen(name) < 127,
                "xvb_campp_set_layer: bad arguments or finalized model");
  const char* fn = "xvb_campp_set_layer";
  const int shape[2] = {rows, cols};
  int rc = h->draft->recs.check(fn, name, shape, w_host, scale_host, shift_host);
  if (rc) return rc;
  XVB_CHECK_ARG((flags & ~(XVB_RELU | XVB_BN)) == 0, "xvb_campp_set_layer(%s): flags %d", name, flags);
  return h->draft->recs.add(fn, name, shape, w_host, bias_host, scale_host, shift_host, flags);
}

static int build(Model* m, RecordStore& recs) {
  const xvb_campp_config_t& c = m->cfg;
  const int g = c.growth_rate;
  m->f8 = c.feat_dim / 8;
  m->bn = c.bn_size * g;
  // a record with its shape, whether it carries a bias and scale / shift, and its flags
  auto need = [&](const std::string& n, int rows, int cols, bool bias, bool bn, int flags, const Rec** out) -> int {
    const int shape[2] = {rows, cols};
    int rc = recs.take("xvb_campp_finalize", n, shape, out);
    if (rc) return rc;
    const Rec* r = *out;
    XVB_CHECK_ARG(r->b.empty() != bias && r->s.empty() != bn && r->flags == flags,
                  "xvb_campp_finalize: record '%s' needs %s bias, %s scale / shift and flags %d (has flags %d)", n.c_str(),
                  bias ? "a" : "no", bn ? "a" : "no", flags, r->flags);
    return XVB_OK;
  };
  auto conv = [&](const std::string& n, int cin, int ksize, int flags, Conv* cv) -> int {
    const Rec* r;
    int rc = need(n, kM, cin * ksize * ksize, false, true, flags, &r);
    if (rc) return rc;
    if ((rc = m->dev.pack(&cv->w, r->w, kM, cin, ksize * ksize, kTaps, ksize * ksize)) || (rc = m->dev.upload(&cv->scale, r->s)) ||
        (rc = m->dev.upload(&cv->shift, r->t)))
      return rc;
    return XVB_OK;
  };
  auto linear = [&](const std::string& n, int cout, int cin, bool bias, int flags, Affine* l) -> int {
    const Rec* r;
    int rc = need(n, cout, cin, bias, false, flags, &r);
    return rc ? rc : pack_affine(m->dev, l, r->w, cout, cin, kTaps, 1, r->b, r->s, r->t, flags);
  };
  auto norm = [&](const std::string& n, int C, float** s, float** t) -> int {
    const Rec* r;
    int rc = need(n, C, 0, false, true, XVB_BN | XVB_RELU, &r);
    if (rc) return rc;
    if ((rc = m->dev.upload(s, r->s)) || (rc = m->dev.upload(t, r->t))) return rc;
    return XVB_OK;
  };
  auto plain = [&](const std::string& n, int rows, int cols, float** w, float** b) -> int {
    const Rec* r;
    int rc = need(n, rows, cols, true, false, 0, &r);
    if (rc) return rc;
    if ((rc = m->dev.upload(w, r->w)) || (rc = m->dev.upload(b, r->b))) return rc;
    return XVB_OK;
  };
  int rc;
  const Rec* r;
  if ((rc = need("head.conv1", kM, 9, false, true, XVB_BN | XVB_RELU, &r)) || (rc = m->dev.upload(&m->conv1_w, r->w)) ||
      (rc = m->dev.upload(&m->conv1_s, r->s)) || (rc = m->dev.upload(&m->conv1_t, r->t)))
    return rc;
  for (int j = 0; j < kResBlocks; ++j) {
    ResBlk& b = m->res[j];
    const std::string p = "head.layer" + std::to_string(j / 2 + 1) + "." + std::to_string(j % 2) + ".";
    b.stride = j % 2 == 0 ? 2 : 1;
    b.has_sc = b.stride != 1;
    if ((rc = conv(p + "conv1", kM, 3, XVB_BN | XVB_RELU, &b.c1)) || (rc = conv(p + "conv2", kM, 3, XVB_BN | XVB_RELU, &b.c2)))
      return rc;
    if (b.has_sc && (rc = conv(p + "shortcut.0", kM, 1, XVB_BN, &b.sc))) return rc;
  }
  if ((rc = conv("head.conv2", kM, 3, XVB_BN | XVB_RELU, &m->conv2)) != XVB_OK) return rc;
  int ch = c.init_channels;
  if ((rc = linear("xvector.tdnn.linear", ch, 5 * m->f8 * kM, true, XVB_RELU, &m->tdnn)) != XVB_OK) return rc;
  for (int bi = 0; bi < kBlocks; ++bi) {
    const std::string p = "xvector.block" + std::to_string(bi + 1) + ".tdnnd";
    const int d = kDilation[bi];
    for (int li = 0; li < kLayers[bi]; ++li) {
      const std::string q = p + std::to_string(li + 1) + ".";
      const int cin = ch + li * g;
      Dense L;
      if ((rc = norm(q + "nonlinear1", cin, &L.s1, &L.t1)) || (rc = linear(q + "linear1", m->bn, cin, true, XVB_RELU, &L.lin1)))
        return rc;
      // linear_local: the dilated k = 3 kernel packed over its whole span, the gap taps as zeros (as ops.PackedAffine
      // packs it)
      const std::string ln = q + "cam_layer.linear_local";
      if ((rc = need(ln, g, m->bn * 3, false, false, 0, &r))) return rc;
      const int span = 2 * d + 1;
      std::vector<float> full((size_t)g * m->bn * span, 0.f);
      for (size_t oc = 0; oc < (size_t)g * m->bn; ++oc)
        for (int k = 0; k < 3; ++k) full[oc * span + k * d] = r->w[oc * 3 + k];
      const int ctx[3] = {-d, 0, d};
      if ((rc = pack_affine(m->dev, &L.local, full, g, m->bn, ctx, 3, r->b, r->s, r->t, 0))) return rc;
      if ((rc = plain(q + "cam_layer.linear1", m->bn / 2, m->bn, &L.gw1, &L.gb1)) ||
          (rc = plain(q + "cam_layer.linear2", g, m->bn / 2, &L.gw2, &L.gb2)))
        return rc;
      m->layers[bi].push_back(std::move(L));
    }
    ch += kLayers[bi] * g;
    m->widths[bi] = ch;
    m->maxw = ch > m->maxw ? ch : m->maxw;
    const std::string t = "xvector.transit" + std::to_string(bi + 1) + ".";
    Transit& tr = m->transit[bi];
    const bool last = bi + 1 == kBlocks;
    if ((rc = norm(t + "nonlinear", ch, &tr.s, &tr.t)) ||
        (rc = linear(t + "linear", ch / 2, ch, last, last ? XVB_RELU : 0, &tr.lin)))
      return rc;
    ch /= 2;
  }
  m->c3 = ch;
  if ((rc = need("xvector.dense.linear", c.embd_dim, 2 * ch, false, true, XVB_BN, &r)) || (rc = m->dev.upload(&m->dense_w, r->w)) ||
      (rc = m->dev.upload(&m->dense_s, r->s)) || (rc = m->dev.upload(&m->dense_t, r->t)))
    return rc;
  return recs.check_all_used("xvb_campp_finalize");
}

extern "C" int xvb_campp_finalize(xvb_campp_t* h) { return publish_built(h, build, "xvb_campp_finalize"); }

extern "C" int xvb_campp_feat_dim(const xvb_campp_t* h) { return h ? h->m->cfg.feat_dim : XVB_EINVAL; }
extern "C" int xvb_campp_embed_dim(const xvb_campp_t* h) { return h ? h->m->cfg.embd_dim : XVB_EINVAL; }
extern "C" int xvb_campp_last_launches(const xvb_campp_t* h) { return h ? h->last_launches : 0; }

extern "C" int xvb_campp_extract(xvb_campp_t* h, const float* feats, int B, int T, float* emb, void* stream) {
  XVB_CHECK_ARG(finalized(h), "xvb_campp_extract: model not finalized");
  XVB_CHECK_ARG(feats && emb && B > 0, "xvb_campp_extract: bad arguments");
  XVB_CHECK_ARG(T >= kMinFrames, "xvb_campp_extract: CAM++ needs at least %d frames per chunk, got %d", kMinFrames, T);
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->cfg.embd_dim;
  int n = 0;
  int rc = for_groups(B, T, kFrameBudget,
                      [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, nullptr, 0, emb + i * E, &n, stream); });
  if (rc) return rc;
  h->last_launches = n;
  return XVB_OK;
}

extern "C" int xvb_campp_extract_lengths(xvb_campp_t* h, const float* feats, const int32_t* lengths_host, int B, int T, float* emb,
                                         void* stream) {
  const char* fn = "xvb_campp_extract_lengths";
  XVB_CHECK_ARG(finalized(h), "%s: model not finalized", fn);
  XVB_CHECK_ARG(feats && lengths_host && emb && B > 0 && T > 0, "%s: bad arguments", fn);
  bool all_T;
  int rc = check_lengths(fn, lengths_host, B, T, &all_T, kMinFrames);
  if (rc) return rc;
  if (all_T) return xvb_campp_extract(h, feats, B, T, emb, stream);   // nothing to mask: the unmasked call itself
  // row 0: L at the head's resolution; row 1: L' = ceil(L / 2), the output length of the stride-2 tdnn (k = 5, pad 2)
  std::vector<int32_t> table((size_t)2 * B);
  for (int b = 0; b < B; ++b) {
    table[b] = lengths_host[b];
    table[(size_t)B + b] = (lengths_host[b] + 1) / 2;
  }
  size_t need[H::kBufs] = {0};
  bool planes[H::kBufs] = {false};
  need[H::kLengths] = table.size();
  uint64_t grown;
  if ((rc = h->ws.reserve(need, planes, &grown))) return rc;
  int* lens = h->ws.i32(H::kLengths);
  // stream-ordered: the previous call's kernels on `stream` have read the old table before this one lands
  XVB_CUDA(cudaMemcpyAsync(lens, table.data(), table.size() * sizeof(int32_t), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  const size_t per_utt = (size_t)T * h->m->cfg.feat_dim, E = (size_t)h->m->cfg.embd_dim;
  int n = 0;
  rc = for_groups(B, T, kFrameBudget,
                  [&](int i, int b) { return extract_group(h, feats + i * per_utt, b, T, lens + i, B, emb + i * E, &n, stream); });
  if (rc) return rc;
  h->last_launches = n;
  return XVB_OK;
}

extern "C" int xvb_campp_chunk_sizes(int T, int max_chunk, int* sizes, int cap) {
  XVB_CHECK_ARG(T >= 1 && max_chunk >= 1, "xvb_campp_chunk_sizes: T %d and max_chunk %d must be >= 1", T, max_chunk);
  // XvectorMixin.split_chunks(even=False): max_chunk-long chunks and a shorter last one, then the last two re-split
  // evenly, the first of them taking the odd frame
  const int num = T / max_chunk + (T % max_chunk ? 1 : 0);
  XVB_CHECK_ARG(sizes && cap >= num, "xvb_campp_chunk_sizes: %d chunks do not fit in %d entries", num, cap);
  for (int i = 0; i + 1 < num; ++i) sizes[i] = max_chunk;
  sizes[num - 1] = T - max_chunk * (num - 1);
  if (num > 1) {
    const int two = sizes[num - 2] + sizes[num - 1];
    sizes[num - 2] = two - two / 2;
    sizes[num - 1] = two / 2;
  }
  return num;
}

// ---- "XVBP0001" model files: the configuration, then the records as handed over (save_records) ------------------
extern "C" int xvb_campp_save(const xvb_campp_t* h, const char* path) {
  XVB_CHECK_ARG(finalized(h) && path, "xvb_campp_save: model not finalized");
  return save_records("xvb_campp_save", path, kFile, &h->m->cfg, h->m->recs);
}

extern "C" int xvb_campp_load(xvb_campp_t** out, const char* path) {
  return load_records(
      "xvb_campp_load", path, kFile, (void**)out,
      [](void** h, const void* cfg) { return xvb_campp_create((xvb_campp_t**)h, (const xvb_campp_config_t*)cfg); },
      [](void* h, const char* name, const int* shape, const float* w, const float* b, const float* s, const float* t, int flags) {
        return xvb_campp_set_layer((xvb_campp_t*)h, name, shape[0], shape[1], w, b, s, t, flags);
      },
      [](void* h) { return xvb_campp_finalize((xvb_campp_t*)h); }, [](void* h) { xvb_campp_destroy((xvb_campp_t*)h); });
}

extern "C" void xvb_campp_destroy(xvb_campp_t* h) { delete h; }
