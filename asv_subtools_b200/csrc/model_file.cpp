// Every model-file layout of the native extractors, written and read here without Python -- the role of
// torch::jit::load in the reference's runtime (runtime/extractor/torch_asv_model.cc:8-17).  All are little-endian.
//
// The tap-layer files of the TDNN and ECAPA-TDNN hold the layers exactly as the reference's state_dict stores them
// (conv weights (Cout, Cin, tot_context) incl. masked taps, eval BatchNorm folded to scale/shift), one tap record each:
//
//   tap record : i32 Cout, Cin, ntaps, tot_context, flags, has_bias, has_bn | i32 ctx[ntaps]
//                | f32 w[Cout*Cin*tot_context] | f32 bias[Cout]? | f32 scale[Cout], shift[Cout]?
//
//   "XVBM0001" (TDNN) | i32 feat_dim | f32 pooling_eps | i32 n_frame | i32 n_segment | n_frame + n_segment tap records
//                       (segment layers with ntaps = tot_context = 1 and ctx = {0})
//   "XVBM0002" (TDNN with an attention pooling, xvb_extractor_set_attention_pooling): the XVBM0001 header, then the
//              pooling record i32 kind, pooled, gdiv, unweighted_var, n_attention (AttnPoolRecord) | for the xi-vector
//              kinds f32 prior_logprec[pooled], prior_mean[pooled] | n_frame + n_attention + n_segment tap records
//              (the attention affines, 1 or 2, between the frame and the segment layers).  Written only for such a
//              model, so XVBM0001 files are written as before.
//   "XVBE0001" (ECAPA-TDNN) | i32 feat_dim, channels, mfa_dim, att_hidden, embed_dim, n_layers
//              | per layer: i32 name_len | name (no NUL) | tap record
//   "XVBE0002" (ECAPA-TDNN with MQMHA pooling): the same with the pooling record {num_head, num_q, hidden, share,
//              affine_layers, time_attention, stddev} after the dims; grouped convs stored as the state_dict holds them.
//   "XVBG0001" (egrecho's ECAPA-TDNN, chained blocks): the XVBE0002 header with i32 residual_form (1: chained,
//              xvb_ecapa_set_chained) after the pooling record, then the named tap records.
//   "XVBE0003" (ECAPA-TDNN whose attentive pooling is set by xvb_ecapa_set_attention, e.g. the launcher model of
//              pytorch/model/ecapa-tdnn-xvector.py): the XVBE0001 header with i32 global_context and the f32 variance
//              floor after the dims, then the named tap records.  Written only for an attention other than the default
//              (1, 1e-5), so XVBE0001 / XVBE0002 / XVBG0001 files are written as before.
//
// The named-record files of the native ResNet, RepVGG, Conformer and CAM++ extractors (save_records / load_records
// below) and the record store behind them (records.h).
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <vector>

#include "../../include/xvb200.h"
#include "records.h"

namespace xvb {
void set_error(const char* fmt, ...);
}
using xvb::set_error;

namespace {
bool rd(FILE* f, void* p, size_t n) { return fread(p, 1, n, f) == n; }

#define FAIL_IF(cond, ...) do { if (cond) { set_error(__VA_ARGS__); return XVB_EINVAL; } } while (0)

// weight elements of a record shape; a ksize outside [0, 4096] counts as too large
int64_t weight_elems(const int* shape, int n) {
  const int64_t rc = (int64_t)shape[0] * shape[1];
  if (n == 2) return rc;
  return shape[2] < 0 || shape[2] > 4096 ? INT64_MAX : rc * shape[2] * shape[2];
}

// the bounds every record shape meets, in set_layer and in a model file
bool shape_ok(const int* shape, int n) {
  return shape[0] > 0 && shape[0] <= 65536 && shape[1] >= 0 && shape[1] <= (1 << 20) &&
         weight_elems(shape, n) <= (int64_t)1 << 28;
}

const char* shape_str(const int* shape, int n, char (&buf)[48]) {
  if (n == 2) snprintf(buf, sizeof buf, "%d x %d", shape[0], shape[1]);
  else snprintf(buf, sizeof buf, "%d x %d x k%d", shape[0], shape[1], shape[2]);
  return buf;
}

bool write_tap(FILE* f, const xvb::TapRec& r) {
  const int32_t hd[7] = {r.Cout, r.Cin, r.ntaps, r.tot(), r.flags, !r.b.empty(), !r.s.empty()};
  return fwrite(hd, 4, 7, f) == 7 && fwrite(r.ctx, 4, r.ntaps, f) == (size_t)r.ntaps &&
         fwrite(r.w.data(), 4, r.w.size(), f) == r.w.size() && fwrite(r.b.data(), 4, r.b.size(), f) == r.b.size() &&
         fwrite(r.s.data(), 4, r.s.size(), f) == r.s.size() && fwrite(r.t.data(), 4, r.t.size(), f) == r.t.size();
}

// One tap record (the name is the caller's).  kBadHeader: a short read of the ints, or Cout, Cin outside (0, inf), ntaps
// outside [1, XVB_MAX_TAPS] or tot_context outside [ntaps, 4096) or not the span of ctx; kTruncated: a short read of the
// arrays.
enum TapRead { kTapOk, kBadHeader, kTruncated };
TapRead read_tap(FILE* f, xvb::TapRec* r) {
  int32_t hd[7];
  if (!rd(f, hd, sizeof hd)) return kBadHeader;
  r->Cout = hd[0]; r->Cin = hd[1]; r->ntaps = hd[2]; r->flags = hd[4];
  const int tot = hd[3];
  if (!(r->Cout > 0 && r->Cin > 0 && r->ntaps >= 1 && r->ntaps <= XVB_MAX_TAPS && tot >= r->ntaps && tot < 4096) ||
      !rd(f, r->ctx, 4 * (size_t)r->ntaps) || tot != r->tot())
    return kBadHeader;
  r->w.resize((size_t)r->Cout * r->Cin * tot);
  r->b.resize(hd[5] ? r->Cout : 0);
  r->s.resize(hd[6] ? r->Cout : 0);
  r->t.resize(r->s.size());
  const bool ok = rd(f, r->w.data(), r->w.size() * 4) && rd(f, r->b.data(), r->b.size() * 4) &&
                  rd(f, r->s.data(), r->s.size() * 4) && rd(f, r->t.data(), r->t.size() * 4);
  return ok ? kTapOk : kTruncated;
}

const float* or_null(const std::vector<float>& v) { return v.empty() ? nullptr : v.data(); }
}  // namespace

namespace xvb {

TapRec tap_record(const char* name, int Cout, int Cin, const int* ctx, int ntaps, const float* w, const float* b,
                  const float* s, const float* t, int flags) {
  TapRec r;
  r.name = name;
  r.Cout = Cout; r.Cin = Cin; r.ntaps = ntaps; r.flags = flags;
  for (int i = 0; i < ntaps; ++i) r.ctx[i] = ctx[i];
  r.w.assign(w, w + (size_t)Cout * Cin * r.tot());
  if (b) r.b.assign(b, b + Cout);
  if (flags & XVB_BN) { r.s.assign(s, s + Cout); r.t.assign(t, t + Cout); }
  return r;
}

int save_tap_file(const char* fn, const char* path, const char* magic, const void* head, size_t head_bytes,
                  const std::vector<const TapRec*>& layers, bool named) {
  FILE* f = fopen(path, "wb");
  FAIL_IF(!f, "%s: cannot open '%s'", fn, path);
  bool ok = fwrite(magic, 1, 8, f) == 8 && fwrite(head, 1, head_bytes, f) == head_bytes;
  for (const TapRec* r : layers) {
    const int32_t nl = (int32_t)r->name.size();
    if (named) ok = ok && fwrite(&nl, 4, 1, f) == 1 && fwrite(r->name.data(), 1, r->name.size(), f) == r->name.size();
    ok = ok && write_tap(f, *r);
  }
  ok = fclose(f) == 0 && ok;
  FAIL_IF(!ok, "%s: write to '%s' failed", fn, path);
  return XVB_OK;
}

int RecordStore::check(const char* fn, const char* name, const int* shape, const float* w, const float* s,
                       const float* t) const {
  char buf[48];
  FAIL_IF(!shape_ok(shape, n), "%s(%s): bad shape %s", fn, name, shape_str(shape, n, buf));
  FAIL_IF((shape[n - 1] > 0) != (w != nullptr) || (w && shape[1] == 0),
          n == 2 ? "%s(%s): a weight needs cols > 0, a norm record cols 0"
                 : "%s(%s): a weight needs ksize 1 or 3 and Cin > 0, a BatchNorm record ksize 0 and no weight",
          fn, name);
  FAIL_IF((s == nullptr) != (t == nullptr), "%s(%s): scale and shift go together", fn, name);
  return XVB_OK;
}

int RecordStore::add(const char* fn, const char* name, const int* shape, const float* w, const float* b,
                     const float* s, const float* t, int flags) {
  FAIL_IF(recs.count(name), "%s: record '%s' set twice", fn, name);
  Rec r;
  for (int i = 0; i < n; ++i) r.shape[i] = shape[i];
  r.flags = flags;
  const size_t rows = (size_t)shape[0];
  if (w) r.w.assign(w, w + (size_t)weight_elems(shape, n));
  if (b) r.b.assign(b, b + rows);
  if (s) { r.s.assign(s, s + rows); r.t.assign(t, t + rows); }
  recs[name] = std::move(r);
  order.push_back(name);
  return XVB_OK;
}

const Rec* RecordStore::find(const std::string& name) const {
  auto it = recs.find(name);
  return it == recs.end() ? nullptr : &it->second;
}

int RecordStore::take(const char* fn, const std::string& name, const int* shape, const Rec** out) {
  const Rec* r = find(name);
  FAIL_IF(!r, "%s: record '%s' is missing", fn, name.c_str());
  char have[48], want[48];
  FAIL_IF(memcmp(r->shape, shape, n * sizeof(int)) != 0, "%s: record '%s' is %s, expected %s", fn, name.c_str(),
          shape_str(r->shape, n, have), shape_str(shape, n, want));
  used.insert(name);
  *out = r;
  return XVB_OK;
}

int RecordStore::check_all_used(const char* fn) const {
  for (const std::string& name : order)
    FAIL_IF(!used.count(name), "%s: record '%s' is not part of this configuration", fn, name.c_str());
  return XVB_OK;
}

// The named-record model files ("XVBR0001" ResNet, "XVBC0001" Conformer, "XVBP0001" CAM++), little-endian:
//
//   magic[8] | configuration block (RecordFormat::cfg_bytes raw bytes) | i32 nrec
//   per record, in set_layer order:
//     i32 name_len | name (no NUL) | i32 shape[nshape] | i32 flags | i32 has_w | i32 has_b | i32 has_s
//     | f32 w[weight elements]? | f32 b[rows]? | f32 s[rows], t[rows]?
//
// Loading refuses a wrong magic, nrec outside [1, max_records], a name length outside (0, 127), a shape outside the
// set_layer bounds (rows in (0, 65536], the second int in [0, 2^20], at most 2^28 weight elements), has_w not equal to
// (last shape int > 0) and a short read; set_layer and finalize then check the records against the configuration.
int save_records(const char* fn, const char* path, const RecordFormat& fmt, const void* cfg, const RecordStore& store) {
  FILE* f = fopen(path, "wb");
  FAIL_IF(!f, "%s: cannot open '%s'", fn, path);
  const int32_t nrec = (int32_t)store.order.size();
  bool ok = fwrite(fmt.magic, 1, 8, f) == 8 && fwrite(cfg, 1, fmt.cfg_bytes, f) == fmt.cfg_bytes && fwrite(&nrec, 4, 1, f) == 1;
  for (const std::string& n : store.order) {
    const Rec& r = store.recs.at(n);
    const int32_t nl = (int32_t)n.size();
    int32_t hd[7];
    int k = 0;
    for (int i = 0; i < fmt.nshape; ++i) hd[k++] = r.shape[i];
    hd[k++] = r.flags; hd[k++] = !r.w.empty(); hd[k++] = !r.b.empty(); hd[k++] = !r.s.empty();
    ok = ok && fwrite(&nl, 4, 1, f) == 1 && fwrite(n.data(), 1, n.size(), f) == n.size() && fwrite(hd, 4, k, f) == (size_t)k &&
         fwrite(r.w.data(), 4, r.w.size(), f) == r.w.size() && fwrite(r.b.data(), 4, r.b.size(), f) == r.b.size() &&
         fwrite(r.s.data(), 4, r.s.size(), f) == r.s.size() && fwrite(r.t.data(), 4, r.t.size(), f) == r.t.size();
  }
  ok = fclose(f) == 0 && ok;
  FAIL_IF(!ok, "%s: write to '%s' failed", fn, path);
  return XVB_OK;
}

int load_records(const char* fn, const char* path, const RecordFormat& fmt, void** out,
                 int (*create)(void** h, const void* cfg),
                 int (*set_layer)(void* h, const char* name, const int* shape, const float* w, const float* b,
                                  const float* s, const float* t, int flags),
                 int (*finalize)(void* h), void (*destroy)(void* h)) {
  FAIL_IF(!out || !path, "%s: null argument", fn);
  FILE* f = fopen(path, "rb");
  FAIL_IF(!f, "%s: cannot open '%s'", fn, path);
  char magic[8];
  std::vector<char> cfg(fmt.cfg_bytes);
  int32_t nrec = 0;
  void* h = nullptr;
  int rc = XVB_EINVAL;
  do {
    if (!rd(f, magic, 8) || memcmp(magic, fmt.magic, 8) != 0 || !rd(f, cfg.data(), cfg.size()) || !rd(f, &nrec, 4) ||
        nrec < 1 || nrec > fmt.max_records) {
      set_error("%s: '%s' is not an %.8s file", fn, path, fmt.magic);
      break;
    }
    if ((rc = create(&h, cfg.data()))) break;
    const int ns = fmt.nshape;
    std::vector<float> w, b, s, t;
    for (int i = 0; i < nrec && rc == XVB_OK; ++i) {
      int32_t nl = 0, hd[7] = {0};   // shape[ns], flags, has_w, has_b, has_s
      char name[128];
      bool ok = rd(f, &nl, 4) && nl > 0 && nl < 127 && rd(f, name, (size_t)nl) && rd(f, hd, 4 * (size_t)(ns + 4)) &&
                shape_ok(hd, ns) && hd[ns + 1] == (hd[ns - 1] > 0);
      const int32_t flags = hd[ns], has_w = hd[ns + 1], has_b = hd[ns + 2], has_s = hd[ns + 3];
      if (ok) {
        name[nl] = 0;
        w.resize(has_w ? (size_t)weight_elems(hd, ns) : 0);
        ok = rd(f, w.data(), w.size() * 4);
        if (ok && has_b) { b.resize(hd[0]); ok = rd(f, b.data(), b.size() * 4); }
        if (ok && has_s) { s.resize(hd[0]); t.resize(hd[0]); ok = rd(f, s.data(), s.size() * 4) && rd(f, t.data(), t.size() * 4); }
      }
      if (!ok) { set_error("%s: '%s' is truncated or corrupt at record %d", fn, path, i); rc = XVB_EINVAL; break; }
      rc = set_layer(h, name, hd, has_w ? w.data() : nullptr, has_b ? b.data() : nullptr, has_s ? s.data() : nullptr,
                     has_s ? t.data() : nullptr, flags);
    }
    if (rc == XVB_OK) rc = finalize(h);
  } while (0);
  fclose(f);
  if (rc != XVB_OK) { if (h) destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}

}  // namespace xvb

extern "C" int xvb_extractor_load(xvb_extractor_t** out, const char* path) {
  if (!out || !path) { set_error("xvb_extractor_load: null argument"); return XVB_EINVAL; }
  FILE* f = fopen(path, "rb");
  if (!f) { set_error("xvb_extractor_load: cannot open '%s'", path); return XVB_EINVAL; }
  xvb_extractor_t* h = nullptr;
  int rc = XVB_EINVAL;
  char magic[8];
  int32_t feat_dim = 0, n_frame = 0, n_seg = 0;
  float eps = 0.f;
  xvb::AttnPoolRecord pool = {0, 0, 0, 0, 0};
  do {
    const bool got_magic = rd(f, magic, 8);
    const bool att = got_magic && memcmp(magic, "XVBM0002", 8) == 0;
    if (!att && (!got_magic || memcmp(magic, "XVBM0001", 8) != 0)) {
      set_error("xvb_extractor_load: '%s' is not an XVBM0001 file or an XVBM0002 file", path);
      break;
    }
    if (!rd(f, &feat_dim, 4) || !rd(f, &eps, 4) || !rd(f, &n_frame, 4) || !rd(f, &n_seg, 4) || feat_dim <= 0 ||
        n_frame <= 0 || n_seg <= 0 || n_frame > 64 || n_seg > 64) { set_error("xvb_extractor_load: bad header in '%s'", path); break; }
    std::vector<float> prior[2];
    if (att && (!rd(f, &pool, sizeof pool) ||
                !(pool.kind == XVB_POOL_ATTENTION || pool.kind == XVB_POOL_XI_POSTMEAN || pool.kind == XVB_POOL_XI_POSTDIST) ||
                pool.pooled <= 0 || pool.pooled > (1 << 20) || pool.n_attention < 1 || pool.n_attention > 2)) {
      set_error("xvb_extractor_load: '%s' is not an XVBM0001 file or an XVBM0002 file: bad pooling record", path);
      break;
    }
    const bool xi = pool.kind == XVB_POOL_XI_POSTMEAN || pool.kind == XVB_POOL_XI_POSTDIST;
    if (xi) {
      prior[0].resize(pool.pooled);
      prior[1].resize(pool.pooled);
      if (!rd(f, prior[0].data(), 4 * (size_t)pool.pooled) || !rd(f, prior[1].data(), 4 * (size_t)pool.pooled)) {
        set_error("xvb_extractor_load: '%s' is truncated in the xi-vector prior", path);
        break;
      }
    }
    if ((rc = xvb_extractor_create(&h, feat_dim)) != XVB_OK) break;
    if (att && (rc = xvb_extractor_set_attention_pooling(h, pool.kind, pool.pooled, pool.gdiv, pool.unweighted,
                                                         xi ? prior[0].data() : nullptr, xi ? prior[1].data() : nullptr)))
      break;
    xvb::TapRec r;
    const int n_att = pool.n_attention;
    int cin = feat_dim;   // the input width add_*_layer gives the layer
    int c_last = 0;       // the last frame layer's channels
    for (int i = 0; rc == XVB_OK && i < n_frame + n_att + n_seg; ++i) {
      if (i == n_frame) c_last = cin;
      if (i == n_frame + n_att)   // mean | std, or the attention pooling's own width
        cin = !att ? 2 * c_last : pool.kind == XVB_POOL_XI_POSTMEAN ? pool.pooled : 2 * pool.pooled;
      const TapRead got = read_tap(f, &r);
      if (got == kBadHeader || r.Cin != cin) { set_error("xvb_extractor_load: bad layer %d header in '%s'", i, path); rc = XVB_EINVAL; break; }
      if (got == kTruncated) { set_error("xvb_extractor_load: '%s' is truncated in layer %d", path, i); rc = XVB_EINVAL; break; }
      if (i < n_frame)
        rc = xvb_extractor_add_frame_layer(h, r.Cout, r.ctx, r.ntaps, r.w.data(), or_null(r.b), or_null(r.s), or_null(r.t), r.flags);
      else if (i < n_frame + n_att)
        rc = xvb_extractor_add_attention_layer(h, r.Cout, r.ctx, r.ntaps, r.w.data(), or_null(r.b), or_null(r.s), or_null(r.t), r.flags);
      else
        rc = xvb_extractor_add_segment_layer(h, r.Cout, r.w.data(), or_null(r.b), or_null(r.s), or_null(r.t), r.flags);
      cin = r.Cout;
    }
    if (rc == XVB_OK) rc = xvb_extractor_finalize(h, eps);
  } while (0);
  fclose(f);
  if (rc != XVB_OK) { if (h) xvb_extractor_destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_extractor_feat_dim(const char* path) {
  FILE* f = path ? fopen(path, "rb") : nullptr;
  if (!f) { set_error("xvb_extractor_feat_dim: cannot open '%s'", path ? path : "(null)"); return XVB_EINVAL; }
  char magic[8];
  int32_t d = 0;
  const bool ok = rd(f, magic, 8) && (memcmp(magic, "XVBM0001", 8) == 0 || memcmp(magic, "XVBM0002", 8) == 0) &&
                  rd(f, &d, 4) && d > 0;
  fclose(f);
  if (!ok) { set_error("xvb_extractor_feat_dim: '%s' is not an XVBM0001 file or an XVBM0002 file", path); return XVB_EINVAL; }
  return d;
}

extern "C" int xvb_ecapa_load(xvb_ecapa_t** out, const char* path) {
  if (!out || !path) { set_error("xvb_ecapa_load: null argument"); return XVB_EINVAL; }
  FILE* f = fopen(path, "rb");
  if (!f) { set_error("xvb_ecapa_load: cannot open '%s'", path); return XVB_EINVAL; }
  char magic[8];
  int32_t hd[6];
  xvb_ecapa_t* h = nullptr;
  int rc = XVB_EINVAL;
  do {
    int32_t pr[8];   // the pooling record, then XVBG0001's residual form; or XVBE0003's attention record
    const bool got = rd(f, magic, 8);
    const bool g = got && memcmp(magic, "XVBG0001", 8) == 0;
    const bool mq = g || (got && memcmp(magic, "XVBE0002", 8) == 0);
    const bool att = got && memcmp(magic, "XVBE0003", 8) == 0;
    const bool ok_magic = mq || att || (got && memcmp(magic, "XVBE0001", 8) == 0);
    if (!ok_magic || !rd(f, hd, sizeof hd) || hd[5] < 1 || hd[5] > 256 || (mq && !rd(f, pr, (g ? 8 : 7) * sizeof(int32_t))) ||
        (att && !rd(f, pr, 2 * sizeof(int32_t)))) {
      set_error("xvb_ecapa_load: '%s' is not an XVBE0001 / XVBE0002 / XVBE0003 / XVBG0001 file", path);
      break;
    }
    if ((rc = xvb_ecapa_create(&h, hd[0], hd[1], hd[2], hd[3], hd[4]))) break;
    if (mq && (rc = xvb_ecapa_set_mqmha(h, pr[0], pr[1], pr[2], pr[3], pr[4], pr[5], pr[6]))) break;
    if (g && (rc = xvb_ecapa_set_chained(h, pr[7]))) break;
    if (att) {
      float floor_;
      memcpy(&floor_, &pr[1], sizeof floor_);
      if (pr[0] == 1 && floor_ == 1e-5f) {   // the default attention is written as XVBE0001
        set_error("xvb_ecapa_load: '%s' is an XVBE0003 file with the default attention", path);
        rc = XVB_EINVAL;
        break;
      }
      if ((rc = xvb_ecapa_set_attention(h, pr[0], floor_))) break;
    }
    xvb::TapRec r;
    for (int i = 0; i < hd[5] && rc == XVB_OK; ++i) {
      int32_t nl = 0;
      char name[128];
      if (!(rd(f, &nl, 4) && nl > 0 && nl < 127 && rd(f, name, (size_t)nl) && read_tap(f, &r) == kTapOk)) {
        set_error("xvb_ecapa_load: '%s' is truncated or corrupt at layer %d", path, i);
        rc = XVB_EINVAL;
        break;
      }
      name[nl] = 0;
      rc = xvb_ecapa_set_layer(h, name, r.Cout, r.Cin, r.ctx, r.ntaps, r.w.data(), or_null(r.b), or_null(r.s), or_null(r.t),
                               r.flags);
    }
    if (rc == XVB_OK) rc = xvb_ecapa_finalize(h);
  } while (0);
  fclose(f);
  if (rc != XVB_OK) { if (h) xvb_ecapa_destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}
