// Host records of the native extractors and their model-file codecs (host code in model_file.cpp; the device-weight
// arena and the workspace are in records.cuh).
//
// The TDNN and ECAPA-TDNN hand over tap layers (TapRec).  The ResNet, RepVGG, Conformer and CAM++ set_layer hands over
// one record per state_dict module path: a small fixed shape, flags and up to four fp32 arrays.  The store keeps host
// copies in insertion order, so that save() writes the records exactly as they were handed over, and finalize() takes
// each record its configuration needs and then refuses any record it did not take.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <map>
#include <set>
#include <string>
#include <vector>

#include "../../include/xvb200.h"

namespace xvb {

// The shape of a TDNN layer as TdnnAffine stores it: Cout x Cin over the taps ctx[0..ntaps), strictly increasing; the
// weight spans the whole context from min(ctx[0], 0) to max(ctx[ntaps-1], 0) (components.py:50-53), unused taps
// included.
struct TapShape {
  int Cout = 0, Cin = 0, ntaps = 0, flags = 0;
  int ctx[XVB_MAX_TAPS] = {0};
  int left() const { return ctx[0] < 0 ? ctx[0] : 0; }
  int tot() const { return (ctx[ntaps - 1] > 0 ? ctx[ntaps - 1] : 0) - left() + 1; }
};

// One TDNN or ECAPA-TDNN layer exactly as handed over: w (Cout, Cin, tot), the bias when given, scale and shift when
// flags has XVB_BN.  name: the ECAPA-TDNN layer name; empty in the TDNN, whose layers are positional.
struct TapRec : TapShape {
  std::string name;
  std::vector<float> w, b, s, t;
};

// Host copies of a layer's arrays (the caller has checked the taps and that XVB_BN comes with scale and shift).
TapRec tap_record(const char* name, int Cout, int Cin, const int* ctx, int ntaps, const float* w, const float* b,
                  const float* s, const float* t, int flags);

// The pooling record of an "XVBM0002" file (a TDNN x-vector with an attention pooling; layout in model_file.cpp): the
// arguments of xvb_extractor_set_attention_pooling and the number of attention affines after the frame layers.
struct AttnPoolRecord { int32_t kind, pooled, gdiv, unweighted, n_attention; };

// The tap-layer files ("XVBM0001" TDNN, "XVBE0001" / "XVBE0002" ECAPA-TDNN; layouts in model_file.cpp): magic, the
// family's header block, then the layers in order, each preceded by its name when `named` (fn: the caller's name).
int save_tap_file(const char* fn, const char* path, const char* magic, const void* head, size_t head_bytes,
                  const std::vector<const TapRec*>& layers, bool named);

struct Rec {   // one named record exactly as handed over
  int shape[3] = {0, 0, 0};        // rows, cols (CAM++, Conformer) or Cout, Cin, ksize (ResNet)
  int flags = 0;
  std::vector<float> w, b, s, t;   // weight, bias, scale, shift; empty when not handed over
};

// One family's records and model file (layout at save_records in model_file.cpp).
struct RecordFormat {
  const char* magic;   // 8 bytes
  size_t cfg_bytes;    // the configuration block
  int nshape;          // 2: rows x cols, weight rows * cols; 3: Cout x Cin x ksize, weight Cout * Cin * ksize^2
  int max_records;
};

struct RecordStore {
  explicit RecordStore(int nshape) : n(nshape) {}
  int n;                              // shape ints per record
  std::map<std::string, Rec> recs;
  std::vector<std::string> order;     // insertion order, for save
  std::set<std::string> used;         // taken by finalize

  // set_layer's shared checks (fn: the caller's name): shape bounds, a weight exactly when the last shape int is > 0,
  // scale and shift together.  Family checks come between check and add.
  int check(const char* fn, const char* name, const int* shape, const float* w, const float* s, const float* t) const;
  // refuses a name set twice, then keeps host copies of the arrays
  int add(const char* fn, const char* name, const int* shape, const float* w, const float* b, const float* s,
          const float* t, int flags);
  const Rec* find(const std::string& name) const;
  // the record `name` with exactly this shape, marked used (fn: the caller's name)
  int take(const char* fn, const std::string& name, const int* shape, const Rec** out);
  // refuses the first record that no take marked used
  int check_all_used(const char* fn) const;
};

// Writes magic, the configuration block and the store's records in insertion order (fn: the caller's name).
int save_records(const char* fn, const char* path, const RecordFormat& fmt, const void* cfg, const RecordStore& store);

// Reads a file written by save_records through the family's entry points: create from the configuration block,
// set_layer per record, finalize; destroys the handle on any failure.  *out is written on success only.
int load_records(const char* fn, const char* path, const RecordFormat& fmt, void** out,
                 int (*create)(void** h, const void* cfg),
                 int (*set_layer)(void* h, const char* name, const int* shape, const float* w, const float* b,
                                  const float* s, const float* t, int flags),
                 int (*finalize)(void* h), void (*destroy)(void* h));

}  // namespace xvb
