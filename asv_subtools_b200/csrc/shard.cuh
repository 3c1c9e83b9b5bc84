// The whole-shard protocol of the TDNN, ECAPA-TDNN and ResNet native extractors, written once: extract_host, the
// device-resident and the host-buffer shard calls, the pipelined submit / wait of single batches and the replicated
// embedding table (peer.cu).  A handle type H derives from Handle (records.cuh), has a `Shard<H> shard` member and
// specialises ShardFamily<H> with
//   static int extract(H*, const float* feats, int B, int T, float* emb, void* stream)   one batch, sets last_launches
//   static H* twin(const H*)                    a new handle on the same model: the second lane
//   static int feat_dim(const H*), embed_dim(const H*)
//
// Batch k of a shard runs on lane k & 1: lane 0 is the handle itself, lane 1 its twin, made on first use and kept until
// the handle is destroyed, each lane on its own stream forked from `stream` and joined back into it.  The wgmma layer
// kernels occupy whole SMs, so the two lanes' GEMMs queue behind one another; what overlaps is everything else: one
// batch's bandwidth-bound kernels run on the SMs' spare slots next to the other batch's GEMM CTAs, and a GEMM's ragged
// tail is filled by the other lane's CTAs.  There are two lanes only when N > batch, XVB_LANES (read on every call, so
// one process can compare both) is not 0 and the caller does not ask for a single lane.
#pragma once
#include <stdlib.h>

#include <memory>

#include "common.cuh"
#include "records.cuh"

namespace xvb {

template <typename H>
struct ShardFamily;

// An fp32 device buffer grown to the largest request.
struct DevBuf {
  float* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  ~DevBuf() { cudaFree(p); }
  int reserve(size_t n) {
    if (n <= cap) return XVB_OK;
    cudaFree(p);
    p = nullptr;
    cap = 0;
    XVB_CUDA(cudaMalloc((void**)&p, n * sizeof(float)));
    cap = n;
    return XVB_OK;
  }
};

template <typename H>
struct Shard {
  using F = ShardFamily<H>;
  // device slots of the host-buffer calls: two per lane, so the copy engine runs up to two batches ahead of a lane;
  // submit / wait use slots 0 and 1
  static constexpr int kSlots = 4;

  std::unique_ptr<H> lane1;
  cudaStream_t lane_stream[2] = {nullptr, nullptr};
  cudaEvent_t ev_fork = nullptr, ev_join[2] = {nullptr, nullptr};
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_h2d[kSlots] = {nullptr}, ev_done[kSlots] = {nullptr};
  DevBuf p_feats[kSlots], p_emb[kSlots];
  bool slot_busy[2] = {false, false};   // submitted and not yet waited for
  DevBuf h_feats, h_emb;                 // staging of extract_host
  // replicated embedding table: every shard batch's rows also go to these copies at row0 + (row inside the shard)
  float* tables[XVB_MAX_PEERS] = {nullptr};
  int n = 0;
  int64_t row0 = 0, ld = 0;

  ~Shard() {
    lane1.reset();
    for (int i = 0; i < 2; ++i) {
      if (lane_stream[i]) cudaStreamDestroy(lane_stream[i]);
      if (ev_join[i]) cudaEventDestroy(ev_join[i]);
    }
    if (ev_fork) cudaEventDestroy(ev_fork);
    for (int i = 0; i < kSlots; ++i) {
      if (ev_h2d[i]) cudaEventDestroy(ev_h2d[i]);
      if (ev_done[i]) cudaEventDestroy(ev_done[i]);
    }
    if (copy_stream) cudaStreamDestroy(copy_stream);
  }

  // The four calls below refuse a null or draft handle and bad sizes ("fn: bad arguments") before they touch it.
  // feats (B, T, F) host -> emb (B, E) host through device staging; synchronises `stream`.
  static int extract_host(H* h, const float* feats_host, int B, int T, float* emb_host, void* stream, const char* fn) {
    XVB_CHECK_ARG(finalized(h) && feats_host && emb_host && B > 0 && T > 0, "%s: bad arguments", fn);
    Shard& d = h->shard;
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t nf = (size_t)B * T * F::feat_dim(h), ne = (size_t)B * F::embed_dim(h);
    int rc;
    if ((rc = d.h_feats.reserve(nf)) || (rc = d.h_emb.reserve(ne))) return rc;
    XVB_CUDA(cudaMemcpyAsync(d.h_feats.p, feats_host, nf * sizeof(float), cudaMemcpyHostToDevice, s));
    if ((rc = F::extract(h, d.h_feats.p, B, T, d.h_emb.p, stream))) return rc;
    XVB_CUDA(cudaMemcpyAsync(emb_host, d.h_emb.p, ne * sizeof(float), cudaMemcpyDeviceToHost, s));
    XVB_CUDA(cudaStreamSynchronize(s));
    return XVB_OK;
  }

  int set_gather(float* const* t, int nt, int64_t r0, int64_t l, int E, const char* fn) {
    XVB_CHECK_ARG(nt >= 0 && nt <= XVB_MAX_PEERS, "%s: bad arguments", fn);
    XVB_CHECK_ARG(nt == 0 || (t && r0 >= 0 && l >= E && l % 4 == 0),
                  "%s: need tables, row0 >= 0, ld >= embed_dim and ld %% 4 == 0", fn);
    for (int k = 0; k < nt; ++k) tables[k] = t[k];
    n = nt; row0 = r0; ld = l;
    return XVB_OK;
  }

  // feats (N, T, F) and emb (N, E) on the device; asynchronous on `stream`.
  static int device(H* h, const float* feats, int64_t N, int T, int batch, float* emb, void* stream, bool single_lane,
                    const char* fn) {
    XVB_CHECK_ARG(finalized(h) && feats && emb && N > 0 && T > 0 && batch > 0, "%s: bad arguments", fn);
    Shard& d = h->shard;
    const size_t Fd = F::feat_dim(h), E = F::embed_dim(h);
    const cudaStream_t s = (cudaStream_t)stream;
    const bool lanes = two_lanes(N, batch, single_lane);
    int rc, launches = 0, k = 0;
    if (lanes && (rc = d.fork(h, s))) return rc;
    for (int64_t i = 0; i < N; i += batch, ++k) {
      const int b = (int)(N - i < batch ? N - i : batch);
      H* lane = (lanes && (k & 1)) ? d.lane1.get() : h;
      const cudaStream_t ls = lanes ? d.lane_stream[k & 1] : s;
      if ((rc = F::extract(lane, feats + (size_t)i * T * Fd, b, T, emb + (size_t)i * E, ls))) return rc;
      launches += lane->last_launches;
      if ((rc = d.scatter(emb + (size_t)i * E, b, (int)E, i, ls, &launches))) return rc;
    }
    if (lanes && (rc = d.join(s))) return rc;
    h->last_launches = launches;
    return XVB_OK;
  }

  // The same through host buffers (pinned, so that the copies are asynchronous): batch k's features cross the link on
  // the copy stream into slot k % kSlots while earlier batches run, its embeddings go back on its lane's stream.  Slot
  // reuse is ordered by events on the device; returns when all of emb_host is written.
  static int host(H* h, const float* feats_host, int64_t N, int T, int batch, float* emb_host, void* stream,
                  bool single_lane, const char* fn) {
    XVB_CHECK_ARG(finalized(h) && feats_host && emb_host && N > 0 && T > 0 && batch > 0, "%s: bad arguments", fn);
    Shard& d = h->shard;
    XVB_CHECK_ARG(!d.slot_busy[0] && !d.slot_busy[1], "%s: a submit_host slot is still in flight", fn);
    const size_t Fd = F::feat_dim(h), E = F::embed_dim(h);
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t bmax = (size_t)(N < batch ? N : batch);
    int rc;
    if ((rc = d.ensure_copy_stream())) return rc;
    for (int slot = 0; slot < kSlots; ++slot)
      if ((rc = d.reserve_slot(slot, bmax * T * Fd, bmax * E))) return rc;
    const bool lanes = two_lanes(N, batch, single_lane);
    if (lanes && (rc = d.fork(h, s))) return rc;
    int launches = 0, k = 0;
    for (int64_t i = 0; i < N; i += batch, ++k) {
      const int b = (int)(N - i < batch ? N - i : batch);
      const int slot = k % kSlots;
      H* lane = (lanes && (k & 1)) ? d.lane1.get() : h;
      const cudaStream_t ls = lanes ? d.lane_stream[k & 1] : s;
      if (k >= kSlots) XVB_CUDA(cudaStreamWaitEvent(d.copy_stream, d.ev_done[slot], 0));   // batch k - kSlots has left the slot
      XVB_CUDA(cudaMemcpyAsync(d.p_feats[slot].p, feats_host + (size_t)i * T * Fd, (size_t)b * T * Fd * sizeof(float),
                               cudaMemcpyHostToDevice, d.copy_stream));
      XVB_CUDA(cudaEventRecord(d.ev_h2d[slot], d.copy_stream));
      XVB_CUDA(cudaStreamWaitEvent(ls, d.ev_h2d[slot], 0));
      if ((rc = F::extract(lane, d.p_feats[slot].p, b, T, d.p_emb[slot].p, ls))) return rc;
      launches += lane->last_launches;
      if ((rc = d.scatter(d.p_emb[slot].p, b, (int)E, i, ls, &launches))) return rc;
      XVB_CUDA(cudaMemcpyAsync(emb_host + (size_t)i * E, d.p_emb[slot].p, (size_t)b * E * sizeof(float), cudaMemcpyDeviceToHost,
                               ls));
      XVB_CUDA(cudaEventRecord(d.ev_done[slot], ls));
    }
    if (lanes && (rc = d.join(s))) return rc;
    XVB_CUDA(cudaStreamSynchronize(s));
    h->last_launches = launches;
    return XVB_OK;
  }

  // One batch into slot 0 or 1 without waiting: the H2D on the copy stream, the stack and the D2H on `stream`.
  static int submit(H* h, const float* feats_host, int B, int T, float* emb_host, int slot, void* stream, const char* fn) {
    XVB_CHECK_ARG(finalized(h) && feats_host && emb_host && B > 0 && T > 0 && (slot == 0 || slot == 1),
                  "%s: bad arguments (slot must be 0 or 1)", fn);
    Shard& d = h->shard;
    XVB_CHECK_ARG(!d.slot_busy[slot], "%s: slot %d still in flight (call the wait of this handle)", fn, slot);
    const cudaStream_t s = (cudaStream_t)stream;
    const size_t nf = (size_t)B * T * F::feat_dim(h), ne = (size_t)B * F::embed_dim(h);
    int rc;
    if ((rc = d.ensure_copy_stream()) || (rc = d.reserve_slot(slot, nf, ne))) return rc;
    XVB_CUDA(cudaMemcpyAsync(d.p_feats[slot].p, feats_host, nf * sizeof(float), cudaMemcpyHostToDevice, d.copy_stream));
    XVB_CUDA(cudaEventRecord(d.ev_h2d[slot], d.copy_stream));
    XVB_CUDA(cudaStreamWaitEvent(s, d.ev_h2d[slot], 0));
    if ((rc = F::extract(h, d.p_feats[slot].p, B, T, d.p_emb[slot].p, stream))) return rc;
    XVB_CUDA(cudaMemcpyAsync(emb_host, d.p_emb[slot].p, ne * sizeof(float), cudaMemcpyDeviceToHost, s));
    XVB_CUDA(cudaEventRecord(d.ev_done[slot], s));
    d.slot_busy[slot] = true;
    return XVB_OK;
  }

  int wait(int slot) {
    if (!slot_busy[slot]) return XVB_OK;
    XVB_CUDA(cudaEventSynchronize(ev_done[slot]));
    slot_busy[slot] = false;
    return XVB_OK;
  }

 private:
  static bool two_lanes(int64_t N, int batch, bool single_lane) {
    const char* v = getenv("XVB_LANES");
    return !single_lane && (!v || atoi(v) != 0) && N > batch;
  }

  // Both lane streams start after everything already queued on `s`; the twin and the streams are made on first use.
  int fork(H* h, cudaStream_t s) {
    if (!lane1) {
      for (int i = 0; i < 2; ++i) {
        XVB_CUDA(cudaStreamCreateWithFlags(&lane_stream[i], cudaStreamNonBlocking));
        XVB_CUDA(cudaEventCreateWithFlags(&ev_join[i], cudaEventDisableTiming));
      }
      XVB_CUDA(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
      lane1.reset(F::twin(h));
    }
    XVB_CUDA(cudaEventRecord(ev_fork, s));
    for (int i = 0; i < 2; ++i) XVB_CUDA(cudaStreamWaitEvent(lane_stream[i], ev_fork, 0));
    return XVB_OK;
  }

  // `s` continues after both lanes.
  int join(cudaStream_t s) {
    for (int i = 0; i < 2; ++i) {
      XVB_CUDA(cudaEventRecord(ev_join[i], lane_stream[i]));
      XVB_CUDA(cudaStreamWaitEvent(s, ev_join[i], 0));
    }
    return XVB_OK;
  }

  int ensure_copy_stream() {
    if (copy_stream) return XVB_OK;
    XVB_CUDA(cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < kSlots; ++i) {
      XVB_CUDA(cudaEventCreateWithFlags(&ev_h2d[i], cudaEventDisableTiming));
      XVB_CUDA(cudaEventCreateWithFlags(&ev_done[i], cudaEventDisableTiming));
    }
    return XVB_OK;
  }

  int reserve_slot(int slot, size_t nf, size_t ne) {
    int rc = p_feats[slot].reserve(nf);
    return rc ? rc : p_emb[slot].reserve(ne);
  }

  // The rows [i, i + b) of the shard, just written to `e` on `ls`, into every table copy; counted as a launch.
  int scatter(const float* e, int b, int E, int64_t i, cudaStream_t ls, int* launches) {
    if (!n) return XVB_OK;
    ++*launches;
    return xvb_scatter_rows(e, b, E, tables, n, row0 + i, ld, ls);
  }
};

}  // namespace xvb
