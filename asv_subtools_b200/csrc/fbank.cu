// Kaldi-compatible fbank / MFCC from raw waveforms on the GPU (SURVEY section 8f, rank 1, second half).
//
// The reference's online path computes features with KaldiFeature (pytorch/libs/egs/kaldi_features.py
// :69-135) -> torchaudio.compliance.kaldi.fbank / .mfcc, and its C++ runtime with kaldifeat
// (runtime/kaldifeat/csrc/feature-fbank.cc, feature-window.cc, mel-computations.cc); both restate Kaldi's
// compute-fbank-feats.  Per frame (snip_edges, dither 0 -- the launchers force it for extraction,
// runEcapaXvector_online.py:380-381):
//   remove DC -> [raw log-energy] -> pre-emphasis (replicate first sample) -> window -> zero-pad to 2^k
//   -> |rFFT|^2 -> triangular mel bank -> log(max(., eps)) [-> DCT-II + lifter for MFCC]
// One warp owns one frame, entirely in shared memory: the N-point real FFT is an N/2-point complex
// radix-2 DIF (bit-reversed output, no permutation pass) plus the even/odd recombination; the mel bank
// is stored sparse (each FFT bin feeds at most two filters).  Work per frame is ~1 % of the network's,
// bytes are 2.5 KB in / 320 B out: nowhere near a roofline, so the kernel is written for accuracy
// (double-precision tables) and simplicity.  Ragged batches: utterances back to back in one sample
// array with (U+1) sample offsets and (U+1) frame offsets.
#include <cuda_runtime.h>
#include <float.h>
#include <math.h>

#include <vector>

#include "common.cuh"

namespace xvb {

struct FbankDev {
  const float* window;
  const float2* tw_m;       // exp(-2 pi i k / M), k < M/2
  const float2* tw_n;       // exp(-2 pi i k / N), k <= M
  const int* mel_start;
  const int* mel_len;
  const int* mel_off;
  const float* mel_w;
  const float* dct;         // (num_mel, num_ceps) or null
  const float* lifter;      // (num_ceps) or null
  int shift, size, N, log2m, num_mel, num_ceps, dim;
  int remove_dc, use_energy, raw_energy, use_log, use_power, htk_compat;
  float preemph, log_energy_floor;   // log_energy_floor = -inf when energy_floor == 0
};

constexpr int kFbankWarps = 8;

// Floats of shared memory per warp: N samples (M float2), M + 4 spectrum values, 128 log-mel energies.  Rounded up to
// a multiple of 4 so that every warp's slice starts 16-byte aligned: the float2 accesses to z compile to 8-byte
// vector loads and stores, and N = 2 (M = 1) would otherwise leave odd warps 4 bytes off.
__host__ __device__ constexpr int fbank_warp_floats(int N) { return (N + (N / 2 + 4) + 128 + 3) & ~3; }

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__global__ void __launch_bounds__(kFbankWarps * 32)
fbank_kernel(const float* __restrict__ wave, const long long* __restrict__ sample_off, const int* __restrict__ frame_off,
             int num_utts, long long total_frames, FbankDev d, float* __restrict__ out) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int M = d.N >> 1;
  float* xs = smem + warp * fbank_warp_floats(d.N);            // N floats == M float2
  float2* z = reinterpret_cast<float2*>(xs);
  float* P = xs + d.N;                           // M + 1 spectrum values
  float* lm = P + (M + 4);                       // log-mel energies (MFCC)
  const long long f = (long long)blockIdx.x * kFbankWarps + warp;
  if (f >= total_frames) return;                 // whole warp leaves together
  // utterance of this frame: last u with frame_off[u] <= f
  int lo = 0, hi = num_utts;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if ((long long)frame_off[mid] <= f) lo = mid; else hi = mid;
  }
  const float* src = wave + sample_off[lo] + (f - frame_off[lo]) * (long long)d.shift;

  float s = 0.f;
  for (int i = lane; i < d.size; i += 32) { const float v = src[i]; xs[i] = v; s += v; }
  const float mean = d.remove_dc ? warp_sum(s) / (float)d.size : 0.f;
  __syncwarp();
  float e = 0.f;
  for (int i = lane; i < d.size; i += 32) { const float v = xs[i] - mean; xs[i] = v; e = fmaf(v, v, e); }
  float energy = warp_sum(e);                    // raw energy (after DC removal, before pre-emphasis)
  __syncwarp();
  // pre-emphasis + window, chunks from the top so that x[i-1] is still the unmodified sample
  for (int base = ((d.size - 1) >> 5) << 5; base >= 0; base -= 32) {
    const int i = base + lane;
    float y = 0.f;
    if (i < d.size) y = (xs[i] - d.preemph * xs[i > 0 ? i - 1 : 0]) * d.window[i];
    __syncwarp();
    if (i < d.size) xs[i] = y;
    __syncwarp();
  }
  for (int i = d.size + lane; i < d.N; i += 32) xs[i] = 0.f;
  __syncwarp();
  if (d.use_energy && !d.raw_energy) {
    e = 0.f;
    for (int i = lane; i < d.size; i += 32) e = fmaf(xs[i], xs[i], e);
    energy = warp_sum(e);
  }
  float log_energy = fmaxf(logf(fmaxf(energy, FLT_EPSILON)), d.log_energy_floor);

  // M-point complex DIF FFT of z[n] = x[2n] + i x[2n+1]; Z[k] ends up at z[bitrev(k)]
  for (int h = M >> 1, tstep = 1; h >= 1; h >>= 1, tstep <<= 1) {
    for (int j = lane; j < (M >> 1); j += 32) {
      const int pos = j & (h - 1);
      const int i0 = ((j - pos) << 1) + pos, i1 = i0 + h;
      const float2 a = z[i0], b = z[i1], w = d.tw_m[pos * tstep];
      const float dx = a.x - b.x, dy = a.y - b.y;
      z[i0] = make_float2(a.x + b.x, a.y + b.y);
      z[i1] = make_float2(dx * w.x - dy * w.y, dx * w.y + dy * w.x);
    }
    __syncwarp();
  }
  // even/odd recombination: X[k] = E[k] + W_N^k O[k], k = 0..M
  const int rsh = 32 - d.log2m;
  for (int k = lane; k <= M; k += 32) {
    const int k0 = k & (M - 1), k1 = (M - k) & (M - 1);
    const float2 a = z[d.log2m ? (__brev((unsigned)k0) >> rsh) : 0];
    const float2 c = z[d.log2m ? (__brev((unsigned)k1) >> rsh) : 0];
    const float ex = 0.5f * (a.x + c.x), ey = 0.5f * (a.y - c.y);      // E = (Z[k] + conj Z[M-k]) / 2
    const float ox = 0.5f * (a.y + c.y), oy = -0.5f * (a.x - c.x);     // O = -i (Z[k] - conj Z[M-k]) / 2
    const float2 w = d.tw_n[k];
    const float xr = ex + (w.x * ox - w.y * oy), xi = ey + (w.x * oy + w.y * ox);
    const float p = xr * xr + xi * xi;
    P[k] = d.use_power ? p : sqrtf(p);
  }
  __syncwarp();
  const bool mfcc = d.num_ceps > 0;
  float* row = out + f * (long long)d.dim;
  const int mel_col0 = (d.use_energy && !d.htk_compat) ? 1 : 0;
  for (int b = lane; b < d.num_mel; b += 32) {
    const int st = d.mel_start[b], n = d.mel_len[b];
    const float* w = d.mel_w + d.mel_off[b];
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(w[j], P[st + j], acc);
    if (d.use_log) acc = logf(fmaxf(acc, FLT_EPSILON));
    if (mfcc) lm[b] = acc;
    else row[mel_col0 + b] = acc;
  }
  if (!mfcc) {
    if (d.use_energy && lane == 0) row[d.htk_compat ? d.num_mel : 0] = log_energy;
    return;
  }
  __syncwarp();
  for (int c = lane; c < d.num_ceps; c += 32) {
    float acc = 0.f;
    for (int b = 0; b < d.num_mel; ++b) acc = fmaf(lm[b], d.dct[b * d.num_ceps + c], acc);
    acc *= d.lifter[c];
    if (c == 0 && d.use_energy) acc = log_energy;
    if (!d.htk_compat) row[c] = acc;
    else if (c > 0) row[c - 1] = acc;
    else row[d.num_ceps - 1] = d.use_energy ? acc : acc * 1.41421356237309515f;
  }
}

}  // namespace xvb

using namespace xvb;

struct xvb_fbank {
  xvb_fbank_opts_t o;
  FbankDev d{};
  std::vector<void*> bufs;
  template <typename T>
  int upload(const std::vector<T>& h, const T** dst) {
    void* p = nullptr;
    XVB_CUDA(cudaMalloc(&p, h.size() * sizeof(T) + 16));
    bufs.push_back(p);
    XVB_CUDA(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
    *dst = static_cast<const T*>(p);
    return XVB_OK;
  }
};

extern "C" void xvb_fbank_default_opts(xvb_fbank_opts_t* o) {
  if (!o) return;
  // torchaudio.compliance.kaldi.fbank / mfcc defaults (= Kaldi's), with dither fixed at 0
  o->sample_frequency = 16000.f; o->frame_length_ms = 25.f; o->frame_shift_ms = 10.f;
  o->preemphasis_coefficient = 0.97f; o->low_freq = 20.f; o->high_freq = 0.f; o->energy_floor = 1.0f;
  o->cepstral_lifter = 22.f; o->blackman_coeff = 0.42f;
  o->num_mel_bins = 23; o->num_ceps = 0; o->use_energy = 0; o->raw_energy = 1; o->remove_dc_offset = 1;
  o->use_log_fbank = 1; o->use_power = 1; o->htk_compat = 0; o->window_type = XVB_WINDOW_POVEY;
}

extern "C" int xvb_fbank_create(xvb_fbank_t** out, const xvb_fbank_opts_t* opts) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(out && opts, "xvb_fbank_create: null argument");
  const xvb_fbank_opts_t& o = *opts;
  const int shift = (int)(o.sample_frequency * o.frame_shift_ms * 0.001f);
  const int size = (int)(o.sample_frequency * o.frame_length_ms * 0.001f);
  XVB_CHECK_ARG(o.sample_frequency > 0 && shift > 0 && size >= 2 && size <= 4096, "xvb_fbank_create: bad frame geometry (window of %d samples)", size);
  XVB_CHECK_ARG(o.num_mel_bins > 3 && o.num_mel_bins <= 128, "xvb_fbank_create: num_mel_bins=%d outside (3, 128]", o.num_mel_bins);
  XVB_CHECK_ARG(o.num_ceps >= 0 && o.num_ceps <= o.num_mel_bins, "xvb_fbank_create: num_ceps=%d cannot exceed num_mel_bins", o.num_ceps);
  XVB_CHECK_ARG(o.preemphasis_coefficient >= 0.f && o.preemphasis_coefficient <= 1.f, "xvb_fbank_create: preemphasis must be in [0,1]");
  XVB_CHECK_ARG(o.window_type >= 0 && o.window_type <= XVB_WINDOW_BLACKMAN, "xvb_fbank_create: unknown window type %d", o.window_type);
  XVB_CHECK_ARG(o.num_ceps == 0 || (o.use_log_fbank && o.use_power), "xvb_fbank_create: MFCC is defined on log power mel energies");
  int N = 1, log2n = 0;
  while (N < size) { N <<= 1; ++log2n; }
  const int M = N / 2;
  const double nyq = 0.5 * o.sample_frequency;
  double hi_f = o.high_freq;
  if (hi_f <= 0.0) hi_f += nyq;
  XVB_CHECK_ARG(o.low_freq >= 0.f && o.low_freq < nyq && hi_f > 0.0 && hi_f <= nyq && o.low_freq < hi_f,
                "xvb_fbank_create: bad low/high frequency %g/%g for Nyquist %g", (double)o.low_freq, hi_f, nyq);

  xvb_fbank* h = new xvb_fbank();
  h->o = o;
  FbankDev& d = h->d;
  d.shift = shift; d.size = size; d.N = N; d.log2m = log2n - 1; d.num_mel = o.num_mel_bins; d.num_ceps = o.num_ceps;
  d.remove_dc = o.remove_dc_offset; d.use_energy = o.use_energy; d.raw_energy = o.raw_energy; d.use_log = o.use_log_fbank;
  d.use_power = o.use_power; d.htk_compat = o.htk_compat; d.preemph = o.preemphasis_coefficient;
  d.log_energy_floor = o.energy_floor == 0.f ? -INFINITY : logf(o.energy_floor);
  d.dim = (o.num_ceps > 0 ? o.num_ceps : o.num_mel_bins + (o.use_energy ? 1 : 0));

  const double pi = 3.14159265358979323846;
  std::vector<float> win(size);
  for (int i = 0; i < size; ++i) {
    const double a = 2.0 * pi / (size - 1), c = cos(a * i);
    double w = 1.0;
    switch (o.window_type) {
      case XVB_WINDOW_POVEY: w = pow(0.5 - 0.5 * c, 0.85); break;
      case XVB_WINDOW_HAMMING: w = 0.54 - 0.46 * c; break;
      case XVB_WINDOW_HANNING: w = 0.5 - 0.5 * c; break;
      case XVB_WINDOW_BLACKMAN: w = o.blackman_coeff - 0.5 * c + (0.5 - o.blackman_coeff) * cos(2 * a * i); break;
      default: break;
    }
    win[i] = (float)w;
  }
  std::vector<float2> twm(M / 2 > 0 ? M / 2 : 1), twn(M + 1);
  for (int k = 0; k < M / 2; ++k) twm[k] = make_float2((float)cos(-2.0 * pi * k / M), (float)sin(-2.0 * pi * k / M));
  for (int k = 0; k <= M; ++k) twn[k] = make_float2((float)cos(-2.0 * pi * k / N), (float)sin(-2.0 * pi * k / N));
  // mel bank (get_mel_banks, vtln_warp = 1), sparse
  auto mel = [](double f) { return 1127.0 * log(1.0 + f / 700.0); };
  const double mlo = mel(o.low_freq), mhi = mel(hi_f), delta = (mhi - mlo) / (o.num_mel_bins + 1);
  std::vector<int> st(o.num_mel_bins), ln(o.num_mel_bins), off(o.num_mel_bins);
  std::vector<float> mw;
  for (int b = 0; b < o.num_mel_bins; ++b) {
    const double left = mlo + b * delta, center = left + delta, right = center + delta;
    int first = -1, last = -2;
    std::vector<float> w(M, 0.f);
    for (int k = 0; k < M; ++k) {
      const double m = mel((double)o.sample_frequency / N * k);
      const double v = fmin((m - left) / (center - left), (right - m) / (right - center));
      if (v > 0.0) { w[k] = (float)v; if (first < 0) first = k; last = k; }
    }
    st[b] = first < 0 ? 0 : first;
    ln[b] = first < 0 ? 0 : last - first + 1;
    off[b] = (int)mw.size();
    for (int k = 0; k < ln[b]; ++k) mw.push_back(w[st[b] + k]);
  }
  if (mw.empty()) mw.push_back(0.f);
  rc = h->upload(win, &d.window);
  if (!rc) rc = h->upload(twm, &d.tw_m);
  if (!rc) rc = h->upload(twn, &d.tw_n);
  if (!rc) rc = h->upload(st, &d.mel_start);
  if (!rc) rc = h->upload(ln, &d.mel_len);
  if (!rc) rc = h->upload(off, &d.mel_off);
  if (!rc) rc = h->upload(mw, &d.mel_w);
  if (!rc && o.num_ceps > 0) {
    const int nb = o.num_mel_bins, nc = o.num_ceps;
    std::vector<float> dct((size_t)nb * nc), lift(nc);
    for (int n = 0; n < nb; ++n)
      for (int k = 0; k < nc; ++k)
        dct[(size_t)n * nc + k] = (float)(k == 0 ? sqrt(1.0 / nb) : cos(pi / nb * (n + 0.5) * k) * sqrt(2.0 / nb));
    for (int i = 0; i < nc; ++i) lift[i] = (float)(o.cepstral_lifter != 0.f ? 1.0 + 0.5 * o.cepstral_lifter * sin(pi * i / o.cepstral_lifter) : 1.0);
    rc = h->upload(dct, &d.dct);
    if (!rc) rc = h->upload(lift, &d.lifter);
  }
  if (rc) { xvb_fbank_destroy(h); return rc; }
  *out = h;
  return XVB_OK;
}

extern "C" int xvb_fbank_dim(const xvb_fbank_t* h) { return h ? h->d.dim : XVB_EINVAL; }

extern "C" int64_t xvb_fbank_num_frames(const xvb_fbank_t* h, int64_t num_samples) {
  if (!h) return XVB_EINVAL;
  return num_samples < h->d.size ? 0 : 1 + (num_samples - h->d.size) / h->d.shift;   // snip_edges (_get_strided)
}

extern "C" int xvb_fbank_compute(xvb_fbank_t* h, const float* wave, const int64_t* sample_offsets,
                                 const int32_t* frame_offsets, int num_utts, int64_t total_frames, float* feats,
                                 void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(h && wave && sample_offsets && frame_offsets && feats && num_utts > 0, "xvb_fbank_compute: bad arguments");
  XVB_CHECK_ARG(total_frames >= 0 && total_frames < (1ll << 31) * kFbankWarps, "xvb_fbank_compute: too many frames for one call");
  if (total_frames == 0) return XVB_OK;
  const size_t smem = (size_t)kFbankWarps * fbank_warp_floats(h->d.N) * sizeof(float);
  XVB_ENSURE_DYN_SMEM((fbank_kernel), 200 * 1024);
  static_assert(sizeof(long long) == sizeof(int64_t), "offset type");
  const unsigned grid = (unsigned)((total_frames + kFbankWarps - 1) / kFbankWarps);
  fbank_kernel<<<grid, kFbankWarps * 32, smem, (cudaStream_t)stream>>>(
      wave, reinterpret_cast<const long long*>(sample_offsets), frame_offsets, num_utts, total_frames, h->d, feats);
  XVB_LAUNCH_CHECK();
  return XVB_OK;
}

extern "C" void xvb_fbank_destroy(xvb_fbank_t* h) {
  if (!h) return;
  for (void* p : h->bufs) cudaFree(p);
  delete h;
}
