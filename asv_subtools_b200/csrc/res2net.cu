// Res2Net block of ECAPA-TDNN as ONE persistent kernel (Res2NetBlock.forward,
// pytorch/model/ecapa_tdnn_xvector.py:61-75).
//
//   y_0 = x_0 ;  y_{i+1} = BN(ReLU(W_i * splice(x_{i+1} + [i>=1] y_i, [-d,0,d]) + b_i)),  i = 0..6
//
// The seven 128->128 dilated TDNN layers form a serial chain, but the chain only couples frames of the
// SAME utterance.  Launched as seven grid-wide GEMMs they leave most of the machine idle in each
// layer's last wave and pay launch + drain seven times.  Here a CTA OWNS utterances: it walks its
// utterance through all seven steps, tile by tile, with the same TMA -> wgmma pipeline as tdnn_gemm.cu
// (bf16x3 split operands, fp32 accumulators in registers).
// Step i reads chunk i+1 of the input tensor and -- as a second A source accumulated into the same
// accumulators (W(a+b) = Wa + Wb) -- chunk i of the OUTPUT tensor, which this very CTA wrote in
// step i-1: the only synchronisation is CTA-local (the consumers fence their stores, then release
// the producer through an mbarrier), no grid-wide barrier and no extra launches.  Chunk 0 is copied
// through by the consumer warps on the way.
#include "res2net.cuh"

namespace xvb {
template int launch_chain<128>(const Res2Params&, const uint16_t*, const uint16_t*, int64_t, const uint16_t*, const uint16_t*,
                               uint16_t*, uint16_t*, int64_t, int, cudaStream_t);
}  // namespace xvb

using namespace xvb;

extern "C" int xvb_res2net_block_ex(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi,
                                    const uint16_t* w_lo, const float* bias, const float* bn_scale, const float* bn_shift,
                                    int dilation, int scale, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, int B, int T,
                                    int width, void* stream) {
  int rc = require_sm90();
  if (rc) return rc;
  XVB_CHECK_ARG(width == 64 || width == 128, "xvb_res2net_block: the chain kernel is built for widths 64 and 128, got %d", width);
  XVB_CHECK_ARG(x_hi && x_lo && w_hi && w_lo && bias && bn_scale && bn_shift && y_hi && y_lo, "xvb_res2net_block: null pointer");
  XVB_CHECK_ARG(B > 0 && T > 0 && scale >= 2 && scale <= 16 && dilation >= 1, "xvb_res2net_block: bad shape");
  const int C = scale * width;
  XVB_CHECK_ARG(ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C, "xvb_res2net_block: pitches must be >= %d and multiples of 8", C);
  XVB_CHECK_ARG(((uintptr_t)x_hi | (uintptr_t)x_lo | (uintptr_t)y_hi | (uintptr_t)y_lo | (uintptr_t)w_hi | (uintptr_t)w_lo) % 16 == 0,
                "xvb_res2net_block: pointers must be 16-byte aligned");
  XVB_CHECK_ARG(x_hi != y_hi && x_lo != y_lo, "xvb_res2net_block: input and output must be distinct tensors");
  Res2Params p{};
  p.B = B; p.T = T; p.C = C; p.num_steps = scale - 1; p.dilation = dilation; p.num_m = (T + 127) / 128;
  p.bias = bias; p.scale = bn_scale; p.shift = bn_shift;
  p.x_hi = reinterpret_cast<const __nv_bfloat16*>(x_hi); p.x_lo = reinterpret_cast<const __nv_bfloat16*>(x_lo);
  p.y_hi = reinterpret_cast<__nv_bfloat16*>(y_hi); p.y_lo = reinterpret_cast<__nv_bfloat16*>(y_lo);
  p.ldx = ldx; p.ldy = ldy;
  return width == 128 ? launch_chain<128>(p, x_hi, x_lo, ldx, w_hi, w_lo, y_hi, y_lo, ldy, scale, (cudaStream_t)stream)
                      : launch_chain<64>(p, x_hi, x_lo, ldx, w_hi, w_lo, y_hi, y_lo, ldy, scale, (cudaStream_t)stream);
}

extern "C" int xvb_res2net_block(const uint16_t* x_hi, const uint16_t* x_lo, int64_t ldx, const uint16_t* w_hi,
                                 const uint16_t* w_lo, const float* bias, const float* bn_scale, const float* bn_shift,
                                 int dilation, int scale, uint16_t* y_hi, uint16_t* y_lo, int64_t ldy, int B, int T,
                                 void* stream) {
  return xvb_res2net_block_ex(x_hi, x_lo, ldx, w_hi, w_lo, bias, bn_scale, bn_shift, dilation, scale, y_hi, y_lo, ldy, B, T,
                              128, stream);
}
