// The width-64 instance of the Res2Net chain kernel (res2net.cuh): ECAPA-TDNN C512, scale 8 x 64 channels.
#include "res2net.cuh"

namespace xvb {
template int launch_chain<64>(const Res2Params&, const uint16_t*, const uint16_t*, int64_t, const uint16_t*, const uint16_t*,
                              uint16_t*, uint16_t*, int64_t, int, cudaStream_t);
}  // namespace xvb
