// fe_stream_dc16h.cu -- streaming front end: DC16H (three 32-bit words per sample, Convert.cpp:288-301).  CS16's launch shape
// (16-sample chunks, a ring of 8, one-warp CTAs); a lane's chunk is 192 bytes, staged as three 64-byte thirds (StFmt), and a staged
// pair is read out of its 48-byte quad (st_read_pair).
#include "fe_stream.cuh"

namespace aisgpu {

template cudaError_t launch_frontend_stream_shape<FE_FMT_DC16H, 16, 8, 1>(const FeParams &, int, bool, int, cudaStream_t);

} // namespace aisgpu
