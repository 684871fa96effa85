// fe_stream_f0e.cu -- streaming front end: CF32, 32-sample chunks, ring of 3, four-warp CTAs (104 KB: room for back-end CTAs beside it).
#include "fe_stream.cuh"

namespace aisgpu {

template cudaError_t launch_frontend_stream_shape<0, 32, 3, 4>(const FeParams &, int, bool, int, cudaStream_t);

} // namespace aisgpu
