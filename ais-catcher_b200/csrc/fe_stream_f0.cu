// fe_stream_f0.cu -- streaming front end: the dispatch to each format's launch shape (one translation unit per shape, see
// fe_stream.cuh, keeps the build parallel) and the lane planner's test hook.
#include "fe_stream.cuh"

namespace aisgpu {

cudaError_t launch_frontend_stream(const FeParams &p, int fmt, int k, bool pre, int forced_L, cudaStream_t s) {
	switch (fmt) {
	// 32-sample visits, four-warp CTAs: the kernel is bound by what DRAM delivers for 32768 concurrent sequential streams, and
	// more resident warps never helped among the shapes measured on the previous target (16 / 32 / 64 samples per visit; one-,
	// two- and four-warp CTAs; rings of 2 .. 8 chunks with one to eight CTAs sharing an SM).  A ring of 3 (104 KB per CTA instead
	// of 174 KB for 5) lets the coherent chains' back-end CTAs (the FFT estimate alone takes 67 KB) fit on the SM beside the front
	// end's.  In front of the resampler it was faster than one-warp CTAs with 16-sample chunks at 6 MSPS.
	case 0: return launch_frontend_stream_shape<0, 32, 3, 4>(p, k, pre, forced_L, s);
	case 1: return launch_frontend_stream_shape<1, 16, 8, 1>(p, k, pre, forced_L, s);
	case 2: return launch_frontend_stream_shape<2, 16, 8, 1>(p, k, pre, forced_L, s);
	case 3: return launch_frontend_stream_shape<3, 16, 8, 1>(p, k, pre, forced_L, s);
	case FE_FMT_FS4: return launch_frontend_stream_shape<FE_FMT_FS4, 16, 8, 1>(p, k, pre, forced_L, s); // CS16's bytes per sample: CS16's shape (the CF32 shape was not measured for it)
	// 12 bytes per sample: CS16's chunk length, ring depth and one-warp CTAs (the one shape measured); its ring is 52 KB per CTA
	case FE_FMT_DC16H: return launch_frontend_stream_shape<FE_FMT_DC16H, 16, 8, 1>(p, k, pre, forced_L, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace aisgpu

// Test hook (not part of include/aisgpu.h): the lane planner of the streaming front end as the launcher calls it, so that the CPU
// suite can check its invariants without a device.  Returns 0 when the block is too short for the streaming kernel.
extern "C" int aisgpu_dbg_plan_lanes(long long n_streams, int super_steps, int warm_super_steps, int warps_per_cta, int cta_slots, int min_ratio, int forced_lanes,
									 int *lanes, int *q, int *r) {
	return aisgpu::st_plan(n_streams, super_steps, warm_super_steps, warps_per_cta, cta_slots, min_ratio, forced_lanes, *lanes, *q, *r) ? 1 : 0;
}
