// fe_disc.cu -- front end of the FM-discriminator input model (-m 3, reference ModelDiscriminator, Model.cpp:702-754).  A stereo
// recording of two discriminator outputs is read as I/Q; ConvertRAW's scaling (Convert.cpp:255-286), then RealPart feeds channel
// A's Filter 37 and ImaginaryPart channel B's (StreamHelpers.cpp:25-49).  So the front end is a conversion and a split: I goes to
// Cbuf row 2 * stream, Q to row 2 * stream + 1, as real 48 kHz samples (sample i at float 2 * c_off + i of the row).  Rates below
// 48 kHz reach this kernel as CF32 blocks of the DSP::Upsample ring (aisgpu.cu, pre-stage 1 with no CIC stage in front).
//
// Shape: nothing is recurrent, so one CTA converts one contiguous segment of one stream.  Each thread loads DISC_PAIRS pairs of
// samples (warp-contiguous) before it stores any, and writes one float2 per pair to each row: every row is written as contiguous
// 256-byte warp stores.  Pairs are read with one vector load where the batch's rows allow it (CF32 16 bytes, CS16 and F32_FS4 8, CU8/CS8 4);
// a DC16H pair is read as its four live words wherever it lies.
#include "fe_common.cuh"
#include "params.h"

namespace aisgpu {

namespace {

constexpr int DISC_THREADS = 256;
constexpr int DISC_PAIRS = 4;                          // sample pairs per thread
constexpr int DISC_SEG = 2 * DISC_PAIRS * DISC_THREADS; // samples per CTA

template <int FMT, bool VEC>
__global__ void __launch_bounds__(DISC_THREADS) k_frontend_disc(const FeParams p, int nseg) {
	const int stream = blockIdx.x / nseg, seg = blockIdx.x - stream * nseg;
	const long long in0 = (long long)stream * p.in_stride;
	float *ra = reinterpret_cast<float *>(p.C + (long long)(2 * stream) * p.c_stride) + 2 * p.c_off;
	float *rb = reinterpret_cast<float *>(p.C + (long long)(2 * stream + 1) * p.c_stride) + 2 * p.c_off;
	float2 a[DISC_PAIRS], b[DISC_PAIRS];
#pragma unroll
	for (int u = 0; u < DISC_PAIRS; u++) {
		const int i = seg * DISC_SEG + 2 * (u * DISC_THREADS + threadIdx.x);
		if (i < p.N) {
			if (VEC) fe_load_pair<FMT>(p.in, in0 + i, i, a[u], b[u]);
			else {
				a[u] = fe_load_one<FMT>(p.in, in0 + i, i);
				b[u] = fe_load_one<FMT>(p.in, in0 + i + 1, i + 1);
			}
		}
	}
#pragma unroll
	for (int u = 0; u < DISC_PAIRS; u++) {
		const int i = seg * DISC_SEG + 2 * (u * DISC_THREADS + threadIdx.x);
		if (i < p.N) {
			*reinterpret_cast<float2 *>(ra + i) = make_float2(a[u].x, b[u].x);
			*reinterpret_cast<float2 *>(rb + i) = make_float2(a[u].y, b[u].y);
		}
	}
}

template <int FMT>
cudaError_t launch_disc_fmt(const FeParams &p, cudaStream_t s) {
	constexpr int BPS = fe_fmt_bps(FMT);
	if (p.N <= 0 || (p.N & 1)) return cudaErrorInvalidValue;
	const int nseg = (p.N + DISC_SEG - 1) / DISC_SEG;
	const unsigned ctas = (unsigned)((long long)p.st_B * nseg);
	// a pair starts at an even sample: one vector load when the batch and its rows are aligned to two samples
	const bool vec = FMT == FE_FMT_DC16H || (((size_t)p.in % (2 * BPS)) == 0 && ((p.in_stride * BPS) % (2 * BPS)) == 0);
	if (vec) k_frontend_disc<FMT, true><<<ctas, DISC_THREADS, 0, s>>>(p, nseg);
	else k_frontend_disc<FMT, false><<<ctas, DISC_THREADS, 0, s>>>(p, nseg);
	return cudaGetLastError();
}

} // namespace

cudaError_t launch_frontend_disc(const FeParams &p, int fmt, cudaStream_t s) {
	switch (fmt) {
	case 0: return launch_disc_fmt<0>(p, s);
	case 1: return launch_disc_fmt<1>(p, s);
	case 2: return launch_disc_fmt<2>(p, s);
	case 3: return launch_disc_fmt<3>(p, s);
	case FE_FMT_FS4: return launch_disc_fmt<FE_FMT_FS4>(p, s);
	case FE_FMT_DC16H: return launch_disc_fmt<FE_FMT_DC16H>(p, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace aisgpu
