// be_fm.cu -- FM back end: Demod::FM + Filter 37 taps (Demod.cpp:27-37, DSP.cpp:249-280).
#include "exact.cuh"
#include "params.h"

namespace aisgpu {

__constant__ float c_taps_receiver[37];

// K2-FM': the same FM + FIR37, five outputs (one symbol slot of the 5-phase deinterleaver, DSP.h:65-73) per thread:
// 41 discriminator values are read once into registers and reused by the five 37-tap sums (each still accumulated
// in the reference's order, k = 0..36 from 0.0f).  Besides the filtered samples the kernel emits what the decoders
// actually consume: one sign bit per (row, sampling phase, slot), packed 32 slots per word by warp ballots.
// REAL: the row already holds the discriminator output (ModelDiscriminator, Model.cpp:716-728: RealPart / ImaginaryPart
// straight into Filter 37), stored as floats in the bytes of the complex row, sample m at float 2 * c_new + m.
template <bool REAL>
__global__ void __launch_bounds__(FM5_THREADS) k_fm_fir5(const Fm5Params p) {
	__shared__ float fm[FM5_SAMPLES + FIRF_T - 1 + 3];
	const int row = blockIdx.y, tid = threadIdx.x;
	const int S0 = blockIdx.x * FM5_THREADS;
	const int M0 = 5 * S0 - p.r0; // new-sample index of the first sample of slot S0
	const float2 *c = p.Cbuf + (long long)row * p.c_stride + p.c_new;
	for (int i = tid; i < FM5_SAMPLES + FIRF_T - 1; i += FM5_THREADS) {
		const int m = M0 + i - (FIRF_T - 1);
		float v = 0.0f;
		if (m < p.n && m >= -(FIRF_T - 1) - 4) {
			if (REAL) {
				fm[i] = reinterpret_cast<const float *>(c)[m];
				continue;
			}
			const float2 a = c[m], pv = c[m - 1];
			const float re = __fsub_rn(__fmul_rn(a.x, pv.x), __fmul_rn(a.y, -pv.y));
			const float im = __fadd_rn(__fmul_rn(a.x, -pv.y), __fmul_rn(a.y, pv.x));
			v = __fdiv_rn(fd_atan2f_common(im, re), 3.14159265358979323846f);
			if (p.tap_fm && m >= 0 && i >= FIRF_T - 1) p.tap_fm[(long long)row * p.tap_stride + m] = v;
		}
		fm[i] = v;
	}
	__syncthreads();
	float x[FIRF_T + 4];
#pragma unroll
	for (int i = 0; i < FIRF_T + 4; i++) x[i] = fm[5 * tid + i];
	float y[5];
#pragma unroll
	for (int j = 0; j < 5; j++) {
		float acc = 0.0f;
#pragma unroll
		for (int k = 0; k < FIRF_T; k++) acc = __fadd_rn(acc, __fmul_rn(c_taps_receiver[k], x[j + k]));
		y[j] = acc;
	}
	const int slot = S0 + tid;
	const int m0 = M0 + 5 * tid;
#pragma unroll
	for (int j = 0; j < 5; j++) {
		const int m = m0 + j;
		if (m >= 0 && m < p.n) {
			if (p.Fbuf) p.Fbuf[(long long)row * p.f_stride + p.f_off + m] = y[j];
			if (p.tap_dec) p.tap_dec[(long long)(row * 5 + j) * p.nslots + slot - (j >= p.r0 ? 0 : 1)] = y[j];
		}
		const unsigned w = __ballot_sync(0xffffffffu, y[j] > 0.0f);
		if ((tid & 31) == j && (slot >> 5) < p.dwords) p.dbits[(long long)(row * 5 + j) * p.dwords + (slot >> 5)] = w;
	}
}

// ---- launch entry points ----
cudaError_t fm_init(const float *taps37) { return cudaMemcpyToSymbol(c_taps_receiver, taps37, FIRF_T * sizeof(float)); }
cudaError_t launch_fm_fir5(const Fm5Params &p, int rows, cudaStream_t s) {
	dim3 grid((p.nslots + FM5_THREADS - 1) / FM5_THREADS, rows);
	if (p.real) k_fm_fir5<true><<<grid, FM5_THREADS, 0, s>>>(p);
	else k_fm_fir5<false><<<grid, FM5_THREADS, 0, s>>>(p);
	return cudaGetLastError();
}

} // namespace aisgpu
