// tune.cu -- the per-stream digital tune (aisgpu_set_tunings): ConvertRAW of the caller's samples, multiplied by the conjugate of a
// phasor at the stream's offset, into CF32 rows that the rest of the engine reads as a CF32 input.  Each input row feeds T adjacent
// streams, each with its own offset.
//
// The definition (include/aisgpu.h, aisgpu_tune_restate): sample n of a stream (counted from its first sample, across submits) with
// offset f and sample rate fs has the phase index k = ((n mod fs) * f) mod fs in [0, fs); k = a * 4096 + b; p = T_hi[a] * T_lo[b] with
// T_hi[a] = exp(2 pi i a 4096 / fs), T_lo[b] = exp(2 pi i b / fs), computed in double and rounded to float once (tune_tables); the
// output is v * conj(p), every product and sum rounded to float in the order tune_mix writes.  An offset of 0 outputs v itself.
// tune_convert, tune_k and tune_mix are that definition, compiled for the device (k_tune) and the host (aisgpu_tune_restate), so both
// agree bit for bit.
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../include/aisgpu.h"
#include "params.h"

namespace aisgpu {

namespace {

// binary32 operations, each rounded once: intrinsics on the device, plain operators on the host (built with -ffp-contract=off)
#ifdef __CUDA_ARCH__
#define TUNE_MUL(a, b) __fmul_rn(a, b)
#define TUNE_ADD(a, b) __fadd_rn(a, b)
#define TUNE_SUB(a, b) __fsub_rn(a, b)
#else
#define TUNE_MUL(a, b) ((a) * (b))
#define TUNE_ADD(a, b) ((a) + (b))
#define TUNE_SUB(a, b) ((a) - (b))
#endif

__host__ __device__ inline float flip_sign(float x) { // -x as a bit operation: -(+0) is -0, never 0 - x
#ifdef __CUDA_ARCH__
	return __uint_as_float(__float_as_uint(x) ^ 0x80000000u);
#else
	unsigned u;
	memcpy(&u, &x, 4);
	u ^= 0x80000000u;
	memcpy(&x, &u, 4);
	return x;
#endif
}

// ConvertRAW of sample i of a row (Utilities/Convert.cpp:255-301, StreamHelpers.cpp:105-118), which is sample n of its stream:
// F32_FS4's x, jx, -x, -jx pattern is indexed by n
__host__ __device__ inline float2 tune_convert(int fmt, const void *row, long long i, long long n) {
	switch (fmt) {
	case 0: return reinterpret_cast<const float2 *>(row)[i];
	case 1: {
		const uchar2 v = reinterpret_cast<const uchar2 *>(row)[i];
		return make_float2(TUNE_MUL((float)((int)v.x - 128), 0.0078125f), TUNE_MUL((float)((int)v.y - 128), 0.0078125f));
	}
	case 2: {
		const char2 v = reinterpret_cast<const char2 *>(row)[i];
		return make_float2(TUNE_MUL((float)(signed char)v.x, 0.0078125f), TUNE_MUL((float)(signed char)v.y, 0.0078125f));
	}
	case 3: {
		const short2 v = reinterpret_cast<const short2 *>(row)[i];
		return make_float2(TUNE_MUL((float)v.x, 3.0517578125e-05f), TUNE_MUL((float)v.y, 3.0517578125e-05f));
	}
	case FE_FMT_FS4: {
		const float x = reinterpret_cast<const float *>(row)[i];
		const float y = (n & 2) ? flip_sign(x) : x;
		return (n & 1) ? make_float2(0.0f, y) : make_float2(y, 0.0f);
	}
	default: { // DC16H: I and Q the low halves of words 0 and 1, sign-extended; Q negated as an integer (Q = 0 stays +0)
		const unsigned *w = reinterpret_cast<const unsigned *>(row) + 3 * i;
		const int iv = (int)(short)(w[0] & 0xFFFFu), qv = -(int)(short)(w[1] & 0xFFFFu);
		return make_float2(TUNE_MUL((float)iv, 3.0517578125e-05f), TUNE_MUL((float)qv, 3.0517578125e-05f));
	}
	}
}

// the phase index of sample n for an offset whose residue modulo fs is fk (0 <= fk < fs)
__host__ __device__ inline unsigned tune_k(long long n, int fk, int fs) { return (unsigned)((n % fs) * (long long)fk % fs); }

// v * conj(hi * lo)
__host__ __device__ inline float2 tune_mix(float2 v, float2 hi, float2 lo) {
	const float pr = TUNE_SUB(TUNE_MUL(hi.x, lo.x), TUNE_MUL(hi.y, lo.y));
	const float pi = TUNE_ADD(TUNE_MUL(hi.x, lo.y), TUNE_MUL(hi.y, lo.x));
	return make_float2(TUNE_ADD(TUNE_MUL(v.x, pr), TUNE_MUL(v.y, pi)), TUNE_SUB(TUNE_MUL(v.y, pr), TUNE_MUL(v.x, pi)));
}

// tables: T_lo[0 .. 4096) then T_hi[0 .. ceil(fs / 4096)); k = a * 4096 + b reads T_hi[a] = tab[TUNE_LO + a] and T_lo[b] = tab[b]
constexpr int TUNE_LO = 4096;

constexpr int TUNE_THREADS = 256, TUNE_RUN = 8; // a CTA visits TUNE_THREADS * TUNE_RUN samples of one row at a time

// One read of the input and one 8-byte write per sample and tuning.  Each CTA copies the tables into shared memory once and then walks
// work items (input row r, segment of TUNE_THREADS * TUNE_RUN samples); thread t converts samples t, t + 256, ... of the segment once,
// then mixes them by each of the row's T streams rT .. rT + T - 1 in turn and stores them to that stream's row, so every load and store
// is coalesced.  Within a stream k steps by 256 * f mod fs from one sample to the next.
template <int FMT>
__global__ void __launch_bounds__(TUNE_THREADS) k_tune(TuneParams p) {
	extern __shared__ float2 tune_tab[];
	for (int i = threadIdx.x; i < p.tab_len; i += TUNE_THREADS) tune_tab[i] = p.tab[i];
	__syncthreads();
	constexpr int SEG = TUNE_THREADS * TUNE_RUN;
	const int segs = (p.N + SEG - 1) / SEG;
	for (long long w = blockIdx.x; w < (long long)segs * p.R; w += gridDim.x) {
		const int r = (int)(w / segs), i0 = (int)(w % segs) * SEG + threadIdx.x;
		const void *row = reinterpret_cast<const unsigned char *>(p.in) + (long long)r * p.in_stride * fe_fmt_bps(FMT);
		float2 v[TUNE_RUN] = {};
#pragma unroll
		for (int j = 0; j < TUNE_RUN; j++) {
			const int i = i0 + j * TUNE_THREADS;
			if (i < p.N) v[j] = tune_convert(FMT, row, i, p.first + i);
		}
#pragma unroll 1
		for (int s = r * p.T; s < (r + 1) * p.T; s++) {
			const int fk = p.fk[s];
			float2 *out = p.out + (long long)s * p.out_stride + p.out_off;
			if (fk) {
				unsigned k = tune_k(p.first + i0, fk, p.fs);
				const unsigned dk = (unsigned)((long long)TUNE_THREADS * fk % p.fs);
#pragma unroll
				for (int j = 0; j < TUNE_RUN; j++) {
					const int i = i0 + j * TUNE_THREADS;
					if (i < p.N) out[i] = tune_mix(v[j], tune_tab[TUNE_LO + (k >> 12)], tune_tab[k & (TUNE_LO - 1)]);
					k += dk;
					if (k >= (unsigned)p.fs) k -= p.fs;
				}
			}
			else {
#pragma unroll
				for (int j = 0; j < TUNE_RUN; j++) {
					const int i = i0 + j * TUNE_THREADS;
					if (i < p.N) out[i] = v[j];
				}
			}
		}
	}
}

template <int FMT>
cudaError_t launch_tune_f(const TuneParams &p, int ctas, cudaStream_t s) {
	const size_t smem = (size_t)(p.tab_len) * sizeof(float2);
	if (cudaError_t e = cudaFuncSetAttribute(k_tune<FMT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) return e;
	k_tune<FMT><<<ctas, TUNE_THREADS, smem, s>>>(p);
	return cudaGetLastError();
}

} // namespace

int tune_table_len(int fs) { return TUNE_LO + (fs + TUNE_LO - 1) / TUNE_LO; }

void tune_tables(int fs, float2 *tab) {
	const double w = 2.0 * M_PI;
	for (int b = 0; b < TUNE_LO; b++) {
		const double t = w * (double)b / (double)fs;
		tab[b] = make_float2((float)cos(t), (float)sin(t));
	}
	for (int a = 0, n = tune_table_len(fs) - TUNE_LO; a < n; a++) {
		const double t = w * (double)((long long)a * TUNE_LO) / (double)fs;
		tab[TUNE_LO + a] = make_float2((float)cos(t), (float)sin(t));
	}
}

cudaError_t launch_tune(const TuneParams &p, int fmt, int ctas, cudaStream_t s) {
	const int segs = (p.N + TUNE_THREADS * TUNE_RUN - 1) / (TUNE_THREADS * TUNE_RUN);
	ctas = (int)std::min<long long>((long long)segs * p.R, ctas);
	if (ctas < 1) return cudaSuccess;
	switch (fmt) {
	case 0: return launch_tune_f<0>(p, ctas, s);
	case 1: return launch_tune_f<1>(p, ctas, s);
	case 2: return launch_tune_f<2>(p, ctas, s);
	case 3: return launch_tune_f<3>(p, ctas, s);
	case FE_FMT_FS4: return launch_tune_f<FE_FMT_FS4>(p, ctas, s);
	case FE_FMT_DC16H: return launch_tune_f<FE_FMT_DC16H>(p, ctas, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace aisgpu

using namespace aisgpu;

extern "C" int aisgpu_tune_restate(int format, int sample_rate, int32_t offset_hz, int64_t first_sample, const void *in, int64_t n, void *out_cf32) {
	const bool known = (format >= AISGPU_FMT_CF32 && format <= AISGPU_FMT_F32_FS4) || format == AISGPU_FMT_DC16H;
	if (!known || sample_rate < 1 || first_sample < 0 || n < 0 || (n > 0 && (!in || !out_cf32)) ||
		!((long long)offset_hz * 2 > -(long long)sample_rate && (long long)offset_hz * 2 < (long long)sample_rate))
		return AISGPU_EINVAL;
	const int fmt = fe_fmt_id(format), fs = sample_rate;
	const int fk = offset_hz < 0 ? offset_hz + fs : offset_hz;
	std::vector<float2> tab(tune_table_len(fs));
	tune_tables(fs, tab.data());
	float2 *out = static_cast<float2 *>(out_cf32);
	for (long long i = 0; i < n; i++) {
		const long long m = first_sample + i;
		float2 v = tune_convert(fmt, in, i, m);
		if (fk) {
			const unsigned k = tune_k(m, fk, fs);
			v = tune_mix(v, tab[TUNE_LO + (k >> 12)], tab[k & (TUNE_LO - 1)]);
		}
		out[i] = v;
	}
	return 0;
}
