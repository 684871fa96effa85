// fe_misc.cu -- small front-end kernels: Rotate phasor table, Upsample, DownsampleKFilter, history carries.
#include <algorithm>

#include "exact.cuh"
#include "params.h"
#include "fe_common.cuh"

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// K0: Rotate phasor table (DSP/DSP.cpp:296-316: rot *= mult per 96 kHz sample, rot /= |rot| once per call)
// The phasor depends only on the sequence of chunk lengths, never on the data, so one table per submit serves
// every stream of the batch.  tab[P96 + i] is the phasor that multiplies 96 kHz sample i of this submit;
// tab[0..P96) repeats the last P96 phasors of the previous submit (warm-up history of the front end).
// ---------------------------------------------------------------------------------------------
__global__ void k_rot_table(float2 *__restrict__ tab, const float2 *__restrict__ prev_tail, const float2 *__restrict__ state_in,
							float2 *__restrict__ state_out, float2 mult, int P96, int n96) {
	if (blockIdx.x != 0) return;
	for (int i = threadIdx.x; i < P96; i += blockDim.x) tab[i] = prev_tail ? prev_tail[i] : make_float2(1.0f, 0.0f);
	if (threadIdx.x != 0) return;
	float2 rot = *state_in;
	float2 *o = tab + P96;
	for (int i = 0; i < n96; i++) {
		o[i] = rot;
		rot = cmul(rot, mult);
	}
	*state_out = cnormalize(rot);
}

// ---------------------------------------------------------------------------------------------
// DSP::Upsample (DSP.cpp:192-212): out = (1 - alpha) * a + alpha * b with a, b consecutive inputs.  alpha is a float
// accumulator that only depends on how many samples have gone by, so the host replays it (same binary32 adds) and
// hands the kernel one (input index, alpha) pair per output; outputs land in a ring of whole reference blocks.
// ---------------------------------------------------------------------------------------------
__global__ void k_upsample(const float2 *__restrict__ D0, long long d0_stride, int d0_off, const int *__restrict__ src, const float *__restrict__ alpha,
						   int M, float2 *__restrict__ S, long long s_stride, long long m0, int cap) {
	const int m = blockIdx.x * blockDim.x + threadIdx.x;
	if (m >= M) return;
	const float2 *d = D0 + (long long)blockIdx.y * d0_stride + d0_off;
	const int i = src[m];
	const float al = alpha[m];
	const float2 a = d[i - 1], b = d[i];
	const float w = __fsub_rn(1.0f, al);
	float2 o;
	o.x = __fadd_rn(__fmul_rn(w, a.x), __fmul_rn(al, b.x));
	o.y = __fadd_rn(__fmul_rn(w, a.y), __fmul_rn(al, b.y));
	S[(long long)blockIdx.y * s_stride + (int)((m0 + m) % cap)] = o;
}

// DSP::DownsampleKFilter with Filters::BlackmanHarris_28_3, K = 3 (DSP.cpp:160-189, Filters.h:43-53; the 288 kS/s
// front end, Model.cpp:308-313): out[j] = sum_k taps[k] * x[n_j - 25 + k], n_j = first + 3 j, accumulated from 0 in
// ascending k.  Input: the submit's samples, negative indices from the previous submit's tail.
__constant__ float c_taps_bh28_3[DSK_T];
template <int FMT>
__global__ void __launch_bounds__(DSK_THREADS) k_dsk(const void *__restrict__ in, long long in_stride, const void *__restrict__ tail, int tail_len, int first,
													  int n_out, float2 *__restrict__ S, long long s_stride, long long j0, int cap) {
	__shared__ float2 x[3 * DSK_THREADS + DSK_T];
	const int stream = blockIdx.y, tid = threadIdx.x;
	const int o0 = blockIdx.x * DSK_THREADS;             // first output of this CTA
	const int lo = first + 3 * o0 - (DSK_T - 1);         // input index of x[0], relative to the submit
	for (int i = tid; i < 3 * DSK_THREADS + DSK_T; i += DSK_THREADS) {
		const int n = lo + i;
		float2 v = make_float2(0.f, 0.f);
		if (n < 0) {
			if (n >= -tail_len) v = fe_load_one<FMT>(tail, (long long)stream * tail_len + tail_len + n);
		}
		else if (n <= first + 3 * (n_out - 1)) v = fe_load_one<FMT>(in, (long long)stream * in_stride + n);
		x[i] = v;
	}
	__syncthreads();
	const int o = o0 + tid;
	if (o >= n_out) return;
	float2 acc = make_float2(0.f, 0.f);
#pragma unroll
	for (int k = 0; k < DSK_T; k++) {
		const float2 dd = x[3 * tid + k];
		acc.x = __fadd_rn(acc.x, __fmul_rn(c_taps_bh28_3[k], dd.x));
		acc.y = __fadd_rn(acc.y, __fmul_rn(c_taps_bh28_3[k], dd.y));
	}
	S[(long long)stream * s_stride + (int)((j0 + o) % cap)] = acc;
}

// new_tail = last P samples of (old_tail ++ chunk); works for any N.  Copies words of sizeof(W) bytes: the launcher picks the
// widest word that divides the input's base, its row stride, N and P in bytes.  A device batch's row stride is any even number of
// samples (aisgpu_check_device_batch), which for CU8 / CS8 is a multiple of 4 bytes but not always of 8.
template <typename W>
__global__ void k_tail_update(W *__restrict__ new_tail, const W *__restrict__ old_tail, const unsigned char *__restrict__ in,
							  long long in_stride_b, long long n_w, int p_w) {
	const int stream = blockIdx.y;
	const W *row = reinterpret_cast<const W *>(in + (long long)stream * in_stride_b);
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p_w; i += gridDim.x * blockDim.x) {
		const long long s = (long long)i + n_w - p_w; // word index relative to chunk start
		new_tail[(long long)stream * p_w + i] = s >= 0 ? row[s] : old_tail[(long long)stream * p_w + (s + p_w)];
	}
}

// ---------------------------------------------------------------------------------------------
// small utility: move `cnt` trailing elements of each row to the slot just before `dst_end`
// (keeps unconsumed samples / filter history in front of the next submit's data)
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void k_carry(T *__restrict__ buf, long long stride, int src_begin, int dst_begin, int cnt) {
	extern __shared__ __align__(16) unsigned char carry_sm[];
	T *tmp = reinterpret_cast<T *>(carry_sm);
	T *row = buf + (long long)blockIdx.x * stride;
	for (int i = threadIdx.x; i < cnt; i += blockDim.x) tmp[i] = row[src_begin + i];
	__syncthreads();
	for (int i = threadIdx.x; i < cnt; i += blockDim.x) row[dst_begin + i] = tmp[i];
}

// copy `cnt` elements of each row from one buffer to another (unconsumed samples / filter history handed to the
// buffer the next submit's front end writes into)
template <typename T>
__global__ void k_carry2(const T *__restrict__ src, T *__restrict__ dst, long long stride, int src_begin, int dst_begin, int cnt) {
	const T *srow = src + (long long)blockIdx.x * stride + src_begin;
	T *drow = dst + (long long)blockIdx.x * stride + dst_begin;
	for (int i = threadIdx.x; i < cnt; i += blockDim.x) drow[i] = srow[i];
}

// One read of n new 48 kHz samples per row, written to up to GROUP_MAX - 1 destinations at a stride and offset of their own:
//  - engine groups: the leader's rows into every member's own ring, at the Cbuf stride and HC (aisgpu.cu, fan_out);
//  - the channel dump: the rows of one inner submit into columns [off, off + n) of the submit's compact export slot (dump_export).
// 16-byte loads and stores: strides, offsets and length are whole float4s.  The destination pointers are unrolled so that they stay
// in the parameter bank.
struct FanoutArgs {
	const float4 *src;
	float4 *dst[GROUP_MAX - 1];
	long long src_stride4, dst_stride4;
	int src_off4, dst_off4, n4, rows, nd;
};
__global__ void __launch_bounds__(256) k_c_fanout(const FanoutArgs a) {
	for (int r = blockIdx.y; r < a.rows; r += gridDim.y) {
		const long long srow = (long long)r * a.src_stride4 + a.src_off4, drow = (long long)r * a.dst_stride4 + a.dst_off4;
		for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < a.n4; j += gridDim.x * blockDim.x) {
			const float4 v = a.src[srow + j];
#pragma unroll
			for (int m = 0; m < GROUP_MAX - 1; m++)
				if (m < a.nd) a.dst[m][drow + j] = v;
		}
	}
}

__global__ void k_d0_carry(float2 *__restrict__ D0, long long d0_stride, int d0_off, int L, int rows) {
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r < rows) D0[(long long)r * d0_stride + d0_off - 1] = D0[(long long)r * d0_stride + d0_off + L - 1]; // Upsample::a = b
}

// ---- launch entry points ----
cudaError_t launch_rot_table(float2 *tab, const float2 *prev_tail, const float2 *state_in, float2 *state_out, float2 mult, int P96, int n96, cudaStream_t s) {
	k_rot_table<<<1, 32, 0, s>>>(tab, prev_tail, state_in, state_out, mult, P96, n96);
	return cudaGetLastError();
}
cudaError_t launch_upsample(const float2 *D0, long long d0_stride, int d0_off, const int *src, const float *alpha, int M, int B, float2 *S, long long s_stride,
							long long m0, int cap, cudaStream_t s) {
	k_upsample<<<dim3((M + 255) / 256, B), 256, 0, s>>>(D0, d0_stride, d0_off, src, alpha, M, S, s_stride, m0, cap);
	return cudaGetLastError();
}
cudaError_t launch_d0_carry(float2 *D0, long long d0_stride, int d0_off, int L, int rows, cudaStream_t s) {
	k_d0_carry<<<(rows + 127) / 128, 128, 0, s>>>(D0, d0_stride, d0_off, L, rows);
	return cudaGetLastError();
}
cudaError_t launch_dsk(int fmt, const void *in, long long in_stride, const void *tail, int tail_len, int first, int n_out, int B, float2 *S, long long s_stride,
					   long long j0, int cap, cudaStream_t s) {
	dim3 grid((n_out + DSK_THREADS - 1) / DSK_THREADS, B);
	switch (fmt) {
	case 0: k_dsk<0><<<grid, DSK_THREADS, 0, s>>>(in, in_stride, tail, tail_len, first, n_out, S, s_stride, j0, cap); break;
	case 1: k_dsk<1><<<grid, DSK_THREADS, 0, s>>>(in, in_stride, tail, tail_len, first, n_out, S, s_stride, j0, cap); break;
	case 2: k_dsk<2><<<grid, DSK_THREADS, 0, s>>>(in, in_stride, tail, tail_len, first, n_out, S, s_stride, j0, cap); break;
	default: k_dsk<3><<<grid, DSK_THREADS, 0, s>>>(in, in_stride, tail, tail_len, first, n_out, S, s_stride, j0, cap); break;
	}
	return cudaGetLastError();
}
template <typename W>
static cudaError_t tail_update_w(void *new_tail, const void *old_tail, const void *in, long long in_stride_b, long long n_b, int p_b, int B, cudaStream_t s) {
	const int p_w = p_b / (int)sizeof(W);
	dim3 grid((p_w + 127) / 128, B);
	k_tail_update<W><<<grid, 128, 0, s>>>((W *)new_tail, (const W *)old_tail, (const unsigned char *)in, in_stride_b, n_b / (long long)sizeof(W), p_w);
	return cudaGetLastError();
}
cudaError_t launch_tail_update(void *new_tail, const void *old_tail, const void *in, long long in_stride_b, long long n_b, int p_b, int B, cudaStream_t s) {
	const unsigned long long m = (unsigned long long)(size_t)in | (unsigned long long)in_stride_b | (unsigned long long)n_b | (unsigned long long)p_b;
	if (m % 8 == 0) return tail_update_w<uint2>(new_tail, old_tail, in, in_stride_b, n_b, p_b, B, s);
	if (m % 4 == 0) return tail_update_w<unsigned>(new_tail, old_tail, in, in_stride_b, n_b, p_b, B, s);
	if (m % 2 == 0) return tail_update_w<unsigned short>(new_tail, old_tail, in, in_stride_b, n_b, p_b, B, s);
	return tail_update_w<unsigned char>(new_tail, old_tail, in, in_stride_b, n_b, p_b, B, s);
}
cudaError_t launch_carry_f2(float2 *buf, long long stride, int src_begin, int dst_begin, int cnt, int rows, cudaStream_t s) {
	k_carry<float2><<<rows, 128, cnt * sizeof(float2), s>>>(buf, stride, src_begin, dst_begin, cnt);
	return cudaGetLastError();
}
cudaError_t launch_carry2_f2(const float2 *src, float2 *dst, long long stride, int src_begin, int dst_begin, int cnt, int rows, cudaStream_t s) {
	k_carry2<float2><<<rows, 128, 0, s>>>(src, dst, stride, src_begin, dst_begin, cnt);
	return cudaGetLastError();
}
cudaError_t launch_c_fanout(const float2 *src, long long src_stride, int src_off, float2 *const *dst, int nd, long long dst_stride, int dst_off, int n,
							int rows, cudaStream_t s) {
	if (nd < 1 || nd > GROUP_MAX - 1 || (src_stride | dst_stride | src_off | dst_off | n) & 1) return cudaErrorInvalidValue;
	FanoutArgs a;
	a.src = reinterpret_cast<const float4 *>(src);
	for (int m = 0; m < GROUP_MAX - 1; m++) a.dst[m] = m < nd ? reinterpret_cast<float4 *>(dst[m]) : nullptr;
	a.src_stride4 = src_stride / 2;
	a.dst_stride4 = dst_stride / 2;
	a.src_off4 = src_off / 2;
	a.dst_off4 = dst_off / 2;
	a.n4 = n / 2;
	a.rows = rows;
	a.nd = nd;
	if (a.n4 == 0) return cudaSuccess;
	const dim3 grid((a.n4 + 255) / 256, std::min(rows, 65535));
	k_c_fanout<<<grid, 256, 0, s>>>(a);
	return cudaGetLastError();
}
cudaError_t set_taps_bh28_3(const float *taps26) { return cudaMemcpyToSymbol(c_taps_bh28_3, taps26, DSK_T * sizeof(float)); }

} // namespace aisgpu
