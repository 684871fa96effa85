// exact.cuh -- exact-rounding arithmetic helpers shared by every kernel of the AIS demodulation hot path.
//
// Every kernel reproduces the IEEE binary32 operation order of the reference block it replaces (file:line cited per
// kernel, relative to /root/reference/Source) so that results are bit-identical: all arithmetic goes through
// __fadd_rn/__fsub_rn/__fmul_rn/__fdiv_rn (never contracted to FMA), std::abs of a complex is evaluated as glibc's
// hypotf does, libm-dependent constants (twiddles, phasor steps) come from host tables, and atan2f is the fdlibm
// algorithm glibc 2.39 ships.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// exact arithmetic helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(__fmul_rn(a.x, s), __fmul_rn(a.y, s)); }
// std::complex<float> product (ac-bd, ad+bc), every product and sum rounded separately
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
	return make_float2(__fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x)));
}
// std::abs(std::complex<float>) == cabsf == glibc 2.39 hypotf for finite inputs (checked on 5e7 patterns, see DESIGN.md)
__device__ __forceinline__ float habs(float2 a) {
	double x = (double)a.x, y = (double)a.y;
	return __double2float_rn(__dsqrt_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y))));
}
__device__ __forceinline__ float2 cnormalize(float2 r) { // rot /= std::abs(rot)
	float a = habs(r);
	return make_float2(__fdiv_rn(r.x, a), __fdiv_rn(r.y, a));
}

// fdlibm atanf/atan2f (the algorithm behind glibc 2.39 __ieee754_atan2f; verified bit-identical on 5e7 inputs)
__device__ __forceinline__ float fd_atanf(float x) {
	const float aT[11] = { 3.3333334327e-01f, -2.0000000298e-01f, 1.4285714924e-01f, -1.1111110449e-01f, 9.0908870101e-02f,
						   -7.6918758452e-02f, 6.6610731184e-02f, -5.8335702866e-02f, 4.9768779427e-02f, -3.6531571299e-02f, 1.6285819933e-02f };
	const int hx = __float_as_int(x), ix = hx & 0x7fffffff;
	if (ix >= 0x4c000000) { // |x| >= 2^25 (rare)
		if (ix > 0x7f800000) return __fadd_rn(x, x);
		const float r = __fadd_rn(1.5707962513e+00f, 7.5497894159e-08f);
		return hx > 0 ? r : -r;
	}
	if (ix < 0x31000000) return x; // |x| < 2^-29 (rare)
	// The four argument reductions of fdlibm are evaluated side by side and selected, so a warp does not serialise
	// over them; the operations on the selected path are exactly the library's.
	const bool small = ix < 0x3ee00000; // |x| < 0.4375: no reduction, x keeps its sign
	const float ax = fabsf(x);
	const int id = ix < 0x3f300000 ? 0 : (ix < 0x3f980000 ? 1 : (ix < 0x401c0000 ? 2 : 3));
	const float n0 = __fsub_rn(__fmul_rn(2.0f, ax), 1.0f), d0 = __fadd_rn(2.0f, ax);
	const float n1 = __fsub_rn(ax, 1.0f), d1 = __fadd_rn(ax, 1.0f);
	const float n2 = __fsub_rn(ax, 1.5f), d2 = __fadd_rn(1.0f, __fmul_rn(1.5f, ax));
	const float num = id == 0 ? n0 : (id == 1 ? n1 : (id == 2 ? n2 : -1.0f));
	const float den = id == 0 ? d0 : (id == 1 ? d1 : (id == 2 ? d2 : ax));
	const float hi = id == 0 ? 4.6364760399e-01f : (id == 1 ? 7.8539812565e-01f : (id == 2 ? 9.8279368877e-01f : 1.5707962513e+00f));
	const float lo = id == 0 ? 5.0121582440e-09f : (id == 1 ? 3.7748947079e-08f : (id == 2 ? 3.4473217170e-08f : 7.5497894159e-08f));
	const float xr = small ? x : __fdiv_rn(num, den);
	const float z = __fmul_rn(xr, xr), w = __fmul_rn(z, z);
	const float s1 = __fmul_rn(z, __fadd_rn(aT[0], __fmul_rn(w, __fadd_rn(aT[2], __fmul_rn(w, __fadd_rn(aT[4], __fmul_rn(w, __fadd_rn(aT[6], __fmul_rn(w, __fadd_rn(aT[8], __fmul_rn(w, aT[10])))))))))));
	const float s2 = __fmul_rn(w, __fadd_rn(aT[1], __fmul_rn(w, __fadd_rn(aT[3], __fmul_rn(w, __fadd_rn(aT[5], __fmul_rn(w, __fadd_rn(aT[7], __fmul_rn(w, aT[9])))))))));
	const float xs = __fmul_rn(xr, __fadd_rn(s1, s2));
	if (small) return __fsub_rn(xr, xs);
	const float r = __fsub_rn(hi, __fsub_rn(__fsub_rn(xs, lo), xr));
	return hx < 0 ? -r : r;
}
__device__ __forceinline__ float fd_atan2f(float y, float x) {
	const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f;
	int hx = __float_as_int(x), ix = hx & 0x7fffffff, hy = __float_as_int(y), iy = hy & 0x7fffffff;
	if (ix > 0x7f800000 || iy > 0x7f800000) return __fadd_rn(x, y);
	if (hx == 0x3f800000) return fd_atanf(y);
	int m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
	if (iy == 0) {
		switch (m) {
		case 0: case 1: return y;
		case 2: return __fadd_rn(pi, tiny);
		default: return __fsub_rn(-pi, tiny);
		}
	}
	if (ix == 0) return hy < 0 ? __fsub_rn(-pi_o_2, tiny) : __fadd_rn(pi_o_2, tiny);
	if (ix == 0x7f800000) {
		if (iy == 0x7f800000) {
			switch (m) {
			case 0: return __fadd_rn(pi_o_4, tiny);
			case 1: return __fsub_rn(-pi_o_4, tiny);
			case 2: return __fadd_rn(__fmul_rn(3.0f, pi_o_4), tiny);
			default: return __fsub_rn(__fmul_rn(-3.0f, pi_o_4), tiny);
			}
		}
		else {
			switch (m) {
			case 0: return 0.0f;
			case 1: return -0.0f;
			case 2: return __fadd_rn(pi, tiny);
			default: return __fsub_rn(-pi, tiny);
			}
		}
	}
	if (iy == 0x7f800000) return hy < 0 ? __fsub_rn(-pi_o_2, tiny) : __fadd_rn(pi_o_2, tiny);
	int k = (iy - ix) >> 23;
	float z;
	if (k > 60) z = __fadd_rn(pi_o_2, __fmul_rn(0.5f, pi_lo));
	else if (hx < 0 && k < -60) z = 0.0f;
	else z = fd_atanf(fabsf(__fdiv_rn(y, x)));
	switch (m) {
	case 0: return z;
	case 1: return __int_as_float(__float_as_int(z) ^ 0x80000000);
	case 2: return __fsub_rn(pi, __fsub_rn(z, pi_lo));
	default: return __fsub_rn(__fsub_rn(z, pi_lo), pi);
	}
}

// fd_atan2f for the discriminators (one call per 48 kHz sample and channel): the same results, with the library's chain of
// rare-case tests (NaN, zeros, infinities, |y/x| outside 2^-29 .. 2^25, x == 1) replaced by ONE range test in front of a
// straight-line common path -- both operands normal and their exponents at most 28 / 23 apart; everything else takes
// fd_atan2f.  On the common path |y/x| lies in [2^-28, 2^24), so atanf needs no special cases; its four argument reductions
// share one division (num / den selected, x / 1 for the unreduced range), "x - x*s" is written as "0 - ((x*s - 0) - x)"
// (identical in binary32) so that both ranges share the final expression, and pi - (z - pi_lo) is taken as the exact negation
// of (z - pi_lo) - pi.  tests/host/atan2_check.c holds the same formulation in C: 1.4e8 arguments on this path against the C
// library, 0 mismatches; the FM taps of the parity tests check the transcription.
static __device__ __noinline__ float fd_atan2f_rare(float y, float x) { return fd_atan2f(y, x); } // out of line: keeps the callers' loops short
__device__ __forceinline__ float fd_atan2f_common(float y, float x) {
	const uint32_t hx = __float_as_uint(x), hy = __float_as_uint(y), ix = hx & 0x7fffffffu, iy = hy & 0x7fffffffu;
	const int k = ((int)iy - (int)ix) >> 23;
	if (!((ix - 0x00800000u) < 0x7f000000u && (iy - 0x00800000u) < 0x7f000000u && (uint32_t)(k + 28) <= 51u && hx != 0x3f800000u)) return fd_atan2f_rare(y, x);
	const float t = fabsf(__fdiv_rn(y, x));
	const uint32_t it = __float_as_uint(t);
	const bool small = it < 0x3ee00000u, c0 = it < 0x3f300000u, c1 = it < 0x3f980000u, c2 = it < 0x401c0000u;
	const float a = c0 ? __fmul_rn(2.0f, t) : t;
	const float nm = __fsub_rn(a, c1 ? 1.0f : 1.5f);
	const float b = (c2 && !c1) ? __fmul_rn(1.5f, t) : t;
	const float dn = __fadd_rn(b, c0 ? 2.0f : 1.0f);
	const float num = small ? t : (c2 ? nm : -1.0f);
	const float den = small ? 1.0f : (c2 ? dn : t);
	const float hi = small ? 0.0f : (c0 ? 4.6364760399e-01f : (c1 ? 7.8539812565e-01f : (c2 ? 9.8279368877e-01f : 1.5707962513e+00f)));
	const float lo = small ? 0.0f : (c0 ? 5.0121582440e-09f : (c1 ? 3.7748947079e-08f : (c2 ? 3.4473217170e-08f : 7.5497894159e-08f)));
	const float xr = __fdiv_rn(num, den);
	const float z = __fmul_rn(xr, xr), w = __fmul_rn(z, z);
	const float s1 = __fmul_rn(z, __fadd_rn(3.3333334327e-01f, __fmul_rn(w, __fadd_rn(1.4285714924e-01f, __fmul_rn(w, __fadd_rn(9.0908870101e-02f,
					 __fmul_rn(w, __fadd_rn(6.6610731184e-02f, __fmul_rn(w, __fadd_rn(4.9768779427e-02f, __fmul_rn(w, 1.6285819933e-02f)))))))))));
	const float s2 = __fmul_rn(w, __fadd_rn(-2.0000000298e-01f, __fmul_rn(w, __fadd_rn(-1.1111110449e-01f, __fmul_rn(w, __fadd_rn(-7.6918758452e-02f,
					 __fmul_rn(w, __fadd_rn(-5.8335702866e-02f, __fmul_rn(w, -3.6531571299e-02f)))))))));
	const float xs = __fmul_rn(xr, __fadd_rn(s1, s2));
	const float zz = __fsub_rn(hi, __fsub_rn(__fsub_rn(xs, lo), xr));
	if ((int)hx >= 0) return __uint_as_float(__float_as_uint(zz) | (hy & 0x80000000u));
	const float v = __fsub_rn(__fsub_rn(zz, -8.7422776573e-08f), 3.1415927410e+00f);
	return __uint_as_float(__float_as_uint(v) ^ (~hy & 0x80000000u));
}

// ---- binary32 pairs: a complex sample is one 64-bit register pair.  sm_90 has no packed FP32 instruction, so a pair
// ---- operation is two scalar __fadd_rn / __fmul_rn (each lane rounded on its own; never contracted into an FMA).
typedef unsigned long long c64;
__device__ __forceinline__ float2 unpack2(c64 v);
__device__ __forceinline__ c64 pack2(float x, float y);
__device__ __forceinline__ c64 padd(c64 a, c64 b) {
	const float2 x = unpack2(a), y = unpack2(b);
	return pack2(__fadd_rn(x.x, y.x), __fadd_rn(x.y, y.y));
}
__device__ __forceinline__ c64 pmul(c64 a, c64 b) {
	const float2 x = unpack2(a), y = unpack2(b);
	return pack2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ c64 pack2(float x, float y) {
	c64 r;
	asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(x), "f"(y));
	return r;
}
__device__ __forceinline__ float2 unpack2(c64 v) {
	float2 r;
	asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(v));
	return r;
}

__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }
__device__ __forceinline__ void cp_async16(void *smem_dst, const void *gsrc) {
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_f(float *smem_dst, const float *gsrc) {
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}
__device__ __forceinline__ void cp_async_f(float2 *smem_dst, const float2 *gsrc) {
	asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc));
}

} // namespace aisgpu
