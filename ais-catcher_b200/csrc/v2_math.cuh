// v2_math.cuh -- the two libm-level functions of the V2 engine (be_v2.cu), in a header of their own so that
// tests/host/exact_math_check.cu can evaluate them on the device and compare them with the host library.
#pragma once
#include <cuda_runtime.h>

namespace aisgpu {

// glibc 2.39 sincosf (sysdeps/ieee754/flt-32/s_sincosf.c): |y| < pi/4 -> polynomial on y, |y| < 120 -> reduce_fast (quadrant
// from a scaled float->int conversion), double arithmetic throughout, results rounded to float once.
// Domain: the engine's two callers stay inside [-1.27, 2 pi).  derotate takes theta = 2 pi f with |f| <= 206 / 1024 (f of
// FreqOffset::Estimate: (256 - (fz + frac + 51)) / 2 / 512 with fz in [-1, 409] and |frac| <= 1/2), learnSlotPhase takes
// theta = (slot offset in [0, 1280)) * 2 pi / 1280.  Only that domain is restated: neither the large-argument reduction
// (|y| >= 120) nor the non-finite returns of the library are here.  tests/test_gpu_exact_math.py compares every float of
// [-8, 8] with the host library, bit for bit.
__device__ __forceinline__ void v2_sincosf(float y, float &sn, float &cs) {
	const double c0 = 0x1p0, c1 = -0x1.ffffffd0c621cp-2, c2 = 0x1.55553e1068f19p-5, c3 = -0x1.6c087e89a359dp-10, c4 = 0x1.99343027bf8c3p-16;
	const double s1 = -0x1.555545995a603p-3, s2 = 0x1.1107605230bc4p-7, s3 = -0x1.994eb3774cf24p-13;
	const unsigned top = (__float_as_uint(y) >> 20) & 0x7ffu;
	double x = (double)y;
	int n = 0;
	double sgn = 1.0, flip = 1.0; // flip: the second table row (n & 2) negates the cosine polynomial's coefficients
	if (top < ((__float_as_uint(0x1.921FB6p-1f) >> 20) & 0x7ffu)) {
		if (top < ((__float_as_uint(0x1p-12f) >> 20) & 0x7ffu)) {
			sn = y;
			cs = 1.0f;
			return;
		}
	}
	else { // reduce_fast: the engine's arguments are bounded by 2 pi (see above)
		const double r = __dmul_rn(x, 0x1.45F306DC9C883p+23);
		n = ((int)r + 0x800000) >> 24;
		x = __dsub_rn(x, __dmul_rn((double)n, 0x1.921FB54442D18p0));
		sgn = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
		if (n & 2) flip = -1.0;
	}
	const double x2 = __dmul_rn(x, x);
	x = __dmul_rn(x, sgn);
	const double x4 = __dmul_rn(x2, x2), x3 = __dmul_rn(x2, x);
	const double pc2 = __dadd_rn(__dmul_rn(flip, c3), __dmul_rn(x2, __dmul_rn(flip, c4)));
	const double ps1 = __dadd_rn(s2, __dmul_rn(x2, s3));
	const double pc1 = __dadd_rn(__dmul_rn(flip, c0), __dmul_rn(x2, __dmul_rn(flip, c1)));
	const double x5 = __dmul_rn(x3, x2), x6 = __dmul_rn(x4, x2);
	const double s = __dadd_rn(x, __dmul_rn(x3, s1));
	const double c = __dadd_rn(pc1, __dmul_rn(x4, __dmul_rn(flip, c2)));
	const float fs = __double2float_rn(__dadd_rn(s, __dmul_rn(x5, ps1)));
	const float fc = __double2float_rn(__dadd_rn(c, __dmul_rn(x6, pc2)));
	sn = (n & 1) ? fc : fs; // odd quadrants swap the two results
	cs = (n & 1) ? fs : fc;
}

// octant-reduced polynomial atan2 of the FM branch (V2Engine.cpp:243-262); 0 when both operands are zero
__device__ __forceinline__ float v2_atan2_fast(float y, float x) {
	const float ax = fabsf(x), ay = fabsf(y);
	const float mx = ax > ay ? ax : ay, mn = ax > ay ? ay : ax;
	if (mx == 0.0f) return 0.0f;
	const float a = __fdiv_rn(mn, mx);
	const float s = __fmul_rn(a, a);
	float r = __fadd_rn(__fmul_rn(-0.0464964749f, s), 0.15931422f);
	r = __fsub_rn(__fmul_rn(r, s), 0.327622764f);
	r = __fadd_rn(__fmul_rn(__fmul_rn(r, s), a), a);
	if (ay > ax) r = __fsub_rn(1.57079637f, r);
	if (x < 0.0f) r = __fsub_rn(3.14159274f, r);
	return y < 0.0f ? -r : r;
}

} // namespace aisgpu
