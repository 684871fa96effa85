// fe_common.cuh -- sample-format conversion shared by the front-end kernels (Utilities/Convert.cpp:255-301, and ConvertRAW's
// F32_FS4 case, Utilities/StreamHelpers.cpp:105-118).
#pragma once
#include "exact.cuh"
#include "params.h"

namespace aisgpu {

// F32_FS4: one real float per sample, shifted by fs/4 -- sample n of a Receive becomes x, jx, -x, -jx for n % 4 = 0 .. 3.  The
// pattern restarts with every Receive, and every block length the engine takes is a multiple of 4, so n % 4 is the sample's
// index in the submit modulo 4 (a negative index reaches into the previous submit's history: two's complement keeps n & 3).
// Readers pass that index as `pos`; the other formats ignore it.  The live component is x with its sign bit kept or flipped
// (never 0 - x: -(+0) is -0), the other the literal +0; nothing is multiplied.
__device__ __forceinline__ float fs4_neg(float x) { return __int_as_float(__float_as_int(x) ^ (int)0x80000000u); }
// samples 2m, 2m + 1 of the pattern from the floats (x0, x1); `neg` = bit 1 of the even sample's position
__device__ __forceinline__ void fs4_pair(float x0, float x1, bool neg, float2 &a, float2 &b) {
	a = make_float2(neg ? fs4_neg(x0) : x0, 0.0f);
	b = make_float2(0.0f, neg ? fs4_neg(x1) : x1);
}

// DC16H (Convert.cpp:288-301): three 32-bit words per sample.  I is the low half of word 0 and Q the low half of word 1, both
// sign-extended; the high halves and word 2 are never read.  Q is negated as a 32-bit integer BEFORE the conversion: Q = 0 stays
// +0.0f (a float negation would make -0.0f, and atan2f tells them apart) and Q = -32768 becomes exactly 1.0f.
__device__ __forceinline__ float2 dc16h_sample(uint32_t wi, uint32_t wq) {
	const int i = (int)(short)(wi & 0xFFFFu), q = -(int)(short)(wq & 0xFFFFu);
	return make_float2(__fmul_rn((float)i, 3.0517578125e-05f), __fmul_rn((float)q, 3.0517578125e-05f));
}

template <int FMT>
__device__ __forceinline__ void fe_load_pair(const void *base, long long idx, int pos, float2 &a, float2 &b) {
	// two consecutive samples starting at even index idx, which is sample `pos` (even) of the submit
	if (FMT == 0) {
		float4 v = __ldg(reinterpret_cast<const float4 *>(reinterpret_cast<const float2 *>(base) + idx));
		a = make_float2(v.x, v.y);
		b = make_float2(v.z, v.w);
	}
	else if (FMT == 1) { // CU8: (u-128)/128  (Utilities/Convert.cpp:255-264); /128 is an exact scaling
		uchar4 v = __ldg(reinterpret_cast<const uchar4 *>(reinterpret_cast<const uchar2 *>(base) + idx));
		a = make_float2(__fmul_rn((float)((int)v.x - 128), 0.0078125f), __fmul_rn((float)((int)v.y - 128), 0.0078125f));
		b = make_float2(__fmul_rn((float)((int)v.z - 128), 0.0078125f), __fmul_rn((float)((int)v.w - 128), 0.0078125f));
	}
	else if (FMT == 2) { // CS8 (Convert.cpp:266-275)
		char4 v = __ldg(reinterpret_cast<const char4 *>(reinterpret_cast<const char2 *>(base) + idx));
		a = make_float2(__fmul_rn((float)v.x, 0.0078125f), __fmul_rn((float)v.y, 0.0078125f));
		b = make_float2(__fmul_rn((float)v.z, 0.0078125f), __fmul_rn((float)v.w, 0.0078125f));
	}
	else if (FMT == 3) { // CS16 (Convert.cpp:277-286)
		short4 v = __ldg(reinterpret_cast<const short4 *>(reinterpret_cast<const short2 *>(base) + idx));
		a = make_float2(__fmul_rn((float)v.x, 3.0517578125e-05f), __fmul_rn((float)v.y, 3.0517578125e-05f));
		b = make_float2(__fmul_rn((float)v.z, 3.0517578125e-05f), __fmul_rn((float)v.w, 3.0517578125e-05f));
	}
	else if (FMT == FE_FMT_FS4) {
		const float2 v = __ldg(reinterpret_cast<const float2 *>(reinterpret_cast<const float *>(base) + idx));
		fs4_pair(v.x, v.y, (pos & 2) != 0, a, b);
	}
	else { // DC16H: 24 bytes, read as the four live words (any word-aligned base)
		static_assert(FMT <= 3 || FMT == FE_FMT_FS4 || FMT == FE_FMT_DC16H, "no conversion for this format id");
		const uint32_t *w = reinterpret_cast<const uint32_t *>(base) + idx * 3;
		a = dc16h_sample(__ldg(w), __ldg(w + 1));
		b = dc16h_sample(__ldg(w + 3), __ldg(w + 4));
	}
}

template <int FMT>
__device__ __forceinline__ float2 fe_load_one(const void *base, long long idx, int pos) { // sample idx of the rows, which is sample `pos` of the submit
	if (FMT == 0) return __ldg(reinterpret_cast<const float2 *>(base) + idx);
	if (FMT == 1) {
		const uchar2 v = __ldg(reinterpret_cast<const uchar2 *>(base) + idx);
		return make_float2(__fmul_rn((float)((int)v.x - 128), 0.0078125f), __fmul_rn((float)((int)v.y - 128), 0.0078125f));
	}
	if (FMT == 2) {
		const char2 v = __ldg(reinterpret_cast<const char2 *>(base) + idx);
		return make_float2(__fmul_rn((float)v.x, 0.0078125f), __fmul_rn((float)v.y, 0.0078125f));
	}
	if (FMT == 3) {
		const short2 v = __ldg(reinterpret_cast<const short2 *>(base) + idx);
		return make_float2(__fmul_rn((float)v.x, 3.0517578125e-05f), __fmul_rn((float)v.y, 3.0517578125e-05f));
	}
	if (FMT == FE_FMT_FS4) {
		const float x = __ldg(reinterpret_cast<const float *>(base) + idx);
		const float y = (pos & 2) ? fs4_neg(x) : x;
		return (pos & 1) ? make_float2(0.0f, y) : make_float2(y, 0.0f);
	}
	static_assert(FMT <= 3 || FMT == FE_FMT_FS4 || FMT == FE_FMT_DC16H, "no conversion for this format id");
	const uint32_t *w = reinterpret_cast<const uint32_t *>(base) + idx * 3;
	return dc16h_sample(__ldg(w), __ldg(w + 1));
}

} // namespace aisgpu
