// The device restatements of the C library functions the reference calls -- fd_atan2f_common / fd_atan2f and habs
// (ais-catcher_b200/csrc/exact.cuh), v2_sincosf and v2_atan2_fast (v2_math.cuh) -- evaluated on the GPU and compared bit for bit
// with the host C library the reference itself is linked against: atan2f, hypotf, sincosf (and sinf / cosf, which std::polar
// calls).  NaN results are compared as a class: the device's canonical NaN is 0x7fffffff, x86's default NaN 0xffc00000.
// tests/test_gpu_exact_math.py compiles this file with the library's nvcc flags and runs it.
//
//   exact_math_check <random atan2 pairs> <random hypotf pairs> <sincosf stride>
//
// Prints one line per check, "<name> checked <n> mismatches <m> ...", and exits non-zero when any check has a mismatch.
#include <cfloat>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "exact.cuh"
#include "v2_math.cuh"

using namespace aisgpu;

// ---- device side ----
__global__ void k_atan2(const float *y, const float *x, float *common, float *full, long long n) {
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
		common[i] = fd_atan2f_common(y[i], x[i]);
		full[i] = fd_atan2f(y[i], x[i]);
	}
}
__global__ void k_habs(const float *y, const float *x, float *out, long long n) {
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
		out[i] = habs(make_float2(x[i], y[i]));
}
// the float with bit pattern first + i * stride, i < n
__global__ void k_sincos(uint32_t first, uint32_t stride, long long n, float *sn, float *cs) {
	for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
		v2_sincosf(__uint_as_float(first + (uint32_t)i * stride), sn[i], cs[i]);
}
__global__ void k_v2_atan2(const float *y, const float *x, float *out, int n) {
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = v2_atan2_fast(y[i], x[i]);
}

// ---- host side ----
static void cuda_check(cudaError_t e, const char *what) {
	if (e != cudaSuccess) {
		fprintf(stderr, "%s: %s\n", what, cudaGetErrorString(e));
		exit(2);
	}
}
#define CK(x) cuda_check((x), #x)

static inline uint32_t f2u(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static inline float u2f(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
static inline bool same(float a, float b) { return (std::isnan(a) && std::isnan(b)) || f2u(a) == f2u(b); }

static uint64_t splitmix(uint64_t &s) {
	uint64_t z = (s += 0x9e3779b97f4a7c15ull);
	z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
	z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
	return z ^ (z >> 31);
}

// runs f(lo, hi, t) over [0, n) on every host thread; f returns its mismatch count
template <typename F>
static long long parallel(long long n, F f) {
	int nt = (int)std::thread::hardware_concurrency();
	nt = nt < 1 ? 1 : (nt > 64 ? 64 : nt);
	std::vector<long long> bad(nt, 0);
	std::vector<std::thread> th;
	for (int t = 0; t < nt; t++)
		th.emplace_back([&, t] { bad[t] = f(n * t / nt, n * (t + 1) / nt, t); });
	for (auto &x : th) x.join();
	long long s = 0;
	for (long long b : bad) s += b;
	return s;
}

static const long long CH = 1 << 24; // elements per device round trip

struct Buffers {
	float *dy, *dx, *d0, *d1;
	std::vector<float> h0, h1;
	Buffers() : h0(CH), h1(CH) {
		CK(cudaMalloc(&dy, CH * 4)); CK(cudaMalloc(&dx, CH * 4)); CK(cudaMalloc(&d0, CH * 4)); CK(cudaMalloc(&d1, CH * 4));
	}
};

// the range test of fd_atan2f_common: true when the pair takes the out-of-line fd_atan2f
static bool atan2_rare(float y, float x) {
	const uint32_t hx = f2u(x), hy = f2u(y), ix = hx & 0x7fffffffu, iy = hy & 0x7fffffffu;
	const int k = ((int)iy - (int)ix) >> 23;
	return !((ix - 0x00800000u) < 0x7f000000u && (iy - 0x00800000u) < 0x7f000000u && (uint32_t)(k + 28) <= 51u && hx != 0x3f800000u);
}

struct Tally {
	long long n = 0, bad = 0, rare = 0;
	void print(const char *name, double s) const {
		printf("%s checked %lld mismatches %lld rare %lld (%.1f s)\n", name, n, bad, rare, s);
	}
};

// fd_atan2f_common and fd_atan2f against atan2f on the pairs (y[i], x[i])
static void atan2_chunk(Buffers &b, const float *y, const float *x, long long n, Tally &t, const char *name) {
	CK(cudaMemcpy(b.dy, y, n * 4, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(b.dx, x, n * 4, cudaMemcpyHostToDevice));
	k_atan2<<<1024, 256>>>(b.dy, b.dx, b.d0, b.d1, n);
	CK(cudaGetLastError());
	CK(cudaMemcpy(b.h0.data(), b.d0, n * 4, cudaMemcpyDeviceToHost));
	CK(cudaMemcpy(b.h1.data(), b.d1, n * 4, cudaMemcpyDeviceToHost));
	const long long printed = t.bad;
	t.bad += parallel(n, [&](long long lo, long long hi, int) {
		long long bad = 0;
		for (long long i = lo; i < hi; i++) {
			const float w = atan2f(y[i], x[i]);
			if (!same(b.h0[i], w) || !same(b.h1[i], w)) {
				if (printed + bad < 4)
					printf("  %s: atan2f(%a [%08x], %a [%08x]) = %08x, fd_atan2f_common %08x, fd_atan2f %08x\n", name, y[i], f2u(y[i]), x[i],
						   f2u(x[i]), f2u(w), f2u(b.h0[i]), f2u(b.h1[i]));
				bad++;
			}
		}
		return bad;
	});
	for (long long i = 0; i < n; i++) t.rare += atan2_rare(y[i], x[i]);
	t.n += n;
}

// habs against hypotf; pin_nonfinite: a pair of an infinity and a NaN must give NaN on the device where hypotf gives inf
static void habs_chunk(Buffers &b, const float *y, const float *x, long long n, Tally &t, const char *name, bool pin_nonfinite) {
	CK(cudaMemcpy(b.dy, y, n * 4, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(b.dx, x, n * 4, cudaMemcpyHostToDevice));
	k_habs<<<1024, 256>>>(b.dy, b.dx, b.d0, n);
	CK(cudaGetLastError());
	CK(cudaMemcpy(b.h0.data(), b.d0, n * 4, cudaMemcpyDeviceToHost));
	const long long printed = t.bad;
	t.bad += parallel(n, [&](long long lo, long long hi, int) {
		long long bad = 0;
		for (long long i = lo; i < hi; i++) {
			const float w = hypotf(x[i], y[i]);
			bool ok = same(b.h0[i], w);
			if (pin_nonfinite && ((std::isinf(x[i]) && std::isnan(y[i])) || (std::isnan(x[i]) && std::isinf(y[i]))))
				ok = std::isnan(b.h0[i]) && std::isinf(w); // the documented difference (DESIGN.md section 2)
			if (!ok) {
				if (printed + bad < 4)
					printf("  %s: hypotf(%a, %a) = %08x, habs %08x\n", name, x[i], y[i], f2u(w), f2u(b.h0[i]));
				bad++;
			}
		}
		return bad;
	});
	t.n += n;
}

static double secs(std::chrono::steady_clock::time_point t0) {
	return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

int main(int argc, char **argv) {
	const long long n_atan2 = argc > 1 ? atoll(argv[1]) : 100000000LL;
	const long long n_hypot = argc > 2 ? atoll(argv[2]) : 50000000LL;
	const uint32_t sc_stride = argc > 3 ? (uint32_t)atoll(argv[3]) : 1u;
	Buffers b;
	bool fail = false;

	// the special values: signed zeros, the smallest and largest subnormals, FLT_MIN, 1 and its neighbours, FLT_MAX, inf, NaN
	std::vector<float> sp;
	for (uint32_t u : {0x00000000u, 0x00000001u, 0x007fffffu, 0x00800000u, 0x3f7fffffu, 0x3f800000u, 0x3f800001u, 0x7f7fffffu, 0x7f800000u})
		for (uint32_t s : {0u, 0x80000000u}) sp.push_back(u2f(u | s));
	sp.push_back(u2f(0x7fc00000u));
	sp.push_back(u2f(0xffc00000u));
	std::vector<float> y, x;
	for (float a : sp)
		for (float c : sp) { y.push_back(a); x.push_back(c); }

	{ // 1. the special values, every pair
		auto t0 = std::chrono::steady_clock::now();
		Tally t;
		atan2_chunk(b, y.data(), x.data(), (long long)y.size(), t, "atan2_special");
		t.print("atan2_special", secs(t0));
		fail |= t.bad != 0;
		Tally h;
		habs_chunk(b, y.data(), x.data(), (long long)y.size(), h, "habs_special", true);
		h.print("habs_special", secs(t0));
		fail |= h.bad != 0;
	}
	{ // 2. every (exponent of y, exponent of x) pair x 4 sign combinations x 4 x 4 mantissas: the k + 28 <= 51 range test of
	  //    fd_atan2f_common and the k > 60 / k < -60 branches of fd_atan2f
		auto t0 = std::chrono::steady_clock::now();
		const uint32_t mant[4] = {0u, 1u, 0x400000u, 0x7fffffu};
		y.clear(); x.clear();
		for (uint32_t ey = 0; ey < 256; ey++)
			for (uint32_t ex = 0; ex < 256; ex++)
				for (uint32_t sg = 0; sg < 4; sg++)
					for (int my = 0; my < 4; my++)
						for (int mx = 0; mx < 4; mx++) {
							y.push_back(u2f((sg & 1u) << 31 | ey << 23 | mant[my]));
							x.push_back(u2f((sg >> 1) << 31 | ex << 23 | mant[(mx + my) & 3]));
						}
		Tally t;
		for (long long o = 0; o < (long long)y.size(); o += CH)
			atan2_chunk(b, y.data() + o, x.data() + o, std::min(CH, (long long)y.size() - o), t, "atan2_exponents");
		t.print("atan2_exponents", secs(t0));
		fail |= t.bad != 0;
	}
	{ // 3. random bit patterns (NaNs and infinities included)
		auto t0 = std::chrono::steady_clock::now();
		uint64_t s = 0xA7A2F00Dull;
		Tally t;
		y.resize(CH); x.resize(CH);
		for (long long o = 0; o < n_atan2; o += CH) {
			const long long n = std::min(CH, n_atan2 - o);
			for (long long i = 0; i < n; i++) {
				const uint64_t r = splitmix(s);
				y[i] = u2f((uint32_t)r);
				x[i] = u2f((uint32_t)(r >> 32));
			}
			atan2_chunk(b, y.data(), x.data(), n, t, "atan2_random");
		}
		t.print("atan2_random", secs(t0));
		fail |= t.bad != 0;
	}
	{ // 4. habs against hypotf on finite pairs: random patterns, subnormals, both near FLT_MAX
		auto t0 = std::chrono::steady_clock::now();
		uint64_t s = 0x4A85ull;
		Tally t;
		y.resize(CH); x.resize(CH);
		for (long long o = 0; o < n_hypot; o += CH) {
			const long long n = std::min(CH, n_hypot - o);
			for (long long i = 0; i < n; i++) {
				const uint64_t r = splitmix(s);
				uint32_t a = (uint32_t)r, c = (uint32_t)(r >> 32);
				switch (i % 4) {
				case 0: break;                                             // any pattern
				case 1: a &= 0x807fffffu; c &= 0x807fffffu; break;         // both subnormal (or zero)
				case 2: a &= 0x807fffffu; c = (c & 0x81ffffffu); break;    // subnormal against a tiny normal
				default: a |= 0x7e000000u; c |= 0x7e000000u; break;        // both within 2^-1 .. 2 of FLT_MAX
				}
				if ((a & 0x7f800000u) == 0x7f800000u) a &= 0xff7fffffu; // keep them finite
				if ((c & 0x7f800000u) == 0x7f800000u) c &= 0xff7fffffu;
				y[i] = u2f(a);
				x[i] = u2f(c);
			}
			habs_chunk(b, y.data(), x.data(), n, t, "habs_random", false);
		}
		t.print("habs_random", secs(t0));
		fail |= t.bad != 0;
	}
	{ // 5. v2_sincosf against sincosf on every float of [-8, 8] (or every sc_stride-th): the engine's domain [-1.27, 2 pi)
	  //    with a margin; sinf / cosf on every 16th
		auto t0 = std::chrono::steady_clock::now();
		Tally t;
		const uint32_t top = f2u(8.0f);
		for (uint32_t sign : {0u, 0x80000000u}) {
			const long long total = (long long)(top / sc_stride) + 1;
			for (long long o = 0; o < total; o += CH) {
				const long long n = std::min(CH, total - o);
				const uint32_t first = sign + (uint32_t)(o * sc_stride);
				k_sincos<<<1024, 256>>>(first, sc_stride, n, b.d0, b.d1);
				CK(cudaGetLastError());
				CK(cudaMemcpy(b.h0.data(), b.d0, n * 4, cudaMemcpyDeviceToHost));
				CK(cudaMemcpy(b.h1.data(), b.d1, n * 4, cudaMemcpyDeviceToHost));
				const long long printed = t.bad;
				t.bad += parallel(n, [&](long long lo, long long hi, int) {
					long long bad = 0;
					for (long long i = lo; i < hi; i++) {
						const float v = u2f(first + (uint32_t)i * sc_stride);
						float sn, cs;
						sincosf(v, &sn, &cs);
						bool ok = f2u(sn) == f2u(b.h0[i]) && f2u(cs) == f2u(b.h1[i]);
						if (ok && (i & 15) == 0) ok = f2u(sinf(v)) == f2u(b.h0[i]) && f2u(cosf(v)) == f2u(b.h1[i]);
						if (!ok) {
							if (printed + bad < 4)
								printf("  sincos: %a [%08x]: sincosf (%08x, %08x), v2_sincosf (%08x, %08x)\n", v, f2u(v), f2u(sn), f2u(cs),
									   f2u(b.h0[i]), f2u(b.h1[i]));
							bad++;
						}
					}
					return bad;
				});
				t.n += n;
			}
		}
		t.print("sincos", secs(t0));
		fail |= t.bad != 0;
	}
	{ // 6. v2_atan2_fast with both operands zero (any signs) is +0, as in the reference's FMDemod
		const float zy[4] = {0.0f, -0.0f, 0.0f, -0.0f}, zx[4] = {0.0f, 0.0f, -0.0f, -0.0f};
		float out[4];
		CK(cudaMemcpy(b.dy, zy, 16, cudaMemcpyHostToDevice));
		CK(cudaMemcpy(b.dx, zx, 16, cudaMemcpyHostToDevice));
		k_v2_atan2<<<1, 32>>>(b.dy, b.dx, b.d0, 4);
		CK(cudaGetLastError());
		CK(cudaMemcpy(out, b.d0, 16, cudaMemcpyDeviceToHost));
		long long bad = 0;
		for (int i = 0; i < 4; i++) bad += f2u(out[i]) != 0u;
		printf("v2_atan2_zero checked 4 mismatches %lld\n", bad);
		fail |= bad != 0;
	}
	return fail ? 1 : 0;
}
