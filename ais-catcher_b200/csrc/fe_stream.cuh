#pragma once
#include "exact.cuh"
#include "params.h"
#include <atomic>
#include <algorithm>

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// K1'': the front end as the reference writes it -- a per-sample streaming pipeline with its state in registers --
// run by every THREAD on its own sub-segment of a stream.  A lane walks [a - P, a + S): the first P samples only warm
// the state up from zero (each CIC stage is a pure function of its last six inputs, see k_frontend), after that every
// 2^(K+1) inputs yield one 48 kHz sample per channel.  Per input pair a Downsample2CIC5 stage costs 9 complex adds and
// one complex multiply (DSP.cpp:93-117, literally: r_k = z; z += h_k / h_k = z; z += r_k), each a pair of scalar
// __fadd_rn / __fmul_rn (exact.cuh: rounded separately, never contracted into an FMA, subnormals kept), and nothing goes
// through shared memory between stages; shared memory only stages the input: the warp fetches the next 16 samples of all 32 lanes with
// coalesced 16-byte cp.async copies (raw format, converted when read) into a ring, four chunks ahead.
// ---------------------------------------------------------------------------------------------
struct Cic5 { c64 h0, h1, h2, h3, h4; };
__device__ __forceinline__ void cic5_zero(Cic5 &s) { s.h0 = s.h1 = s.h2 = s.h3 = s.h4 = 0ull; }
// one even/odd input pair of Downsample2CIC5 -> one output
__device__ __forceinline__ c64 ds2_pair(Cic5 &s, c64 xe, c64 xo, c64 sc) {
	c64 z = xe;
	const c64 r0 = z; z = padd(z, s.h0);
	const c64 r1 = z; z = padd(z, s.h1);
	const c64 r2 = z; z = padd(z, s.h2);
	const c64 r3 = z; z = padd(z, s.h3);
	const c64 r4 = z; z = padd(z, s.h4);
	const c64 out = pmul(z, sc);
	z = xo;
	s.h0 = z; z = padd(z, r0);
	s.h1 = z; z = padd(z, r1);
	s.h2 = z; z = padd(z, r2);
	s.h3 = z; z = padd(z, r3);
	s.h4 = z;
	(void)r4;
	return out;
}
// one even/odd input pair of FilterCIC5 -> two outputs (DSP.cpp:132-157)
__device__ __forceinline__ void fcic_pair(Cic5 &s, c64 xe, c64 xo, c64 sc, c64 &oe, c64 &oo) {
	c64 z = xe;
	const c64 r0 = z; z = padd(z, s.h0);
	const c64 r1 = z; z = padd(z, s.h1);
	const c64 r2 = z; z = padd(z, s.h2);
	const c64 r3 = z; z = padd(z, s.h3);
	const c64 r4 = z; z = padd(z, s.h4);
	oe = pmul(z, sc);
	z = xo;
	s.h0 = z; z = padd(z, r0);
	s.h1 = z; z = padd(z, r1);
	s.h2 = z; z = padd(z, r2);
	s.h3 = z; z = padd(z, r3);
	s.h4 = z; z = padd(z, r4);
	oo = pmul(z, sc);
}
// ---- -go FP_DS on (Model.cpp:233-236): DSP::Downsample16_CU8 = four DS_UINT16 stages on I/Q packed as two uint16 in one
// ---- uint32 (DSP.cpp:499-665, shifts 3, 4, 5, then 0 with the conversion to float).  Plain integer adds: bit-exact by
// ---- construction, including the carry of I into Q that the reference's masks "clean up" after the shift.
struct Cic5u { uint32_t h0, h1, h2, h3, h4; };
__device__ __forceinline__ void cic5u_zero(Cic5u &s) { s.h0 = s.h1 = s.h2 = s.h3 = s.h4 = 0u; }
template <int SHIFT>
__device__ __forceinline__ uint32_t ds2u_pair(Cic5u &s, uint32_t xe, uint32_t xo) { // MA1 x 5, emit, MA2 x 5 (DSP.cpp:85-90, 508-527)
	constexpr uint32_t m16 = 0xFFFFu >> SHIFT, mask = m16 | (m16 << 16);
	uint32_t z = xe;
	const uint32_t r0 = z; z += s.h0;
	const uint32_t r1 = z; z += s.h1;
	const uint32_t r2 = z; z += s.h2;
	const uint32_t r3 = z; z += s.h3;
	z += s.h4;
	const uint32_t out = (z >> SHIFT) & mask;
	z = xo;
	s.h0 = z; z += r0;
	s.h1 = z; z += r1;
	s.h2 = z; z += r2;
	s.h3 = z; z += r3;
	s.h4 = z;
	return out;
}
// last stage: uint16 pair -> int16 pair (sign bits flipped) -> float / 32768 (DSP.cpp:610-617)
__device__ __forceinline__ c64 u16pair_to_c64(uint32_t z) {
	z ^= 0x80008000u;
	return pack2(__fmul_rn((float)(short)(z & 0xFFFFu), 3.0517578125e-05f), __fmul_rn((float)(short)(z >> 16), 3.0517578125e-05f));
}

template <int FMT, int G>
struct StFmt {
	static constexpr int BPS = FMT == 0 ? 8 : (FMT == 3 ? 4 : 2); // FMT 4: CU8 through the integer CIC stages (-go FP_DS on)
	static constexpr int CHUNK = G * BPS;         // bytes of one lane's chunk (G = 16: 128 / 32 / 32 / 64)
	static constexpr int PIECES = CHUNK / 16;     // 16-byte pieces per lane chunk = cp.async instructions per warp chunk
	static constexpr int SLOT = CHUNK + 16;       // lane stride in the ring (odd multiple of 16 bytes: conflict-free 16-byte reads)
};
// sample pair j (samples 2j, 2j+1) of a staged chunk
template <int FMT>
__device__ __forceinline__ void st_read_pair(const unsigned char *slot, int j, c64 &xe, c64 &xo) {
	if (FMT == 0) {
		const ulonglong2 v = *reinterpret_cast<const ulonglong2 *>(slot + j * 16);
		xe = v.x;
		xo = v.y;
	}
	else if (FMT == 1) {
		const uchar4 v = *reinterpret_cast<const uchar4 *>(slot + j * 4);
		xe = pack2(__fmul_rn((float)((int)v.x - 128), 0.0078125f), __fmul_rn((float)((int)v.y - 128), 0.0078125f));
		xo = pack2(__fmul_rn((float)((int)v.z - 128), 0.0078125f), __fmul_rn((float)((int)v.w - 128), 0.0078125f));
	}
	else if (FMT == 2) {
		const char4 v = *reinterpret_cast<const char4 *>(slot + j * 4);
		xe = pack2(__fmul_rn((float)v.x, 0.0078125f), __fmul_rn((float)v.y, 0.0078125f));
		xo = pack2(__fmul_rn((float)v.z, 0.0078125f), __fmul_rn((float)v.w, 0.0078125f));
	}
	else {
		const short4 v = *reinterpret_cast<const short4 *>(slot + j * 8);
		xe = pack2(__fmul_rn((float)v.x, 3.0517578125e-05f), __fmul_rn((float)v.y, 3.0517578125e-05f));
		xo = pack2(__fmul_rn((float)v.z, 3.0517578125e-05f), __fmul_rn((float)v.w, 3.0517578125e-05f));
	}
}

// ST_WARPS: warps per CTA (independent of each other), ST_NB: chunks in each warp's staging ring.  CF32 runs four-warp CTAs with
// 32-sample chunks and a ring of 3 (104 KB per CTA); the integer formats one-warp CTAs with 16-sample chunks and a ring of 8.
// ST_G: samples a lane fetches per visit of its sub-segment.  Every lane is an independent sequential stream for DRAM (1024 warps
// = 32768 streams, far more than there are banks), so the bytes per visit decide the row-buffer locality: 16 samples = one
// 128-byte line per visit, 64 samples = four consecutive lines.
template <int FMT, int K, int ST_G, int ST_NB, int ST_WARPS, bool PRE = false>
__global__ void __launch_bounds__(ST_WARPS * 32) k_frontend_st(const FeParams p) {
	static_assert(K >= 3 && K <= 7, "streaming front end: 768 kS/s .. 12288 kS/s");
	static_assert(ST_G <= (1 << (K + 2)) && (ST_G % 16) == 0, "a chunk must not be longer than a super-step");
	typedef StFmt<FMT, ST_G> F;
	constexpr int SS = 1 << (K + 2);     // inputs per super-step: two 48 kHz samples per channel
	constexpr int NCH = SS / ST_G;       // chunks per super-step
	constexpr int N96 = SS >> K;         // 96 kHz samples per super-step (4)
	extern __shared__ __align__(16) unsigned char st_ring[]; // [ST_WARPS][ST_NB][32 * SLOT]
	const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
	// Lane mapping: global lane g owns sub-segment (g % L) of stream (g / L).  A stream's nss = q * L + r super-steps are split
	// unevenly -- the first L - r lanes take q, the last r take q + 1 -- so that L need not divide the block: the host picks L such
	// that all CTAs are resident at once (one wave over the SMs) with the longest sub-segments that allow (launch_st_one).
	const long long g0 = ((long long)blockIdx.x * ST_WARPS + wib) * 32;
	const int L = p.st_L;
	if (g0 >= (long long)p.st_B * L) return; // whole warp
	int stream = (int)((g0 + lane) / L), sub = (int)((g0 + lane) - (long long)stream * L);
	const bool ghost = stream >= p.st_B; // the last warp's spare lanes replay the batch's last lane without storing
	if (ghost) { stream = p.st_B - 1; sub = L - 1; }
	const int n_short = L - p.st_r;
	const int n_main = ghost ? 0 : p.st_q + (sub >= n_short ? 1 : 0); // super-steps this lane delivers
	unsigned char(*ring)[32 * F::SLOT] = reinterpret_cast<unsigned char(*)[32 * F::SLOT]>(st_ring + (size_t)wib * ST_NB * 32 * F::SLOT);
	// the lane owns samples [a, a + n_main * SS); every lane of every warp walks warm_super + q + (r ? 1 : 0) super-steps (a short
	// lane's last one re-reads the head of its right neighbour's sub-segment -- same stream -- and is not stored)
	const long long a = ((long long)sub * p.st_q + max(0, sub - n_short)) * SS;
	const int n_super = p.P / SS + p.st_q + (p.st_r ? 1 : 0);
	const int warp_chunks = n_super * NCH; // warm-up included
	// staging: in instruction `it` lane j fetches 16-byte piece (j % PIECES) of the chunk of owner it*(32/PIECES) + j / PIECES;
	// only the first sub-segment of a stream starts in the previous submit: its warm-up chunks come from the tail buffer
	constexpr int OWN_PER_IT = 32 / F::PIECES;
	const int o0 = lane / F::PIECES, q0 = lane % F::PIECES;
	// Where the owners' sub-segments start: every lane computes its own start and the fetching lane collects, once, the starts of
	// the PIECES owners it fetches for (a table in shared memory would put an LDS in front of every LDGSTS, and ptxas pads that
	// pair with three dummy issue slots).  Main phase: 32-bit offsets in 16-byte units from in0 = p.in - P samples (the launcher
	// declines batches of 64 GB and more) -- two instructions per 16-byte copy; warm-up phase (the first P / ST_G chunks,
	// warp-uniform): full addresses by shuffle, because a stream's first lane reads the tail buffer.
	const unsigned char *in0 = reinterpret_cast<const unsigned char *>(p.in) - (long long)p.P * F::BPS;
	const unsigned my_off = (unsigned)((((long long)stream * p.in_stride + a) * F::BPS) >> 4);
	const unsigned long long my_warm = sub == 0 ? (unsigned long long)(reinterpret_cast<const unsigned char *>(p.tail) + (long long)stream * p.P * F::BPS)
												: (unsigned long long)(in0 + ((unsigned long long)my_off << 4));
	const int dst_off = o0 * F::SLOT + q0 * 16;
	unsigned own_off[F::PIECES]; // the owners this lane fetches for, one per instruction of a chunk (registers are not the scarce resource: one CTA per SM)
#pragma unroll
	for (int it = 0; it < F::PIECES; it++) own_off[it] = __shfl_sync(0xffffffffu, my_off, it * OWN_PER_IT + o0);
	auto prefetch = [&](int c) {
		if (c < warp_chunks) {
			const long long coff = (long long)c * (ST_G * F::BPS) + q0 * 16;
			unsigned char *dst = &ring[c % ST_NB][dst_off];
			if (c * ST_G < p.P) { // a rolled loop: this branch runs for 5 % of the chunks and would otherwise be inlined at every prefetch site (K + 2 .. 20 of them)
#pragma unroll 1
				for (int it = 0; it < F::PIECES; it++) {
					const unsigned long long w = __shfl_sync(0xffffffffu, my_warm, it * OWN_PER_IT + o0);
					cp_async16(dst + it * OWN_PER_IT * F::SLOT, reinterpret_cast<const unsigned char *>(w) + coff);
				}
			}
			else {
				unsigned long long base = (unsigned long long)(in0 + coff);
				asm volatile("" : "+l"(base)); // one register pair: otherwise ptxas keeps p.in uniform and adds it to every address again
#pragma unroll
				for (int it = 0; it < F::PIECES; it++) cp_async16(dst + it * OWN_PER_IT * F::SLOT, reinterpret_cast<const unsigned char *>(base + ((unsigned long long)own_off[it] << 4)));
			}
		}
		cp_async_commit();
	};
	const c64 sc = pack2(0.03125f, 0.03125f);
	static_assert(FMT != 4 || (K == 4 && !PRE), "the integer front end exists for the exact 1536K bucket only (Model.cpp:222-236)");
	Cic5 lv[K], chA, chB, fA, fB;
	Cic5u lu[4];
	uint32_t pendu[4];
#pragma unroll
	for (int l = 0; l < 4; l++) { cic5u_zero(lu[l]); pendu[l] = 0u; }
#pragma unroll
	for (int l = 0; l < K; l++) cic5_zero(lv[l]);
	cic5_zero(chA); cic5_zero(chB); cic5_zero(fA); cic5_zero(fB);
	c64 fd1 = 0ull, fd2 = 0ull; // FilterComplex3Tap h1, h2
	// PRE: decimation in front of DSP::Upsample -- the level-K samples go to D0 and nothing else is computed
	const float2 *rot_g = PRE ? nullptr : p.rot + (p.P >> K) + ((a - p.P) >> K);
	float2 *Cg = PRE ? p.D0 + (long long)stream * p.d0_stride + p.d0_off + ((a - p.P) >> K)
					 : p.C + (long long)(stream * 2) * p.c_stride + p.c_off + ((a - p.P) >> (K + 1));
	const int warm_super = p.P / SS;
#pragma unroll
	for (int c = 0; c < ST_NB - 1; c++) prefetch(c);
	// Rotate phasors: loaded two super-steps ahead of their use (under load a global load can take longer than one
	// super-step of arithmetic)
	float2 rt_n1[N96], rt_n2[N96];
#pragma unroll
	for (int i = 0; i < N96; i++) {
		rt_n1[i] = PRE ? make_float2(0.f, 0.f) : __ldg(rot_g + i);
		rt_n2[i] = PRE ? make_float2(0.f, 0.f) : __ldg(rot_g + (n_super > 1 ? N96 : 0) + i);
	}
	// Tried on this loop on the previous target and dropped, each slower live (not re-measured on the H100): two super-steps per
	//   trip (fewer back-edge register moves, but more registers and twice the code); the droop filter selected instead of branched;
	//   a register cap that spills; the chunk loop below rolled (smaller kernel, but the state moves are paid per chunk).
	for (int ss = 0; ss < n_super; ss++) {
		float2 rt[N96];
#pragma unroll
		for (int i = 0; i < N96; i++) {
			rt[i] = rt_n1[i];
			rt_n1[i] = rt_n2[i];
		}
		if (!PRE && ss + 2 < n_super) {
#pragma unroll
			for (int i = 0; i < N96; i++) rt_n2[i] = __ldg(rot_g + (ss + 2) * N96 + i);
		}
		c64 lvK[N96]; // PRE: the super-step's level-K outputs
		c64 pend[K + 1];  // pend[l]: even-indexed input waiting at level l+1 (l = 1..K-1), pend[K]: unused
		c64 upE = 0ull, dnE = 0ull, waE = 0ull, wbE = 0ull;
		c64 outA0 = 0ull, outA1 = 0ull, outB0 = 0ull, outB1 = 0ull;
#pragma unroll
		for (int cc = 0; cc < NCH; cc++) {
			const int c = ss * NCH + cc;
			prefetch(c + ST_NB - 1);
			cp_async_wait<ST_NB - 1>(); // chunk c has landed
			__syncwarp();
			{
				const unsigned char *slot = &ring[c % ST_NB][lane * F::SLOT];
#pragma unroll
				for (int j = 0; j < ST_G / 2; j++) {
					const int n1 = cc * (ST_G / 2) + j; // index of this pair's output at level 1 within the super-step
					c64 y = 0ull;
					int idx = n1;
					bool live = true;
					if (FMT == 4) { // integer stages 1..4; the fourth one delivers the 96 kHz float sample
						const uchar4 v = *reinterpret_cast<const uchar4 *>(slot + j * 4);
						uint32_t yu = ds2u_pair<3>(lu[0], (uint32_t)v.x | ((uint32_t)v.y << 16), (uint32_t)v.z | ((uint32_t)v.w << 16));
						if ((idx & 1) == 0) { pendu[1] = yu; live = false; }
						else { yu = ds2u_pair<4>(lu[1], pendu[1], yu); idx >>= 1; }
						if (live) {
							if ((idx & 1) == 0) { pendu[2] = yu; live = false; }
							else { yu = ds2u_pair<5>(lu[2], pendu[2], yu); idx >>= 1; }
						}
						if (live) {
							if ((idx & 1) == 0) { pendu[3] = yu; live = false; }
							else {
								y = u16pair_to_c64(ds2u_pair<0>(lu[3], pendu[3], yu));
								// before the first sample of a stream the reference's float stages hold 0.0f, while the all-zero bytes
								// of the (virtual) history convert to -1.0f: silence the warm-up outputs of the stream's first lane
								if (p.st_first && sub == 0 && ss < warm_super) y = 0ull;
								idx >>= 1;
							}
						}
					}
					else {
						c64 xe, xo;
						st_read_pair<FMT == 4 ? 1 : FMT>(slot, j, xe, xo);
						y = ds2_pair(lv[0], xe, xo, sc);
						// ripple through the deeper levels: an output with an odd index completes a pair one level down
#pragma unroll
						for (int l = 1; l < K; l++) {
							if (live) {
								if ((idx & 1) == 0) { pend[l] = y; live = false; }
								else { y = ds2_pair(lv[l], pend[l], y, sc); idx >>= 1; }
							}
						}
					}
					if (live && PRE) lvK[idx] = y;
					if (live && !PRE) { // y is 96 kHz sample idx (0..N96-1) of the super-step
						c64 x = y;
						if (p.use_fdc) { // FilterComplex3Tap: alpha * (h1 + x) + h2 * beta (DSP.cpp:283-293)
							// FilterComplex3Tap's own operation order, each product and sum rounded separately
							const float2 h1 = unpack2(fd1), h2 = unpack2(fd2), yv = unpack2(y);
							const float tx = __fadd_rn(h1.x, yv.x), ty = __fadd_rn(h1.y, yv.y);
							x = pack2(__fadd_rn(__fmul_rn(p.fdc_alpha, tx), __fmul_rn(h2.x, p.fdc_beta)),
									  __fadd_rn(__fmul_rn(p.fdc_alpha, ty), __fmul_rn(h2.y, p.fdc_beta)));
							fd1 = fd2;
							fd2 = y;
						}
						const float2 xv = unpack2(x);
						const float2 r = rt[idx];
						const float RR = __fmul_rn(xv.x, r.x), II = __fmul_rn(xv.y, r.y), RI = __fmul_rn(xv.x, r.y), IR = __fmul_rn(xv.y, r.x);
						const c64 up = pack2(__fsub_rn(RR, II), __fadd_rn(IR, RI));
						const c64 dn = pack2(__fadd_rn(RR, II), __fsub_rn(IR, RI));
						if ((idx & 1) == 0) { upE = up; dnE = dn; }
						else {
							const c64 wa = ds2_pair(chA, upE, up, sc), wb = ds2_pair(chB, dnE, dn, sc);
							if ((idx & 2) == 0) { waE = wa; wbE = wb; }
							else {
								fcic_pair(fA, waE, wa, sc, outA0, outA1);
								fcic_pair(fB, wbE, wb, sc, outB0, outB1);
							}
						}
					}
				}
			}
			__syncwarp(); // the ring slot may be refilled by a later prefetch
		}
		if (PRE) {
			if (ss >= warm_super && ss - warm_super < n_main) {
				float2 *o = Cg + ss * N96;
#pragma unroll
				for (int i = 0; i < N96; i += 2) *reinterpret_cast<ulonglong2 *>(o + i) = make_ulonglong2(lvK[i], lvK[i + 1]);
			}
		}
		else if (ss >= warm_super && ss - warm_super < n_main) { // two 48 kHz samples per channel
			float2 *o = Cg + ss * 2;
			*reinterpret_cast<ulonglong2 *>(o) = make_ulonglong2(outA0, outA1);
			*reinterpret_cast<ulonglong2 *>(o + p.c_stride) = make_ulonglong2(outB0, outB1);
		}
	}
	cp_async_wait<0>();
}

// ---- launch entry point of one sample format (instantiated by fe_stream_f<FMT>.cu) ----
// Lanes per stream: the cost of a launch is modelled as waves x (super-steps per lane, warm-up included), a wave being what
// the SMs hold at once (SM count x resident CTAs of this shape).  Sub-segments shorter than `min_ratio` warm-ups are not considered;
// among (nearly) equal costs the fewest lanes win -- every lane re-reads P samples of warm-up.
// 1024 streams x 2048 super-steps, four-warp CTAs, one per SM on 132 SMs: L = 16 (128 CTAs, 128 + 6 super-steps) against
// 140 for the split L = 32 (256 CTAs = 2 waves of 64 + 6).
static inline bool st_plan(long long B, int nss, int warm, int wpc, int slots, int min_ratio, int forced_L, int &L, int &q, int &r) {
	const int q_min = warm * min_ratio > 0 ? warm * min_ratio : 1;
	if (nss < q_min) return false;
	const int L_max = nss / q_min;
	auto cost = [&](int l) {
		const long long ctas = ((B * l + 31) / 32 + wpc - 1) / wpc;
		const long long waves = (ctas + slots - 1) / slots;
		return (double)waves * ((nss + l - 1) / l + warm);
	};
	int best = 1;
	double cb = cost(1);
	for (int l = 2; l <= L_max; l++) {
		const double c = cost(l);
		if (c < cb * 0.97) { cb = c; best = l; }
	}
	if (forced_L > 0) best = forced_L < L_max ? forced_L : L_max;
	L = best;
	q = nss / L;
	r = nss - q * L;
	return true;
}
// SMs x resident CTAs of one kernel instantiation, and the SM count: asked once per process and instantiation (the caller's
// static cache; all devices of a box are alike)
struct CtaSlots { std::atomic<int> slots{0}, sms{0}; };
template <typename Kernel>
static cudaError_t cta_slots(CtaSlots &cache, Kernel *kernel, int threads, size_t smem, int &slots, int &sms) {
	slots = cache.slots.load();
	sms = cache.sms.load();
	if (slots) return cudaSuccess;
	int dev = 0, occ = 0;
	cudaError_t e;
	if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
	if ((e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)) != cudaSuccess) return e;
	if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, threads, smem)) != cudaSuccess) return e;
	slots = sms * (occ > 0 ? occ : 1);
	cache.sms.store(sms); // before slots: a thread that sees slots != 0 also sees sms
	cache.slots.store(slots);
	return cudaSuccess;
}

template <int FMT, int K, int G, int NB, int WPC, bool PRE>
static cudaError_t launch_st_one(const FeParams &p_in, int forced_L, cudaStream_t s) {
	constexpr int GG = G <= (1 << (K + 2)) ? G : (1 << (K + 2)); // K = 3: a super-step is 32 samples
	constexpr int SS = 1 << (K + 2);
	const size_t smem = (size_t)WPC * NB * 32 * StFmt<FMT, GG>::SLOT;
	cudaError_t e = cudaFuncSetAttribute(k_frontend_st<FMT, K, GG, NB, WPC, PRE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); // per device
	if (e != cudaSuccess) return e;
	static CtaSlots cache;
	int slots = 0, sms = 0;
	if ((e = cta_slots(cache, k_frontend_st<FMT, K, GG, NB, WPC, PRE>, WPC * 32, smem, slots, sms)) != cudaSuccess) return e;
	if (p_in.st_cap > 0) slots = std::min(slots, sms * p_in.st_cap);
	FeParams p = p_in;
	if (p.N % SS || p.P % SS) return cudaErrorNotSupported; // the caller falls back to the tiled kernel
	if ((unsigned long long)p.st_B * (unsigned long long)p.in_stride * StFmt<FMT, GG>::BPS >= (1ull << 36)) return cudaErrorNotSupported; // 32-bit lane offsets (16-byte units)
	// the integer front end only needs a sub-segment to cover its own warm-up; the float one wants >= 4 warm-ups per lane
	if (!st_plan(p.st_B, p.N / SS, p.P / SS, WPC, slots, FMT == 4 ? 1 : 4, forced_L, p.st_L, p.st_q, p.st_r)) return cudaErrorNotSupported;
	const long long n_warps = ((long long)p.st_B * p.st_L + 31) / 32;
	const unsigned ctas = (unsigned)((n_warps + WPC - 1) / WPC);
	k_frontend_st<FMT, K, GG, NB, WPC, PRE><<<ctas, WPC * 32, smem, s>>>(p);
	return cudaGetLastError();
}
// One launch shape (chunk length G, ring depth NB, warps per CTA WPC) of one format, for every K it is instantiated for:
// 3 .. 7 CIC stages (768 kS/s .. 12288 kS/s), or 3 .. 5 in front of DSP::Upsample (pre).  Any other K: cudaErrorNotSupported.
template <int FMT, int G, int NB, int WPC>
cudaError_t launch_frontend_stream_shape(const FeParams &p, int k, bool pre, int forced_L, cudaStream_t s) {
	if (pre) {
		switch (k) {
		case 3: return launch_st_one<FMT, 3, G, NB, WPC, true>(p, forced_L, s);
		case 4: return launch_st_one<FMT, 4, G, NB, WPC, true>(p, forced_L, s);
		case 5: return launch_st_one<FMT, 5, G, NB, WPC, true>(p, forced_L, s);
		default: return cudaErrorNotSupported;
		}
	}
	switch (k) {
	case 3: return launch_st_one<FMT, 3, G, NB, WPC, false>(p, forced_L, s);
	case 4: return launch_st_one<FMT, 4, G, NB, WPC, false>(p, forced_L, s);
	case 5: return launch_st_one<FMT, 5, G, NB, WPC, false>(p, forced_L, s);
	case 6: return launch_st_one<FMT, 6, G, NB, WPC, false>(p, forced_L, s);
	case 7: return launch_st_one<FMT, 7, G, NB, WPC, false>(p, forced_L, s);
	default: return cudaErrorNotSupported;
	}
}
// The shapes that exist, each compiled by its own translation unit only (fe_stream_f0e.cu .. fe_stream_f3.cu)
extern template cudaError_t launch_frontend_stream_shape<0, 32, 3, 4>(const FeParams &, int, bool, int, cudaStream_t);
extern template cudaError_t launch_frontend_stream_shape<1, 16, 8, 1>(const FeParams &, int, bool, int, cudaStream_t);
extern template cudaError_t launch_frontend_stream_shape<2, 16, 8, 1>(const FeParams &, int, bool, int, cudaStream_t);
extern template cudaError_t launch_frontend_stream_shape<3, 16, 8, 1>(const FeParams &, int, bool, int, cudaStream_t);

} // namespace aisgpu
