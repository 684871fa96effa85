// be_sym.cu -- symbol timing + bit decoders: PhaseSearch[EMA], AIS::Decoder x 5 with the Reset cross-connect, SimplePLL.
#include "exact.cuh"
#include "params.h"
#include "dec_core.cuh"
#include <cstdlib>

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// K3: symbol timing + demodulation + bit decoder.
//   ModelDefault : ScatterPLL (DSP.h:95-117) -> 5 x PhaseSearchEMA / PhaseSearch (Demod.cpp:39-170) -> 5 x Decoder
//   ModelStandard: Deinterleave (DSP.h:65-73) -> 5 x Decoder
//   ModelBase    : SimplePLL (DSP.cpp:28-57) -> 1 x Decoder
// One thread per (row, sampling phase); the five phases of a row sit in five adjacent lanes of one warp so the
// decoder's Reset broadcast (AIS.cpp:47-49, Model.cpp:566-573) is a warp vote.  Frame bits live in shared memory.
// ---------------------------------------------------------------------------------------------
__constant__ float c_ps_cos[8];
__constant__ float c_ps_sin[8];

// ---------------------------------------------------------------------------------------------
// K3a: PhaseSearchEMA / PhaseSearch (Demod.cpp:39-170), hypothesis-parallel.  Half a warp per (row, sampling
// phase): lane h owns hypothesis h (its EMA / 12-sample history and its last 5 sign decisions); the +-1 (+-2)
// neighbourhood argmax is three (five) shuffles.  The only thing leaving the kernel is one bit per symbol.
// ---------------------------------------------------------------------------------------------

__global__ void __launch_bounds__(PS_THREADS) k_phase_search(const K3Params p) {
	__shared__ float2 tile[PS_THREADS / 32][2][2 * K3_ROWLEN];
	const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
	const int half = lane >> 4, h = lane & 15;
	const long long ninst = (long long)p.rows * 5;
	const long long warp_global = (long long)blockIdx.x * (PS_THREADS / 32) + wib;
	const long long inst = warp_global * 2 + half;
	const bool active = inst < ninst;
	const int row = active ? (int)(inst / 5) : 0, phase = active ? (int)(inst - (long long)row * 5) : 0;
	const unsigned hmask = 0xffffu << (half * 16);
	const int j = h < 8 ? h : 15 - h;
	const float cj = c_ps_cos[j];
	const float sj = h < 8 ? c_ps_sin[j] : -c_ps_sin[j]; // a - b == a + (-b) and im * (-s) == -(im * s), exactly
	const float weight = 0.85f, omw = __fsub_rn(1.0f, 0.85f);

	float ma = 0.0f, mem[12];
	uint32_t hist = 0; // bit d = sign decision of this hypothesis d symbols ago (uint8_t bits[] of the reference, low 5 bits)
	int max_idx = 0, rot = 0, last = 0;
#pragma unroll
	for (int l = 0; l < 12; l++) mem[l] = 0.0f;
	if (active) {
		const PsState &st = p.ps[inst];
		ma = st.ma[h];
#pragma unroll
		for (int dd = 0; dd < 5; dd++) hist |= ((st.plane[dd] >> h) & 1u) << dd;
		max_idx = st.max_idx;
		rot = st.rot;
		last = st.last;
		if (!p.ps_ema) {
#pragma unroll
			for (int l = 0; l < 12; l++) mem[l] = p.ps_mem[(long long)(h * 12 + l) * ninst + inst];
		}
	}
	const int nsamp = p.nsym * 5;
	float2(*mytile)[2 * K3_ROWLEN] = tile[wib];
	// each half stages the samples of its own row
	auto prefetch = [&](int buf, int s0) {
		const int base = s0 * 5;
		if (active) {
			const float2 *src = p.Ec + (long long)row * p.e_stride + p.e_begin + base;
			float2 *dst = &mytile[buf][half * K3_ROWLEN];
			for (int e = h; e < K3_ROWLEN; e += 16)
				if (base + e < nsamp) cp_async_f(dst + e, src + e);
		}
		cp_async_commit();
	};
	const int ntiles = (p.nsym + K3_TS - 1) / K3_TS;
	if (ntiles > 0) prefetch(0, 0);
	for (int t = 0; t < ntiles; t++) {
		if (t + 1 < ntiles) {
			prefetch((t + 1) & 1, (t + 1) * K3_TS);
			cp_async_wait<1>();
		}
		else cp_async_wait<0>();
		__syncwarp();
		const float2 *my = &mytile[t & 1][half * K3_ROWLEN + phase];
		const int s_end = min(K3_TS, p.nsym - t * K3_TS);
		uint32_t word = 0;
		for (int sl = 0; sl < s_end; sl++) {
			const float2 x = my[sl * 5];
			// (1j)^rot pre-rotation (Demod.cpp:44-65), branch free: swap on odd rot, negate on rot >= 2 (sign flips are exact)
			float re = (rot & 1) ? -x.y : x.x, im = (rot & 1) ? x.x : x.y;
			if (rot & 2) { re = -re; im = -im; }
			rot = (rot + 1) & 3;
			const float tt = __fadd_rn(__fmul_rn(re, cj), __fmul_rn(im, sj));
			hist = (hist << 1) | (tt > 0.0f ? 1u : 0u);
			const float at = fabsf(tt);
			if (p.ps_ema) { // Demod.cpp:67-91
				ma = __fadd_rn(__fmul_rn(weight, ma), __fmul_rn(omw, at));
				const int i0 = (max_idx - 1) & 15;
				const float v0 = __shfl_sync(0xffffffffu, ma, half * 16 + i0);
				const float v1 = __shfl_sync(0xffffffffu, ma, half * 16 + ((i0 + 1) & 15));
				const float v2 = __shfl_sync(0xffffffffu, ma, half * 16 + ((i0 + 2) & 15));
				float mv = v0;
				int best = i0;
				if (v1 > mv) { mv = v1; best = (i0 + 1) & 15; }
				if (v2 > mv) { mv = v2; best = (i0 + 2) & 15; }
				max_idx = best;
			}
			else { // Demod.cpp:129-160: ring slot `last` takes |t|, sums run over slots 0..11 in slot order
#pragma unroll
				for (int l = 0; l < 12; l++) mem[l] = (l == last) ? at : mem[l];
				last = (last + 1) % 12;
				float avg = mem[0];
#pragma unroll
				for (int l = 1; l < 12; l++) avg = __fadd_rn(avg, mem[l]);
				float mv = 0.0f;
				const int prev_max = max_idx;
#pragma unroll
				for (int q = -2; q <= 2; q++) {
					const int jj = (prev_max + q) & 15;
					const float v = __shfl_sync(0xffffffffu, avg, half * 16 + jj);
					if (v > mv) { mv = v; max_idx = jj; }
				}
			}
			const uint32_t hb = __shfl_sync(0xffffffffu, hist, half * 16 + max_idx);
			const uint32_t bit = ((hb >> 3) ^ (hb >> 4)) & 1u; // nDelay = 3 (Model.h:219)
			word |= bit << sl;
			if (p.tap_dec && active && h == 0) p.tap_dec[inst * p.nsym + t * K3_TS + sl] = bit ? 1.0f : -1.0f;
		}
		if (active && h == 0) p.dbits[inst * p.dwords + t] = word;
		if (active && phase == 0 && p.mode_level) { // ScatterPLL level: ((((0+n0)+n1)+n2)+n3)+n4, then / 5
			const float2 *rowt = &mytile[t & 1][half * K3_ROWLEN];
			for (int sl = h; sl < s_end; sl += 16) {
				float acc = 0.0f;
#pragma unroll
				for (int jx = 0; jx < 5; jx++) {
					const float2 x = rowt[sl * 5 + jx];
					acc = __fadd_rn(acc, __fadd_rn(__fmul_rn(x.x, x.x), __fmul_rn(x.y, x.y)));
				}
				p.lvl[(long long)row * p.lvl_stride + t * K3_TS + sl] = __fdiv_rn(acc, 5.0f);
			}
		}
		__syncwarp();
	}
	if (active) {
		PsState &st = p.ps[inst];
		st.ma[h] = ma;
#pragma unroll
		for (int dd = 0; dd < 5; dd++) {
			const uint32_t pl = __ballot_sync(hmask, (hist >> dd) & 1u) >> (half * 16);
			if (h == 0) st.plane[dd] = pl;
		}
		if (h == 0) { st.max_idx = max_idx; st.rot = rot; st.last = last; }
		if (!p.ps_ema) {
#pragma unroll
			for (int l = 0; l < 12; l++) p.ps_mem[(long long)(h * 12 + l) * ninst + inst] = mem[l];
		}
	}
}

// ---------------------------------------------------------------------------------------------
// K3a': PhaseSearchEMA (Demod.cpp:39-101) with four hypotheses per lane.  A one-warp CTA owns eight consecutive (row, sampling
// phase) instances, four lanes each (lane q holds hypotheses 4q .. 4q+3: their EMAs and their sign histories).  Per symbol:
//   * t, |t| and the EMA update of the lane's four hypotheses -- plain per-lane arithmetic in the reference's order;
//   * the (1j)^rot pre-rotation costs nothing: symbols are walked in groups of four, the kernel is instantiated per value of
//     rot at the start of the submit (the host knows it: symbols delivered so far & 3), so which of (x.re, x.im) feeds "re" is
//     static and the signs go into the constants (-(x) * c == x * (-c) exactly);
//   * (1 - w) * |t| is taken as |(1 - w) * t| -- the absolute value rides as an operand modifier on the following add;
//   * the neighbourhood argmax "best of (i0, i0+1, i0+2)" is evaluated lazily: the lanes put their EMAs into shared memory (one
//     16-byte store per lane and symbol) and only the three values around the previous maximum are read back and compared
//     (Demod.cpp:80-91), with no shuffle on the sequential chain;
//   * the stores of group g and the lookups of group g - 1 sit between the same two __syncwarp()s, so the sequential chain
//     (address from max_idx -> three loads -> two compares -> max_idx) of one group runs under the arithmetic of the next;
//   * the lane that holds hypothesis max_idx contributes the demodulated bit (its decisions 3 and 4 symbols ago, XORed).
// One hypothesis per lane (16 lanes per instance) and eight per lane (2 lanes) were both slower than four lanes at 1024 x 131072
// @1536K on the previous target (not re-measured on the H100): below four lanes the per-warp dependency chains are no longer
// hidden by other warps.  Demod::PhaseSearch (PS_EMA off) keeps the one-hypothesis-per-lane kernel above.
// ---------------------------------------------------------------------------------------------
constexpr int PS2_INST = 8;                   // (row, phase) instances per warp; a CTA is ONE warp -- no CTA barrier anywhere
constexpr int PS2_TROWS = 3;                  // rows eight consecutive instances can touch
constexpr int PS2_ROWP = K3_ROWLEN + 5;       // padded tile row: the instances of a warp read different banks
constexpr int PS3_G = 4;        // symbols per group
constexpr int PS3_STRIDE = 20;  // floats per (instance, symbol): 16 EMAs, the first two again (the window wraps), 2 unused
template <int R0>
__global__ void __launch_bounds__(32, 28) k_phase_search_ema4b(const K3Params p) { // 61 registers, no spills: left alone ptxas takes 110 and the 1280 one-warp CTAs of the bench shape no longer fit next to the other kernels' CTAs
	__shared__ float2 tile[2][PS2_TROWS][PS2_ROWP];
	__shared__ __align__(16) float mav[2][PS3_G][PS2_INST][PS3_STRIDE];
	const int lane = threadIdx.x;
	const long long ninst = (long long)p.rows * 5;
	const long long inst0 = (long long)blockIdx.x * PS2_INST; // first instance of this warp
	const int il = lane >> 2;                              // instance within the warp
	const long long gi = inst0 + il;
	const int q = lane & 3, q4 = 4 * q;                    // hypothesis group
	const bool active = gi < ninst;
	const long long inst = active ? gi : ninst - 1;
	const int row = (int)(inst / 5), phase = (int)(inst - (long long)row * 5);
	const int r_lo = (int)(inst0 / 5);                    // first row the warp touches
	const int rin = row - r_lo;
	auto or4 = [](uint32_t v) {
		v |= __shfl_xor_sync(0xffffffffu, v, 1);
		v |= __shfl_xor_sync(0xffffffffu, v, 2);
		return v;
	};
	const float weight = 0.85f, omw = __fsub_rn(1.0f, 0.85f);
	float cj[4], sj[4];
#pragma unroll
	for (int k = 0; k < 4; k++) {
		const int h = 4 * q + k, j = h < 8 ? h : 15 - h;
		cj[k] = c_ps_cos[j];
		sj[k] = h < 8 ? c_ps_sin[j] : -c_ps_sin[j]; // a - b == a + (-b) and im * (-s) == -(im * s), exactly
	}
	const c64 cP01 = pack2(cj[0], cj[1]), cP23 = pack2(cj[2], cj[3]), sP01 = pack2(sj[0], sj[1]), sP23 = pack2(sj[2], sj[3]);
	const c64 cN01 = pack2(-cj[0], -cj[1]), cN23 = pack2(-cj[2], -cj[3]), sN01 = pack2(-sj[0], -sj[1]), sN23 = pack2(-sj[2], -sj[3]);
	const c64 w2 = pack2(weight, weight), o2 = pack2(omw, omw);
	float ma[4] = { 0.f, 0.f, 0.f, 0.f };
	uint32_t hist = 0u; // nibble d (bits 4d .. 4d+3) = the sign decisions of the lane's four hypotheses d symbols ago
	int max_idx = 0;
	if (active) {
		const PsState &st = p.ps[inst];
#pragma unroll
		for (int k = 0; k < 4; k++) ma[k] = st.ma[4 * q + k];
#pragma unroll
		for (int dd = 0; dd < 5; dd++) hist |= ((st.plane[dd] >> (4 * q)) & 0xfu) << (4 * dd);
		max_idx = st.max_idx;
	}
	const int nsamp = p.nsym * 5;
	// a tile row is K3_ROWLEN = 5 x 32 samples: five 8-byte copies per lane and row, no index arithmetic beyond the row's base
	static_assert(K3_ROWLEN == 5 * 32, "tile row = five warp-wide copies");
	const float2 *rowsrc[PS2_TROWS];
#pragma unroll
	for (int r = 0; r < PS2_TROWS; r++) rowsrc[r] = p.Ec + (long long)min(r_lo + r, p.rows - 1) * p.e_stride + p.e_begin + lane;
	auto prefetch = [&](int buf, int s0) {
		const int base = s0 * 5;
		if (base + K3_ROWLEN <= nsamp) { // a whole tile (all but the submit's last one)
#pragma unroll
			for (int r = 0; r < PS2_TROWS; r++)
				if (r_lo + r < p.rows) {
#pragma unroll
					for (int j = 0; j < 5; j++) cp_async_f(&tile[buf][r][lane + 32 * j], rowsrc[r] + base + 32 * j);
				}
		}
		else {
			for (int e = lane; e < PS2_TROWS * K3_ROWLEN; e += 32) {
				const int r = e / K3_ROWLEN, c = e - r * K3_ROWLEN;
				if (r_lo + r < p.rows && base + c < nsamp) cp_async_f(&tile[buf][r][c], p.Ec + (long long)(r_lo + r) * p.e_stride + p.e_begin + base + c);
			}
		}
		cp_async_commit();
	};
	// one symbol, first half: hypotheses, EMAs, decisions; the EMAs go to shared memory for the lookup half
	uint32_t xm[2][PS3_G]; // bit k: the demodulated bit hypothesis 4q + k would deliver for this symbol (nDelay = 3, Model.h:219)
	auto first_half = [&](const float2 x, const int k, const int buf) {
		const int r = (R0 + k) & 3;
		// (1j)^rot (Demod.cpp:44-65): rot 0: (re, im) = (x.re, x.im); 1: (-x.im, x.re); 2: (-x.re, -x.im); 3: (x.im, -x.re)
		const float X = (r & 1) ? x.y : x.x, Y = (r & 1) ? x.x : x.y;
		const bool nA = r == 1 || r == 2, nB = r >= 2;
		const c64 X2 = pack2(X, X), Y2 = pack2(Y, Y);
		// products two hypotheses per pmul, then the sums, each rounded separately (__fmul_rn / __fadd_rn, never an FMA)
		const float2 a01 = unpack2(pmul(X2, nA ? cN01 : cP01)), a23 = unpack2(pmul(X2, nA ? cN23 : cP23));
		const float2 b01 = unpack2(pmul(Y2, nB ? sN01 : sP01)), b23 = unpack2(pmul(Y2, nB ? sN23 : sP23));
		const float t0 = __fadd_rn(a01.x, b01.x), t1 = __fadd_rn(a01.y, b01.y), t2 = __fadd_rn(a23.x, b23.x), t3 = __fadd_rn(a23.y, b23.y);
		hist <<= 4;
		if (t0 > 0.0f) hist |= 1u;
		if (t1 > 0.0f) hist |= 2u;
		if (t2 > 0.0f) hist |= 4u;
		if (t3 > 0.0f) hist |= 8u;
		{ // ma = weight * ma + (1 - weight) * |t| (Demod.cpp:67-78); (1 - weight) > 0, so (1 - weight) * |t| == |(1 - weight) * t| bit for bit
			const float2 w01 = unpack2(pmul(w2, pack2(ma[0], ma[1]))), w23 = unpack2(pmul(w2, pack2(ma[2], ma[3])));
			const float2 u01 = unpack2(pmul(o2, pack2(t0, t1))), u23 = unpack2(pmul(o2, pack2(t2, t3)));
			ma[0] = __fadd_rn(w01.x, fabsf(u01.x));
			ma[1] = __fadd_rn(w01.y, fabsf(u01.y));
			ma[2] = __fadd_rn(w23.x, fabsf(u23.x));
			ma[3] = __fadd_rn(w23.y, fabsf(u23.y));
		}
		const uint32_t hs = hist >> 12;
		xm[buf][k] = (hs ^ (hs >> 4)) & 0xfu;
		float *mv = &mav[buf][k][il][0];
		*reinterpret_cast<float4 *>(mv + q4) = make_float4(ma[0], ma[1], ma[2], ma[3]);
		if (q == 0) *reinterpret_cast<float2 *>(mv + 16) = make_float2(ma[0], ma[1]);
	};
	// second half: best of (i0, i0+1, i0+2), strict >, the first maximum wins (Demod.cpp:80-91); every lane of the instance
	// evaluates it (same addresses: a broadcast), the lane that holds hypothesis max_idx contributes the demodulated bit
	uint32_t word = 0;
	auto second_half = [&](const int k, const int buf) {
		const int i0 = (max_idx - 1) & 15;
		const float *v = &mav[buf][k][il][i0];
		const float v0 = v[0], v1 = v[1], v2 = v[2];
		const bool p1 = v1 > v0;
		const float mvv = p1 ? v1 : v0;
		const int best = v2 > mvv ? 2 : (p1 ? 1 : 0);
		max_idx = (i0 + best) & 15;
		// xm >> (max_idx - 4q) is 0 unless 0 <= max_idx - 4q < 4 (the funnel shift clamps the distance at 32); its bit 0 enters the
		// word from the top: after 32 symbols the first one sits in bit 0
		const uint32_t sh = __funnelshift_rc(xm[buf][k], 0u, (uint32_t)(max_idx - q4));
		word = __funnelshift_r(word, sh, 1);
	};
	const int ntiles = (p.nsym + K3_TS - 1) / K3_TS;
	if (ntiles > 0) prefetch(0, 0);
	for (int t = 0; t < ntiles; t++) {
		if (t + 1 < ntiles) {
			prefetch((t + 1) & 1, (t + 1) * K3_TS);
			cp_async_wait<1>();
		}
		else cp_async_wait<0>();
		__syncwarp();
		const float2 *my = &tile[t & 1][rin][phase];
		const int s_end = min(K3_TS, p.nsym - t * K3_TS);
		const int ngrp = (s_end + PS3_G - 1) / PS3_G;
		word = 0;
		auto trip = [&](const int g, const int buf) { // buf is a literal at both call sites: xm[][] stays in registers
			const int cnt1 = g < ngrp ? s_end - g * PS3_G : 0;      // symbols of group g (>= 4 except in the last group of the last tile)
			const int cnt2 = g > 0 ? s_end - (g - 1) * PS3_G : 0;   // symbols of group g - 1
			const float2 *x = my + g * (PS3_G * 5);
			if (cnt1 >= PS3_G && cnt2 >= PS3_G) { // the common trip, one basic block: the lookups of group g - 1 run under the arithmetic of group g
#pragma unroll
				for (int k = 0; k < PS3_G; k++) first_half(x[k * 5], k, buf);
#pragma unroll
				for (int k = 0; k < PS3_G; k++) second_half(k, buf ^ 1);
			}
			else {
#pragma unroll
				for (int k = 0; k < PS3_G; k++)
					if (k < cnt1) first_half(x[k * 5], k, buf);
#pragma unroll
				for (int k = 0; k < PS3_G; k++)
					if (k < cnt2) second_half(k, buf ^ 1);
			}
			__syncwarp(); // group g's EMAs are visible to the lookups of the next trip; buffer g & 1 is rewritten two trips later
		};
		if (s_end == K3_TS) { // a whole tile: eight groups, the trip structure is static (no per-trip counts, no per-symbol tests)
			static_assert(K3_TS == 8 * PS3_G, "eight groups per tile");
			auto full_trip = [&](const int g, const int buf) { // first halves of group g, lookups of group g - 1
				const float2 *x = my + g * (PS3_G * 5);
#pragma unroll
				for (int k = 0; k < PS3_G; k++) first_half(x[k * 5], k, buf);
#pragma unroll
				for (int k = 0; k < PS3_G; k++) second_half(k, buf ^ 1);
				__syncwarp();
			};
#pragma unroll
			for (int k = 0; k < PS3_G; k++) first_half(my[k * 5], k, 0);
			__syncwarp();
			for (int g = 1; g < 7; g += 2) {
				full_trip(g, 1);
				full_trip(g + 1, 0);
			}
			full_trip(7, 1);
#pragma unroll
			for (int k = 0; k < PS3_G; k++) second_half(k, 1);
			__syncwarp();
		}
		else {
			for (int g = 0; g <= ngrp; g += 2) {
				trip(g, 0);
				if (g + 1 <= ngrp) trip(g + 1, 1);
			}
		}
		word >>= (32 - s_end) & 31; // a short last tile: the first symbol goes to bit 0
		word = or4(word);
		if (active && q == 0) p.dbits[inst * p.dwords + t] = word;
		if (p.tap_dec && active) { // decoder input tap: one float per symbol, eight symbols per lane of the instance
			for (int sx = 8 * q; sx < min(8 * q + 8, s_end); sx++) p.tap_dec[inst * p.nsym + t * K3_TS + sx] = ((word >> sx) & 1u) ? 1.0f : -1.0f;
		}
		if (p.mode_level) { // ScatterPLL level: ((((0+n0)+n1)+n2)+n3)+n4, then / 5 (DSP.h:100-106), by the warp that holds the row's phase 0
#pragma unroll
			for (int r = 0; r < PS2_TROWS; r++) {
				const long long first = (long long)(r_lo + r) * 5; // the row's phase-0 instance
				if (first >= inst0 && first < inst0 + PS2_INST && r_lo + r < p.rows && lane < s_end) {
					const float2 *rowt = &tile[t & 1][r][lane * 5];
					float acc = 0.0f;
#pragma unroll
					for (int jx = 0; jx < 5; jx++) {
						const float2 xx = rowt[jx];
						acc = __fadd_rn(acc, __fadd_rn(__fmul_rn(xx.x, xx.x), __fmul_rn(xx.y, xx.y)));
					}
					p.lvl[(long long)(r_lo + r) * p.lvl_stride + t * K3_TS + lane] = __fdiv_rn(acc, 5.0f);
				}
			}
		}
		__syncwarp();
	}
	// state back: the bit planes are OR-combined over the four lanes of the instance
	uint32_t planes[5];
#pragma unroll
	for (int dd = 0; dd < 5; dd++) planes[dd] = or4(((hist >> (4 * dd)) & 0xfu) << (4 * q));
	if (active) {
		PsState &st = p.ps[inst];
#pragma unroll
		for (int k = 0; k < 4; k++) st.ma[4 * q + k] = ma[k];
		if (q == 0) {
#pragma unroll
			for (int dd = 0; dd < 5; dd++) st.plane[dd] = planes[dd];
			st.max_idx = max_idx;
			st.rot = (R0 + p.nsym) & 3;
		}
	}
}

// positions at which Decoder::cannotBeValid (AIS.cpp:111-142) can fire: 30 62 96 168 184 192 336 385 448,
// plus MAX_FRAME_BITS (AIS.h:172) -- one bit per frame position
__constant__ uint32_t c_abort_bits[35];

// Outside a frame the decoder is a tiny automaton; q encodes it in one register:
//   q = 0..5   TRAINING with min(position, 5) alternations seen (only "position > 4" is ever tested, AIS.h:105-113)
//   q = 8..14  STARTFLAG with position = q - 7 (AIS.h:116-137)
__device__ __forceinline__ int dec_q_from_state(const DecState &d) {
	return d.state == ST_TRAINING ? min(d.position, 5) : (d.state == ST_STARTFLAG ? 7 + d.position : 0);
}

// K3b: the five AIS::Decoder instances of one row (AIS.h:91-181) in lanes 0..4 of one warp, one symbol per
// iteration for all of them.  Every lane runs the same straight-line code each symbol -- the out-of-frame automaton
// (one table lookup) and the in-frame bit collector (bits gathered in a register, flushed to shared memory once per
// 32) are both evaluated and masked -- so a row costs the same whether or not it is collecting a frame; only the
// rare events (frame start, word flush, abort positions, closing flag + CRC + Reset vote) branch.

template <int MODEL>
__global__ void __launch_bounds__(DK_THREADS) k_decode(const K3Params p) {
	__shared__ uint32_t frames_all[DK_THREADS / 32][DEC_WORDS * 32];
	__shared__ float tile_all[DK_THREADS / 32][2][K3_ROWLEN]; // MODEL 0: the row's FIR37 samples; MODEL 2: its 32 symbol levels
	__shared__ uint8_t lut_all[DK_THREADS / 32][64];
	const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
	const int row = blockIdx.x * (DK_THREADS / 32) + wib;
	if (row >= p.rows) return; // whole warp
	const int phase = lane;
	const bool active = lane < 5;
	float(*tile)[K3_ROWLEN] = tile_all[wib];
	// transition table of the out-of-frame automaton, index (q << 2) | (alt << 1) | Bit:
	// bits 0-3 next q, bit 4 TRAINING->STARTFLAG (start_idx is taken), bit 5 0111111|0 seen: the frame starts
	uint8_t *lut = lut_all[wib];
	for (int i = lane; i < 64; i += 32) {
		const int qq = i >> 2, al = (i >> 1) & 1, bt = i & 1;
		int qn;
		if (qq < 8) qn = al ? min(qq + 1, 5) : (qq == 5 ? 8 + 2 * bt : 0);  // TRAINING (AIS.h:103-114)
		else qn = qq == 14 ? (bt ? 0 : 15) : (bt ? qq + 1 : 0);             // STARTFLAG (AIS.h:116-137)
		const int to_sf = qq < 8 && qn >= 8, enter = qn == 15;
		lut[i] = (uint8_t)((enter ? 0 : qn) | (to_sf << 4) | (enter << 5));
	}
	__syncwarp();

	DecCtx ctx;
	ctx.frame = frames_all[wib] + lane;
	ctx.mode_level = p.mode_level;
	ctx.stride = K3_THREADS;
	DecState d;
	const int sidx = row * 5 + (active ? phase : 0);
	const long long nthr_total = (long long)p.rows * 5;
	if (active) {
		d = p.dec[sidx];
		for (int w = 0; w < DEC_WORDS; w++) ctx.frame[w * K3_THREADS] = p.dec_data[(long long)w * nthr_total + sidx];
	}
	else {
		d.state = ST_TRAINING; d.lastBit = 0; d.prev = 0; d.position = 0; d.one_seq = 0; d.level = 0.f; d.start_idx = 0;
	}
	const long long clk0 = clock64();
	int n_slow = 0, n_crc = 0, n_crcbits = 0;
	int in_data = active && d.state == ST_DATAFCS;
	int q = dec_q_from_state(d);
	int prev = d.prev, lastBit = d.lastBit;
	int pos = in_data ? d.position : 0, ones = in_data ? d.one_seq : 0;
	float level = d.level;
	uint32_t cur = in_data ? ctx.frame[(pos >> 5) * K3_THREADS] : 0u; // the partially filled frame word
	int start_rel = -1; // slot*5+phase of the most recent TRAINING -> STARTFLAG transition in this submit
	// slots in which this phase has a sample (Deinterleave forwards partial groups at both ends of a submit)
	const int lo_rel = (int)(p.abs_lo - p.abs_begin), hi_rel = (int)(p.abs_hi - p.abs_begin);
	const int slot_lo = phase >= lo_rel ? 0 : 1;
	const int slot_hi = (hi_rel - phase + 4) / 5;
	const int per_sym = MODEL == 2 ? 1 : 5;
	const int nelem = p.nsym * per_sym;
	const float *src_row = MODEL == 2 ? p.lvl + (long long)row * p.lvl_stride : p.Ef + (long long)row * p.e_stride + p.e_begin;
	auto prefetch = [&](int buf, int s0) {
		const int base = s0 * per_sym;
		for (int e = lane; e < K3_TS * per_sym; e += 32)
			if (base + e < nelem) cp_async_f(&tile[buf][e], src_row + base + e);
		cp_async_commit();
	};
	const int ntiles = (p.nsym + K3_TS - 1) / K3_TS;
	if (ntiles > 0) prefetch(0, 0);
	for (int t = 0; t < ntiles; t++) {
		if (t + 1 < ntiles) {
			prefetch((t + 1) & 1, (t + 1) * K3_TS);
			cp_async_wait<1>();
		}
		else cp_async_wait<0>();
		__syncwarp();
		const int s_end = min(K3_TS, p.nsym - t * K3_TS);
		// decision bits and validity of this lane's 32 slots
		uint32_t dword = 0, vword = 0;
		if (MODEL == 2) {
			if (active) {
				dword = p.dbits[(long long)sidx * p.dwords + t];
				vword = s_end >= 32 ? 0xffffffffu : ((1u << s_end) - 1u);
			}
		}
		else if (active) {
			const float *my = &tile[t & 1][phase];
			for (int sl = 0; sl < s_end; sl++) {
				const int slot = t * K3_TS + sl;
				const float bsmp = my[sl * 5];
				const bool valid = slot >= slot_lo && slot < slot_hi;
				dword |= (bsmp > 0.0f ? 1u : 0u) << sl;
				vword |= (valid ? 1u : 0u) << sl;
			}
		}
		for (int sl = 0; sl < s_end; sl++) {
			const int dd = (dword >> sl) & 1u;
			const int valid = (vword >> sl) & 1u;
			const int Bit = 1 ^ dd ^ prev; // NRZI (AIS.h:93-96)
			const int lastBit_before = lastBit;
			const int alt = Bit ^ lastBit_before;
			const int tv = lut[(q << 2) | (alt << 1) | Bit];
			const int upd = valid & (in_data ^ 1), dat = valid & in_data;
			const int start_before = start_rel;
			const float level_before = level;
			// ---- out of frame: TRAINING / STARTFLAG automaton ----
			const int ev = upd ? (tv >> 4) : 0; // bit 0: start_idx taken, bit 1: the frame starts
			start_rel = (ev & 1) ? (t * K3_TS + sl) * 5 + phase : start_rel;
			q = upd ? (tv & 15) : q;
			// ---- in frame: DATAFCS (AIS.h:141-175) ----
			const int five = ones == 5;
			const int append = dat & ((five & (Bit ^ 1)) ^ 1); // a 0 after five 1s is a stuffing bit and is dropped
			cur |= (uint32_t)(append & Bit) << (pos & 31);
			const int pos_n = pos + append;
			if (MODEL == 2) {
				const float lv = tile[t & 1][sl];
				level = (dat && ctx.mode_level) ? __fadd_rn(level, lv) : level;
			}
			ones = dat ? (Bit ? ones + 1 : 0) : ones;
			const int closing = dat & Bit & five; // sixth 1 in a row: closing flag (AIS.h:151-161)
			const int full = append & ((pos_n & 31) == 0);
			const int abortpos = dat & ((c_abort_bits[pos_n >> 5] >> (pos_n & 31)) & 1u);
			pos = pos_n;
			prev = valid ? dd : prev;
			lastBit = valid ? Bit : lastBit;
			if ((ev >> 1) | full | abortpos) { // lane-local rare events
				if (ev >> 1) { // 0111111|0: the frame starts (AIS.h:120-124)
					in_data = 1;
					q = 0;
					pos = 0; ones = 0; level = 0.0f; cur = 0u;
					d.start_idx = start_rel >= 0 ? p.abs_begin + start_rel : d.start_idx;
					for (int w = 0; w < DEC_WORDS; w++) ctx.frame[w * K3_THREADS] = 0u; // msg.clear()
				}
				if (full) {
					ctx.frame[((pos >> 5) - 1) * K3_THREADS] = cur;
					cur = 0u;
				}
				if (abortpos && !closing) { // position == MaxBits || cannotBeValid(position) (AIS.h:172)
					if (pos & 31) ctx.frame[(pos >> 5) * K3_THREADS] = cur;
					if (pos == MAX_FRAME_BITS || dec_cannot_be_valid(ctx, pos)) { in_data = 0; q = 0; }
				}
			}
			const unsigned closers = __ballot_sync(0xffffffffu, closing);
			if (!closers) continue;
			// ---- some decoder of the row saw a closing flag: CRC, frame emission, Reset of the siblings ----
			n_slow++;
			int fr_len = 0;
			float fr_level = 0.0f;
			bool found = false;
			if (closing) {
				if (pos & 31) ctx.frame[(pos >> 5) * K3_THREADS] = cur;
				fr_level = ctx.mode_level ? __fdiv_rn(level, (float)pos) : 0.0f;
				const int len = pos - 7;
				if (len >= 16 && dec_crc16(ctx, len)) {
					found = true;
					fr_len = len;
				}
				in_data = 0;
				q = 0;
				if (p.dbg) { n_crc++; n_crcbits += len > 0 ? len : 0; }
			}
			const unsigned vote = __ballot_sync(0xffffffffu, found);
			if (vote) { // FOUNDMESSAGE -> Reset to the four sibling decoders (AIS.cpp:47-49,98-108)
				const int winner = __ffs(vote) - 1; // lowest phase runs first (DSP.h:108-112)
				const int rel = (t * K3_TS + sl) * 5 + phase;
				if (lane == winner) {
					float ppm = 0.0f;
					if (MODEL == 2 && p.ppmtab) { // tag.ppm of the CGF block that delivered the group's 5th sample
						const long long last_of_group = p.abs_begin + (long long)(t * K3_TS + sl) * 5 + 4;
						int bi = (int)((last_of_group - p.blk_abs0) >> 9);
						bi = bi < 0 ? 0 : (bi >= p.nblk ? p.nblk - 1 : bi);
						ppm = p.ppmtab[p.stepidx[row * p.nblk + bi]];
					}
					emit_frame(p.ring, p.ring_head, p.ring_limit, p.ring_cap, p.chunk, p.blk, ctx, row, phase, fr_len, fr_level, ppm, d.start_idx, p.abs_begin + rel);
				}
				else if (active && (lane < winner || !valid)) { // already stepped this symbol (or no sample in this slot), then reset
					in_data = 0;
					q = 0;
				}
				else if (active) { // reset first, then step this symbol from TRAINING/0: only the NRZI memory survives
					in_data = 0;
					level = level_before;
					start_rel = start_before;
					q = alt ? 1 : 0;
				}
			}
		}
		__syncwarp();
	}
	if (p.dbg) {
		const long long dt = clock64() - clk0;
		for (int o = 16; o > 0; o >>= 1) {
			n_crc += __shfl_xor_sync(0xffffffffu, n_crc, o);
			n_crcbits += __shfl_xor_sync(0xffffffffu, n_crcbits, o);
		}
		if (lane == 0) {
			p.dbg[row * 4 + 0] = dt;
			p.dbg[row * 4 + 1] = n_slow;
			p.dbg[row * 4 + 2] = n_crc;
			p.dbg[row * 4 + 3] = n_crcbits;
		}
	}
	if (active) {
		if (in_data) {
			d.state = ST_DATAFCS;
			d.position = pos;
			d.one_seq = ones;
			if (pos & 31) ctx.frame[(pos >> 5) * K3_THREADS] = cur; // keep the partial word with the persisted frame
		}
		else if (q < 8) { d.state = ST_TRAINING; d.position = q; d.one_seq = 0; }
		else { d.state = ST_STARTFLAG; d.position = q - 7; d.one_seq = 0; }
		if (!in_data && q >= 8 && start_rel >= 0) d.start_idx = p.abs_begin + start_rel;
		d.level = level;
		d.prev = prev;
		d.lastBit = lastBit;
		for (int w = 0; w < DEC_WORDS; w++) p.dec_data[(long long)w * nthr_total + sidx] = ctx.frame[w * K3_THREADS];
		p.dec[sidx] = d;
	}
}
// K3c: the five decoders of a row, fully word-parallel.  Every state of AIS::Decoder::Run (AIS.h:91-181) consumes a
// run of bits of the 32-symbol word with bitwise operations instead of one step per bit:
//   TRAINING  : candidate TRAINING->STARTFLAG transitions are  E = ~alt & alt<<1 & .. & alt<<5  (a repeat after five
//               alternations); one counts only if its five alternations come after the last reset (index e).  What
//               STARTFLAG does with it is read off the next bits (count of ones that follow) in the same iteration.
//   STARTFLAG : only when a flag straddles a word boundary: position so far in sfP.
//   DATAFCS   : closing flag = first run of six ones (carry-in `ones` prepended), stuffing bits = zeros after five
//               ones, both by shifted ANDs; the surviving bits are squeezed together and appended to the frame;
//               the cannotBeValid()/MaxBits exits (AIS.cpp:111-142) are evaluated only when the position crosses one
//               of their lengths; the signal level is summed bit by bit in the reference's order.
// A CRC-valid frame is rare; when one closes in a word, the row rolls back to the state at the start of the word
// section, replays it up to that bit (its siblings one bit less if they come later in the round-robin order of
// DSP.h:108-112), applies the Reset broadcast (AIS.cpp:47-49, Model.cpp:566-573) and carries on.
struct Dk3 {
	int mode;        // 0 TRAINING, 1 STARTFLAG, 2 DATAFCS
	int sfP;         // STARTFLAG: position (1..7)
	int pos, ones;   // DATAFCS: position, one_seq_count
	float level;
	uint32_t cur;    // partially filled frame word
	int e;           // TRAINING: alternations count only at bit indices > e (relative to the current word)
	int start_rel;   // slot*5+phase of the latest TRAINING->STARTFLAG transition of this submit, -1 if none
};

__device__ __forceinline__ uint32_t lowmask(int n) { return n >= 32 ? 0xffffffffu : ((1u << n) - 1u); }

// Consumes bits [i0, i1) of the word.  Returns 32, or the index of the bit at which a CRC-valid frame closed (the
// state is then TRAINING with e = that bit, the frame bits are complete in shared memory, fr_len / fr_level set).
template <bool LEVEL>
__device__ __forceinline__ int dk3_run(Dk3 &st, const DecCtx &ctx, uint32_t Bitw, uint32_t E, int i0, int i1, const float *__restrict__ lvl,
									   int slot0, int phase, int &fr_len, float &fr_level) {
	int i = i0;
	while (i < i1) {
		if (st.mode == 0) {
			uint32_t Em = E & ~lowmask(i) & lowmask(i1);
			bool done = true;
			while (Em) {
				const int j = __ffs(Em) - 1;
				Em &= Em - 1;
				if (j - 5 <= st.e) continue; // some of the five alternations precede the last reset
				// TRAINING -> STARTFLAG at bit j (AIS.h:107-111); position = Bit ? 3 : 1
				st.start_rel = (slot0 + j) * 5 + phase;
				const int b = (Bitw >> j) & 1;
				const int need = b ? 4 : 6; // ones still to come before the 0 that ends the flag
				const int n = i1 - (j + 1);
				const uint32_t W = n > 0 ? ((Bitw >> (j + 1)) | ~lowmask(n)) : 0xffffffffu; // j + 1 may be 32
				const int t1 = ~W ? __ffs(~W) - 1 : 32; // ones that follow
				const int m = min(t1, need);
				if (m >= n) { // the word ends inside the flag
					st.mode = 1;
					st.sfP = (b ? 3 : 1) + n;
					i = i1;
					done = false;
					break;
				}
				const int decide = j + 1 + m;
				if (t1 == need) { // 0111111|0: the frame starts (AIS.h:120-124)
					st.mode = 2;
					st.pos = 0; st.ones = 0; st.level = 0.0f; st.cur = 0u;
					i = decide + 1;
					done = false;
					break;
				}
				st.e = decide; // the flag failed there: NextState(TRAINING, 0)
			}
			if (done) i = i1;
		}
		else if (st.mode == 1) {
			const int n = i1 - i;
			const uint32_t W = (Bitw >> i) | ~lowmask(n);
			const int t1 = ~W ? __ffs(~W) - 1 : 32;
			const int need = 7 - st.sfP;
			const int m = min(t1, need);
			if (m >= n) {
				st.sfP += n;
				i = i1;
			}
			else {
				const int decide = i + m;
				if (t1 == need) {
					st.mode = 2;
					st.pos = 0; st.ones = 0; st.level = 0.0f; st.cur = 0u;
				}
				else {
					st.mode = 0;
					st.e = decide;
				}
				i = decide + 1;
			}
		}
		else {
			const int n = i1 - i;
			const uint32_t W = (Bitw >> i) & lowmask(n);
			const unsigned long long X = ((unsigned long long)W << st.ones) | ((1ull << st.ones) - 1ull); // carried-in ones first
			const unsigned long long R5 = X & (X << 1) & (X << 2) & (X << 3) & (X << 4);
			const unsigned long long R6 = R5 & (X << 5);
			const int c = R6 ? (__ffsll((long long)R6) - 1 - st.ones) : 64; // closing flag: the sixth 1 in a row (AIS.h:151-161)
			const int endb = c < n ? c : n - 1;                              // last bit consumed if no early exit
			const uint32_t Sw = (uint32_t)((~X & (R5 << 1)) >> st.ones) & lowmask(endb + 1); // stuffing zeros
			uint32_t bits = W & lowmask(endb + 1);
			for (uint32_t tmp = Sw; tmp;) { // squeeze the stuffing bits out, highest first
				const int sb = 31 - __clz((int)tmp);
				tmp &= ~(1u << sb);
				bits = (bits & lowmask(sb)) | ((sb >= 31 ? 0u : (bits >> (sb + 1))) << sb);
			}
			const int cnt = endb + 1 - __popc(Sw);
			const int pos0 = st.pos;
			const int sh = pos0 & 31;
			uint32_t cur = st.cur | (bits << sh);
			if (sh + cnt >= 32) {
				ctx.frame[(pos0 >> 5) * K3_THREADS] = cur;
				cur = sh ? (bits >> (32 - sh)) : 0u;
			}
			const int newpos = pos0 + cnt;
			// exits by length: position == MaxBits || cannotBeValid(position), tested after every bit (AIS.h:172)
			int exit_m = -1;
			{
				const int w0 = (pos0 + 1) >> 5, w1 = newpos >> 5;
				bool any = false;
				for (int w = w0; w <= w1 && w < 35; w++) {
					uint32_t ab = c_abort_bits[w];
					if (w == w0) ab &= ~lowmask((pos0 + 1) & 31);
					if (w == w1) ab &= lowmask((newpos & 31) + 1);
					any |= ab != 0;
				}
				if (any) {
					ctx.frame[(newpos >> 5) * K3_THREADS] = cur; // type / mmsi fields must be readable
					for (int Pa = pos0 + 1; Pa <= newpos; Pa++) {
						if (!((c_abort_bits[Pa >> 5] >> (Pa & 31)) & 1u)) continue;
						const int r = Pa - pos0 - 1; // ordinal of the appended bit that makes position == Pa
						int m = r;
						for (;;) {
							const int m2 = r + __popc(Sw & lowmask(m + 1));
							if (m2 == m) break;
							m = m2;
						}
						if (m == c) break; // closing flag on the same bit: NextState(TRAINING) came first
						if (Pa == MAX_FRAME_BITS || dec_cannot_be_valid(ctx, Pa)) {
							exit_m = m;
							break;
						}
					}
				}
			}
			if (exit_m >= 0) {
				st.mode = 0;
				st.e = i + exit_m;
				i += exit_m + 1;
				continue;
			}
			if (LEVEL && ctx.mode_level) { // level += tag.sample_lvl for every bit in DATAFCS, in order (AIS.h:146-147)
				float lv = st.level;
#pragma unroll
				for (int m = 0; m < 32; m++) {
					const float v = lvl[min(i + m, 31)];
					lv = m <= endb ? __fadd_rn(lv, v) : lv;
				}
				st.level = lv;
			}
			if (c < n) { // closing flag
				if (newpos & 31) ctx.frame[(newpos >> 5) * K3_THREADS] = cur;
				st.mode = 0;
				st.e = i + c;
				i += c + 1;
				const int len = newpos - 7;
				if (len >= 16 && dec_crc16_bytes(ctx, len)) {
					fr_len = len;
					fr_level = ctx.mode_level ? __fdiv_rn(st.level, (float)newpos) : 0.0f;
					st.pos = newpos;
					return i - 1;
				}
			}
			else {
				st.pos = newpos;
				st.cur = cur;
				const int tot = n + st.ones; // trailing ones of the consumed bits (a stuffing zero resets the count)
				const unsigned long long Y = ~(X << (64 - tot));
				st.ones = Y ? __clzll((long long)Y) : tot;
				i = i1;
			}
		}
	}
	return 32;
}


template <int MODEL, int RPW>
__global__ void __launch_bounds__(DK3_WARPS * 32) k_decode3(const K3Params p) {
	__shared__ uint32_t frames_all[DK3_WARPS][DEC_WORDS * 32];
	__shared__ float tile_all[DK3_WARPS][RPW][3][K3_TS];
	const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
	const int g = lane / 5, phase = lane - 5 * g;
	const int row0 = (blockIdx.x * DK3_WARPS + wib) * RPW;
	if (row0 >= p.rows) return; // whole warp
	const int row = row0 + g;
	const bool active = g < RPW && row < p.rows;
	const int gbase = 5 * (g < RPW ? g : 0);
	float(*tile)[3][K3_TS] = tile_all[wib];

	DecCtx ctx;
	ctx.frame = frames_all[wib] + lane;
	ctx.mode_level = p.mode_level;
	ctx.stride = K3_THREADS;
	DecState d;
	const int sidx = active ? row * 5 + phase : 0;
	const long long nthr_total = (long long)p.rows * 5;
	Dk3 st;
	st.mode = 0; st.sfP = 0; st.pos = 0; st.ones = 0; st.level = 0.0f; st.cur = 0u; st.e = -1; st.start_rel = -1;
	int prev = 0, lastBit = 0;
	uint32_t altprev = 0u;
	if (active) {
		d = p.dec[sidx];
		prev = d.prev;
		lastBit = d.lastBit;
		if (d.state == ST_DATAFCS) {
			st.mode = 2;
			st.pos = d.position;
			st.ones = d.one_seq;
			st.level = d.level;
			const int nw = (d.position >> 5) + 1;
			for (int w = 0; w < nw && w < DEC_WORDS; w++) ctx.frame[w * K3_THREADS] = p.dec_data[(long long)w * nthr_total + sidx];
			st.cur = (d.position & 31) ? ctx.frame[(d.position >> 5) * K3_THREADS] : 0u;
		}
		else if (d.state == ST_STARTFLAG) {
			st.mode = 1;
			st.sfP = d.position;
		}
		else { // TRAINING with `position` alternations counted so far (only "> 4" is ever tested)
			const int q = min(d.position, 5);
			st.e = -1 - q;
			altprev = q ? (0xffffffffu << (32 - q)) : 0u;
		}
	}
	const int lo_rel = (int)(p.abs_lo - p.abs_begin), hi_rel = (int)(p.abs_hi - p.abs_begin);
	const int slot_lo = phase >= lo_rel ? 0 : 1; // Deinterleave forwards partial groups at both ends of a submit
	const int slot_hi = (hi_rel - phase + 4) / 5;
	const int ntiles = (p.nsym + K3_TS - 1) / K3_TS;
	auto prefetch = [&](int buf, int s0) {
		if (MODEL == 2) {
#pragma unroll
			for (int g2 = 0; g2 < RPW; g2++) {
				const int r2 = row0 + g2;
				if (r2 < p.rows && s0 + lane < p.nsym) cp_async_f(&tile[g2][buf][lane], p.lvl + (long long)r2 * p.lvl_stride + s0 + lane);
			}
		}
		cp_async_commit();
	};
	auto load_dbits = [&](int t) -> uint32_t { return (active && t < ntiles) ? p.dbits[(long long)sidx * p.dwords + t] : 0u; };
	uint32_t pre0 = load_dbits(0), pre1 = load_dbits(1), pre2 = load_dbits(2);
	if (ntiles > 0) {
		prefetch(0, 0);
		if (ntiles > 1) prefetch(1, K3_TS);
		else cp_async_commit();
	}
	int nbits_total = 0; // valid bits seen by this lane in this submit
	for (int t = 0; t < ntiles; t++) {
		if (t + 2 < ntiles) prefetch((t + 2) % 3, (t + 2) * K3_TS);
		else cp_async_commit();
		cp_async_wait<2>(); // tile t has landed
		__syncwarp();
		uint32_t dword = pre0;
		pre0 = pre1;
		pre1 = pre2;
		pre2 = load_dbits(t + 3);
		// valid slots of this word for this lane: [lo, hi)
		int lo = max(0, slot_lo - t * K3_TS), hi = min(K3_TS, min(p.nsym, slot_hi) - t * K3_TS);
		if (!active) hi = 0;
		const int nb = max(0, hi - lo);
		const int slot0 = t * K3_TS + lo;
		dword >>= lo;
		const uint32_t Bitw = ~(dword ^ ((dword << 1) | (uint32_t)prev)); // NRZI (AIS.h:93-96)
		const uint32_t alt = Bitw ^ ((Bitw << 1) | (uint32_t)lastBit);
		uint32_t run5 = __funnelshift_l(altprev, alt, 1);
		run5 &= __funnelshift_l(altprev, alt, 2);
		run5 &= __funnelshift_l(altprev, alt, 3);
		run5 &= __funnelshift_l(altprev, alt, 4);
		run5 &= __funnelshift_l(altprev, alt, 5);
		const uint32_t E = ~alt & run5 & lowmask(nb);
		const float *lvl = &tile[g < RPW ? g : 0][t % 3][lo];
		int i = 0;
		for (;;) {
			const Dk3 saved = st;
			const int i_saved = i;
			int fr_len = 0;
			float fr_level = 0.0f;
			const int x = dk3_run<MODEL == 2>(st, ctx, Bitw, E, i, nb, lvl, slot0, phase, fr_len, fr_level);
			i = x < 32 ? x + 1 : nb;
			if (!__any_sync(0xffffffffu, x < 32)) break;
			// a frame with a good CRC closed somewhere in the warp: per row, the first one in (bit, phase) order wins
			const int key = x < 32 ? (x + lo) * 8 + phase : 0x7fffffff; // bit index in slot units (lanes of a row may differ in lo)
			int rowmin = 0x7fffffff;
#pragma unroll
			for (int k2 = 0; k2 < 5; k2++) rowmin = min(rowmin, __shfl_sync(0xffffffffu, key, gbase + k2));
			if (rowmin == 0x7fffffff || !active) continue; // nothing in this row: its lanes have finished the word already
			const int xs = rowmin >> 3, pw = rowmin & 7; // slot (relative to the word) and phase of the winner
			if (key == rowmin) { // FOUNDMESSAGE: publish, Reset goes to the four siblings (AIS.cpp:47-49,98-108)
				float ppm = 0.0f;
				const int slot = t * K3_TS + xs;
				if (MODEL == 2 && p.ppmtab) { // tag.ppm of the CGF block that delivered the group's 5th sample
					const long long last_of_group = p.abs_begin + (long long)slot * 5 + 4;
					int bi = (int)((last_of_group - p.blk_abs0) >> 9);
					bi = bi < 0 ? 0 : (bi >= p.nblk ? p.nblk - 1 : bi);
					ppm = p.ppmtab[p.stepidx[row * p.nblk + bi]];
				}
				const long long sidx0 = st.start_rel >= 0 ? p.abs_begin + st.start_rel : d.start_idx;
				FrameRec *rp = ring_claim(p.ring, p.ring_head, p.ring_limit, p.ring_cap);
				if (rp) {
					FrameRec &r = *rp;
					r.row = row; r.phase = phase; r.nbits = fr_len - 16; r.level = fr_level; r.ppm = ppm; r.chunk = p.chunk; r.blk = p.blk;
					r.start_idx = sidx0;
					r.end_idx = p.abs_begin + (long long)slot * 5 + phase;
					const int nw = (st.pos + 31) >> 5;
					for (int w = 0; w < DEC_WORDS; w++) r.data[w] = w < nw ? frame_word(ctx, w) : 0u; // msg.clear() left the rest zero
				}
			}
			else { // sibling: replay up to the winner's bit, then Reset -> NextState(TRAINING, 0)
				st = saved;
				const int xl = xs - lo; // the winner's slot as a bit index of this lane's word (may be -1 when lo = 1)
				const int stop = max(i_saved, min(nb, phase < pw ? xl + 1 : xl)); // earlier phases have already stepped that symbol
				int fl = 0;
				float fv = 0.0f;
				if (stop > i_saved) dk3_run<MODEL == 2>(st, ctx, Bitw, E, i_saved, stop, lvl, slot0, phase, fl, fv);
				st.mode = 0;
				st.e = stop - 1;
				i = stop;
			}
		}
		if (nb > 0) {
			altprev = nb >= 32 ? alt : ((alt << (32 - nb)) | (altprev >> nb)); // keep "bit 31 = latest alternation flag"
			lastBit = (int)((Bitw >> (nb - 1)) & 1u);
			prev = (int)((dword >> (nb - 1)) & 1u);
			st.e = max(st.e - nb, -64);
			nbits_total += nb;
		}
		__syncwarp();
	}
	if (active) {
		if (st.mode == 2) {
			d.state = ST_DATAFCS;
			d.position = st.pos;
			d.one_seq = st.ones;
			if (st.pos & 31) ctx.frame[(st.pos >> 5) * K3_THREADS] = st.cur;
			const int nw = (st.pos >> 5) + 1;
			for (int w = 0; w < nw && w < DEC_WORDS; w++) p.dec_data[(long long)w * nthr_total + sidx] = ctx.frame[w * K3_THREADS];
		}
		else if (st.mode == 1) { d.state = ST_STARTFLAG; d.position = st.sfP; d.one_seq = 0; }
		else { // TRAINING: alternations counted = trailing alternation flags that come after the last reset
			const int n_alt = __clz((int)~altprev);
			d.state = ST_TRAINING;
			d.position = max(0, min(min(5, n_alt), -1 - st.e));
			d.one_seq = 0;
		}
		if (st.mode != 0 && st.start_rel >= 0) d.start_idx = p.abs_begin + st.start_rel;
		d.level = st.level;
		d.prev = prev;
		d.lastBit = lastBit;
		p.dec[sidx] = d;
	}
}

// K3d: ModelChallenger (Model.cpp:601-678): per row FIVE decoders behind the coherent branch (ScatterPLL: a group of five symbols
// is handed out when its fifth sample has arrived) and FIVE behind the FM branch (Deinterleave: every sample is handed out at
// once), all ten cross-connected by the Reset signal.  Both branches hang off one sample-by-sample throttle, so within a
// group of five samples the reference's order is  f0 f1 f2 f3 | a0 a1 a2 a3 a4 | f4  (FM decoder j at sample 5g + j, the
// coherent ones when sample 5g + 4 has passed the FIR).  Same word-parallel machine as k_decode3 with ten lanes per row and
// that rank deciding who has "already stepped" when a frame completes.  The FM decoders see the signal level ScatterPLL
// left in the tag: the previous group's for f0..f3, the current one's for f4 (DSP.h:100-106, the TAG travels by reference --
// across the two channels as well: a row's first group of a block sees the level the other channel's chain left behind).
template <int RPW>
__global__ void __launch_bounds__(DK3_WARPS * 32) k_decode10(const K3Params p) {
	constexpr int MODEL = 2;
	__shared__ uint32_t frames_all[DK3_WARPS][DEC_WORDS * 32];
	__shared__ float tile_all[DK3_WARPS][RPW][3][K3_TS + 2]; // entry 0: the level of the slot in front of the word; +1 over-read slack
	const int tid = threadIdx.x, lane = tid & 31, wib = tid >> 5;
	const int g = lane / 10, ph10 = lane - 10 * g;
	const bool fm = ph10 >= 5;
	const int phase = fm ? ph10 - 5 : ph10;
	const int rank = fm ? (phase < 4 ? phase : 9) : 4 + phase; // order of the ten decoders within a group of five samples
	const int row0 = (blockIdx.x * DK3_WARPS + wib) * RPW;
	if (row0 >= p.rows) return; // whole warp
	const int row = row0 + g;
	const bool active = g < RPW && row < p.rows;
	const int gbase = 10 * (g < RPW ? g : 0);
	float(*tile)[3][K3_TS + 2] = tile_all[wib];

	DecCtx ctx;
	ctx.frame = frames_all[wib] + lane;
	ctx.mode_level = p.mode_level;
	ctx.stride = K3_THREADS;
	DecState d;
	const int sidx = active ? row * 10 + ph10 : 0;
	const long long nthr_total = (long long)p.rows * 10;
	Dk3 st;
	st.mode = 0; st.sfP = 0; st.pos = 0; st.ones = 0; st.level = 0.0f; st.cur = 0u; st.e = -1; st.start_rel = -1;
	int prev = 0, lastBit = 0;
	uint32_t altprev = 0u;
	if (active) {
		d = p.dec[sidx];
		prev = d.prev;
		lastBit = d.lastBit;
		if (d.state == ST_DATAFCS) {
			st.mode = 2;
			st.pos = d.position;
			st.ones = d.one_seq;
			st.level = d.level;
			const int nw = (d.position >> 5) + 1;
			for (int w = 0; w < nw && w < DEC_WORDS; w++) ctx.frame[w * K3_THREADS] = p.dec_data[(long long)w * nthr_total + sidx];
			st.cur = (d.position & 31) ? ctx.frame[(d.position >> 5) * K3_THREADS] : 0u;
		}
		else if (d.state == ST_STARTFLAG) {
			st.mode = 1;
			st.sfP = d.position;
		}
		else { // TRAINING with `position` alternations counted so far (only "> 4" is ever tested)
			const int q = min(d.position, 5);
			st.e = -1 - q;
			altprev = q ? (0xffffffffu << (32 - q)) : 0u;
		}
	}
	const int lo_rel = (int)(p.abs_lo - p.abs_begin), hi_rel = (int)(p.abs_hi - p.abs_begin);
	// FM lanes: Deinterleave forwards partial groups at both ends of a submit; coherent lanes: complete groups only
	const int slot_lo = fm ? (phase >= lo_rel ? 0 : 1) : 0;
	const int slot_hi = fm ? (hi_rel - phase + 4) / 5 : p.nsym;
	const int nslots = max(p.nsym, p.nslots_fm);
	const int ntiles = (nslots + K3_TS - 1) / K3_TS;
	auto prefetch = [&](int buf, int s0) {
#pragma unroll
		for (int g2 = 0; g2 < RPW; g2++) {
			const int r2 = row0 + g2;
			if (r2 >= p.rows) continue;
			for (int e = lane; e < K3_TS + 1; e += 32) { // entry e = level of slot s0 + e - 1
				const int sl = s0 + e - 1;
				if (sl < 0) { // the level the tag carries into this row's first group: the OTHER channel's last group (same TAG object,
					// Rotate feeds channel A's chain, then B's, DSP.cpp:312-313) -- for B the one A has just left in this block; in
					// single-channel mode only the one chain touches the tag: the row's own last level of the previous block
					if ((r2 & 1) && !p.lvl_own) cp_async_f(&tile[g2][buf][e], p.lvl + (long long)(r2 - 1) * p.lvl_stride + p.nsym - 1);
					else cp_async_f(&tile[g2][buf][e], p.lvl_prev + r2);
				}
				else if (sl < p.nsym) cp_async_f(&tile[g2][buf][e], p.lvl + (long long)r2 * p.lvl_stride + sl);
			}
		}
		cp_async_commit();
	};
	const uint32_t *mybits = (fm ? p.dbits2 : p.dbits) + (long long)(row * 5 + phase) * p.dwords;
	auto load_dbits = [&](int t) -> uint32_t { return (active && t < ntiles) ? mybits[t] : 0u; };
	uint32_t pre0 = load_dbits(0), pre1 = load_dbits(1), pre2 = load_dbits(2);
	if (ntiles > 0) {
		prefetch(0, 0);
		if (ntiles > 1) prefetch(1, K3_TS);
		else cp_async_commit();
	}
	int nbits_total = 0; // valid bits seen by this lane in this submit
	for (int t = 0; t < ntiles; t++) {
		if (t + 2 < ntiles) prefetch((t + 2) % 3, (t + 2) * K3_TS);
		else cp_async_commit();
		cp_async_wait<2>(); // tile t has landed
		__syncwarp();
		uint32_t dword = pre0;
		pre0 = pre1;
		pre1 = pre2;
		pre2 = load_dbits(t + 3);
		// valid slots of this word for this lane: [lo, hi)
		int lo = max(0, slot_lo - t * K3_TS), hi = min(K3_TS, min(nslots, slot_hi) - t * K3_TS);
		if (!active) hi = 0;
		const int nb = max(0, hi - lo);
		const int slot0 = t * K3_TS + lo;
		dword >>= lo;
		const uint32_t Bitw = ~(dword ^ ((dword << 1) | (uint32_t)prev)); // NRZI (AIS.h:93-96)
		const uint32_t alt = Bitw ^ ((Bitw << 1) | (uint32_t)lastBit);
		uint32_t run5 = __funnelshift_l(altprev, alt, 1);
		run5 &= __funnelshift_l(altprev, alt, 2);
		run5 &= __funnelshift_l(altprev, alt, 3);
		run5 &= __funnelshift_l(altprev, alt, 4);
		run5 &= __funnelshift_l(altprev, alt, 5);
		const uint32_t E = ~alt & run5 & lowmask(nb);
		const float *lvl = &tile[g < RPW ? g : 0][t % 3][lo + ((fm && phase < 4) ? 0 : 1)];
		int i = 0;
		for (;;) {
			const Dk3 saved = st;
			const int i_saved = i;
			int fr_len = 0;
			float fr_level = 0.0f;
			const int x = dk3_run<MODEL == 2>(st, ctx, Bitw, E, i, nb, lvl, slot0, phase, fr_len, fr_level);
			i = x < 32 ? x + 1 : nb;
			if (!__any_sync(0xffffffffu, x < 32)) break;
			// a frame with a good CRC closed somewhere in the warp: per row, the first one in (bit, phase) order wins
			const int key = x < 32 ? (x + lo) * 16 + rank : 0x7fffffff; // bit index in slot units (lanes of a row may differ in lo)
			int rowmin = 0x7fffffff;
#pragma unroll
			for (int k2 = 0; k2 < 10; k2++) rowmin = min(rowmin, __shfl_sync(0xffffffffu, key, gbase + k2));
			if (rowmin == 0x7fffffff || !active) continue; // nothing in this row: its lanes have finished the word already
			const int xs = rowmin >> 4, pw = rowmin & 15; // slot (relative to the word) and rank of the winner
			if (key == rowmin) { // FOUNDMESSAGE: publish, Reset goes to the four siblings (AIS.cpp:47-49,98-108)
				float ppm = 0.0f;
				const int slot = t * K3_TS + xs;
				if (p.ppmtab) { // tag.ppm of the CGF block that delivered the group's 5th sample (coherent) / this sample (FM)
					const long long last_of_group = p.abs_begin + (long long)slot * 5 + (fm ? phase : 4);
					int bi = (int)((last_of_group - p.blk_abs0) >> 9);
					bi = bi < 0 ? 0 : (bi >= p.nblk ? p.nblk - 1 : bi);
					ppm = p.ppmtab[p.stepidx[row * p.nblk + bi]];
				}
				const long long sidx0 = st.start_rel >= 0 ? p.abs_begin + st.start_rel : d.start_idx;
				FrameRec *rp = ring_claim(p.ring, p.ring_head, p.ring_limit, p.ring_cap);
				if (rp) {
					FrameRec &r = *rp;
					r.row = row; r.phase = ph10; r.nbits = fr_len - 16; r.level = fr_level; r.ppm = ppm; r.chunk = p.chunk; r.blk = p.blk;
					r.start_idx = sidx0;
					r.end_idx = p.abs_begin + (long long)slot * 5 + phase;
					const int nw = (st.pos + 31) >> 5;
					for (int w = 0; w < DEC_WORDS; w++) r.data[w] = w < nw ? frame_word(ctx, w) : 0u; // msg.clear() left the rest zero
				}
			}
			else { // sibling: replay up to the winner's bit, then Reset -> NextState(TRAINING, 0)
				st = saved;
				const int xl = xs - lo; // the winner's slot as a bit index of this lane's word (may be -1 when lo = 1)
				const int stop = max(i_saved, min(nb, rank < pw ? xl + 1 : xl)); // decoders of lower rank have already stepped that group
				int fl = 0;
				float fv = 0.0f;
				if (stop > i_saved) dk3_run<MODEL == 2>(st, ctx, Bitw, E, i_saved, stop, lvl, slot0, phase, fl, fv);
				st.mode = 0;
				st.e = stop - 1;
				i = stop;
			}
		}
		if (nb > 0) {
			altprev = nb >= 32 ? alt : ((alt << (32 - nb)) | (altprev >> nb)); // keep "bit 31 = latest alternation flag"
			lastBit = (int)((Bitw >> (nb - 1)) & 1u);
			prev = (int)((dword >> (nb - 1)) & 1u);
			st.e = max(st.e - nb, -64);
			nbits_total += nb;
		}
		__syncwarp();
	}
	if (active) {
		if (st.mode == 2) {
			d.state = ST_DATAFCS;
			d.position = st.pos;
			d.one_seq = st.ones;
			if (st.pos & 31) ctx.frame[(st.pos >> 5) * K3_THREADS] = st.cur;
			const int nw = (st.pos >> 5) + 1;
			for (int w = 0; w < nw && w < DEC_WORDS; w++) p.dec_data[(long long)w * nthr_total + sidx] = ctx.frame[w * K3_THREADS];
		}
		else if (st.mode == 1) { d.state = ST_STARTFLAG; d.position = st.sfP; d.one_seq = 0; }
		else { // TRAINING: alternations counted = trailing alternation flags that come after the last reset
			const int n_alt = __clz((int)~altprev);
			d.state = ST_TRAINING;
			d.position = max(0, min(min(5, n_alt), -1 - st.e));
			d.one_seq = 0;
		}
		if (st.mode != 0 && st.start_rel >= 0) d.start_idx = p.abs_begin + st.start_rel;
		d.level = st.level;
		d.prev = prev;
		d.lastBit = lastBit;
		p.dec[sidx] = d;
		// ScatterPLL's level stays in the tag for the FM decoders of the next group: keep the last one for the next submit
		if (ph10 == 0 && p.nsym > 0) {
			if (p.lvl_own) p.lvl_prev_out[row] = p.lvl[(long long)row * p.lvl_stride + p.nsym - 1];
			else if (row & 1) p.lvl_prev_out[row - 1] = p.lvl[(long long)row * p.lvl_stride + p.nsym - 1]; // B's last level is what A starts the next block with
		}
	}
}


// ModelBase: SimplePLL (DSP.cpp:28-57) + one Decoder per row; strictly sequential per row.
__global__ void __launch_bounds__(K3_THREADS) k_base(const float *__restrict__ Ef, long long e_stride, int e_begin, int n, int rows,
													   PllState *__restrict__ pll, DecState *__restrict__ dec, uint32_t *__restrict__ dec_data, FrameRec *__restrict__ ring,
													   unsigned long long *__restrict__ ring_head, unsigned long long ring_limit, int ring_cap, int chunk, int blk, float *__restrict__ tap_dec,
													   int *__restrict__ tap_cnt) {
	__shared__ uint32_t frames[DEC_WORDS * K3_THREADS];
	const int tid = threadIdx.x;
	const int row = blockIdx.x * K3_THREADS + tid;
	if (row >= rows) return;
	DecCtx ctx;
	ctx.frame = frames + tid;
	ctx.mode_level = 1;
	ctx.stride = K3_THREADS;
	DecState d = dec[row * 5];
	const long long nthr_total = (long long)rows * 5;
	for (int w = 0; w < DEC_WORDS; w++) frames[w * K3_THREADS + tid] = dec_data[(long long)w * nthr_total + row * 5];
	PllState pl = pll[row];
	const float *e = Ef + (long long)row * e_stride + e_begin;
	int ntap = 0;
	for (int i = 0; i < n; i++) {
		const float x = e[i];
		const int bit = x > 0.0f;
		if (bit != pl.prev) pl.pll = __fadd_rn(pl.pll, __fmul_rn(__fsub_rn(0.5f, pl.pll), pl.fast ? 0.6f : 0.05f));
		pl.pll = __fadd_rn(pl.pll, 0.2f);
		if (pl.pll >= 1.0f) {
			if (tap_dec) tap_dec[(long long)row * n + ntap++] = x;
			int fr_len = 0, lb = 0;
			float fr_level = 0.f;
			const bool found = dec_step(d, ctx, x, 0.0f, 0, fr_len, fr_level, lb);
			if (found) emit_frame(ring, ring_head, ring_limit, ring_cap, chunk, blk, ctx, row, 0, fr_len, fr_level, 0.0f, d.start_idx, 0);
			// DecoderMessage -> SimplePLL::Signal (Model.cpp:434-435; DSP.cpp:46-57): the last NextState decides
			pl.fast = (d.state == ST_TRAINING) ? 1 : (d.state == ST_STARTFLAG ? 0 : pl.fast);
			pl.pll = __fsub_rn(pl.pll, (float)(int)pl.pll);
		}
		pl.prev = bit;
	}
	for (int w = 0; w < DEC_WORDS; w++) dec_data[(long long)w * nthr_total + row * 5] = frames[w * K3_THREADS + tid];
	dec[row * 5] = d;
	pll[row] = pl;
	if (tap_cnt) tap_cnt[row] = ntap;
}

// ---- launch entry points ----
cudaError_t sym_init(const float *ps_cos8, const float *ps_sin8, const uint32_t *abort_bits35) {
	cudaError_t e = cudaMemcpyToSymbol(c_ps_cos, ps_cos8, 8 * sizeof(float));
	if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_ps_sin, ps_sin8, 8 * sizeof(float));
	if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_abort_bits, abort_bits35, 35 * sizeof(uint32_t));
	return e;
}
cudaError_t launch_phase_search(const K3Params &p, cudaStream_t s) {
	if (p.ps_ema) { // four hypotheses per lane (PhaseSearchEMA only)
		const unsigned grid = (unsigned)(((long long)p.rows * 5 + PS2_INST - 1) / PS2_INST);
		switch (p.ps_rot0 & 3) { // (1j)^rot at the first symbol of the submit
		case 0: k_phase_search_ema4b<0><<<grid, 32, 0, s>>>(p); break;
		case 1: k_phase_search_ema4b<1><<<grid, 32, 0, s>>>(p); break;
		case 2: k_phase_search_ema4b<2><<<grid, 32, 0, s>>>(p); break;
		default: k_phase_search_ema4b<3><<<grid, 32, 0, s>>>(p); break;
		}
		return cudaGetLastError();
	}
	const long long ps_warps = ((long long)p.rows * 5 + 1) / 2;
	k_phase_search<<<(unsigned)((ps_warps + PS_THREADS / 32 - 1) / (PS_THREADS / 32)), PS_THREADS, 0, s>>>(p);
	return cudaGetLastError();
}
// Five AIS::Decoder instances per row.  decoder = 1: plain bit-serial kernel, one row per warp, kept as the cross-check the
// decoder fuzz test runs against the same oracle; anything else: word-parallel kernel, rpw rows share a warp (1, 3, 6).
template <int MODEL>
static cudaError_t launch_decode_model(int decoder, int rpw, const K3Params &p, cudaStream_t s) {
	if (decoder == 1) {
		const int grid = (p.rows + DK_THREADS / 32 - 1) / (DK_THREADS / 32);
		k_decode<MODEL><<<grid, DK_THREADS, 0, s>>>(p);
	}
	else {
		const int grid = (p.rows + rpw * DK3_WARPS - 1) / (rpw * DK3_WARPS);
		if (rpw == 1) k_decode3<MODEL, 1><<<grid, DK3_WARPS * 32, 0, s>>>(p);
		else if (rpw == 3) k_decode3<MODEL, 3><<<grid, DK3_WARPS * 32, 0, s>>>(p);
		else k_decode3<MODEL, 6><<<grid, DK3_WARPS * 32, 0, s>>>(p);
	}
	return cudaGetLastError();
}
cudaError_t launch_decode10(int rpw, const K3Params &p, cudaStream_t s) {
	if (rpw == 1) k_decode10<1><<<(p.rows + DK3_WARPS - 1) / DK3_WARPS, DK3_WARPS * 32, 0, s>>>(p);
	else k_decode10<3><<<(p.rows + 3 * DK3_WARPS - 1) / (3 * DK3_WARPS), DK3_WARPS * 32, 0, s>>>(p);
	return cudaGetLastError();
}
cudaError_t launch_decode(int model, int decoder, int rpw, const K3Params &p, cudaStream_t s) {
	return model == 2 ? launch_decode_model<2>(decoder, rpw, p, s) : launch_decode_model<0>(decoder, rpw, p, s);
}
cudaError_t launch_base(const float *Ef, long long e_stride, int e_begin, int n, int rows, PllState *pll, DecState *dec, uint32_t *dec_data,
						const FrameOut &out, float *tap_dec, int *tap_cnt, cudaStream_t s) {
	k_base<<<(rows + K3_THREADS - 1) / K3_THREADS, K3_THREADS, 0, s>>>(Ef, e_stride, e_begin, n, rows, pll, dec, dec_data, out.ring, out.ring_head, out.ring_limit,
																		  out.ring_cap, out.chunk, out.blk, tap_dec, tap_cnt);
	return cudaGetLastError();
}

} // namespace aisgpu
