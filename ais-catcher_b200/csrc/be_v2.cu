// be_v2.cu -- V2::Engine (reference Source/DSP/Decoder/V2/V2Engine.{h,cpp}; model 11 "v2_base", Model.cpp:440-460): the
// newer per-channel engine on the same 48 kHz channel samples -- slot-predicted, sub-bin interpolated frequency estimate
// (FreqOffset::Estimate / Engine::CGF), folded FIR17, five decision-directed PhaseTrackers feeding five decoders, and an FM
// branch (polynomial atan2, folded FIR37, BitPLL) feeding a sixth; any decoder that completes a frame resets all six.
//
// Unlike ModelDefault the blocks of a row cannot be processed independently: what the frequency estimator does with block
// b depends on the decoder states and on the slot-phase predictor left behind by block b - 1.  So ONE WARP OWNS ONE ROW and
// walks its 512-sample blocks in order; inside a block the FFT (registers, fft512.cuh), the FIRs and the discriminator are
// spread over the 32 lanes, the float recurrences the reference runs sample by sample (rolling sum, derotation phasor) are
// replayed by the whole warp in lock step, and the six decoders live in lanes 0..5.  The five strobe decoders take every
// fifth sample each, so lanes 0..4 step one sample per iteration while lane 5 steps the FM branch over the same five
// samples; only when a frame completes somewhere in such a group of five (rare) the group is rolled back and replayed
// sample by sample in the reference's order (strobe decoder, then FM decoder, V2Engine.cpp:333-361).
//
// libm on the path: std::polar / cosf / sinf are glibc's sincosf (the double-precision polynomial of sincosf_poly /
// reduce_fast, v2_sincosf in v2_math.cuh, checked against the host library by tests/test_gpu_exact_math.py), atan2f is
// fd_atan2f (exact.cuh).
#include "exact.cuh"
#include "params.h"
#include "dec_core.cuh"
#include "fft512.cuh"
#include "v2_math.cuh"

namespace aisgpu {

static __constant__ float c_v2_taps17[17];
static __constant__ float c_v2_taps37[37];

constexpr int V2_SLOT = 1280; // SOTDMA slot at 48 kHz (V2Engine.h:105)
constexpr int V2_PRE = 155;   // start-flag anchor -> burst start (V2Engine.h:106)
constexpr int V2_WARPS = 4;   // rows per CTA
constexpr float V2_PI = 3.14159265358979323846f; // PI of Library/Common.h:318 as a float

struct V2Params {
	const float2 *Cbuf;
	long long c_stride;
	int c_begin, nproc, rows;
	V2State *st;
	DecState *dec;      // [rows * 6]
	uint32_t *dec_data; // [DEC_WORDS][rows * 6]
	FrameRec *ring;
	unsigned long long *ring_head, ring_limit;
	int ring_cap, chunk, blk;
	const uint32_t *level_rows;
	const float2 *omega_g;
	float w_train, w_track;
	float2 *tap_fc, *tap_coh; // optional [rows][nproc * 512]: the blocks this launch processed
	float *tap_fmf;
	long long tap_stride;
};

constexpr int V2_A = 16 + 512;                 // float2: 16 history + derotated block; later the FIR37 output (512 floats)
constexpr int V2_BC_BYTES = 544 * 8 + 512 * 4; // FFT tile + magnitudes, later coh[512] float2 + fmd[36 + 512] float
constexpr int V2_FR = DEC_WORDS * 8;           // frame words of the six decoders, stride 8
constexpr int V2_WARP_BYTES = V2_A * 8 + V2_BC_BYTES + V2_FR * 4;

__global__ void __launch_bounds__(V2_WARPS * 32, 4) k_v2_engine(const V2Params p) {
	extern __shared__ __align__(16) unsigned char v2_sm[];
	const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
	const int row = blockIdx.x * V2_WARPS + wib;
	if (row >= p.rows) return; // whole warp
	unsigned char *base = v2_sm + (size_t)wib * V2_WARP_BYTES;
	float2 *bufA = reinterpret_cast<float2 *>(base);
	float *fmf = reinterpret_cast<float *>(base); // aliases bufA once the FIR17 has consumed it
	unsigned char *bc = base + V2_A * 8;
	float2 *tb = reinterpret_cast<float2 *>(bc);
	float *mag = reinterpret_cast<float *>(bc + 544 * 8);
	float2 *coh = reinterpret_cast<float2 *>(bc);
	float *fmd = reinterpret_cast<float *>(bc + 512 * 8); // [36 + 512]
	uint32_t *frames = reinterpret_cast<uint32_t *>(base + V2_A * 8 + V2_BC_BYTES);
	const unsigned FULL = 0xffffffffu;

	float2 tw[15];
	fft512_lane_twiddles(p.omega_g, lane, tw);

	// ---- state: scalars are kept identical in every lane; the decoder lanes (0..5) also hold their decoder / tracker ----
	V2State &S = p.st[row];
	float2 fo_rot = S.fo_rot, slot_ema = S.slot_ema, fm_prev = S.fm_prev;
	float last_f = S.last_f, ppm = S.ppm, pll_phase = S.pll_phase;
	int slot_phase = S.slot_phase, di = S.di, pll_last = S.pll_last;
	long long sample_idx = S.sample_idx;
	float2 h17 = lane < 16 ? S.f17_hist[lane] : make_float2(0.f, 0.f);
	float h37a = S.f37_hist[lane], h37b = lane < 4 ? S.f37_hist[32 + lane] : 0.0f;
	unsigned trk_rot = 0;
	float2 trk_s = make_float2(0.f, 0.f);
	int trk_prev = 0;
	if (lane < 5) {
		trk_rot = S.trk_rot[lane];
		trk_s = S.trk_s[lane];
		trk_prev = S.trk_prev[lane];
	}
	DecCtx ctx;
	ctx.frame = frames + (lane < 6 ? lane : 0);
	ctx.mode_level = row_level(p.level_rows, row);
	ctx.stride = 8;
	DecState d;
	d.state = ST_TRAINING; d.lastBit = 0; d.prev = 0; d.position = 0; d.one_seq = 0; d.level = 0.f; d.start_idx = 0;
	const long long ndec = (long long)p.rows * 6;
	const long long didx = (long long)row * 6 + (lane < 6 ? lane : 0);
	if (lane < 6) {
		d = p.dec[didx];
		for (int w = 0; w < DEC_WORDS; w++) ctx.frame[w * 8] = p.dec_data[(long long)w * ndec + didx];
	}
	__syncwarp();

	const float2 *Crow = p.Cbuf + (long long)row * p.c_stride + p.c_begin;
	const float k_th = __fdiv_rn(__fmul_rn(2.0f, V2_PI), (float)V2_SLOT); // 2 pi / SLOT
	const float k_ph = __fdiv_rn((float)V2_SLOT, __fmul_rn(2.0f, V2_PI)); // SLOT / 2 pi
	const float w_keep = __fsub_rn(1.0f, 0.2f);                            // 1 - LEARN_W

	// FreqOffset::Derotate (V2Engine.cpp:138-151) over [i0, i1) of the block: the phasor chain is replayed by all lanes, lane
	// (i & 31) parks phasor i in the output array; then every lane multiplies its samples.  rot is renormalised per call.
	auto derotate = [&](float fv, const float2 *in, int i0, int i1) {
		float sn, cs;
		v2_sincosf(__fmul_rn(__fmul_rn(fv, 2.0f), V2_PI), sn, cs);
		const float2 step = make_float2(cs, sn); // std::polar(1.0f, theta)
		float2 r = fo_rot;
#pragma unroll 8
		for (int i = i0; i < i1; i++) {
			r = cmul(r, step);
			if ((i & 31) == lane) bufA[16 + i] = r;
		}
		__syncwarp();
		for (int i = (i0 & ~31) + lane; i < i1; i += 32)
			if (i >= i0) bufA[16 + i] = cmul(in[i], bufA[16 + i]);
		fo_rot = cnormalize(r);
		last_f = fv;
		__syncwarp();
	};

	// FreqOffset::Estimate (V2Engine.cpp:56-136) on a 512-sample window; returns f, sets prominence
	float prominence = 0.0f;
	auto estimate = [&](const float2 *win) -> float {
		cgf_fft_block<false>(win, tb, mag, lane, tw);
		__syncwarp();
		float f = 0.0f, prom = 0.0f;
		if (lane == 0) {
			float rs = 0.0f;
			for (int j = 0; j < 133; j++) rs = __fadd_rn(rs, mag[j]);
			float wm = __fadd_rn(rs, __fmul_rn(0.6f, __fadd_rn(mag[15], mag[15 + 102])));
			int wi = 0;
			for (int i = 1; i <= 512 - 133; i++) {
				rs = __fadd_rn(__fsub_rn(rs, mag[i - 1]), mag[i + 132]);
				const float v = __fadd_rn(rs, __fmul_rn(0.6f, __fadd_rn(mag[i + 15], mag[i + 15 + 102])));
				if (v > wm) { wm = v; wi = i; }
			}
			int fz = -1;
			float mx = 0.0f;
			for (int i = wi; i < wi + 31; i++) {
				const float hh = __fadd_rn(mag[i], mag[i + 102]);
				if (hh > mx) { mx = hh; fz = i; }
			}
			float total = 0.0f;
			for (int i = 0; i < 512; i++) total = __fadd_rn(total, mag[i]);
			prom = total > 0.0f ? __fdiv_rn(__fmul_rn(mx, 256.0f), total) : 0.0f;
			if (fz >= 0) {
				float frac = 0.0f;
				if (fz > 0 && fz + 102 + 1 < 512) { // sub-bin parabola through the three pair sums around the peak
					const float a = __fadd_rn(mag[fz - 1], mag[fz - 1 + 102]);
					const float c = __fadd_rn(mag[fz + 1], mag[fz + 1 + 102]);
					const float den = __fadd_rn(__fsub_rn(a, __fmul_rn(2.0f, mx)), c);
					if (den < 0.0f) {
						frac = __fdiv_rn(__fmul_rn(0.5f, __fsub_rn(a, c)), den);
						frac = frac > 0.5f ? 0.5f : (frac < -0.5f ? -0.5f : frac);
					}
				}
				f = __fdiv_rn(__fdiv_rn(__fsub_rn(256.0f, __fadd_rn(__fadd_rn((float)fz, frac), 51.0f)), 2.0f), 512.0f);
			}
		}
		f = __shfl_sync(FULL, f, 0);
		prominence = __shfl_sync(FULL, prom, 0);
		__syncwarp();
		return f;
	};

	for (int b = 0; b < p.nproc; b++) {
		const float2 *in = Crow + (long long)b * 512; // raw[0, 1024): the block to decode and the lookahead
		slot_ema = make_float2(__fmul_rn(slot_ema.x, 0.9999f), __fmul_rn(slot_ema.y, 0.9999f));
		const bool busy = __ballot_sync(FULL, lane < 5 && d.state != ST_TRAINING) != 0u;
		const bool locked = __fadd_rn(__fmul_rn(slot_ema.x, slot_ema.x), __fmul_rn(slot_ema.y, slot_ema.y)) >= 0.64f;
		const int e = (int)((((long long)slot_phase - sample_idx) % V2_SLOT + V2_SLOT) % V2_SLOT);
		const float ppm_prev = ppm;
		int split = 0;
		float f;
		// ---- Engine::CGF (V2Engine.cpp:292-321) ----
		if (locked && e < 512) {
			split = e; // [0, e) keeps the previous block's frequency
			derotate(last_f, in, 0, e);
			f = estimate(in + e);
			derotate(f, in, e, 512);
		}
		else {
			bool mid = false;
			if (!busy) { // midWins (V2Engine.cpp:279-290): energy of input[512, 768) against input[0, 256), summed in order
				for (int i = lane; i < 256; i += 32) {
					const float2 u = in[i], v = in[512 + i];
					mag[i] = __fadd_rn(__fmul_rn(u.x, u.x), __fmul_rn(u.y, u.y));
					mag[256 + i] = __fadd_rn(__fmul_rn(v.x, v.x), __fmul_rn(v.y, v.y));
				}
				__syncwarp();
				int m = 0;
				if (lane == 0) {
					float head = 0.0f, tail = 0.0f;
					for (int i = 0; i < 256; i++) {
						head = __fadd_rn(head, mag[i]);
						tail = __fadd_rn(tail, mag[256 + i]);
					}
					m = tail > head;
				}
				mid = __shfl_sync(FULL, m, 0) != 0;
				__syncwarp();
			}
			f = estimate(in + (mid ? 256 : 0));
			if (busy && prominence < 5.5f) f = last_f; // tone gate: hold while a decode is in flight
			derotate(f, in, 0, 512);
		}
		ppm = __fdiv_rn(__fmul_rn(f, 48000.0f), 162.0f);

		// ---- FilterFL17 (V2Engine.cpp:153-175): coh[n] = dot17(&x[n - 16]), folded taps ----
		if (lane < 16) bufA[lane] = h17;
		__syncwarp();
		for (int n = lane; n < 512; n += 32) {
			const float2 *a = bufA + n;
			float2 sum = make_float2(0.f, 0.f);
#pragma unroll
			for (int i = 0; i < 8; i++) {
				const float tx = __fadd_rn(a[i].x, a[16 - i].x), ty = __fadd_rn(a[i].y, a[16 - i].y);
				sum.x = __fadd_rn(sum.x, __fmul_rn(tx, c_v2_taps17[i]));
				sum.y = __fadd_rn(sum.y, __fmul_rn(ty, c_v2_taps17[i]));
			}
			sum.x = __fadd_rn(sum.x, __fmul_rn(a[8].x, c_v2_taps17[8]));
			sum.y = __fadd_rn(sum.y, __fmul_rn(a[8].y, c_v2_taps17[8]));
			coh[n] = sum;
			if (p.tap_fc) {
				p.tap_fc[(long long)row * p.tap_stride + b * 512 + n] = a[16];
				p.tap_coh[(long long)row * p.tap_stride + b * 512 + n] = sum;
			}
		}
		if (lane < 16) h17 = bufA[512 + lane];
		// ---- FMDemod (V2Engine.cpp:264-272) on the RAW block, then FilterFL37 ----
		fmd[lane] = h37a;
		if (lane < 4) fmd[32 + lane] = h37b;
		for (int i = lane; i < 512; i += 32) {
			const float2 cur = in[i], pv = i ? in[i - 1] : fm_prev;
			const float re = __fsub_rn(__fmul_rn(cur.x, pv.x), __fmul_rn(cur.y, -pv.y));
			const float im = __fadd_rn(__fmul_rn(cur.x, -pv.y), __fmul_rn(cur.y, pv.x));
			fmd[36 + i] = __fdiv_rn(v2_atan2_fast(im, re), V2_PI);
		}
		fm_prev = in[511];
		__syncwarp(); // coh complete, bufA dead from here on: the FIR37 output may take its place
		for (int n = lane; n < 512; n += 32) {
			const float *a = fmd + n;
			float sum = 0.0f;
#pragma unroll
			for (int i = 0; i < 18; i++) sum = __fadd_rn(sum, __fmul_rn(__fadd_rn(a[i], a[36 - i]), c_v2_taps37[i]));
			sum = __fadd_rn(sum, __fmul_rn(a[18], c_v2_taps37[18]));
			fmf[n] = sum;
			if (p.tap_fmf) p.tap_fmf[(long long)row * p.tap_stride + b * 512 + n] = sum;
		}
		h37a = fmd[512 + lane];
		if (lane < 4) h37b = fmd[544 + lane];
		__syncwarp();

		// ---- the sample loop (V2Engine.cpp:333-361), five samples per iteration ----
		const int o = lane < 5 ? ((lane - di) % 5 + 5) % 5 : 0; // first sample of the block that strobe decoder `lane` takes
		// one strobe decoder step on sample i (lane < 5); returns found
		auto strobe_step = [&](int i, int &fr_len, float &fr_level) -> bool {
			const float2 z0 = coh[i];
			// PhaseTracker::Rotate90 (V2Engine.cpp:190-203)
			const float sre = (trk_rot & 1u) ? z0.y : z0.x, sim = (trk_rot & 1u) ? z0.x : z0.y;
			const float zr = ((trk_rot ^ (trk_rot >> 1)) & 1u) ? -sre : sre, zi = (trk_rot & 2u) ? -sim : sim;
			trk_rot = (trk_rot + 1u) & 3u;
			const float alpha = d.state == ST_TRAINING ? p.w_train : p.w_track;
			const float beta = __fsub_rn(1.0f, alpha);
			const float proj = __fadd_rn(__fmul_rn(zr, trk_s.x), __fmul_rn(zi, trk_s.y));
			const float bd = __fmul_rn(beta, proj >= 0.0f ? 1.0f : -1.0f);
			trk_s = make_float2(__fadd_rn(__fmul_rn(alpha, trk_s.x), __fmul_rn(bd, zr)), __fadd_rn(__fmul_rn(alpha, trk_s.y), __fmul_rn(bd, zi)));
			const int decision = proj > 0.0f ? 1 : 0;
			const int bit = decision ^ trk_prev;
			trk_prev = decision;
			const float lvl = __fadd_rn(__fmul_rn(z0.x, z0.x), __fmul_rn(z0.y, z0.y)); // tag.sample_lvl = norm2(coh_filtered[i])
			int lb;
			return dec_step(d, ctx, bit ? 1.0f : -1.0f, lvl, sample_idx + i, fr_len, fr_level, lb);
		};
		// the FM branch on sample i (lane 5): BitPLL (V2Engine.cpp:225-240), then the decoder when it strobes
		auto fm_step = [&](int i, int &fr_len, float &fr_level) -> bool {
			const float smp = fmf[i];
			const int bit = smp > 0.0f ? 1 : 0;
			if (bit != pll_last) pll_phase = __fadd_rn(pll_phase, __fmul_rn(__fsub_rn(0.5f, pll_phase), d.state == ST_TRAINING ? 0.6f : 0.05f));
			pll_last = bit;
			pll_phase = __fadd_rn(pll_phase, 0.2f);
			if (pll_phase < 1.0f) return false;
			pll_phase = __fsub_rn(pll_phase, (float)(int)pll_phase);
			const float2 z0 = coh[i];
			const float lvl = __fadd_rn(__fmul_rn(z0.x, z0.x), __fmul_rn(z0.y, z0.y));
			int lb;
			return dec_step(d, ctx, smp, lvl, sample_idx + i, fr_len, fr_level, lb);
		};
		auto reset_all = [&]() { // Engine::resetDecoders: NextState(TRAINING, 0) on all six
			if (lane < 6) { d.state = ST_TRAINING; d.position = 0; d.one_seq = 0; }
		};
		for (int g0 = 0; g0 < 512; g0 += 5) {
			const int gn = min(5, 512 - g0);
			// fast path: nobody completes a frame in this group
			const DecState d_sv = d;
			const unsigned rot_sv = trk_rot;
			const float2 s_sv = trk_s;
			const int prev_sv = trk_prev, pl_sv = pll_last;
			const float ph_sv = pll_phase;
			bool found = false;
			int fl = 0;
			float fv = 0.0f;
			if (lane < 5) {
				const int i = g0 + ((o - g0) % 5 + 5) % 5;
				if (i < g0 + gn) found = strobe_step(i, fl, fv);
			}
			else if (lane == 5) {
				for (int i = g0; i < g0 + gn; i++) found |= fm_step(i, fl, fv);
			}
			if (__any_sync(FULL, found)) { // replay the group in the reference's order
				d = d_sv; trk_rot = rot_sv; trk_s = s_sv; trk_prev = prev_sv; pll_last = pl_sv; pll_phase = ph_sv;
				for (int i = g0; i < g0 + gn; i++) {
					const int L = (di + i) % 5;
					const float tag_ppm = i >= split ? ppm : ppm_prev;
					bool fnd = false;
					int len = 0;
					float lev = 0.0f;
					if (lane == L) fnd = strobe_step(i, len, lev);
					if (__any_sync(FULL, fnd)) {
						if (fnd) emit_frame(p.ring, p.ring_head, p.ring_limit, p.ring_cap, p.chunk, p.blk, ctx, row, lane, len, lev, tag_ppm, d.start_idx, sample_idx + i);
						// learnSlotPhase (V2Engine.cpp:298-307) from the decoder that found the message
						const long long sidx0 = __shfl_sync(FULL, d.start_idx, L);
						const long long a = sidx0 - V2_PRE;
						const float th = __fmul_rn((float)((a % V2_SLOT + V2_SLOT) % V2_SLOT), k_th);
						float sn, cs;
						v2_sincosf(th, sn, cs);
						slot_ema = make_float2(__fadd_rn(__fmul_rn(w_keep, slot_ema.x), __fmul_rn(0.2f, cs)), __fadd_rn(__fmul_rn(w_keep, slot_ema.y), __fmul_rn(0.2f, sn)));
						const float ph = __fmul_rn(fd_atan2f(slot_ema.y, slot_ema.x), k_ph);
						slot_phase = (int)__fadd_rn(__fadd_rn(ph, (float)V2_SLOT), 0.5f) % V2_SLOT;
						reset_all();
					}
					fnd = false;
					if (lane == 5) fnd = fm_step(i, len, lev);
					if (__any_sync(FULL, fnd)) {
						if (fnd) emit_frame(p.ring, p.ring_head, p.ring_limit, p.ring_cap, p.chunk, p.blk, ctx, row, 5, len, lev, tag_ppm, d.start_idx, sample_idx + i);
						reset_all();
					}
				}
			}
			__syncwarp();
		}
		sample_idx += 512;
		di = (di + 512) % 5;
		__syncwarp();
	}

	// ---- state back ----
	if (lane == 0) {
		S.fo_rot = fo_rot; S.slot_ema = slot_ema; S.fm_prev = fm_prev;
		S.last_f = last_f; S.ppm = ppm; S.pll_phase = pll_phase;
		S.slot_phase = slot_phase; S.di = di; S.pll_last = pll_last;
		S.sample_idx = sample_idx;
	}
	// the FM branch state lives in lane 5
	const float pp = __shfl_sync(FULL, pll_phase, 5);
	const int pl = __shfl_sync(FULL, pll_last, 5);
	if (lane == 0) { S.pll_phase = pp; S.pll_last = pl; }
	if (lane < 16) S.f17_hist[lane] = h17;
	S.f37_hist[lane] = h37a;
	if (lane < 4) S.f37_hist[32 + lane] = h37b;
	if (lane < 5) {
		S.trk_rot[lane] = trk_rot;
		S.trk_s[lane] = trk_s;
		S.trk_prev[lane] = trk_prev;
	}
	if (lane < 6) {
		p.dec[didx] = d;
		for (int w = 0; w < DEC_WORDS; w++) p.dec_data[(long long)w * ndec + didx] = ctx.frame[w * 8];
	}
}

// ---- launch entry points ----
cudaError_t v2_init(const float *taps17, const float *taps37, const float2 *omega256) {
	cudaError_t e = cudaMemcpyToSymbol(c_v2_taps17, taps17, 17 * sizeof(float));
	if (e == cudaSuccess) e = cudaMemcpyToSymbol(c_v2_taps37, taps37, 37 * sizeof(float));
	if (e == cudaSuccess) e = fft512_set_omega(omega256);
	if (e == cudaSuccess) e = cudaFuncSetAttribute(k_v2_engine, cudaFuncAttributeMaxDynamicSharedMemorySize, V2_WARPS * V2_WARP_BYTES);
	return e;
}
cudaError_t launch_v2_engine(const float2 *Cbuf, long long c_stride, int c_begin, int nproc, int rows, V2State *st, DecState *dec, uint32_t *dec_data,
							 const FrameOut &out, const float2 *omega_g, float w_train, float w_track, float2 *tap_fc, float2 *tap_coh, float *tap_fmf,
							 long long tap_stride, cudaStream_t s) {
	V2Params p;
	p.Cbuf = Cbuf; p.c_stride = c_stride; p.c_begin = c_begin; p.nproc = nproc; p.rows = rows; p.st = st; p.dec = dec; p.dec_data = dec_data;
	p.ring = out.ring; p.ring_head = out.ring_head; p.ring_limit = out.ring_limit; p.ring_cap = out.ring_cap; p.chunk = out.chunk; p.blk = out.blk;
	p.level_rows = out.level_rows;
	p.omega_g = omega_g; p.w_train = w_train; p.w_track = w_track; p.tap_fc = tap_fc; p.tap_coh = tap_coh; p.tap_fmf = tap_fmf; p.tap_stride = tap_stride;
	k_v2_engine<<<(rows + V2_WARPS - 1) / V2_WARPS, V2_WARPS * 32, V2_WARPS * V2_WARP_BYTES, s>>>(p);
	return cudaGetLastError();
}

} // namespace aisgpu
