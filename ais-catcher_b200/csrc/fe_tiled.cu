// fe_tiled.cu -- the tiled (shared-memory staged, TMA bulk copy) front end: serves the rates below 768 kS/s and any
// block shape the streaming kernel (fe_stream.cuh) does not take.
#include "exact.cuh"
#include "params.h"
#include "fe_common.cuh"

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// K1: fused front end.  input rate -> k x Downsample2CIC5 (DSP.cpp:93-117) -> FilterComplex3Tap (DSP.cpp:283-293)
//     -> Rotate (DSP.cpp:296-316) -> per channel Downsample2CIC5 -> FilterCIC5 (DSP.cpp:132-157) -> Cbuf.
// One CTA owns (segment, stream) and walks the segment tile by tile, every stage array living in shared memory
// as [HIST history | tile]; the history is what the reference keeps in h0..h4 / h1,h2 / rot.  A segment starts P
// samples early (from the previous submit's tail for segment 0) with zero history: after P >= h_k samples every
// stage's history is exact because each CIC stage is a pure function of its last 6 inputs
// (u_{s+1}[n] = fl(u_s[n] + u_s[n-1]), y[j] = u_5[2j]/32).
// ---------------------------------------------------------------------------------------------

// R consecutive outputs of one Downsample2CIC5 from 2R+4 inputs held in registers: 9R+6 complex adds.
// sm = the CTA's shared array; in_off / out_off = index of sample 0 of the stage input / output (history at
// negative indices); j0 = first output index.  Outputs past the valid count land in the arrays' slack.
template <int R>
__device__ __forceinline__ void ds2_run(float2 *__restrict__ sm, int in_off, int out_off, int j0) {
	c64 v[2 * R + 6];
	const ulonglong2 *p = reinterpret_cast<const ulonglong2 *>(sm + in_off + 2 * j0 - 6);
#pragma unroll
	for (int q = R + 2; q >= 0; q--) {
		const ulonglong2 t = p[q];
		v[2 * q] = t.x;
		v[2 * q + 1] = t.y;
	}
#pragma unroll
	for (int s = 1; s <= 4; s++) {
#pragma unroll
		for (int n = 2 * R + 4; n >= s + 1; n--) v[n] = padd(v[n], v[n - 1]);
	}
	const c64 sc = pack2(0.03125f, 0.03125f);
	c64 *o = reinterpret_cast<c64 *>(sm + out_off + j0);
#pragma unroll
	for (int q = 0; q < R; q++) {
		const int n = 6 + 2 * q;
		o[q] = pmul(padd(v[n], v[n - 1]), sc);
	}
}

// R consecutive outputs of FilterCIC5 (no decimation) from R+5 inputs: 5R+10 complex adds; straight to HBM.
template <int R>
__device__ __forceinline__ void fcic_run(const float2 *__restrict__ sm, int in_off, float2 *__restrict__ out, int m0, int m_lo, int n_out) {
	c64 v[R + 5];
	const c64 *p = reinterpret_cast<const c64 *>(sm + in_off + m0 - 5);
#pragma unroll
	for (int q = 0; q < R + 5; q++) v[q] = p[q];
#pragma unroll
	for (int s = 1; s <= 5; s++) {
#pragma unroll
		for (int n = R + 4; n >= s; n--) v[n] = padd(v[n], v[n - 1]);
	}
	const c64 sc = pack2(0.03125f, 0.03125f);
	c64 *o = reinterpret_cast<c64 *>(out);
#pragma unroll
	for (int q = 0; q < R; q++)
		if (m0 + q >= m_lo && m0 + q < n_out) o[m0 + q] = pmul(v[5 + q], sc);
}

// ---- mbarrier + 1-D bulk async copy (TMA, SASS UBLKCP): global -> shared without touching registers ----
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
	asm volatile(
		"{\n\t.reg .pred p;\n\t"
		"WAIT_%=:\n\t"
		"mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
		"@p bra DONE_%=;\n\t"
		"bra WAIT_%=;\n\t"
		"DONE_%=:\n\t}" ::"r"((unsigned)__cvta_generic_to_shared(bar)),
		"r"(parity)
		: "memory");
}
__device__ __forceinline__ void bulk_g2s(void *smem_dst, const void *gsrc, unsigned bytes, uint64_t *bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
					 (unsigned)__cvta_generic_to_shared(smem_dst)),
				 "l"(gsrc), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
				 : "memory");
}

// One CTA of NW = 4 warps owns (segment, stream) and walks [seg_start - P, seg_end) in tiles of p.tile input samples,
// starting from zero history: after P >= h_k samples every stage's history is exact, so only 48 kHz outputs that
// belong to [seg_start, seg_end) are written.  Thread 0 keeps a two-deep ring of bulk async copies (input tile + its
// Rotate phasors) in flight; all threads then run the stages of the tile back to back out of the CTA's shared-memory
// arrays ([HIST history | tile] each).  The arrays of one CTA serve NW warps, so the shared-memory footprint per
// resident warp -- what capped the one-warp version at 6 warps per SM -- drops NW-fold; the deeper (shorter) stages
// simply occupy fewer warps.  After the barrier that ends a stage, three threads move the last HIST inputs of that
// stage to the front of the array the next tile will read (the reference's h0..h4 / h1,h2 carried state).
constexpr int NW = 4;

// History for the next tile: dst[-HIST .. 0) = src[n - HIST .. n) for a group of stage arrays, n = len >> shift (even;
// when n < HIST part of the old history moves up -- one warp instruction loads all entries before any is stored).
// Array descriptors (src offset, dst offset, shift) sit in shared memory; three threads of warp 0 serve one array.
struct FeCarryDesc { int src, dst, shift, pad; };
__device__ __forceinline__ void fe_carry_group(float2 *__restrict__ sm, const FeCarryDesc *__restrict__ desc, int first, int count, int len, int tid) {
	if (tid < 3 * count) {
		const int a = tid / 3, e = 2 * (tid - 3 * a);
		const FeCarryDesc d = desc[first + a];
		const int n = len >> d.shift;
		const float4 v = *reinterpret_cast<const float4 *>(sm + d.src + n - FE_HIST + e);
		*reinterpret_cast<float4 *>(sm + d.dst - FE_HIST + e) = v;
	}
}

template <int FMT, int K, bool PRE = false>
__global__ void __launch_bounds__(NW * 32) k_frontend(const FeParams p) {
	constexpr int NT = NW * 32;
	extern __shared__ __align__(16) float2 sm[];
	__shared__ __align__(8) uint64_t mbar[2];
	__shared__ FeCarryDesc cdesc[2][FE_MAXK + 6]; // [parity of the tile][array]: input ring, levels 1..K, up, dn | wa, wb
	const int tid = threadIdx.x;
	const int stream = blockIdx.y;
	const long long seg_start = (long long)blockIdx.x * p.seg_len;
	if (seg_start >= p.N) return;
	const int seg_n = (int)min((long long)p.seg_len, (long long)p.N - seg_start); // samples of this segment
	const int span = seg_n + p.P;                                                  // samples walked, warm-up included
	const int n_tiles = (span + p.tile - 1) / p.tile;
	const long long base = seg_start - p.P; // first sample walked, relative to the submit (negative: previous submit's tail)
	const float2 *rot_g = p.rot + (p.P >> K) + (base >> K);
	float2 *Cg = p.C + (long long)(stream * 2) * p.c_stride + p.c_off + (base >> (K + 1));
	const int m_first = p.P >> (K + 1); // first 48 kHz output (relative to base) that belongs to the segment
	const int off_up = p.off_up + FE_HIST, off_dn = p.off_dn + FE_HIST, off_wa = p.off_wa + FE_HIST, off_wb = p.off_wb + FE_HIST;

	// zero what acts as history or may be read before written (the whole array is small enough to clear)
	for (int i = tid; i < p.smem_f2; i += NT) sm[i] = make_float2(0.f, 0.f);
	if (tid == 0) {
		mbar_init(&mbar[0], 1);
		mbar_init(&mbar[1], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
	}
	if (tid < 2 * (K + 5)) {
		const int par = tid / (K + 5), a = tid - par * (K + 5);
		FeCarryDesc d;
		d.pad = 0;
		if (a == 0) { d.src = p.off_in[par] + FE_HIST; d.dst = p.off_in[par ^ 1] + FE_HIST; d.shift = 0; }
		else if (a <= K) { d.src = d.dst = p.off_lv[a] + FE_HIST; d.shift = a; }
		else if (a == K + 1) { d.src = d.dst = off_up; d.shift = K; }
		else if (a == K + 2) { d.src = d.dst = off_dn; d.shift = K; }
		else if (a == K + 3) { d.src = d.dst = off_wa; d.shift = K + 1; }
		else { d.src = d.dst = off_wb; d.shift = K + 1; }
		cdesc[par][a] = d;
	}
	__syncthreads();

	auto issue = [&](int t) {
		const int rel = t * p.tile;
		const int len = min(p.tile, span - rel);
		const int b = t & 1;
		const int n96 = len >> K;
		unsigned bytes = PRE ? 0u : (unsigned)n96 * 8u;
		if (FMT == 0) bytes += (unsigned)len * 8u;
		mbar_expect_tx(&mbar[b], bytes);
		if (!PRE) bulk_g2s(sm + p.off_rot[b], rot_g + (rel >> K), (unsigned)n96 * 8u, &mbar[b]);
		if (FMT == 0) {
			const long long pos = base + rel;
			float2 *dst = sm + p.off_in[b] + FE_HIST;
			const float2 *in = reinterpret_cast<const float2 *>(p.in) + (long long)stream * p.in_stride;
			const float2 *tl = reinterpret_cast<const float2 *>(p.tail) + (long long)stream * p.P + p.P;
			if (pos >= 0) bulk_g2s(dst, in + pos, (unsigned)len * 8u, &mbar[b]);
			else if (pos + len <= 0) bulk_g2s(dst, tl + pos, (unsigned)len * 8u, &mbar[b]);
			else { // the tile straddles the first sample of the submit
				const int nt = (int)(-pos);
				bulk_g2s(dst, tl + pos, (unsigned)nt * 8u, &mbar[b]);
				bulk_g2s(dst + nt, in, (unsigned)(len - nt) * 8u, &mbar[b]);
			}
		}
	};
	if (tid == 0) issue(0);

	for (int t = 0; t < n_tiles; t++) {
		const int rel = t * p.tile;
		const int len = min(p.tile, span - rel);
		const int b = t & 1;
		if (tid == 0 && t + 1 < n_tiles) issue(t + 1); // ring slot b^1 was released by the barriers of tile t-1
		const int off_in = (b ? p.off_in[1] : p.off_in[0]) + FE_HIST;
		if (FMT != 0) { // integer formats, F32_FS4 and DC16H: convert while loading (registers), no bulk copy
			// F32_FS4: pos, the tile's first sample relative to the submit, is a multiple of 4 -- seg_len is whole tiles, a tile a whole
			// number of super-steps (or the whole block), P a whole number of super-steps -- but the pattern position is taken from
			// pos + i itself, so nothing here depends on it
			const long long pos = base + rel;
			const long long tbase = (long long)stream * p.P + p.P + pos;
			const long long ibase = (long long)stream * p.in_stride + pos;
			for (int i = tid * 2; i < len; i += 2 * NT) {
				float2 x, y;
				if (pos + i < 0) fe_load_pair<FMT>(p.tail, tbase + i, (int)(pos + i), x, y);
				else fe_load_pair<FMT>(p.in, ibase + i, (int)(pos + i), x, y);
				*reinterpret_cast<float4 *>(sm + off_in + i) = make_float4(x.x, x.y, y.x, y.y);
			}
			__syncthreads();
		}
		mbar_wait(&mbar[b], (unsigned)((t >> 1) & 1));
		// The deeper stages only have work for one or two warps.  Warp w of every CTA sits on scheduler w % 4, so a fixed
		// assignment would pile all of that work on one of the SM's four schedulers; the work index vt is therefore
		// rotated by one warp per stage and per tile, which spreads it evenly (CTAs are at different tiles).
		int rotw = t + blockIdx.x;
#define FE_VT() ((tid + 32 * ((rotw++) & (NW - 1))) & (NT - 1))
		// ---- K cascaded Downsample2CIC5 at the input rate ----
		int src = off_in;
#pragma unroll
		for (int l = 0; l < K; l++) {
			const int dst = p.off_lv[l + 1] + FE_HIST;
			const int n_out = len >> (l + 1);
			const int vt = FE_VT();
			for (int j0 = vt * 5; j0 < n_out; j0 += 5 * NT) ds2_run<5>(sm, src, dst, j0);
			__syncthreads();
			if (l == 0 && !PRE) fe_carry_group(sm, cdesc[b], K + 3, 2, p.tile, tid); // wa, wb of the previous (always full) tile; its FilterCIC5 pass is two barriers back
			src = dst;
		}
		if (PRE) { // decimation in front of DSP::Upsample (Model.cpp:183-189): the level-K samples go to HBM
			const int nK = len >> K, iK = rel >> K, firstK = p.P >> K; // samples before firstK are warm-up
			float2 *o = p.D0 + (long long)stream * p.d0_stride + p.d0_off + (base >> K) + iK;
			const int vt_o = FE_VT();
			for (int i = vt_o; i < nK; i += NT)
				if (iK + i >= firstK) o[i] = sm[src + i];
			__syncthreads();
			fe_carry_group(sm, cdesc[b], 0, K + 1, len, tid);
			__syncthreads();
			continue;
		}
		// ---- FilterComplex3Tap + Rotate at 96 kHz ----
		const int n96 = len >> K;
		const int off_rt = b ? p.off_rot[1] : p.off_rot[0];
		const int vt_r = FE_VT();
		for (int i = vt_r; i < n96; i += NT) {
			float2 x = sm[src + i];
			if (p.use_fdc) { // alpha * (h1 + data[i]) + h2 * beta
				const float2 tt = cadd(sm[src + i - 2], x);
				const float2 h2 = sm[src + i - 1];
				x = make_float2(__fadd_rn(__fmul_rn(p.fdc_alpha, tt.x), __fmul_rn(h2.x, p.fdc_beta)),
								__fadd_rn(__fmul_rn(p.fdc_alpha, tt.y), __fmul_rn(h2.y, p.fdc_beta)));
			}
			const float2 r = sm[off_rt + i];
			const float RR = __fmul_rn(x.x, r.x), II = __fmul_rn(x.y, r.y), RI = __fmul_rn(x.x, r.y), IR = __fmul_rn(x.y, r.x);
			sm[off_up + i] = make_float2(__fsub_rn(RR, II), __fadd_rn(IR, RI));
			sm[off_dn + i] = make_float2(__fadd_rn(RR, II), __fsub_rn(IR, RI));
		}
		__syncthreads();
		if (K == 0) fe_carry_group(sm, cdesc[b], K + 3, 2, p.tile, tid);
		// ---- per channel Downsample2CIC5 96k -> 48k ----
		const int n48 = n96 >> 1;
		const int runs = (n48 + 4) / 5;
		if (K == 0) __syncthreads(); // the wa/wb history move above reads what this pass overwrites
		const int vt_c = FE_VT();
		for (int r = vt_c; r < 2 * runs; r += NT) {
			const int ch = r >= runs;
			ds2_run<5>(sm, ch ? off_dn : off_up, ch ? off_wb : off_wa, (ch ? r - runs : r) * 5);
		}
		__syncthreads();
		// every stage that reads the input ring, the level arrays, up and dn has run: move their histories
		fe_carry_group(sm, cdesc[b], 0, K + 3, len, tid);
		// ---- per channel FilterCIC5 at 48k, straight to HBM ----
		const int m_rel = rel >> (K + 1); // 48 kHz index of the tile's first output, relative to base
		if (m_rel + n48 > m_first) {
			const int m_lo = m_first - m_rel; // outputs before it are warm-up
			const int vt_f = FE_VT();
			for (int r = vt_f; r < 2 * runs; r += NT) {
				const int ch = r >= runs;
				fcic_run<5>(sm, ch ? off_wb : off_wa, Cg + (ch ? p.c_stride : 0) + m_rel, (ch ? r - runs : r) * 5, m_lo, n48);
			}
		}
		__syncthreads();
	}
}

// ---- launch entry point ----
template <int FMT, int K, bool PRE>
static cudaError_t launch_tiled_one(const FeParams &p, dim3 grid, size_t smem, cudaStream_t s) {
	cudaError_t e = cudaFuncSetAttribute(k_frontend<FMT, K, PRE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
	if (e != cudaSuccess) return e;
	k_frontend<FMT, K, PRE><<<grid, NW * 32, smem, s>>>(p);
	return cudaGetLastError();
}
template <int FMT>
static cudaError_t launch_tiled_fmt(const FeParams &p, int k, bool pre, dim3 grid, size_t smem, cudaStream_t s) {
	if (pre) {
		switch (k) { // CIC stages in front of DSP::Upsample (kA <= 5)
		case 0: return launch_tiled_one<FMT, 0, true>(p, grid, smem, s);
		case 1: return launch_tiled_one<FMT, 1, true>(p, grid, smem, s);
		case 2: return launch_tiled_one<FMT, 2, true>(p, grid, smem, s);
		case 3: return launch_tiled_one<FMT, 3, true>(p, grid, smem, s);
		case 4: return launch_tiled_one<FMT, 4, true>(p, grid, smem, s);
		default: return launch_tiled_one<FMT, 5, true>(p, grid, smem, s);
		}
	}
	switch (k) {
	case 0: return launch_tiled_one<FMT, 0, false>(p, grid, smem, s);
	case 1: return launch_tiled_one<FMT, 1, false>(p, grid, smem, s);
	case 2: return launch_tiled_one<FMT, 2, false>(p, grid, smem, s);
	case 3: return launch_tiled_one<FMT, 3, false>(p, grid, smem, s);
	case 4: return launch_tiled_one<FMT, 4, false>(p, grid, smem, s);
	case 5: return launch_tiled_one<FMT, 5, false>(p, grid, smem, s);
	case 6: return launch_tiled_one<FMT, 6, false>(p, grid, smem, s);
	default: return launch_tiled_one<FMT, 7, false>(p, grid, smem, s);
	}
}
cudaError_t launch_frontend_tiled(const FeParams &p, int fmt, int k, bool pre, dim3 grid, size_t smem, cudaStream_t s) {
	switch (fmt) {
	case 0: return launch_tiled_fmt<0>(p, k, pre, grid, smem, s);
	case 1: return launch_tiled_fmt<1>(p, k, pre, grid, smem, s);
	case 2: return launch_tiled_fmt<2>(p, k, pre, grid, smem, s);
	case 3: return launch_tiled_fmt<3>(p, k, pre, grid, smem, s);
	case FE_FMT_FS4: return launch_tiled_fmt<FE_FMT_FS4>(p, k, pre, grid, smem, s);
	case FE_FMT_DC16H: return launch_tiled_fmt<FE_FMT_DC16H>(p, k, pre, grid, smem, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace aisgpu
