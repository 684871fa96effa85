// be_cgf.cu -- ModelDefault back end, first half: SquareFreqOffsetCorrection + FilterComplex (DSP.cpp:215-246, 417-489).
#include "exact.cuh"
#include "params.h"
#include "fft512.cuh"

namespace aisgpu {

// ---------------------------------------------------------------------------------------------
// K2a: SquareFreqOffsetCorrection, estimation half (DSP.cpp:417-455, FFT.h:93-130).
// One warp per 512-sample block.  The reference's radix-2 DIT butterflies (t = Omega[j * N / 2m] * x[hi]; x[hi] = x[lo] - t;
// x[lo] += t, FFT.h:104-129) are evaluated with the block held in REGISTERS, 16 complex values per lane -- every butterfly
// is the reference's own arithmetic on the reference's own operands, only who computes it changes, so the spectrum is
// bit-identical whatever the schedule:
//   layout A  lane = p[8:4], register = p[3:0]  (p = position in the bit-reversed array): stages 0..3 are lane-local,
//             stage 4 pairs lane l with l ^ 1 (one shuffle per value; both lanes form t, a - t is evaluated as a + (-t));
//   layout C  lane = p[4:0], register = p[8:5]  after one transpose through a padded shared tile: stages 5..8 lane-local.
// Twiddles of stages 0..4 are warp-uniform (constant memory), those of stages 5..8 are 15 per-lane registers loaded once.
// |F| in fftshift order goes to shared memory; then (one lane per block) the sequential float cumsum, then the parallel
// first-maximum searches.  Result: an index into the host-built phasor-step table.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(CGF_THREADS) k_cgf_estimate(const float2 *__restrict__ Cbuf, long long c_stride, int c_begin, int nblk,
																 int total_blocks, const float2 *__restrict__ omega_g, int wide,
																 int *__restrict__ stepidx) {
	extern __shared__ __align__(16) unsigned char cgf_sm[];
	float *mag = reinterpret_cast<float *>(cgf_sm);                       // [16][513]
	unsigned char *scratch = cgf_sm + CGF_BLK_PER_CTA * CGF_ROWP * 4;     // transpose tiles (8 x 544 float2), later cumsum [16][513]
	float *cum = reinterpret_cast<float *>(scratch);

	const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
	float2 tw[15];
	fft512_lane_twiddles(omega_g, lane, tw);

	const int blk0 = blockIdx.x * CGF_BLK_PER_CTA;
	float2 *tb = reinterpret_cast<float2 *>(scratch) + w * CGF_TB;
	for (int rep = 0; rep < 2; rep++) {
		const int lb = w + rep * 8;
		const int id = blk0 + lb;
		if (id < total_blocks) {
			const int row = id / nblk, b = id - row * nblk;
			const float2 *src = Cbuf + (long long)row * c_stride + c_begin + (long long)b * CGF_N;
			cgf_fft_block<true>(src, tb, mag + lb * CGF_ROWP, lane, tw);
		}
		__syncwarp();
	}
	__syncthreads(); // all FFT buffers dead, mags complete
	if (wide && tid < CGF_BLK_PER_CTA && blk0 + tid < total_blocks) {
		const float *mg = mag + tid * CGF_ROWP;
		float *cs = cum + tid * CGF_ROWP;
		float c = 0.0f;
		cs[0] = 0.0f;
#pragma unroll 16
		for (int i = 1; i < CGF_N; i++) {
			c = __fadd_rn(c, mg[i]);
			cs[i] = c;
		}
	}
	__syncthreads();
	for (int rep = 0; rep < 2; rep++) {
		const int lb = w + rep * 8;
		const int id = blk0 + lb;
		if (id >= total_blocks) continue;
		const float *mg = mag + lb * CGF_ROWP;
		const float *cs = cum + lb * CGF_ROWP;
		int wi = 0;
		if (wide) { // DSP.cpp:424-446: M = 133, ofs = 15, delta = 102
			float bv = -1.0f;
			int bi = 1 << 30;
			for (int i = lane; i < CGF_N - 133; i += 32) {
				float v = __fadd_rn(__fsub_rn(cs[i + 133], cs[i]), __fmul_rn(0.6f, __fadd_rn(mg[i + 15], mg[i + 117])));
				if (v > bv) { bv = v; bi = i; }
			}
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) {
				float ov = __shfl_xor_sync(0xffffffffu, bv, o);
				int oi = __shfl_xor_sync(0xffffffffu, bi, o);
				if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
			}
			wi = (bi == (1 << 30)) ? 0 : bi;
			wi = wi + 66 - 256;
		}
		// DSP.cpp:448-455: i in [wi+187, wi+223)
		float bv = 0.0f;
		int bi = 1 << 30;
		for (int c = lane; c < 36; c += 32) {
			const int i = wi + 187 + c;
			float h = __fadd_rn(mg[i & 511], mg[(i + 102) & 511]);
			if (h > bv) { bv = h; bi = i; }
		}
#pragma unroll
		for (int o = 16; o > 0; o >>= 1) {
			float ov = __shfl_xor_sync(0xffffffffu, bv, o);
			int oi = __shfl_xor_sync(0xffffffffu, bi, o);
			if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
		}
		if (lane == 0) stepidx[id] = (bi == (1 << 30)) ? CGF_IDX_NONE : bi + CGF_IDX_OFFSET;
	}
}

__constant__ float c_taps_coherent[FIRC_T]; // FilterComplex 17 taps (Filters.h:35-41)

// ---------------------------------------------------------------------------------------------
// K2bc: the derotation phasor chain, output[i] *= rot and FilterComplex 17 taps in ONE kernel (DSP.cpp:457-465, 215-246).
// The chain rot *= rot_step is strictly sequential per row (4096 dependent complex products per submit at the bench
// shape: their latency is the floor for the whole stage), everything else is parallel.  A CTA owns CF_ROWS rows: warp 0 runs
// the chains, one lane per row, CF_T steps ahead into a double-buffered shared tile; meanwhile the two consumer warps
// derotate the previous tile (coalesced loads of the 48 kHz samples, requested one tile ahead), and run the FIR out of a
// shared ring that keeps the 16-sample history.  The phasors never travel through HBM (an earlier version wrote them out, 67 MB per submit, and read them back).  FIR: products
// by scalar __fmul_rn, the (re, im) accumulation by padd (two scalar __fadd_rn): two roundings per tap, as in the reference.
// ---------------------------------------------------------------------------------------------
constexpr int CF_T = 64;               // samples per tile and row (a 512-block = 8 tiles)
// CF_ROWS rows per CTA, CF_CONS = CF_ROWS / 2 consumer warps (four outputs per thread and tile): 4 rows -> 512 CTAs at 2048 rows
// (3-4 per SM, one CTA's barrier waits overlap another's arithmetic); 8 rows halve the chain warp's share of the issue slots
constexpr int CF_DERP = 2 * CF_T + 2 * CF_T / 4; // ring row: two tiles, one pad slot after every four samples
// ring position n (0 .. 2 CF_T - 1) -> slot: threads that own four consecutive outputs read n = 4c + i; 5c + i hits 16 different
// 8-byte banks over a half warp
__device__ __forceinline__ int cf_slot(int n) { return n + (n >> 2); }

struct CfParams {
	const float2 *Cbuf;
	long long c_stride;
	int c_begin;
	const int *stepidx;     // [rows][nblk]
	const float2 *steptab;
	float2 *rot_state;      // [rows]
	int nblk, rows;
	const float2 *hist_old; // [rows][16]
	float2 *hist_new;
	float2 *Ebuf;
	long long e_stride;
	int e_off;
	float2 *tap_cgf;        // optional
	long long tap_stride;
};

template <int CF_ROWS>
__global__ void __launch_bounds__(32 + 16 * CF_ROWS) k_cgf_fused(const CfParams p) {
	constexpr int CF_CONS = CF_ROWS / 2;
	__shared__ __align__(16) float2 rotb[2][CF_ROWS][CF_T + 2]; // +2: the chain lanes (one row each) store to different banks
	__shared__ __align__(16) float2 der[CF_ROWS][CF_DERP]; // der[r][cf_slot((t & 1) * CF_T + j)] = derotated sample j of tile t
	const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const int row0 = blockIdx.x * CF_ROWS;
	const int ntiles = p.nblk * (CGF_N / CF_T);
	const int ct = tid - 32; // consumer thread index 0..63 (negative in the chain warp)
	if (warp != 0) { // FIR history of the previous submit sits where "tile -1" would have left it
		for (int i = ct; i < CF_ROWS * (FIRC_T - 1); i += 32 * CF_CONS) {
			const int r = i / (FIRC_T - 1), k = i - r * (FIRC_T - 1);
			const int row = row0 + r;
			der[r][cf_slot(CF_T + CF_T - (FIRC_T - 1) + k)] = row < p.rows ? p.hist_old[row * (FIRC_T - 1) + k] : make_float2(0.f, 0.f);
		}
	}
	// chain state (warp 0, lanes < CF_ROWS)
	const int crow = row0 + lane;
	const bool chain = warp == 0 && lane < CF_ROWS && crow < p.rows;
	float2 rot = chain ? p.rot_state[crow] : make_float2(1.0f, 0.0f);
	float2 st = make_float2(1.0f, 0.0f);
	constexpr int CF_PER = CF_ROWS * CF_T / (32 * CF_CONS);
	float2 cpre[CF_PER]; // the consumer threads' 48 kHz samples of the tile about to be derotated
#pragma unroll
	for (int u = 0; u < CF_PER; u++) {
		const int q = ct + u * 32 * CF_CONS;
		const int r = q / CF_T, j = q - r * CF_T;
		cpre[u] = (warp != 0 && row0 + r < p.rows) ? p.Cbuf[(long long)(row0 + r) * p.c_stride + p.c_begin + j] : make_float2(0.f, 0.f);
	}
	__syncthreads();
	for (int it = 0; it <= ntiles; it++) {
		if (warp == 0) {
			if (it < ntiles && lane < CF_ROWS) {
				const int b = it / (CGF_N / CF_T);
				if ((it % (CGF_N / CF_T)) == 0 && chain) st = p.steptab[p.stepidx[crow * p.nblk + b]];
				float2 *o = rotb[it & 1][lane];
#pragma unroll 16
				for (int i = 0; i < CF_T; i++) {
					rot = cmul(rot, st);
					o[i] = rot;
				}
				if ((it % (CGF_N / CF_T)) == (CGF_N / CF_T) - 1) rot = cnormalize(rot); // once per 512-block (DSP.cpp:465)
			}
		}
		else if (it >= 1) {
			const int t = it - 1;
			const int half = (t & 1) * CF_T;
			// derotate: thread -> (row r, sample j), a warp covers 32 consecutive samples of one row.  The 48 kHz samples of the
			// NEXT tile are requested before this tile is touched, so their HBM/L2 latency hides behind the FIR below.
			float2 cnext[CF_PER];
#pragma unroll
			for (int u = 0; u < CF_PER; u++) {
				const int q = ct + u * 32 * CF_CONS;
				const int r = q / CF_T, j = q - r * CF_T;
				cnext[u] = (row0 + r < p.rows && t + 1 < ntiles) ? p.Cbuf[(long long)(row0 + r) * p.c_stride + p.c_begin + (t + 1) * CF_T + j] : make_float2(0.f, 0.f);
			}
#pragma unroll
			for (int u = 0; u < CF_PER; u++) {
				const int q = ct + u * 32 * CF_CONS;
				const int r = q / CF_T, j = q - r * CF_T;
				const int row = row0 + r;
				float2 v = make_float2(0.f, 0.f);
				if (row < p.rows) {
					const int n = t * CF_T + j;
					v = cmul(cpre[u], rotb[t & 1][r][j]);
					if (p.tap_cgf) p.tap_cgf[(long long)row * p.tap_stride + n] = v;
				}
				der[r][cf_slot(half + j)] = v;
			}
#pragma unroll
			for (int u = 0; u < CF_PER; u++) cpre[u] = cnext[u];
			asm volatile("bar.sync 1, %0;" ::"n"(32 * CF_CONS));
			// FIR: thread -> (row r, four consecutive outputs j0..j0+3): 20 ring samples in registers
			{
				const int r = ct >> 4, j0 = (ct & 15) * 4;
				const int row = row0 + r;
				float2 x[FIRC_T + 3];
#pragma unroll
				for (int i = 0; i < FIRC_T + 3; i++) x[i] = der[r][cf_slot((half + j0 - (FIRC_T - 1) + i) & (2 * CF_T - 1))];
				if (row < p.rows) {
					float2 y[4];
#pragma unroll
					for (int o = 0; o < 4; o++) {
						c64 acc = pack2(0.0f, 0.0f);
#pragma unroll
						for (int k = 0; k < FIRC_T; k++)
							acc = padd(acc, pack2(__fmul_rn(c_taps_coherent[k], x[o + k].x), __fmul_rn(c_taps_coherent[k], x[o + k].y)));
						y[o] = unpack2(acc);
					}
					// Ebuf rows start at an even float2 index (e_stride and e_off are even), j0 is a multiple of 4: 16-byte stores
					float4 *e = reinterpret_cast<float4 *>(p.Ebuf + (long long)row * p.e_stride + p.e_off + t * CF_T + j0);
					e[0] = make_float4(y[0].x, y[0].y, y[1].x, y[1].y);
					e[1] = make_float4(y[2].x, y[2].y, y[3].x, y[3].y);
				}
			}
		}
		__syncthreads();
	}
	if (chain) p.rot_state[crow] = rot;
	if (warp != 0) { // history for the next submit: the last 16 derotated samples
		const int half = ((ntiles - 1) & 1) * CF_T;
		for (int i = ct; i < CF_ROWS * (FIRC_T - 1); i += 32 * CF_CONS) {
			const int r = i / (FIRC_T - 1), k = i - r * (FIRC_T - 1);
			const int row = row0 + r;
			if (row < p.rows) p.hist_new[row * (FIRC_T - 1) + k] = der[r][cf_slot(half + CF_T - (FIRC_T - 1) + k)];
		}
	}
}

// ---- launch entry points ----
constexpr int CGF_EST_SMEM = CGF_BLK_PER_CTA * CGF_ROWP * 4 + (8 * CGF_TB * 8 > CGF_BLK_PER_CTA * CGF_ROWP * 4 ? 8 * CGF_TB * 8 : CGF_BLK_PER_CTA * CGF_ROWP * 4);
cudaError_t cgf_init(const float *taps17, const float2 *omega256) {
	cudaError_t e = cudaMemcpyToSymbol(c_taps_coherent, taps17, FIRC_T * sizeof(float));
	if (e != cudaSuccess) return e;
	e = fft512_set_omega(omega256);
	if (e != cudaSuccess) return e;
	return cudaFuncSetAttribute(k_cgf_estimate, cudaFuncAttributeMaxDynamicSharedMemorySize, CGF_EST_SMEM);
}
cudaError_t launch_cgf_estimate(const float2 *Cbuf, long long c_stride, int c_begin, int nblk, int total_blocks, const float2 *omega, int wide, int *stepidx,
								cudaStream_t s) {
	const int ctas = (total_blocks + CGF_BLK_PER_CTA - 1) / CGF_BLK_PER_CTA;
	k_cgf_estimate<<<ctas, CGF_THREADS, CGF_EST_SMEM, s>>>(Cbuf, c_stride, c_begin, nblk, total_blocks, omega, wide, stepidx);
	return cudaGetLastError();
}
cudaError_t launch_cgf_fused(const float2 *Cbuf, long long c_stride, int c_begin, const int *stepidx, const float2 *steptab, float2 *rot_state, int nblk, int rows,
							 const float2 *hist_old, float2 *hist_new, float2 *Ebuf, long long e_stride, int e_off, float2 *tap_cgf, long long tap_stride, int rows_per_cta, cudaStream_t s) {
	CfParams p;
	p.Cbuf = Cbuf; p.c_stride = c_stride; p.c_begin = c_begin; p.stepidx = stepidx; p.steptab = steptab; p.rot_state = rot_state;
	p.nblk = nblk; p.rows = rows; p.hist_old = hist_old; p.hist_new = hist_new; p.Ebuf = Ebuf; p.e_stride = e_stride; p.e_off = e_off;
	p.tap_cgf = tap_cgf; p.tap_stride = tap_stride;
	if (rows_per_cta == 8) k_cgf_fused<8><<<(rows + 7) / 8, 32 + 16 * 8, 0, s>>>(p);
	else k_cgf_fused<4><<<(rows + 3) / 4, 32 + 16 * 4, 0, s>>>(p);
	return cudaGetLastError();
}

} // namespace aisgpu
