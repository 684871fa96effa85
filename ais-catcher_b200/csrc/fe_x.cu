// fe_x.cu -- front end of single-channel mode (-c X, reference Model.cpp:35-107): a complex baseband stream already centred on
// one AIS channel at 48 / 96 / 192 kS/s goes through K x Downsample2CIC5 -> [FilterComplex3Tap at 48 kHz] -> FilterCIC5 and
// yields ONE 48 kHz row of Cbuf per stream (no Rotate, no second channel).  Non-bucket rates reach this kernel as CF32 blocks
// from the DSP::Upsample ring (aisgpu.cu, pre-stage 1 with no CIC stage in front of the resampler).
//
// Shape: the per-thread streaming pipeline of fe_stream.cuh without Rotate.  Every lane owns a sub-segment of one stream and
// walks it chunk by chunk with the filter state in registers, after P samples of warm-up from zero state (every stage is a pure
// function of its last few inputs).  A chunk is 128 bytes of input per lane (16 CF32, 32 CS16, 64 CU8/CS8 samples); the warp
// stages the chunks of its 32 lanes through a shared-memory ring with coalesced 16-byte cp.async copies, NB - 1 chunks ahead.
// Each input byte is read once, plus P samples per sub-segment.  The lanes per stream come from the same planner as the
// streaming front end (st_plan): as few as give one balanced wave over the SMs.
#include "fe_stream.cuh"

namespace aisgpu {

namespace {

constexpr int X_NB = 6; // chunks in a warp's staging ring (5 in flight while one is consumed): 27 KB per one-warp CTA

template <int FMT>
struct XFmt {
	static constexpr int BPS = FMT == 0 ? 8 : (FMT == 3 ? 4 : 2);
	static constexpr int G = 128 / BPS; // samples per lane chunk
	typedef StFmt<FMT, G> F;            // CHUNK = 128 bytes, PIECES = 8, SLOT = 144
};

template <int FMT, int K>
__global__ void __launch_bounds__(32) k_frontend_x(const FeParams p) {
	typedef typename XFmt<FMT>::F F;
	constexpr int G = XFmt<FMT>::G;
	constexpr int N48 = G >> K; // 48 kHz outputs per chunk (even)
	static_assert(K >= 0 && K <= 2 && N48 >= 4, "buckets 48K, 96K, 192K");
	extern __shared__ __align__(16) unsigned char x_ring[]; // [X_NB][32 * SLOT]
	const int lane = threadIdx.x;
	const long long g = (long long)blockIdx.x * 32 + lane;
	const int L = p.st_L;
	int stream = (int)(g / L), sub = (int)(g - (long long)stream * L);
	const bool ghost = stream >= p.st_B; // spare lanes of the last warp replay the batch's last lane without storing
	if (ghost) { stream = p.st_B - 1; sub = L - 1; }
	const int n_short = L - p.st_r;
	const int n_main = ghost ? 0 : p.st_q + (sub >= n_short ? 1 : 0); // chunks this lane delivers
	// the lane owns samples [a, a + n_main * G); every lane walks warm + q + (r ? 1 : 0) chunks (a short lane's last one re-reads
	// the head of its right neighbour's sub-segment -- same stream -- and stores nothing)
	const long long a = ((long long)sub * p.st_q + max(0, sub - n_short)) * G;
	const int warm = p.P / G;
	const int n_chunks = warm + p.st_q + (p.st_r ? 1 : 0);
	const unsigned char *in_row = reinterpret_cast<const unsigned char *>(p.in) + ((long long)stream * p.in_stride + a - p.P) * F::BPS;
	// warm-up chunks of a stream's first sub-segment come from the previous submit's last P samples (the tail buffer)
	const unsigned long long my_warm = sub == 0 ? (unsigned long long)(reinterpret_cast<const unsigned char *>(p.tail) + (long long)stream * p.P * F::BPS)
												: (unsigned long long)in_row;
	const unsigned long long my_main = (unsigned long long)in_row;
	// instruction `it` of a chunk: lane j copies 16-byte piece (j % 8) of the chunk of owner it * 4 + j / 8 -- four owners' 128-byte
	// chunks per warp instruction
	constexpr int OWN_PER_IT = 32 / F::PIECES;
	const int o0 = lane / F::PIECES, q0 = lane % F::PIECES;
	unsigned char(*ring)[32 * F::SLOT] = reinterpret_cast<unsigned char(*)[32 * F::SLOT]>(x_ring);
	auto prefetch = [&](int c) {
		if (c < n_chunks) {
			const unsigned long long base = c < warm ? my_warm : my_main; // warp-uniform choice
			unsigned char *dst = &ring[c % X_NB][o0 * F::SLOT + q0 * 16];
#pragma unroll
			for (int it = 0; it < F::PIECES; it++) {
				const unsigned long long w = __shfl_sync(0xffffffffu, base, it * OWN_PER_IT + o0);
				cp_async16(dst + it * OWN_PER_IT * F::SLOT, reinterpret_cast<const unsigned char *>(w) + (long long)c * F::CHUNK + q0 * 16);
			}
		}
		cp_async_commit();
	};
	const c64 sc = pack2(0.03125f, 0.03125f);
	Cic5 lv[K > 0 ? K : 1], fc;
#pragma unroll
	for (int l = 0; l < K; l++) cic5_zero(lv[l]);
	cic5_zero(fc);
	c64 fd1 = 0ull, fd2 = 0ull; // FilterComplex3Tap h1, h2
	c64 pend[K > 0 ? K : 1];    // pend[l]: even-indexed sample waiting at level l (l = 1 .. K-1)
	c64 e48 = 0ull;             // even-indexed 48 kHz sample waiting for FilterCIC5
	float2 *Cg = p.C + (long long)stream * p.c_stride + p.c_off + (a >> K);
#pragma unroll
	for (int c = 0; c < X_NB - 1; c++) prefetch(c);
	for (int c = 0; c < n_chunks; c++) {
		prefetch(c + X_NB - 1);
		cp_async_wait<X_NB - 1>(); // chunk c has landed
		__syncwarp();
		const unsigned char *slot = &ring[c % X_NB][lane * F::SLOT];
		const bool store = c >= warm && c - warm < n_main;
		float2 *o = Cg + (long long)(c - warm) * N48;
#pragma unroll
		for (int j = 0; j < G / 2; j++) {
			c64 xe, xo;
			st_read_pair<FMT>(slot, j, xe, xo);
			if (K == 0) { // 48K: convert >> FCIC5 (no droop filter, Model.cpp:91-93)
				c64 o0v, o1v;
				fcic_pair(fc, xe, xo, sc, o0v, o1v);
				if (store) *reinterpret_cast<ulonglong2 *>(o + 2 * j) = make_ulonglong2(o0v, o1v);
				continue;
			}
			c64 y = ds2_pair(lv[0], xe, xo, sc);
			int idx = j;
			bool live = true;
#pragma unroll
			for (int l = 1; l < K; l++) { // an output with an odd index completes a pair one level down
				if (live) {
					if ((idx & 1) == 0) { pend[l] = y; live = false; }
					else { y = ds2_pair(lv[l], pend[l], y, sc); idx >>= 1; }
				}
			}
			if (!live) continue;
			// y is 48 kHz sample idx of the chunk
			c64 x = y;
			if (p.use_fdc) { // FilterComplex3Tap: alpha * (h1 + x) + h2 * beta (DSP.cpp:283-293), each product and sum rounded separately
				const float2 h1 = unpack2(fd1), h2 = unpack2(fd2), yv = unpack2(y);
				const float tx = __fadd_rn(h1.x, yv.x), ty = __fadd_rn(h1.y, yv.y);
				x = pack2(__fadd_rn(__fmul_rn(p.fdc_alpha, tx), __fmul_rn(h2.x, p.fdc_beta)), __fadd_rn(__fmul_rn(p.fdc_alpha, ty), __fmul_rn(h2.y, p.fdc_beta)));
				fd1 = fd2;
				fd2 = y;
			}
			if ((idx & 1) == 0) e48 = x;
			else {
				c64 o0v, o1v;
				fcic_pair(fc, e48, x, sc, o0v, o1v);
				if (store) *reinterpret_cast<ulonglong2 *>(o + idx - 1) = make_ulonglong2(o0v, o1v);
			}
		}
		__syncwarp(); // the ring slot may be refilled by a later prefetch
	}
	cp_async_wait<0>();
}

template <int FMT, int K>
cudaError_t launch_x_one(FeParams p, int forced_L, cudaStream_t s) {
	constexpr int G = XFmt<FMT>::G;
	constexpr size_t smem = (size_t)X_NB * 32 * XFmt<FMT>::F::SLOT;
	if (p.N % G || p.P % G || p.N <= 0) return cudaErrorInvalidValue;
	static CtaSlots cache;
	int slots = 0, sms = 0;
	if (const cudaError_t e = cta_slots(cache, k_frontend_x<FMT, K>, 32, smem, slots, sms)) return e;
	const int nss = p.N / G, warm = p.P / G;
	// sub-segments of at least four warm-ups when the block allows it, else one lane per stream
	if (!st_plan(p.st_B, nss, warm, 1, slots, 4, forced_L, p.st_L, p.st_q, p.st_r)) {
		p.st_L = 1;
		p.st_q = nss;
		p.st_r = 0;
	}
	const unsigned ctas = (unsigned)(((long long)p.st_B * p.st_L + 31) / 32);
	k_frontend_x<FMT, K><<<ctas, 32, smem, s>>>(p);
	return cudaGetLastError();
}

template <int FMT>
cudaError_t launch_x_fmt(const FeParams &p, int k, int forced_L, cudaStream_t s) {
	switch (k) {
	case 0: return launch_x_one<FMT, 0>(p, forced_L, s);
	case 1: return launch_x_one<FMT, 1>(p, forced_L, s);
	case 2: return launch_x_one<FMT, 2>(p, forced_L, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace

int frontend_x_granule(int fmt) { return fmt == 0 ? XFmt<0>::G : (fmt == 3 ? XFmt<3>::G : XFmt<1>::G); }

cudaError_t launch_frontend_x(const FeParams &p, int fmt, int k, int forced_L, cudaStream_t s) {
	switch (fmt) {
	case 0: return launch_x_fmt<0>(p, k, forced_L, s);
	case 1: return launch_x_fmt<1>(p, k, forced_L, s);
	case 2: return launch_x_fmt<2>(p, k, forced_L, s);
	case 3: return launch_x_fmt<3>(p, k, forced_L, s);
	default: return cudaErrorInvalidValue;
	}
}

} // namespace aisgpu
