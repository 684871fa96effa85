// params.h -- parameter blocks, per-row state records and launch entry points of the kernels (host and device view).
//
// Layout in HBM (one engine == one batch of B independent IQ streams, "row" = stream*2 + channel; single-channel mode: row = stream):
//   in     [B][N]              input samples of one submit (CF32 float2, CU8/CS8/CS16, F32_FS4 floats, or DC16H word triples)
//   tail   [B][P]              last P input samples of the previous submit (front-end warm-up history)
//   rot    [P96 + N>>k]        Rotate phasor table of the submit (shared by all streams), with P96 history
//   Cbuf   [2B][HC + n48max]   48 kHz channel samples; new samples land at offset HC, unconsumed/history before (FM-discriminator
//                              input: real samples in the same bytes, new ones from float 2 * HC)
//   Ebuf   [2B][HE + nEmax]    samples entering the symbol-timing stage (FIR17 out, or FIR37 out for FM models)
//   state  PS/decoder/CGF/FIR  small per-row / per-(row,phase) structs
//   frames ring of FrameRec    decoded frames of the submit
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace aisgpu {

constexpr int FE_HIST = 6;   // >= 5, even so that even sample indices stay 16-byte aligned
constexpr int FE_SLACK = 12; // over-read room behind each array for partial runs
constexpr int FE_MAXK = 7;

// The kernels' FMT template parameter.  0 .. 3 are the public AISGPU_FMT_* values; 4 is CU8 through the integer CIC stages
// (-go FP_DS on, fe_stream.cuh), so F32_FS4 (public value 4) and DC16H (public value 7) have ids of their own.  fe_fmt_id is the
// one place the public value is translated: every launch entry point below takes its result.
constexpr int FE_FMT_FPDS = 4, FE_FMT_FS4 = 5, FE_FMT_DC16H = 6;
inline int fe_fmt_id(int public_format) { return public_format == 4 ? FE_FMT_FS4 : (public_format == 7 ? FE_FMT_DC16H : public_format); }
__host__ __device__ constexpr int fe_fmt_bps(int fmt) { // bytes per sample
	return fmt == 0 ? 8 : (fmt == FE_FMT_DC16H ? 12 : ((fmt == 3 || fmt == FE_FMT_FS4) ? 4 : 2));
}

struct FeParams {
	const void *in;       // [B][in_stride] samples
	const void *tail;     // [B][P]
	long long in_stride;  // in samples
	int format, k, N, P, seg_len, tile;
	int use_fdc;
	float fdc_alpha, fdc_beta;
	const float2 *rot;    // [P96 + N>>k]
	float2 *C;            // [2B][c_stride]
	long long c_stride;
	int c_off;
	int off_in[2];           // smem offsets (float2 units) of the two input-ring buffers (level 0, each [HIST | tile])
	int off_rot[2];          // phasors of the tile
	int off_lv[FE_MAXK + 1]; // level arrays 1..k (off_lv[0] unused)
	int off_up, off_dn, off_wa, off_wb;
	int st_L, st_q, st_r, st_B; // streaming kernel: lanes per stream, super-steps per lane (the last st_r lanes of a stream take st_q + 1), streams
	int st_first;           // 1 in the first block of a stream (the integer front end's virtual history, see fe_stream.cuh)
	int st_cap;             // resident CTAs per SM the lane planner counts on (0 = what fits)
	int smem_f2;          // total float2
	float2 *D0;           // PRE mode (decimation in front of DSP::Upsample): level-K samples, [B][d0_stride], sample i at d0_off + i
	long long d0_stride;
	int d0_off;
};

constexpr int CGF_N = 512;
constexpr int CGF_BLK_PER_CTA = 16;
constexpr int CGF_THREADS = 256;
constexpr int CGF_ROWP = 513;           // padded row (floats) so 16 lanes scanning 16 rows hit 16 banks
constexpr int CGF_IDX_OFFSET = 3;       // idx = i + 3, i in [-3, 410]
constexpr int CGF_IDX_NONE = 414;       // no bin above zero: fz = -1
constexpr int CGF_NIDX = 415;

constexpr int FIRC_T = 17;
constexpr int FIRC_TILE = 256;

constexpr int FIRF_T = 37;
constexpr int FIRF_TILE = 256;
constexpr int FM5_THREADS = 128; // slots per CTA
constexpr int FM5_SAMPLES = FM5_THREADS * 5;
struct Fm5Params {
	const float2 *Cbuf;
	long long c_stride;
	int c_new, n;        // new samples start at Cbuf[row][c_new], n of them
	int r0;              // abs index of new sample 0 modulo 5: slot 0 starts r0 samples before it
	int nslots;
	float *Fbuf;         // FIR37 output, [rows][f_stride], new sample m at f_off + m; NULL: nobody reads it (the decoders take dbits)
	long long f_stride;
	int f_off;
	uint32_t *dbits;     // [rows*5][dwords]
	int dwords;
	float *tap_fm;       // optional
	long long tap_stride;
	float *tap_dec;      // optional: decoder input samples [rows*5][nslots], valid ones only, packed per phase
	int real;            // 1: the rows hold real samples (the FM-discriminator input model) that go straight into FIR37
};

enum { ST_TRAINING = 0, ST_STARTFLAG = 1, ST_DATAFCS = 3 };
constexpr int DEC_WORDS = 35;     // 140 bytes (Message.h:69 data[MAX_AIS_FRAME_BYTES + 4])
constexpr int MAX_FRAME_BITS = 1087; // MAX_AIS_FRAME_LENGTH (Message.h:41)
constexpr int K3_THREADS = 32; // one warp per CTA: the rows are few, spread them over all SMs

struct DecState { // one per (row, phase); persisted between submits (frame bits live in a separate array)
	int state, lastBit, prev, position, one_seq;
	float level;
	long long start_idx;
};
struct PsState { // PhaseSearchEMA (Demod.h:68-86) / PhaseSearch (Demod.h:41-66)
	float ma[16];
	uint32_t plane[5]; // plane[d] bit h = decision of hypothesis h, d symbols ago (bits[h] >> d & 1)
	int max_idx, rot, last;
};
struct FrameRec {
	int row, phase, nbits;
	float level;          // TAG::level before the dB conversion (AIS.h:147)
	float ppm;
	int chunk;            // ordinal of the submit
	long long start_idx, end_idx;
	uint32_t data[DEC_WORDS];
	int blk;              // ordinal of the front-end block (several per submit behind a resampler)
};

// Host side: the frame ring of one decoder launch, as the launchers take it (the kernels receive the fields one by one)
struct FrameOut {
	FrameRec *ring;
	unsigned long long *ring_head; // frames emitted since the engine was created (tickets); slot = ticket % ring_cap
	unsigned long long ring_limit; // tickets below this may be written: frames drained by the host at launch time + ring_cap
	int ring_cap;
	int chunk;                     // ordinal of the caller's submit
	int blk;                       // ordinal of the front-end block
	const uint32_t *level_rows;    // bit r of word r >> 5: row r's frames carry the signal level (its stream's tag_mode & 1)
};

// Whether row r's frames carry the signal level (FrameOut::level_rows)
__host__ __device__ __forceinline__ int row_level(const uint32_t *level_rows, int r) { return (int)((level_rows[r >> 5] >> (r & 31)) & 1u); }


struct K3Params {
	int ps_ema;
	int ps_rot0;          // PhaseSearchEMA: (symbols delivered before this submit) & 3 = the (1j)^rot phase of its first symbol
	int rows;
	int nsym;             // symbol slots (groups of 5 samples) to walk this submit
	long long e_stride;
	int e_begin;          // index in the row of the sample with absolute index abs_begin
	long long abs_begin;  // absolute per-channel index (TAG::sample_idx, DSP.h:110) of slot 0 / phase 0; multiple of 5
	long long abs_lo, abs_hi; // samples with abs_lo <= index < abs_hi exist this submit (Deinterleave forwards partial groups)
	const float2 *Ec;     // ModelDefault: FIR17 output
	const float *Ef;      // FM models: FIR37 output
	PsState *ps;
	float *ps_mem;        // PhaseSearch history |t| [16*12][rows*5] (only when !ps_ema)
	uint32_t *dbits;      // ModelDefault: demodulated bits, [rows*5][dwords], bit (s & 31) of word (s >> 5) = symbol s
	uint32_t *dbits2;     // ModelChallenger: the FM branch's decision bits, same layout
	int nslots_fm;        // ModelChallenger: slots the FM branch covers this submit
	const float *lvl_prev; // ModelChallenger: [rows] the level the tag carries into this block (read)
	float *lvl_prev_out;   //                  ... and into the next one (written; double buffered by launch)
	int lvl_own;           //                  1 (single-channel mode): a row carries its own last level; 0: channel A the one B left
	int dwords;
	float *lvl;           // ModelDefault: ScatterPLL level of symbol s (TAG::sample_lvl, DSP.h:100-106), [rows][lvl_stride]
	int lvl_stride;
	DecState *dec;
	uint32_t *dec_data;   // [DEC_WORDS][rows*5]
	FrameRec *ring;
	unsigned long long *ring_head; // frames emitted since the engine was created (tickets); slot = ticket % ring_cap
	unsigned long long ring_limit; // tickets below this may be written: frames drained by the host at launch time + ring_cap
	int ring_cap;
	int chunk;
	int blk;
	const uint32_t *level_rows; // FrameOut::level_rows
	// tag.ppm lookup (ModelDefault): block index of a sample = (abs_idx - blk_abs0) >> 9
	const int *stepidx;
	const float *ppmtab;
	long long blk_abs0;
	int nblk;
	float *tap_dec;       // optional: decoder input samples [rows*5][nsym]
	long long *dbg;       // optional per-row counters [rows][4]: cycles, frame-collecting steps, CRC runs, CRC bits
};

constexpr int K3_TS = 32;                 // symbols staged per tile
constexpr int K3_ROWLEN = K3_TS * 5;      // samples of one row in a tile

struct PllState { int prev; float pll; int fast; };

constexpr int PS_THREADS = 128;
constexpr int DK_THREADS = 128;
constexpr int DK3_WARPS = 2;
constexpr int DSK_T = 26;
constexpr int DSK_THREADS = 256;


// V2::Engine (Decoder/V2/V2Engine.h:95-155) per (stream, channel): everything the engine carries from block to block
struct V2State {
	float2 fo_rot;        // FreqOffset::rot
	float2 slot_ema;      // slot-phase EMA
	float2 fm_prev;       // FMDemod::prev
	float last_f, ppm, pll_phase;
	int slot_phase, di, pll_last;
	long long sample_idx;
	float2 f17_hist[16];  // FilterFL17::buffer
	float f37_hist[36];   // FilterFL37::buffer
	unsigned trk_rot[5];  // PhaseTracker x 5
	float2 trk_s[5];
	int trk_prev[5];
};

// ---- launch entry points (one translation unit per kernel family; every function returns cudaGetLastError()); `fmt` is a
// ---- kernel format id (fe_fmt_id), cudaErrorInvalidValue for one the family has no kernel for ----
// fe_misc.cu
cudaError_t launch_rot_table(float2 *tab, const float2 *prev_tail, const float2 *state_in, float2 *state_out, float2 mult, int P96, int n96, cudaStream_t s);
cudaError_t launch_upsample(const float2 *D0, long long d0_stride, int d0_off, const int *src, const float *alpha, int M, int B, float2 *S, long long s_stride,
                            long long m0, int cap, cudaStream_t s);
cudaError_t launch_d0_carry(float2 *D0, long long d0_stride, int d0_off, int L, int rows, cudaStream_t s);
cudaError_t launch_dsk(int fmt, const void *in, long long in_stride, const void *tail, int tail_len, int first, int n_out, int B, float2 *S, long long s_stride,
                       long long j0, int cap, cudaStream_t s);
// last p_b bytes of (old_tail ++ the first n_b bytes of each input row) -> new_tail; rows of `in` are in_stride_b bytes apart
cudaError_t launch_tail_update(void *new_tail, const void *old_tail, const void *in, long long in_stride_b, long long n_b, int p_b, int B, cudaStream_t s);
cudaError_t launch_carry_f2(float2 *buf, long long stride, int src_begin, int dst_begin, int cnt, int rows, cudaStream_t s);
cudaError_t launch_carry2_f2(const float2 *src, float2 *dst, long long stride, int src_begin, int dst_begin, int cnt, int rows, cudaStream_t s);
cudaError_t set_taps_bh28_3(const float *taps26);
// engine groups (aisgpu_attach) and the channel dump (aisgpu_dump_open): float2 elements [src_off, src_off + n) of every row of src
// (rows src_stride apart) into elements [dst_off, dst_off + n) of the same row of each of the nd (<= GROUP_MAX - 1) buffers dst[]
// (rows dst_stride apart); strides, offsets and n are even
constexpr int GROUP_MAX = 8; // engines in one group, the leader included
cudaError_t launch_c_fanout(const float2 *src, long long src_stride, int src_off, float2 *const *dst, int nd, long long dst_stride, int dst_off, int n,
							int rows, cudaStream_t s);
// tune.cu: the per-stream digital tune (aisgpu_set_tunings).  R input rows of N samples in format fmt (in_stride samples apart) -> R * T
// CF32 rows of out (out_stride apart, from element out_off), input row r feeding streams rT .. rT + T - 1; sample i of the submit is
// sample first + i of its stream; fk[s]: stream s's offset modulo fs in [0, fs) (0: converted only); tab: tune_tables(fs), tab_len =
// tune_table_len(fs) entries.  At most `ctas` CTAs.
struct TuneParams {
	const void *in;
	long long in_stride;
	float2 *out;
	long long out_stride;
	int out_off;
	int N, R, T, fs, tab_len;
	long long first;
	const int *fk;
	const float2 *tab;
};
int tune_table_len(int fs);
void tune_tables(int fs, float2 *tab);
cudaError_t launch_tune(const TuneParams &p, int fmt, int ctas, cudaStream_t s);
// fe_tiled.cu
cudaError_t launch_frontend_tiled(const FeParams &p, int fmt, int k, bool pre, dim3 grid, size_t smem, cudaStream_t s);
// fe_stream_f*.cu: the launcher picks the lanes per stream (st_plan in fe_stream.cuh) unless forced_L > 0
cudaError_t launch_frontend_stream(const FeParams &p, int fmt, int k, bool pre, int forced_L, cudaStream_t s); // cudaErrorNotSupported: no shape for k, or the block does not fit the kernel
cudaError_t launch_frontend_stream_fpds(const FeParams &p, int forced_L, cudaStream_t s); // fe_stream_fp.cu: CU8, integer CIC stages, 1536K
// fe_x.cu: single-channel mode, k = 0 .. 2 CIC stages, one Cbuf row per stream; p.N and p.P multiples of frontend_x_granule(fmt)
cudaError_t launch_frontend_x(const FeParams &p, int fmt, int k, int forced_L, cudaStream_t s);
int frontend_x_granule(int fmt);
// fe_disc.cu: FM-discriminator input (-m 3), ConvertRAW and the I / Q split into real rows 2 * stream (I) and 2 * stream + 1 (Q) of
// p.C, sample i at float 2 * p.c_off + i; p.N even
cudaError_t launch_frontend_disc(const FeParams &p, int fmt, cudaStream_t s);
// be_cgf.cu
cudaError_t cgf_init(const float *taps17, const float2 *omega256);
cudaError_t launch_cgf_estimate(const float2 *Cbuf, long long c_stride, int c_begin, int nblk, int total_blocks, const float2 *omega, int wide, int *stepidx, cudaStream_t s);
cudaError_t launch_cgf_fused(const float2 *Cbuf, long long c_stride, int c_begin, const int *stepidx, const float2 *steptab, float2 *rot_state, int nblk, int rows,
                             const float2 *hist_old, float2 *hist_new, float2 *Ebuf, long long e_stride, int e_off, float2 *tap_cgf, long long tap_stride, cudaStream_t s);
// be_v2.cu
cudaError_t v2_init(const float *taps17, const float *taps37, const float2 *omega256);
cudaError_t launch_v2_engine(const float2 *Cbuf, long long c_stride, int c_begin, int nproc, int rows, V2State *st, DecState *dec, uint32_t *dec_data,
                             const FrameOut &out, const float2 *omega_g, float w_train, float w_track, float2 *tap_fc, float2 *tap_coh, float *tap_fmf,
                             long long tap_stride, cudaStream_t s);
// be_fm.cu
cudaError_t fm_init(const float *taps37);
cudaError_t launch_fm_fir5(const Fm5Params &p, int rows, cudaStream_t s);
// be_sym.cu
cudaError_t sym_init(const float *ps_cos8, const float *ps_sin8, const uint32_t *abort_bits35);
cudaError_t launch_phase_search(const K3Params &p, cudaStream_t s);
cudaError_t launch_decode(int model, int decoder, int rpw, const K3Params &p, cudaStream_t s);
cudaError_t launch_decode10(int rpw, const K3Params &p, cudaStream_t s);
// out.level_rows is not read: k_base always sums the level (its sample levels are 0)
cudaError_t launch_base(const float *Ef, long long e_stride, int e_begin, int n, int rows, PllState *pll, DecState *dec, uint32_t *dec_data,
                        const FrameOut &out, float *tap_dec, int *tap_cnt, cudaStream_t s);

} // namespace aisgpu
