// aisgpu.cu -- host side of the C ABI declared in include/aisgpu.h.
//
// Mirrors, for a batch of streams, what AIS::ModelFrontend::buildModel + ModelDefault/Standard/Base::buildModel
// wire up for one stream (reference Source/DSP/Model.cpp:27-356, 419-438, 484-577): the rate -> chain table, the
// filter parameters, and the per-submit launch sequence of the kernels in aisgpu_kernels.cuh.  The only
// arithmetic done on the host is the libm-dependent constant tables (Rotate step, FFT twiddles, CGF phasor
// steps, Model.cpp:31, FFT.h:81-83, DSP.cpp:457-458) and the per-frame tail of AIS::Decoder::processData
// (dB level, validate, buildNMEA: AIS.cpp:66-96, Message.cpp:398-413, 569-686).  No CPU fallback exists.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <chrono>
#include <deque>
#include <memory>
#include <string>
#include <vector>

#include "../../include/aisgpu.h"
#include "be_json.h"
#include "dump.h"
#include "params.h"

using namespace aisgpu;

namespace {

thread_local std::string g_create_error;

const float PI_F = 3.14159265358979323846f; // Library/Common.h:318

float2 polar1(float theta) { // std::polar(1.0f, theta) through sincosf, as the reference build resolves it
	float s, c;
	sincosf(theta, &s, &c);
	return make_float2(1.0f * c, 1.0f * s);
}

const float H_TAPS_RECEIVER[37] = { // DSP/Filters.h:24-33
	0.00119025f, -0.00148464f, -0.00282428f, -0.00200561f, -0.00068852f, 0.00343044f, 0.00902093f, 0.01367867f,
	0.01147965f, 0.0027259f, -0.01766614f, -0.04244429f, -0.0577468f, -0.05245161f, -0.01072754f, 0.0732564f,
	0.17643278f, 0.25582214f, 0.28200453f, 0.25582214f, 0.17643278f, 0.0732564f, -0.01072754f, -0.05245161f,
	-0.0577468f, -0.04244429f, -0.01766614f, 0.0027259f, 0.01147965f, 0.01367867f, 0.00902093f, 0.00343044f,
	-0.00068852f, -0.00200561f, -0.00282428f, -0.00148464f, 0.00119025f };
const float H_TAPS_COHERENT[17] = { // DSP/Filters.h:35-41
	2.06995719e-06f, 3.18610148e-05f, 3.40605309e-04f, 2.52892989e-03f, 1.30411453e-02f, 4.67076746e-02f,
	1.16186141e-01f, 2.00730781e-01f, 2.40861391e-01f, 2.00730781e-01f, 1.16186141e-01f, 4.67076746e-02f,
	1.30411453e-02f, 2.52892989e-03f, 3.40605309e-04f, 3.18610148e-05f, 2.06995719e-06f };
const float H_TAPS_BH28_3[26] = { // DSP/Filters.h:43-53
	6.32542387e-05f, -2.90015252e-04f, -1.54206250e-03f, -1.64972455e-03f, 3.12793899e-03f, 1.09494413e-02f,
	9.04975801e-03f, -1.43685846e-02f, -4.45615933e-02f, -3.44883647e-02f, 5.53474269e-02f, 2.01827915e-01f,
	3.16534610e-01f, 3.16534610e-01f, 2.01827915e-01f, 5.53474269e-02f, -3.44883647e-02f, -4.45615933e-02f,
	-1.43685846e-02f, 9.04975801e-03f, 1.09494413e-02f, 3.12793899e-03f, -1.64972455e-03f, -1.54206250e-03f,
	-2.90015252e-04f, 6.32542387e-05f };
const float H_PS_COS[8] = { 9.9518472640441780e-01f, 9.5694033335306883e-01f, 8.8192125790916542e-01f, 7.7301044123076901e-01f,
							6.3439326515712957e-01f, 4.7139671032286945e-01f, 2.9028464326824349e-01f, 9.8017099547459546e-02f }; // Demod.h:29-31
const float H_PS_SIN[8] = { 9.8017143048367339e-02f, 2.9028468509743588e-01f, 4.7139674887287397e-01f, 6.3439329894649099e-01f,
							7.7301046896098113e-01f, 8.8192127851457169e-01f, 9.5694034604181499e-01f, 9.9518473068888236e-01f };

constexpr int HC = 1024; // room in front of new 48 kHz samples: unconsumed CGF samples (<512), FM/FIR history (37), or the V2 engine's
                         // block awaiting its lookahead plus a partial block (<1024)
constexpr int V2_BLK = 512; // V2::BLOCK_SIZE (V2Engine.h:30)
constexpr int HD = 48;  // ModelChallenger: derotated samples kept in front of the new ones (FM needs 1, FIR37 36, a partial group 4)
constexpr int HE = 8;   // room in front of new symbol-stage samples: an incomplete group of 5 (<=4)

// the tiled front end (the CIC stages below 768 kS/s, and of blocks the streaming kernel declines): input samples per tile --
// one run of 5 outputs per thread of a four-warp CTA at the first CIC stage, 2 x 5 x 128 -- and the CTAs a submit is cut into
// (segments x streams, several waves over the SMs)
constexpr int FE_TILE = 1280;
constexpr int FE_CTAS = 4096;

constexpr int X_GRANULE = 64; // single-channel mode: a multiple of every format's front-end lane chunk (frontend_x_granule); also the
                              // FM-discriminator input model's granule

int bytes_per_sample(int fmt) { return fe_fmt_bps(fe_fmt_id(fmt)); }
bool format_known(int fmt) { return (fmt >= AISGPU_FMT_CF32 && fmt <= AISGPU_FMT_F32_FS4) || fmt == AISGPU_FMT_DC16H; } // 5 and 6 are not formats

// A ring of pre-stage output (Upsample's at the bucket rate, DownsampleKFilter's at 96 kS/s), one row of `stride` samples per stream;
// positions only grow, position p lives in slot p % cap.
struct PreRing {
	float2 *d = nullptr;
	int cap = 0;
	long long stride = 0;
	long long produced = 0, consumed = 0; // samples written / handed to the next stage
	long long last = 0;                   // produced when the last submit began: AISGPU_TAP_PRE / _PRE2 read [last, produced)
};

// What runs behind the 48 kHz rows, chosen once from the model: each chain has its own state, allocation and step function.
enum class Chain {
	Fm,       // ModelStandard, ModelBase, ModelDiscriminator: FM -> FIR37 -> five decoders, or Base's SimplePLL tail
	Coherent, // ModelDefault, ModelChallenger: CGF -> derotation + FIR17 -> phase search -> decoders (+ Challenger's FM branch)
	V2,       // ModelV2: one kernel per block of the V2 engine
};

// The back-end stages that are pipelined over two streams (aisgpu_handle::be_streams), named by what they carry from one submit
// into the next.
enum Stage {
	STAGE_FM_FIR,       // FM chain: FM + FIR37 + slicer (Ef is single buffered)
	STAGE_DEROT_FIR,    // coherent chain: phasor chain + derotation + FIR17 (CGF rotation state, FIR17 history)
	STAGE_PHASE_SEARCH, // coherent chain: phase search state, and the incomplete group of 5 carried into the other Ec buffer
	STAGE_DECODE,       // decoder state
	STAGE_CBUF_CARRY,   // the samples carried in front of HC of the next submit's Cbuf
	STAGE_FM_BRANCH,    // ModelChallenger: FM branch on the derotated samples (reads Ed, single buffered, and carries its history)
	NSTAGE
};

// What aisgpu_set_receivers gives each stream: its channel letters, own MMSI and tag mode (what drain_ring reads), and the TAG fields
// its records are printed with.  Without a table every stream holds the config's fields.
struct Receiver {
	char channel_a = 'A', channel_b = 'B';
	int32_t station = 0, own_mmsi = -1;
	uint32_t tag_mode = 3;
	int32_t driver = 0;
	std::string hardware;
	uint32_t ipv4 = 0;
};

// The receive time of every submit (aisgpu_set_clock), one per group: the leader's submits append to it and the members read it.
// at[c] is S_c, the samples per stream submitted through submit c (counters[2] after it), for a recording clock, and the system
// clock in microseconds since the epoch, read by submit c, for a live one.
struct Clock {
	bool live = false;
	long long fs = 0;
	std::vector<long long> start_us; // recording: the time of each stream's first sample
	std::vector<long long> at;
	// start_us[s] + floor(S_c * 10^6 / fs) without overflow, or the wall time of submit c
	long long stamp(int s, long long c) const {
		if (live) return at[(size_t)c];
		const long long S = at[(size_t)c], q = S / fs, r = S % fs;
		return start_us[(size_t)s] + q * 1000000 + r * 1000000 / fs;
	}
};

} // namespace

struct aisgpu_handle {
	aisgpu_config cfg;
	int k = 0, P = 0, P96 = 0, bps = 8;
	// Rates the reference serves through DSP::Upsample (non-bucket rates, Model.cpp:134-149) or DSP::DownsampleKFilter
	// (the DSK buckets, Model.cpp:208-218, 308-313) get a pre-stage of up to three stages, in this order:
	//  - CIC: kA x Downsample2CIC5 of the caller's input into D0 (with kA = 0 only the format conversion), when Upsample runs or kA > 0;
	//  - Upsample: D0 -> us_ring;
	//  - DSK: DownsampleKFilter(BlackmanHarris_28_3, 3) of the caller's input, of D0 or of every whole Upsample block -> dsk_ring.
	// The front end proper then runs once per whole block of the last ring with k = the CIC stages behind the resampler ("inner" submits).
	bool pre_us = false, pre_dsk = false;
	int kA = 0, PA = 0;   // CIC stage: its stages and their warm-up history (input samples)
	int in_fmt = 0;       // sample format the front end proper reads (CF32 behind a pre-stage)
	int outer_N = 0;      // submit length of an Upsample engine (must not change: the reference's block sizes depend on it)
	int blk = 0;          // reference block length entering the front end proper (L_us or 8192)
	int us_blk = 0;       // Upsample block: outer_N >> kA
	long long d0_stride = 0;
	float us_alpha = 0.0f, us_inc = 1.0f;     // Upsample::alpha / increment (DSP.h:165)
	int dsk_first = 0;                         // DownsampleKFilter::idx_in
	PreRing us_ring, dsk_ring;
	unsigned char *d_raw_tail[2] = { nullptr, nullptr }; // raw-format history of the stage that reads the caller's input (CIC or DSK)
	int raw_tail_cur = 0;
	float2 *d_cf_tail[2] = { nullptr, nullptr };         // CF32 history of a DSK behind the CIC stage (it reads D0 or Upsample blocks)
	int cf_tail_cur = 0;
	float2 *d_D0 = nullptr;
	int *d_us_src = nullptr;
	float *d_us_alpha = nullptr;
	FeParams fe_pre;
	long long msg_chunk = 0; // ordinal of the caller's submit (what frames are tagged with)
	int obps = 8;            // bytes per sample of the caller's format (bps: of what the front end proper reads)
	int pbps = 8;            // bytes per sample of what the pre-stage reads: the caller's format, CF32 behind the tune
	int inner_max = 0;       // longest block the front end proper can be handed
	int use_fdc = 0;
	int fp_ds = 0; // integer CIC front end (DS_UINT16 x 4, DSP.cpp:499-665): CU8 @1536K with -go FP_DS on
	int xmode = 0; // single-channel mode (AISGPU_MODE_X): no Rotate, one back-end row per stream
	int disc = 0;  // FM-discriminator input (AISGPU_MODEL_DISCRIMINATOR): I and Q are two real 48 kHz rows, no Rotate, no CIC stage
	int us_ratio = 0; // ceil(bucket / rate): most DSP::Upsample outputs per input sample (AB: 2, X and model 3: <= 4)
	float fdc_alpha = 0, fdc_beta = 1;
	int rows = 0;
	int max_n48 = 0;
	int st_L = 0; // AISGPU_ST_L: lanes per stream of the streaming front end (0: the launcher plans)
	Chain chain = Chain::Fm;
	int dec_rpw = 3, decoder = 3; // AISGPU_DEC_RPW: rows per warp of the word-parallel decoder; AISGPU_DECODER=1: the bit-serial one
	// fe_stream: front end + input history; stream: everything behind the 48 kHz buffers (the stream handed to callers
	// for timing).  The front end of submit c+1 overlaps the back end of submit c; Cbuf is double buffered for that.
	cudaStream_t stream = nullptr, copy_stream = nullptr, fe_stream = nullptr;
	// Back-end stages of consecutive submits are pipelined: submit c runs on be_streams[c & 1] (be_streams[0] == stream);
	// stage s (enum Stage) of submit c waits for stage s of submit c-1 (its carried state) through ev_stage[s][(c-1) & 1]; the
	// buffers between stages are double buffered (index c & 1).  With taps enabled everything stays on one stream.
	cudaStream_t be_streams[2] = { nullptr, nullptr }, bs = nullptr;
	cudaEvent_t ev_stage[NSTAGE][2] = {};
	bool stage_rec[NSTAGE][2] = {};
	// Ec (FIR17 output, coherent chains) is double buffered: the fused derotation kernel of submit c + 1 writes one buffer while the
	// phase search of submit c still reads the other (with a single buffer the chain fused -> phase search of ALL submits was one
	// serial sequence).  ec_cur: the buffer the next block of symbols goes to; ev_ec_read[i]: the last reader of buffer i.
	int ec_cur = 0, ec_last = 0;
	cudaEvent_t ev_ec_read[2] = { nullptr, nullptr };
	bool ec_read_rec[2] = { false, false };
	cudaEvent_t ev_join = nullptr;
	int pb = 0; // buffer parity of the submit being enqueued
	static const int NC = 3; // ring of 48 kHz buffers: the front end may run two submits ahead of the back end
	cudaEvent_t ev_fe_done[3] = { nullptr, nullptr, nullptr }, ev_be_done[3] = { nullptr, nullptr, nullptr };
	bool be_recorded[3] = { false, false, false };
	static const int NEV = 128;
	cudaEvent_t ev_fe0s[128] = { nullptr }, ev_fe1s[128] = { nullptr };
	cudaEvent_t ev_copy[2] = { nullptr, nullptr }, ev_done[2] = { nullptr, nullptr };
	bool fe_timed = false;
	// input staging for host submits
	unsigned char *d_in[2] = { nullptr, nullptr };
	int in_cur = 0;
	bool in_used[2] = { false, false };
	unsigned char *d_tail[2] = { nullptr, nullptr };
	int tail_cur = 0;
	// Rotate
	// Rotate: table c lives in slot c % 3, rot state after chunk c in d_rot_state[1 + c % 3] (slot 0 = initial state);
	// tables are produced on side_stream, one submit ahead when the chunk length repeats
	float2 *d_rot[3] = { nullptr, nullptr, nullptr };
	int rot_n96[3] = { 0, 0, 0 };
	long long rot_ready_chunk = -1; // newest chunk whose table has been enqueued on side_stream
	int rot_cur = 0;
	float2 *d_rot_state = nullptr;  // [4]
	cudaStream_t side_stream = nullptr;
	cudaEvent_t ev_rot[3] = { nullptr, nullptr, nullptr }, ev_k1[3] = { nullptr, nullptr, nullptr };
	bool k1_recorded[3] = { false, false, false };
	float2 mult;
	// 48 kHz channel buffer
	float2 *d_C2[3] = { nullptr, nullptr, nullptr };
	int c_last = 0; // buffer the last submit's front end wrote
	long long c_stride = 0;
	int c_hist = 0; // samples kept in front of HC
	// CGF
	long long cgf_abs = 0;
	int *d_stepidx2[2] = { nullptr, nullptr };
	float2 *d_steptab = nullptr, *d_omega = nullptr, *d_cgf_rot = nullptr;
	float *d_ppmtab = nullptr;
	long long r_stride = 0;
	float2 *d_fir_hist[2] = { nullptr, nullptr };
	int fir_cur = 0;
	float2 *d_tap_cgf = nullptr;
	// symbol stage
	float2 *d_Ec2[2] = { nullptr, nullptr };
	float *d_Ef = nullptr; // FIR37 output (FM chain, ModelChallenger's FM branch), single buffered
	long long e_stride = 0;
	int e_left = 0;
	long long e_abs = 0;
	PsState *d_ps = nullptr;
	float *d_ps_mem = nullptr;
	long long *d_dbg = nullptr; // AISGPU_DEBUG=1: per-row decoder counters (tap 6)
	uint32_t *d_dbits2[2] = { nullptr, nullptr };
	float *d_lvl2[2] = { nullptr, nullptr };
	int dwords = 0;
	DecState *d_dec = nullptr;
	uint32_t *d_dec_data = nullptr;
	uint32_t *d_level_rows = nullptr; // bit per row: its frames carry the signal level (FrameOut::level_rows)
	PllState *d_pll = nullptr;
	V2State *d_v2 = nullptr;     // V2 engine: per-row state
	float2 *d_Ed = nullptr;      // ModelChallenger: derotated 48 kHz samples [rows][HD + nE]
	long long ed_stride = 0;
	uint32_t *d_dbitsF[2] = { nullptr, nullptr };
	float *d_lvl_prev = nullptr; // [2][rows], double buffered by decode launch
	int lvlp_cur = 0;
	float2 *d_tap_coh = nullptr;
	float *d_tap_dec = nullptr, *d_tap_fm = nullptr;
	int *d_tap_cnt = nullptr;
	// frames
	// Circular frame ring.  Tickets (frames emitted since creation) only grow; the host owns `drained`.  Every submit
	// records, in stream order behind its decoders, the ring head into a pinned slot plus an event: aisgpu_poll_upto waits
	// for one submit only and later submits keep running.
	FrameRec *d_ring = nullptr;
	unsigned long long *d_ring_head = nullptr;
	int ring_cap = 0;
	unsigned long long drained = 0;           // tickets delivered to (or dropped for) the host
	static const int NT = 1024;               // submits whose completion record is kept
	unsigned long long *pin_head = nullptr;   // [NT] pinned: ring head after submit t (slot t % NT)
	cudaEvent_t ev_ticket[1024] = { nullptr };
	cudaEvent_t ev_mark = nullptr;
	std::deque<unsigned long long> launch_limit; // per undrained submit: drained-at-launch + ring_cap (what its kernels were given)
	long long polled_ticket = -1;             // newest submit whose frames have been drained
	bool overflow_pending = false;
	std::vector<FrameRec> h_ring;
	std::vector<aisgpu_msg> out_queue;
	size_t out_pos = 0;
	std::shared_ptr<Clock> clock; // aisgpu_set_clock (a member: its leader's); null: every record takes the output's rxtime_us
	std::vector<int> seq; // per-stream multi-sentence sequence id (Message.cpp:28-39 is process-global in the reference)
	std::vector<Receiver> rx; // per stream: the config's fields, or the receiver aisgpu_set_receivers installed
	bool rx_table = false;    // aisgpu_set_receivers has been called: the records take the receivers' TAG fields
	// The per-stream digital tune (aisgpu_set_tunings, tune.cu).  With a table every submit first runs k_tune on fe_stream: the
	// caller's n_streams / per_input input rows, converted and mixed by each stream's offset (input row r feeds streams
	// r * per_input .. r * per_input + per_input - 1), into d_tune [n_streams][tune_stride] as CF32, which everything behind it then
	// reads as a CF32 input (src_fmt); behind a resampler with no CIC stage (kA = 0) k_tune writes D0 directly and is the pre-stage's
	// conversion.  Without a table nothing of this is allocated or launched, and per_input is 1.
	bool tuned = false;
	int per_input = 1;
	float2 *d_tune = nullptr, *d_tune_tab = nullptr;
	long long tune_stride = 0;
	int *d_tune_fk = nullptr;
	int tune_ctas = 0;
	// last-submit geometry (for taps)
	int last_n = 0, last_n48 = 0, last_nE = 0, last_nsym = 0, last_launches = 0;
	uint64_t counters[8] = { 0 };
	long long chunk = 0;
	std::string err;
	int poisoned = 0; // a CUDA failure inside a submit leaves the carried state half-advanced: every later call returns this code
	FeParams fe;
	// pinned double buffer of the Upsample (input index, alpha) schedule
	int *pin_us_src[2] = { nullptr, nullptr };
	float *pin_us_alpha[2] = { nullptr, nullptr };
	cudaEvent_t ev_us[2] = { nullptr, nullptr };
	bool us_used[2] = { false, false };
	int us_cur = 0, us_cap = 0;
	// NCCL (resolved at run time): communicator of the job's ranks, device scratch of the counter all-reduce
	void *nccl_lib = nullptr, *nccl_comm = nullptr;
	unsigned long long *d_counts = nullptr;
	// Engine groups (aisgpu_attach): a member has no front end of its own; every inner submit of its leader copies the leader's new
	// 48 kHz rows into the member's own Cbuf ring (k_c_fanout on the leader's fe_stream, then ev_fan) and runs the member's back end.
	aisgpu_config given;                    // the caller's config as passed to aisgpu_create / aisgpu_attach (the rule compares these)
	bool member = false;                    // created by aisgpu_attach (stays set when the leader is destroyed)
	aisgpu_handle *leader = nullptr;        // member: its leader while both exist
	std::vector<aisgpu_handle *> members;   // leader: in attach order
	cudaEvent_t ev_fan = nullptr;           // leader: recorded behind k_c_fanout, waited on by every member's back end
	// The 48 kHz channel dump (aisgpu_dump_open).  Each inner submit's new rows are gathered (k_c_fanout on fe_stream, behind
	// ev_fe_done) into columns [dump_off, dump_off + n48) of the submit's device slot [rows][dump_n]; after the last pass dump_stream
	// copies the slot into its pinned twin and records ev_dump.  The caller's thread writes the pinned slot to the files (dump_write).
	// Slot s is reused by submit j only after the host has written its previous contents, which also means that the previous copy
	// out of d_dump[s] has finished.  Nothing of this is allocated or launched while no dump has been opened.
	static const int ND = 3;
	aisgpu::ChannelDump *dump = nullptr;
	cudaStream_t dump_stream = nullptr;
	float2 *d_dump[3] = { nullptr, nullptr, nullptr }, *pin_dump[3] = { nullptr, nullptr, nullptr };
	cudaEvent_t ev_dump[3] = { nullptr, nullptr, nullptr }, ev_export = nullptr;
	long long dump_cap = 0;  // samples per row a slot holds: the most one submit can yield
	long long dump_next = 0; // submits that have filled a slot; slot dump_next % ND is the next one
	struct DumpPending {
		long long ticket, n;
		int slot;
	};
	std::deque<DumpPending> dump_pending; // slots copied or being copied, not yet written, in submit order
	int dump_slot = -1;                   // the submit being enqueued: its slot (-1: no export), row length and columns exported so far
	long long dump_n = 0, dump_off = 0;
	// The output records (aisgpu_lines_enable; aisgpu_json_enable is JSON_FULL with suffix "\n").  Every drain of the frame ring
	// uploads the frames it publishes to d_jmsg, kJsonBatch at a time, and formats them on json_stream (be_json.cu: the NMEA_TAG
	// group counts, a record per frame into its slot, the placement within json_cap bytes per submit, the packed text); the text
	// comes back through pin_jtext and is appended to json_buf, which aisgpu_poll_lines / aisgpu_poll_json hand out from json_pos
	// on, and the kept records' lengths (pin_jkeep) to rec_len.  fmt_records / fmt_groups are the engine's counters (frames
	// published, multi-sentence ones among them), carried from batch to batch.  Frames and records are queued side by side and
	// each is read by its own poll; neither queue keeps more than ring_cap unread entries: the oldest are dropped and the next poll
	// of that kind returns AISGPU_EOVERFLOW.  Nothing of this exists while no format has been enabled.
	bool json_on = false, json_api = false;
	int fmt = 0, json_slot = 0, rec_cap = 0;
	long long json_cap = 0, fmt_records = 0, fmt_groups = 0;
	// The output's tag (its strings owned here): with a receiver table, stream s's records are printed with it and s's receiver's
	// station, driver, hardware, mode and ipv4, one context per stream.
	aisgpu_tag fmt_tag = {};
	std::string fmt_hw, fmt_uuid, fmt_suffix;
	std::string fmt_strings; // uuid and suffix, then every context's hardware and full-JSON prefix, each NUL-terminated
	FmtCtx *d_fctx = nullptr; // [1], or [n_streams] with a receiver table
	cudaStream_t json_stream = nullptr;
	char *d_jstrings = nullptr, *d_jslots = nullptr, *d_jtext = nullptr;
	aisgpu_msg *d_jmsg = nullptr;
	int *d_jlen = nullptr, *d_jseg = nullptr, *d_jkeep = nullptr, *pin_jkeep = nullptr;
	long long *d_jstamp = nullptr;    // with a clock: the stamps of a batch's frames, beside d_jmsg
	std::vector<long long> json_stamp;
	long long *d_jpsum = nullptr, *d_joff = nullptr, *d_jtotal = nullptr, *pin_jtotal = nullptr, *d_jgroups = nullptr;
	char *pin_jtext = nullptr;
	std::vector<int> json_seg;
	std::deque<int> rec_len; // the unread records' lengths
	bool queue_overflow_pending = false;
	std::string json_buf;
	size_t json_pos = 0;
	bool json_overflow_pending = false;
	// everything dalloc, halloc and new_event created: aisgpu_destroy releases these (the streams are destroyed one by one)
	std::vector<void *> dev_mem, host_mem;
	std::vector<cudaEvent_t> events;
};

namespace {

// The back end's rows and the (stream, channel) they stand for: AB rows are stream * 2 + channel, single-channel rows are streams.
int rows_of(const aisgpu_handle *h) { return h->xmode ? h->cfg.n_streams : 2 * h->cfg.n_streams; }
int row_of(const aisgpu_handle *h, int stream, int channel) { return h->xmode ? stream : stream * 2 + channel; }
int stream_of_row(const aisgpu_handle *h, int row) { return h->xmode ? row : row >> 1; }
int channel_of_row(const aisgpu_handle *h, int row) { return h->xmode ? 0 : row & 1; }

#define CU(call)                                                                                   \
	do {                                                                                           \
		cudaError_t e_ = (call);                                                                   \
		if (e_ != cudaSuccess) {                                                                   \
			char b_[256];                                                                          \
			snprintf(b_, sizeof(b_), "%s:%d %.120s: %s", "aisgpu.cu", __LINE__, #call, cudaGetErrorString(e_)); \
			h->err = b_;                                                                           \
			return AISGPU_ECUDA;                                                                   \
		}                                                                                          \
	} while (0)

template <typename T>
int dalloc(aisgpu_handle *h, T **p, size_t n) {
	{
		const cudaError_t e = cudaMalloc((void **)p, n * sizeof(T));
		if (e == cudaErrorMemoryAllocation) {
			char b[160];
			snprintf(b, sizeof(b), "out of device memory allocating %zu bytes", n * sizeof(T));
			h->err = b;
			(void)cudaGetLastError();
			*p = nullptr;
			return AISGPU_ENOMEM;
		}
		CU(e);
	}
	h->dev_mem.push_back(*p);
	CU(cudaMemsetAsync(*p, 0, n * sizeof(T), h->stream));
	return 0;
}

template <typename T>
int halloc(aisgpu_handle *h, T **p, size_t n) { // pinned host memory
	if (cudaMallocHost((void **)p, n * sizeof(T)) != cudaSuccess) {
		h->err = "out of pinned host memory";
		(void)cudaGetLastError();
		*p = nullptr;
		return AISGPU_ENOMEM;
	}
	h->host_mem.push_back(*p);
	return 0;
}

// Releases a buffer of dalloc / halloc before the handle is destroyed (nothing may still use it)
template <typename T>
void dfree(aisgpu_handle *h, T *&p) {
	if (!p) return;
	h->dev_mem.erase(std::find(h->dev_mem.begin(), h->dev_mem.end(), (void *)p));
	cudaFree(p);
	p = nullptr;
}
template <typename T>
void hfree(aisgpu_handle *h, T *&p) {
	if (!p) return;
	h->host_mem.erase(std::find(h->host_mem.begin(), h->host_mem.end(), (void *)p));
	cudaFreeHost(p);
	p = nullptr;
}

cudaError_t new_event(aisgpu_handle *h, cudaEvent_t *ev, unsigned flags = cudaEventDisableTiming) {
	const cudaError_t e = cudaEventCreateWithFlags(ev, flags);
	if (e == cudaSuccess) h->events.push_back(*ev);
	return e;
}

// Where this submit's decoders write their frames: they may fill the ring up to ring_cap tickets past what the host had drained
// when they were launched (mark_ticket keeps that limit for drain_ring).
FrameOut frame_out(const aisgpu_handle *h) {
	return FrameOut{ h->d_ring, h->d_ring_head, h->drained + (unsigned long long)h->ring_cap, h->ring_cap, (int)h->msg_chunk, (int)h->chunk,
					 h->d_level_rows };
}

void set_frame_out(K3Params &p, const FrameOut &o) {
	p.ring = o.ring;
	p.ring_head = o.ring_head;
	p.ring_limit = o.ring_limit;
	p.ring_cap = o.ring_cap;
	p.chunk = o.chunk;
	p.blk = o.blk;
	p.level_rows = o.level_rows;
}

// The level switch of every row from its stream's tag mode (bit 0: the frames carry the signal level, AIS.cpp:73-75) into
// d_level_rows, before the first submit
int put_level_rows(aisgpu_handle *h) {
	std::vector<uint32_t> bits((size_t)(h->rows + 31) / 32, 0u);
	for (int r = 0; r < h->rows; r++)
		if (h->rx[stream_of_row(h, r)].tag_mode & 1) bits[r >> 5] |= 1u << (r & 31);
	CU(cudaMemcpyAsync(h->d_level_rows, bits.data(), bits.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
	CU(cudaStreamSynchronize(h->stream));
	return 0;
}

bool has_cic(const aisgpu_handle *h) { return h->pre_us || h->kA > 0; }

// The format the first stage reads: the caller's, or the CF32 rows of the tune (aisgpu_set_tuning)
int src_fmt(const aisgpu_handle *h) { return h->tuned ? AISGPU_FMT_CF32 : h->cfg.format; }

// The rows the caller's submits hold: one per stream, or one per per_input streams behind a fan of tunings (aisgpu_set_tunings)
int inputs(const aisgpu_handle *h) { return h->cfg.n_streams / h->per_input; }

// A tuned engine whose CIC stage would only convert (a resampler behind no CIC stage): the tune writes D0 in its place
bool tune_into_d0(const aisgpu_handle *h) { return h->tuned && h->pre_us && h->kA == 0; }

// The CIC stage's warm-up history for h->kA stages (5 input samples per stage and level), rounded up to a whole number of
// super-steps of the streaming kernel (and even tiles at every level)
void plan_cic(aisgpu_handle *h) {
	const int g = std::max(4, 4 << h->kA);
	h->PA = std::max(g, (5 * ((1 << h->kA) - 1) + g - 1) / g * g);
}

// Upsample from sr to target behind h->kA CIC stages (Upsample::setParams, DSP.h:172-178)
void plan_upsample(aisgpu_handle *h, int sr, int target) {
	h->pre_us = true;
	h->in_fmt = AISGPU_FMT_CF32;
	h->us_inc = (float)sr / (float)target;
	h->us_ratio = (target + sr - 1) / sr;
	plan_cic(h);
}

// Model.cpp:35-107 (mode X): bucket 48K / 96K / 192K, k = 0 .. 2 CIC stages, Upsample straight behind convert at other rates
// (kA = 0), FilterComplex3Tap at 48 kHz behind the CIC stages (none at 48K); -go DSK / FP_DS / SOXR / SRC / MA are never read.
int plan_frontend_x(aisgpu_handle *h) {
	const int sr = h->cfg.sample_rate;
	if (sr < 12000 || sr > 192000) {
		h->err = "Model: sample rate must be between 12k and 192k (inclusive).";
		return AISGPU_EINVAL;
	}
	int bucket = 48000;
	while (bucket < sr) bucket *= 2;
	h->kA = 0;
	h->fp_ds = 0;
	h->in_fmt = src_fmt(h);
	h->k = bucket == 192000 ? 2 : (bucket == 96000 ? 1 : 0);
	if (bucket != sr) plan_upsample(h, sr, bucket); // "sample rate ...K upsampled to ...K." (Model.cpp:58-59)
	h->use_fdc = (h->cfg.droop && h->k > 0) ? 1 : 0;
	h->fdc_alpha = h->k == 2 ? -1.1f : -0.8f;
	h->fdc_beta = 1 - 2 * h->fdc_alpha; // DSP.h:293-297
	// history in input samples: FCIC5 5 + FDC 2 at 48 kHz, h_l = 2 h_{l-1} + 5 per CIC stage, rounded up to whole lane chunks
	int hk = 7;
	for (int i = 0; i < h->k; i++) hk = 2 * hk + 5;
	const int g = frontend_x_granule(fe_fmt_id(h->in_fmt));
	h->P = (hk + g - 1) / g * g;
	h->P96 = 0;
	return 0;
}

// Model.cpp:702-731 (-m 3): convert at 48 kHz, Upsample(fs -> 48000) straight behind convert below it, never a CIC stage; the
// channel mode is not read (ModelDiscriminator is a Model, not a ModelFrontend), and neither are droop / DSK / FP_DS.
int plan_frontend_disc(aisgpu_handle *h) {
	const int sr = h->cfg.sample_rate;
	if (sr > 48000) {
		h->err = "Internal error: sample rate not supported in FM discriminator model.";
		return AISGPU_EINVAL;
	}
	if (sr < 12000) { // the reference takes any lower rate; the Upsample ring here holds ratios up to 4 (< 1.25 samples per symbol below)
		h->err = "FM discriminator model: sample rate must be between 12k and 48k (inclusive).";
		return AISGPU_EINVAL;
	}
	h->disc = 1;
	h->kA = 0;
	h->k = 0;
	h->fp_ds = 0;
	h->in_fmt = src_fmt(h);
	if (sr != 48000) plan_upsample(h, sr, 48000); // US.setParams(sample_rate, 48000) (Model.cpp:722-728)
	h->use_fdc = 0;
	h->P = 0; // the split has no filter state: no warm-up history
	h->P96 = 0;
	return 0;
}

// Model.cpp:129-338: which bucket, how many CIC stages, droop taps, resampler.  Returns <0 when unsupported.
int plan_frontend(aisgpu_handle *h) {
	const int sr = h->cfg.sample_rate;
	if (h->cfg.channel_mode != AISGPU_MODE_AB && h->cfg.channel_mode != AISGPU_MODE_X) {
		h->err = "unknown channel_mode (AISGPU_MODE_AB or AISGPU_MODE_X)";
		return AISGPU_EINVAL;
	}
	if (h->cfg.model == AISGPU_MODEL_DISCRIMINATOR) return plan_frontend_disc(h); // the same two-row chain in AB and X
	h->xmode = h->cfg.channel_mode == AISGPU_MODE_X;
	if (h->xmode) return plan_frontend_x(h);
	if (sr < 96000 || sr > 12288000) {
		h->err = "Model: sample rate must be between 96K and 12288K (inclusive).";
		return AISGPU_EINVAL;
	}
	static const int rates_nodsk[] = { 96000, 192000, 288000, 384000, 768000, 1536000, 3072000, 6144000, 12288000 };                           // Model.cpp:129
	static const int rates_dsk[] = { 96000, 192000, 288000, 384000, 576000, 768000, 1152000, 1536000, 2304000, 3072000, 6144000, 12288000 }; // Model.cpp:130 (-go DSK on)
	int bucket = 0;
	if (h->cfg.dsk) {
		for (int b : rates_dsk)
			if (b >= sr) { bucket = b; break; }
	}
	else {
		for (int b : rates_nodsk)
			if (b >= sr) { bucket = b; break; }
	}
	const bool interp = bucket != sr; // "sample rate ...K upsampled to ...K." (Model.cpp:146-147)
	h->kA = 0;
	h->fp_ds = 0;
	h->in_fmt = src_fmt(h);
	int k_total = 0;
	if (bucket == 288000 || bucket == 576000 || bucket == 1152000 || bucket == 2304000) {
		// [kA x Downsample2CIC5 ->] [Upsample ->] DownsampleKFilter(BlackmanHarris_28_3, 3) -> ROT, no droop filter
		// (Model.cpp:208-218, 248-258, 278-288, 308-313)
		for (int b = bucket; b > 288000; b >>= 1) h->kA++;
		h->pre_dsk = true;
		if (interp) plan_upsample(h, sr, bucket);
		else if (h->kA) plan_cic(h);
		h->k = 0;
		h->blk = 8192; // DownsampleKFilter::outputSize (DSP.h:193)
		h->in_fmt = AISGPU_FMT_CF32;
	}
	else {
		for (int b = bucket; b > 96000; b >>= 1) k_total++;
		if (interp) { // Upsample sits in front of the last min(k, 2) CIC stages (Model.cpp:183-189 and siblings)
			const int post = k_total < 2 ? k_total : 2;
			h->kA = k_total - post;
			h->k = post;
			plan_upsample(h, sr, bucket);
		}
		else h->k = k_total;
	}
	if (h->cfg.fp_ds) { // -go FP_DS on: only the exact 1536K bucket has an integer front end, and it is fed by convert.outCU8 (Model.cpp:222-236)
		if (sr == 1536000 && h->cfg.format == AISGPU_FMT_CU8) h->fp_ds = 1;
		else if (sr == 1536000) {
			h->err = "FP_DS on: the integer front end (Downsample16_CU8, Model.cpp:233-236) needs CU8 input";
			return AISGPU_EINVAL;
		}
	}
	h->use_fdc = (h->cfg.droop && k_total > 0) ? 1 : 0;
	float a = 0.0f;
	switch (bucket) {
	case 12288000: case 6144000: a = -2.0f; break;
	case 3072000: a = -1.5f; break;
	case 1536000: case 768000: a = -1.2f; break;
	case 384000: a = -1.1f; break;
	case 192000: a = -0.8f; break;
	default: break;
	}
	h->fdc_alpha = a;
	h->fdc_beta = 1 - 2 * a; // DSP.h:293-297
	// history needed in input samples: h_0 = 17 (FDC 2 + DS2 5 + FCIC5 2*5), h_l = 2 h_{l-1} + 5
	const int k = h->k;
	int hk = 17;
	for (int i = 0; i < k; i++) hk = 2 * hk + 5;
	const int q = 1 << (k + 2);
	h->P = (hk + q - 1) / q * q;
	h->P96 = h->P >> k;
	return 0;
}

// granule of the caller's submit length: every CIC stage needs an even block (DSP.cpp:94,135)
int outer_granule(const aisgpu_handle *h) {
	if (h->xmode || h->disc) return X_GRANULE;
	if (h->fp_ds) return 16384; // 32 lane sub-segments of 512 samples: the shortest the streaming kernel takes (sub-segment >= warm-up history, 384)
	return h->pre_dsk ? std::max(64, 1 << (h->kA + 2)) : (1 << (h->k + h->kA + 2));
}

void layout_frontend(FeParams &p, int k, int tile) {
	int off = 0;
	auto take = [&](int n) {
		int o = off;
		off += (FE_HIST + n + FE_SLACK + 1) & ~1;
		return o;
	};
	p.off_in[0] = take(tile);
	p.off_in[1] = take(tile);
	p.off_rot[0] = take(tile >> k);
	p.off_rot[1] = take(tile >> k);
	p.off_lv[0] = 0;
	for (int l = 1; l <= k; l++) p.off_lv[l] = take(tile >> l);
	p.off_up = take(tile >> k);
	p.off_dn = take(tile >> k);
	p.off_wa = take(tile >> (k + 1));
	p.off_wb = take(tile >> (k + 1));
	p.smem_f2 = off;
	p.tile = tile;
}

// single-channel mode: K x Downsample2CIC5 -> [FDC] -> FilterCIC5 into Cbuf row `stream` (fe_x.cu)
int launch_frontend_single(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	FeParams &p = h->fe;
	p.in = dev_in;
	p.tail = h->d_tail[h->tail_cur];
	p.in_stride = stride;
	p.format = h->in_fmt;
	p.k = h->k;
	p.N = N;
	p.P = h->P;
	p.use_fdc = h->use_fdc;
	p.fdc_alpha = h->fdc_alpha;
	p.fdc_beta = h->fdc_beta;
	p.rot = nullptr;
	p.C = h->d_C2[h->chunk % aisgpu_handle::NC];
	p.c_stride = h->c_stride;
	p.c_off = HC;
	p.st_B = h->cfg.n_streams;
	CU(launch_frontend_x(p, fe_fmt_id(h->in_fmt), h->k, h->st_L, h->fe_stream));
	return 0;
}

// FM-discriminator input: ConvertRAW, I into Cbuf row 2 * stream and Q into row 2 * stream + 1 as real samples (fe_disc.cu)
int launch_frontend_split(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	FeParams &p = h->fe;
	p.in = dev_in;
	p.in_stride = stride;
	p.format = h->in_fmt;
	p.N = N;
	p.C = h->d_C2[h->chunk % aisgpu_handle::NC];
	p.c_stride = h->c_stride;
	p.c_off = HC;
	p.st_B = h->cfg.n_streams;
	CU(launch_frontend_disc(p, fe_fmt_id(h->in_fmt), h->fe_stream));
	return 0;
}

// The CIC stages of the AB front end over p.N samples per stream of public format fmt (bps bytes per sample): k x Downsample2CIC5, then
// [FilterComplex3Tap ->] Rotate -> per channel Downsample2CIC5 + FilterCIC5 into Cbuf; pre: only the level-k samples, into D0 in
// front of the resampler.  The per-thread streaming kernel (768 kS/s and above) takes the block when the rows are 16-byte aligned:
// its launcher splits every stream over as many lanes as make one balanced wave (st_plan, fe_stream.cuh) and declines a k it has
// no shape for and blocks shorter than four warm-ups.  The tiled kernel takes the rest.
int launch_cic(aisgpu_handle *h, FeParams &p, int fmt, int bps, int k, bool pre) {
	const int B = h->cfg.n_streams;
	// F32_FS4: the kernels take a sample's place in the x, jx, -x, -jx pattern from its index in the block and in the history behind it
	if (fmt == AISGPU_FMT_F32_FS4 && (p.N % 4 || p.P % 4)) {
		h->err = "internal: an F32_FS4 block or its history is not a multiple of 4 samples";
		return AISGPU_ECUDA;
	}
	if (((p.in_stride * bps) % 16) == 0 && (((size_t)p.in) % 16) == 0) {
		p.st_B = B;
		// CF32's four-warp CTAs (fe_stream_f0.cu) are planned as ONE balanced wave of one CTA per SM, chosen over power-of-two lane
		// splits on live step times at 1024 x 131072 on the previous target (not re-measured on the H100): the rest of the SM is left
		// to the back-end CTAs that run beside the front end of the next submit.  The integer formats' one-warp CTAs: as many as fit.
		p.st_cap = fmt == 0 ? 1 : 0;
		const cudaError_t e = h->fp_ds ? launch_frontend_stream_fpds(p, h->st_L, h->fe_stream) : launch_frontend_stream(p, fe_fmt_id(fmt), k, pre, h->st_L, h->fe_stream);
		if (e == cudaSuccess) return 0;
		if (e != cudaErrorNotSupported) CU(e);
	}
	if (h->fp_ds) { // the integer CIC stages only exist in the streaming kernel; check_placement and the granule make it take every valid block
		h->err = "internal: the FP_DS streaming front end declined the block";
		return AISGPU_ECUDA;
	}
	const int q = 1 << (k + 2); // a tile is a whole number of super-steps
	int tile = (FE_TILE + q - 1) / q * q;
	if (tile > p.N) tile = p.N;
	if (tile != p.tile) layout_frontend(p, k, tile);
	const int tiles_total = (p.N + tile - 1) / tile;
	const int n_seg = std::max(1, std::min((FE_CTAS + B - 1) / B, tiles_total));
	p.seg_len = (tiles_total + n_seg - 1) / n_seg * tile;
	const dim3 grid((p.N + p.seg_len - 1) / p.seg_len, B);
	CU(launch_frontend_tiled(p, fe_fmt_id(fmt), k, pre, grid, (size_t)p.smem_f2 * sizeof(float2), h->fe_stream));
	return 0;
}

int launch_frontend(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	if (h->xmode) return launch_frontend_single(h, dev_in, stride, N);
	if (h->disc) return launch_frontend_split(h, dev_in, stride, N);
	FeParams &p = h->fe;
	p.in = dev_in;
	p.tail = h->d_tail[h->tail_cur];
	p.in_stride = stride;
	p.format = h->in_fmt;
	p.k = h->k;
	p.N = N;
	p.P = h->P;
	p.use_fdc = h->use_fdc;
	p.fdc_alpha = h->fdc_alpha;
	p.fdc_beta = h->fdc_beta;
	p.rot = h->d_rot[h->rot_cur];
	p.C = h->d_C2[h->chunk % aisgpu_handle::NC];
	p.c_stride = h->c_stride;
	p.c_off = HC;
	p.st_first = h->chunk == 0 ? 1 : 0;
	return launch_cic(h, p, h->in_fmt, h->bps, h->k, false);
}

// stage s of this submit may start when stage s of the previous submit (other stream) has finished
int stage_begin(aisgpu_handle *h, Stage s) {
	const int prev = h->pb ^ 1;
	if (h->be_streams[1] != h->be_streams[0] && h->stage_rec[s][prev]) CU(cudaStreamWaitEvent(h->bs, h->ev_stage[s][prev], 0));
	return 0;
}
int stage_end(aisgpu_handle *h, Stage s) {
	if (h->be_streams[1] != h->be_streams[0]) {
		CU(cudaEventRecord(h->ev_stage[s][h->pb], h->bs));
		h->stage_rec[s][h->pb] = true;
	}
	return 0;
}

int carry(aisgpu_handle *h, float2 *buf, long long stride, int src_begin, int dst_begin, int cnt) {
	if (cnt <= 0 || src_begin == dst_begin) return 0;
	CU(launch_carry_f2(buf, stride, src_begin, dst_begin, cnt, h->rows, h->bs));
	h->last_launches++;
	return 0;
}

int carry2(aisgpu_handle *h, const float2 *src, float2 *dst, long long stride, int src_begin, int dst_begin, int cnt) {
	if (cnt <= 0) return 0;
	CU(launch_carry2_f2(src, dst, stride, src_begin, dst_begin, cnt, h->rows, h->bs));
	h->last_launches++;
	return 0;
}

// ModelStandard's tail, Filter 37 -> Deinterleave(5) -> 5 cross-reset decoders (Model.cpp:484-518), which ModelDiscriminator
// repeats behind its real rows (Model.cpp:732-751); ModelBase has SimplePLL -> 1 decoder instead
bool standard_tail(const aisgpu_handle *h) { return h->cfg.model == AISGPU_MODEL_STANDARD || h->cfg.model == AISGPU_MODEL_DISCRIMINATOR; }

// The back end of this submit has read Cbuf[chunk % NC] for the last time: the front end of submit chunk + NC may overwrite it.
int be_done(aisgpu_handle *h) {
	const int cb = (int)(h->chunk % aisgpu_handle::NC);
	CU(cudaEventRecord(h->ev_be_done[cb], h->bs));
	h->be_recorded[cb] = true;
	return 0;
}

// Enqueue the Rotate phasor table of chunk c (n96 samples at 96 kHz) on the side stream.
int enqueue_rot_table(aisgpu_handle *h, long long c, int n96) {
	const int slot = (int)(c % 3), prev = (int)((c + 2) % 3);
	// slot was last read by the front end of chunk c-3
	if (h->k1_recorded[slot]) CU(cudaStreamWaitEvent(h->side_stream, h->ev_k1[slot], 0));
	const float2 *prev_tail = c > 0 ? h->d_rot[prev] + h->rot_n96[prev] : nullptr;
	const float2 *state_in = c > 0 ? h->d_rot_state + 1 + prev : h->d_rot_state;
	CU(launch_rot_table(h->d_rot[slot], prev_tail, state_in, h->d_rot_state + 1 + slot, h->mult, h->P96, n96, h->side_stream));
	CU(cudaEventRecord(h->ev_rot[slot], h->side_stream));
	h->rot_n96[slot] = n96;
	h->rot_ready_chunk = c;
	return 0;
}

int fan_out(aisgpu_handle *h, int cb, int n48);
int dump_export(aisgpu_handle *h, int cb, int n48);
int backend_begin(aisgpu_handle *h, cudaEvent_t ready, int N, int n48);
int backend_step(aisgpu_handle *h, float2 *Ccur, float2 *Cnext, int n48);

// One Receive() of the front end proper: N samples per stream (a whole reference block) -> frames, for the engine and the members
// of its group.
int submit_common(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	const int q = (h->xmode || h->disc) ? X_GRANULE : 1 << (h->k + 2);
	if (N <= 0 || N > h->inner_max || (N % q) != 0) {
		char b[160];
		snprintf(b, sizeof(b), "internal: block of %d samples must be a positive multiple of %d and <= %d", N, q, h->inner_max);
		h->err = b;
		return AISGPU_ECUDA; // cannot come from the caller's arguments (check_outer has passed): poisons the handle
	}
	const int k = h->k, B = h->cfg.n_streams;
	const int n96 = N >> k, n48 = (h->xmode || h->disc) ? n96 : n96 >> 1; // X: the k CIC stages end at 48 kHz; -m 3: no CIC stage
	// ---- K0: Rotate phasor table (side stream; normally already enqueued by the previous submit); single-channel mode and the
	// FM-discriminator input have none ----
	if (!h->xmode && !h->disc) {
		const long long c = h->chunk;
		const int slot = (int)(c % 3);
		if (!(h->rot_ready_chunk == c && h->rot_n96[slot] == n96)) {
			if (int rc = enqueue_rot_table(h, c, n96)) return rc;
		}
		CU(cudaStreamWaitEvent(h->fe_stream, h->ev_rot[slot], 0));
		h->rot_cur = slot;
	}
	const int cb = (int)(h->chunk % aisgpu_handle::NC);
	float2 *Ccur = h->d_C2[cb], *Cnext = h->d_C2[(cb + 1) % aisgpu_handle::NC];
	h->c_last = cb;
	// ---- K1: fused front end (its own stream: overlaps the back end of the previous submit) ----
	if (h->be_recorded[cb]) CU(cudaStreamWaitEvent(h->fe_stream, h->ev_be_done[cb], 0)); // back end of submit c-3 still reads Cbuf[cb]
	const int evi = (int)(h->chunk % aisgpu_handle::NEV);
	CU(cudaEventRecord(h->ev_fe0s[evi], h->fe_stream));
	if (int rc = launch_frontend(h, dev_in, stride, N)) return rc;
	CU(cudaEventRecord(h->ev_fe1s[evi], h->fe_stream));
	CU(cudaEventRecord(h->ev_k1[h->chunk % 3], h->fe_stream));
	h->k1_recorded[h->chunk % 3] = true;
	h->fe_timed = true;
	if (h->xmode || h->disc) h->last_launches++;
	else {
		h->last_launches += 2; // front end + this submit's phasor table
		// speculate that the next submit has the same length: build its phasor table now, off the critical path
		if (int rc = enqueue_rot_table(h, h->chunk + 1, n96)) return rc;
	}
	// ---- front-end history for the next submit (none for the FM-discriminator input's split) ----
	if (h->P) {
		const int nxt = h->tail_cur ^ 1;
		CU(launch_tail_update(h->d_tail[nxt], h->d_tail[h->tail_cur], dev_in, stride * h->bps, (long long)N * h->bps, h->P * h->bps, B, h->fe_stream));
		h->tail_cur = nxt;
		h->last_launches++;
	}
	CU(cudaEventRecord(h->ev_fe_done[cb], h->fe_stream));
	if (!h->members.empty())
		if (int rc = fan_out(h, cb, n48)) return rc;
	if (h->dump_slot >= 0)
		if (int rc = dump_export(h, cb, n48)) return rc;
	if (int rc = backend_begin(h, h->ev_fe_done[cb], N, n48)) return rc;
	if (int rc = backend_step(h, Ccur, Cnext, n48)) return rc;
	for (aisgpu_handle *m : h->members) {
		int rc = backend_begin(m, h->ev_fan, N, n48);
		if (!rc) rc = backend_step(m, m->d_C2[cb], m->d_C2[(cb + 1) % aisgpu_handle::NC], n48);
		if (rc) {
			h->err = m->err;
			return rc;
		}
	}
	return 0;
}

// Engine groups: the leader's new rows [HC, HC + n48) of Cbuf[cb] into every member's Cbuf[cb], on the leader's fe_stream behind its
// front end.  A member's Cbuf[cb] was last read by its back end of submit c-3.
int fan_out(aisgpu_handle *h, int cb, int n48) {
	float2 *dst[GROUP_MAX - 1];
	int nd = 0;
	for (aisgpu_handle *m : h->members) {
		if (m->be_recorded[cb]) CU(cudaStreamWaitEvent(h->fe_stream, m->ev_be_done[cb], 0));
		dst[nd++] = m->d_C2[cb];
	}
	CU(launch_c_fanout(h->d_C2[cb], h->c_stride, HC, dst, nd, h->c_stride, HC, n48, h->rows, h->fe_stream));
	CU(cudaEventRecord(h->ev_fan, h->fe_stream));
	h->last_launches++;
	return 0;
}

// ---- the channel dump (aisgpu_dump_open) ----

// Before the first pass of a submit that yields n 48 kHz samples per row: pick its slot.  The host has already written the slot's
// previous contents (dump_reclaim); the front-end stream still waits for the copy out of it, which has finished by then.
int dump_begin(aisgpu_handle *h, long long n) {
	h->dump_slot = -1;
	if (!h->dump || n == 0) return 0;
	const int s = (int)(h->dump_next % aisgpu_handle::ND);
	if (n > h->dump_cap || h->dump_pending.size() >= (size_t)aisgpu_handle::ND) {
		h->err = "internal: channel dump slot overrun";
		return AISGPU_ECUDA;
	}
	if (h->dump_next >= aisgpu_handle::ND) CU(cudaStreamWaitEvent(h->fe_stream, h->ev_dump[s], 0));
	h->dump_slot = s;
	h->dump_n = n;
	h->dump_off = 0;
	return 0;
}

// One inner submit: its rows [HC, HC + n48) of Cbuf[cb] into columns [dump_off, dump_off + n48) of the slot, on fe_stream behind
// ev_fe_done[cb] (no back end waits for it) and behind a leader's fan-out (no member waits for it either).
int dump_export(aisgpu_handle *h, int cb, int n48) {
	if (h->dump_off + n48 > h->dump_n) {
		h->err = "internal: channel dump export overrun";
		return AISGPU_ECUDA;
	}
	float2 *dst = h->d_dump[h->dump_slot];
	CU(launch_c_fanout(h->d_C2[cb], h->c_stride, HC, &dst, 1, h->dump_n, (int)h->dump_off, n48, h->rows, h->fe_stream));
	h->dump_off += n48;
	h->last_launches++;
	return 0;
}

// After the last pass: one copy of the whole slot into its pinned twin on dump_stream.
int dump_end(aisgpu_handle *h, long long ticket) {
	const int s = h->dump_slot;
	if (s < 0) return 0;
	h->dump_slot = -1;
	if (h->dump_off != h->dump_n) {
		h->err = "internal: channel dump rows missing";
		return AISGPU_ECUDA;
	}
	CU(cudaEventRecord(h->ev_export, h->fe_stream));
	CU(cudaStreamWaitEvent(h->dump_stream, h->ev_export, 0));
	CU(cudaMemcpyAsync(h->pin_dump[s], h->d_dump[s], (size_t)h->rows * h->dump_n * sizeof(float2), cudaMemcpyDeviceToHost, h->dump_stream));
	CU(cudaEventRecord(h->ev_dump[s], h->dump_stream));
	h->dump_pending.push_back({ ticket, h->dump_n, s });
	h->dump_next++;
	return 0;
}

// Writes the pending slots of the submits up to `ticket` (all of them for ticket < 0) to the files, in submit order, on the caller's
// thread.  After a file error the rows are dropped (the dump has stopped); the error surfaces at the next submit.
int dump_write(aisgpu_handle *h, long long ticket) {
	while (!h->dump_pending.empty() && (ticket < 0 || h->dump_pending.front().ticket <= ticket)) {
		const aisgpu_handle::DumpPending p = h->dump_pending.front();
		CU(cudaEventSynchronize(h->ev_dump[p.slot]));
		h->dump_pending.pop_front();
		if (h->dump && !h->dump->failed()) h->dump->write(reinterpret_cast<const float *>(h->pin_dump[p.slot]), p.n);
	}
	return 0;
}

// At the entry of every submit, before anything is enqueued: a stopped dump refuses the submit (the reference's StopRequest());
// otherwise the slot this submit may fill is written out first if it still holds an earlier submit's rows.
int dump_reclaim(aisgpu_handle *h) {
	if (!h->dump) return 0;
	if (h->dump_pending.size() >= (size_t)aisgpu_handle::ND)
		if (int rc = dump_write(h, h->dump_pending.front().ticket)) return rc;
	if (h->dump->failed()) {
		h->err = h->dump->error();
		return AISGPU_EIO;
	}
	return 0;
}

// The back end of one inner submit starts when its 48 kHz rows are ready: the engine's own front end, or its leader's fan-out.
int backend_begin(aisgpu_handle *h, cudaEvent_t ready, int N, int n48) {
	h->c_last = (int)(h->chunk % aisgpu_handle::NC);
	h->pb = (int)(h->chunk & 1);
	h->bs = h->be_streams[h->pb];
	CU(cudaStreamWaitEvent(h->bs, ready, 0));
	h->last_n = N;
	h->last_n48 = n48;
	h->last_nE = 0;
	h->last_nsym = 0;
	return 0;
}

// The FM chain's state: the FIR37 history carried in front of HC, Ef, the slicer's decision bits, ModelBase's SimplePLL and taps.
// nEmax: most samples per row entering the chain.
int alloc_fm(aisgpu_handle *h, int nEmax) {
	h->c_hist = FIRF_T;
	if (int rc = dalloc(h, &h->d_Ef, (size_t)h->rows * h->e_stride)) return rc;
	h->dwords = (nEmax / 5 + 2 + K3_TS - 1) / K3_TS + 1;
	for (int i = 0; i < 2; i++)
		if (int rc = dalloc(h, &h->d_dbits2[i], (size_t)h->rows * 5 * h->dwords)) return rc;
	if (!standard_tail(h)) {
		if (int rc = dalloc(h, &h->d_pll, (size_t)h->rows)) return rc;
		std::vector<PllState> pl(h->rows);
		for (auto &x : pl) { x.prev = 0; x.pll = 0.0f; x.fast = 1; }
		CU(cudaMemcpyAsync(h->d_pll, pl.data(), pl.size() * sizeof(PllState), cudaMemcpyHostToDevice, h->stream));
		CU(cudaStreamSynchronize(h->stream));
	}
	if (h->cfg.enable_taps) {
		if (!h->disc)
			if (int rc = dalloc(h, &h->d_tap_fm, (size_t)h->rows * h->r_stride)) return rc;
		if (int rc = dalloc(h, &h->d_tap_cnt, (size_t)h->rows)) return rc;
	}
	return 0;
}

// FM chain: ModelStandard and ModelDiscriminator (FM, or the real rows, -> Filter 37 -> 5-phase slicer -> five decoders) and ModelBase
// (FM -> Filter 37 -> SimplePLL -> one decoder).  n48 new samples per row at [HC, HC + n48) of Ccur.
int step_fm(aisgpu_handle *h, float2 *Ccur, float2 *Cnext, int n48) {
	const bool standard = standard_tail(h);
	if (int rc = stage_begin(h, STAGE_CBUF_CARRY)) return rc;
	if (h->disc) { // FIR history of the real rows: the last 36 samples (n48 is even), moved as 18 float2
		if (int rc = carry2(h, Ccur, Cnext, h->c_stride, HC + n48 / 2 - (FIRF_T - 1) / 2, HC - (FIRF_T - 1) / 2, (FIRF_T - 1) / 2)) return rc;
	}
	else if (int rc = carry2(h, Ccur, Cnext, h->c_stride, HC + n48 - FIRF_T, HC - FIRF_T, FIRF_T)) return rc; // FM + FIR history
	if (int rc = stage_end(h, STAGE_CBUF_CARRY)) return rc;
	// the 5-phase deinterleaver's slots are aligned to absolute sample indices (DSP.h:65-73)
	const long long a0 = h->e_abs, a1 = a0 + n48;
	const long long g0 = a0 - a0 % 5;
	const int nslots = (int)((a1 - g0 + 4) / 5);
	Fm5Params f;
	memset(&f, 0, sizeof(f));
	f.Cbuf = Ccur;
	f.c_stride = h->c_stride;
	f.c_new = HC;
	f.n = n48;
	f.r0 = standard ? (int)(a0 - g0) : 0;
	f.nslots = nslots;
	// the filtered samples themselves are only read by k_base, the bit-serial cross-check decoder and the taps
	f.Fbuf = (!standard || h->decoder == 1 || h->cfg.enable_taps) ? h->d_Ef : nullptr;
	f.f_stride = h->e_stride;
	f.f_off = HE;
	f.dbits = h->d_dbits2[h->pb];
	f.dwords = h->dwords;
	f.tap_fm = h->cfg.enable_taps ? h->d_tap_fm : nullptr; // not allocated for the FM-discriminator input (no FM stage)
	f.tap_stride = h->r_stride;
	f.tap_dec = (h->cfg.enable_taps && standard) ? h->d_tap_dec : nullptr;
	f.real = h->disc;
	if (int rc = stage_begin(h, STAGE_FM_FIR)) return rc; // Ef (single buffered) is only read by taps / k_base, which do not pipeline
	CU(launch_fm_fir5(f, h->rows, h->bs));
	if (int rc = stage_end(h, STAGE_FM_FIR)) return rc;
	h->last_launches++;
	h->last_nE = n48;
	if (int rc = be_done(h)) return rc;
	if (!standard) {
		CU(launch_base(h->d_Ef, h->e_stride, HE, n48, h->rows, h->d_pll, h->d_dec, h->d_dec_data, frame_out(h), h->cfg.enable_taps ? h->d_tap_dec : nullptr,
					   h->cfg.enable_taps ? h->d_tap_cnt : nullptr, h->bs));
		h->last_launches++;
		return 0;
	}
	// Deinterleave (DSP.h:65-73) forwards every sample at once, so partial groups at both ends are walked with a per-phase validity test
	K3Params p;
	memset(&p, 0, sizeof(p));
	p.rows = h->rows;
	p.nsym = nslots;
	p.e_stride = h->e_stride;
	p.e_begin = HE - (int)(a0 - g0);
	p.abs_begin = g0;
	p.abs_lo = a0;
	p.abs_hi = a1;
	p.Ef = h->d_Ef;
	p.dec = h->d_dec;
	p.dec_data = h->d_dec_data;
	set_frame_out(p, frame_out(h));
	p.tap_dec = nullptr; // the decoder input samples are recorded by the FM/FIR kernel
	p.dbg = h->d_dbg;
	p.dbits = h->d_dbits2[h->pb];
	p.dwords = h->dwords;
	if (int rc = stage_begin(h, STAGE_DECODE)) return rc;
	CU(launch_decode(0, h->decoder, h->dec_rpw, p, h->bs));
	if (int rc = stage_end(h, STAGE_DECODE)) return rc;
	h->last_launches++;
	h->last_nsym = nslots;
	h->e_abs = a1;
	return 0;
}

// The coherent chain's state: CGF tables and rotation, Ec, phase search, decision bits and levels, and ModelChallenger's FM branch.
int alloc_coherent(aisgpu_handle *h, int nEmax) {
	h->c_hist = 0;
	for (int i = 0; i < 2; i++) {
		if (int rc = dalloc(h, &h->d_stepidx2[i], (size_t)h->rows * (nEmax / CGF_N + 1))) return rc;
	}
	if (int rc = dalloc(h, &h->d_cgf_rot, (size_t)h->rows)) return rc;
	for (int i = 0; i < 2; i++)
		if (int rc = dalloc(h, &h->d_Ec2[i], (size_t)h->rows * h->e_stride)) return rc;
	if (int rc = dalloc(h, &h->d_ps, (size_t)h->rows * 5)) return rc;
	h->dwords = (nEmax / 5 + 1 + K3_TS - 1) / K3_TS + 1;
	for (int i = 0; i < 2; i++) {
		if (int rc = dalloc(h, &h->d_dbits2[i], (size_t)h->rows * 5 * h->dwords)) return rc;
		if (int rc = dalloc(h, &h->d_lvl2[i], (size_t)h->rows * h->dwords * K3_TS)) return rc;
	}
	if (!h->cfg.ps_ema)
		if (int rc = dalloc(h, &h->d_ps_mem, (size_t)h->rows * 5 * 16 * 12)) return rc;
	if (h->cfg.model == AISGPU_MODEL_CHALLENGER) { // FM branch on the derotated samples (Model.cpp:637-639)
		h->ed_stride = (HD + nEmax + 8 + 1) & ~1LL;
		if (int rc = dalloc(h, &h->d_Ed, (size_t)h->rows * h->ed_stride)) return rc;
		if (int rc = dalloc(h, &h->d_Ef, (size_t)h->rows * h->e_stride)) return rc;
		for (int i = 0; i < 2; i++)
			if (int rc = dalloc(h, &h->d_dbitsF[i], (size_t)h->rows * 5 * h->dwords)) return rc;
		if (int rc = dalloc(h, &h->d_lvl_prev, (size_t)2 * h->rows)) return rc;
	}
	if (int rc = dalloc(h, &h->d_steptab, CGF_NIDX)) return rc;
	if (int rc = dalloc(h, &h->d_ppmtab, CGF_NIDX)) return rc;
	if (int rc = dalloc(h, &h->d_omega, CGF_N)) return rc;
	std::vector<float2> one(h->rows, make_float2(1.0f, 0.0f));
	CU(cudaMemcpyAsync(h->d_cgf_rot, one.data(), one.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
	std::vector<float2> om(CGF_N), st(CGF_NIDX);
	std::vector<float> pp(CGF_NIDX);
	for (int s = 0; s < CGF_N; s++) om[s] = polar1((float)(-2.0 * PI_F) * (float)s / (float)CGF_N); // FFT.h:81-83
	for (int idx = 0; idx < CGF_NIDX; idx++) { // DSP.cpp:453,457-458,466
		float fz = -1;
		if (idx != CGF_IDX_NONE) {
			int i = idx - CGF_IDX_OFFSET;
			fz = (CGF_N / 2 - (i + 102 / 2.0f));
		}
		float f = fz / 2.0f / CGF_N;
		st[idx] = polar1((float)(f * 2 * PI_F));
		pp[idx] = f * 48000.0f / 162.0f;
	}
	CU(cudaMemcpyAsync(h->d_omega, om.data(), om.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
	CU(cudaMemcpyAsync(h->d_steptab, st.data(), st.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
	CU(cudaMemcpyAsync(h->d_ppmtab, pp.data(), pp.size() * sizeof(float), cudaMemcpyHostToDevice, h->stream));
	CU(cudaStreamSynchronize(h->stream)); // host vectors go out of scope
	if (h->cfg.enable_taps)
		if (int rc = dalloc(h, &h->d_tap_cgf, (size_t)h->rows * h->r_stride)) return rc;
	return 0;
}

// Coherent chain: ModelDefault (CGF -> derotation + FIR17 -> 5 x PhaseSearch[EMA] -> 5 decoders, Model.cpp:520-577), and
// ModelChallenger, which adds an FM branch on the derotated samples and decodes both with ten cross-reset decoders (Model.cpp:601-678).
// Only whole 512-blocks enter the chain.
int step_coherent(aisgpu_handle *h, float2 *Ccur, float2 *Cnext, int n48) {
	const bool challenger = h->cfg.model == AISGPU_MODEL_CHALLENGER;
	const int cnt = h->c_hist; // unconsumed samples in front of HC
	const int total = cnt + n48;
	const int nblk = total / CGF_N;
	const int c_begin = HC - cnt;
	const int newcnt = total - nblk * CGF_N;
	// samples that do not fill a 512-block go to the front of the next submit's buffer; the estimator of the next
	// submit only has to wait for this copy (and this one for the copy of the previous submit)
	if (int rc = stage_begin(h, STAGE_CBUF_CARRY)) return rc;
	if (int rc = carry2(h, Ccur, Cnext, h->c_stride, c_begin + nblk * CGF_N, HC - newcnt, newcnt)) return rc;
	if (int rc = stage_end(h, STAGE_CBUF_CARRY)) return rc;
	h->c_hist = newcnt;
	if (nblk == 0) return be_done(h);
	const int nE = nblk * CGF_N;
	// stepidx / dbits / lvl are double buffered by submit parity == stream, so stream order protects them
	int *stepidx = h->d_stepidx2[h->pb];
	CU(launch_cgf_estimate(Ccur, h->c_stride, c_begin, nblk, h->rows * nblk, h->d_omega, h->cfg.afc_wide, stepidx, h->bs));
	// phasor chain + derotation + FIR17 in one kernel: waits for what carries its state and for the last reader of the Ec buffer it
	// writes (the phase search two blocks of symbols ago); ModelChallenger's Ed (single buffered) is free once the previous
	// submit's FM branch has read it
	if (int rc = stage_begin(h, STAGE_DEROT_FIR)) return rc;
	if (h->ec_read_rec[h->ec_cur]) CU(cudaStreamWaitEvent(h->bs, h->ev_ec_read[h->ec_cur], 0));
	if (challenger)
		if (int rc = stage_begin(h, STAGE_FM_BRANCH)) return rc;
	CU(launch_cgf_fused(Ccur, h->c_stride, c_begin, stepidx, h->d_steptab, h->d_cgf_rot, nblk, h->rows, h->d_fir_hist[h->fir_cur], h->d_fir_hist[h->fir_cur ^ 1],
						h->d_Ec2[h->ec_cur], h->e_stride, HE, challenger ? h->d_Ed + HD : (h->cfg.enable_taps ? h->d_tap_cgf : nullptr),
						challenger ? h->ed_stride : h->r_stride, h->bs));
	if (int rc = stage_end(h, STAGE_DEROT_FIR)) return rc;
	h->fir_cur ^= 1;
	h->last_launches += 2;
	h->last_nE = nE;
	if (int rc = be_done(h)) return rc;
	// ScatterPLL (DSP.h:95-117) only forwards complete groups of 5: e_left older samples sit just before HE, and the incomplete group
	// at the end moves to the front of the OTHER Ec buffer, where the next block of symbols lands
	const int e_total = h->e_left + nE;
	const int nsym = e_total / 5;
	const int e_begin = HE - h->e_left;
	const int nl = e_total - nsym * 5;
	h->last_nsym = nsym;
	K3Params p;
	memset(&p, 0, sizeof(p));
	p.ps_ema = h->cfg.ps_ema;
	p.ps_rot0 = (int)((h->e_abs / 5) & 3); // e_abs counts from 0 at creation: symbols delivered so far
	p.rows = h->rows;
	p.nsym = nsym;
	p.e_stride = h->e_stride;
	p.e_begin = e_begin;
	p.abs_begin = h->e_abs;
	p.abs_lo = h->e_abs;
	p.abs_hi = h->e_abs + (long long)nsym * 5;
	p.Ec = h->d_Ec2[h->ec_cur];
	p.Ef = h->d_Ef;
	p.ps = h->d_ps;
	p.ps_mem = h->d_ps_mem;
	p.dec = h->d_dec;
	p.dec_data = h->d_dec_data;
	set_frame_out(p, frame_out(h));
	p.stepidx = stepidx;
	p.ppmtab = h->d_ppmtab;
	p.blk_abs0 = h->cgf_abs;
	p.nblk = nblk;
	p.tap_dec = h->cfg.enable_taps ? h->d_tap_dec : nullptr;
	p.dbg = h->d_dbg;
	p.dbits = h->d_dbits2[h->pb];
	p.dwords = h->dwords;
	p.lvl = h->d_lvl2[h->pb];
	p.lvl_stride = h->dwords * K3_TS;
	if (int rc = stage_begin(h, STAGE_PHASE_SEARCH)) return rc;
	CU(launch_phase_search(p, h->bs));
	h->last_launches++;
	if (int rc = carry2(h, h->d_Ec2[h->ec_cur], h->d_Ec2[h->ec_cur ^ 1], h->e_stride, e_begin + nsym * 5, HE - nl, nl)) return rc;
	if (int rc = stage_end(h, STAGE_PHASE_SEARCH)) return rc;
	CU(cudaEventRecord(h->ev_ec_read[h->ec_cur], h->bs));
	h->ec_read_rec[h->ec_cur] = true;
	if (challenger) {
		// FM branch on the derotated samples: Demod::FM -> Filter 37 -> Deinterleave (Model.cpp:637-639), all new samples at once
		const long long a0 = h->e_abs + h->e_left, a1 = a0 + nE; // absolute indices of the new samples
		Fm5Params f;
		memset(&f, 0, sizeof(f));
		f.Cbuf = h->d_Ed;
		f.c_stride = h->ed_stride;
		f.c_new = HD;
		f.n = nE;
		f.r0 = h->e_left;
		f.nslots = (int)((a1 - h->e_abs + 4) / 5);
		f.Fbuf = h->cfg.enable_taps ? h->d_Ef : nullptr; // k_decode10 takes the decision bits
		f.f_stride = h->e_stride;
		f.f_off = HE;
		f.dbits = h->d_dbitsF[h->pb];
		f.dwords = h->dwords;
		if (int rc = stage_begin(h, STAGE_FM_BRANCH)) return rc;
		CU(launch_fm_fir5(f, h->rows, h->bs));
		h->last_launches++;
		if (int rc = carry(h, h->d_Ed, h->ed_stride, nE, 0, HD)) return rc; // the last HD derotated samples stay in front
		if (int rc = stage_end(h, STAGE_FM_BRANCH)) return rc;
		p.dbits2 = h->d_dbitsF[h->pb];
		p.nslots_fm = f.nslots;
		p.lvl_prev = h->d_lvl_prev + (size_t)h->lvlp_cur * h->rows;
		p.lvl_prev_out = h->d_lvl_prev + (size_t)(h->lvlp_cur ^ 1) * h->rows;
		p.lvl_own = h->xmode;
		h->lvlp_cur ^= 1;
		p.abs_lo = a0;
		p.abs_hi = a1;
	}
	if (int rc = stage_begin(h, STAGE_DECODE)) return rc;
	CU(challenger ? launch_decode10(h->dec_rpw == 1 ? 1 : 3, p, h->bs) : launch_decode(2, h->decoder, h->dec_rpw, p, h->bs));
	if (int rc = stage_end(h, STAGE_DECODE)) return rc;
	h->last_launches++;
	h->ec_last = h->ec_cur;
	h->ec_cur ^= 1;
	h->e_left = nl;
	h->e_abs += (long long)nsym * 5;
	h->cgf_abs += nE;
	return 0;
}

// The V2 chain's state: one V2State per row, the FFT twiddles and the kernel's constant tables, and its taps.
int alloc_v2(aisgpu_handle *h) {
	h->c_hist = V2_BLK; // Engine::raw starts as a block of zeros that is decoded when the first real block has arrived (V2Engine.cpp:274-277, 379-395)
	if (int rc = dalloc(h, &h->d_v2, (size_t)h->rows)) return rc;
	if (int rc = dalloc(h, &h->d_omega, CGF_N)) return rc;
	{
		std::vector<V2State> init(h->rows);
		memset(init.data(), 0, init.size() * sizeof(V2State));
		for (auto &v : init) {
			v.fo_rot = make_float2(1.0f, 0.0f);
			v.fm_prev = make_float2(1.0f, 0.0f);
		}
		std::vector<float2> om(CGF_N);
		for (int s = 0; s < CGF_N; s++) om[s] = polar1((float)(-2.0 * PI_F) * (float)s / (float)CGF_N);
		CU(cudaMemcpyAsync(h->d_v2, init.data(), init.size() * sizeof(V2State), cudaMemcpyHostToDevice, h->stream));
		CU(cudaMemcpyAsync(h->d_omega, om.data(), om.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
		CU(cudaStreamSynchronize(h->stream));
		CU(v2_init(H_TAPS_COHERENT, H_TAPS_RECEIVER, om.data()));
	}
	if (h->cfg.enable_taps) {
		if (int rc = dalloc(h, &h->d_tap_cgf, (size_t)h->rows * h->r_stride)) return rc;
		if (int rc = dalloc(h, &h->d_tap_coh, (size_t)h->rows * h->r_stride)) return rc;
		if (int rc = dalloc(h, &h->d_tap_fm, (size_t)h->rows * h->r_stride)) return rc;
	}
	return 0;
}

// V2 chain: Engine::Receive (V2Engine.cpp:379-395) in one kernel.  A block is decoded once the NEXT block is complete (it is the
// estimator's lookahead), so one whole block plus the partial one wait in front of the new samples.
int step_v2(aisgpu_handle *h, float2 *Ccur, float2 *Cnext, int n48) {
	const int cnt = h->c_hist;
	const int total = cnt + n48;
	const int nproc = std::max(0, total / V2_BLK - 1);
	const int c_begin = HC - cnt;
	const int newcnt = total - nproc * V2_BLK;
	if (int rc = carry2(h, Ccur, Cnext, h->c_stride, c_begin + nproc * V2_BLK, HC - newcnt, newcnt)) return rc;
	h->c_hist = newcnt;
	if (nproc > 0) {
		const bool taps = h->cfg.enable_taps;
		CU(launch_v2_engine(Ccur, h->c_stride, c_begin, nproc, h->rows, h->d_v2, h->d_dec, h->d_dec_data, frame_out(h), h->d_omega, h->cfg.dd_train,
							h->cfg.dd_weight, taps ? h->d_tap_cgf : nullptr, taps ? h->d_tap_coh : nullptr, taps ? h->d_tap_fm : nullptr, h->r_stride, h->bs));
		h->last_launches++;
	}
	h->last_nE = nproc * V2_BLK;
	return be_done(h);
}

// Everything behind the 48 kHz rows of one inner submit: n48 new samples per row at [HC, HC + n48) of Ccur; what the chain carries
// into the next submit goes in front of HC in Cnext.  Stage-pipelined over consecutive submits, see aisgpu_handle::be_streams.
int backend_step(aisgpu_handle *h, float2 *Ccur, float2 *Cnext, int n48) {
	const int rc = h->chain == Chain::Fm ? step_fm(h, Ccur, Cnext, n48)
				   : h->chain == Chain::Coherent ? step_coherent(h, Ccur, Cnext, n48) : step_v2(h, Ccur, Cnext, n48);
	if (rc) return rc;
	h->chunk++;
	return 0;
}

// History of the stage that reads the caller's input: the CIC stage's warm-up, or DownsampleKFilter's taps
int raw_tail_len(const aisgpu_handle *h) { return has_cic(h) ? h->PA : 32; }

// The CIC stage: kA x Downsample2CIC5 of the caller's N samples into D0 (Model.cpp:183-189, 208-218)
int pre_cic(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	FeParams &pp = h->fe_pre;
	pp.in = dev_in;
	pp.tail = h->d_raw_tail[h->raw_tail_cur];
	pp.in_stride = stride;
	pp.format = src_fmt(h);
	pp.k = h->kA;
	pp.N = N;
	pp.P = h->PA;
	pp.use_fdc = 0;
	pp.rot = nullptr;
	pp.C = nullptr;
	pp.D0 = h->d_D0;
	pp.d0_stride = h->d0_stride;
	pp.d0_off = 2;
	if (int rc = launch_cic(h, pp, src_fmt(h), h->pbps, h->kA, true)) return rc;
	h->last_launches++;
	return 0;
}

// Replays Upsample's float accumulator over L inputs: one (input index, alpha) pair per output (DSP.cpp:196-209).  Returns the
// number of outputs, or -1 when they would not fit the table.
int us_schedule(aisgpu_handle *h, int L, int *us_src, float *us_al) {
	float alpha = h->us_alpha;
	const float inc = h->us_inc;
	int M = 0;
	for (int i = 0; i < L; i++) {
		do {
			if (M >= h->us_cap) return -1;
			us_src[M] = i;
			us_al[M++] = alpha;
			alpha += inc;
		} while (alpha < 1.0f);
		alpha -= 1.0f;
	}
	h->us_alpha = alpha;
	return M;
}

// Upsample (DSP.cpp:192-212): the N >> kA samples of D0 -> us_ring.  The schedule goes through a pinned double buffer, so the copy
// is a true asynchronous one and the caller's thread never waits for the front-end stream here.
int pre_upsample(aisgpu_handle *h, int N) {
	PreRing &r = h->us_ring;
	const int L = N >> h->kA;
	if (!h->outer_N) {
		h->outer_N = N;
		h->us_blk = L;
		if (!h->pre_dsk) h->blk = L;
		r.cap = (h->us_ratio + 2) * L; // whole blocks: < L left over + up to us_ratio * L (+ a few) new samples
	}
	const int ub = h->us_cur;
	if (h->us_used[ub]) CU(cudaEventSynchronize(h->ev_us[ub])); // the copy issued two submits ago has read this buffer
	const int M = us_schedule(h, L, h->pin_us_src[ub], h->pin_us_alpha[ub]);
	if (M < 0) {
		h->err = "Upsample schedule overflow";
		return AISGPU_ECUDA;
	}
	CU(cudaMemcpyAsync(h->d_us_src, h->pin_us_src[ub], (size_t)M * sizeof(int), cudaMemcpyHostToDevice, h->fe_stream));
	CU(cudaMemcpyAsync(h->d_us_alpha, h->pin_us_alpha[ub], (size_t)M * sizeof(float), cudaMemcpyHostToDevice, h->fe_stream));
	CU(cudaEventRecord(h->ev_us[ub], h->fe_stream));
	h->us_used[ub] = true;
	h->us_cur ^= 1;
	const int B = h->cfg.n_streams;
	CU(launch_upsample(h->d_D0, h->d0_stride, 2, h->d_us_src, h->d_us_alpha, M, B, r.d, r.stride, r.produced, r.cap, h->fe_stream));
	CU(launch_d0_carry(h->d_D0, h->d0_stride, 2, L, B, h->fe_stream));
	r.produced += M;
	h->last_launches += 2;
	return 0;
}

// DownsampleKFilter(BlackmanHarris_28_3, 3) (Model.cpp:308-313; DSP.cpp:160-189): N samples per stream of src -> dsk_ring.  Behind
// the CIC stage src is CF32 (D0 or an Upsample block) with a CF32 history of its own; otherwise it is the caller's input in the
// caller's format, and the raw-format history serves.
int pre_dsk(aisgpu_handle *h, const void *src, long long stride, int N) {
	// DownsampleKFilter::Receive returns at once on a block shorter than its taps minus one (DSP.cpp:165-166): the block is dropped
	// and the filter's history, phase and output block stay as they were
	if (N < DSK_T - 1) return 0;
	PreRing &r = h->dsk_ring;
	const bool cf32 = has_cic(h);
	const int B = h->cfg.n_streams, c = h->cf_tail_cur;
	const void *tail = cf32 ? (const void *)h->d_cf_tail[c] : (const void *)h->d_raw_tail[h->raw_tail_cur];
	const int first = h->dsk_first;
	const int n_out = first < N ? (N - first + 2) / 3 : 0;
	if (n_out > 0) {
		CU(launch_dsk(fe_fmt_id(cf32 ? AISGPU_FMT_CF32 : src_fmt(h)), src, stride, tail, 32, first, n_out, B, r.d, r.stride, r.produced, r.cap, h->fe_stream));
		h->last_launches++;
	}
	h->dsk_first = first + 3 * n_out - N;
	r.produced += n_out;
	if (cf32) {
		CU(launch_tail_update(h->d_cf_tail[c ^ 1], h->d_cf_tail[c], src, stride * 8, (long long)N * 8, 32 * 8, B, h->fe_stream));
		h->cf_tail_cur = c ^ 1;
		h->last_launches++;
	}
	return 0;
}

int sync_backend(aisgpu_handle *h) {
	CU(cudaStreamSynchronize(h->be_streams[0]));
	if (h->be_streams[1] != h->be_streams[0]) CU(cudaStreamSynchronize(h->be_streams[1]));
	return 0;
}

int check_outer(aisgpu_handle *h, int N) {
	const int q = outer_granule(h);
	if (N <= 0 || N > h->cfg.max_chunk_samples || (N % q) != 0) {
		char b[160];
		snprintf(b, sizeof(b), "n_samples=%d must be a positive multiple of %d and <= max_chunk_samples=%d", N, q, h->cfg.max_chunk_samples);
		h->err = b;
		return AISGPU_EINVAL;
	}
	if (h->pre_us && h->outer_N && N != h->outer_N) {
		h->err = "at an interpolated sample rate every submit must have the same length (DSP::Upsample re-blocks by it, DSP.cpp:203)";
		return AISGPU_EINVAL;
	}
	return 0;
}

// Where a device batch (aisgpu_submit_device) may lie, from what the readers of the planned chain load:
//  - the tiled front end and pre-stage (fe_tiled.cu) load pairs of samples at even indices with one vector load of two samples
//    (fe_common.cuh) and copy CF32 tiles with cp.async.bulk, which needs 16-byte sources: base aligned to two samples, even stride;
//  - the streaming kernels (fe_stream.cuh) are only chosen for 16-byte rows; the integer front end of FP_DS and single-channel
//    mode (fe_x.cu) exist only as such kernels: base and rows 16-byte aligned, and FP_DS's lane offsets fit 32 bits of 16-byte units;
//  - the FM-discriminator split at 48 kHz (fe_disc.cu) loads single samples where pairs are not aligned: any sample-aligned base;
//  - DownsampleKFilter (k_dsk) and the warm-up tail copy (k_tail_update) read single samples;
//  - F32_FS4: base 16-byte aligned and a stride of whole x, jx, -x, -jx patterns (four samples = 16 bytes), at every rate and in
//    every mode: each row is then a 16-byte aligned run of whole patterns, which is what every reader above asks for;
//  - DC16H: the same rule for another reason -- at 12 bytes per sample four samples are 48 bytes, so a 16-byte aligned base and a
//    stride that is a multiple of 4 samples put every row on a 16-byte boundary, which the streaming kernels' 16-byte copies need
//    (the other readers load single 32-bit words).
int check_placement(aisgpu_handle *h, const void *dev, int64_t stride) {
	const unsigned long long a = (unsigned long long)(size_t)dev;
	const int bps = bytes_per_sample(h->cfg.format);
	if (h->cfg.format == AISGPU_FMT_F32_FS4 && (stride < 0 || stride % 4 || a % 16)) {
		h->err = "F32_FS4: the base of a device batch must be 16-byte aligned and stride_samples a non-negative multiple of 4";
		return AISGPU_EINVAL;
	}
	if (h->cfg.format == AISGPU_FMT_DC16H) { // the whole rule of the format: "two samples" below would be 24 bytes
		if (stride < 0 || stride % 4 || a % 16) {
			h->err = "DC16H: the base of a device batch must be 16-byte aligned and stride_samples a non-negative multiple of 4";
			return AISGPU_EINVAL;
		}
		return 0;
	}
	if (stride < 0 || (stride & 1)) {
		h->err = "stride_samples must be even and non-negative";
		return AISGPU_EINVAL;
	}
	if (h->xmode || h->fp_ds) {
		if (a % 16 || (stride * bps) % 16) {
			h->err = h->xmode ? "single-channel mode: the rows of a device batch must be 16-byte aligned"
							  : "FP_DS on: the rows of a device batch must be 16-byte aligned";
			return AISGPU_EINVAL;
		}
		if (h->fp_ds && (unsigned long long)h->cfg.n_streams * (unsigned long long)stride * (unsigned long long)bps >= (1ull << 36)) {
			h->err = "FP_DS on: a device batch must span less than 64 GiB";
			return AISGPU_EINVAL;
		}
		return 0;
	}
	const int align = (h->disc && !h->pre_us) ? bps : 2 * bps;
	if (a % align) {
		char b[160];
		snprintf(b, sizeof(b), "the base of a device batch must be aligned to %d bytes (%s)", align,
				 align == bps ? "one sample" : "two samples");
		h->err = b;
		return AISGPU_EINVAL;
	}
	return 0;
}

int mark_ticket(aisgpu_handle *h, long long t);

// The tune stage (aisgpu_set_tunings): the caller's N samples per input row, sample 0 being sample counters[2] of every stream,
// converted and mixed into the rows of the row's streams in d_tune (or in D0, tune_into_d0); what follows reads d_tune in place of the
// caller's rows.
int tune_input(aisgpu_handle *h, const void *&dev_in, long long &stride, int N) {
	TuneParams p;
	p.in = dev_in;
	p.in_stride = stride;
	p.out = h->d_tune ? h->d_tune : h->d_D0;
	p.out_stride = h->d_tune ? h->tune_stride : h->d0_stride;
	p.out_off = h->d_tune ? 0 : 2;
	p.N = N;
	p.R = inputs(h);
	p.T = h->per_input;
	p.fs = h->cfg.sample_rate;
	p.tab_len = tune_table_len(p.fs);
	p.first = (long long)h->counters[2];
	p.fk = h->d_tune_fk;
	p.tab = h->d_tune_tab;
	CU(launch_tune(p, fe_fmt_id(h->cfg.format), h->tune_ctas, h->fe_stream));
	h->last_launches++;
	dev_in = h->d_tune;
	stride = h->tune_stride;
	return 0;
}

// The caller's Receive(): N samples per stream in the caller's format.
int submit_outer(aisgpu_handle *h, const void *dev_in, long long stride, int N) {
	if (int rc = check_outer(h, N)) return rc;
	// Message::Stamp's reading of the system clock, once for every frame this submit completes
	const long long wall_us = h->clock && h->clock->live ? (long long)std::chrono::duration_cast<std::chrono::microseconds>(
															   std::chrono::system_clock::now().time_since_epoch()).count()
														 : 0;
	h->last_launches = 0;
	if (h->tuned)
		if (int rc = tune_input(h, dev_in, stride, N)) return rc;
	h->msg_chunk = (long long)h->counters[3];
	for (aisgpu_handle *m : h->members) {
		m->last_launches = 0;
		m->msg_chunk = h->msg_chunk;
	}
	if (!h->pre_us && !h->pre_dsk) {
		if (int rc = dump_begin(h, N >> (h->k + 1))) return rc; // a dump is AB only: two 48 kHz rows per stream
		if (int rc = submit_common(h, dev_in, stride, N)) return rc;
	}
	else {
		h->us_ring.last = h->us_ring.produced;
		h->dsk_ring.last = h->dsk_ring.produced;
		if (has_cic(h) && !tune_into_d0(h))
			if (int rc = pre_cic(h, dev_in, stride, N)) return rc;
		if (h->pre_us) {
			if (int rc = pre_upsample(h, N)) return rc;
		}
		else if (int rc = has_cic(h) ? pre_dsk(h, h->d_D0 + 2, h->d0_stride, N >> h->kA) : pre_dsk(h, dev_in, stride, N)) return rc;
		if (!tune_into_d0(h)) { // raw-format history of the pre-stage for the next submit
			const int cur = h->raw_tail_cur, tl = raw_tail_len(h);
			CU(launch_tail_update(h->d_raw_tail[cur ^ 1], h->d_raw_tail[cur], dev_in, stride * h->pbps, (long long)N * h->pbps, tl * h->pbps, h->cfg.n_streams, h->fe_stream));
			h->raw_tail_cur = cur ^ 1;
			h->last_launches++;
		}
		if (h->pre_us && h->pre_dsk) // every whole Upsample block goes through DownsampleKFilter
			for (PreRing &u = h->us_ring; u.produced - u.consumed >= h->us_blk; u.consumed += h->us_blk)
				if (int rc = pre_dsk(h, u.d + u.consumed % u.cap, u.stride, h->us_blk)) return rc;
		// hand every whole reference block of the last ring to the front end proper
		PreRing &r = h->pre_dsk ? h->dsk_ring : h->us_ring;
		if (int rc = dump_begin(h, (r.produced - r.consumed) / h->blk * (h->blk >> (h->k + 1)))) return rc;
		for (; r.produced - r.consumed >= h->blk; r.consumed += h->blk)
			if (int rc = submit_common(h, r.d + r.consumed % r.cap, r.stride, h->blk)) return rc;
	}
	if (int rc = dump_end(h, (long long)h->counters[3])) return rc;
	if (int rc2 = mark_ticket(h, (long long)h->counters[3])) return rc2;
	for (aisgpu_handle *m : h->members) {
		if (int rc2 = mark_ticket(m, (long long)h->counters[3])) {
			h->err = m->err;
			return rc2;
		}
		m->counters[2] += (uint64_t)N;
		m->counters[3] += 1;
	}
	h->counters[2] += (uint64_t)N;
	h->counters[3] += 1;
	if (h->clock) h->clock->at.push_back(h->clock->live ? wall_us : (long long)h->counters[2]);
	return 0;
}

// The payload of a frame as NMEA six-bit letters, one pass over the bit stream (what Message::getLetter does letter by
// letter, Message.cpp:643-662): letter i = bits [6i, 6i + 6), MSB first; bits past the message end read as 0; a letter that
// would cross bit 1064 is the NUL byte the reference returns there; value v prints as v + 48 (v < 40) or v + 56.
int armour_payload(const uint8_t *data, int nbits, char *out) {
	const int n = (nbits + 5) / 6;
	uint32_t window = 0; // the next `have` unread bits, right-aligned
	int have = 0, next_byte = 0;
	for (int i = 0; i < n; i++) {
		if (have < 6) {
			window = (window << 8) | data[next_byte++];
			have += 8;
		}
		have -= 6;
		unsigned v = (window >> have) & 0x3Fu;
		const int past = 6 * (i + 1) - nbits; // bits of this letter beyond the end of the message
		if (past > 0) v &= 0x3Fu << past;
		out[i] = 6 * (i + 1) > 1064 ? (char)0 : (char)(v + (v < 40 ? 48 : 56));
	}
	return n;
}

bool msg_validate(const uint8_t *d, int length) { // Message.cpp:398-413
	static const int ml[28] = { 149, 149, 149, 168, 418, 88, 72, 56, 168, 70, 168, 72, 40, 40, 88, 92, 80, 168, 312, 70, 271, 145, 154, 160, 72, 60, 96, 168 };
	if (length == 0) return true;
	if (length > 1064) return false;
	unsigned t = d[0] >> 2;
	if (t < 1 || t > 28) return false;
	return length >= ml[t - 1];
}

// Message::buildNMEA (Message.cpp:569-631): "!AIVDM,<sentences>,<index>,<seq>,<channel>,<up to 56 letters>,<fill>*<checksum>";
// own-ship frames read !AIVDO; the sequence id (Message::nextSeqId, Message.cpp:28-39; one counter per stream here instead of
// one per process) only exists for multi-sentence messages; fill bits are reported on the last sentence.
void build_nmea(aisgpu_msg &m, int own_mmsi, int *seq_counter) {
	char letters[180];
	const int nletters = armour_payload(m.data, m.nbits, letters);
	const int nsent = nletters ? (nletters + 55) / 56 : 1;
	const uint32_t mmsi = ((uint32_t)m.data[1] << 22) | ((uint32_t)m.data[2] << 14) | ((uint32_t)m.data[3] << 6) | (m.data[4] >> 2);
	char seq = 0;
	if (nsent > 1) {
		seq = (char)('0' + *seq_counter);
		*seq_counter = (*seq_counter + 1) % 10;
	}
	m.n_sentences = nsent;
	for (int s = 0; s < nsent && s < 4; s++) {
		char *line = m.nmea[s];
		int at = 0;
		uint8_t sum = 0; // XOR of everything between '!' and '*'
		auto put = [&](char ch) { line[at++] = ch; sum ^= (uint8_t)ch; };
		line[at++] = '!';
		for (const char *t = (own_mmsi == (int)mmsi) ? "AIVDO," : "AIVDM,"; *t; t++) put(*t);
		put((char)('0' + nsent));
		put(',');
		put((char)('1' + s));
		put(',');
		if (seq) put(seq);
		put(',');
		if (m.channel != '?') put(m.channel);
		put(',');
		const int first = 56 * s, count = std::min(56, nletters - first);
		for (int k = 0; k < count; k++) put(letters[first + k]);
		put(',');
		put((char)('0' + (s == nsent - 1 ? 6 * nletters - m.nbits : 0)));
		line[at++] = '*';
		line[at++] = "0123456789ABCDEF"[sum >> 4];
		line[at++] = "0123456789ABCDEF"[sum & 15];
		line[at] = 0;
		m.nmea_len[s] = at; // a 1064-bit message ends in a NUL letter, so strlen() is not enough
	}
}

const int kJsonBatch = 4096; // frames decoded per launch group

// Drops the oldest unread records beyond ring_cap (a caller that polls only frames does not let json_buf grow without bound).
void json_trim(aisgpu_handle *h) {
	if ((long long)h->rec_len.size() <= h->ring_cap) return;
	while ((long long)h->rec_len.size() > h->ring_cap) {
		h->json_pos += (size_t)h->rec_len.front();
		h->rec_len.pop_front();
	}
	h->json_overflow_pending = true;
}

// The records of out_queue[q0, end) (the frames a drain just published) -> json_buf, on the device (be_json.cu), in batches of
// kJsonBatch frames; a submit split over two batches carries the bytes its records have used into the second, and every batch
// carries the engine's counters into the next.
int json_decode(aisgpu_handle *h, size_t q0) {
	const int n_all = (int)(h->out_queue.size() - q0);
	if (n_all <= 0) return 0;
	h->json_buf.erase(0, h->json_pos); // what has been read
	h->json_pos = 0;
	cudaStream_t st = h->json_stream;
	long long carry = 0;
	for (int b0 = 0; b0 < n_all; b0 += kJsonBatch) {
		const int n = std::min(kJsonBatch, n_all - b0);
		const aisgpu_msg *q = h->out_queue.data() + q0 + b0;
		// submits are contiguous in out_queue: seg[i] = the first frame of frame i's submit within this batch
		h->json_seg.resize((size_t)n);
		for (int i = 0; i < n; i++) h->json_seg[i] = (i > 0 && q[i].chunk == q[i - 1].chunk) ? h->json_seg[i - 1] : i;
		if (b0 == 0 || q[0].chunk != q[-1].chunk) carry = 0;
		CU(cudaMemcpyAsync(h->d_jmsg, q, (size_t)n * sizeof(aisgpu_msg), cudaMemcpyHostToDevice, st));
		CU(cudaMemcpyAsync(h->d_jseg, h->json_seg.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice, st));
		if (h->clock) { // each frame's stamp, from its stream and the submit that completed it
			h->json_stamp.resize((size_t)n);
			for (int i = 0; i < n; i++) h->json_stamp[i] = h->clock->stamp(q[i].stream, q[i].chunk);
			CU(cudaMemcpyAsync(h->d_jstamp, h->json_stamp.data(), (size_t)n * sizeof(long long), cudaMemcpyHostToDevice, st));
		}
		CU(fmt_launch(h->d_jmsg, h->clock ? h->d_jstamp : nullptr, n, h->d_fctx, h->rx_table, h->fmt_records, h->fmt_groups, h->d_jgroups, h->d_jslots, h->json_slot, h->rec_cap,
					  h->d_jlen, h->d_jseg, h->json_cap, carry, h->d_jpsum, h->d_joff, h->d_jkeep, h->d_jtotal, h->d_jtext, st));
		CU(cudaMemcpyAsync(h->pin_jtotal, h->d_jtotal, 4 * sizeof(long long), cudaMemcpyDeviceToHost, st));
		CU(cudaMemcpyAsync(h->pin_jkeep, h->d_jkeep, (size_t)n * sizeof(int), cudaMemcpyDeviceToHost, st));
		CU(cudaStreamSynchronize(st));
		const long long total = h->pin_jtotal[0], kept = h->pin_jtotal[1];
		carry = h->pin_jtotal[2];
		h->fmt_records += n;
		h->fmt_groups += h->pin_jtotal[3];
		if (total > 0) {
			CU(cudaMemcpyAsync(h->pin_jtext, h->d_jtext, (size_t)total, cudaMemcpyDeviceToHost, st));
			CU(cudaStreamSynchronize(st));
			h->json_buf.append(h->pin_jtext, (size_t)total);
		}
		for (int i = 0; i < n; i++)
			if (h->pin_jkeep[i] >= 0) h->rec_len.push_back(h->pin_jkeep[i]);
		if (kept < n) h->json_overflow_pending = true; // records that did not fit their submit's json_cap bytes
	}
	json_trim(h);
	return 0;
}

// Copies the frames with tickets [a, b) to the end of h_ring; tickets at or above `limit` were dropped by the kernels.
int fetch_frames(aisgpu_handle *h, unsigned long long a, unsigned long long b, unsigned long long limit) {
	const unsigned long long hi = std::min(b, std::max(a, limit));
	if (b > hi) {
		h->counters[4] += (uint64_t)(b - hi);
		h->overflow_pending = true;
	}
	const unsigned long long cap = (unsigned long long)h->ring_cap;
	while (a < hi) {
		const size_t off = (size_t)(a % cap);
		const size_t n = (size_t)std::min<unsigned long long>(hi - a, cap - off);
		const size_t at = h->h_ring.size();
		h->h_ring.resize(at + n);
		CU(cudaMemcpy(h->h_ring.data() + at, h->d_ring + off, n * sizeof(FrameRec), cudaMemcpyDeviceToHost));
		a += n;
	}
	return 0;
}

// Records, behind everything enqueued for submit `t`, the ring head (into a pinned slot) and the completion event.
int mark_ticket(aisgpu_handle *h, long long t) {
	cudaStream_t st = h->bs ? h->bs : h->stream;
	CU(cudaEventRecord(h->ev_mark, h->fe_stream)); // a pre-stage submit may have launched nothing behind the front-end stream
	CU(cudaStreamWaitEvent(st, h->ev_mark, 0));
	const int slot = (int)(t % aisgpu_handle::NT);
	// With two back-end streams the snapshots of consecutive submits sit on different streams: chain them, so that the recorded
	// heads are monotonic in t and record t also covers everything submit t-1 wrote (a submit without back-end work would otherwise
	// take its snapshot while the previous submit's decoders are still running)
	if (t > 0 && h->be_streams[1] != h->be_streams[0]) CU(cudaStreamWaitEvent(st, h->ev_ticket[(t - 1) % aisgpu_handle::NT], 0));
	CU(cudaMemcpyAsync(&h->pin_head[slot], h->d_ring_head, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
	CU(cudaEventRecord(h->ev_ticket[slot], st));
	h->launch_limit.push_back(frame_out(h).ring_limit);
	return 0;
}

// Frames of the submits (polled_ticket, upto] -> out_queue.  upto < 0: everything, after a full synchronisation.
int drain_ring(aisgpu_handle *h, long long upto) {
	const long long latest = (long long)h->counters[3] - 1;
	if (latest < 0) return 0;
	if (upto < 0 || upto > latest) {
		CU(cudaStreamSynchronize(h->fe_stream));
		if (int rc = sync_backend(h)) return rc;
		upto = latest;
	}
	if (upto <= h->polled_ticket) return 0;
	if (latest - upto >= aisgpu_handle::NT) upto = latest; // its completion record has been recycled: wait for the newest one
	CU(cudaEventSynchronize(h->ev_ticket[upto % aisgpu_handle::NT]));
	h->h_ring.clear();
	const long long first = h->polled_ticket + 1;
	if (latest - first < aisgpu_handle::NT) { // every submit's own record is still there: exact limits per submit
		for (long long t = first; t <= upto; t++) {
			const unsigned long long head = std::max(h->drained, (unsigned long long)h->pin_head[t % aisgpu_handle::NT]);
			if (int rc = fetch_frames(h, h->drained, head, h->launch_limit.front())) return rc;
			h->drained = head;
			h->launch_limit.pop_front();
		}
	}
	else { // more submits than records since the last poll: they all ran against the oldest one's limit or a later (larger) one
		const unsigned long long head = std::max(h->drained, (unsigned long long)h->pin_head[upto % aisgpu_handle::NT]);
		if (int rc = fetch_frames(h, h->drained, head, h->launch_limit.front())) return rc;
		h->drained = head;
		for (long long t = first; t <= upto; t++) h->launch_limit.pop_front();
	}
	h->polled_ticket = upto;
	if (h->h_ring.empty()) return 0;
	// reference emission order: per submit, stream-major, channel A (ROT.up) before B (DSP.cpp:312-313), then time
	std::stable_sort(h->h_ring.begin(), h->h_ring.end(), [](const FrameRec &a, const FrameRec &b) {
		if (a.chunk != b.chunk) return a.chunk < b.chunk;
		if (a.blk != b.blk) return a.blk < b.blk; // Rotate sends whole blocks: A then B per block (DSP.cpp:312-313)
		return a.row < b.row;
	});
	if (h->json_on && h->out_pos > 0) { // frames and lines are queued side by side: keep only what has not been read
		h->out_queue.erase(h->out_queue.begin(), h->out_queue.begin() + (long)h->out_pos);
		h->out_pos = 0;
	}
	const size_t q0 = h->out_queue.size();
	for (const FrameRec &r : h->h_ring) {
		h->counters[0]++;
		aisgpu_msg m;
		memset(&m, 0, sizeof(m));
		m.stream = stream_of_row(h, r.row);
		const Receiver &rx = h->rx[m.stream]; // the config's fields unless a receiver table was installed
		m.channel = channel_of_row(h, r.row) ? rx.channel_b : rx.channel_a;
		m.nbits = (r.nbits >= 0 && r.nbits <= 1064) ? r.nbits : 0; // Message::setLength (Message.h:288-292)
		m.start_idx = r.start_idx;
		m.end_idx = r.end_idx;
		m.ppm = r.ppm;
		m.chunk = r.chunk;
		float lvl = r.level;
		if ((rx.tag_mode & 1) && lvl != 0.0) lvl = (float)(10.0f * log10((double)lvl)); // AIS.cpp:74-75: the reference resolves to the double log10
		m.level = lvl;
		memcpy(m.data, r.data, 140);
		if (!msg_validate(m.data, m.nbits)) continue; // AIS.cpp:87-93: dropped, siblings were still reset
		build_nmea(m, rx.own_mmsi, &h->seq[m.stream]);
		h->counters[1]++;
		h->counters[channel_of_row(h, r.row) ? 6 : 5]++;
		h->out_queue.push_back(m);
	}
	if (!h->json_on) return 0;
	if (int rc = json_decode(h, q0)) return rc;
	// a caller that polls only lines: the frames it does not read are kept up to ring_cap
	if ((long long)h->out_queue.size() > h->ring_cap) {
		h->out_queue.erase(h->out_queue.begin(), h->out_queue.end() - h->ring_cap);
		h->queue_overflow_pending = true;
	}
	return 0;
}

} // namespace

extern "C" {

int aisgpu_abi_version(void) { return AISGPU_ABI_VERSION; }

void aisgpu_default_config(aisgpu_config *cfg) {
	memset(cfg, 0, sizeof(*cfg));
	cfg->struct_size = sizeof(*cfg);
	cfg->model = AISGPU_MODEL_DEFAULT;
	cfg->sample_rate = 1536000;
	cfg->format = AISGPU_FMT_CF32;
	cfg->n_streams = 1;
	cfg->max_chunk_samples = 131072;
	cfg->ps_ema = 1;
	cfg->afc_wide = 1;
	cfg->droop = 1;
	cfg->channel_a = 'A';
	cfg->channel_b = 'B';
	cfg->station = 0;
	cfg->own_mmsi = -1;
	cfg->tag_mode = 3;
	cfg->device = 0;
	cfg->enable_taps = 0;
	cfg->max_frames = 0;
	cfg->host_staging = 1;
	cfg->dsk = 0;
	cfg->fp_ds = 0;
	cfg->dd_train = 0.75f;
	cfg->dd_weight = 0.86f;
	cfg->channel_mode = AISGPU_MODE_AB;
}

const char *aisgpu_last_error(aisgpu_handle *h) { return h ? h->err.c_str() : g_create_error.c_str(); }

// hooks for the host-only units of the library (host_internal.h)
const aisgpu_config *aisgpu_internal_config(aisgpu_handle *h) { return &h->cfg; }
int aisgpu_internal_inputs(aisgpu_handle *h) { return inputs(h); }
void aisgpu_internal_set_error(aisgpu_handle *h, const char *msg) { (h ? h->err : g_create_error) = msg; }
int aisgpu_internal_grouped(aisgpu_handle *h) { return h->member || !h->members.empty(); }

static int create_impl(aisgpu_handle *h) {
	const aisgpu_config &c = h->cfg;
	if (c.model != AISGPU_MODEL_DEFAULT && c.model != AISGPU_MODEL_STANDARD && c.model != AISGPU_MODEL_BASE && c.model != AISGPU_MODEL_V2 &&
		c.model != AISGPU_MODEL_CHALLENGER && c.model != AISGPU_MODEL_DISCRIMINATOR) {
		h->err = "unknown model kind";
		return AISGPU_EINVAL;
	}
	if (!format_known(c.format) || c.n_streams < 1 || c.max_chunk_samples < 1) {
		h->err = "bad format / n_streams / max_chunk_samples";
		return AISGPU_EINVAL;
	}
	if (int rc = plan_frontend(h)) return rc;
	h->chain = c.model == AISGPU_MODEL_V2 ? Chain::V2 : (c.model == AISGPU_MODEL_DEFAULT || c.model == AISGPU_MODEL_CHALLENGER) ? Chain::Coherent : Chain::Fm;
	// rows per warp of the decoder kernel, chosen on the previous target (not re-measured on the H100): ModelDefault's 1; 3 for the
	// FM chain with the current front-end shape (slightly faster than 6 rows per warp) and for ModelChallenger's k_decode10
	h->dec_rpw = c.model == AISGPU_MODEL_DEFAULT ? 1 : 3;
	if (const char *e = getenv("AISGPU_DEC_RPW")) {
		h->dec_rpw = atoi(e);
		if (h->dec_rpw != 1 && h->dec_rpw != 3) h->dec_rpw = 6;
	}
	if (const char *e = getenv("AISGPU_DECODER")) h->decoder = atoi(e) == 1 ? 1 : 3;
	if (c.model == AISGPU_MODEL_CHALLENGER) { // ModelChallenger always demodulates with PhaseSearchEMA (Model.cpp:646-652) and needs the fused kernel's derotated output
		h->cfg.ps_ema = 1;
	}
	if (const char *e = getenv("AISGPU_ST_L")) h->st_L = atoi(e);
	int ndev = 0;
	if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
		h->err = "no CUDA device (the CUDA path has no CPU fallback)";
		return AISGPU_ENODEV;
	}
	if (c.device < 0 || c.device >= ndev) {
		h->err = "CUDA device ordinal out of range";
		return AISGPU_ENODEV;
	}
	CU(cudaSetDevice(c.device));
	// Back-end kernels are small and latency bound; give them priority so that their CTAs are dispatched as soon as the
	// (large-grid) front end of the next submit frees a slot, instead of queueing behind all of its CTAs.
	int prio_lo = 0, prio_hi = 0;
	CU(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));
	CU(cudaStreamCreateWithPriority(&h->stream, cudaStreamNonBlocking, prio_hi));
	h->be_streams[0] = h->be_streams[1] = h->stream;
	{
		const char *e = getenv("AISGPU_BE_PIPE");
		// Overlapping the stages of consecutive submits over two back-end streams paid a few per cent for the FM chain on the previous
		// target.  For the coherent chain it is what keeps the step time stable: with one back-end stream the run can lock into a serial
		// pattern (front end c+1 starved while back end c runs, back end c+1 then waiting for it) that costs about half again per step,
		// self-sustaining from the first submits on (tools/default_probe.py shows which pattern a process lands in).
		// ModelV2 is one kernel, and ModelBase's k_base reads the single-buffered FIR37 output: they stay on one stream.
		const bool staged = h->chain == Chain::Coherent || (h->chain == Chain::Fm && standard_tail(h));
		const bool pipe = staged && !c.enable_taps && (e ? atoi(e) != 0 : true);
		if (pipe) CU(cudaStreamCreateWithPriority(&h->be_streams[1], cudaStreamNonBlocking, prio_hi));
	}
	h->bs = h->stream;
	for (int st = 0; st < NSTAGE; st++)
		for (int i = 0; i < 2; i++) CU(new_event(h, &h->ev_stage[st][i]));
	for (int i = 0; i < 2; i++) CU(new_event(h, &h->ev_ec_read[i]));
	CU(new_event(h, &h->ev_join));
	CU(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
	CU(cudaStreamCreateWithFlags(&h->side_stream, cudaStreamNonBlocking));
	CU(cudaStreamCreateWithPriority(&h->fe_stream, cudaStreamNonBlocking, prio_lo));
	for (int i = 0; i < aisgpu_handle::NC; i++) {
		CU(new_event(h, &h->ev_fe_done[i]));
		CU(new_event(h, &h->ev_be_done[i]));
	}
	for (int i = 0; i < 3; i++) {
		CU(new_event(h, &h->ev_rot[i]));
		CU(new_event(h, &h->ev_k1[i]));
	}
	for (int i = 0; i < aisgpu_handle::NEV; i++) {
		CU(new_event(h, &h->ev_fe0s[i], cudaEventDefault));
		CU(new_event(h, &h->ev_fe1s[i], cudaEventDefault));
	}
	for (int i = 0; i < 2; i++) {
		CU(new_event(h, &h->ev_copy[i]));
		CU(new_event(h, &h->ev_done[i]));
	}
	const int B = c.n_streams, k = h->k;
	const int q = outer_granule(h);
	const int maxN = (c.max_chunk_samples + q - 1) / q * q;
	h->cfg.max_chunk_samples = maxN;
	h->rows = rows_of(h);
	h->obps = bytes_per_sample(c.format);
	h->pbps = h->obps;
	h->bps = bytes_per_sample(h->in_fmt);
	h->inner_max = h->pre_dsk ? h->blk : (h->pre_us ? (maxN >> h->kA) : maxN);
	h->max_n48 = h->inner_max >> ((h->xmode || h->disc) ? k : k + 1);
	h->seq.assign(B, 0);
	{
		Receiver r;
		r.channel_a = c.channel_a;
		r.channel_b = c.channel_b;
		r.station = c.station;
		r.own_mmsi = c.own_mmsi;
		r.tag_mode = c.tag_mode;
		h->rx.assign(B, r);
	}
	// a group member (aisgpu_attach) has no front end: no pre-stage, warm-up tails, Rotate tables or input staging
	if ((h->pre_us || h->pre_dsk) && !h->member) { // resampler pre-stage: raw-format history, level-kA stream, schedule tables, rings
		const int tl = raw_tail_len(h);
		for (int i = 0; i < 2; i++) {
			if (int rc = dalloc(h, &h->d_raw_tail[i], (size_t)B * tl * h->obps)) return rc;
			if (c.format == AISGPU_FMT_CU8) CU(cudaMemsetAsync(h->d_raw_tail[i], 0x80, (size_t)B * tl * h->obps, h->stream));
		}
		const int Lmax = maxN >> h->kA;
		if (has_cic(h)) {
			h->d0_stride = (Lmax + 4 + 1) & ~1LL;
			if (int rc = dalloc(h, &h->d_D0, (size_t)B * h->d0_stride)) return rc;
			memset(&h->fe_pre, 0, sizeof(h->fe_pre));
		}
		if (h->pre_us) {
			if (int rc = dalloc(h, &h->d_us_src, (size_t)h->us_ratio * Lmax + 8)) return rc;
			if (int rc = dalloc(h, &h->d_us_alpha, (size_t)h->us_ratio * Lmax + 8)) return rc;
			h->us_ring.stride = (long long)(h->us_ratio + 2) * Lmax; // its cap is set by the first submit, whose length fixes the block
			if (int rc = dalloc(h, &h->us_ring.d, (size_t)B * h->us_ring.stride)) return rc;
		}
		if (h->pre_dsk) {
			const int cap96 = ((2 * maxN / 3 + 1 + h->blk + h->blk - 1) / h->blk + 1) * h->blk; // behind Upsample up to 2x the samples
			CU(set_taps_bh28_3(H_TAPS_BH28_3));
			h->dsk_ring.cap = cap96;
			h->dsk_ring.stride = cap96;
			if (int rc = dalloc(h, &h->dsk_ring.d, (size_t)B * cap96)) return rc;
			if (has_cic(h))
				for (int i = 0; i < 2; i++)
					if (int rc = dalloc(h, &h->d_cf_tail[i], (size_t)B * 32)) return rc;
		}
	}
	for (int i = 0; i < 2; i++) {
		if (h->P && !h->member) {
			if (int rc = dalloc(h, &h->d_tail[i], (size_t)B * h->P * h->bps)) return rc;
			// F32_FS4 stays zero bytes.  +0 floats expand to (+0, 0), (0, +0), (-0, 0), (0, -0), and warming up on them from the
			// reference's all +0 state leaves +0 everywhere but in the imaginary part of a first stage's h0 (the last odd sample,
			// stored as it is).  The first thing added to that component is the literal +0 of the next even sample, and
			// +0 + -0 = +0 + +0: no output can tell the -0 from the reference's +0.
			if (h->in_fmt == AISGPU_FMT_CU8 && !h->fp_ds) // the reference's zero initial filter state is byte value 128 in CU8 (0 for the unbiased integer pipeline)
				CU(cudaMemsetAsync(h->d_tail[i], 0x80, (size_t)B * h->P * h->bps, h->stream));
		}
		if (int rc = dalloc(h, &h->d_fir_hist[i], (size_t)h->rows * 16)) return rc;
	}
	if (!h->xmode && !h->disc && !h->member) {
		for (int i = 0; i < 3; i++)
			if (int rc = dalloc(h, &h->d_rot[i], (size_t)h->P96 + (h->inner_max >> k) + 8)) return rc;
		if (int rc = dalloc(h, &h->d_rot_state, 4)) return rc;
		float2 one = make_float2(1.0f, 0.0f);
		CU(cudaMemcpyAsync(h->d_rot_state, &one, sizeof(one), cudaMemcpyHostToDevice, h->stream)); // after the memset on the same stream
		h->mult = polar1((float)(PI_F * 25000.0 / 48000.0)); // Model.cpp:31
	}
	h->c_stride = (HC + h->max_n48 + 8 + 1) & ~1LL;
	for (int i = 0; i < 2; i++)
		if (int rc = dalloc(h, &h->d_C2[i], (size_t)h->rows * h->c_stride)) return rc;
	if (int rc = dalloc(h, &h->d_C2[2], (size_t)h->rows * h->c_stride)) return rc;
	const int nEmax = HC + h->max_n48;
	h->e_stride = (HE + nEmax + 8 + 1) & ~1LL;
	h->r_stride = nEmax;
	const int ndec = h->chain == Chain::V2 ? 6 : (c.model == AISGPU_MODEL_CHALLENGER ? 10 : 5); // decoders per row
	if (int rc = dalloc(h, &h->d_dec, (size_t)h->rows * ndec)) return rc;
	if (int rc = dalloc(h, &h->d_dec_data, (size_t)h->rows * ndec * DEC_WORDS)) return rc;
	if (int rc = dalloc(h, &h->d_level_rows, (size_t)(h->rows + 31) / 32)) return rc;
	if (int rc = put_level_rows(h)) return rc;
	if (int rc = h->chain == Chain::Fm ? alloc_fm(h, nEmax) : h->chain == Chain::Coherent ? alloc_coherent(h, nEmax) : alloc_v2(h)) return rc;
	if (c.enable_taps)
		if (int rc = dalloc(h, &h->d_tap_dec, (size_t)h->rows * 5 * (nEmax / 5 + 2))) return rc;
	if (getenv("AISGPU_DEBUG"))
		if (int rc = dalloc(h, &h->d_dbg, (size_t)h->rows * 4)) return rc;
	{
		std::vector<float2> om(CGF_N / 2);
		for (int s = 0; s < CGF_N / 2; s++) om[s] = polar1((float)(-2.0 * PI_F) * (float)s / (float)CGF_N); // FFT.h:81-83
		CU(cgf_init(H_TAPS_COHERENT, om.data()));
	}
	CU(fm_init(H_TAPS_RECEIVER));
	{
		uint32_t ab[35] = { 0 };
		const int pos[] = { 30, 62, 96, 168, 184, 192, 336, 385, 448, MAX_FRAME_BITS }; // AIS.cpp:111-142, AIS.h:172
		for (int q : pos) ab[q >> 5] |= 1u << (q & 31);
		CU(sym_init(H_PS_COS, H_PS_SIN, ab));
	}
	h->ring_cap = c.max_frames > 0 ? c.max_frames : std::max(4096, B * 64);
	if (int rc = dalloc(h, &h->d_ring, (size_t)h->ring_cap)) return rc;
	if (int rc = dalloc(h, &h->d_ring_head, 1)) return rc;
	if (int rc = dalloc(h, &h->d_counts, 16)) return rc;
	if (int rc = halloc(h, &h->pin_head, aisgpu_handle::NT)) return rc;
	memset(h->pin_head, 0, aisgpu_handle::NT * sizeof(unsigned long long));
	for (int i = 0; i < aisgpu_handle::NT; i++) CU(new_event(h, &h->ev_ticket[i]));
	CU(new_event(h, &h->ev_mark));
	if (h->pre_us && !h->member) {
		h->us_cap = h->us_ratio * (maxN >> h->kA) + 8; // Upsample emits at most ceil(bucket / rate) samples per input
		for (int i = 0; i < 2; i++) {
			if (int rc = halloc(h, &h->pin_us_src[i], (size_t)h->us_cap)) return rc;
			if (int rc = halloc(h, &h->pin_us_alpha[i], (size_t)h->us_cap)) return rc;
			CU(new_event(h, &h->ev_us[i]));
		}
	}
	if (c.host_staging && !h->member) // the H2D staging buffers of aisgpu_submit / _v / _async (otherwise allocated by the first host submit)
		for (int i = 0; i < 2; i++)
			if (int rc = dalloc(h, &h->d_in[i], (size_t)B * maxN * h->obps)) return rc;
	memset(&h->fe, 0, sizeof(h->fe));
	CU(cudaStreamSynchronize(h->stream));
	return 0;
}

// The caller's config: the current layout, or the one before channel_mode was appended (then AB).
static bool copy_config(const aisgpu_config *cfg, aisgpu_config *c) {
	if (!cfg || (cfg->struct_size != sizeof(aisgpu_config) && cfg->struct_size != offsetof(aisgpu_config, channel_mode))) return false;
	memset(c, 0, sizeof(*c));
	memcpy(c, cfg, cfg->struct_size);
	c->struct_size = sizeof(aisgpu_config);
	if (cfg->struct_size != sizeof(aisgpu_config)) c->channel_mode = AISGPU_MODE_AB;
	return true;
}

int aisgpu_create(const aisgpu_config *cfg, aisgpu_handle **out) {
	aisgpu_config c;
	if (!out || !copy_config(cfg, &c)) {
		g_create_error = "aisgpu_create: null argument or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	aisgpu_handle *h = new aisgpu_handle();
	h->cfg = c;
	h->given = c;
	int rc = create_impl(h);
	if (rc) {
		g_create_error = h->err;
		aisgpu_destroy(h);
		*out = nullptr;
		return rc;
	}
	*out = h;
	return 0;
}

// a CUDA failure (or an internal inconsistency) inside a submit leaves carried state half-advanced: poison the handle
// (a group's submit advances every member's state too: the whole group is poisoned)
static int poison(aisgpu_handle *h, int rc) {
	if (rc != 0 && rc != AISGPU_EINVAL && !h->poisoned) {
		h->poisoned = rc;
		for (aisgpu_handle *m : h->members)
			if (!m->poisoned) {
				m->poisoned = rc;
				m->err = h->err;
			}
	}
	return rc;
}
#define ENTER(h)                                  \
	do {                                          \
		if (!(h)) return AISGPU_EINVAL;           \
		if ((h)->poisoned) return (h)->poisoned;  \
		CU(cudaSetDevice((h)->cfg.device));       \
	} while (0)

// a group member is fed by its leader's submits only
static int refuse_member(aisgpu_handle *h) {
	if (!h->member) return 0;
	h->err = "this engine is a member of a group: submit to the group's leader";
	return AISGPU_EINVAL;
}

// The checks of every submit before anything is enqueued: the length, then the channel dump (a stopped dump refuses the submit with
// AISGPU_EIO, which does not poison the handle; a slot still holding rows is written out)
static int submit_gate(aisgpu_handle *h, int n_samples) {
	if (int rc = check_outer(h, n_samples)) return rc;
	return dump_reclaim(h);
}

int aisgpu_submit_device(aisgpu_handle *h, const void *dev_samples, int64_t stride_samples, int n_samples) {
	ENTER(h);
	if (int rc = refuse_member(h)) return rc;
	if (!dev_samples) return AISGPU_EINVAL;
	if (int rc = check_placement(h, dev_samples, stride_samples)) return rc;
	if (stride_samples < n_samples) {
		h->err = "stride_samples must be >= n_samples";
		return AISGPU_EINVAL;
	}
	if (int rc = submit_gate(h, n_samples)) return rc; // all argument checks come before any state is touched
	return poison(h, submit_outer(h, dev_samples, stride_samples, n_samples));
}

// Host submits: the batch (one row per input, inputs(h)) goes through one of two device staging buffers (copy stream), the front end
// of the submit before last being the previous reader of that buffer.  `ptrs` != nullptr: one host pointer per input row.
static int submit_host(aisgpu_handle *h, const void *host_samples, const void *const *ptrs, int n_samples, bool wait_copy, int64_t *ticket) {
	if (int rc = check_outer(h, n_samples)) return rc;
	const size_t row_bytes = (size_t)n_samples * h->obps;
	const int cur = h->in_cur, R = inputs(h);
	if (!h->d_in[cur]) {
		if (int rc = dalloc(h, &h->d_in[cur], (size_t)R * h->cfg.max_chunk_samples * h->obps)) return rc;
		CU(cudaStreamSynchronize(h->stream)); // dalloc clears on h->stream
	}
	if (h->in_used[cur]) CU(cudaStreamWaitEvent(h->copy_stream, h->ev_done[cur], 0));
	if (ptrs) {
		for (int s = 0; s < R; s++) {
			if (!ptrs[s]) {
				h->err = "null stream pointer";
				return AISGPU_EINVAL;
			}
		}
		for (int s = 0; s < R; s++)
			CU(cudaMemcpyAsync(h->d_in[cur] + (size_t)s * row_bytes, ptrs[s], row_bytes, cudaMemcpyHostToDevice, h->copy_stream));
	}
	else CU(cudaMemcpyAsync(h->d_in[cur], host_samples, row_bytes * R, cudaMemcpyHostToDevice, h->copy_stream));
	CU(cudaEventRecord(h->ev_copy[cur], h->copy_stream));
	CU(cudaStreamWaitEvent(h->fe_stream, h->ev_copy[cur], 0));
	if (ticket) *ticket = (int64_t)h->counters[3];
	if (int rc = submit_outer(h, h->d_in[cur], n_samples, n_samples)) return rc;
	CU(cudaEventRecord(h->ev_done[cur], h->fe_stream)); // the front end is the only reader of the staging buffer
	h->in_used[cur] = true;
	h->in_cur ^= 1;
	// aisgpu_submit / _v: the caller's buffer is only borrowed for the call (Stream.h:41 semantics): wait for the copy, not
	// for the kernels
	if (wait_copy) CU(cudaEventSynchronize(h->ev_copy[cur]));
	return 0;
}

int aisgpu_submit(aisgpu_handle *h, const void *host_samples, int n_samples) {
	ENTER(h);
	if (int rc = refuse_member(h)) return rc;
	if (!host_samples) return AISGPU_EINVAL;
	if (int rc = submit_gate(h, n_samples)) return rc;
	return poison(h, submit_host(h, host_samples, nullptr, n_samples, true, nullptr));
}

int aisgpu_submit_v(aisgpu_handle *h, const void *const *stream_ptrs, int n_samples) {
	ENTER(h);
	if (int rc = refuse_member(h)) return rc;
	if (!stream_ptrs) return AISGPU_EINVAL;
	if (int rc = submit_gate(h, n_samples)) return rc;
	return poison(h, submit_host(h, nullptr, stream_ptrs, n_samples, true, nullptr));
}

int aisgpu_submit_async(aisgpu_handle *h, const void *host_samples, int n_samples, int64_t *ticket) {
	ENTER(h);
	if (int rc = refuse_member(h)) return rc;
	if (!host_samples) return AISGPU_EINVAL;
	if (int rc = submit_gate(h, n_samples)) return rc;
	return poison(h, submit_host(h, host_samples, nullptr, n_samples, false, ticket));
}

int aisgpu_sync(aisgpu_handle *h) {
	ENTER(h);
	CU(cudaStreamSynchronize(h->copy_stream));
	CU(cudaStreamSynchronize(h->fe_stream));
	if (int rc = sync_backend(h)) return rc;
	for (aisgpu_handle *m : h->members)
		if (int rc = sync_backend(m)) {
			h->err = m->err;
			return rc;
		}
	return dump_write(h, -1);
}

int aisgpu_poll_upto(aisgpu_handle *h, int64_t ticket, aisgpu_msg *out, int max, int *n) {
	if (!n || (max > 0 && !out)) return AISGPU_EINVAL;
	ENTER(h);
	if (int rc = dump_write(h, ticket > (int64_t)h->counters[3] - 1 ? -1 : (long long)ticket)) return rc;
	if (h->out_pos >= h->out_queue.size()) {
		h->out_queue.clear();
		h->out_pos = 0;
		if (int rc = drain_ring(h, (long long)ticket)) return rc;
	}
	int k = 0;
	while (k < max && h->out_pos < h->out_queue.size()) out[k++] = h->out_queue[h->out_pos++];
	*n = k;
	if (h->overflow_pending) { // reported once per loss, together with the frames that survived
		h->overflow_pending = false;
		h->err = "frame ring overflow: frames were dropped (see counters[4]); raise aisgpu_config.max_frames or poll more often";
		return AISGPU_EOVERFLOW;
	}
	if (h->queue_overflow_pending) {
		h->queue_overflow_pending = false;
		h->err = "frames were dropped from the host queue: with JSON enabled, more than max_frames frames were left unread";
		return AISGPU_EOVERFLOW;
	}
	return 0;
}

int aisgpu_poll(aisgpu_handle *h, aisgpu_msg *out, int max, int *n) { return aisgpu_poll_upto(h, -1, out, max, n); }

namespace {

// The tag stream s's records are printed with: the output's, with a receiver table the receiver's station, driver, hardware, mode
// and ipv4
aisgpu_tag tag_of(const aisgpu_handle *h, int s) {
	aisgpu_tag t = h->fmt_tag;
	t.hardware = h->fmt_hw.c_str();
	t.uuid = h->fmt_uuid.c_str();
	t.suffix = h->fmt_suffix.c_str();
	if (h->rx_table) {
		const Receiver &r = h->rx[s];
		t.station = r.station;
		t.driver = r.driver;
		t.hardware = r.hardware.c_str();
		t.mode = (int32_t)r.tag_mode;
		t.ipv4 = r.ipv4;
	}
	return t;
}

// The format's contexts -- one, or one per stream with a receiver table -- with their strings in one packed buffer, and the slots and
// text sized for the longest of them.  lines_enable calls it, and aisgpu_set_receivers again when a format is already enabled: the
// buffers that depend on the strings are then made anew (nothing has been submitted, so nothing uses them).
int fmt_setup(aisgpu_handle *h) {
	const int nctx = h->rx_table ? h->cfg.n_streams : 1;
	std::vector<aisgpu_tag> tags((size_t)nctx);
	std::vector<AjPrefix> prefixes((size_t)nctx);
	std::vector<size_t> hw_at((size_t)nctx), prefix_at((size_t)nctx);
	std::string strings = h->fmt_uuid + '\0' + h->fmt_suffix + '\0';
	size_t longest = 0, longest_prefix = 0;
	for (int i = 0; i < nctx; i++) {
		tags[i] = tag_of(h, i);
		prefixes[i] = aj_prefix(&tags[i]);
		hw_at[i] = strings.size();
		strings += std::string(tags[i].hardware) + '\0';
		prefix_at[i] = strings.size();
		strings += prefixes[i].text + '\0';
		// the full-JSON line holds the prefix and, where the mode prints them, the time members of any stamp
		const size_t line_head = prefixes[i].text.size() + ((tags[i].mode & 2) ? kAjTimeMax : 0);
		longest = std::max(longest, line_head + strlen(tags[i].hardware) * 6);
		longest_prefix = std::max(longest_prefix, line_head);
	}
	h->fmt_strings = strings;
	// a record's room: the longest record of its format with the tag's strings (the hardware name escaped, uuid and suffix once per
	// sentence) -- four fully escaped sentences (2.4 KB) plus the longest fields (1.3 KB) after the full-JSON prefix, and for
	// JSON_ANNOTATED their units and descriptions besides; JSON_SPARSE and JSON_ANNOTATED add a scratch full line to the slot
	const size_t strs = longest + (h->fmt_uuid.size() + h->fmt_suffix.size()) * 4;
	const int fmt = h->fmt;
	const bool rewritten = fmt == AISGPU_MSGFORMAT_JSON_SPARSE || fmt == AISGPU_MSGFORMAT_JSON_ANNOTATED;
	h->rec_cap = (int)((strs + (fmt == AISGPU_MSGFORMAT_JSON_ANNOTATED ? 20480 : 4096) + 15) / 16 * 16);
	h->json_slot = h->rec_cap + (rewritten ? (int)((longest_prefix + 4096 + 15) / 16 * 16) : 0);
	if (!h->json_stream) {
		CU(cudaStreamCreateWithFlags(&h->json_stream, cudaStreamNonBlocking));
		if (int rc = dalloc(h, &h->d_jtotal, 4)) return rc;
		if (int rc = halloc(h, &h->pin_jtotal, 4)) return rc;
		if (int rc = dalloc(h, &h->d_jmsg, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_jlen, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_jseg, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_jkeep, kJsonBatch)) return rc;
		if (int rc = halloc(h, &h->pin_jkeep, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_jgroups, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_jpsum, kJsonBatch)) return rc;
		if (int rc = dalloc(h, &h->d_joff, kJsonBatch)) return rc;
	}
	if (h->clock && !h->d_jstamp)
		if (int rc = dalloc(h, &h->d_jstamp, kJsonBatch)) return rc;
	dfree(h, h->d_jstrings);
	dfree(h, h->d_fctx);
	dfree(h, h->d_jslots);
	dfree(h, h->d_jtext);
	hfree(h, h->pin_jtext);
	const size_t text = (size_t)kJsonBatch * h->rec_cap;
	if (int rc = dalloc(h, &h->d_jstrings, strings.size())) return rc;
	if (int rc = dalloc(h, &h->d_fctx, (size_t)nctx)) return rc;
	if (int rc = dalloc(h, &h->d_jslots, (size_t)kJsonBatch * h->json_slot)) return rc;
	if (int rc = dalloc(h, &h->d_jtext, text)) return rc;
	if (int rc = halloc(h, &h->pin_jtext, text)) return rc;
	// dalloc zeroes each buffer on h->stream: the strings and the contexts are written after that, not under it
	CU(cudaStreamSynchronize(h->stream));
	CU(cudaMemcpy(h->d_jstrings, strings.data(), strings.size(), cudaMemcpyHostToDevice));
	std::vector<FmtCtx> ctx((size_t)nctx);
	for (int i = 0; i < nctx; i++) {
		ctx[i] = fmt_ctx(&tags[i], fmt, h->fmt_suffix.c_str(), prefixes[i]);
		ctx[i].uuid = h->d_jstrings;
		ctx[i].suffix = h->d_jstrings + h->fmt_uuid.size() + 1;
		ctx[i].hardware = h->d_jstrings + hw_at[i];
		ctx[i].prefix = h->d_jstrings + prefix_at[i];
	}
	CU(cudaMemcpy(h->d_fctx, ctx.data(), ctx.size() * sizeof(FmtCtx), cudaMemcpyHostToDevice));
	return 0;
}

// aisgpu_lines_enable and aisgpu_json_enable (who: the entry point, for the messages)
int lines_enable(aisgpu_handle *h, int fmt, const aisgpu_tag *tag, const char *suffix, int max_bytes_per_submit, bool json_api,
				 const char *who) {
	ENTER(h);
	if (!tag || max_bytes_per_submit <= 0 || fmt < AISGPU_MSGFORMAT_NMEA || fmt > AISGPU_MSGFORMAT_JSON_ANNOTATED) {
		h->err = std::string(who) + ": bad argument";
		return AISGPU_EINVAL;
	}
	if (h->counters[3] > 0 || h->json_on) {
		h->err = std::string(who) + (h->json_on ? ": a format is already enabled" : ": the engine has been submitted to");
		return AISGPU_EINVAL;
	}
	h->fmt_tag = *tag;
	h->fmt_hw = tag->hardware ? tag->hardware : "";
	h->fmt_uuid = tag->uuid ? tag->uuid : "";
	h->fmt_suffix = suffix;
	h->fmt = fmt;
	h->json_api = json_api;
	h->json_cap = max_bytes_per_submit;
	if (int rc = fmt_setup(h)) return rc;
	h->json_on = true;
	return 0;
}

// aisgpu_poll_lines and aisgpu_poll_json: whole records from the queue until the next would pass cap
int poll_records(aisgpu_handle *h, int64_t ticket, char *out, size_t cap, size_t *n_bytes, int *n_records, const char *who) {
	*n_bytes = 0;
	*n_records = 0;
	if (h->rec_len.empty())
		if (int rc = drain_ring(h, (long long)ticket)) return rc;
	size_t k = 0;
	int recs = 0;
	while (recs < (int)h->rec_len.size() && k + (size_t)h->rec_len[recs] <= cap) k += (size_t)h->rec_len[recs++];
	if (recs == 0 && !h->rec_len.empty()) {
		h->err = std::string(who) + (h->json_api ? ": cap is smaller than the next line" : ": cap is smaller than the next record");
		return AISGPU_EINVAL;
	}
	if (k) memcpy(out, h->json_buf.data() + h->json_pos, k);
	h->json_pos += k;
	h->rec_len.erase(h->rec_len.begin(), h->rec_len.begin() + recs);
	*n_bytes = k;
	*n_records = recs;
	if (h->json_overflow_pending) {
		h->json_overflow_pending = false;
		h->err = h->json_api ? "JSON text overflow: lines were dropped; raise max_bytes_per_submit of aisgpu_json_enable"
							 : "record overflow: records were dropped; raise max_bytes_per_submit of aisgpu_lines_enable";
		return AISGPU_EOVERFLOW;
	}
	return 0;
}

} // namespace

int aisgpu_json_enable(aisgpu_handle *h, const aisgpu_tag *tag, int max_bytes_per_submit) {
	return lines_enable(h, AISGPU_MSGFORMAT_JSON_FULL, tag, "\n", max_bytes_per_submit, true, "aisgpu_json_enable");
}

int aisgpu_lines_enable(aisgpu_handle *h, int msgformat, const aisgpu_tag *tag, int max_bytes_per_submit) {
	return lines_enable(h, msgformat, tag, tag && tag->suffix ? tag->suffix : "\r\n", max_bytes_per_submit, false,
						"aisgpu_lines_enable");
}

int aisgpu_poll_json(aisgpu_handle *h, int64_t ticket, char *out, size_t cap, size_t *n_bytes, int *n_lines) {
	if (!n_bytes || !n_lines || (cap > 0 && !out)) return AISGPU_EINVAL;
	ENTER(h);
	if (!h->json_api) {
		h->err = h->json_on ? "aisgpu_poll_json: the engine formats another message format (aisgpu_poll_lines)"
							: "aisgpu_poll_json: JSON is not enabled (aisgpu_json_enable)";
		return AISGPU_EINVAL;
	}
	return poll_records(h, ticket, out, cap, n_bytes, n_lines, "aisgpu_poll_json");
}

int aisgpu_poll_lines(aisgpu_handle *h, int64_t ticket, char *out, size_t cap, size_t *n_bytes, int *n_records) {
	if (!n_bytes || !n_records || (cap > 0 && !out)) return AISGPU_EINVAL;
	ENTER(h);
	if (!h->json_on) {
		h->err = "aisgpu_poll_lines: no format is enabled (aisgpu_lines_enable)";
		return AISGPU_EINVAL;
	}
	return poll_records(h, ticket, out, cap, n_bytes, n_records, "aisgpu_poll_lines");
}

namespace {

// Receiver::setChannel's test of a designation letter (Application/Receiver.cpp:103-105): alphanumeric or '?'
bool channel_letter_ok(char c) { return (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || (c >= '0' && c <= '9') || c == '?'; }

// The rules of aisgpu_set_receivers that need no device: "" or the reason.  channel_b is read where a stream has two channels (AB
// mode, and the FM-discriminator input model in either mode).
std::string receivers_refusal(const aisgpu_config &c, const aisgpu_receiver *r, int n) {
	if (!r) return "aisgpu_set_receivers: null receiver table";
	if (n != c.n_streams) return "aisgpu_set_receivers: " + std::to_string(n) + " receivers for " + std::to_string(c.n_streams) + " streams";
	const bool two = c.channel_mode != AISGPU_MODE_X || c.model == AISGPU_MODEL_DISCRIMINATOR;
	for (int s = 0; s < n; s++) {
		if (!channel_letter_ok(r[s].channel_a)) return "invalid NMEA channel designation: " + std::string(1, r[s].channel_a);
		if (two && !channel_letter_ok(r[s].channel_b)) return "invalid NMEA channel designation: " + std::string(1, r[s].channel_b);
	}
	return "";
}

} // namespace

int aisgpu_check_receivers(const aisgpu_config *cfg, const aisgpu_receiver *r, int n) {
	aisgpu_config c;
	if (!copy_config(cfg, &c)) {
		g_create_error = "aisgpu_check_receivers: null config or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	const std::string why = receivers_refusal(c, r, n);
	if (!why.empty()) {
		g_create_error = why;
		return AISGPU_EINVAL;
	}
	return 0;
}

int aisgpu_set_receivers(aisgpu_handle *h, const aisgpu_receiver *r, int n) {
	ENTER(h);
	std::string why = receivers_refusal(h->given, r, n);
	if (why.empty() && h->rx_table) why = "aisgpu_set_receivers: a receiver table is already installed";
	if (why.empty() && h->counters[3] > 0) why = "aisgpu_set_receivers: the engine has been submitted to (install the table before the first submit)";
	if (!why.empty()) {
		h->err = why;
		return AISGPU_EINVAL;
	}
	std::vector<Receiver> rx((size_t)n);
	for (int s = 0; s < n; s++) {
		rx[s].channel_a = r[s].channel_a;
		rx[s].channel_b = r[s].channel_b;
		rx[s].station = r[s].station;
		rx[s].own_mmsi = r[s].own_mmsi;
		rx[s].tag_mode = r[s].tag_mode;
		rx[s].driver = r[s].driver;
		rx[s].hardware = r[s].hardware ? r[s].hardware : "";
		rx[s].ipv4 = r[s].ipv4;
	}
	h->rx.swap(rx);
	h->rx_table = true;
	if (int rc = put_level_rows(h)) return rc;
	if (h->json_on)
		if (int rc = fmt_setup(h)) return rc;
	return 0;
}

namespace {

// The rules of aisgpu_set_tunings that need no device: "" or the reason.  fp_ds: the engine runs the integer CIC front end.
std::string tuning_refusal(const aisgpu_config &c, bool fp_ds, const int32_t *f, int n, int per_input) {
	if (!f) return "aisgpu_set_tuning: null offset table";
	if (n != c.n_streams) return "aisgpu_set_tuning: " + std::to_string(n) + " offsets for " + std::to_string(c.n_streams) + " streams";
	if (per_input < 1 || c.n_streams % per_input)
		return "aisgpu_set_tunings: per_input " + std::to_string(per_input) + " must be at least 1 and divide n_streams " +
			   std::to_string(c.n_streams);
	if (c.model == AISGPU_MODEL_DISCRIMINATOR)
		return "aisgpu_set_tuning: the FM-discriminator input model reads I and Q as two real audio channels: there is nothing to tune";
	if (fp_ds) return "aisgpu_set_tuning: FP_DS on: the integer front end reads the caller's CU8 samples directly and cannot take tuned ones";
	const long long fs = c.sample_rate;
	for (int s = 0; s < n; s++)
		if (2 * (long long)f[s] <= -fs || 2 * (long long)f[s] >= fs)
			return "aisgpu_set_tuning: stream " + std::to_string(s) + ": offset " + std::to_string(f[s]) +
				   " Hz must lie strictly between -fs/2 and fs/2 (fs = " + std::to_string(fs) + ")";
	return "";
}

} // namespace

int aisgpu_check_tunings(const aisgpu_config *cfg, const int32_t *offset_hz, int n, int per_input) {
	aisgpu_config c;
	if (!copy_config(cfg, &c)) {
		g_create_error = "aisgpu_check_tuning: null config or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	// plan_frontend's FP_DS condition: the exact 1536K bucket of AB mode fed CU8
	const bool fp_ds = c.fp_ds && c.channel_mode == AISGPU_MODE_AB && c.model != AISGPU_MODEL_DISCRIMINATOR && c.sample_rate == 1536000 &&
					   c.format == AISGPU_FMT_CU8;
	const std::string why = tuning_refusal(c, fp_ds, offset_hz, n, per_input);
	if (!why.empty()) {
		g_create_error = why;
		return AISGPU_EINVAL;
	}
	return 0;
}

int aisgpu_check_tuning(const aisgpu_config *cfg, const int32_t *offset_hz, int n) { return aisgpu_check_tunings(cfg, offset_hz, n, 1); }

int aisgpu_set_tunings(aisgpu_handle *h, const int32_t *offset_hz, int n, int per_input) {
	ENTER(h);
	std::string why = tuning_refusal(h->given, h->fp_ds != 0, offset_hz, n, per_input);
	if (why.empty() && h->member)
		why = "aisgpu_set_tuning: this engine is a member of a group and reads its leader's front end: install the table on the leader";
	if (why.empty() && h->tuned) why = "aisgpu_set_tuning: a tuning table is already installed";
	if (why.empty() && h->counters[3] > 0) why = "aisgpu_set_tuning: the engine has been submitted to (install the table before the first submit)";
	if (!why.empty()) {
		h->err = why;
		return AISGPU_EINVAL;
	}
	// Everything behind the tune reads CF32: plan the front end again for it (it passed for the caller's format at creation, and the
	// plan only differs in the format it reads and the warm-up history that follows from it), and give the warm-up histories CF32 size.
	const int B = h->cfg.n_streams, fs = h->cfg.sample_rate;
	h->tuned = true;
	h->per_input = per_input;
	if (int rc = plan_frontend(h)) return poison(h, rc == AISGPU_EINVAL ? AISGPU_ECUDA : rc);
	h->bps = bytes_per_sample(h->in_fmt);
	h->pbps = bytes_per_sample(AISGPU_FMT_CF32);
	for (int i = 0; i < 2; i++) {
		dfree(h, h->d_tail[i]);
		if (h->P)
			if (int rc = dalloc(h, &h->d_tail[i], (size_t)B * h->P * h->bps)) return poison(h, rc);
		if (h->d_raw_tail[i]) {
			dfree(h, h->d_raw_tail[i]);
			if (int rc = dalloc(h, &h->d_raw_tail[i], (size_t)B * raw_tail_len(h) * h->pbps)) return poison(h, rc);
		}
		// host staging allocated at creation holds one row per stream; no submit has used it yet: one row per input from now on
		if (h->d_in[i] && per_input > 1) {
			dfree(h, h->d_in[i]);
			if (int rc = dalloc(h, &h->d_in[i], (size_t)inputs(h) * h->cfg.max_chunk_samples * h->obps)) return poison(h, rc);
		}
	}
	if (!tune_into_d0(h)) {
		h->tune_stride = h->cfg.max_chunk_samples; // a multiple of the granule: even, so every CF32 row is 16-byte aligned
		if (int rc = dalloc(h, &h->d_tune, (size_t)B * h->tune_stride)) return poison(h, rc);
	}
	std::vector<float2> tab((size_t)tune_table_len(fs));
	tune_tables(fs, tab.data());
	std::vector<int> fk((size_t)B);
	for (int s = 0; s < B; s++) fk[s] = offset_hz[s] < 0 ? offset_hz[s] + fs : offset_hz[s];
	if (int rc = dalloc(h, &h->d_tune_tab, tab.size())) return poison(h, rc);
	if (int rc = dalloc(h, &h->d_tune_fk, fk.size())) return poison(h, rc);
	CU(cudaMemcpyAsync(h->d_tune_tab, tab.data(), tab.size() * sizeof(float2), cudaMemcpyHostToDevice, h->stream));
	CU(cudaMemcpyAsync(h->d_tune_fk, fk.data(), fk.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
	CU(cudaStreamSynchronize(h->stream));
	// k_tune keeps the tables in shared memory (at most 56.3 KB): four CTAs per SM, each walking many segments
	int sms = 0;
	CU(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, h->cfg.device));
	h->tune_ctas = 4 * sms;
	return 0;
}

int aisgpu_set_tuning(aisgpu_handle *h, const int32_t *offset_hz, int n) { return aisgpu_set_tunings(h, offset_hz, n, 1); }

namespace {

const long long kClockEnd = 253402300800000000LL; // 10000-01-01T00:00:00Z in microseconds: rxtime stays YYYYMMDDHHMMSS below it

// The rules of aisgpu_set_clock that need no device: "" or the reason.
std::string clock_refusal(const aisgpu_config &c, const int64_t *start_us, int n) {
	if (n != c.n_streams) return "aisgpu_set_clock: " + std::to_string(n) + " start times for " + std::to_string(c.n_streams) + " streams";
	if (start_us)
		for (int s = 0; s < n; s++)
			if (start_us[s] < 0 || start_us[s] >= kClockEnd)
				return "aisgpu_set_clock: stream " + std::to_string(s) + ": start " + std::to_string((long long)start_us[s]) +
					   " us must lie in [0, " + std::to_string(kClockEnd) + ") (1970-01-01 .. 9999-12-31)";
	return "";
}

} // namespace

int aisgpu_check_clock(const aisgpu_config *cfg, const int64_t *start_us, int n) {
	aisgpu_config c;
	if (!copy_config(cfg, &c)) {
		g_create_error = "aisgpu_check_clock: null config or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	const std::string why = clock_refusal(c, start_us, n);
	if (!why.empty()) {
		g_create_error = why;
		return AISGPU_EINVAL;
	}
	return 0;
}

int aisgpu_set_clock(aisgpu_handle *h, const int64_t *start_us, int n) {
	ENTER(h);
	std::string why = clock_refusal(h->given, start_us, n);
	if (why.empty() && h->member)
		why = "aisgpu_set_clock: this engine is a member of a group: its leader's clock stamps the group's frames (set it on the leader)";
	if (why.empty() && h->clock) why = "aisgpu_set_clock: a clock is already set";
	if (why.empty() && h->counters[3] > 0) why = "aisgpu_set_clock: the engine has been submitted to (set the clock before the first submit)";
	if (!why.empty()) {
		h->err = why;
		return AISGPU_EINVAL;
	}
	auto clk = std::make_shared<Clock>();
	clk->live = start_us == nullptr;
	clk->fs = h->given.sample_rate;
	if (start_us) clk->start_us.assign(start_us, start_us + n);
	std::vector<aisgpu_handle *> group(1, h);
	group.insert(group.end(), h->members.begin(), h->members.end());
	for (aisgpu_handle *e : group) {
		e->clock = clk;
		if (e->json_on && !e->d_jstamp) { // a format enabled before the clock: the stamps' device buffer
			if (int rc = dalloc(e, &e->d_jstamp, kJsonBatch)) return poison(h, rc);
			CU(cudaStreamSynchronize(e->stream));
		}
	}
	return 0;
}

int aisgpu_stamp(aisgpu_handle *h, int stream, int64_t chunk, int64_t *rxtime_us) {
	if (!h || !rxtime_us) return AISGPU_EINVAL;
	if (!h->clock) {
		h->err = "aisgpu_stamp: the engine has no clock (aisgpu_set_clock)";
		return AISGPU_EINVAL;
	}
	if (stream < 0 || stream >= h->cfg.n_streams) {
		h->err = "aisgpu_stamp: no stream " + std::to_string(stream);
		return AISGPU_EINVAL;
	}
	if (chunk < 0 || chunk >= (int64_t)h->clock->at.size()) {
		h->err = "aisgpu_stamp: no submit " + std::to_string((long long)chunk) + " (" + std::to_string(h->clock->at.size()) + " so far)";
		return AISGPU_EINVAL;
	}
	*rxtime_us = h->clock->stamp(stream, chunk);
	return 0;
}

int aisgpu_tap(aisgpu_handle *h, int tap, int stream, int channel, void *dst, size_t dst_bytes, size_t *n_out) {
	if (!h || !n_out || stream < 0 || stream >= h->cfg.n_streams || channel < 0 || channel > 9) return AISGPU_EINVAL;
	CU(cudaSetDevice(h->cfg.device));
	CU(cudaStreamSynchronize(h->fe_stream));
	if (int rc = sync_backend(h)) return rc;
	if (h->xmode && (tap == AISGPU_TAP_ROT || (channel & 1))) {
		h->err = "single-channel mode has no Rotate and no channel 1";
		return AISGPU_EINVAL;
	}
	if (h->disc && tap == AISGPU_TAP_ROT) {
		h->err = "the FM discriminator model has no Rotate";
		return AISGPU_EINVAL;
	}
	if (h->member && (tap == AISGPU_TAP_ROT || tap == AISGPU_TAP_PRE || tap == AISGPU_TAP_PRE2)) {
		h->err = "a group member has no front end: read the front-end taps from the group's leader";
		return AISGPU_EINVAL;
	}
	const int row = row_of(h, stream, channel & 1);
	const void *src = nullptr;
	size_t n = 0, esz = 8;
	switch (tap) {
	case AISGPU_TAP_C:
		src = h->d_C2[h->c_last] + (long long)row * h->c_stride + HC; // note: valid until the next submit only for [0, n48)
		n = h->last_n48;
		if (h->disc) esz = 4; // real rows
		break;
	case AISGPU_TAP_CGF:
		if (!h->d_tap_cgf) { h->err = "taps not enabled or not a ModelDefault engine"; return AISGPU_EINVAL; }
		src = h->d_tap_cgf + (long long)row * h->r_stride;
		n = h->last_nE;
		break;
	case AISGPU_TAP_FIR: // the filter in front of the symbol stage: FIR17 (V2, ModelDefault), or Filter 37 of the FM chain and of ModelChallenger's FM branch
		if (h->chain == Chain::V2) {
			if (!h->d_tap_coh) { h->err = "taps not enabled"; return AISGPU_EINVAL; }
			src = h->d_tap_coh + (long long)row * h->r_stride;
		}
		else if (h->cfg.model == AISGPU_MODEL_DEFAULT) src = h->d_Ec2[h->ec_last] + (long long)row * h->e_stride + HE;
		else {
			if (!h->cfg.enable_taps && h->cfg.model != AISGPU_MODEL_BASE) { h->err = "taps not enabled"; return AISGPU_EINVAL; } // the FIR37 output is not stored then
			src = h->d_Ef + (long long)row * h->e_stride + HE;
			esz = 4;
		}
		n = h->last_nE;
		break;
	case AISGPU_TAP_ROT:
		CU(cudaStreamSynchronize(h->side_stream));
		src = h->d_rot[h->rot_cur] + h->P96;
		n = h->rot_n96[h->rot_cur];
		break;
	case 4: { // decoder input of sampling phase (channel / 2): channel = ch + 2 * phase
		if (!h->d_tap_dec) { h->err = "taps not enabled"; return AISGPU_EINVAL; }
		const int phase = channel >> 1;
		esz = 4;
		if (h->cfg.model == AISGPU_MODEL_BASE) {
			int cnt = 0;
			CU(cudaMemcpy(&cnt, h->d_tap_cnt + row, sizeof(int), cudaMemcpyDeviceToHost));
			src = h->d_tap_dec + (long long)row * h->last_nE;
			n = cnt;
		}
		else {
			src = h->d_tap_dec + (long long)(row * 5 + phase) * h->last_nsym;
			n = h->last_nsym;
			if (standard_tail(h)) { // samples of this phase among the last submit's [a0, a1)
				const long long a1 = h->e_abs, a0 = a1 - h->last_nE;
				n = 0;
				for (long long a = a0; a < a1; a++) n += (a % 5) == phase;
			}
		}
		break;
	}
	case AISGPU_TAP_PRE:
	case AISGPU_TAP_PRE2: { // what the resampler in front of the decimation chain produced in the last submit (stream, channel ignored):
		// PRE the first resampler stage (Upsample, else DSK), PRE2 the DSK behind Upsample
		const bool second = tap == AISGPU_TAP_PRE2;
		const PreRing *r = h->pre_us ? (second ? &h->dsk_ring : &h->us_ring) : (second ? nullptr : &h->dsk_ring);
		if (!r || !r->d || r->cap <= 0) { h->err = "this rate has no resampler stage"; return AISGPU_EINVAL; }
		const int cap = r->cap;
		const long long a = r->last;
		size_t cnt = (size_t)std::min<long long>(r->produced - a, cap);
		if (dst_bytes < cnt * 8) cnt = dst_bytes / 8;
		for (size_t i = 0; i < cnt;) { // the ring may wrap
			const size_t off = (size_t)((a + (long long)i) % cap), run = std::min(cnt - i, (size_t)cap - off);
			if (dst) CU(cudaMemcpy((float2 *)dst + i, r->d + (long long)stream * r->stride + off, run * 8, cudaMemcpyDeviceToHost));
			i += run;
		}
		*n_out = cnt;
		return 0;
	}
	case 6: // debug counters of the decoder kernel, 4 x int64 per row (stream/channel ignored, all rows)
		if (!h->d_dbg) { h->err = "AISGPU_DEBUG not set"; return AISGPU_EINVAL; }
		src = h->d_dbg;
		n = (size_t)h->rows * 4;
		break;
	case 5:
		if (!h->d_tap_fm) { h->err = "taps not enabled or not an FM engine"; return AISGPU_EINVAL; }
		src = h->d_tap_fm + (long long)row * h->r_stride;
		n = h->last_nE;
		esz = 4;
		break;
	default:
		h->err = "unknown tap";
		return AISGPU_EINVAL;
	}
	if (dst_bytes < n * esz) n = dst_bytes / esz;
	if (n && dst) CU(cudaMemcpy(dst, src, n * esz, cudaMemcpyDeviceToHost));
	*n_out = n;
	return 0;
}

int aisgpu_counters(aisgpu_handle *h, uint64_t counters[8]) {
	if (!h || !counters) return AISGPU_EINVAL;
	memcpy(counters, h->counters, sizeof(h->counters));
	return 0;
}

// ---- NCCL, resolved at run time: the counters are the only thing that ever crosses NVLink (SURVEY.md 8e) ----
namespace {
struct nccl_uid { char internal[128]; };
struct NcclApi {
	void *lib = nullptr;
	int (*GetUniqueId)(nccl_uid *) = nullptr;
	int (*CommInitRank)(void **, int, nccl_uid, int) = nullptr;
	int (*AllReduce)(const void *, void *, size_t, int, int, void *, cudaStream_t) = nullptr;
	int (*CommDestroy)(void *) = nullptr;
	const char *(*GetErrorString)(int) = nullptr;
};
NcclApi *nccl_api(std::string &err) {
	static NcclApi api;
	static bool tried = false;
	if (!tried) {
		tried = true;
		const char *names[] = { "libnccl.so.2", "libnccl.so" };
		for (const char *nm : names)
			if ((api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL))) break;
		if (api.lib) {
			api.GetUniqueId = (int (*)(nccl_uid *))dlsym(api.lib, "ncclGetUniqueId");
			api.CommInitRank = (int (*)(void **, int, nccl_uid, int))dlsym(api.lib, "ncclCommInitRank");
			api.AllReduce = (int (*)(const void *, void *, size_t, int, int, void *, cudaStream_t))dlsym(api.lib, "ncclAllReduce");
			api.CommDestroy = (int (*)(void *))dlsym(api.lib, "ncclCommDestroy");
			api.GetErrorString = (const char *(*)(int))dlsym(api.lib, "ncclGetErrorString");
			if (!api.GetUniqueId || !api.CommInitRank || !api.AllReduce || !api.CommDestroy) {
				dlclose(api.lib);
				api.lib = nullptr;
			}
		}
	}
	if (!api.lib) {
		err = "NCCL not found (dlopen libnccl.so.2)";
		return nullptr;
	}
	return &api;
}
} // namespace

int aisgpu_nccl_unique_id(void *id128) {
	if (!id128) return AISGPU_EINVAL;
	NcclApi *api = nccl_api(g_create_error);
	if (!api) return AISGPU_ENODEV;
	nccl_uid id;
	if (int rc = api->GetUniqueId(&id)) {
		g_create_error = std::string("ncclGetUniqueId: ") + (api->GetErrorString ? api->GetErrorString(rc) : "error");
		return AISGPU_ECUDA;
	}
	memcpy(id128, &id, sizeof(id));
	return 0;
}

int aisgpu_comm_init(aisgpu_handle *h, const void *id128, int n_ranks, int rank) {
	if (!h || !id128 || n_ranks < 1 || rank < 0 || rank >= n_ranks) return AISGPU_EINVAL;
	CU(cudaSetDevice(h->cfg.device));
	NcclApi *api = nccl_api(h->err);
	if (!api) return AISGPU_ENODEV;
	if (h->nccl_comm) {
		api->CommDestroy(h->nccl_comm);
		h->nccl_comm = nullptr;
	}
	nccl_uid id;
	memcpy(&id, id128, sizeof(id));
	if (int rc = api->CommInitRank(&h->nccl_comm, n_ranks, id, rank)) {
		h->err = std::string("ncclCommInitRank: ") + (api->GetErrorString ? api->GetErrorString(rc) : "error");
		h->nccl_comm = nullptr;
		return AISGPU_ECUDA;
	}
	return 0;
}

int aisgpu_allreduce_counts(aisgpu_handle *h, uint64_t totals[8]) {
	if (!h || !totals) return AISGPU_EINVAL;
	CU(cudaSetDevice(h->cfg.device));
	if (!h->nccl_comm) { // a single engine is its own job
		memcpy(totals, h->counters, sizeof(h->counters));
		return 0;
	}
	NcclApi *api = nccl_api(h->err);
	if (!api) return AISGPU_ENODEV;
	CU(cudaMemcpyAsync(h->d_counts, h->counters, 8 * sizeof(uint64_t), cudaMemcpyHostToDevice, h->stream));
	if (int rc = api->AllReduce(h->d_counts, h->d_counts + 8, 8, /*ncclUint64*/ 5, /*ncclSum*/ 0, h->nccl_comm, h->stream)) {
		h->err = std::string("ncclAllReduce: ") + (api->GetErrorString ? api->GetErrorString(rc) : "error");
		return AISGPU_ECUDA;
	}
	CU(cudaMemcpyAsync(totals, h->d_counts + 8, 8 * sizeof(uint64_t), cudaMemcpyDeviceToHost, h->stream));
	CU(cudaStreamSynchronize(h->stream));
	return 0;
}

void *aisgpu_cuda_stream(aisgpu_handle *h) { return h ? (void *)h->stream : nullptr; }

int aisgpu_join(aisgpu_handle *h) {
	if (!h) return AISGPU_EINVAL;
	if (h->be_streams[1] != h->be_streams[0]) {
		CU(cudaEventRecord(h->ev_join, h->be_streams[1]));
		CU(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
	}
	for (aisgpu_handle *m : h->members) // the event is captured by each wait, so one serves every back-end stream of the group
		for (int i = 0; i < (m->be_streams[1] != m->be_streams[0] ? 2 : 1); i++) {
			CU(cudaEventRecord(h->ev_join, m->be_streams[i]));
			CU(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
		}
	if (h->dump_stream) { // the copies of the channel dump
		CU(cudaEventRecord(h->ev_join, h->dump_stream));
		CU(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
	}
	return 0;
}

float aisgpu_last_frontend_ms(aisgpu_handle *h) {
	float ms = -1.0f;
	int n = 0;
	if (aisgpu_frontend_times(h, &ms, 1, &n) || n != 1) return -1.0f;
	return ms;
}

int aisgpu_frontend_times(aisgpu_handle *h, float *ms_out, int max, int *n) {
	if (!h || !ms_out || !n) return AISGPU_EINVAL;
	*n = 0;
	if (!h->fe_timed) return 0;
	CU(cudaStreamSynchronize(h->fe_stream));
	if (int rc = sync_backend(h)) return rc;
	long long cnt = std::min<long long>(std::min<long long>(h->chunk, aisgpu_handle::NEV), max);
	for (long long i = 0; i < cnt; i++) { // newest first
		const int evi = (int)((h->chunk - 1 - i) % aisgpu_handle::NEV);
		CU(cudaEventElapsedTime(&ms_out[i], h->ev_fe0s[evi], h->ev_fe1s[evi]));
	}
	*n = (int)cnt;
	return 0;
}

int aisgpu_last_launches(aisgpu_handle *h) { return h ? h->last_launches : 0; }

int aisgpu_chunk_granule(const aisgpu_config *cfg) {
	aisgpu_config c;
	if (!copy_config(cfg, &c)) {
		g_create_error = "aisgpu_chunk_granule: null argument or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	aisgpu_handle tmp;
	tmp.cfg = c;
	if (int rc = plan_frontend(&tmp)) {
		g_create_error = tmp.err;
		return rc;
	}
	return outer_granule(&tmp);
}

int aisgpu_check_device_batch(const aisgpu_config *cfg, const void *dev_samples, int64_t stride_samples) {
	aisgpu_config c;
	if (!copy_config(cfg, &c) || !dev_samples) {
		g_create_error = "aisgpu_check_device_batch: null argument or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	if (!format_known(c.format) || c.n_streams < 1) {
		g_create_error = "bad format / n_streams";
		return AISGPU_EINVAL;
	}
	aisgpu_handle tmp;
	tmp.cfg = c;
	int rc = plan_frontend(&tmp);
	if (!rc) rc = check_placement(&tmp, dev_samples, stride_samples);
	if (rc) g_create_error = tmp.err;
	return rc;
}

// The rule of aisgpu_attach on two caller configs: every field the front end reads is equal, and neither engine is the
// FM-discriminator input model (its front end is the I/Q split, not the CIC chain the others share).
static int check_attach_cfg(const aisgpu_config &L, const aisgpu_config &M, std::string &err) {
	const struct {
		const char *name;
		long long a, b;
	} fields[] = { { "sample_rate", L.sample_rate, M.sample_rate }, { "format", L.format, M.format }, { "n_streams", L.n_streams, M.n_streams },
				   { "max_chunk_samples", L.max_chunk_samples, M.max_chunk_samples }, { "channel_mode", L.channel_mode, M.channel_mode },
				   { "droop", L.droop, M.droop }, { "dsk", L.dsk, M.dsk }, { "fp_ds", L.fp_ds, M.fp_ds }, { "device", L.device, M.device } };
	for (const auto &f : fields)
		if (f.a != f.b) {
			err = std::string("aisgpu_attach: ") + f.name + " differs from the leader's (a group shares the leader's front end)";
			return AISGPU_EINVAL;
		}
	if (L.model == AISGPU_MODEL_DISCRIMINATOR || M.model == AISGPU_MODEL_DISCRIMINATOR) {
		err = std::string("aisgpu_attach: the FM discriminator model cannot be in a group (as the ") +
			  (L.model == AISGPU_MODEL_DISCRIMINATOR ? "leader)" : "member)");
		return AISGPU_EINVAL;
	}
	return 0;
}

int aisgpu_check_attach(const aisgpu_config *leader, const aisgpu_config *member) {
	aisgpu_config l, m;
	if (!copy_config(leader, &l) || !copy_config(member, &m)) {
		g_create_error = "aisgpu_check_attach: null argument or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	return check_attach_cfg(l, m, g_create_error);
}

int aisgpu_attach(aisgpu_handle *leader, const aisgpu_config *cfg, aisgpu_handle **out) {
	aisgpu_config c;
	if (!leader || !out || !copy_config(cfg, &c)) {
		g_create_error = "aisgpu_attach: null argument or struct_size mismatch";
		return AISGPU_EINVAL;
	}
	*out = nullptr;
	if (leader->poisoned) {
		g_create_error = "aisgpu_attach: the leader has failed: " + leader->err;
		return leader->poisoned;
	}
	if (int rc = check_attach_cfg(leader->given, c, g_create_error)) return rc;
	if (leader->member) {
		g_create_error = "aisgpu_attach: a member cannot lead a group";
		return AISGPU_EINVAL;
	}
	if (leader->counters[3] != 0) {
		g_create_error = "aisgpu_attach: the leader has already been submitted to (attach every member before the first submit)";
		return AISGPU_EINVAL;
	}
	if ((int)leader->members.size() + 1 >= GROUP_MAX) {
		g_create_error = "aisgpu_attach: a group holds at most 8 engines";
		return AISGPU_EINVAL;
	}
	if (cudaSetDevice(leader->cfg.device) != cudaSuccess || (!leader->ev_fan && new_event(leader, &leader->ev_fan) != cudaSuccess)) {
		(void)cudaGetLastError();
		g_create_error = "aisgpu_attach: CUDA event creation failed";
		return AISGPU_ECUDA;
	}
	aisgpu_handle *h = new aisgpu_handle();
	h->cfg = c;
	h->given = c;
	h->member = true;
	int rc = create_impl(h);
	if (!rc && (h->rows != leader->rows || h->c_stride != leader->c_stride || h->inner_max != leader->inner_max)) {
		h->err = "internal: a member's 48 kHz rows differ from its leader's";
		rc = AISGPU_EINVAL;
	}
	if (rc) {
		g_create_error = h->err;
		aisgpu_destroy(h);
		return rc;
	}
	h->leader = leader;
	h->clock = leader->clock; // a clock set before the attach (one set after it reaches the member through the leader)
	leader->members.push_back(h);
	*out = h;
	return 0;
}

static int dump_refuse(aisgpu_handle *h, const char *why) {
	h->err = std::string("aisgpu_dump_open: ") + why;
	return AISGPU_EINVAL;
}

int aisgpu_dump_open(aisgpu_handle *h, const char *const *prefixes) {
	ENTER(h);
	if (!prefixes) return dump_refuse(h, "null prefix array");
	if (h->member) return dump_refuse(h, "a group member has no front end of its own (dump the group's leader)");
	if (h->cfg.model == AISGPU_MODEL_DISCRIMINATOR) return dump_refuse(h, "the FM-discriminator input model has no 48 kHz channel dump (ModelDiscriminator refuses the key)");
	if (h->xmode) return dump_refuse(h, "single-channel mode writes no channel dump (the reference wires none in mode X)");
	if (h->dump) return dump_refuse(h, "a dump is already open");
	if (h->counters[3] != 0) return dump_refuse(h, "the engine has already been submitted to (open the dump before the first submit)");
	// the most 48 kHz samples per row one submit can yield: whole blocks of the last pre-stage ring (< one block left over plus what
	// one submit adds, within the ring's capacity) times a block's samples, or one submit's without a pre-stage
	const long long nblk = h->pre_dsk ? h->dsk_ring.cap / h->blk : (h->pre_us ? h->us_ratio + 2 : 1);
	const long long cap = nblk * h->max_n48;
	if (!h->dump_stream) {
		CU(cudaStreamCreateWithFlags(&h->dump_stream, cudaStreamNonBlocking));
		CU(new_event(h, &h->ev_export));
		for (int i = 0; i < aisgpu_handle::ND; i++) {
			if (int rc = dalloc(h, &h->d_dump[i], (size_t)h->rows * cap)) return rc;
			if (int rc = halloc(h, &h->pin_dump[i], (size_t)h->rows * cap)) return rc;
			CU(new_event(h, &h->ev_dump[i]));
		}
		CU(cudaStreamSynchronize(h->stream)); // dalloc clears on h->stream
		h->dump_cap = cap;
	}
	h->dump = new aisgpu::ChannelDump(prefixes, h->cfg.n_streams);
	return 0;
}

int aisgpu_dump_close(aisgpu_handle *h) {
	if (!h) return AISGPU_EINVAL;
	if (!h->dump) return 0;
	CU(cudaSetDevice(h->cfg.device));
	const int rc = h->poisoned ? h->poisoned : dump_write(h, -1); // a poisoned engine's slots are not trusted: close with what was written
	h->dump_pending.clear();
	const bool ok = h->dump->close();
	if (!ok) h->err = h->dump->error();
	delete h->dump;
	h->dump = nullptr;
	return rc ? rc : (ok ? 0 : AISGPU_EIO);
}

int aisgpu_validate(const uint8_t *data, int nbits) {
	if (!data || nbits < 0) return 0;
	return msg_validate(data, nbits) ? 1 : 0;
}

int aisgpu_build_nmea(aisgpu_msg *m, int own_mmsi, int *seq) {
	if (!m || !seq || m->nbits < 0 || m->nbits > 1064 || *seq < 0 || *seq > 9) return AISGPU_EINVAL;
	build_nmea(*m, own_mmsi, seq);
	return 0;
}

void aisgpu_destroy(aisgpu_handle *h) {
	if (!h) return;
	if (h->dump) aisgpu_dump_close(h);
	if (h->leader) { // detach: the leader's fe_stream may still be writing this member's rows
		cudaSetDevice(h->leader->cfg.device);
		cudaStreamSynchronize(h->leader->fe_stream);
		auto &v = h->leader->members;
		v.erase(std::remove(v.begin(), v.end(), h), v.end());
		h->leader = nullptr;
	}
	if (h->fe_stream) cudaStreamSynchronize(h->fe_stream);
	for (aisgpu_handle *m : h->members) { // their back ends were waiting on this engine's front end
		cudaStreamSynchronize(m->be_streams[0]);
		if (m->be_streams[1] != m->be_streams[0]) cudaStreamSynchronize(m->be_streams[1]);
		m->leader = nullptr;
		if (!m->poisoned) m->poisoned = AISGPU_EINVAL;
		m->err = "the group's leader was destroyed (destroy the members first)";
	}
	if (h->stream) cudaStreamSynchronize(h->stream);
	if (h->be_streams[1] && h->be_streams[1] != h->stream) { cudaStreamSynchronize(h->be_streams[1]); cudaStreamDestroy(h->be_streams[1]); }
	if (h->nccl_comm) {
		std::string e;
		if (NcclApi *api = nccl_api(e)) api->CommDestroy(h->nccl_comm);
	}
	if (h->copy_stream) cudaStreamSynchronize(h->copy_stream);
	if (h->side_stream) cudaStreamSynchronize(h->side_stream);
	if (h->dump_stream) cudaStreamSynchronize(h->dump_stream);
	if (h->json_stream) {
		cudaStreamSynchronize(h->json_stream);
		cudaStreamDestroy(h->json_stream);
	}
	for (void *p : h->dev_mem) cudaFree(p);
	for (void *p : h->host_mem) cudaFreeHost(p);
	for (cudaEvent_t e : h->events) cudaEventDestroy(e);
	if (h->side_stream) cudaStreamDestroy(h->side_stream);
	if (h->fe_stream) cudaStreamDestroy(h->fe_stream);
	if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
	if (h->dump_stream) cudaStreamDestroy(h->dump_stream);
	if (h->stream) cudaStreamDestroy(h->stream);
	delete h;
}

} // extern "C"
