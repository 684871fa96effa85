/* aisgpu.h -- C ABI of the H100-native AIS demodulation engine.
 *
 * Drop-in boundary for ONE hot path of jvde-github/AIS-catcher: raw IQ ->
 * decimate -> +/-25 kHz channelise -> (CGF, FIR, coherent phase search | FM
 * discriminator, FIR) -> 5-phase symbol timing -> NRZI/HDLC/CRC -> AIS frames
 * (reference Source/DSP/Model.cpp:27-356 ModelFrontend, :419-438 ModelBase,
 * :484-518 ModelStandard, :520-577 ModelDefault; Source/Marine/AIS.h:91-181),
 * run over a batch of independent IQ streams on one GPU.
 *
 * The reference has no FFI for this path (it is a C++ class graph wired with
 * operator>>, Source/Library/Stream.h:136-167); what a maintainer binds is one
 * more AIS::Model subclass (Source/DSP/Model.h:76-126) whose buildModel()
 * connects the device's Connection<RAW> to a sink that forwards every RAW block
 * to aisgpu_submit() and publishes the frames returned by aisgpu_poll() through
 * the inherited Util::PassThrough<Message> output.  That adapter is
 * ais-catcher_b200/host/ModelGPU.h; INTEGRATION.md shows the three registration
 * edits.  Every entry point below cites the reference interface it stands for.
 *
 * Conventions: all functions return 0 on success, a negative AISGPU_E* code on
 * failure (never throw, never abort); aisgpu_last_error() gives the text.  The
 * caller's thread model is the reference's: one thread per handle
 * (Source/Device/FileRAW.cpp:205-206).  There is NO CPU fallback: without a
 * CUDA device aisgpu_create() fails with AISGPU_ENODEV.
 */
#ifndef AISGPU_H
#define AISGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* 3 since the engine groups; later additions are new entry points only (the full AIS JSON: aisgpu_msg_json_full, aisgpu_json_enable,
 * aisgpu_poll_json; the output records: aisgpu_msg_format, aisgpu_lines_enable, aisgpu_poll_lines; the receivers:
 * aisgpu_set_receivers, aisgpu_check_receivers; the tuning: aisgpu_set_tuning, aisgpu_check_tuning, aisgpu_tune_restate; the
 * tunings of one input: aisgpu_set_tunings, aisgpu_check_tunings; the receive time: aisgpu_set_clock, aisgpu_check_clock, aisgpu_stamp), so the number callers check against stays 3.  A caller that
 * needs those entry points looks them up (dlsym) instead of relying on the number. */
#define AISGPU_ABI_VERSION 3

/* model kinds: the reference's "-m" numbers (Source/Application/Receiver.cpp:155-195) */
#define AISGPU_MODEL_STANDARD 0 /* FM -> FIR37 -> 5-phase deinterleave -> 5 decoders (Model.cpp:484-518) */
#define AISGPU_MODEL_BASE 1     /* FM -> FIR37 -> SimplePLL -> 1 decoder            (Model.cpp:419-438) */
#define AISGPU_MODEL_DEFAULT 2  /* CGF -> FIR17 -> 5 x PhaseSearch[EMA] -> 5 decoders (Model.cpp:520-577) */
#define AISGPU_MODEL_CHALLENGER 4 /* CGF -> { FIR17 -> 5 x PhaseSearchEMA | FM -> FIR37 } -> 10 cross-reset decoders (Model.cpp:601-678) */
#define AISGPU_MODEL_V2 11      /* V2::Engine per channel: slot-predicted CGF, 5 PhaseTrackers + FM/BitPLL, 6 decoders (Model.cpp:440-460,
                                   DSP/Decoder/V2/V2Engine.cpp) */
#define AISGPU_MODEL_DISCRIMINATOR 3 /* FM-discriminator input (ModelDiscriminator, Model.cpp:702-754): I and Q are the audio of two
                                        discriminator taps (channel A, channel B); each goes through FIR37 -> 5-phase deinterleave ->
                                        5 decoders.  12000..48000 S/s, see below. */

/* AISGPU_MODEL_DISCRIMINATOR: the stereo recording of two VHF receivers' discriminator outputs, read as I/Q (a stereo WAV is CS16,
 * CU8 or CF32, Device/FileWAV.cpp:84-95).  Real part -> Filter 37 -> channel_a, imaginary part -> Filter 37 -> channel_b.  Rates below
 * 48000 go through DSP::Upsample to 48 kHz (Model.cpp:722-728).  Above 48000 aisgpu_create fails with the reference's "Internal
 * error: sample rate not supported in FM discriminator model."; below 12000 it fails as well, which the reference does not do: the
 * Upsample stage here holds ratios up to 4, and below 12 kS/s a 9600 Bd symbol has fewer than 1.25 input samples.  AB and X
 * channel_mode build the same two-channel chain (the model ignores the channel mode); droop, dsk, fp_ds, ps_ema and afc_wide are
 * ignored.  The granule is 64 samples at every rate and format.  Taps: AISGPU_TAP_C is the real 48 kHz row of the channel (float,
 * 4-byte elements), AISGPU_TAP_FIR the Filter 37 output, AISGPU_TAP_PRE the Upsample output (float2, both channels), tap 4 the
 * per-phase decoder input; AISGPU_TAP_ROT, AISGPU_TAP_CGF and AISGPU_TAP_PRE2 are AISGPU_EINVAL. */

/* input sample formats: the formats of enum class Format (Source/Library/Common.h:89-104) that ConvertRAW takes */
#define AISGPU_FMT_CF32 0
#define AISGPU_FMT_CU8 1
#define AISGPU_FMT_CS8 2
#define AISGPU_FMT_CS16 3
/* Format::F32_FS4 (ConvertRAW, Source/Utilities/StreamHelpers.cpp:105-118): ONE real float per sample, 4 bytes, made complex by the
 * fs/4 shift 1, j, -1, -j -- sample n of a Receive becomes (x, 0), (0, x), (-x, 0), (0, -x) for n % 4 = 0 .. 3.  It is what the Airspy
 * and HydraSDR devices deliver in real mode (-gm REAL_MODE on, Device/AIRSPY.cpp:112-116, 292-298; Device/HYDRASDR.cpp:117, 300)
 * and what -gr FORMAT F32_FS4 reads from a recording (Utilities/Parse.cpp:186).  sample_rate is the rate of the real samples: one
 * real sample gives one complex sample, and the rate -> chain table, the granules and every mode and model apply unchanged
 * (AISGPU_MODEL_DISCRIMINATOR reads the real / imaginary parts of the expanded samples like ModelDiscriminator's own ConvertRAW).
 * The pattern restarts with every submit; every granule is a multiple of 4, so a sample's place in it is its index in the submit
 * modulo 4.  A submit of n_samples is n_samples floats per stream. */
#define AISGPU_FMT_F32_FS4 4
/* Format::DC16H (typedef uint32_t DC16H[3], Source/Library/Common.h:87; Convert::toFloat, Source/Utilities/Convert.cpp:288-301):
 * THREE 32-bit words per sample, 12 bytes.  I is the sign-extended low 16 bits of word 0, Q the sign-extended low 16 bits of word 1;
 * the high halves of both and the whole of word 2 are never read.  re = I / 32768, im = (-Q) / 32768 with Q negated as a 32-bit
 * integer before the division: Q = 0 gives +0.0f (never -0.0f) and Q = -32768 gives exactly 1.0f.  It is what -gr FORMAT DC16H reads
 * from a recording (Utilities/Parse.cpp:188-189); ConvertRAW takes size / 12 samples of a buffer and drops the bytes short of one
 * (StreamHelpers.cpp:120-126).  sample_rate is the rate of the complex samples; the rate -> chain table, the granules and every
 * mode, model and switch apply unchanged, FP_DS as for CS16 and CF32 (the integer CIC stages take CU8 only, Model.cpp:231-237).
 * A submit of n_samples is 3 * n_samples words per stream.  aisgpu_wav_probe never returns it (no WAV layout maps to it).
 * Its value is 7: 5 and 6 are not formats and stay AISGPU_EINVAL ("bad format"), the answer callers have always had for them. */
#define AISGPU_FMT_DC16H 7

#define AISGPU_OK 0
#define AISGPU_EINVAL -1   /* bad argument / unsupported configuration (reference: std::runtime_error at buildModel, Model.cpp:109-110) */
#define AISGPU_ENODEV -2   /* no usable CUDA device */
#define AISGPU_ECUDA -3    /* CUDA runtime error; adapter converts to Error()<<...; StopRequest() (FileRAW.cpp:111-115) */
#define AISGPU_ENOMEM -4   /* device or pinned-host allocation failed */
#define AISGPU_EOVERFLOW -5 /* returned by aisgpu_poll*(): the frame ring overflowed since the last poll and frames were dropped; the frames
                              that survived were still delivered (out / *n are valid).  Size the ring with aisgpu_config.max_frames. */
#define AISGPU_EIO -6      /* a channel dump file (aisgpu_dump_open) could not be created or written */

/* tap ids for aisgpu_tap(): intermediates for parity tests */
#define AISGPU_TAP_C 0     /* 48 kHz channel samples after FilterCIC5 (Model.cpp:345-346 C_a/C_b), float2; AISGPU_MODEL_DISCRIMINATOR:
                              the real 48 kHz samples of the channel (RealPart / ImaginaryPart), float */
#define AISGPU_TAP_CGF 1   /* after SquareFreqOffsetCorrection (DSP.cpp:475-489), float2, whole 512-blocks of this submit */
#define AISGPU_TAP_FIR 2   /* after FilterComplex (ModelDefault, float2) or Filter (FM models, float) */
#define AISGPU_TAP_ROT 3   /* the Rotate phasor table of the last submit (DSP.cpp:296-316), float2 */
#define AISGPU_TAP_PRE 7   /* resampled rates: output of DSP::Upsample (or of DownsampleKFilter when there is no Upsample) in the last submit */
#define AISGPU_TAP_PRE2 8  /* Upsample -> DownsampleKFilter rates: the /3 filter's output in the last submit */

typedef struct aisgpu_config {
	uint32_t struct_size;       /* = sizeof(aisgpu_config) */
	int32_t model;              /* AISGPU_MODEL_*                                   (Receiver.cpp:155-195) */
	int32_t sample_rate;        /* 96000..12288000 (X mode: 12000..192000; AISGPU_MODEL_DISCRIMINATOR: 12000..48000); non-bucket rates are upsampled, 288000 is /3-filtered (Model.cpp:109-149, 308-313) */
	int32_t format;             /* AISGPU_FMT_*                                      (Common.h:290-295 RAW.format) */
	int32_t n_streams;          /* batch of independent IQ streams, >= 1 */
	int32_t max_chunk_samples;  /* upper bound of n_samples per stream per submit */
	int32_t ps_ema;             /* -go PS_EMA   (Model.cpp:583-585), default 1 */
	int32_t afc_wide;           /* -go AFC_WIDE (Model.cpp:586-588), default 1 */
	int32_t droop;              /* -go DROOP    (Model.cpp:384-386), default 1 */
	char channel_a, channel_b;  /* CH1/CH2 of buildModel (Model.cpp:547-548), default 'A','B' (a receiver table overrides: aisgpu_set_receivers) */
	int32_t station;            /* Model::station  (Model.h:79) (a receiver table overrides) */
	int32_t own_mmsi;           /* Model::own_mmsi (Model.h:80): sentences of this MMSI read !AIVDO (a receiver table overrides) */
	uint32_t tag_mode;          /* TAG::mode (Common.h:242): bit0 = signal level, default 3 (a receiver table overrides) */
	int32_t device;             /* CUDA device ordinal */
	int32_t enable_taps;        /* keep intermediates readable through aisgpu_tap() */
	int32_t max_frames;         /* capacity of the device frame ring = frames that may wait between two polls (0 = default) */
	int32_t host_staging;       /* 1 (default): the device staging buffers behind aisgpu_submit*() are allocated by aisgpu_create;
	                               0: at the first host submit (engines that are only fed with aisgpu_submit_device) */
	int32_t dsk;                /* -go DSK   (Model.cpp:377-379): adds the 576K / 1152K / 2304K buckets (CIC stages -> /3 filter), default 0 */
	int32_t fp_ds;              /* -go FP_DS (Model.cpp:362-365): integer CIC stages for CU8 input at exactly 1536000 (DSP.cpp:499-665), default 0 */
	float dd_train, dd_weight;  /* -go DD_TRAIN / DD_WEIGHT of the V2 engine (Model.cpp:462-474; Model.h:272), defaults 0.75 / 0.86 */
	int32_t channel_mode;       /* AISGPU_MODE_AB (default) or AISGPU_MODE_X (Model::setMode, Model.h:104); added after dd_weight:
	                               a caller that passes struct_size == offsetof(aisgpu_config, channel_mode) gets AB */
} aisgpu_config;

/* channel modes: the values of AIS::Mode (Model.h:41-47).  AB also serves CD: the reference builds the same chain for both and
 * only the channel letters (channel_a / channel_b) and the tuning differ.
 * AISGPU_MODE_X: single-channel mode (-c X, Model.cpp:35-107).  Each stream is a complex baseband stream already centred on one AIS
 * channel at 12000..192000 S/s; rates other than 48K / 96K / 192K are upsampled to the next of them (DSP::Upsample).  The chain
 * is K x Downsample2CIC5 -> [FilterComplex3Tap at 48 kHz when droop is on and K > 0] -> FilterCIC5, one channel per stream whose
 * frames carry channel_a; channel_b, dsk and fp_ds are ignored, AISGPU_TAP_ROT and taps of channel 1 are AISGPU_EINVAL.  The
 * granule is 64 samples at every rate and format (one 128-byte chunk of the byte formats' front-end lanes), and a device batch
 * (aisgpu_submit_device) must have 16-byte aligned rows. */
#define AISGPU_MODE_AB 0
#define AISGPU_MODE_X 3

/* One decoded frame == one AIS::Message the reference would Send (Source/Marine/AIS.cpp:66-96). */
typedef struct aisgpu_msg {
	int32_t stream;             /* index in the batch */
	char channel;               /* Message::channel (Message.h:300-305) */
	int32_t nbits;              /* Message::getLength() */
	int64_t start_idx, end_idx; /* Message::start_idx/end_idx: 48 kHz symbol-sample counters (AIS.h:112,151) */
	float level;                /* TAG::level in dB (AIS.cpp:74-75) */
	float ppm;                  /* TAG::ppm   (DSP.cpp:484) */
	int64_t chunk;              /* ordinal of the submit that completed the frame */
	uint8_t data[140];          /* Message::data (Message.h:69), payload bytes, MSB-first fields */
	int32_t n_sentences;        /* Message::sentences().size() */
	char nmea[4][100];          /* NUL-terminated !AIVDM sentences (Message.cpp:569-631) */
	int32_t nmea_len[4];        /* their lengths: the last letter of a 1064-bit message is a NUL byte in the reference
	                               (Message::getLetter returns 0 when the letter crosses bit 1064, Message.cpp:646-647) */
} aisgpu_msg;

typedef struct aisgpu_handle aisgpu_handle;

/* Fills *cfg with the reference's defaults (Model.h:218-222, 138-143; Common.h:242). */
void aisgpu_default_config(aisgpu_config *cfg);

/* == AIS::Model::buildModel(CH1, CH2, sample_rate, timerOn, device) (Model.h:94, Model.cpp:27,520).  cfg->struct_size is
 * sizeof(aisgpu_config), or offsetof(aisgpu_config, channel_mode) for callers built before that field existed (AB mode). */
int aisgpu_create(const aisgpu_config *cfg, aisgpu_handle **out);

/* Checks the rate -> chain table of ModelFrontend::buildModel (Model.cpp:35-338) without touching the GPU and returns
 * the granule every n_samples passed to aisgpu_submit must be a multiple of (> 0), or AISGPU_EINVAL with the
 * reference's wording in aisgpu_last_error(NULL).  AB: 2^(CIC stages + 2) input samples; X: 64.  cfg->struct_size may be
 * sizeof(aisgpu_config) or offsetof(aisgpu_config, channel_mode), as for aisgpu_create. */
int aisgpu_chunk_granule(const aisgpu_config *cfg);

/* == StreamIn<RAW>::Receive(const RAW*, 1, TAG&) for every stream of the batch (Stream.h:41; Model.cpp:33).
 * host_samples: n_streams contiguous runs of n_samples samples (stream-major), borrowed for the call only (the call
 * returns when the host-to-device copy into the engine's staging buffer has completed; the kernels run
 * asynchronously).  n_samples must be a multiple of aisgpu_chunk_granule() -- every CIC stage needs an even block
 * (DSP.cpp:94,135 assert(len%2==0)) -- and, at rates the reference serves through DSP::Upsample, the same for every
 * call (Upsample re-blocks by the length of its input block, DSP.cpp:203).  Pinned host memory gives full PCIe speed.
 * After a CUDA failure inside a submit the handle is poisoned: every later call returns the stored error. */
int aisgpu_submit(aisgpu_handle *h, const void *host_samples, int n_samples);

/* Same, one host pointer per stream: stream_ptrs[s] -> n_samples samples of stream s.  This is the shape the reference's
 * receivers deliver -- every device thread hands its own FIFO block to Receive (RAW.data, Common.h:290-295;
 * FileRAW.cpp:132-136) -- so n_streams independent receivers need no repacking on the host. */
int aisgpu_submit_v(aisgpu_handle *h, const void *const *stream_ptrs, int n_samples);

/* Asynchronous form of aisgpu_submit for callers that own (at least two) pinned buffers: enqueues the host-to-device copy
 * and the kernels and returns at once.  host_samples must stay untouched until aisgpu_poll_upto(ticket) (or any later
 * poll / aisgpu_sync) has returned.  *ticket receives the ordinal of this submit (0, 1, 2, ...; every aisgpu_submit*
 * call takes one).  The pattern  submit_async(c); poll_upto(c - 1)  overlaps the copy of step c with the host work of
 * step c - 1. */
int aisgpu_submit_async(aisgpu_handle *h, const void *host_samples, int n_samples, int64_t *ticket);

/* Same, with the batch already resident in device memory ([n_streams][stride_samples], first n_samples used).  n_samples may
 * change from call to call as for aisgpu_submit, and so may dev_samples and stride_samples.  Placement rule (checked by
 * aisgpu_check_device_batch, which this calls first; a batch that breaks it is AISGPU_EINVAL with the handle untouched):
 *   - stride_samples is even and >= n_samples;
 *   - dev_samples is aligned to two samples: 16 bytes for CF32, 8 for CS16, 4 for CU8 / CS8;
 *   - AISGPU_MODE_X and FP_DS: dev_samples and every row are 16-byte aligned (stride_samples * bytes per sample % 16 == 0);
 *   - AISGPU_MODEL_DISCRIMINATOR at exactly 48000 S/s: dev_samples only needs to be aligned to one sample;
 *   - AISGPU_FMT_F32_FS4, in every mode and model: dev_samples is 16-byte aligned and stride_samples is a multiple of 4, so every row
 *     starts a new 1, j, -1, -j pattern on a 16-byte boundary;
 *   - AISGPU_FMT_DC16H, in every mode and model: dev_samples is 16-byte aligned and stride_samples is a multiple of 4 (four samples
 *     are 48 bytes), so every row starts on a 16-byte boundary. */
int aisgpu_submit_device(aisgpu_handle *h, const void *dev_samples, int64_t stride_samples, int n_samples);

/* The placement rule of aisgpu_submit_device for an engine created with *cfg, without touching the GPU (dev_samples is only
 * inspected as a number): 0 if the batch may lie there, else AISGPU_EINVAL (also for a configuration aisgpu_create refuses) with
 * the reason in aisgpu_last_error(NULL).  stride_samples >= n_samples is aisgpu_submit_device's own check. */
int aisgpu_check_device_batch(const aisgpu_config *cfg, const void *dev_samples, int64_t stride_samples);

/* Waits for all submitted work (cudaStreamSynchronize). */
int aisgpu_sync(aisgpu_handle *h);

/* == Model::Output() / StreamOut<Message> (Model.h:96): returns frames completed by submits so far, in the
 * reference's emission order (per submit: stream-major, channel A before B, then time; DSP.cpp:312-313).
 * Implies aisgpu_sync().  *n receives the count written (<= max); call again until *n == 0. */
int aisgpu_poll(aisgpu_handle *h, aisgpu_msg *out, int max, int *n);

/* aisgpu_poll that only waits for the submits up to `ticket` (see aisgpu_submit_async) and returns their frames; later
 * submits keep running.  ticket < 0 or beyond the last submit == aisgpu_poll. */
int aisgpu_poll_upto(aisgpu_handle *h, int64_t ticket, aisgpu_msg *out, int max, int *n);

/* Intermediates of the LAST submit for one stream/channel; *n_out = elements written (float2 or float). */
int aisgpu_tap(aisgpu_handle *h, int tap, int stream, int channel, void *dst, size_t dst_bytes, size_t *n_out);

/* counters[0]=frames (CRC ok), [1]=messages published (validate ok), [2]=samples/stream, [3]=submits,
 * [4]=frames dropped by ring overflow, [5]=ch A messages, [6]=ch B messages, [7]=reserved */
int aisgpu_counters(aisgpu_handle *h, uint64_t counters[8]);

/* Multi-GPU: the stream batch is sharded over one engine (process) per GPU and nothing but these counters ever crosses
 * NVLink (SURVEY.md 8e).  aisgpu_nccl_unique_id fills a 128-byte ncclUniqueId on one rank (the caller ships it to the
 * others: MPI, a file, torch.distributed ...), aisgpu_comm_init joins the communicator (ncclCommInitRank; NCCL is resolved
 * at run time with dlopen("libnccl.so.2"), AISGPU_ENODEV if absent), aisgpu_allreduce_counts sums aisgpu_counters() of all
 * ranks (ncclAllReduce, uint64, on the engine's stream).  Without a communicator totals == the local counters. */
int aisgpu_nccl_unique_id(void *id128);
int aisgpu_comm_init(aisgpu_handle *h, const void *id128, int n_ranks, int rank);
int aisgpu_allreduce_counts(aisgpu_handle *h, uint64_t totals[8]);

/* The CUDA stream the kernels are launched on (cudaStream_t as void*), for event timing by the caller. */
void *aisgpu_cuda_stream(aisgpu_handle *h);

/* The back end runs on more than one internal stream; this makes the stream returned by aisgpu_cuda_stream() wait
 * (on the device, no host synchronisation) for everything submitted so far -- call it before recording an event that
 * should mark the end of all submitted work. */
int aisgpu_join(aisgpu_handle *h);

/* Device time of the front-end kernel of the last submit in ms (CUDA events on the launch stream), <0 if n/a. */
float aisgpu_last_frontend_ms(aisgpu_handle *h);

/* Device times (ms) of the front-end kernel of the most recent submits, newest first (up to 128 kept).
 * Implies aisgpu_sync().  This is the live roofline measurement bench.py reports. */
int aisgpu_frontend_times(aisgpu_handle *h, float *ms_out, int max, int *n);

/* Number of kernels launched by the last submit. */
int aisgpu_last_launches(aisgpu_handle *h);

/* Host-only pieces of the per-frame tail of AIS::Decoder::processData (AIS.cpp:66-96), exported so that they can be
 * checked without a GPU:
 *   aisgpu_validate   == AIS::Message::validate (Message.cpp:398-413): 1 if the frame would be published.
 *   aisgpu_build_nmea == AIS::Message::buildNMEA (Message.cpp:569-631): fills n_sentences / nmea / nmea_len of *m from
 *                        m->data, m->nbits, m->channel.  *seq (0..9) is the multi-sentence sequence id and is advanced
 *                        exactly like Message::nextSeqId (Message.cpp:28-39). */
int aisgpu_validate(const uint8_t *data, int nbits);
int aisgpu_build_nmea(aisgpu_msg *m, int own_mmsi, int *seq);

/* ---- Formats either side of the path (SURVEY.md 8f rank 4) ---- */

/* The TAG / receiver fields the reference's outputs print next to a message (Source/Library/Common.h:218-250 TAG;
 * Message::rxtime/toa/station, Message.h:60-75).  level and ppm are taken from the aisgpu_msg.  On an engine with a receiver table
 * (aisgpu_set_receivers), the records of stream s take driver, hardware, mode, ipv4 and station from the stream's receiver; version,
 * status, rxtime_us, toa_us, include_ssl, uuid and suffix stay the output's, for every stream. */
typedef struct aisgpu_tag {
	int32_t version;      /* TAG::version */
	int32_t driver;       /* TAG::driver (Type enum as int) */
	const char *hardware; /* TAG::hardware, may be NULL (printed as "") */
	int32_t mode;         /* TAG::mode: bit 0 -> signalpower/ppm are printed, bit 1 -> rxuxtime is printed */
	int32_t status;       /* TAG::status, printed as msg_status when non-zero */
	uint32_t ipv4;        /* TAG::ipv4, printed when non-zero */
	int64_t rxtime_us;    /* Message::rxtime (microseconds since the epoch, Message::Stamp); an engine with a clock prints each frame's
	                         stamp instead (aisgpu_set_clock) */
	int64_t toa_us;       /* Message::toa, printed when non-zero */
	int32_t station;      /* Message::getStation(), printed as station_id when non-zero */
	int32_t include_ssl;  /* getNMEAJSON's include_ssl: print ssc (start_idx) and sl (end_idx - start_idx) */
	const char *uuid;     /* getNMEAJSON's uuid argument, may be NULL or "" */
	const char *suffix;   /* getNMEAJSON's suffix argument (e.g. "\r\n"), may be NULL */
} aisgpu_tag;

/* == AIS::Message::getNMEAJSON(out, tag, include_ssl, uuid, suffix) (Message.cpp:93-191): the JSON line of the UDP/TCP/HTTP
 * "NMEA JSON" outputs, number formatting as JSON::Writer (Writer.h:174-218).  Returns the bytes written (no NUL is appended),
 * AISGPU_EOVERFLOW if cap is too small. Host-only. */
int aisgpu_msg_json(const aisgpu_msg *m, const aisgpu_tag *tag, char *out, int cap);

/* == the line JSON::Serializer(JSON_DICT_FULL) writes for AIS::JSONAIS::ProcessMsg(msg, tag) (Source/JSON/JSONAIS.cpp:1092-1533,
 * Source/JSON/Writer.h): the full AIS JSON of -o 5, MSGFORMAT JSON_FULL and the HTTP / UDP / MQTT JSON outputs, decoded by the
 * table interpreter the engine runs on the device (aisgpu_poll_json), built for the host.  From *tag it takes version, driver,
 * hardware, mode (bit 0: signalpower / ppm from the aisgpu_msg unless 1024; bit 1: rxtime / rxuxtime from rxtime_us; bit 2: country
 * and country_code of the MMSI's MID), toa_us (printed when non-zero), station (station_id when non-zero) and suffix (appended);
 * status, ipv4, include_ssl and uuid are not part of this line.  The sentences under "nmea" are m's own.  Every message type and
 * every application message (DAC, FI) of types 6, 8, 25 and 26 that the reference decodes into fields is decoded (ProcessMsg6Data /
 * ProcessMsg8Data, JSONAIS.cpp:979-1044), repeated records included; any other (DAC, FI) is printed as "data", as the reference
 * prints it.  Returns the bytes written (no NUL), AISGPU_EOVERFLOW if cap is too small, AISGPU_EINVAL for a NULL argument.
 * Host-only. */
int aisgpu_msg_json_full(const aisgpu_msg *m, const aisgpu_tag *tag, char *out, int cap);

/* The full AIS JSON of every published frame, decoded on the GPU.  aisgpu_json_enable (before the first submit; once) fixes the tag
 * every line is printed with (as for aisgpu_msg_json_full; suffix is not used) and max_bytes_per_submit, the text one submit's
 * lines may take, newlines included.  From then on every poll of the frame ring -- aisgpu_poll, aisgpu_poll_upto, aisgpu_poll_json
 * and the feeders' -- decodes the frames it publishes on the device: one upload of those frames and three kernels on a stream of
 * its own, never the front end or the demodulation kernels, so frames, taps and counters do not change.  A group member decodes
 * its own frames (enable it on the member).
 *
 * aisgpu_poll_json is aisgpu_poll_upto for the lines: it drains the frames of the submits up to ticket if no line is waiting, and
 * copies whole lines, each ended by '\n', in the order aisgpu_poll returns the frames, until the next would pass cap; *n_bytes and
 * *n_lines receive what was written.  Call it again until *n_lines == 0.  Line i is frame i: the frames and the lines a poll
 * publishes are queued side by side, and each queue is read by its own call (aisgpu_poll* / aisgpu_poll_json), so a caller may
 * take both, or only one of them.  Neither queue keeps more than max_frames (aisgpu_config) unread entries: beyond that the oldest
 * are dropped, and the next poll of that kind returns AISGPU_EOVERFLOW with what survived -- a caller that takes only lines (or
 * only frames) thus holds at most max_frames of the other in host memory.  Lines past a submit's max_bytes_per_submit are dropped,
 * later lines of that submit too, and the next aisgpu_poll_json returns AISGPU_EOVERFLOW with the lines that survived, as the frame
 * ring does.  AISGPU_EINVAL when JSON is not enabled, or when cap is smaller than the next line.  The engine allocates, at enable,
 * about 8.6 KB of device memory and 4.3 KB of pinned host memory per frame of a 4096-frame decode batch. */
int aisgpu_json_enable(aisgpu_handle *h, const aisgpu_tag *tag, int max_bytes_per_submit);
int aisgpu_poll_json(aisgpu_handle *h, int64_t ticket, char *out, size_t cap, size_t *n_bytes, int *n_lines);

/* Message formats: the position of each in the reference's enum class MessageFormat (Source/Library/Common.h:144-156), as MSGFORMAT
 * selects them for an output (IO/MsgOut.h:282-289).  0 (SILENT) is not a format here.  The record of a frame is exactly what
 * OutputMessage::formatInto (IO/MsgOut.h:58-122) -- or, for the three JSON formats, OutputMessage::Receive of the JSON stream --
 * appends for that message, "suffix" being the output's line suffix (aisgpu_tag.suffix; NULL: "\r\n"):
 *   NMEA           each sentence + suffix
 *   NMEA_TAG       per sentence "\s:s<station>,c:<rxtime s>[,g:<i>-<n>-<group>]*hh\" + sentence + "\r\n" (getNMEATagBlock)
 *   COMMUNITY_HUB  the JSON_NMEA record for the engine's frames 0, 100, 200, ...; the BINARY_NMEA record for the others
 *   BINARY_NMEA    getBinaryNMEA(tag, crc = 0): possibly empty (aisgpu_msg_binary)
 *   FULL           per sentence "<s> ( MSG: t, REPEAT: r, MMSI: m[, signalpower: %g, ppm: %g][, timestamp: YYYYMMDDHHMMSS][, ID: station])\n";
 *                  signalpower / ppm when mode bit 0 is set and neither is 1024 (undefined), the timestamp when mode bit 1 is set
 *   JSON_NMEA      getNMEAJSON(tag, include_ssl, uuid, suffix) (aisgpu_msg_json)
 *   JSON_SPARSE    the full AIS JSON object under the sparse dictionary + suffix: keys renamed, a key without a sparse name left out
 *                  with its value
 *   JSON_FULL      the full AIS JSON line (aisgpu_msg_json_full) + suffix
 *   JSON_ANNOTATED the full AIS JSON object with every member's value written as {"value":v[,"unit":..][,"description":..][,"text":..]}
 *                  ("text": the lookup entry of a number's value, where its key has a table) + suffix
 * JSON_SPARSE and JSON_ANNOTATED are the JSON_FULL line rewritten member by member, as JSON::Serializer writes the same members.
 * Two counters make a record depend on the frames before it.  The reference keeps them per output (hub_lines) and per process (the
 * NMEA_TAG group id); here both are the engine's, start at 0 as in a fresh process, and sit beside the per-stream NMEA sequence id
 * (aisgpu_msg.nmea) as the engine's state:
 *   - records: the frames the engine has published; COMMUNITY_HUB prints JSON_NMEA where it is a multiple of 100;
 *   - groups: the multi-sentence frames among them; the k-th such frame has NMEA_TAG group ((k - 1) % 9999) + 1.
 * Both advance over every published frame in emission order, including frames whose records the byte budget drops.  The engine
 * computes them on the device (a scan with a base carried from one 4096-frame batch to the next); aisgpu_format_state is the same
 * pair for aisgpu_msg_format. */
#define AISGPU_MSGFORMAT_NMEA 1
#define AISGPU_MSGFORMAT_NMEA_TAG 2
#define AISGPU_MSGFORMAT_COMMUNITY_HUB 3
#define AISGPU_MSGFORMAT_BINARY_NMEA 4
#define AISGPU_MSGFORMAT_FULL 5
#define AISGPU_MSGFORMAT_JSON_NMEA 6
#define AISGPU_MSGFORMAT_JSON_SPARSE 7
#define AISGPU_MSGFORMAT_JSON_FULL 8
#define AISGPU_MSGFORMAT_JSON_ANNOTATED 9

/* The engine's counters (above), for the host formatter. */
typedef struct aisgpu_format_state {
	int64_t records; /* frames formatted so far */
	int64_t groups;  /* multi-sentence frames among them */
} aisgpu_format_state;

/* The record of m in msgformat (1..9), printed with *tag (version, driver, hardware, mode, status, ipv4, rxtime_us, toa_us, station,
 * include_ssl, uuid; suffix NULL: "\r\n"), by the code the engine runs on the device for aisgpu_poll_lines, built for the host.
 * With st (may be NULL: both counters 0), the record uses *st and, when it is written, advances it exactly as the engine advances
 * its counters (records by one, groups by one for a frame of more than one sentence): a caller that formats every frame aisgpu_poll
 * returns, in order, from a zeroed state gets the engine's records.  Sentence lengths (nmea_len) are taken up to the 100 bytes of
 * aisgpu_msg.nmea, here and in aisgpu_msg_json.
 * Returns the bytes written (no NUL; 0 for an empty record), AISGPU_EOVERFLOW if cap is too small (st unchanged), AISGPU_EINVAL
 * for a NULL argument or an unknown format.  Host-only. */
int aisgpu_msg_format(const aisgpu_msg *m, const aisgpu_tag *tag, int msgformat, aisgpu_format_state *st, char *out, int cap);

/* The records of every published frame in one format, formatted on the GPU.  aisgpu_lines_enable (before the first submit; once,
 * and not together with aisgpu_json_enable: one engine has one format) fixes the format, the tag every record is printed with (as
 * for aisgpu_msg_format) and max_bytes_per_submit, the bytes one submit's records may take.  From then on every poll of the frame
 * ring formats the frames it publishes on the device, exactly as aisgpu_json_enable decodes them (which is this with JSON_FULL and
 * suffix "\n"): frames, taps and counters do not change, a group member formats its own frames, both queues are bounded by
 * max_frames, and records past a submit's budget are dropped and reported as AISGPU_EOVERFLOW by the next aisgpu_poll_lines.
 *
 * aisgpu_poll_lines is aisgpu_poll_upto for the records: it copies whole records, in the order aisgpu_poll returns the frames, until
 * the next would pass cap; *n_bytes and *n_records receive what was written.  Record i is frame i, also when it is empty (a
 * BINARY_NMEA frame of no valid length).  AISGPU_EINVAL when no format is enabled, or when cap is smaller than the next record.
 * aisgpu_poll_json reads the same queue on an engine enabled with aisgpu_json_enable, and is AISGPU_EINVAL on one enabled with
 * aisgpu_lines_enable.  The engine allocates, at enable, a slot per frame of a 4096-frame batch on the device and pinned host room
 * for the text: about 4.3 KB each (NMEA .. JSON_FULL), 8.5 / 4.3 KB (JSON_SPARSE) or 25 / 20.6 KB (JSON_ANNOTATED), plus the tag's
 * strings. */
int aisgpu_lines_enable(aisgpu_handle *h, int msgformat, const aisgpu_tag *tag, int max_bytes_per_submit);
int aisgpu_poll_lines(aisgpu_handle *h, int64_t ticket, char *out, size_t cap, size_t *n_bytes, int *n_records);

/* ---- Receivers: one per stream (the reference's repeated receiver objects, Application/Config.cpp:421) ----
 *
 * Every stream of a batch is a receiver of its own.  Without a table every stream takes the config's channel_a / channel_b, station,
 * own_mmsi and tag_mode, and every record the engine formats takes the aisgpu_tag of aisgpu_lines_enable / aisgpu_json_enable.
 * aisgpu_set_receivers installs r[0 .. n_streams - 1]: from then on stream s behaves as if its engine had been created with r[s]'s
 * channel_a / channel_b, station, own_mmsi and tag_mode --
 *   - its frames carry r[s].channel_a / channel_b (aisgpu_msg.channel) and read !AIVDO for r[s].own_mmsi (Receiver::setOwnMMSI,
 *     Receiver.cpp:221);
 *   - tag_mode bit 0 decides, per stream, whether its frames carry the signal level and convert it to dB (AIS.cpp:73-75): the back
 *     ends read a level switch per 48 kHz row;
 * -- and its records (aisgpu_poll_lines, aisgpu_poll_json) are printed with the output's tag whose station, driver, hardware, mode
 * (= tag_mode) and ipv4 are r[s]'s (Message::setOrigin, Message.h:300-306; the TAG of -M DTM, Receiver.cpp:26-66).  version, status,
 * rxtime_us (each frame's stamp on an engine with a clock), toa_us, include_ssl, uuid and suffix stay the output's, and so do the
 * COMMUNITY_HUB and NMEA_TAG counters (per engine).
 * counters[5] / [6] keep counting each stream's first and second channel, whatever its letters.  So the records expected for stream s
 * are exactly aisgpu_msg_format(frame, tag of s, ...).
 *
 * Rules (AISGPU_EINVAL with the reason in aisgpu_last_error(h), the handle untouched): n == n_streams; before the first submit; at
 * most once.  Every letter the engine prints must pass Receiver::setChannel's test (Receiver.cpp:103-105), alphanumeric or '?', else
 * the reason is the reference's "invalid NMEA channel designation: <c>"; channel_b is only read where a stream has two channels (AB
 * mode, and AISGPU_MODEL_DISCRIMINATOR in both modes).  It may come before or after aisgpu_lines_enable / aisgpu_json_enable: the
 * per-stream record contexts are made when both are known.  A group member takes a table of its own; the leader's does not reach
 * it.  hardware is copied (NULL: "").
 *
 * Memory: a level bit per row (always).  With a table and a format enabled, the device holds one record context (96 bytes) and the
 * stream's hardware name and full-JSON prefix (about 100 bytes plus the name) per stream, and every record slot (above) is sized for
 * the longest hardware name and prefix among the streams. */
typedef struct aisgpu_receiver {
	char channel_a, channel_b; /* the receiver's NMEA designation (CH1 / CH2 of buildModel); X mode: channel_b unused */
	int32_t station;           /* Model::station: NMEA_TAG s:, station_id, FULL's ID */
	int32_t own_mmsi;          /* Model::own_mmsi: this MMSI's sentences read !AIVDO */
	uint32_t tag_mode;         /* TAG::mode of the receiver: bit 0 level in dB + signalpower / ppm printed, bit 1 time, bit 2 country */
	int32_t driver;            /* TAG::driver */
	const char *hardware;      /* TAG::hardware, may be NULL ("") */
	uint32_t ipv4;             /* TAG::ipv4 */
} aisgpu_receiver;

int aisgpu_set_receivers(aisgpu_handle *h, const aisgpu_receiver *r, int n);
/* The rules of aisgpu_set_receivers that need no device, for an engine created with *cfg (struct_size as for aisgpu_create): 0, or
 * AISGPU_EINVAL with the reason in aisgpu_last_error(NULL). */
int aisgpu_check_receivers(const aisgpu_config *cfg, const aisgpu_receiver *r, int n);

/* ---- Tuning: a digital tune per stream (DESIGN.md 7d) ----
 *
 * Without a table the engine takes each capture as centred where the reference tunes its receiver: AB mode expects the channel pair
 * at -25 / +25 kHz (162.000 MHz for A/B, 156.800 MHz for C/D), X mode its channel at 0 Hz.  aisgpu_set_tuning gives stream s an
 * integer offset offset_hz[s]: the frequency of what must land at 0 Hz, relative to the capture's centre -- the pair's centre in AB
 * mode, the channel in X mode.  From then on every submit first mixes each stream to 0 Hz on the GPU (one read of the input and one
 * CF32 write per sample), and the rest of the engine runs unchanged on those rows, as on a CF32 input: stream s then yields exactly
 * the frames (and AISGPU_TAP_C rows, and channel dump) of an untuned engine fed aisgpu_tune_restate(format, sample_rate,
 * offset_hz[s], 0, its whole input) as CF32 -- which is what the reference yields on that signal.  A stream whose offset is 0 is
 * converted only, never multiplied: its frames are those of an untuned engine on its raw input, bit for bit.  Host submits, device
 * batches (any stride and base aisgpu_submit_device takes), aisgpu_feed_files and aisgpu_feed_wav_files all go through the tune.
 * A group leader's table tunes the rows its whole group reads.
 *
 * Several tunings of one input (aisgpu_set_tunings, per_input = T > 1): the engine still decodes n_streams streams, but the caller
 * supplies R = n_streams / T input rows, and stream s reads input row s / T with its own offset offset_hz[s] -- the T tunings of one
 * input are adjacent streams.  A wideband marine-band capture with T = 2 and offsets +2.6 MHz / -2.6 MHz gives the A/B pair on the even
 * streams and the C/D pair on the odd ones (their letters come from aisgpu_set_receivers).  Stream s yields exactly what an untuned CF32
 * engine yields on aisgpu_tune_restate(format, sample_rate, offset_hz[s], 0, input row s / T).  Every entry point that takes the
 * caller's samples takes R rows: aisgpu_submit / _async (R x n_samples contiguous), aisgpu_submit_v (R pointers),
 * aisgpu_submit_device (R rows, stride_samples apart, under the same placement rules), aisgpu_feed_files and aisgpu_feed_wav_files (R
 * paths, file r feeding streams rT .. rT + T - 1).  Everything indexed by stream stays n_streams: receivers, clock starts, dump
 * prefixes, aisgpu_msg.stream, counters, taps, aisgpu_stamp.  The tune reads each input sample once and writes T CF32 samples.
 * aisgpu_set_tuning(h, f, n) is aisgpu_set_tunings(h, f, n, 1).
 *
 * Rules (AISGPU_EINVAL with the reason in aisgpu_last_error(h), the handle untouched): n == n_streams; per_input >= 1 and divides
 * n_streams; before the first submit; at most once; -sample_rate/2 < offset_hz[s] < sample_rate/2.  Refused outright:
 * AISGPU_MODEL_DISCRIMINATOR (its I and Q are two real audio channels: nothing to tune), an engine that runs the FP_DS integer front end
 * (it reads CU8 directly), and a group member (its front end is the leader's).
 *
 * Memory: the tables (about 36 KB at 1536 kS/s, 56 KB at 12.288 MS/s), and n_streams x max_chunk_samples CF32 samples of scratch,
 * except behind a resampler with no CIC stage in front of it, where the tune writes the resampler's input directly.  The host staging
 * of aisgpu_submit / _v / _async and the feeders' pinned buffers hold R rows. */
int aisgpu_set_tunings(aisgpu_handle *h, const int32_t *offset_hz, int n, int per_input);
int aisgpu_set_tuning(aisgpu_handle *h, const int32_t *offset_hz, int n);
/* The rules of aisgpu_set_tunings that need no device, for an engine created with *cfg: 0, or AISGPU_EINVAL with the reason in
 * aisgpu_last_error(NULL).  aisgpu_check_tuning(cfg, f, n) is aisgpu_check_tunings(cfg, f, n, 1). */
int aisgpu_check_tunings(const aisgpu_config *cfg, const int32_t *offset_hz, int n, int per_input);
int aisgpu_check_tuning(const aisgpu_config *cfg, const int32_t *offset_hz, int n);
/* The definition of the tune, on the host: n samples of one stream in `format` (samples first_sample .. first_sample + n - 1 of it)
 * -> n CF32 samples.  Sample m converts as the reference's ConvertRAW does (F32_FS4's 1, j, -1, -j pattern indexed by m) to v; with
 * f = offset_hz and fs = sample_rate, k = ((m mod fs) * f) mod fs in [0, fs) (int64), k = a * 4096 + b, and
 *   p = T_hi[a] * T_lo[b],  T_hi[a] = exp(2 pi i a 4096 / fs),  T_lo[b] = exp(2 pi i b / fs)  (each in double, rounded to float),
 *   out = v * conj(p):  pr = hi.re lo.re - hi.im lo.im, pi = hi.re lo.im + hi.im lo.re, out = (v.re pr + v.im pi, v.im pr - v.re pi),
 * every product and sum rounded to float.  f = 0: out = v.  The engine computes the same bits on the GPU.  0, or AISGPU_EINVAL for an
 * unknown format, sample_rate < 1, first_sample < 0, n < 0, null buffers, or an offset outside (-fs/2, fs/2). */
int aisgpu_tune_restate(int format, int sample_rate, int32_t offset_hz, int64_t first_sample, const void *in, int64_t n, void *out_cf32);

/* ---- Receive time: a clock per stream (DESIGN.md 7e) ----
 *
 * Without a clock every record the engine formats prints the output's aisgpu_tag.rxtime_us.  aisgpu_set_clock stamps every frame
 * with its own receive time instead, at the reference's granularity: its decoder thread stamps a message (Message::Stamp,
 * AIS.cpp:76-77) while it processes the block that completes it, so here a frame's stamp is a function of its stream s and of
 * aisgpu_msg.chunk, the submit c that completed it:
 *   - recording clock (start_us != NULL; start_us[s] = the time of stream s's first sample, microseconds since the epoch):
 *     stamp(s, c) = start_us[s] + floor(S_c * 10^6 / fs), computed as q * 10^6 + (r * 10^6) / fs with q = S_c / fs, r = S_c % fs.
 *     S_c is the number of samples per stream submitted through submit c inclusive (counters[2] right after it) and fs the config's
 *     sample_rate (F32_FS4: the rate of the real samples; AISGPU_MODEL_DISCRIMINATOR: the audio rate).  Submit lengths may vary;
 *     the zero-padded tail blocks of aisgpu_feed_files / aisgpu_feed_wav_files are submits and count as signal time;
 *   - live clock (start_us == NULL): every stream's stamp for submit c is std::chrono::system_clock's time in microseconds since
 *     the epoch, as Message::Stamp reads it, read once by the aisgpu_submit* call (or feeder block) that made submit c, between
 *     that call's entry and its return.
 * The record of every published frame, in every format and on every path (aisgpu_poll_lines, aisgpu_poll_json, the feeders'
 * polls), is then exactly aisgpu_msg_format(frame, tag', ...), tag' being the record's tag (the output's, or its stream's with a
 * receiver table) with rxtime_us = the frame's stamp.  Mode bit 1 still decides, per stream, whether the JSON formats and FULL
 * print the time; NMEA_TAG, BINARY_NMEA and COMMUNITY_HUB print it always.  aisgpu_poll's frames are unchanged (aisgpu_msg has no
 * time): aisgpu_stamp(h, frame.stream, frame.chunk) gives it.
 *
 * Rules (AISGPU_EINVAL with the reason in aisgpu_last_error(h), the handle untouched): n == n_streams, also for start_us == NULL;
 * before the first submit; at most once; every start_us[s] in [0, 253402300800000000) (before 10000-01-01, so that rxtime stays
 * YYYYMMDDHHMMSS).  Refused on a group member: the leader's clock stamps the whole group's frames (as the leader's tuning tunes
 * the rows the group reads), and a member's records and aisgpu_stamp follow the leader's submits.  It may come before or after
 * aisgpu_lines_enable / aisgpu_json_enable and aisgpu_set_receivers.
 *
 * Memory: 8 bytes of host memory per submit for the life of the engine (S_c or the wall time, shared by a group), plus the start
 * times (8 bytes per stream); with a format enabled, a device buffer of one 8-byte stamp per frame of a 4096-frame batch (32 KB),
 * uploaded beside the frames.  Without a clock nothing of this is allocated, uploaded or launched.  (The record slots of every
 * engine hold the longest time members any stamp can print.) */
int aisgpu_set_clock(aisgpu_handle *h, const int64_t *start_us, int n);
/* The rules of aisgpu_set_clock that need no device, for an engine created with *cfg: 0, or AISGPU_EINVAL with the reason in
 * aisgpu_last_error(NULL). */
int aisgpu_check_clock(const aisgpu_config *cfg, const int64_t *start_us, int n);
/* *rxtime_us = the stamp of the frames of stream `stream` completed by submit `chunk` (aisgpu_msg.chunk), for any submit made so far
 * (a member: its leader's submits).  AISGPU_EINVAL without a clock, and for a stream or chunk out of range. */
int aisgpu_stamp(aisgpu_handle *h, int stream, int64_t chunk, int64_t *rxtime_us);

/* == AIS::Message::getBinaryNMEA(out, tag, crc) (Message.cpp:277-396): 0xAC 0x00 framed, byte-stuffed binary record with an
 * optional CRC-16 (Helper.cpp:42-57).  Returns the bytes written, 0 when the reference would emit nothing. Host-only. */
int aisgpu_msg_binary(const aisgpu_msg *m, const aisgpu_tag *tag, int crc, uint8_t *out, int cap);

/* == n_streams Device::RAWFile receivers (Source/Device/FileRAW.cpp:36-165) feeding one engine: paths[s] is the recording of
 * stream s in the engine's sample format (F32_FS4: 4-byte real samples; the padding is +0 floats.  DC16H: 12-byte samples;
 * the padding is zero words, samples (+0, +0)); the files are read in blocks of n_samples (a multiple of aisgpu_chunk_granule),
 * the tail of each file is zero-padded to a whole block (FileRAW.cpp:91-94) and the run ends with the longest file.  Reading
 * block c+1 (threads), the copy and kernels of block c and the delivery of the frames of block c-1 to fn overlap (two pinned
 * buffers, aisgpu_submit_async / aisgpu_poll_upto).  fn may be NULL (count only: aisgpu_counters).  *n_blocks receives the
 * number of blocks submitted.  Returns 0, AISGPU_EOVERFLOW (frames were dropped, the rest delivered) or the first error. */
typedef void (*aisgpu_msg_fn)(const aisgpu_msg *msgs, int n, void *user);
int aisgpu_feed_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks);

/* == Device::WAVFile::Open (Source/Device/FileWAV.cpp:49-98), host only: reads the header of the WAV file at path as the reference
 * does, so that a caller can fill aisgpu_config from a recording.  The 12-byte RIFF header must read "RIFF" ... "WAVE"; chunks are
 * walked until "data", "fmt " may come anywhere before it, and every other chunk is skipped by its size rounded up to an even
 * number.  The first 16 bytes of "fmt " are read and the rest of it is skipped.  The file must have 2 channels (I/Q), and
 * tag 3 / 32 bits is AISGPU_FMT_CF32, tag 1 / 8 bits AISGPU_FMT_CU8, tag 1 / 16 bits AISGPU_FMT_CS16; every other format,
 * WAVE_FORMAT_EXTENSIBLE (0xFFFE) included, is refused.  *sample_rate is dwSamplesPerSec, *data_offset the byte after the data
 * chunk's header.  The data chunk's size is not read: the samples run from there to the end of the file, so chunks after "data"
 * (LIST, ...) are read as samples, as WAVFile::isStreaming reads them (FileWAV.cpp:107-120).  A WAV never maps to
 * AISGPU_FMT_CS8 or AISGPU_FMT_F32_FS4.  AISGPU_EINVAL, with the reference's text in aisgpu_last_error(NULL) ("cannot open WAV
 * file: ...", "cannot read header from WAV file: ...", "not a supported WAV-file.", "invalid fmt chunk in WAV-file.", "cannot
 * read fmt chunk from WAV-file.", "no data in WAV-file.", "WAV-file must have 2 channels (I/Q).", "format not supported"), for a
 * file the reference refuses; the outputs are then untouched. */
int aisgpu_wav_probe(const char *path, int32_t *format, uint32_t *sample_rate, int64_t *data_offset);

/* == n_streams Device::WAVFile receivers feeding one engine: aisgpu_feed_files with stream s read from the data offset that
 * aisgpu_wav_probe gives for paths[s] to the end of the file.  The blocks, the zero-padding of each file's tail, the end of the run
 * with the longest file, fn, *n_blocks and the return values are aisgpu_feed_files's.  Before anything is read or submitted,
 * every file is probed: one the reference refuses, or one whose format or sample rate differs from the engine's, is AISGPU_EINVAL
 * with the file and the reason (the reference's text, or the field that differs) in aisgpu_last_error(h).  An engine group is
 * refused as for aisgpu_feed_files.  AISGPU_MODEL_DISCRIMINATOR reads the stereo recording as I/Q, as ModelDiscriminator does. */
int aisgpu_feed_wav_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks);

/* ---- Engine groups: several models on one front end (the reference's repeated -m, Receiver.cpp:126-244) ----
 *
 * Makes *out a member of leader's group: an engine with a back end of its own (cfg->model with its own ps_ema, afc_wide, dd_train,
 * dd_weight, channel_a/b, station, own_mmsi, tag_mode, enable_taps, max_frames) that is fed with the 48 kHz channel rows of the
 * leader's front end instead of running the front end again.  Call it before the leader's first submit.  AISGPU_EINVAL (reason in
 * aisgpu_last_error(NULL)) when aisgpu_check_attach refuses the pair, when the leader has been submitted to, when leader is itself a
 * member, or when the group would exceed 8 engines.
 *
 * A member behaves exactly like a standalone engine of its own config that received the leader's submits:
 *   - aisgpu_poll, aisgpu_poll_upto (with the leader's tickets), aisgpu_counters and aisgpu_tap act on the member's own frame ring
 *     and state: emission order, msg.chunk, sequence ids, AISGPU_EOVERFLOW and the counters are the standalone engine's; counters[2]
 *     and [3] follow the leader's submits;
 *   - only the leader is submitted to (aisgpu_submit, _v, _async, _device); one leader submit runs every member's back end.
 *     aisgpu_submit* on a member, and aisgpu_feed_files or aisgpu_feed_wav_files on a group's engine, return AISGPU_EINVAL;
 *   - aisgpu_sync(leader) and aisgpu_join(leader) cover the whole group (events on the leader's stream time the group);
 *   - a member has no front end: AISGPU_TAP_ROT, _PRE and _PRE2 are AISGPU_EINVAL, aisgpu_last_frontend_ms() is -1 and
 *     aisgpu_frontend_times() gives n = 0;
 *   - a CUDA failure in a group submit poisons every engine of the group;
 *   - destroying a member detaches it (the leader's frames do not change); destroying a leader that still has members poisons
 *     them, so destroy the members first.
 * One thread drives a whole group, as for a single handle. */
int aisgpu_attach(aisgpu_handle *leader, const aisgpu_config *cfg, aisgpu_handle **out);

/* The compatibility rule of aisgpu_attach without touching the GPU: 0, or AISGPU_EINVAL with the reason (naming the first field that
 * differs) in aisgpu_last_error(NULL).  Every front-end field must be equal -- sample_rate, format, n_streams, max_chunk_samples,
 * channel_mode, droop, dsk, fp_ds, device -- and neither config may be AISGPU_MODEL_DISCRIMINATOR.  struct_size as for
 * aisgpu_create. */
int aisgpu_check_attach(const aisgpu_config *leader, const aisgpu_config *member);

/* ---- The 48 kHz channel dump (the reference's -go DUMP <prefix>, Model.cpp:348-353, 390-396) ----
 *
 * Writes the two 48 kHz channel streams of stream s (the FilterCIC5 outputs C_a / C_b, what AISGPU_TAP_C reads) to
 * "<prefixes[s]>_A.wav" (row 2s) and "<prefixes[s]>_B.wav" (row 2s + 1) as Util::WriteWAV does (StreamHelpers.cpp:135-229): a 44-byte
 * header (IEEE float, 2 channels, 32 bits, 48000 S/s), then every block of samples raw as CF32; the two sizes are patched at close,
 * as uint32_t.  The letters are A and B in CD mode too.  prefixes[s] == NULL: stream s is not written.  Each file is created at the
 * first submit that yields 48 kHz samples, and one file descriptor per file stays open until the dump is closed.
 *
 * Every submit's rows are gathered on the GPU and copied into one of three pinned slots; the files are written on the caller's
 * thread, never by a thread of the engine.  The rows of submit t are in the files no later than the return of aisgpu_poll_upto(t),
 * aisgpu_poll, aisgpu_sync or aisgpu_dump_close; an aisgpu_submit* that needs a slot whose rows have not been written writes them
 * first.  Frames, taps and counters are the same with and without a dump.
 *
 * aisgpu_dump_open is AISGPU_EINVAL, with the handle untouched and the reason in aisgpu_last_error(h), when prefixes is NULL, after
 * the first submit, when a dump is already open, in AISGPU_MODE_X (the reference writes nothing there, Model.cpp:106), for
 * AISGPU_MODEL_DISCRIMINATOR (ModelDiscriminator refuses the key, Model.h:107-122) and on a group member (it has no front end: dump
 * the leader; a leader's dump leaves its members unchanged).  It allocates three device and three pinned slots of
 * rows x (most 48 kHz samples one submit can yield) CF32 samples.
 *
 * A failed create or write stops the dump (the reference's StopRequest()): the reason, in the reference's wording ("WAV out: ..."),
 * goes to aisgpu_last_error, and every later aisgpu_submit* returns AISGPU_EIO without enqueuing anything until aisgpu_dump_close
 * has been called.  aisgpu_poll* are not affected and the handle is not poisoned.  aisgpu_feed_files on an engine with an open dump
 * writes the channels of every block it submits, the zero-padded ones included; AISGPU_EIO is then its first error.
 *
 * aisgpu_dump_close writes what is pending, patches the headers and closes the files: 0, or AISGPU_EIO if a create or write failed
 * (the files are closed with the sizes written so far).  aisgpu_destroy closes an open dump. */
int aisgpu_dump_open(aisgpu_handle *h, const char *const *prefixes);
int aisgpu_dump_close(aisgpu_handle *h);

const char *aisgpu_last_error(aisgpu_handle *h); /* h may be NULL: error of the last failed aisgpu_create / aisgpu_attach */

/* == ~Model */
void aisgpu_destroy(aisgpu_handle *h);

int aisgpu_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif
