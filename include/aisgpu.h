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

/* input sample formats: subset of enum class Format (Source/Library/Common.h:89-104) */
#define AISGPU_FMT_CF32 0
#define AISGPU_FMT_CU8 1
#define AISGPU_FMT_CS8 2
#define AISGPU_FMT_CS16 3

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
	char channel_a, channel_b;  /* CH1/CH2 of buildModel (Model.cpp:547-548), default 'A','B' */
	int32_t station;            /* Model::station  (Model.h:79) */
	int32_t own_mmsi;           /* Model::own_mmsi (Model.h:80): sentences of this MMSI read !AIVDO */
	uint32_t tag_mode;          /* TAG::mode (Common.h:242): bit0 = signal level, default 3 */
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
 *   - AISGPU_MODEL_DISCRIMINATOR at exactly 48000 S/s: dev_samples only needs to be aligned to one sample. */
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
 * Message::rxtime/toa/station, Message.h:60-75).  level and ppm are taken from the aisgpu_msg. */
typedef struct aisgpu_tag {
	int32_t version;      /* TAG::version */
	int32_t driver;       /* TAG::driver (Type enum as int) */
	const char *hardware; /* TAG::hardware, may be NULL (printed as "") */
	int32_t mode;         /* TAG::mode: bit 0 -> signalpower/ppm are printed, bit 1 -> rxuxtime is printed */
	int32_t status;       /* TAG::status, printed as msg_status when non-zero */
	uint32_t ipv4;        /* TAG::ipv4, printed when non-zero */
	int64_t rxtime_us;    /* Message::rxtime (microseconds since the epoch, Message::Stamp) */
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

/* == AIS::Message::getBinaryNMEA(out, tag, crc) (Message.cpp:277-396): 0xAC 0x00 framed, byte-stuffed binary record with an
 * optional CRC-16 (Helper.cpp:42-57).  Returns the bytes written, 0 when the reference would emit nothing. Host-only. */
int aisgpu_msg_binary(const aisgpu_msg *m, const aisgpu_tag *tag, int crc, uint8_t *out, int cap);

/* == n_streams Device::RAWFile receivers (Source/Device/FileRAW.cpp:36-165) feeding one engine: paths[s] is the recording of
 * stream s in the engine's sample format; the files are read in blocks of n_samples (a multiple of aisgpu_chunk_granule),
 * the tail of each file is zero-padded to a whole block (FileRAW.cpp:91-94) and the run ends with the longest file.  Reading
 * block c+1 (threads), the copy and kernels of block c and the delivery of the frames of block c-1 to fn overlap (two pinned
 * buffers, aisgpu_submit_async / aisgpu_poll_upto).  fn may be NULL (count only: aisgpu_counters).  *n_blocks receives the
 * number of blocks submitted.  Returns 0, AISGPU_EOVERFLOW (frames were dropped, the rest delivered) or the first error. */
typedef void (*aisgpu_msg_fn)(const aisgpu_msg *msgs, int n, void *user);
int aisgpu_feed_files(aisgpu_handle *h, const char *const *paths, int n_samples, aisgpu_msg_fn fn, void *user, uint64_t *n_blocks);

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
 *     aisgpu_submit* on a member, and aisgpu_feed_files on a leader with members, return AISGPU_EINVAL;
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
