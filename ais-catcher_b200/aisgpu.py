"""ctypes binding of the C ABI in include/aisgpu.h (test / bench harness side).

The product is libaisgpu.so (csrc/*.cu, built by __graft_entry__.build()); this file only marshals
arguments.  It fails loudly when the library is missing -- there is no fallback implementation.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("AISGPU_LIB") or os.path.join(HERE, "libaisgpu.so")  # AISGPU_LIB: A/B of two builds of the library on one machine

MODEL_STANDARD, MODEL_BASE, MODEL_DEFAULT, MODEL_CHALLENGER, MODEL_V2 = 0, 1, 2, 4, 11
MODEL_DISCRIMINATOR = 3  # FM-discriminator input: I and Q are the audio of two discriminator taps (channels A and B)
FMT_CF32, FMT_CU8, FMT_CS8, FMT_CS16 = 0, 1, 2, 3
FMT_F32_FS4 = 4  # one real float32 per sample, made complex by the fs/4 shift 1, j, -1, -j (Airspy / HydraSDR real mode)
FMT_DC16H = 7  # three uint32 per sample: I and Q are the low 16 bits of words 0 and 1 (Q negated), the rest is not read; 5 and 6 are no formats
MODE_AB, MODE_X = 0, 3  # aisgpu_config.channel_mode: two channels (also CD) / single channel (-c X)
TAP_C, TAP_CGF, TAP_FIR, TAP_ROT, TAP_DEC, TAP_FM, TAP_PRE, TAP_PRE2 = 0, 1, 2, 3, 4, 5, 7, 8

EXPORTS = ["aisgpu_abi_version", "aisgpu_default_config", "aisgpu_create", "aisgpu_submit", "aisgpu_submit_device",
           "aisgpu_sync", "aisgpu_poll", "aisgpu_tap", "aisgpu_counters", "aisgpu_cuda_stream",
           "aisgpu_last_frontend_ms", "aisgpu_frontend_times", "aisgpu_last_launches", "aisgpu_last_error", "aisgpu_destroy",
           "aisgpu_validate", "aisgpu_build_nmea", "aisgpu_chunk_granule", "aisgpu_join", "aisgpu_submit_v", "aisgpu_submit_async",
           "aisgpu_poll_upto", "aisgpu_nccl_unique_id", "aisgpu_comm_init", "aisgpu_allreduce_counts",
           "aisgpu_msg_json", "aisgpu_msg_binary", "aisgpu_feed_files", "aisgpu_check_device_batch", "aisgpu_attach",
           "aisgpu_check_attach", "aisgpu_dump_open", "aisgpu_dump_close", "aisgpu_wav_probe", "aisgpu_feed_wav_files",
           "aisgpu_msg_json_full", "aisgpu_json_enable", "aisgpu_poll_json", "aisgpu_msg_format", "aisgpu_lines_enable",
           "aisgpu_poll_lines", "aisgpu_set_receivers", "aisgpu_check_receivers",
           "aisgpu_set_tuning", "aisgpu_check_tuning", "aisgpu_tune_restate", "aisgpu_set_clock", "aisgpu_check_clock",
           "aisgpu_stamp", "aisgpu_set_tunings", "aisgpu_check_tunings"]

OK, EINVAL, ENODEV, ECUDA, ENOMEM, EOVERFLOW, EIO = 0, -1, -2, -3, -4, -5, -6
# message formats: positions in the reference's enum class MessageFormat (MSGFORMAT of its outputs); include/aisgpu.h describes each record
(MSGFORMAT_NMEA, MSGFORMAT_NMEA_TAG, MSGFORMAT_COMMUNITY_HUB, MSGFORMAT_BINARY_NMEA, MSGFORMAT_FULL, MSGFORMAT_JSON_NMEA,
 MSGFORMAT_JSON_SPARSE, MSGFORMAT_JSON_FULL, MSGFORMAT_JSON_ANNOTATED) = range(1, 10)
MSGFORMATS = {"NMEA": 1, "NMEA_TAG": 2, "COMMUNITY_HUB": 3, "BINARY_NMEA": 4, "FULL": 5, "JSON_NMEA": 6, "JSON_SPARSE": 7,
              "JSON_FULL": 8, "JSON_ANNOTATED": 9}


class FormatState(C.Structure):
    """aisgpu_format_state: the engine's counters for msg_format (records formatted, multi-sentence frames among them)."""
    _fields_ = [("records", C.c_int64), ("groups", C.c_int64)]


class Config(C.Structure):
    _fields_ = [("struct_size", C.c_uint32), ("model", C.c_int32), ("sample_rate", C.c_int32), ("format", C.c_int32),
                ("n_streams", C.c_int32), ("max_chunk_samples", C.c_int32), ("ps_ema", C.c_int32), ("afc_wide", C.c_int32),
                ("droop", C.c_int32), ("channel_a", C.c_char), ("channel_b", C.c_char), ("station", C.c_int32),
                ("own_mmsi", C.c_int32), ("tag_mode", C.c_uint32), ("device", C.c_int32), ("enable_taps", C.c_int32),
                ("max_frames", C.c_int32), ("host_staging", C.c_int32), ("dsk", C.c_int32), ("fp_ds", C.c_int32), ("dd_train", C.c_float), ("dd_weight", C.c_float),
                ("channel_mode", C.c_int32)]


class MsgStruct(C.Structure):
    _fields_ = [("stream", C.c_int32), ("channel", C.c_char), ("nbits", C.c_int32), ("start_idx", C.c_int64),
                ("end_idx", C.c_int64), ("level", C.c_float), ("ppm", C.c_float), ("chunk", C.c_int64),
                ("data", C.c_uint8 * 140), ("n_sentences", C.c_int32), ("nmea", (C.c_char * 100) * 4),
                ("nmea_len", C.c_int32 * 4)]


class TagStruct(C.Structure):
    _fields_ = [("version", C.c_int32), ("driver", C.c_int32), ("hardware", C.c_char_p), ("mode", C.c_int32), ("status", C.c_int32),
                ("ipv4", C.c_uint32), ("rxtime_us", C.c_int64), ("toa_us", C.c_int64), ("station", C.c_int32),
                ("include_ssl", C.c_int32), ("uuid", C.c_char_p), ("suffix", C.c_char_p)]


class Receiver(C.Structure):
    """aisgpu_receiver: one stream's receiver (channel letters, station, own MMSI, tag mode, and the TAG's driver, hardware, ipv4)."""
    _fields_ = [("channel_a", C.c_char), ("channel_b", C.c_char), ("station", C.c_int32), ("own_mmsi", C.c_int32),
                ("tag_mode", C.c_uint32), ("driver", C.c_int32), ("hardware", C.c_char_p), ("ipv4", C.c_uint32)]


def make_receiver(channels="AB", station=0, own_mmsi=-1, tag_mode=3, driver=0, hardware=None, ipv4=0):
    """A Receiver from keyword arguments; channels: the two designation letters (X mode: the second is not read)."""
    enc = lambda t: None if t is None else (t if isinstance(t, bytes) else t.encode("latin-1"))
    ch = channels.encode("latin-1") if isinstance(channels, str) else bytes(channels)
    return Receiver(ch[0:1], ch[1:2] or ch[0:1], station, own_mmsi, tag_mode, driver, enc(hardware), ipv4)


def receiver_table(receivers):
    """A ctypes array of Receiver from Receiver structures or dicts of make_receiver keyword arguments."""
    rs = [r if isinstance(r, Receiver) else make_receiver(**r) for r in receivers]
    return (Receiver * max(len(rs), 1))(*rs)


def check_receivers(receivers, **engine):
    """aisgpu_check_receivers (no GPU needed): the rules of Engine.set_receivers for an engine of keyword arguments `engine`.
    Raises with the reason (the reference's text for a bad letter) if the table would be refused."""
    lib = load()
    rc = lib.aisgpu_check_receivers(C.byref(make_config(**engine)), receiver_table(receivers), len(receivers))
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode("latin-1")))


def _offsets(offsets):
    return (C.c_int32 * max(len(offsets), 1))(*[int(f) for f in offsets])


def check_tuning(offsets, per_input=1, **engine):
    """aisgpu_check_tunings (no GPU needed): the rules of Engine.set_tuning for an engine of keyword arguments `engine`.
    Raises with the reason if the offsets (Hz, one per stream), per_input tunings of each input, would be refused."""
    lib = load()
    rc = lib.aisgpu_check_tunings(C.byref(make_config(**engine)), _offsets(offsets), len(offsets), int(per_input))
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode("latin-1")))


def _starts(start_us):
    return None if start_us is None else (C.c_int64 * max(len(start_us), 1))(*[int(t) for t in start_us])


def check_clock(start_us, n=None, **engine):
    """aisgpu_check_clock (no GPU needed): the rules of Engine.set_clock for an engine of keyword arguments `engine`.  start_us: one
    start time (microseconds since the epoch) per stream, or None for the live clock; n: the count passed (default: len(start_us),
    or n_streams for None).  Raises with the reason if the clock would be refused."""
    lib = load()
    if n is None:
        n = engine.get("n_streams", 1) if start_us is None else len(start_us)
    rc = lib.aisgpu_check_clock(C.byref(make_config(**engine)), _starts(start_us), int(n))
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode("latin-1")))


def tune_restate(fmt, sample_rate, offset_hz, first_sample, samples):
    """aisgpu_tune_restate: one stream's samples in format fmt (a numpy array of the format's layout: complex64 for CF32, bytes
    (u)int8 / int16 pairs, float32 for F32_FS4, uint32 triples for DC16H), samples first_sample .. of the stream, mixed by
    offset_hz -> complex64 array: what a tuned engine's rows after the tune hold."""
    lib = load()
    a = np.ascontiguousarray(samples)
    n = a.nbytes // BPS[fmt]
    out = np.empty(n, np.complex64)
    rc = lib.aisgpu_tune_restate(int(fmt), int(sample_rate), int(offset_hz), int(first_sample), a.ctypes.data_as(C.c_void_p), n,
                                 out.ctypes.data_as(C.c_void_p))
    if rc:
        raise AisGpuError("aisgpu_tune_restate rc=%d" % rc)
    return out


BPS = {FMT_CF32: 8, FMT_CU8: 2, FMT_CS8: 2, FMT_CS16: 4, FMT_F32_FS4: 4, FMT_DC16H: 12}  # bytes per sample of each input format

MSG_FN = C.CFUNCTYPE(None, C.POINTER(MsgStruct), C.c_int, C.c_void_p)


class Msg:
    __slots__ = ("stream", "channel", "nbits", "start_idx", "end_idx", "level", "ppm", "chunk", "payload", "nmea", "data")

    def __init__(self, m):
        self.stream = m.stream
        self.channel = m.channel.decode()
        self.nbits = m.nbits
        self.start_idx = m.start_idx
        self.end_idx = m.end_idx
        self.level = m.level
        self.ppm = m.ppm
        self.chunk = m.chunk
        self.payload = bytes(m.data[:(m.nbits + 7) // 8])
        self.nmea = [m.nmea[i].raw[:m.nmea_len[i]].decode("latin-1") for i in range(min(m.n_sentences, 4))]
        self.data = bytes(m.data)  # all of aisgpu_msg::data: the full JSON reads bits past nbits as the reference does

    def key(self):
        return (self.channel, self.nbits, self.payload, tuple(self.nmea))

    def __repr__(self):
        return "Msg(s%d,%s,%d,%s)" % (self.stream, self.channel, self.nbits, " ".join(self.nmea))


_lib = None


def load():
    """dlopen libaisgpu.so and declare prototypes.  Raises if the library was not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("%s not built: run `python -c 'import __graft_entry__ as g; g.build()'` (no CPU fallback exists)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    lib.aisgpu_abi_version.restype = C.c_int
    lib.aisgpu_default_config.argtypes = [C.POINTER(Config)]
    lib.aisgpu_default_config.restype = None
    lib.aisgpu_create.argtypes = [C.POINTER(Config), C.POINTER(C.c_void_p)]
    lib.aisgpu_submit.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    lib.aisgpu_submit_device.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int]
    lib.aisgpu_submit_v.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.c_int]
    lib.aisgpu_submit_async.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int64)]
    lib.aisgpu_poll_upto.argtypes = [C.c_void_p, C.c_int64, C.POINTER(MsgStruct), C.c_int, C.POINTER(C.c_int)]
    lib.aisgpu_nccl_unique_id.argtypes = [C.c_void_p]
    lib.aisgpu_comm_init.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    lib.aisgpu_allreduce_counts.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.aisgpu_sync.argtypes = [C.c_void_p]
    lib.aisgpu_poll.argtypes = [C.c_void_p, C.POINTER(MsgStruct), C.c_int, C.POINTER(C.c_int)]
    lib.aisgpu_tap.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    lib.aisgpu_counters.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    lib.aisgpu_join.argtypes = [C.c_void_p]
    lib.aisgpu_cuda_stream.argtypes = [C.c_void_p]
    lib.aisgpu_cuda_stream.restype = C.c_void_p
    lib.aisgpu_last_frontend_ms.argtypes = [C.c_void_p]
    lib.aisgpu_last_frontend_ms.restype = C.c_float
    lib.aisgpu_frontend_times.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int)]
    lib.aisgpu_last_launches.argtypes = [C.c_void_p]
    lib.aisgpu_last_error.argtypes = [C.c_void_p]
    lib.aisgpu_last_error.restype = C.c_char_p
    lib.aisgpu_chunk_granule.argtypes = [C.POINTER(Config)]
    if hasattr(lib, "aisgpu_check_device_batch"):  # absent from libraries built before the placement rule (AISGPU_LIB)
        lib.aisgpu_check_device_batch.argtypes = [C.POINTER(Config), C.c_void_p, C.c_int64]
    if hasattr(lib, "aisgpu_attach"):  # absent from libraries built before engine groups (AISGPU_LIB)
        lib.aisgpu_attach.argtypes = [C.c_void_p, C.POINTER(Config), C.POINTER(C.c_void_p)]
        lib.aisgpu_check_attach.argtypes = [C.POINTER(Config), C.POINTER(Config)]
    if hasattr(lib, "aisgpu_dump_open"):  # absent from libraries built before the channel dump (AISGPU_LIB)
        lib.aisgpu_dump_open.argtypes = [C.c_void_p, C.POINTER(C.c_char_p)]
        lib.aisgpu_dump_close.argtypes = [C.c_void_p]
    if hasattr(lib, "aisgpu_wav_probe"):  # absent from libraries built before WAV input (AISGPU_LIB)
        lib.aisgpu_wav_probe.argtypes = [C.c_char_p, C.POINTER(C.c_int32), C.POINTER(C.c_uint32), C.POINTER(C.c_int64)]
        lib.aisgpu_feed_wav_files.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.c_int, MSG_FN, C.c_void_p, C.POINTER(C.c_uint64)]
    if hasattr(lib, "aisgpu_msg_json_full"):  # absent from libraries built before the full JSON (AISGPU_LIB)
        lib.aisgpu_msg_json_full.argtypes = [C.POINTER(MsgStruct), C.POINTER(TagStruct), C.c_char_p, C.c_int]
        lib.aisgpu_json_enable.argtypes = [C.c_void_p, C.POINTER(TagStruct), C.c_int]
        lib.aisgpu_poll_json.argtypes = [C.c_void_p, C.c_int64, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
    if hasattr(lib, "aisgpu_msg_format"):  # absent from libraries built before the output records (AISGPU_LIB)
        lib.aisgpu_msg_format.argtypes = [C.POINTER(MsgStruct), C.POINTER(TagStruct), C.c_int, C.POINTER(FormatState), C.c_char_p,
                                          C.c_int]
        lib.aisgpu_lines_enable.argtypes = [C.c_void_p, C.c_int, C.POINTER(TagStruct), C.c_int]
        lib.aisgpu_poll_lines.argtypes = [C.c_void_p, C.c_int64, C.c_char_p, C.c_size_t, C.POINTER(C.c_size_t), C.POINTER(C.c_int)]
    if hasattr(lib, "aisgpu_set_receivers"):  # absent from libraries built before the receiver tables (AISGPU_LIB)
        lib.aisgpu_set_receivers.argtypes = [C.c_void_p, C.POINTER(Receiver), C.c_int]
        lib.aisgpu_check_receivers.argtypes = [C.POINTER(Config), C.POINTER(Receiver), C.c_int]
    if hasattr(lib, "aisgpu_set_tuning"):  # absent from libraries built before the tuning tables (AISGPU_LIB)
        lib.aisgpu_set_tuning.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int]
        lib.aisgpu_check_tuning.argtypes = [C.POINTER(Config), C.POINTER(C.c_int32), C.c_int]
        lib.aisgpu_tune_restate.argtypes = [C.c_int, C.c_int, C.c_int32, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    if hasattr(lib, "aisgpu_set_tunings"):  # absent from libraries built before several tunings of one input (AISGPU_LIB)
        lib.aisgpu_set_tunings.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int, C.c_int]
        lib.aisgpu_check_tunings.argtypes = [C.POINTER(Config), C.POINTER(C.c_int32), C.c_int, C.c_int]
    if hasattr(lib, "aisgpu_set_clock"):  # absent from libraries built before the clocks (AISGPU_LIB)
        lib.aisgpu_set_clock.argtypes = [C.c_void_p, C.POINTER(C.c_int64), C.c_int]
        lib.aisgpu_check_clock.argtypes = [C.POINTER(Config), C.POINTER(C.c_int64), C.c_int]
        lib.aisgpu_stamp.argtypes = [C.c_void_p, C.c_int, C.c_int64, C.POINTER(C.c_int64)]
    lib.aisgpu_validate.argtypes = [C.c_char_p, C.c_int]
    lib.aisgpu_build_nmea.argtypes = [C.POINTER(MsgStruct), C.c_int, C.POINTER(C.c_int)]
    lib.aisgpu_msg_json.argtypes = [C.POINTER(MsgStruct), C.POINTER(TagStruct), C.c_char_p, C.c_int]
    lib.aisgpu_msg_binary.argtypes = [C.POINTER(MsgStruct), C.POINTER(TagStruct), C.c_int, C.c_char_p, C.c_int]
    lib.aisgpu_feed_files.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.c_int, MSG_FN, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.aisgpu_destroy.argtypes = [C.c_void_p]
    lib.aisgpu_destroy.restype = None
    _lib = lib
    return lib


def chunk_granule(sample_rate, model=MODEL_DEFAULT, dsk=False, fp_ds=False, fmt=FMT_CF32, channel_mode=MODE_AB):
    """Granule (samples) every submit length must be a multiple of; raises with the reference's wording if unsupported."""
    lib = load()
    cfg = Config()
    lib.aisgpu_default_config(C.byref(cfg))
    cfg.sample_rate, cfg.model, cfg.dsk, cfg.fp_ds, cfg.format = sample_rate, model, int(dsk), int(fp_ds), fmt
    cfg.channel_mode = channel_mode
    g = lib.aisgpu_chunk_granule(C.byref(cfg))
    if g <= 0:
        raise AisGpuError("rc=%d: %s" % (g, lib.aisgpu_last_error(None).decode()))
    return g


def check_device_batch(dev_ptr, stride_samples, sample_rate=1536000, model=MODEL_DEFAULT, fmt=FMT_CF32, dsk=False, fp_ds=False,
                       channel_mode=MODE_AB, n_streams=1):
    """aisgpu_check_device_batch: the placement rule of submit_device (no GPU needed).  Raises with the reason if the batch
    may not lie at dev_ptr with rows stride_samples apart."""
    lib = load()
    cfg = Config()
    lib.aisgpu_default_config(C.byref(cfg))
    cfg.sample_rate, cfg.model, cfg.dsk, cfg.fp_ds, cfg.format = sample_rate, model, int(dsk), int(fp_ds), fmt
    cfg.channel_mode, cfg.n_streams = channel_mode, n_streams
    rc = lib.aisgpu_check_device_batch(C.byref(cfg), C.c_void_p(dev_ptr), stride_samples)
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode()))


def wav_probe(path):
    """aisgpu_wav_probe (no GPU needed): (format, sample_rate, data_offset) of a WAV recording, read as the reference's
    Device::WAVFile reads it.  Raises with the reference's text if the reference refuses the file."""
    lib = load()
    fmt, rate, off = C.c_int32(0), C.c_uint32(0), C.c_int64(0)
    rc = lib.aisgpu_wav_probe(os.fsencode(path), C.byref(fmt), C.byref(rate), C.byref(off))
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode()))
    return fmt.value, rate.value, off.value


def make_msg(payload_bytes, nbits, channel="A", start_idx=0, end_idx=0, level=0.0, ppm=0.0, sentences=()):
    """An aisgpu_msg from raw fields (host-only helpers take it)."""
    m = MsgStruct()
    m.nbits = nbits
    m.channel = channel.encode()
    m.start_idx, m.end_idx, m.level, m.ppm = start_idx, end_idx, level, ppm
    for i, b in enumerate(payload_bytes[:140]):
        m.data[i] = b
    m.n_sentences = len(sentences)
    for i, t in enumerate(sentences):
        raw = t if isinstance(t, bytes) else t.encode("latin-1")
        C.memmove(m.nmea[i], raw, len(raw))
        m.nmea_len[i] = len(raw)
    return m


def make_tag(version=0, driver=0, hardware=None, mode=3, status=0, ipv4=0, rxtime_us=0, toa_us=0, station=0, include_ssl=False,
             uuid=None, suffix=None):
    enc = lambda t: None if t is None else (t if isinstance(t, bytes) else t.encode("latin-1"))
    return TagStruct(version, driver, enc(hardware), mode, status, ipv4, rxtime_us, toa_us, station, 1 if include_ssl else 0, enc(uuid), enc(suffix))


def msg_json(m, tag, cap=4096):
    """Host-only: aisgpu_msg_json (reference Message::getNMEAJSON, Message.cpp:93-191) -> bytes."""
    buf = C.create_string_buffer(cap)
    n = load().aisgpu_msg_json(C.byref(m), C.byref(tag), buf, cap)
    if n < 0:
        raise AisGpuError("aisgpu_msg_json rc=%d" % n)
    return buf.raw[:n]


def msg_json_full(m, tag, cap=65536):
    """Host-only: aisgpu_msg_json_full (the reference's JSONAIS line, JSON::Serializer(JSON_DICT_FULL)) -> bytes.
    m: an aisgpu_msg (make_msg) or a polled Msg."""
    if isinstance(m, Msg):
        m = msg_struct(m)
    buf = C.create_string_buffer(cap)
    n = load().aisgpu_msg_json_full(C.byref(m), C.byref(tag), buf, cap)
    if n < 0:
        raise AisGpuError("aisgpu_msg_json_full rc=%d" % n)
    return buf.raw[:n]


def msg_format(m, tag, fmt, state=None, cap=1 << 16):
    """Host-only: aisgpu_msg_format, the record of m (make_msg or a polled Msg) in MSGFORMAT fmt (1..9) with tag -> bytes.
    state: a FormatState, advanced as the engine advances its counters (None: both 0)."""
    if isinstance(m, Msg):
        m = msg_struct(m)
    buf = C.create_string_buffer(cap)
    n = load().aisgpu_msg_format(C.byref(m), C.byref(tag), int(fmt), C.byref(state) if state is not None else None, buf, cap)
    if n < 0:
        raise AisGpuError("aisgpu_msg_format rc=%d" % n)
    return buf.raw[:n]


def msg_struct(msg):
    """The aisgpu_msg of a polled Msg (every byte of data, the sentences, channel, level, ppm, indices)."""
    m = make_msg(msg.data, msg.nbits, msg.channel, msg.start_idx, msg.end_idx, msg.level, msg.ppm, msg.nmea)
    m.stream, m.chunk = msg.stream, msg.chunk
    return m


def msg_binary(m, tag, crc, cap=1024):
    """Host-only: aisgpu_msg_binary (reference Message::getBinaryNMEA, Message.cpp:277-396) -> bytes."""
    buf = C.create_string_buffer(cap)
    n = load().aisgpu_msg_binary(C.byref(m), C.byref(tag), 1 if crc else 0, buf, cap)
    if n < 0:
        raise AisGpuError("aisgpu_msg_binary rc=%d" % n)
    return buf.raw[:n]


def build_nmea(payload_bytes, nbits, channel="A", own_mmsi=-1, seq=0):
    """Host-only: (sentences, next seq) for a frame, through aisgpu_build_nmea (reference Message.cpp:569-631)."""
    lib = load()
    m = MsgStruct()
    m.nbits = nbits
    m.channel = channel.encode()
    for i, b in enumerate(payload_bytes[:140]):
        m.data[i] = b
    s = C.c_int(seq)
    rc = lib.aisgpu_build_nmea(C.byref(m), own_mmsi, C.byref(s))
    if rc:
        raise AisGpuError("aisgpu_build_nmea rc=%d" % rc)
    return Msg(m).nmea, s.value


class AisGpuError(RuntimeError):
    pass


def nccl_unique_id():
    """128-byte ncclUniqueId (bytes) from the library's run-time-resolved NCCL; one rank creates it, all ranks join."""
    lib = load()
    buf = C.create_string_buffer(128)
    rc = lib.aisgpu_nccl_unique_id(buf)
    if rc:
        raise AisGpuError("aisgpu_nccl_unique_id rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode()))
    return buf.raw


def make_config(model=MODEL_DEFAULT, sample_rate=1536000, fmt=FMT_CF32, n_streams=1, max_chunk=131072, ps_ema=True, afc_wide=True,
                droop=True, own_mmsi=-1, device=0, taps=False, max_frames=0, tag_mode=3, host_staging=True, dsk=False, fp_ds=False,
                channel_mode=MODE_AB, channels="AB", dd_train=0.75, dd_weight=0.86):
    """aisgpu_config from Engine's keyword arguments (the library's defaults for everything else)."""
    cfg = Config()
    load().aisgpu_default_config(C.byref(cfg))
    cfg.model, cfg.sample_rate, cfg.format = model, sample_rate, fmt
    cfg.n_streams, cfg.max_chunk_samples = n_streams, max_chunk
    cfg.ps_ema, cfg.afc_wide, cfg.droop = int(ps_ema), int(afc_wide), int(droop)
    cfg.own_mmsi, cfg.device, cfg.enable_taps, cfg.max_frames, cfg.tag_mode = own_mmsi, device, int(taps), max_frames, tag_mode
    cfg.host_staging, cfg.dsk, cfg.fp_ds = int(host_staging), int(dsk), int(fp_ds)
    cfg.dd_train, cfg.dd_weight = dd_train, dd_weight
    cfg.channel_mode = channel_mode
    cfg.channel_a, cfg.channel_b = channels[0].encode(), channels[1].encode()  # CH1 / CH2 of buildModel
    return cfg


# what a group member may set for itself (aisgpu_attach); every other field is the leader's
MEMBER_KEYS = ("model", "ps_ema", "afc_wide", "dd_train", "dd_weight", "channels", "own_mmsi", "taps", "max_frames", "tag_mode")


def check_attach(leader, member):
    """aisgpu_check_attach (no GPU needed): leader and member are dicts of Engine keyword arguments.  Raises with the reason (the
    first front-end field that differs) if the member may not join the leader's group."""
    lib = load()
    rc = lib.aisgpu_check_attach(C.byref(make_config(**leader)), C.byref(make_config(**member)))
    if rc:
        raise AisGpuError("rc=%d: %s" % (rc, lib.aisgpu_last_error(None).decode()))


class Engine:
    """One batch engine == one AIS::Model instance per stream of the batch (reference Source/DSP/Model.h:76-126)."""

    def __init__(self, model=MODEL_DEFAULT, sample_rate=1536000, fmt=FMT_CF32, n_streams=1, max_chunk=131072,
                 ps_ema=True, afc_wide=True, droop=True, own_mmsi=-1, device=0, taps=False, max_frames=0, tag_mode=3, host_staging=True,
                 dsk=False, fp_ds=False, channel_mode=MODE_AB, channels="AB", dd_train=0.75, dd_weight=0.86):
        self.lib = load()
        self.kwargs = dict(model=model, sample_rate=sample_rate, fmt=fmt, n_streams=n_streams, max_chunk=max_chunk, ps_ema=ps_ema,
                           afc_wide=afc_wide, droop=droop, own_mmsi=own_mmsi, device=device, taps=taps, max_frames=max_frames,
                           tag_mode=tag_mode, host_staging=host_staging, dsk=dsk, fp_ds=fp_ds, channel_mode=channel_mode,
                           channels=channels, dd_train=dd_train, dd_weight=dd_weight)
        cfg = make_config(**self.kwargs)
        self.cfg = cfg
        self.leader = None
        self.h = C.c_void_p()
        rc = self.lib.aisgpu_create(C.byref(cfg), C.byref(self.h))
        if rc:
            raise AisGpuError("aisgpu_create rc=%d: %s" % (rc, self.lib.aisgpu_last_error(None).decode()))
        self.n_streams = n_streams
        self.inputs = n_streams  # the rows every submit holds: n_streams / per_input after set_tuning
        self.fmt = fmt
        self.overflows = 0  # polls that reported AISGPU_EOVERFLOW (frames were dropped; the survivors were delivered)

    def attach(self, **member):
        """aisgpu_attach: a new engine of this one's group with its own back end (keyword arguments: MEMBER_KEYS, the rest is this
        engine's).  It is fed by this engine's submits; its own submit methods raise.  Attach before the first submit, and close
        the members before the leader."""
        bad = sorted(set(member) - set(MEMBER_KEYS))
        if bad:
            raise TypeError("attach() sets only the back end (%s); the front end is the leader's: %s" % (", ".join(MEMBER_KEYS), ", ".join(bad)))
        if len(member.get("channels", "AB")) != 2:
            raise ValueError("channels must be two letters (CH1, CH2), got %r" % (member["channels"],))
        kw = dict(self.kwargs, **member)
        cfg = make_config(**kw)
        h = C.c_void_p()
        rc = self.lib.aisgpu_attach(self.h, C.byref(cfg), C.byref(h))
        if rc:
            raise AisGpuError("aisgpu_attach rc=%d: %s" % (rc, self.lib.aisgpu_last_error(None).decode()))
        m = Engine.__new__(Engine)
        m.lib, m.kwargs, m.cfg, m.h = self.lib, kw, cfg, h
        m.leader = self  # keeps the leader alive while the member exists
        m.n_streams, m.inputs, m.fmt, m.overflows = self.n_streams, self.inputs, self.fmt, 0
        return m

    def _chk(self, rc):
        if rc == EOVERFLOW:
            self.overflows += 1
            return
        if rc:
            raise AisGpuError("rc=%d: %s" % (rc, self.lib.aisgpu_last_error(self.h).decode()))

    def _check_rows(self, what, rows):
        if rows != self.inputs:
            raise ValueError("%s: %d rows for an engine of %d inputs (n_streams %d)" % (what, rows, self.inputs, self.n_streams))

    def submit(self, host_array, n_samples):
        """host_array: contiguous numpy array holding inputs x n_samples samples (input-major; inputs is n_streams unless
        set_tuning gave each input several tunings)."""
        a = np.ascontiguousarray(host_array)
        if a.ndim >= 2:
            self._check_rows("submit", a.shape[0])
        if a.nbytes < self.inputs * n_samples * BPS[self.fmt]:
            raise ValueError("submit: %d bytes for %d inputs x %d samples" % (a.nbytes, self.inputs, n_samples))
        self._chk(self.lib.aisgpu_submit(self.h, a.ctypes.data_as(C.c_void_p), n_samples))

    def submit_ptr(self, host_ptr, n_samples):
        self._chk(self.lib.aisgpu_submit(self.h, C.c_void_p(host_ptr), n_samples))

    def submit_v(self, host_arrays, n_samples):
        """One host array per input (the shape independent receivers deliver)."""
        arrs = [np.ascontiguousarray(a) for a in host_arrays]
        self._check_rows("submit_v", len(arrs))
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        self._chk(self.lib.aisgpu_submit_v(self.h, ptrs, n_samples))

    def submit_async_ptr(self, host_ptr, n_samples):
        """Enqueue copy + kernels and return the ticket; the buffer must stay untouched until poll_upto(ticket) returned."""
        t = C.c_int64(-1)
        self._chk(self.lib.aisgpu_submit_async(self.h, C.c_void_p(host_ptr), n_samples, C.byref(t)))
        return t.value

    def feed_files(self, paths, n):
        """aisgpu_feed_files: one recording per input, blocks of n samples; returns (messages, blocks submitted)."""
        return self._feed(self.lib.aisgpu_feed_files, paths, n)

    def feed_wav_files(self, paths, n):
        """aisgpu_feed_wav_files: one WAV recording per input, in the engine's format and at its rate, read from its data chunk
        to its end in blocks of n samples; returns (messages, blocks submitted)."""
        return self._feed(self.lib.aisgpu_feed_wav_files, paths, n)

    def _feed(self, f, paths, n):
        self._check_rows(f.__name__, len(paths))
        arr = (C.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
        out = []
        cb = MSG_FN(lambda msgs, k, user: out.extend(Msg(msgs[i]) for i in range(k)))
        nb = C.c_uint64(0)
        rc = f(self.h, arr, n, cb, None, C.byref(nb))
        if rc == EOVERFLOW:
            self.overflows += 1
        else:
            self._chk(rc)
        return out, nb.value

    def poll_upto(self, ticket, batch=256):
        out = []
        buf = (MsgStruct * batch)()
        n = C.c_int(0)
        while True:
            self._chk(self.lib.aisgpu_poll_upto(self.h, ticket, buf, batch, C.byref(n)))
            if n.value == 0:
                break
            out.extend(Msg(buf[i]) for i in range(n.value))
        return out

    def poll_upto_count(self, ticket, batch=4096):
        """poll_upto without building Python objects: (frames, sentences) of the submits up to `ticket` (-1: all)."""
        if getattr(self, "_pbuf", None) is None or len(self._pbuf) < batch:
            self._pbuf = (MsgStruct * batch)()
        n = C.c_int(0)
        frames = sentences = 0
        while True:
            self._chk(self.lib.aisgpu_poll_upto(self.h, ticket, self._pbuf, batch, C.byref(n)))
            if n.value == 0:
                break
            frames += n.value
            sentences += n.value  # single-sentence messages dominate; exact count is in the structs if needed
            if n.value < batch:
                break
        return frames, sentences

    def comm_init(self, id128, n_ranks, rank):
        self._chk(self.lib.aisgpu_comm_init(self.h, id128, n_ranks, rank))

    def allreduce_counts(self):
        c = (C.c_uint64 * 8)()
        self._chk(self.lib.aisgpu_allreduce_counts(self.h, c))
        return list(c)

    def submit_device(self, dev_ptr, stride_samples, n_samples, rows=None):
        """aisgpu_submit_device: `inputs` rows of the engine's format, stride_samples apart, from dev_ptr.  rows: how many rows the
        caller's batch holds, checked against inputs when given."""
        if rows is not None:
            self._check_rows("submit_device", rows)
        self._chk(self.lib.aisgpu_submit_device(self.h, C.c_void_p(dev_ptr), stride_samples, n_samples))

    def sync(self):
        self._chk(self.lib.aisgpu_sync(self.h))

    def json_enable(self, tag=None, max_bytes_per_submit=1 << 24):
        """aisgpu_json_enable: from the first submit on, every polled frame is also decoded into the full AIS JSON on the GPU
        with tag (make_tag(); default: make_tag()), at most max_bytes_per_submit bytes of lines per submit."""
        self._json_tag = tag if tag is not None else make_tag()  # the tag's strings must outlive the call only; kept anyway
        self._chk(self.lib.aisgpu_json_enable(self.h, C.byref(self._json_tag), int(max_bytes_per_submit)))

    def poll_json(self, ticket=None, cap=1 << 20):
        """aisgpu_poll_json: the lines (str, UTF-8) of the frames of the submits up to ticket (None: all), in frame order."""
        t = -1 if ticket is None else int(ticket)
        buf = C.create_string_buffer(cap)
        nb, nl = C.c_size_t(0), C.c_int(0)
        out = []
        while True:
            self._chk(self.lib.aisgpu_poll_json(self.h, t, buf, cap, C.byref(nb), C.byref(nl)))
            if nl.value == 0:
                break
            out.extend(buf.raw[:nb.value].decode("utf-8", "surrogateescape").split("\n")[:-1])
        return out

    def lines_enable(self, fmt, tag=None, max_bytes_per_submit=1 << 24):
        """aisgpu_lines_enable: from the first submit on, every polled frame is also formatted on the GPU as its record in
        MSGFORMAT fmt (1..9) with tag (make_tag(); default: make_tag(); suffix None: CR LF), at most max_bytes_per_submit bytes of
        records per submit."""
        self._json_tag = tag if tag is not None else make_tag()
        self._chk(self.lib.aisgpu_lines_enable(self.h, int(fmt), C.byref(self._json_tag), int(max_bytes_per_submit)))

    def set_receivers(self, receivers):
        """aisgpu_set_receivers: one receiver per stream (Receiver structures or dicts of make_receiver keyword arguments), before
        the first submit and at most once.  Stream s then has receivers[s]'s letters, own MMSI and tag mode, and its records are
        printed with its station, driver, hardware, mode and ipv4."""
        self._receivers = receiver_table(receivers)  # copied by the library; kept anyway
        self._chk(self.lib.aisgpu_set_receivers(self.h, self._receivers, len(receivers)))

    def set_tuning(self, offsets, per_input=1):
        """aisgpu_set_tunings: one offset in Hz per stream (the channel pair's centre, or in X mode the channel, relative to the
        capture's centre), before the first submit and at most once.  Each submit is then mixed on the GPU so that it lands at 0 Hz.
        per_input > 1: each input row feeds per_input adjacent streams, and every submit and feed takes n_streams / per_input rows."""
        self._chk(self.lib.aisgpu_set_tunings(self.h, _offsets(offsets), len(offsets), int(per_input)))
        self.inputs = self.n_streams // int(per_input)

    def set_clock(self, start_us=None):
        """aisgpu_set_clock: start_us, one start time per stream in microseconds since the epoch (a recording clock), or None (the
        live clock), before the first submit and at most once.  Every record then carries its frame's own receive time."""
        n = self.n_streams if start_us is None else len(start_us)
        self._chk(self.lib.aisgpu_set_clock(self.h, _starts(start_us), n))

    def stamp(self, stream, chunk):
        """aisgpu_stamp: the receive time (microseconds since the epoch) of the frames of `stream` completed by submit `chunk`."""
        t = C.c_int64(0)
        self._chk(self.lib.aisgpu_stamp(self.h, int(stream), int(chunk), C.byref(t)))
        return t.value

    def poll_lines(self, ticket=None, cap=1 << 20):
        """aisgpu_poll_lines: (bytes, number of records) of the frames of the submits up to ticket (None: all), in frame order."""
        t = -1 if ticket is None else int(ticket)
        buf = C.create_string_buffer(cap)
        nb, nr = C.c_size_t(0), C.c_int(0)
        out, n = [], 0
        while True:
            self._chk(self.lib.aisgpu_poll_lines(self.h, t, buf, cap, C.byref(nb), C.byref(nr)))
            if nr.value == 0:
                break
            out.append(buf.raw[:nb.value])
            n += nr.value
        return b"".join(out), n

    def poll(self, batch=256):
        out = []
        buf = (MsgStruct * batch)()
        n = C.c_int(0)
        while True:
            self._chk(self.lib.aisgpu_poll(self.h, buf, batch, C.byref(n)))
            if n.value == 0:
                break
            out.extend(Msg(buf[i]) for i in range(n.value))
        return out

    def poll_count(self, batch=4096):
        """Drains the frame queue like poll() but leaves the frames in the ctypes buffer (no Python objects are built):
        returns (number of frames, number of NMEA sentences).  The library work is identical -- device sync, D2H copy
        of the frame ring, validation and NMEA armouring on the host."""
        if getattr(self, "_pbuf", None) is None or len(self._pbuf) < batch:
            self._pbuf = (MsgStruct * batch)()
        n = C.c_int(0)
        frames = sentences = 0
        while True:
            self._chk(self.lib.aisgpu_poll(self.h, self._pbuf, batch, C.byref(n)))
            if n.value == 0:
                break
            frames += n.value
            sentences += n.value  # single-sentence messages dominate; exact count is in the structs if needed
            if n.value < batch:
                break
        return frames, sentences

    def tap(self, tap, stream=0, channel=0, dtype=np.complex64, max_elems=1 << 22):
        out = np.empty(max_elems, dtype=dtype)
        n = C.c_size_t(0)
        self._chk(self.lib.aisgpu_tap(self.h, tap, stream, channel, out.ctypes.data_as(C.c_void_p), out.nbytes, C.byref(n)))
        return out[:n.value].copy()

    def counters(self):
        c = (C.c_uint64 * 8)()
        self._chk(self.lib.aisgpu_counters(self.h, c))
        return list(c)

    def join(self):
        self._chk(self.lib.aisgpu_join(self.h))

    def cuda_stream(self):
        return self.lib.aisgpu_cuda_stream(self.h)

    def last_frontend_ms(self):
        return float(self.lib.aisgpu_last_frontend_ms(self.h))

    def frontend_times(self, max_n=128):
        buf = (C.c_float * max_n)()
        n = C.c_int(0)
        self._chk(self.lib.aisgpu_frontend_times(self.h, buf, max_n, C.byref(n)))
        return [buf[i] for i in range(n.value)]

    def last_launches(self):
        return int(self.lib.aisgpu_last_launches(self.h))

    def dump_open(self, prefixes):
        """aisgpu_dump_open (-go DUMP): prefixes is one entry per stream, a path prefix (str or os.PathLike) or None for a stream
        that is not dumped.  Stream s goes to <prefix>_A.wav and <prefix>_B.wav.  Open before the first submit."""
        prefixes = list(prefixes)
        if len(prefixes) != self.n_streams:
            raise ValueError("dump_open: %d prefixes for %d streams" % (len(prefixes), self.n_streams))
        arr = (C.c_char_p * len(prefixes))(*[None if p is None else os.fsencode(p) for p in prefixes])
        rc = self.lib.aisgpu_dump_open(self.h, arr)
        if rc:
            raise AisGpuError("rc=%d: %s" % (rc, self.lib.aisgpu_last_error(self.h).decode()))

    def dump_close(self):
        """aisgpu_dump_close: writes what is pending, patches the WAV headers and closes the files."""
        rc = self.lib.aisgpu_dump_close(self.h)
        if rc:
            raise AisGpuError("rc=%d: %s" % (rc, self.lib.aisgpu_last_error(self.h).decode()))

    def close(self):
        if self.h:
            self.lib.aisgpu_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
