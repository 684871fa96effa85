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
MODE_AB, MODE_X = 0, 3  # aisgpu_config.channel_mode: two channels (also CD) / single channel (-c X)
TAP_C, TAP_CGF, TAP_FIR, TAP_ROT, TAP_DEC, TAP_FM, TAP_PRE, TAP_PRE2 = 0, 1, 2, 3, 4, 5, 7, 8

EXPORTS = ["aisgpu_abi_version", "aisgpu_default_config", "aisgpu_create", "aisgpu_submit", "aisgpu_submit_device",
           "aisgpu_sync", "aisgpu_poll", "aisgpu_tap", "aisgpu_counters", "aisgpu_cuda_stream",
           "aisgpu_last_frontend_ms", "aisgpu_frontend_times", "aisgpu_last_launches", "aisgpu_last_error", "aisgpu_destroy",
           "aisgpu_validate", "aisgpu_build_nmea", "aisgpu_chunk_granule", "aisgpu_join", "aisgpu_submit_v", "aisgpu_submit_async",
           "aisgpu_poll_upto", "aisgpu_nccl_unique_id", "aisgpu_comm_init", "aisgpu_allreduce_counts",
           "aisgpu_msg_json", "aisgpu_msg_binary", "aisgpu_feed_files", "aisgpu_check_device_batch", "aisgpu_attach",
           "aisgpu_check_attach", "aisgpu_dump_open", "aisgpu_dump_close"]

OK, EINVAL, ENODEV, ECUDA, ENOMEM, EOVERFLOW, EIO = 0, -1, -2, -3, -4, -5, -6


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


MSG_FN = C.CFUNCTYPE(None, C.POINTER(MsgStruct), C.c_int, C.c_void_p)


class Msg:
    __slots__ = ("stream", "channel", "nbits", "start_idx", "end_idx", "level", "ppm", "chunk", "payload", "nmea")

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
        m.n_streams, m.fmt, m.overflows = self.n_streams, self.fmt, 0
        return m

    def _chk(self, rc):
        if rc == EOVERFLOW:
            self.overflows += 1
            return
        if rc:
            raise AisGpuError("rc=%d: %s" % (rc, self.lib.aisgpu_last_error(self.h).decode()))

    def submit(self, host_array, n_samples):
        """host_array: contiguous numpy array holding n_streams x n_samples samples (stream-major)."""
        a = np.ascontiguousarray(host_array)
        self._chk(self.lib.aisgpu_submit(self.h, a.ctypes.data_as(C.c_void_p), n_samples))

    def submit_ptr(self, host_ptr, n_samples):
        self._chk(self.lib.aisgpu_submit(self.h, C.c_void_p(host_ptr), n_samples))

    def submit_v(self, host_arrays, n_samples):
        """One host array per stream (the shape n_streams independent receivers deliver)."""
        arrs = [np.ascontiguousarray(a) for a in host_arrays]
        ptrs = (C.c_void_p * len(arrs))(*[a.ctypes.data for a in arrs])
        self._chk(self.lib.aisgpu_submit_v(self.h, ptrs, n_samples))

    def submit_async_ptr(self, host_ptr, n_samples):
        """Enqueue copy + kernels and return the ticket; the buffer must stay untouched until poll_upto(ticket) returned."""
        t = C.c_int64(-1)
        self._chk(self.lib.aisgpu_submit_async(self.h, C.c_void_p(host_ptr), n_samples, C.byref(t)))
        return t.value

    def feed_files(self, paths, n):
        """aisgpu_feed_files: one recording per stream, blocks of n samples; returns (messages, blocks submitted)."""
        assert len(paths) == self.n_streams
        arr = (C.c_char_p * len(paths))(*[os.fsencode(p) for p in paths])
        out = []
        cb = MSG_FN(lambda msgs, k, user: out.extend(Msg(msgs[i]) for i in range(k)))
        nb = C.c_uint64(0)
        rc = self.lib.aisgpu_feed_files(self.h, arr, n, cb, None, C.byref(nb))
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

    def submit_device(self, dev_ptr, stride_samples, n_samples):
        self._chk(self.lib.aisgpu_submit_device(self.h, C.c_void_p(dev_ptr), stride_samples, n_samples))

    def sync(self):
        self._chk(self.lib.aisgpu_sync(self.h))

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
