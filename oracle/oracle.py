"""TEST INFRASTRUCTURE -- ctypes front ends for the two CPU checkers.

* ``RefModel``  : the UNMODIFIED reference (oracle/_ref/libaisref*.so, built by oracle/Makefile
                  from /root/reference where it lies; see ref_harness.cpp).
* ``PortModel`` : the plain-C restatement (oracle/libaisoracle.so, ais_oracle.c): models 0, 1, 2 and 4 (ModelChallenger), and
                  ModelChallenger in single-channel mode at 48 kS/s (FLAG_MODE_X).

Both expose the same methods so tests can swap them.  Only tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs may import this module; the product never does.
"""
import ctypes as C
import os
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

MODEL_STANDARD, MODEL_BASE, MODEL_DEFAULT, MODEL_CHALLENGER, MODEL_V2 = 0, 1, 2, 4, 11  # V2: reference harness only
FMT_CF32, FMT_CU8, FMT_CS8, FMT_CS16 = 0, 1, 2, 3
FLAG_PS_EMA, FLAG_AFC_WIDE, FLAG_DROOP, FLAG_TAPS, FLAG_FP_DS, FLAG_DSK = 1, 2, 4, 8, 16, 32  # FP_DS / DSK: reference harness only
FLAG_MODE_X = 64  # the port only: single-channel mode (-c X), ModelChallenger at 48 kS/s; the reference's is oracle_x.RefModelX
# ModelChallenger's decoders as publishers() numbers them: 0..4 the coherent phases a0..a4, 5..9 the FM phases f0..f4.  The
# reference steps them in this order within each group of five 48 kHz samples (PortModel.challenger_order replaces it).
CHALLENGER_ORDER = (5, 6, 7, 8, 0, 1, 2, 3, 4, 9)
DEFAULT_FLAGS = FLAG_PS_EMA | FLAG_AFC_WIDE | FLAG_DROOP

# complex taps
TAP_ROT_IN, TAP_UP, TAP_DOWN, TAP_CA, TAP_CB, TAP_CGF_A, TAP_CGF_B, TAP_FC_A, TAP_FC_B, TAP_US, TAP_DSK = range(11)  # US / DSK: reference harness only
# float taps
TAP_DEC_A0, TAP_DEC_B0, TAP_FM_A, TAP_FM_B, TAP_FR_A, TAP_FR_B = 0, 5, 10, 11, 12, 13


def ref_lib_path(fast=False):
    return os.path.join(HERE, "_ref", "libaisref_fast.so" if fast else "libaisref.so")


def port_lib_path():
    return os.path.join(HERE, "libaisoracle.so")


def have_ref(fast=False):
    return os.path.exists(ref_lib_path(fast))


def have_port():
    return os.path.exists(port_lib_path())


class Msg:
    __slots__ = ("channel", "nbits", "start_idx", "end_idx", "level", "ppm", "payload", "nmea")

    def __init__(self, line):
        p = line.split("|")
        self.channel = p[0]
        self.nbits = int(p[1])
        self.start_idx = int(p[2])
        self.end_idx = int(p[3])
        self.level = float(p[4])
        self.ppm = float(p[5])
        self.payload = bytes.fromhex(p[6])
        self.nmea = p[7].split(" ") if p[7] else []

    def key(self):
        return (self.channel, self.nbits, self.payload, tuple(self.nmea))

    def __repr__(self):
        return "Msg(%s,%d,%s)" % (self.channel, self.nbits, ";".join(self.nmea))


def _bind(lib, prefix):
    f = getattr(lib, prefix + "_create")
    f.restype = C.c_void_p
    f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int]
    f = getattr(lib, prefix + "_push")
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
    for n in ("_tap_c", "_tap_ppm", "_tap_f"):
        f = getattr(lib, prefix + n)
        f.restype = C.c_long
        f.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_long]
    f = getattr(lib, prefix + "_msg_count")
    f.restype = C.c_long
    f.argtypes = [C.c_void_p]
    f = getattr(lib, prefix + "_messages")
    f.restype = C.c_long
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_long]
    f = getattr(lib, prefix + "_destroy")
    f.restype = None
    f.argtypes = [C.c_void_p]
    f = getattr(lib, prefix + "_publishers", None)
    if f is not None:
        f.restype = C.c_long
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_long]


_libs = {}


def ref_format(kind, payload, nbits, channel="A", station=0, own_mmsi=-1, start_idx=0, end_idx=0, rxtime_us=0, toa_us=0, level=0.0,
               ppm=0.0, version=0, driver=0, hardware="", mode=3, status=0, ipv4=0, uuid="", include_ssl=False, suffix=None):
    """The reference's own formatters on a message built from these fields (ref_harness.cpp aisref_format):
    kind 0 Message::getNMEAJSON, 1 getBinaryNMEA without CRC, 2 with CRC.  Returns (output bytes, [sentence bytes])."""
    lib = _load(ref_lib_path(False), "aisref")
    f = lib.aisref_format
    f.restype = C.c_long
    f.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_longlong, C.c_longlong, C.c_longlong, C.c_longlong,
                  C.c_float, C.c_float, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_uint, C.c_char_p, C.c_int, C.c_char_p,
                  C.c_char_p, C.c_long, C.c_char_p, C.c_long]
    out = C.create_string_buffer(8192)
    nm = C.create_string_buffer(1024)
    data = bytes(payload) + bytes(140 - len(payload))
    n = f(kind, data, nbits, ord(channel), station, own_mmsi, start_idx, end_idx, rxtime_us, toa_us, level, ppm, version, driver,
          hardware.encode("latin-1"), mode, status, ipv4, uuid.encode("latin-1"), 1 if include_ssl else 0,
          None if suffix is None else suffix.encode("latin-1"), out, 8192, nm, 1024)
    if n < 0:
        raise RuntimeError("aisref_format: buffer too small")
    return out.raw[:n], nm.raw.split(b"\n")[:-1]


def _load(path, prefix):
    if path not in _libs:
        lib = C.CDLL(path)
        _bind(lib, prefix)
        _libs[path] = lib
    return _libs[path]


class _Model:
    _prefix = None

    def __init__(self, lib, model=MODEL_DEFAULT, sample_rate=1536000, fmt=FMT_CF32, flags=DEFAULT_FLAGS,
                 taps=False, own_mmsi=-1):
        self.lib = lib
        self.p = self._prefix
        if taps:
            flags |= FLAG_TAPS
        self.h = getattr(lib, self.p + "_create")(model, sample_rate, fmt, flags, own_mmsi)
        if not self.h:
            raise RuntimeError("%s_create failed (model=%d rate=%d)" % (self.p, model, sample_rate))
        self.fmt = fmt

    def push(self, chunk):
        """One device callback: chunk is complex64[n] (CF32) or uint8/int8/int16[2n]."""
        a = np.ascontiguousarray(chunk)
        getattr(self.lib, self.p + "_push")(self.h, a.ctypes.data_as(C.c_void_p), a.nbytes)

    def run(self, x, chunk):
        """Feed x in chunks of `chunk` complex samples (the tail that does not fill a chunk is dropped)."""
        per = 1 if self.fmt == FMT_CF32 else 2
        n = (len(x) // per) // chunk
        for i in range(n):
            self.push(x[i * chunk * per:(i + 1) * chunk * per])
        return self

    def _tap(self, fn, tap, dtype):
        f = getattr(self.lib, self.p + fn)
        n = f(self.h, tap, None, 0)
        if n < 0:
            raise ValueError("bad tap %d" % tap)
        out = np.empty(n, dtype=np.float32)
        if n:
            f(self.h, tap, out.ctypes.data_as(C.c_void_p), n)
        return out.view(dtype)

    def tap_c(self, tap):
        return self._tap("_tap_c", tap, np.complex64)

    def tap_ppm(self, tap):
        return self._tap("_tap_ppm", tap, np.float32)

    def tap_f(self, tap):
        return self._tap("_tap_f", tap, np.float32)

    def msg_count(self):
        return getattr(self.lib, self.p + "_msg_count")(self.h)

    def messages(self):
        f = getattr(self.lib, self.p + "_messages")
        n = f(self.h, None, 0)
        buf = C.create_string_buffer(n + 1)
        f(self.h, buf, n)
        txt = buf.raw[:n].decode("ascii", "replace")
        return [Msg(l) for l in txt.split("\n") if l]

    def publishers(self):
        """The decoder that published each message messages() has not yet returned, in order (see CHALLENGER_ORDER for
        ModelChallenger's numbering; the reference harness records ModelChallenger's only).  Call it before messages()."""
        f = getattr(self.lib, self.p + "_publishers")
        n = f(self.h, None, 0)
        out = np.zeros(n, dtype=np.int32)
        if n:
            f(self.h, out.ctypes.data_as(C.c_void_p), n)
        return out.tolist()

    def close(self):
        if self.h:
            getattr(self.lib, self.p + "_destroy")(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RefModel(_Model):
    _prefix = "aisref"

    def __init__(self, *a, fast=False, **kw):
        super().__init__(_load(ref_lib_path(fast), "aisref"), *a, **kw)


class PortModel(_Model):
    _prefix = "aisorc"

    def __init__(self, *a, **kw):
        super().__init__(_load(port_lib_path(), "aisorc"), *a, **kw)

    def challenger_order(self, order):
        """Test hook: step ModelChallenger's ten decoders in this order (a permutation of 0..9) within each group."""
        f = self.lib.aisorc_challenger_order
        f.restype = C.c_int
        f.argtypes = [C.c_void_p, C.c_void_p]
        a = (C.c_int * 10)(*order)
        if f(self.h, a) != 0:
            raise ValueError("not a permutation of the ten decoders: %r" % (order,))
