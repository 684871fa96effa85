"""TEST INFRASTRUCTURE -- ctypes front end of the reference's output records (oracle/_ref/libaisref_fmt.so, built by oracle/fmt.mk
from ref_harness_fmt.cpp).

``ref_record(fmt, data, nbits, ...)`` : the bytes the UNMODIFIED reference's IO::OutputMessage appends for that message in
MessageFormat ``fmt`` (1 NMEA .. 9 JSON_ANNOTATED).  ``hub(v)`` reads (and with v >= 0 sets) the output's COMMUNITY_HUB line count;
``group_seed(g)`` makes the next NMEA_TAG group ``(g % 9999) + 1``.  ``key_count()`` / ``key(k, dict, enhanced, v)`` serialise one
member for the table generator.  Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_AIS_BYTES = 133  # (MAX_AIS_LENGTH + 7) / 8: Message::setBytes takes no more
_lib = None
_out = None


def lib_path():
    return os.path.join(HERE, "_ref", "libaisref_fmt.so")


def have_ref():
    return os.path.exists(lib_path())


def _load():
    global _lib, _out
    if _lib is None:
        lib = C.CDLL(lib_path())
        lib.aisreff_record.restype = C.c_long
        lib.aisreff_record.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p),
                                       C.POINTER(C.c_int), C.c_float, C.c_float, C.c_int, C.c_int, C.c_char_p, C.c_int,
                                       C.c_longlong, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int,
                                       C.c_uint, C.c_char_p, C.c_char_p, C.c_long]
        lib.aisreff_hub.restype = C.c_longlong
        lib.aisreff_hub.argtypes = [C.c_longlong]
        lib.aisreff_group_seed.restype = C.c_int
        lib.aisreff_group_seed.argtypes = [C.c_int]
        lib.aisreff_key_count.restype = C.c_int
        lib.aisreff_key.restype = C.c_long
        lib.aisreff_key.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_long]
        _out = C.create_string_buffer(1 << 18)
        _lib = lib
    return _lib


def _b(s):
    if s is None:
        return None
    return s.encode("latin-1") if isinstance(s, str) else bytes(s)


def ref_record(fmt, data, nbits, channel="A", sentences=(), level=1024.0, ppm=1024.0, version=0, driver=0, hardware="", mode=3,
               rxtime_us=0, toa_us=0, station=0, include_ssl=False, start_idx=0, end_idx=0, uuid="", status=0, ipv4=0,
               suffix=None):
    lib = _load()
    data = bytes(data)[:MAX_AIS_BYTES]
    sents = [_b(s) for s in sentences]
    arr = (C.c_char_p * max(len(sents), 1))(*sents)
    lens = (C.c_int * max(len(sents), 1))(*[len(s) for s in sents])
    ch = channel if isinstance(channel, int) else ord(channel)
    n = lib.aisreff_record(int(fmt), data, len(data), int(nbits), ch, len(sents), arr, lens, float(level), float(ppm), int(version),
                           int(driver), _b(hardware) or b"", int(mode), int(rxtime_us), int(toa_us), int(station), int(bool(include_ssl)),
                           int(start_idx), int(end_idx), _b(uuid) or b"", int(status), int(ipv4), _b(suffix), _out, len(_out))
    if n < 0:
        raise RuntimeError("reference record longer than 256 KiB")
    return _out.raw[:n]


def hub(v=-1):
    return int(_load().aisreff_hub(int(v)))


def group_seed(g):
    n = _load().aisreff_group_seed(int(g))
    if n < 0:
        raise RuntimeError("group id %d not reached" % g)
    return n


def key_count():
    return int(_load().aisreff_key_count())


def key(k, dict_=0, enhanced=False, v=0):
    lib = _load()
    n = lib.aisreff_key(int(k), int(dict_), int(bool(enhanced)), int(v), _out, len(_out))
    if n < 0:
        raise RuntimeError("key text too long")
    return _out.raw[:n]
