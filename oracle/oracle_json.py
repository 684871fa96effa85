"""TEST INFRASTRUCTURE -- ctypes front end of the reference's full AIS JSON (oracle/_ref/libaisref_json.so, built by oracle/json.mk
from ref_harness_json.cpp).

``ref_line(data, nbits, channel, sentences, level, ppm, version, driver, hardware, mode, rxtime_us, toa_us, station)`` : the line
the UNMODIFIED reference's JSONAIS + Serializer(JSON_DICT_FULL) writes for that message, as bytes without a newline.
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
MAX_AIS_BYTES = 133  # (MAX_AIS_LENGTH + 7) / 8: Message::setBytes takes no more
_lib = None


def lib_path():
    return os.path.join(HERE, "_ref", "libaisref_json.so")


def have_ref():
    return os.path.exists(lib_path())


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(lib_path())
        lib.aisrefj_line.restype = C.c_long
        lib.aisrefj_line.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int),
                                     C.c_float, C.c_float, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_longlong, C.c_longlong,
                                     C.c_int, C.c_char_p, C.c_long]
        _lib = lib
    return _lib


_out = None


def ref_line(data, nbits, channel="A", sentences=(), level=1024.0, ppm=1024.0, version=0, driver=0, hardware="", mode=3,
             rxtime_us=0, toa_us=0, station=0):
    global _out
    lib = _load()
    data = bytes(data)[:MAX_AIS_BYTES]
    sents = [s.encode("latin-1") if isinstance(s, str) else bytes(s) for s in sentences]
    arr = (C.c_char_p * max(len(sents), 1))(*sents)
    lens = (C.c_int * max(len(sents), 1))(*[len(s) for s in sents])
    ch = channel if isinstance(channel, int) else ord(channel)
    if _out is None:
        _out = C.create_string_buffer(1 << 16)
    n = lib.aisrefj_line(data, len(data), int(nbits), ch, len(sents), arr, lens, float(level), float(ppm), int(version), int(driver),
                         hardware.encode() if isinstance(hardware, str) else hardware, int(mode), int(rxtime_us), int(toa_us),
                         int(station), _out, 1 << 16)
    if n < 0:
        raise RuntimeError("reference JSON line longer than 64 KiB")
    return _out.raw[:n]
