"""TEST INFRASTRUCTURE -- ctypes front end of the reference's Device::WAVFile (oracle/_ref/libaisref_wav.so, built by oracle/wav.mk
from ref_harness_wav.cpp).

``ref_open(path)`` : (format, sample_rate, read position after Open) as the UNMODIFIED reference opens the file, or RefWavError
                     with the text of the exception it throws.
``ref_read(path)`` : every byte the reference's device delivers as samples.
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


class RefWavError(RuntimeError):
    pass


def lib_path():
    return os.path.join(HERE, "_ref", "libaisref_wav.so")


def have_ref():
    return os.path.exists(lib_path())


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(lib_path())
        lib.aisrefw_open.restype = C.c_int
        lib.aisrefw_open.argtypes = [C.c_char_p, C.POINTER(C.c_int), C.POINTER(C.c_uint), C.POINTER(C.c_longlong), C.c_char_p, C.c_long]
        lib.aisrefw_read.restype = C.c_long
        lib.aisrefw_read.argtypes = [C.c_char_p, C.c_void_p, C.c_long, C.c_char_p, C.c_long]
        _lib = lib
    return _lib


def ref_open(path):
    lib = _load()
    fmt, rate, pos = C.c_int(0), C.c_uint(0), C.c_longlong(0)
    err = C.create_string_buffer(1024)
    if lib.aisrefw_open(os.fsencode(path), C.byref(fmt), C.byref(rate), C.byref(pos), err, 1024):
        raise RefWavError(err.value.decode())
    return fmt.value, rate.value, pos.value


def ref_read(path):
    lib = _load()
    err = C.create_string_buffer(1024)
    n = lib.aisrefw_read(os.fsencode(path), None, 0, err, 1024)
    if n < 0:
        raise RefWavError(err.value.decode())
    buf = C.create_string_buffer(max(n, 1))
    lib.aisrefw_read(os.fsencode(path), buf, n, err, 1024)
    return buf.raw[:n]
