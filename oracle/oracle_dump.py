"""TEST INFRASTRUCTURE -- ctypes front end of the reference harness with the 48 kHz channel dump (-go DUMP <prefix>).

``RefModelDump`` : the UNMODIFIED reference with SetKey(KEY_SETTING_DUMP, prefix) before buildModel (oracle/_ref/libaisref_dump.so,
                   built by oracle/dump.mk from ref_harness_dump.cpp).  Same methods as oracle.RefModel; with taps=True the complex
                   taps 3 / 4 are C_a / C_b.  The reference writes <prefix>_A.wav / <prefix>_B.wav and completes them at close().
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import os

import oracle as O


def refdump_lib_path():
    return os.path.join(O.HERE, "_ref", "libaisref_dump.so")


def have_refdump():
    return os.path.exists(refdump_lib_path())


def adapter_dump_path():
    return os.path.join(O.HERE, "_ref", "adapter_dump_test")


class RefModelDump(O._Model):
    _prefix = "aisref"  # push / taps / messages / destroy are the harness's own entry points

    def __init__(self, prefix, model=O.MODEL_DEFAULT, sample_rate=1536000, fmt=O.FMT_CF32, flags=O.DEFAULT_FLAGS, taps=False, own_mmsi=-1,
                 channel_mode=0, channels="AB"):
        import ctypes as C
        self.lib = O._load(refdump_lib_path(), "aisref")
        self.p = self._prefix
        f = self.lib.aisref_create_dump
        f.restype = C.c_void_p
        f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int, C.c_int, C.c_char, C.c_char, C.c_char_p]
        self.h = f(model, sample_rate, fmt, flags | (O.FLAG_TAPS if taps else 0), own_mmsi, channel_mode, channels[0].encode(),
                   channels[1].encode(), None if prefix is None else os.fsencode(prefix))
        if not self.h:
            raise RuntimeError("aisref_create_dump failed (model=%d rate=%d)" % (model, sample_rate))
        self.fmt = fmt
