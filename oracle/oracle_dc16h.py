"""TEST INFRASTRUCTURE -- ctypes front end of the reference harnesses fed Format::DC16H (three 32-bit words per sample).

``RefModelDC16H`` : the UNMODIFIED reference behind oracle/_ref/libaisref_dc16h.so (kind "ab"), libaisrefx_dc16h.so ("x",
                   single-channel mode) or libaisrefd_dc16h.so ("disc", the FM-discriminator input model), built by oracle/dc16h.mk
                   from ref_harness_dc16h.cpp: the harness of that kind, created as CF32 and switched to DC16H before the first push.
Same methods and taps as oracle.RefModel / oracle_x.RefModelX / oracle_disc.RefModelDisc; push takes uint32[3 n].
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

import oracle as O

FMT_DC16H = 7
_LIBS = {"ab": "libaisref_dc16h.so", "x": "libaisrefx_dc16h.so", "disc": "libaisrefd_dc16h.so"}


def lib_path(kind="ab"):
    return os.path.join(O.HERE, "_ref", _LIBS[kind])


def have_ref(kind="ab"):
    return os.path.exists(lib_path(kind))


class RefModelDC16H(O._Model):
    _prefix = "aisref"  # push / taps / messages are the harness's own entry points

    def __init__(self, model=O.MODEL_DEFAULT, sample_rate=1536000, flags=O.DEFAULT_FLAGS, taps=False, own_mmsi=-1, kind="ab", letters="AB"):
        self.lib = O._load(lib_path(kind), "aisref")
        self.p = self._prefix
        self.kind = kind
        if taps:
            flags |= O.FLAG_TAPS
        if kind == "disc":
            f = self.lib.aisrefd_create
            f.restype = C.c_void_p
            f.argtypes = [C.c_int, C.c_int, C.c_uint, C.c_int, C.c_char_p]
            self.lib.aisrefd_destroy.restype = None
            self.lib.aisrefd_destroy.argtypes = [C.c_void_p]
            self.h = f(sample_rate, O.FMT_CF32, flags & O.FLAG_TAPS, own_mmsi, letters.encode())
        else:
            f = self.lib.aisrefx_create if kind == "x" else self.lib.aisref_create
            f.restype = C.c_void_p
            f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int]
            self.h = f(model, sample_rate, O.FMT_CF32, flags, own_mmsi)
        if not self.h:
            raise RuntimeError("reference harness (%s) create failed (model=%d rate=%d)" % (kind, model, sample_rate))
        s = self.lib.aisref_set_format_dc16h
        s.restype = None
        s.argtypes = [C.c_void_p]
        s(self.h)
        self.fmt = FMT_DC16H

    def close(self):
        if self.h and self.kind == "disc":
            self.lib.aisrefd_destroy(self.h)  # the handle owns a ModelDiscriminator: aisref_destroy would not free it
            self.h = None
        super().close()
