"""TEST INFRASTRUCTURE -- ctypes front end of the reference harness in single-channel mode (-c X).

``RefModelX`` : the UNMODIFIED reference with setMode(X) (oracle/_ref/libaisrefx.so, built by oracle/mode_x.mk from
               ref_harness_x.cpp).  Same methods as oracle.RefModel; taps as in ref_harness_x.cpp (tap 0 = what feeds FCIC5_a).
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import os

import oracle as O


def refx_lib_path():
    return os.path.join(O.HERE, "_ref", "libaisrefx.so")


def have_refx():
    return os.path.exists(refx_lib_path())


class RefModelX(O._Model):
    _prefix = "aisref"  # push / taps / messages / destroy are the harness's own entry points

    def __init__(self, model=O.MODEL_DEFAULT, sample_rate=48000, fmt=O.FMT_CF32, flags=O.DEFAULT_FLAGS, taps=False, own_mmsi=-1):
        import ctypes as C
        self.lib = O._load(refx_lib_path(), "aisref")
        self.p = self._prefix
        f = self.lib.aisrefx_create
        f.restype = C.c_void_p
        f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int]
        self.h = f(model, sample_rate, fmt, flags | (O.FLAG_TAPS if taps else 0), own_mmsi)
        if not self.h:
            raise RuntimeError("aisrefx_create failed (model=%d rate=%d)" % (model, sample_rate))
        self.fmt = fmt
