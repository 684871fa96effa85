"""TEST INFRASTRUCTURE -- ctypes front end of the frequency-correction probe (oracle/ref_harness_afc.cpp, built by oracle/afc.mk).

``RefModelAFC`` : the UNMODIFIED reference behind oracle/_ref/libaisref_afc.so (mode "ab") or libaisrefx_afc.so ("x", single-channel
                  mode): the harness of that mode, plus v2_state() (the V2 engines' state after the last push) and the DD_TRAIN /
                  DD_WEIGHT pair of model 11.  Same methods and taps as oracle.RefModel / oracle_x.RefModelX.
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

import numpy as np

import oracle as O

_LIBS = {"ab": "libaisref_afc.so", "x": "libaisrefx_afc.so"}


def lib_path(mode="ab"):
    return os.path.join(O.HERE, "_ref", _LIBS[mode])


def have_ref(mode="ab"):
    return os.path.exists(lib_path(mode))


class V2State:
    """One V2::Engine after a push: slot_ema (complex64), norm2 (float32, as the reference computes it), slot_phase, ppm, ppm_prev,
    ppm_split, prominence, last_f, sample_idx, busy (what the next block reads) and mag (float32[512], the last estimate's
    fftshift-ordered magnitudes)."""
    __slots__ = ("slot_ema", "norm2", "slot_phase", "ppm", "ppm_prev", "ppm_split", "prominence", "last_f", "sample_idx", "busy", "mag")


class RefModelAFC(O._Model):
    _prefix = "aisref"  # push / taps / messages / destroy are the harness's own entry points

    def __init__(self, model=O.MODEL_V2, sample_rate=1536000, fmt=O.FMT_CF32, flags=O.DEFAULT_FLAGS, taps=False, own_mmsi=-1, mode="ab",
                 weights=None):
        self.lib = O._load(lib_path(mode), "aisref")
        self.p = self._prefix
        f = self.lib.aisrefx_create if mode == "x" else self.lib.aisref_create
        f.restype = C.c_void_p
        f.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int]
        self.h = f(model, sample_rate, fmt, flags | (O.FLAG_TAPS if taps else 0), own_mmsi)
        if not self.h:
            raise RuntimeError("reference harness (%s) create failed (model=%d rate=%d)" % (mode, model, sample_rate))
        self.fmt = fmt
        s = self.lib.aisref_v2_state
        s.restype = C.c_int
        s.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        w = self.lib.aisref_v2_weights
        w.restype = C.c_int
        w.argtypes = [C.c_void_p, C.c_float, C.c_float]
        if weights is not None and w(self.h, weights[0], weights[1]):
            raise RuntimeError("DD_TRAIN / DD_WEIGHT need model 11")

    def v2_state(self, ch=0):
        f = np.zeros(7, np.float32)
        i = np.zeros(4, np.int64)
        mag = np.zeros(512, np.float32)
        if self.lib.aisref_v2_state(self.h, ch, f.ctypes.data, i.ctypes.data, mag.ctypes.data):
            raise RuntimeError("v2_state needs model 11")
        s = V2State()
        s.slot_ema = np.complex64(complex(f[0], f[1]))
        s.ppm, s.ppm_prev, s.prominence, s.last_f, s.norm2 = f[2], f[3], f[4], f[5], f[6]
        s.slot_phase, s.ppm_split, s.sample_idx, s.busy = int(i[0]), int(i[1]), int(i[2]), bool(i[3])
        s.mag = mag
        return s
