"""TEST INFRASTRUCTURE -- ctypes front end of the reference harness for the FM-discriminator input model (-m 3).

``RefModelDisc`` : the UNMODIFIED reference's ModelDiscriminator (oracle/_ref/libaisrefd.so, built by oracle/disc.mk from
                   ref_harness_disc.cpp).  Same methods as oracle.RefModel; taps as in ref_harness_disc.cpp.
Only tests/ and the tools that check the engine may import this module; the product never does.
"""
import ctypes as C
import os

import oracle as O

# float taps of the harness (ref_harness_disc.cpp); complex tap 9 (O.TAP_US) is the Upsample output
TAP_RP, TAP_IP = O.TAP_FM_A, O.TAP_FM_B  # the real rows that feed FR_a / FR_b


def refd_lib_path():
    return os.path.join(O.HERE, "_ref", "libaisrefd.so")


def have_refd():
    return os.path.exists(refd_lib_path())


class RefModelDisc(O._Model):
    _prefix = "aisref"  # push / taps / messages are the harness's own entry points

    def __init__(self, sample_rate=48000, fmt=O.FMT_CF32, taps=False, own_mmsi=-1, letters="AB"):
        self.lib = O._load(refd_lib_path(), "aisref")
        self.p = self._prefix
        f = self.lib.aisrefd_create
        f.restype = C.c_void_p
        f.argtypes = [C.c_int, C.c_int, C.c_uint, C.c_int, C.c_char_p]
        d = self.lib.aisrefd_destroy
        d.restype = None
        d.argtypes = [C.c_void_p]
        self.h = f(sample_rate, fmt, O.FLAG_TAPS if taps else 0, own_mmsi, letters.encode())
        if not self.h:
            raise RuntimeError("aisrefd_create failed (rate=%d)" % sample_rate)
        self.fmt = fmt

    def close(self):
        if self.h:
            self.lib.aisrefd_destroy(self.h)  # the handle owns a ModelDiscriminator: aisref_destroy would not free it
            self.h = None
