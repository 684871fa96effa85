"""Shared pieces of the DC16H tests (three uint32 per sample; Convert::toFloat, Utilities/Convert.cpp:288-301): a complex stream
packed into DC16H words, and the conversion the format stands for, written out on the host.

I is the low half of word 0 and Q the low half of word 1; the sample is (I / 32768, (-Q) / 32768) with Q negated as an integer.
The two high halves and the whole third word are never read: the packer fills them with seeded garbage, so a reader that touches
them does not reproduce the reference."""
import numpy as np

import aisgpu

DC16H = aisgpu.FMT_DC16H


def pack_iq(i16, q16, seed=0):
    """uint32[3 n] from int16 I and Q (Q as stored, before the negation): garbage everywhere the format does not read."""
    i16, q16 = np.asarray(i16, dtype=np.int16), np.asarray(q16, dtype=np.int16)
    n = len(i16)
    w = np.random.default_rng(0xDC16 + seed).integers(0, 1 << 32, size=(n, 3), dtype=np.uint64).astype(np.uint32)
    w[:, 0] = (w[:, 0] & np.uint32(0xFFFF0000)) | i16.view(np.uint16).astype(np.uint32)
    w[:, 1] = (w[:, 1] & np.uint32(0xFFFF0000)) | q16.view(np.uint16).astype(np.uint32)
    return w.reshape(3 * n)


def iq_of(z):
    """int16 (I, Q as stored) of a complex64 stream: I = round(32767 re), Q = -round(32767 im), both within +-32767."""
    z = np.asarray(z, dtype=np.complex64)
    i = np.clip(np.round(z.real * 32767.0), -32767, 32767).astype(np.int16)
    q = (-np.clip(np.round(z.imag * 32767.0), -32767, 32767)).astype(np.int16)
    return i, q


def from_complex(z, seed=0):
    """(uint32[3 n], 3): the stream quantised to 16 bits and packed, in the (raw array, elements per sample) form of the suite."""
    i, q = iq_of(z)
    return pack_iq(i, q, seed), 3


def unpack(words):
    """What ConvertRAW makes of one Receive of DC16H words: complex64[size // 12 bytes]; -Q is an int32 negation, so Q = 0 gives +0.0
    and Q = -32768 gives 1.0."""
    w = np.asarray(words, dtype=np.uint32)
    n = len(w) // 3
    w = w[:3 * n].reshape(n, 3)
    i = (w[:, 0] & np.uint32(0xFFFF)).astype(np.uint16).view(np.int16).astype(np.int32)
    q = -(w[:, 1] & np.uint32(0xFFFF)).astype(np.uint16).view(np.int16).astype(np.int32)
    out = np.empty((n, 2), dtype=np.float32)
    out[:, 0] = i.astype(np.float32) / np.float32(32768.0)
    out[:, 1] = q.astype(np.float32) / np.float32(32768.0)
    return out.view(np.complex64).reshape(n)


def to_cs16(words):
    """int16[2 n] (I, -Q) of DC16H words: the CS16 stream with the same converted samples (needs Q != -32768)."""
    w = np.asarray(words, dtype=np.uint32).reshape(-1, 3)
    i = (w[:, 0] & np.uint32(0xFFFF)).astype(np.uint16).view(np.int16)
    q = (w[:, 1] & np.uint32(0xFFFF)).astype(np.uint16).view(np.int16)
    assert q.min(initial=0) > -32768
    out = np.empty(2 * len(w), dtype=np.int16)
    out[0::2], out[1::2] = i, -q
    return out
