"""WAV files for the tests, built byte by byte with struct (never with the code under test)."""
import struct

import numpy as np

import aisgpu

TAG_BITS = {aisgpu.FMT_CF32: (3, 32), aisgpu.FMT_CU8: (1, 8), aisgpu.FMT_CS16: (1, 16)}
DTYPE = {aisgpu.FMT_CF32: np.float32, aisgpu.FMT_CU8: np.uint8, aisgpu.FMT_CS16: np.int16}


def chunk(cid, body, pad=True):
    """One RIFF chunk: id, little-endian size, body, and the pad byte of an odd body unless pad is False."""
    return cid + struct.pack("<I", len(body)) + body + (b"\0" if pad and len(body) & 1 else b"")


def fmt_chunk(tag=1, channels=2, rate=48000, bits=16, extra=b""):
    align = channels * bits // 8
    return chunk(b"fmt ", struct.pack("<HHIIHH", tag, channels, rate, rate * align, align, bits) + extra)


def riff(*chunks, riff_id=b"RIFF", wave=b"WAVE"):
    body = wave + b"".join(chunks)
    return riff_id + struct.pack("<I", len(body)) + body


def data_header(n_bytes):
    return b"data" + struct.pack("<I", n_bytes)


def wav_bytes(samples, fmt, rate, before=(), after=()):
    """A stereo WAV of the raw samples (bytes or array) in the engine's format fmt: chunks `before` between RIFF and fmt, `after`
    after the data chunk.  Returns (file bytes, data offset)."""
    tag, bits = TAG_BITS[fmt]
    data = samples if isinstance(samples, bytes) else np.ascontiguousarray(samples).tobytes()
    off = len(riff(*before, fmt_chunk(tag, 2, rate, bits))) + 8
    b = riff(*before, fmt_chunk(tag, 2, rate, bits), chunk(b"data", data), *after)
    return b, off


def write_wav(path, samples, fmt, rate, before=(), after=()):
    b, off = wav_bytes(samples, fmt, rate, before, after)
    with open(path, "wb") as f:
        f.write(b)
    return off
