"""Shared pieces of the single-channel (-c X) tests: the cases of tests/golden/mode_x.json, their seeded inputs in every raw
format, and the reference run that produced the file (tests/golden/make_golden_x.py)."""
import hashlib
import json
import os

import numpy as np

import aissynth as S
import oracle as O
import oracle_x as OX

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_X = os.path.join(HERE, "golden", "mode_x.json")

NOEMA = O.FLAG_AFC_WIDE | O.FLAG_DROOP
NODROOP = O.FLAG_PS_EMA | O.FLAG_AFC_WIDE

# name, model, fs, N (samples per submit), nchunks, fmt, flags, seed
CASES = [
    ("default_48k", O.MODEL_DEFAULT, 48000, 4096, 6, O.FMT_CF32, O.DEFAULT_FLAGS, 1),
    ("standard_48k", O.MODEL_STANDARD, 48000, 4096, 6, O.FMT_CF32, O.DEFAULT_FLAGS, 2),
    ("base_48k", O.MODEL_BASE, 48000, 4096, 6, O.FMT_CF32, O.DEFAULT_FLAGS, 3),
    # short blocks: bursts straddle block boundaries, so the level a row carries from block to block is exercised
    ("challenger_48k", O.MODEL_CHALLENGER, 48000, 1024, 24, O.FMT_CF32, O.DEFAULT_FLAGS, 4),
    ("v2_48k", O.MODEL_V2, 48000, 4096, 6, O.FMT_CF32, O.DEFAULT_FLAGS, 5),
    ("default_96k_cu8", O.MODEL_DEFAULT, 96000, 8192, 6, O.FMT_CU8, O.DEFAULT_FLAGS, 6),
    ("default_192k_cs16", O.MODEL_DEFAULT, 192000, 16384, 6, O.FMT_CS16, O.DEFAULT_FLAGS, 7),
    ("default_96k_nodroop", O.MODEL_DEFAULT, 96000, 8192, 6, O.FMT_CF32, NODROOP, 8),
    ("default_96k_noema", O.MODEL_DEFAULT, 96000, 8192, 6, O.FMT_CF32, NOEMA, 9),
    ("default_12k", O.MODEL_DEFAULT, 12000, 1024, 8, O.FMT_CF32, O.DEFAULT_FLAGS, 10),
    ("default_150k", O.MODEL_DEFAULT, 150000, 12800, 6, O.FMT_CF32, O.DEFAULT_FLAGS, 11),
]

CTAPS = {"IN": O.TAP_ROT_IN, "C": O.TAP_CA, "CGF": O.TAP_CGF_A, "FC": O.TAP_FC_A, "US": O.TAP_US}
FTAPS = {"FM": O.TAP_FM_A, "FR": O.TAP_FR_A}
FTAPS.update({"DEC%d" % i: O.TAP_DEC_A0 + i for i in range(5)})


def x_stream(fs, n_samples, stream_id, bursts_per_sec=(4, 10), noise_sigma=0.02, base_seed=0x5C11A7):
    """Single-channel (-c X) stimulus: complex baseband already centred on one AIS channel, bursts at 0 Hz plus a small
    offset (+-600 Hz).  Returns (complex64 samples, list of aissynth.Burst).  Its own RNG streams, built from aissynth's pieces."""
    rng = np.random.default_rng(base_seed + stream_id)
    dur = n_samples / fs
    k = int(rng.integers(bursts_per_sec[0], bursts_per_sec[1] + 1) * dur + 0.999)
    bursts = []
    t = 0
    for _ in range(k):
        bits = S.random_message_bits(rng)
        ln = S.burst_len_samples(len(bits), fs)
        gap = int(rng.integers(ln // 8, max(ln // 8 + 1, (n_samples // max(k, 1)) - ln)))
        start = t + gap
        if start + ln >= n_samples:
            break
        bursts.append(S.Burst(start, "X", bits, amp=rng.uniform(0.05, 0.6), foffs=rng.uniform(-600, 600), timing=rng.uniform(0, 1)))
        t = start + ln
    rng2 = np.random.default_rng(base_seed * 7 + stream_id)
    x = (rng2.standard_normal(n_samples) + 1j * rng2.standard_normal(n_samples)) * noise_sigma
    for b in bursts:
        bb = S.gmsk_baseband(S.frame_bits(b.bits), fs, timing_frac=b.timing)
        n1 = min(n_samples, b.start + len(bb))
        kk = np.arange(b.start, n1)
        x[b.start:n1] += b.amp * bb[:n1 - b.start] * np.exp(1j * (2 * np.pi * b.foffs * kk / fs + rng2.uniform(0, 2 * np.pi)))
    return x.astype(np.complex64), bursts


def to_raw(x, fmt):
    """(raw array, elements per complex sample) of a complex64 stream in one of the engine's input formats."""
    if fmt == O.FMT_CF32:
        return x, 1
    if fmt == O.FMT_CU8:
        return S.to_cu8(x), 2
    if fmt == O.FMT_CS8:
        return (S.to_cu8(x).astype(np.int16) - 128).astype(np.int8), 2
    v = np.empty(2 * len(x), dtype=np.float32)
    v[0::2], v[1::2] = x.real, x.imag
    return np.clip(np.round(v * 32767.0), -32768, 32767).astype(np.int16), 2


def stream_input(fs, n, seed, fmt):
    return to_raw(x_stream(fs, n, seed)[0], fmt)


def fbits(v):
    return int(np.float32(v).view(np.uint32))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def ref_run(model, fs, N, nchunks, fmt, flags, raw, per):
    """The compiled reference in mode X over one stream: messages per chunk, and (count, sha256) of every tap."""
    m = OX.RefModelX(model=model, sample_rate=fs, fmt=fmt, flags=flags, taps=True)
    taps = {k: [] for k in list(CTAPS) + list(FTAPS)}
    chunks = []
    for c in range(nchunks):
        m.push(raw[c * N * per:(c + 1) * N * per])
        for k, t in CTAPS.items():
            taps[k].append(m.tap_c(t))
        for k, t in FTAPS.items():
            taps[k].append(m.tap_f(t))
        chunks.append([{"ch": q.channel, "nbits": q.nbits, "payload": q.payload.hex(), "nmea": q.nmea, "start": q.start_idx,
                        "end": q.end_idx, "level": fbits(q.level), "ppm": fbits(q.ppm)} for q in m.messages()])
    m.close()
    return chunks, taps


def record(chunks, taps):
    return {"messages": chunks, "taps": {k: [int(sum(len(a) for a in v)), sha(np.concatenate(v) if v else np.zeros(0, np.float32))]
                                         for k, v in taps.items()}}


def load():
    with open(GOLDEN_X) as f:
        return json.load(f)["cases"]


def case_input(case):
    raw, per = stream_input(case["fs"], case["N"] * case["nchunks"], case["seed"], case["fmt"])
    assert sha(raw) == case["input_sha256"], "seeded generator no longer reproduces the golden input"
    return raw, per
