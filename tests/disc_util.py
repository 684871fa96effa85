"""Shared pieces of the FM-discriminator input model (-m 3) tests: a seeded stereo stimulus (two discriminator outputs, channel A in
I and channel B in Q), writers for the four raw formats, the cases of tests/golden/disc.json, and the reference run that produced the
file (tests/golden/make_golden_disc.py)."""
import hashlib
import json
import os

import numpy as np

import aissynth as S
import oracle as O
import oracle_disc as OD

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DISC = os.path.join(HERE, "golden", "disc.json")

# name, fs, N (samples per submit), nchunks, fmt, letters, seed
CASES = [
    ("cs16_48k", 48000, 4096, 6, O.FMT_CS16, "AB", 1),
    ("cf32_48k", 48000, 4096, 6, O.FMT_CF32, "AB", 2),
    ("cu8_48k", 48000, 4096, 6, O.FMT_CU8, "AB", 3),
    ("cs8_48k", 48000, 4096, 6, O.FMT_CS8, "AB", 4),
    ("cs16_48k_xx", 48000, 2048, 12, O.FMT_CS16, "XX", 5),
    ("cs16_44k1", 44100, 4416, 6, O.FMT_CS16, "AB", 6),
    ("cf32_32k", 32000, 3200, 8, O.FMT_CF32, "AB", 7),
    ("cs16_22k05", 22050, 2240, 10, O.FMT_CS16, "XX", 8),
    ("cf32_12k", 12000, 1024, 16, O.FMT_CF32, "AB", 9),
    ("type5_48k", 48000, 8192, 4, O.FMT_CS16, "AB", 10),
]

# engine taps <-> harness taps (ref_harness_disc.cpp); per channel
FTAPS = {"C": (OD.TAP_RP, OD.TAP_IP), "FR": (O.TAP_FR_A, O.TAP_FR_B)}
FTAPS.update({"DEC%d" % i: (O.TAP_DEC_A0 + i, O.TAP_DEC_B0 + i) for i in range(5)})


def _burst_train(rng, fs, n, per_sec, type5=False):
    """Bursts (start, bits) of one side.  type5: a two-sentence type 5 first, then the reference's known answers."""
    k = int(rng.integers(per_sec[0], per_sec[1] + 1) * n / fs + 0.999)
    fixed = [S.type5_like_bits(rng), S.payload_to_bits(S.SAMPLE_A), S.payload_to_bits(S.SAMPLE_B)] if type5 else []
    out, t = [], 0
    for i in range(max(k, len(fixed))):
        bits = fixed[i] if i < len(fixed) else S.random_message_bits(rng)
        ln = S.burst_len_samples(len(bits), fs)
        gap = int(rng.integers(ln // 8, max(ln // 8 + 1, n // max(k, 1) - ln)))
        start = t + gap
        if start + ln >= n:
            break
        out.append((start, bits))
        t = start + ln
    return out


def discriminator_audio(fs, n, bursts, rng, noise_sigma=0.05):
    """What a receiver's discriminator tap gives for one channel: the phase increment angle(x[n] conj(x[n-1])) / pi of a noisy GMSK
    baseband, times a random gain, plus a small DC offset, clipped to the sound card's [-1, 1)."""
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * noise_sigma
    for start, bits in bursts:
        bb = S.gmsk_baseband(S.frame_bits(bits), fs, timing_frac=rng.uniform(0, 1))
        n1 = min(n, start + len(bb))
        x[start:n1] += rng.uniform(0.3, 1.0) * bb[:n1 - start] * np.exp(1j * rng.uniform(0, 2 * np.pi))
    d = np.zeros(n)
    d[1:] = np.angle(x[1:] * np.conj(x[:-1])) / np.pi
    return np.clip(d * rng.uniform(2.0, 6.0) + rng.uniform(-0.02, 0.02), -1.0, 1.0 - 2.0 ** -15)


def stereo(fs, n, seed, type5=False):
    """complex64[n]: channel A's discriminator audio in I, channel B's in Q, independent traffic (bursts on one side only, too).
    type5: each side starts with its own two-sentence type 5, then SAMPLE_A and SAMPLE_B, at its own times."""
    rng = np.random.default_rng(0xD15C00 + seed)
    a = _burst_train(rng, fs, n, (4, 9), type5)
    b = _burst_train(rng, fs, n, (2, 5), type5)
    x = discriminator_audio(fs, n, a, rng) + 1j * discriminator_audio(fs, n, b, rng)
    return x.astype(np.complex64)


def to_raw(x, fmt):
    """(raw array, elements per stereo frame) of the stereo signal in one of the four formats (CS16 is what a sound card gives)."""
    if fmt == O.FMT_CF32:
        return x, 1
    v = np.empty(2 * len(x), dtype=np.float64)
    v[0::2], v[1::2] = x.real, x.imag
    if fmt == O.FMT_CS16:
        return np.clip(np.round(v * 32768.0), -32768, 32767).astype(np.int16), 2
    q = np.clip(np.round(v * 128.0), -128, 127)
    if fmt == O.FMT_CS8:
        return q.astype(np.int8), 2
    return (q + 128).astype(np.uint8), 2


def stream_input(fs, n, seed, fmt, type5=False):
    return to_raw(stereo(fs, n, seed, type5), fmt)


def fbits(v):
    return int(np.float32(v).view(np.uint32))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def msg_rec(q):
    return {"ch": q.channel, "nbits": q.nbits, "payload": q.payload.hex(), "nmea": q.nmea, "start": q.start_idx, "end": q.end_idx,
            "level": fbits(q.level), "ppm": fbits(q.ppm)}


def ref_run(fs, N, nchunks, fmt, letters, raw, per):
    """The compiled reference's ModelDiscriminator over one stream: messages per chunk, and per tap name and channel the arrays each
    chunk produced (tap "US" is the complex Upsample output)."""
    m = OD.RefModelDisc(sample_rate=fs, fmt=fmt, taps=True, letters=letters)
    taps = {"%s_%d" % (k, ch): [] for k in FTAPS for ch in (0, 1)}
    taps["US"] = []
    chunks = []
    for c in range(nchunks):
        m.push(raw[c * N * per:(c + 1) * N * per])
        for k, t in FTAPS.items():
            for ch in (0, 1):
                taps["%s_%d" % (k, ch)].append(m.tap_f(t[ch]))
        taps["US"].append(m.tap_c(O.TAP_US))
        chunks.append([msg_rec(q) for q in m.messages()])
    m.close()
    return chunks, taps


def record(chunks, taps):
    return {"messages": chunks, "taps": {k: [int(sum(len(a) for a in v)), sha(np.concatenate(v) if v else np.zeros(0, np.float32))]
                                         for k, v in taps.items()}}


def load():
    with open(GOLDEN_DISC) as f:
        return json.load(f)["cases"]


def case_input(case):
    raw, per = stream_input(case["fs"], case["N"] * case["nchunks"], case["seed"], case["fmt"], case["name"].startswith("type5"))
    assert sha(raw) == case["input_sha256"], "seeded generator no longer reproduces the golden input"
    return raw, per
