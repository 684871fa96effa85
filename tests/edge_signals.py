"""Seeded edge-case stimuli: the input a real receiver delivers and Gaussian noise never does -- digital silence, dropouts, DC,
carriers, real-only and clipped samples, a few quantisation codes, very loud and subnormal floats.  Each one reaches a branch of the
engine that ordinary traffic never takes (an argmax without a maximum, exact ties, subnormals behind the front end, the rare
paths of atan2f, the FP_DS stages at full scale); tests/test_edge_signals.py proves on the reference that it does, and
tests/test_gpu_edge_signals.py compares the engine with the reference on it, bit for bit.

make(name, fs, n, seed, fmt, kind, submit, granule) returns (raw array, array elements per sample) in any of the four input
formats.  kind is the traffic the stimulus is built from: AB (two channels at -/+25 kHz, aissynth.random_stream), X (one channel
at 0 Hz, mode_x_util.x_stream) or DISC (two discriminator outputs, disc_util.stereo).

S1  silence          exact zeros for the whole run (CF32 +0.0, CU8 128, CS8 0, CS16 0)
S2  signed_zero      CF32: -0.0, then zeros of random sign
S3  gaps             traffic with exact-zero gaps (gap_ranges): one granule mid-submit, one 48 kHz CGF block (512 samples) across
                     the boundary of submits 1 and 2, and GAP_SECONDS starting inside a burst (a dropout mid-frame)
S4  dc, dc_traffic   a constant of -1 LSB of CU8 on I and Q (-1/128; CS8 -1, CS16 -256), alone and added to traffic
S5  carrier_*        a complex tone on an exact bin of the 48 kHz channel's 512-point FFT (bin, 750 Hz) or half-way between two
                     (between, 796.875 Hz), alone and under traffic (*_traffic)
S6  real_only        CF32 traffic whose imaginary parts are exactly +0.0
S7  clipped          traffic at CLIP_GAIN x full scale, clipped to the rails: CU8 0 / 255, CS8 -128 / 127, CS16 -32768 / 32767,
                     CF32 hard-limited to +-1.0
S8  quantised        CU8: noise below one LSB (codes 127 and 128 only) under bursts a few LSB strong; CS16 (DISC): audio of at
                     most +-8 LSB
S9  loud, loud_max   CF32 traffic x 2^12, and x 2^LOUD_MAX_EXP: the largest power of two for which every reference tap stays
                     finite (tests/test_edge_signals.py checks both that and that the next power overflows)
S10 subnormal        CF32 traffic x 2^-130: every input sample subnormal or zero
"""
import numpy as np

import aissynth as S
import disc_util as D
import mode_x_util as X
import oracle as O

AB, X_, DISC = "ab", "x", "disc"
CF32, CU8, CS8, CS16 = O.FMT_CF32, O.FMT_CU8, O.FMT_CS8, O.FMT_CS16

GAP_SECONDS = 0.16  # PhaseSearchEMA's level decays by 0.85 per symbol: subnormal after ~530 symbols, 0 after ~630 (66 ms at 9600 Bd)
CLIP_GAIN = 6.0
LOUD_EXP = 12
LOUD_MAX_EXP = 64  # every reference tap stays finite up to here; at 2^65 the FM taps of models 0 and 1 overflow (tests/test_edge_signals.py)
SUBNORMAL_EXP = -130
TONE_BIN_HZ, TONE_BETWEEN_HZ = 750.0, 796.875  # 48 kHz / 512 = 93.75 Hz per bin: bin 8, and bin 8.5
DC = -1.0 / 128.0

NAMES = ["silence", "signed_zero", "gaps", "dc", "dc_traffic", "carrier_bin", "carrier_between", "carrier_bin_traffic",
         "carrier_between_traffic", "real_only", "clipped", "quantised", "loud", "loud_max", "subnormal"]
CF32_ONLY = {"signed_zero", "real_only", "loud", "loud_max", "subnormal"}


def traffic(fs, n, seed, kind=AB, noise_sigma=0.02, dense=True):
    """(complex64[n], [(start, length)] of the bursts in input samples; None for DISC)."""
    if kind == DISC:
        return D.stereo(fs, n, seed), None
    per_sec = (10, 16) if dense else (2, 8)
    if kind == X_:
        x, bursts = X.x_stream(fs, n, seed, bursts_per_sec=per_sec, noise_sigma=noise_sigma)
    else:
        x, bursts = S.random_stream(fs, n, seed, bursts_per_sec=per_sec, noise_sigma=noise_sigma)
    return x, [(b.start, S.burst_len_samples(len(b.bits), fs)) for b in bursts]


def to_raw(x, fmt, kind=AB):
    return D.to_raw(x, fmt) if kind == DISC else X.to_raw(x, fmt)


def cgf_block(fs):
    """Input samples of one 512-sample block at 48 kHz."""
    return 512 * fs // 48000


def gap_ranges(fs, n, submit, granule, bursts):
    """The [start, end) input ranges S3 zeroes: one granule in the middle of submit 0, one CGF block across the boundary of
    submits 1 and 2, and GAP_SECONDS from the middle of the first burst that starts 70 ms after that (or from the middle of submit 3 when the
    traffic has no burst list), all inside [0, n)."""
    g0 = submit // 2 // granule * granule
    blk = cgf_block(fs)
    g1 = 2 * submit - blk // 2
    long_n = int(np.ceil(GAP_SECONDS * fs))
    start = None
    for b0, ln in sorted(bursts or []):
        s = b0 + ln // 2
        if s > g1 + blk + int(0.07 * fs) and s + long_n < n:  # one whole burst fits between the CGF gap and this one
            start = s
            break
    if start is None:
        start = 3 * submit + submit // 2
    out = [(g0, g0 + granule), (g1, g1 + blk), (start, min(n, start + long_n))]
    assert all(0 <= a < b <= n for a, b in out), (out, n)
    return out


def _tone(fs, n, hz, kind, amp=0.3):
    f = hz if kind == X_ else -25000.0 + hz
    k = np.arange(n, dtype=np.float64)
    return (amp * np.exp(2j * np.pi * f * k / fs)).astype(np.complex64)


def _const(n, fmt, cf32, code):
    if fmt == CF32:
        return np.full(n, cf32, np.complex64), 1
    dt = {CU8: np.uint8, CS8: np.int8, CS16: np.int16}[fmt]
    return np.full(2 * n, code, dt), 2


def _offset(raw, fmt, lsb):
    """raw integer samples moved by lsb codes, clipped to the format's rails."""
    lo, hi = {CU8: (0, 255), CS8: (-128, 127), CS16: (-32768, 32767)}[fmt]
    return np.clip(raw.astype(np.int32) + lsb, lo, hi).astype(raw.dtype)


def make(name, fs, n, seed, fmt=CF32, kind=AB, submit=None, granule=1):
    """(raw array, array elements per sample) of stimulus `name` (NAMES) with n samples."""
    if name in CF32_ONLY and fmt != CF32:
        raise ValueError("%s is a CF32 stimulus" % name)
    if name == "silence":
        return _const(n, fmt, 0.0, 128 if fmt == CU8 else 0)
    if name == "signed_zero":
        rng = np.random.default_rng(seed)
        bits = np.zeros(2 * n, np.uint32)
        bits[:n] = 0x80000000  # the first half -0.0 on I and Q, then zeros of random sign
        bits[n:] = rng.integers(0, 2, n, dtype=np.uint32) << np.uint32(31)
        return bits.view(np.float32).view(np.complex64), 1
    if name == "dc":
        return _const(n, fmt, complex(DC, DC), {CU8: 127, CS8: -1, CS16: -256}.get(fmt, 0))
    if name.startswith("carrier"):
        if kind == DISC:
            raise ValueError("no carrier stimulus for the discriminator input")
        x = _tone(fs, n, TONE_BIN_HZ if "_bin" in name else TONE_BETWEEN_HZ, kind)
        if name.endswith("_traffic"):
            x = (x + traffic(fs, n, seed, kind)[0]).astype(np.complex64)
        return to_raw(x, fmt, kind)
    if name == "quantised":
        rng = np.random.default_rng(seed)
        if kind == DISC:
            assert fmt == CS16, "the quantised discriminator stimulus is CS16"
            x = traffic(fs, n, seed, kind)[0]  # audio in [-1, 1): +-8 LSB of CS16
            return to_raw((x * np.float32(8.0 / 32768.0)).astype(np.complex64), fmt, kind)
        assert fmt == CU8, "the quantised stimulus is CU8"
        burst = traffic(fs, n, seed, kind, noise_sigma=0.0)[0]  # bursts of amplitude 0.05 .. 0.6, nothing else
        v = np.empty(2 * n)
        v[0::2], v[1::2] = burst.real, burst.imag
        noise = np.clip(-0.5 + 0.2 * rng.standard_normal(2 * n), -1.45, 0.45)  # rounds to -1 or 0: codes 127 / 128
        return (128 + np.round(noise + v * (6.0 / 0.6))).clip(0, 255).astype(np.uint8), 2
    x, bursts = traffic(fs, n, seed, kind)
    if name == "gaps":
        assert submit, "the gap layout depends on the submit length"
        x = x.copy()
        for a, b in gap_ranges(fs, n, submit, granule, bursts):
            x[a:b] = 0
        return to_raw(x, fmt, kind)
    if name == "dc_traffic":
        if fmt == CF32:
            return (x + np.complex64(complex(DC, DC))).astype(np.complex64), 1
        raw, per = to_raw(x, fmt, kind)
        return _offset(raw, fmt, -256 if fmt == CS16 else -1), per
    if name == "real_only":
        return x.real.astype(np.float32).astype(np.complex64), 1
    if name == "clipped":
        y = x.astype(np.complex128) * CLIP_GAIN
        if fmt == CF32:
            return (np.clip(y.real, -1.0, 1.0) + 1j * np.clip(y.imag, -1.0, 1.0)).astype(np.complex64), 1
        return to_raw(y, fmt, kind)
    if name in ("loud", "loud_max", "subnormal"):
        e = {"loud": LOUD_EXP, "loud_max": LOUD_MAX_EXP, "subnormal": SUBNORMAL_EXP}[name]
        return (x.astype(np.complex128) * 2.0 ** e).astype(np.complex64), 1
    raise ValueError("unknown stimulus %r" % name)
