"""Seeded stimuli for frequency correction over its whole range: AIS traffic whose carrier sits anywhere the estimators can reach
and beyond, a carrier that drifts across the whole range, and slot-aligned traffic that locks the V2 engine's slot predictor.
tests/test_afc.py proves on the reference that each one reaches the branch it exists for; tests/test_gpu_afc.py compares the
engine with the reference on them, bit for bit.

The carriers, in Hz at 48 kHz (one bin of the squared 512-point spectrum is 93.75 Hz, so a carrier moves 46.875 Hz per bin):
  ModelDefault / ModelChallenger, AFC wide (the default)   about +-9.7 kHz   (fz in [-205, 208])
  ModelDefault / ModelChallenger, AFC narrow               about +-0.8 kHz   (fz in [-17, 18])
  ModelEngineV2 (FreqOffset::Estimate)                     about +-9.6 kHz

rows(fs, offsets, seconds, seed)  one stream per carrier offset: dense traffic on channel A at +offset and on channel B at -offset,
                                  so the two channels' estimates differ; every 512-sample block at 48 kHz carries a burst
drift(fs, seconds, seed)          the carrier ramps from -DRIFT_HZ to +DRIFT_HZ over the run (channel B the other way)
slotted(fs, phase, seed, ...)     bursts that start at 48 kHz sample k * 1280 + phase (+- a few samples), in consecutive slots,
                                  on carriers that alternate from burst to burst; then bursts at random phases, then noise
mode X (kind=X_): one channel at 0 Hz instead of A and B.

The bursts are a small pool of messages rendered once at baseband (aissynth.gmsk_baseband) and mixed to their carriers here, so a
sweep of a hundred rows costs seconds.  The generators of aissynth / mode_x_util are used, not changed.
"""
import numpy as np

import aissynth as S
import mode_x_util as X

AB, X_ = "ab", "x"
SLOT = 1280  # SOTDMA slot at 48 kHz

# the sweep: a coarse grid past both edges, fine grids across the edges of the wide (V2 and CGF) and of the narrow range
COARSE = [float(f) for f in np.arange(-12000.0, 12000.0 + 1, 500.0)]
FINE_WIDE = [float(s * f) for s in (-1, 1) for f in np.arange(9300.0, 9900.0 + 1, 25.0)]
FINE_NARROW = [float(s * f) for s in (-1, 1) for f in np.arange(650.0, 950.0 + 1, 25.0)]
SWEEP = COARSE + FINE_WIDE + FINE_NARROW
DRIFT_HZ = 9000.0
SLOT_OFFSETS = (-1500.0, 2000.0)  # carriers the slot-aligned bursts alternate between (channel B: the negated pair)

_pools = {}


def _pool(fs, k=8):
    """k baseband bursts (unit amplitude, complex128) of random 168-bit messages at rate fs, rendered once per rate."""
    if fs not in _pools:
        rng = np.random.default_rng(0xAFC0 + fs % 9973)
        _pools[fs] = [S.gmsk_baseband(S.frame_bits(S.random_message_bits(rng)), fs, timing_frac=float(rng.uniform(0, 1)))
                      for _ in range(k)]
    return _pools[fs]


def _place(y, starts, pool, rng, amp):
    """Adds bursts from the pool to y at the given input-sample starts, each with its own amplitude and phase."""
    n = len(y)
    for s in starts:
        b = pool[int(rng.integers(0, len(pool)))]
        e = min(n, s + len(b))
        if e > s:
            y[s:e] += (rng.uniform(*amp) * np.exp(2j * np.pi * rng.uniform(0, 1))) * b[:e - s]
    return y


def _dense_starts(fs, n, rng, gap_ms=(0.5, 4.0)):
    """Burst starts back to back with gaps of gap_ms: no 512-sample block at 48 kHz (10.7 ms) lies between two bursts."""
    ln = len(_pool(fs)[0])
    out, t = [], int(rng.integers(0, fs // 200))
    while t < n:
        out.append(t)
        t += ln + int(rng.uniform(*gap_ms) * fs / 1000.0)
    return out


def _mix(parts, fs, n, rng, noise_sigma):
    """Noise plus each (baseband, carrier) where carrier is a frequency in Hz or an array of per-sample frequencies."""
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * noise_sigma
    k = np.arange(n, dtype=np.float64)
    for y, f in parts:
        if np.ndim(f) == 0:
            ph = 2 * np.pi * f * k / fs
        else:
            ph = 2 * np.pi * np.concatenate([[0.0], np.cumsum(f[:-1])]) / fs
        x += y * np.exp(1j * ph)
    return x.astype(np.complex64)


def _centre(kind, ch):
    return 0.0 if kind == X_ else (-25000.0 if ch == 0 else 25000.0)


def row(fs, n, offset, seed, kind=AB, noise_sigma=0.02):
    """One sweep row: dense traffic on channel A at +offset and on channel B at -offset (mode X: one channel at +offset)."""
    rng = np.random.default_rng(0xAFC1 + seed)
    parts = []
    for ch, sign in ((0, 1.0), (1, -1.0))[:1 if kind == X_ else 2]:
        y = _place(np.zeros(n, np.complex128), _dense_starts(fs, n, rng), _pool(fs), rng, (0.15, 0.6))
        parts.append((y, _centre(kind, ch) + sign * offset))
    return _mix(parts, fs, n, rng, noise_sigma)


def rows(fs, n, offsets, seed=0, kind=AB):
    return [row(fs, n, f, seed + i, kind) for i, f in enumerate(offsets)]


def drift(fs, n, seed, kind=AB, hz=DRIFT_HZ):
    """Dense traffic whose carrier ramps linearly from -hz to +hz over the n samples (channel B from +hz to -hz)."""
    rng = np.random.default_rng(0xAFC2 + seed)
    ramp = np.linspace(-hz, hz, n)
    parts = []
    for ch, sign in ((0, 1.0), (1, -1.0))[:1 if kind == X_ else 2]:
        y = _place(np.zeros(n, np.complex128), _dense_starts(fs, n, rng), _pool(fs), rng, (0.15, 0.6))
        parts.append((y, _centre(kind, ch) + sign * ramp))
    return _mix(parts, fs, n, rng, noise_sigma=0.02)


def slotted(fs, n, phase, seed, kind=AB, aligned=12, misaligned=6, jitter=2, offsets=SLOT_OFFSETS, b_shift=128, every=2):
    """Slot-aligned traffic: `aligned` bursts in consecutive slots, burst j starting at 48 kHz sample (j + 1) * SLOT + phase +
    U[-jitter, jitter], on carriers that alternate between offsets[0] and offsets[1]; then `misaligned` bursts one and a half slots
    apart plus a random shift (their slot phases disagree and the lock decays); then noise to the end.  Channel B (AB) has the same
    layout at phase + b_shift and the negated carriers.  Returns complex64[n]."""
    rng = np.random.default_rng(0xAFC3 + seed)
    r = fs / 48000.0
    pool = _pool(fs)
    parts = []
    for ch, sign, ph in ((0, 1.0, phase), (1, -1.0, phase + b_shift))[:1 if kind == X_ else 2]:
        y = np.zeros(n, np.complex128)
        f = np.full(n, _centre(kind, ch))
        t48 = []
        for j in range(aligned):
            t48.append((every * j + 1) * SLOT + ph + int(rng.integers(-jitter, jitter + 1)))
        t = t48[-1]
        for j in range(misaligned):
            t += SLOT + SLOT // 2 + int(rng.integers(0, SLOT // 2))
            t48.append(t)
        starts = [int(round(s * r)) for s in t48]
        for j, s in enumerate(starts):
            if s >= n:
                break
            e = min(n, s + int(SLOT * r))
            f[s:e] += sign * offsets[j % 2]
            _place(y, [s], pool, rng, (0.5, 0.6))
        parts.append((y, f))
    return _mix(parts, fs, n, rng, noise_sigma=0.02)


def slot_span(aligned=10, misaligned=6):
    """48 kHz samples until the last slotted burst has ended (the noise after it is what decays the lock in silence)."""
    return (aligned + 1) * SLOT + misaligned * 2 * SLOT + 2 * SLOT


def to_raw(x, fmt):
    return X.to_raw(x, fmt)


# the run length of one sweep row, in 48 kHz samples (16 blocks of 512: 0.17 s), and of the drift row
SWEEP_N48 = 8192
DRIFT_N48 = 96000
# slot phases (48 kHz samples) that put the learned slot phase P at 0, 1 and 255 mod 256, so that the split e = P - sample_idx
# (mod 1280) of the locked blocks is 0 / 256, 1 / 257 and 255 / 511; channel B sits 128 samples later (AB at 1536 kS/s, mode X at
# 48 kS/s: the front ends delay the channel differently).  tests/test_afc.py checks the splits they reach.
SLOT_PHASES = {AB: (9, 10, 8), X_: (13, 14, 12)}
SLOT_N48 = 48000
SILENT_N48 = 48000 * 26  # 0.9999 per block: a lock of |slot_ema| ~ 0.93 decays below 0.8 after ~1500 blocks (16 s) of noise


def v2_estimate(mag):
    """FreqOffset::Estimate's search on the magnitudes it left behind (V2Engine.cpp:74-130), in binary32 and in its order:
    (wi, fz, frac before the clamp, frac, f).  tests/test_afc.py checks f against the reference's own last_f."""
    m = np.asarray(mag, np.float32)
    f32 = np.float32
    rs = f32(0.0)
    for j in range(133):
        rs = f32(rs + m[j])
    wm = f32(rs + f32(f32(0.6) * f32(m[15] + m[117])))
    wi = 0
    for i in range(1, 512 - 133 + 1):
        rs = f32(f32(rs - m[i - 1]) + m[i + 132])
        v = f32(rs + f32(f32(0.6) * f32(m[i + 15] + m[i + 117])))
        if v > wm:
            wm, wi = v, i
    fz, mx = -1, f32(0.0)
    for i in range(wi, wi + 31):
        h = f32(m[i] + m[i + 102])
        if h > mx:
            mx, fz = h, i
    if fz < 0:
        return wi, fz, None, None, f32(0.0)
    raw = frac = f32(0.0)
    if fz > 0 and fz + 103 < 512:
        a = f32(m[fz - 1] + m[fz + 101])
        c = f32(m[fz + 1] + m[fz + 103])
        den = f32(f32(a - f32(f32(2.0) * mx)) + c)
        if den < 0:
            raw = f32(f32(f32(0.5) * f32(a - c)) / den)
            frac = f32(min(max(raw, f32(-0.5)), f32(0.5)))
    f = f32(f32(f32(256.0) - f32(f32(f32(fz) + frac) + f32(51.0))) / f32(2.0)) / f32(512.0)
    return wi, fz, raw, frac, f32(f)


# two tones whose squares fall on bins b and b + 102 of the squared 512-point spectrum at 48 kHz (fftshift order, bin k at
# -24000 + 93.75 k Hz): FreqOffset::Estimate's window sits at an end of its range and its peak on the window's first bin, fz = 0
# (no bin below it for the sub-bin step) or fz = 409 (no bin above its partner)
EDGE_TONE_BINS = (0, 409)


def edge_tones(fs, n, fz, seed, kind=AB):
    """The tone pair of EDGE_TONE_BINS entry fz on every channel (relative to its centre), under noise.  The tone at the end of the
    spectrum is strong (0.9), its partner weak (0.05): with partners of equal strength the window moves inwards to take in their
    cross product half-way between them."""
    rng = np.random.default_rng(0xAFC4 + seed)
    k = np.arange(n, dtype=np.float64)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 0.02
    for ch in range(1 if kind == X_ else 2):
        for b, amp in zip((fz, fz + 102), (0.9, 0.05) if fz < 256 else (0.05, 0.9)):
            f = _centre(kind, ch) + (-24000.0 + 93.75 * b) / 2.0
            x += amp * np.exp(1j * (2 * np.pi * f * k / fs + rng.uniform(0, 2 * np.pi)))
    return x.astype(np.complex64)
