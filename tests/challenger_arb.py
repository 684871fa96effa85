"""Stimulus for ModelChallenger's ten cross-reset decoders, built where their order within a group decides what is published.

ModelChallenger (Source/DSP/Model.cpp:601-678) runs, per channel, five decoders behind the coherent branch (FIR17 -> ScatterPLL ->
PhaseSearchEMA, a0..a4) and five behind the FM branch (FM -> Filter 37 -> Deinterleave, f0..f4), all joined by Reset.  Within a group
of five 48 kHz samples they step f0 f1 f2 f3 | a0 .. a4 | f4.  On clean bursts an FM decoder closes a frame a group or more before
any coherent one, so the order is never consulted.  The families below make it count:

* threshold: type 1 / 5 / 18 frames at amplitudes stepped across the gap between the FM and the coherent sensitivity, at timing
  offsets on a 1/20-symbol grid and carrier offsets within the CGF's range.  Coherent decoders win at the low end, FM decoders at the
  high end.  The coherent branch closes a frame 4..9 samples after the FM branch, so the two close in one group only for f0.
* null: a burst the FM branch would win, with 1..3 short deep amplitude nulls (1..3 samples at 48 kHz) on chosen data bits.  Each
  clicks the FM discriminator and barely moves the phase search, so a coherent decoder wins, at whichever phase the timing favours.
* replay: two frames back to back on one channel, built at the bit level: frame 1's closing flag, k alternations 1 0 1 .. (k = 1..4,
  one run with the flag's last bits), frame 2's flag.  Frame 2 is lost at k <= 2 and found from k = 3: the alternations counted
  after frame 1's Reset sit on the decoder's "> 4" threshold.  Three short deep nulls late in frame 1 hand it to a coherent decoder,
  so the FM decoders, a bit ahead of it, are the Reset's siblings.  Whether the winner's group counts as an alternation for a
  sibling (it does when the sibling steps after the winner, f4 after a0..a4) decides which decoder finds frame 2.
* straddle: frames placed in one-sample steps of their 48 kHz start so that the closing group straddles a 512-sample CGF block
  boundary at each of its four inner positions, with a carrier offset between FFT bins, so consecutive blocks' ppm differ.

Bits come from decoder_limits (onair_bits, hdlc), the waveform from aissynth.gmsk_baseband.  Everything is seeded.
split_schedule() derives submit lengths from the reference's own end_idx so that a submit boundary falls inside closing groups.
"""
import numpy as np

import aissynth as S
import decoder_limits as DL

BAUD = 9600.0
BLOCK = 512            # SquareFreqOffsetCorrection's block (Model.cpp:621)
LEAD = 2048            # 48 kHz samples of noise in front of a track's first burst
GAP = 640              # 48 kHz samples of noise between bursts (the decoders return to TRAINING)
FM_CLOSE_DELAY = {False: 23, True: 21}  # 48 kHz samples from the sixth closing-flag 1 (at 5 samples per bit) to an FM decoder's
                                        # end_idx, AB mode (through Downsample2CIC5) and single-channel mode at 48 kS/s
REPLAY_K = (1, 2, 3, 4)                 # alternations between the two frames of a replay item
COHERENT_LAG = 6       # the coherent branch closes a frame 4..9 samples after the FM branch (test_challenger_arb.test_branch_lag)
AMPS = (0.017, 0.02, 0.023, 0.026, 0.03, 0.034, 0.04, 0.05)  # over noise sigma 0.02 per component at 96 kS/s
TYPES = ((1, 168), (5, 424), (18, 168))
NOISE = 0.02


class Item:
    """One burst: tx bits (before NRZI), 48 kHz start sample, timing offset in 1/20 symbol, amplitude, carrier offset (Hz) and
    amplitude nulls [(48 kHz sample offset from the start, width)]."""
    __slots__ = ("family", "bits", "start", "frac", "amp", "foffs", "nulls", "k", "close")

    def __init__(self, family, bits, amp, foffs, frac=0, nulls=(), k=None):
        self.family, self.bits, self.amp, self.foffs, self.frac = family, bits, amp, foffs, frac
        self.nulls, self.k = list(nulls), k
        self.start = None
        self.close = len(bits) - 10  # tx bit index of the last frame's sixth closing-flag 1 (hdlc: flag + 8 tail bits follow)

    def n48(self):
        return 5 * len(self.bits) + 40


def _frame(rng, msg_type, nbits, tail=8, preamble=24):
    on = DL.onair_bits(nbits, msg_type, int(rng.integers(200000000, 780000000)), rng)
    return DL.hdlc(on, preamble=preamble, tail=tail)


def _threshold(rng, n):
    out = []
    for i in range(n):
        t, nb = TYPES[int(rng.integers(0, len(TYPES)))]
        out.append(Item("threshold", _frame(rng, t, nb), AMPS[i % len(AMPS)], rng.uniform(-2000, 2000), frac=int(rng.integers(0, 20))))
    return out


def _null(rng, n):
    out = []
    for i in range(n):
        t, nb = TYPES[int(rng.integers(0, len(TYPES)))]
        bits = _frame(rng, t, nb)
        ndata = len(bits) - 24 - 16 - 8
        nulls = []
        for _ in range(1 + i % 3):  # at chosen data bits, somewhere inside the symbol
            b = 32 + int(rng.integers(8, ndata - 8))
            nulls.append((5 * b + int(rng.integers(0, 5)), 1 + int(rng.integers(0, 3))))
        out.append(Item("null", bits, float(rng.uniform(0.03, 0.06)), rng.uniform(-2000, 2000), frac=int(rng.integers(0, 20)),
                        nulls=nulls))
    return out


def _replay(rng, n):
    out = []
    for i in range(n):
        k = REPLAY_K[i % len(REPLAY_K)]
        b1 = _frame(rng, 1, 168, tail=0)
        b2 = _frame(rng, 18, 168, preamble=k + 1)[1:]  # 1 0 1 0 ...: one alternation run from frame 1's closing 1s into the flag
        amp = float(rng.choice((0.04, 0.05, 0.07, 0.3)))
        # nulls 30, 45 and 60 bits before frame 1's end break it for the FM branch only
        nulls = [(5 * (len(b1) - b) + int(rng.integers(0, 5)), 3) for b in (30, 45, 60)]
        out.append(Item("replay", np.concatenate([b1, b2]), amp, rng.uniform(-2000, 2000), frac=int(rng.integers(0, 20)),
                        nulls=nulls, k=k))
    return out


def _straddle(rng, n):
    """Item k: split position 1 + k % 4, closing sample u = (k // 4) % 5 into the group; odd k // 20 at amplitudes where a coherent
    decoder wins (its frames close COHERENT_LAG samples later, so they are placed that much earlier)."""
    out = []
    for i in range(n):
        t, nb = TYPES[int(rng.integers(0, len(TYPES)))]
        coh = (i // 20) % 2 == 1
        amp = float(rng.choice((0.018, 0.02, 0.022))) if coh else float(rng.choice((0.04, 0.05, 0.3)))
        # a carrier offset halfway between two of the CGF's 512-point bins makes its estimate flip between blocks
        foffs = (int(rng.integers(-20, 21)) + 0.5) * 48000.0 / BLOCK / 2
        out.append(Item("straddle", _frame(rng, t, nb), amp, foffs, frac=0, k=i))
    return out


class Track:
    """The items of one channel, laid out one after the other from LEAD; straddle items so that their FM close lands around a CGF
    block boundary at one of the four inner positions of a group."""

    def __init__(self, items, x_mode=False):
        self.items = items
        delay = FM_CLOSE_DELAY[x_mode]
        pos = LEAD
        for it in items:
            if it.family == "straddle":
                # the first block boundary B far enough ahead that falls `want` samples into a group; the frame's close at sample u
                # of that group, in one-sample steps of the start
                want, u = 1 + it.k % 4, (it.k // 4) % 5
                lag = COHERENT_LAG if (it.k // 20) % 2 else 0
                B = -(-(pos + 5 * it.close + delay + 20) // BLOCK) * BLOCK
                while B % 5 != want:
                    B += BLOCK
                it.start = B - want + u - 5 * it.close - delay - lag
            else:
                it.start = pos
            pos = it.start + it.n48() + GAP
        self.n48 = pos + LEAD


def build(n_streams, per_family=(16, 10, 32, 40), seed=0, x_mode=False):
    """n_streams streams; each carries tracks for A and B (AB) or one track (X).  Returns [[Track per channel] per stream]."""
    streams = []
    for s in range(n_streams):
        chans = []
        for c in range(1 if x_mode else 2):
            rng = np.random.default_rng([0xC4A1, seed, s, c])
            items = _threshold(rng, per_family[0]) + _null(rng, per_family[1]) + _replay(rng, per_family[2]) + \
                _straddle(rng, per_family[3])
            order = rng.permutation(len(items))
            chans.append(Track([items[i] for i in order], x_mode))
        streams.append(chans)
    return streams


def n48(streams, quantum=BLOCK):
    n = max(t.n48 for st in streams for t in st)
    return -(-n // quantum) * quantum


def _burst(it, fs, fc, n, rng):
    """The item's complex burst at fs on carrier fc, placed at its start; returns (first sample, samples)."""
    r = fs / 48000.0
    sps = fs / BAUD
    off = it.frac / 20.0 * sps  # timing offset in samples at fs
    bb = S.gmsk_baseband(it.bits, fs, timing_frac=off - np.floor(off))
    p0 = int(round(it.start * r)) + int(np.floor(off))
    env = np.ones(len(bb))
    for o, w in it.nulls:
        env[int(o * r):int((o + w) * r)] = 0.0
    m = min(len(bb), n - p0)
    k = np.arange(p0, p0 + m)
    gain = np.sqrt(96000.0 / fs)  # the same SNR in the 48 kHz channel at every input rate (NOISE is per input sample)
    return p0, gain * it.amp * env[:m] * bb[:m] * np.exp(1j * (2 * np.pi * (fc + it.foffs) * k / fs + rng.uniform(0, 2 * np.pi)))


def render(streams, fs, seed=0):
    """complex64[n_streams][n]: AB (two tracks) at -/+25 kHz, or X (one track) at 0 Hz, over complex AWGN of NOISE per component."""
    n = int(n48(streams) * fs // 48000)
    out = np.empty((len(streams), n), np.complex64)
    for s, chans in enumerate(streams):
        rng = np.random.default_rng([0x5EED, seed, s, fs])
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * NOISE
        for c, tr in enumerate(chans):
            fc = 0.0 if len(chans) == 1 else (-25000.0, 25000.0)[c]
            for it in tr.items:
                p0, b = _burst(it, fs, fc, n, rng)
                x[p0:p0 + len(b)] += b
        out[s] = x
    return out


def closing_splits(end_idx):
    """For frames closing at these 48 kHz samples: {CGF block boundary B inside the closing group: split position B - 5 g}."""
    out = {}
    for e in end_idx:
        g = e // 5
        B = -(-(5 * g + 1) // BLOCK) * BLOCK
        if B <= 5 * g + 4:
            out[B] = B - 5 * g
    return out


def split_schedule(end_idx, fs, n, max_len):
    """Submit lengths (input samples at fs, summing to n) with a boundary at every CGF block boundary that falls inside the closing
    group of one of these frames, so that the block before it is decoded in one submit and the rest of the group in the next.
    Segments longer than max_len are cut in max_len pieces."""
    r = fs // 48000
    cuts = sorted({B * r for B in closing_splits(end_idx)} | {0, n})
    lengths = []
    for a, b in zip(cuts, cuts[1:]):
        while b - a > max_len:
            lengths.append(max_len)
            a += max_len
        if b > a:
            lengths.append(b - a)
    return lengths


def submit_edges(lengths, fs):
    """48 kHz samples at which a submit's CGF output starts (a block boundary that a submit crossed), from submit lengths at fs."""
    r = fs / 48000.0
    edges, tot, last = set(), 0, 0
    for L in lengths:
        tot += L
        B = int(tot / r) // BLOCK * BLOCK
        if B > last:
            edges.add(last)
            last = B
    edges.discard(0)
    return sorted(edges)
