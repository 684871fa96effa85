"""Boundary stimulus for the frame decoders: AIS frames of any bit length, built so that the reference's length rules decide their
fate, with a plain restatement of the reference's bit decoder that says which of them are published.

The reference's bit decoder (Source/Marine/AIS.h:91-181, AIS.cpp:111-142) resets after every DATAFCS bit when `position` reaches
MaxBits (1087) or when cannotBeValid(position) fires at one of the positions in ABORT_POSITIONS.  The closing flag is processed
before that test, so a frame whose sixth closing 1 lands exactly on such a position (payload L = P - 23, "the tie") is still
decoded, while the same frame one bit longer (L = P - 22) is dropped one bit before its flag completes.  aissynth.frame_bits only
makes whole bytes, which never lands on those positions; the frames here are cut at the bit.

* onair_bits / hdlc: message fields written MSB first per byte, sent LSB first per byte, cut to any length L, CRC-16/X.25 of
  exactly those L bits, bit stuffing, flags.  A run of five ones can be forced so that a stuffing zero falls on a chosen position.
* designs(): ties and neighbours at every abort position and at MaxBits, with a field that makes the test fire and one that does
  not, frames aborted in mid-frame with a stuffing zero next to the abort position, and ties with a stuffing zero in their last bits.
* predict(): Decoder::Run + processData + Message::validate (Message.cpp:398-413) on the designed bits.  It says, per design,
  whether a frame is published and with which nbits and payload bytes (the trailing partial byte carries FCS bits, as the
  reference leaves them), and where the decoder closed or aborted -- so a test can show the stimulus reaches each boundary.
* Stimulus: every design at 32 consecutive one-symbol start offsets (the boundary bit visits every position of a 32-symbol decoder
  word whatever the chain's delay), spread over the two channels of several streams; the bursts of a channel form one continuous
  clean GMSK signal (filler zeros between frames keep every decoder in TRAINING, so noise cannot start a false frame).  Rendered
  as A/B IQ (render_ab), single-channel IQ (render_x) or a stereo discriminator recording (render_disc).
"""
import numpy as np

import aissynth as S

ABORT_POSITIONS = (30, 62, 96, 168, 184, 192, 336, 385, 448)  # AIS.cpp:111-142: 24 + the field length each one checks
MAX_BITS = 1087       # MAX_AIS_FRAME_LENGTH (Message.h:41): 1064 payload + 16 FCS + 7 closing-flag bits
MAX_PAYLOAD = 1064    # MAX_AIS_LENGTH
MIN_BITS = (149, 149, 149, 168, 418, 88, 72, 56, 168, 70, 168, 72, 40, 40, 88, 92, 80, 168, 312, 70, 271, 145, 154, 160, 72, 60, 96,
            168)      # Message::validate, per type 1..28
OFFSETS = 32          # one-symbol start offsets per design (a decoder word holds 32 symbols)
BAUD = 9600.0

# Per position: (fields that make cannotBeValid fire there, fields that do not).  Type 8 fires nowhere and validates from 56 bits;
# at 62 both are type 13 (valid from 40 bits), so the untriggered neighbour L = 40 is published.
FIELDS = {
    30: (dict(type=0), dict(type=13)),
    62: (dict(type=13, mmsi=1050000000), dict(type=13, mmsi=211000001)),
    96: (dict(type=10), dict(type=8)),
    168: (dict(type=16), dict(type=8)),
    184: (dict(type=20), dict(type=8)),
    192: (dict(type=1), dict(type=8)),
    336: (dict(type=19), dict(type=8)),
    385: (dict(type=21), dict(type=8)),
    448: (dict(type=5), dict(type=8)),
    MAX_BITS: (dict(type=8), dict(type=8)),
}


class Design:
    """One designed frame.  kind: 'tie' (L = P-24 .. P-22 around position P), 'maxbits', 'abort' (longer than P, of the type that
    fires at P, stuffing zero at `stuff`), 'tie_stuff' (a tie or its neighbour with a stuffing zero at `stuff`)."""
    __slots__ = ("kind", "P", "L", "trig", "type", "mmsi", "stuff", "seed", "onair", "bits", "outcome")

    def __init__(self, kind, P, L, trig, fields, stuff=None, seed=0):
        self.kind, self.P, self.L, self.trig, self.stuff, self.seed = kind, P, L, trig, stuff, seed
        self.type = fields["type"]
        self.mmsi = fields.get("mmsi", 211000000 + 1000 * P + L)
        self.onair = self.bits = self.outcome = None

    def name(self):
        s = "%s_P%d_L%d_%s" % (self.kind, self.P, self.L, "fire" if self.trig else "pass")
        return s + ("_stuff%d" % self.stuff if self.stuff is not None else "")

    def __repr__(self):
        return self.name()

    def frame(self):
        """(nbits, payload bytes) the frame would be published with if nothing stopped it: the designed bits and the FCS after
        them, packed as Message::setBit packs them, ceil(L / 8) bytes."""
        crc = S.crc16_x25(self.onair)
        bits = np.concatenate([self.onair, np.array([(crc >> k) & 1 for k in range(16)], dtype=np.uint8)])
        n = (self.L + 7) // 8
        return self.L, bytes(np.packbits(bits[:8 * n].reshape(n, 8)[:, ::-1], axis=1).reshape(-1))

    def closed_at(self):
        """Decoder positions at which the designed frame closed or was aborted (the predicted events of its own bits)."""
        return [(e[0], e[1]) for e in self.outcome]


def onair_bits(L, msg_type, mmsi, rng, stuff=None):
    """L on-air data bits: random message bits with the type (bits 0-5) and MMSI (bits 8-37) fields, MSB first per byte, each byte
    sent LSB first, cut after L bits.  stuff = s: on-air bits s-6 .. s-1 are 0 11111, so a stuffing zero follows the s-th bit."""
    nbytes = (L + 7) // 8
    msg = rng.integers(0, 2, nbytes * 8).astype(np.uint8)
    for k in range(6):
        msg[k] = (msg_type >> (5 - k)) & 1
    for k in range(30):
        if 8 + k < len(msg):
            msg[8 + k] = (mmsi >> (29 - k)) & 1
    tx = msg.reshape(nbytes, 8)[:, ::-1].reshape(-1)[:L].copy()
    if stuff is not None:
        assert 6 <= stuff <= L
        tx[stuff - 6] = 0
        tx[stuff - 5:stuff] = 1
    return tx


def hdlc(onair, preamble=24, tail=8):
    """On-air data bits -> transmitted bits (before NRZI): preamble, flag, data + CRC-16/X.25 of exactly those bits (LSB first),
    stuffed, flag, tail (as aissynth.frame_bits, without rounding the data up to whole bytes)."""
    crc = S.crc16_x25(onair)
    data = np.concatenate([onair, np.array([(crc >> k) & 1 for k in range(16)], dtype=np.uint8)])
    stuffed, ones = [], 0
    for b in data:
        stuffed.append(int(b))
        ones = ones + 1 if b else 0
        if ones == 5:
            stuffed.append(0)
            ones = 0
    flag = [0, 1, 1, 1, 1, 1, 1, 0]
    return np.array([k & 1 for k in range(preamble)] + flag + stuffed + flag + [0] * tail, dtype=np.uint8)


# ---------------------------------------------------------------------------------------------------------------------------------
# the reference's decoder, restated bit by bit on decoded bits (after NRZI)

def _type(buf):
    return buf[0] >> 2


def _mmsi(buf):
    return (buf[1] << 22) | (buf[2] << 14) | (buf[3] << 6) | (buf[4] >> 2)


def cannot_be_valid(buf, pos):
    """AIS.cpp:111-142."""
    if pos == 30:
        t = _type(buf)
        return t > 28 or t == 0
    if pos == 62:
        return _mmsi(buf) > 999999999
    t = _type(buf)
    return {96: t == 10, 168: t == 16, 184: t in (15, 20, 23), 192: t in (1, 2, 3, 4, 7, 9, 11, 18, 22, 24, 25, 27, 28), 336: t == 19,
            385: t == 21, 448: t == 5}.get(pos, False)


def validate(buf, nbits):
    """Message::validate (Message.cpp:398-413)."""
    if nbits == 0:
        return True
    if nbits > MAX_PAYLOAD:
        return False
    t = _type(buf)
    return 1 <= t <= 28 and nbits >= MIN_BITS[t - 1]


def _crc_ok(buf, n):
    crc = 0xFFFF
    for i in range(n):
        b = (buf[i >> 3] >> (i & 7)) & 1
        crc = (crc >> 1) ^ 0x8408 if (b ^ crc) & 1 else crc >> 1
    return crc == 0xF0B8


def predict(bits):
    """Decoder::Run (AIS.h:91-181) from TRAINING over decoded bits, with processData (AIS.cpp:66-96) and Message::validate.
    Returns (events, final state): ("frame", position, nbits, payload bytes, published), ("crc", position) for a closing flag whose
    CRC fails, ("abort", position) for a reset by MaxBits / cannotBeValid.  State 0 is TRAINING."""
    TRAINING, STARTFLAG, DATAFCS = 0, 1, 2
    state, position, ones, last = TRAINING, 0, 0, 0
    buf = bytearray((MAX_BITS + 7) // 8 + 4)
    events = []
    for b in bits:
        b = int(b)
        if state == TRAINING:
            if b != last:
                position += 1
            elif position > 4:
                state, position = STARTFLAG, (3 if b else 1)
            else:
                position = 0
        elif state == STARTFLAG:
            if position == 7:
                if b == 0:
                    state, position, ones = DATAFCS, 0, 0
                    buf[:] = bytes(len(buf))
                else:
                    state, position = TRAINING, 0
            elif b:
                position += 1
            else:
                state, position = TRAINING, 0
        else:
            if position < MAX_BITS:  # Message::setBit
                if b:
                    buf[position >> 3] |= 1 << (position & 7)
                else:
                    buf[position >> 3] &= ~(1 << (position & 7)) & 0xFF
            position += 1
            if b:
                if ones == 5:  # closing flag: processData, then NextState(TRAINING) -- before the length test below
                    n = position - 7
                    if n >= 16 and _crc_ok(buf, n):
                        nbits = n - 16
                        length = nbits if nbits <= MAX_PAYLOAD else 0  # Message::setLength ignores longer lengths
                        events.append(("frame", position, length, bytes(buf[:(length + 7) // 8]), validate(buf, length)))
                    else:
                        events.append(("crc", position))
                    state, position, ones = TRAINING, 0, 0
                else:
                    ones += 1
            else:
                if ones == 5:
                    position -= 1  # bit-destuff
                ones = 0
            if state == DATAFCS and (position == MAX_BITS or cannot_be_valid(buf, position)):
                events.append(("abort", position))
                state, position, ones = TRAINING, 0, 0
        last = b
    return events, state


def published(events):
    return [(e[2], e[3]) for e in events if e[0] == "frame" and e[4]]


# ---------------------------------------------------------------------------------------------------------------------------------
# designs

def _build(d):
    """Draws the design's payload; redraws until the decoder is back in TRAINING 16 bits after the frame, so one design cannot
    reach into the next one (after an abort in mid-frame the rest of the frame is read as training bits)."""
    for attempt in range(64):
        rng = np.random.default_rng([0xB0DE, d.P, d.L, int(d.trig), 0 if d.stuff is None else d.stuff + 1, d.seed, attempt])
        onair = onair_bits(d.L, d.type, d.mmsi, rng, d.stuff)
        bits = hdlc(onair)
        events, state = predict(np.concatenate([bits, np.zeros(16, np.uint8)]))
        if state == 0:
            d.onair, d.bits, d.outcome = onair, bits, events
            return d
    raise AssertionError("no payload of %s leaves the decoder in TRAINING" % d.name())


def designs():
    out = []
    for P in ABORT_POSITIONS:
        for trig in (True, False):
            for L in (P - 24, P - 23, P - 22):
                out.append(Design("tie", P, L, trig, FIELDS[P][0 if trig else 1]))
    for L in (MAX_PAYLOAD - 1, MAX_PAYLOAD, MAX_PAYLOAD + 1, 1100):
        out.append(Design("maxbits", MAX_BITS, L, True, FIELDS[MAX_BITS][0]))
    for P in ABORT_POSITIONS + (MAX_BITS,):  # frames that run past P, with a stuffing zero at each of P-2 .. P+2
        L = 1100 if P == MAX_BITS else P + 40
        for s in range(P - 2, P + 3):
            out.append(Design("abort", P, L, True, FIELDS[P][0], stuff=s))
    for P in ABORT_POSITIONS[2:] + (MAX_BITS,):  # ties and neighbours whose last data bits end in a stuffing zero
        for L in (P - 23, P - 22):
            for s in (L - 2, L - 1, L):
                out.append(Design("tie_stuff", P, L, True, FIELDS[P][0], stuff=s))
    return [_build(d) for d in out]


def tie_designs():
    """The ties and their neighbours only (the scale case's stimulus)."""
    return [d for d in designs() if d.kind in ("tie", "maxbits")]


# ---------------------------------------------------------------------------------------------------------------------------------
# layout and rendering

class Stimulus:
    """Every design at OFFSETS start offsets, instance i on track i % (2 B): stream track % B, channel A for the first B tracks.
    tracks[t] = (decoded bits of the whole track, [(start symbol, design)]).  n_sym: symbols per track (all equal)."""

    def __init__(self, dsg, n_streams, offsets=range(OFFSETS), lead=64, gap=8):
        self.designs = dsg
        self.n_streams = n_streams
        ntr = 2 * n_streams
        inst = [(d, k) for k in offsets for d in dsg]
        seqs = [[np.zeros(lead, np.uint8)] for _ in range(ntr)]
        cur = [lead] * ntr
        placed = [[] for _ in range(ntr)]
        for i, (d, k) in enumerate(inst):
            t = i % ntr
            s = cur[t] + gap
            s += (k - s) % OFFSETS
            seqs[t].append(np.zeros(s - cur[t], np.uint8))
            seqs[t].append(d.bits)
            placed[t].append((s, d))
            cur[t] = s + len(d.bits)
        self.n_sym = max(cur) + lead
        self.tracks = []
        for t in range(ntr):
            seqs[t].append(np.zeros(self.n_sym - cur[t], np.uint8))
            self.tracks.append((np.concatenate(seqs[t]), placed[t]))

    def track(self, s, ch):
        return self.tracks[s + (0 if ch == "A" else self.n_streams)]

    def expected(self, s, ch):
        """(nbits, payload) of the frames the reference publishes on channel ch of stream s, in order."""
        return [f for _, d in self.track(s, ch)[1] for f in published(d.outcome)]

    def n_samples(self, fs, quantum=32768):
        n = int(np.ceil(self.n_sym * fs / BAUD))
        return -(-n // quantum) * quantum

    def _tone(self, bits, fs, n, fc, timing, amp, rng):
        bb = S.gmsk_baseband(bits, fs, timing_frac=timing)
        m = min(n, len(bb))
        k = np.arange(m)
        out = np.zeros(n, np.complex128)
        out[:m] = amp * bb[:m] * np.exp(1j * (2 * np.pi * fc * k / fs + rng.uniform(0, 2 * np.pi)))
        return out

    def render_ab(self, fs, seed=0, amp=0.5, noise_sigma=0.01, quantum=32768):
        """complex64[n_streams][n]: channel A at -25 kHz and B at +25 kHz (plus a small carrier offset), over complex AWGN."""
        n = self.n_samples(fs, quantum)
        out = np.empty((self.n_streams, n), np.complex64)
        for s in range(self.n_streams):
            rng = np.random.default_rng([0xAB, seed, s])
            x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * noise_sigma
            for ch, fc in (("A", -25000.0), ("B", 25000.0)):
                x += self._tone(self.track(s, ch)[0], fs, n, fc + rng.uniform(-300, 300), rng.uniform(0, 1), amp, rng)
            out[s] = x
        return out

    def render_x(self, fs, seed=0, amp=0.5, noise_sigma=0.01, quantum=32768):
        """complex64[2 n_streams][n] for single-channel mode: stream s carries the A track of stream s (s < n_streams) or the B
        track of stream s - n_streams, at 0 Hz plus a small offset."""
        n = self.n_samples(fs, quantum)
        out = np.empty((2 * self.n_streams, n), np.complex64)
        for t, (bits, _) in enumerate(self.tracks):
            rng = np.random.default_rng([0x58, seed, t])
            x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * noise_sigma
            out[t] = x + self._tone(bits, fs, n, rng.uniform(-300, 300), rng.uniform(0, 1), amp, rng)
        return out

    def render_disc(self, fs, seed=0, amp=0.5, noise_sigma=0.003, quantum=32768):
        """complex64[n_streams][n] for the FM-discriminator input model: channel A's discriminator audio in I, B's in Q -- the
        phase increment of a noisy GMSK baseband over pi, times a gain, plus a small DC offset, clipped to [-1, 1) (the model of
        disc_util.discriminator_audio, on the designed bits).  Less noise than the IQ renderings: the phase increment of the
        complex noise at 5 samples per symbol would otherwise flip a bit of a long frame now and then."""
        n = self.n_samples(fs, quantum)
        out = np.empty((self.n_streams, n), np.complex64)
        for s in range(self.n_streams):
            rng = np.random.default_rng([0xD1, seed, s])
            iq = []
            for ch in "AB":
                x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)) * noise_sigma
                x += self._tone(self.track(s, ch)[0], fs, n, 0.0, rng.uniform(0, 1), amp, rng)
                d = np.zeros(n)
                d[1:] = np.angle(x[1:] * np.conj(x[:-1])) / np.pi
                iq.append(np.clip(d * rng.uniform(2.0, 6.0) + rng.uniform(-0.02, 0.02), -1.0, 1.0 - 2.0 ** -15))
            out[s] = iq[0] + 1j * iq[1]
        return out


def assert_boundaries(dsg, seen, label, offsets=OFFSETS):
    """seen: Counter of published (nbits, payload).  Per design: its frame published at each of its start offsets when the
    restated decoder publishes it, at none when not; and per position, that the ties and the dropped neighbours are among them."""
    bad = []
    for d in dsg:
        n = seen[d.frame()]
        want = offsets if published(d.outcome) else 0
        if n != want:
            bad.append((d.name(), n, want))
    assert not bad, "%s: designs published a wrong number of times (name, got, want): %r" % (label, bad[:12])
    for P in ABORT_POSITIONS + (MAX_BITS,):
        ties = [d for d in dsg if d.P == P and d.L == P - 23 and d.kind in ("tie", "maxbits", "tie_stuff")]
        drops = [d for d in dsg if d.P == P and d.L == P - 22 and d.trig]
        assert ties and drops, (label, P)
        assert all(seen[d.frame()] == (0 if P in (30, 62) else offsets) for d in ties), (label, P, "tie")
        assert all(seen[d.frame()] == 0 for d in drops), (label, P, "dropped neighbour")
