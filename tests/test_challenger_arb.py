"""CPU (-m "not gpu"): ModelChallenger's ten cross-reset decoders where their order within a group decides what is published.

The stimulus is tests/challenger_arb.py's (threshold sweep, FM-only nulls, back-to-back frames on the alternation threshold, closing
groups across CGF blocks, submit boundaries inside closing groups).  Three things are checked:

* the plain-C restatement (oracle/ais_oracle.c, model 4) equals the compiled reference on all of it: every frame with its level and
  ppm bit patterns and end_idx, and which of the ten decoders published it;
* the stimulus reaches the cases where the order matters, counted from the published records and the decoders' publishers: winners
  at each decoder, closes of both branches in one group, frames found after a Reset only by decoders ranked above its sender, FM
  winners whose CGF block is not their group's fifth sample's, channel B FM winners that read the level channel A left behind, and
  every split position of a closing group across submits;
* each plausible mis-ordering of the ten decoders (f4 before the coherent ones, the coherent ones before f0..f3, the FM phases
  reversed) changes the restatement's published frames on this stimulus.

tests/golden/challenger_arb.json holds a SHA-256 of the reference's records per case, written by `python
tests/test_challenger_arb.py`; where oracle/_ref was not built, the restatement is checked against it and counted from.
"""
import functools
import hashlib
import json
import os
from collections import Counter

import numpy as np
import pytest

import challenger_arb as CA
import oracle as O
import oracle_x as OX

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "challenger_arb.json")
FS_AB, FS_X = 96000, 48000
N_AB, N_X = 16, 16
CHUNK = 4096
NARROW = O.FLAG_PS_EMA | O.FLAG_DROOP  # AFC_WIDE off
ORDER = O.CHALLENGER_ORDER
RANK = {d: r for r, d in enumerate(ORDER)}
ORDERS = {"f4_before_coherent": (5, 6, 7, 8, 9, 0, 1, 2, 3, 4), "coherent_before_fm": tuple(range(10)),
          "fm_reversed": (9, 8, 7, 6, 0, 1, 2, 3, 4, 5)}
# name: (single-channel mode, flags, submits: "chunk" = CHUNK each, "split" = split_schedule of the "chunk" case's end_idx)
CASES = {"ab": (False, O.DEFAULT_FLAGS, "chunk"), "ab_narrow": (False, NARROW, "chunk"), "ab_split": (False, O.DEFAULT_FLAGS, "split"),
         "x": (True, O.DEFAULT_FLAGS, "chunk"), "x_split": (True, O.DEFAULT_FLAGS, "split")}
MIN = 20  # every coverage class below, per channel where it is per channel


class Rec:
    """A published frame with the decoder that published it."""
    __slots__ = ("channel", "nbits", "start", "end", "level", "ppm", "payload", "nmea", "pub")

    def __init__(self, m, pub):
        self.channel, self.nbits, self.start, self.end = m.channel, m.nbits, m.start_idx, m.end_idx
        self.level = int(np.float32(m.level).view(np.uint32))
        self.ppm = int(np.float32(m.ppm).view(np.uint32))
        self.payload, self.nmea, self.pub = m.payload.hex(), tuple(m.nmea), pub

    def key(self):
        return (self.channel, self.nbits, self.start, self.end, self.level, self.ppm, self.payload, self.nmea)

    def full(self):
        return self.key() + (self.pub,)

    def rkey(self):
        """What the order of the decoders decides besides level and ppm: which frames are found, where and by whom."""
        return (self.channel, self.nbits, self.start, self.end, self.payload, self.pub)


@functools.lru_cache(maxsize=None)
def stimulus(x_mode):
    streams = CA.build(N_X if x_mode else N_AB, x_mode=x_mode)
    return streams, CA.render(streams, FS_X if x_mode else FS_AB)


def make(kind, x_mode, flags, taps=False):
    if kind == "ref":
        if x_mode:
            return OX.RefModelX(model=O.MODEL_CHALLENGER, sample_rate=FS_X, flags=flags, taps=taps)
        return O.RefModel(model=O.MODEL_CHALLENGER, sample_rate=FS_AB, flags=flags, taps=taps)
    return O.PortModel(model=O.MODEL_CHALLENGER, sample_rate=FS_X if x_mode else FS_AB,
                       flags=flags | (O.FLAG_MODE_X if x_mode else 0), taps=taps)


def feed(m, x, lengths):
    """Pushes x in the given submits; returns the records."""
    recs, pos = [], 0
    for n in lengths:
        m.push(x[pos:pos + n])
        pos += n
        pubs = m.publishers()
        msgs = m.messages()
        assert len(pubs) == len(msgs)
        recs += [Rec(q, p) for q, p in zip(msgs, pubs)]
    m.close()
    return recs


def chunks(n, chunk=CHUNK):
    return [min(chunk, n - p) for p in range(0, n, chunk)]


@functools.lru_cache(maxsize=None)
def schedules(name):
    """Per stream submit lengths of the case."""
    x_mode, flags, sub = CASES[name]
    _, xs = stimulus(x_mode)
    if sub == "chunk":
        return [chunks(xs.shape[1])] * len(xs)
    base = runs("x" if x_mode else "ab", "port")
    fs = FS_X if x_mode else FS_AB
    return [CA.split_schedule([r.end for r in recs], fs, xs.shape[1], 2 * CHUNK) for recs in base]


@functools.lru_cache(maxsize=None)
def runs(name, kind, order=None):
    """Per stream records of the case, by the reference ("ref") or the restatement ("port", with another decoder order)."""
    x_mode, flags, _ = CASES[name]
    _, xs = stimulus(x_mode)
    out = []
    for s, lengths in enumerate(schedules(name)):
        m = make(kind, x_mode, flags)
        if order is not None:
            m.challenger_order(order)
        out.append(feed(m, xs[s], lengths))
    return out


def digest(recs_per_stream, lengths_per_stream):
    h = hashlib.sha256()
    for recs, lengths in zip(recs_per_stream, lengths_per_stream):
        h.update(repr(lengths).encode())
        for r in recs:
            h.update(repr(r.full()).encode())
    return h.hexdigest()


def load_golden():
    with open(GOLDEN) as f:
        return json.load(f)


@functools.lru_cache(maxsize=None)
def checked(name):
    """The case's records, equal to the stored reference digest (and to the reference itself, where it was built)."""
    port = runs(name, "port")
    want = load_golden()[name]
    if O.have_ref() and (not CASES[name][0] or OX.have_refx()):
        ref = runs(name, "ref")
        for s, (g, w) in enumerate(zip(port, ref)):
            assert [r.full() for r in g] == [r.full() for r in w], "stream %d: the restatement differs from the reference: %r" % (
                s, [(a.full(), b.full()) for a, b in zip(g, w) if a.full() != b.full()][:2] or (len(g), len(w)))
        assert digest(ref, schedules(name)) == want["sha256"], "the reference no longer reproduces %s" % GOLDEN
    assert digest(port, schedules(name)) == want["sha256"], "the restatement differs from the reference's stored records"
    return port


def item_of(streams, s, rec):
    """The stimulus item whose burst the frame closed in."""
    chans = streams[s]
    tr = chans[0] if len(chans) == 1 else chans["AB".index(rec.channel)]
    for it in tr.items:
        if it.start <= rec.end < it.start + it.n48() + CA.GAP:
            return it
    return None


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_equals_reference(built, name):
    recs = checked(name)
    assert sum(len(r) for r in recs) >= 500 * (N_X if CASES[name][0] else N_AB) // 16


def test_winners_at_every_decoder(built):
    c = Counter((r.channel, r.pub) for recs in checked("ab") + checked("ab_narrow") for r in recs)
    c.update(("X", r.pub) for recs in checked("x") for r in recs)
    low = {k: c[k] for k in [(ch, d) for ch in "ABX" for d in range(10)] if c[k] < MIN}
    assert not low, "decoders with fewer than %d winners (channel, decoder): %r" % (MIN, low)


def test_same_group_closes(built):
    """A frame published by f0..f3 that a coherent decoder closes in the same group: it publishes it there when ranked first.  The
    coherent branch closes a frame 4..9 samples after the FM branch (test_branch_lag), so only f0 with a lag of 4 samples ties; the
    timing grid yields a handful.  A coherent winner that f4 closes in the same group would need a lag below 0: none exists."""
    n = Counter()
    for name in ("ab", "x"):
        other = runs(name, "port", ORDERS["coherent_before_fm"])
        for recs, orecs in zip(checked(name), other):
            there = {(r.channel, r.payload, r.end // 5): r.pub for r in orecs}
            for r in recs:
                if 5 <= r.pub <= 8 and there.get((r.channel, r.payload, r.end // 5), 9) < 5:
                    n[r.channel] += 1
    # a known thin class (measured A 2, B 1, X 2): the ties need the smallest lag of test_branch_lag's distribution
    assert sum(n.values()) >= 4, dict(n)


def test_branch_lag(built):
    """How many 48 kHz samples after the FM branch the coherent branch closes the same frame, over the timing grid: ModelDefault
    with PS_EMA is ModelChallenger's coherent branch alone (the same CGF, FIR17 and PhaseSearchEMA with nDelay 3).  Measured on
    this stimulus: 4..9 samples (mostly 5..7), so in the FM winner's group only when the winner is f0 and the lag 4, never for f4."""
    _, xs = stimulus(False)
    lag, glag = Counter(), Counter()
    for s, recs in enumerate(checked("ab")):
        m = O.PortModel(model=O.MODEL_DEFAULT, sample_rate=FS_AB)
        m.run(xs[s], CHUNK)
        coh = {(q.channel, q.payload.hex()): q.end_idx for q in m.messages()}
        m.close()
        for r in recs:
            if r.pub >= 5 and (r.channel, r.payload) in coh:
                e = coh[(r.channel, r.payload)]
                lag[e - r.end] += 1
                glag[(r.pub - 5, e // 5 - r.end // 5)] += 1
    assert sum(lag.values()) >= 1000 and min(lag) >= 4 and max(lag) <= 9, sorted(lag.items())
    assert all(g >= 1 for (ph, g) in glag if ph > 0), sorted(glag.items())


def counter_order(p1, p2):
    """One of ORDERS that steps decoder p2 before decoder p1, where p2 steps after p1 in the reference's order (None for pairs within
    one branch): f4 after a0..a4, a0..a4 after f0..f3."""
    if p1 < 5 and p2 == 9:
        return ORDERS["f4_before_coherent"]
    if 5 <= p1 <= 8 and p2 < 5:
        return ORDERS["coherent_before_fm"]
    return None


def test_replay_boundary(built):
    """Back-to-back frames with k alternations between them.  Frame 2 is lost for k <= 2 and found from k = 3: the count after frame
    1's Reset sits on the "> 4" threshold.  Count the second frames found only because their decoder stepped after frame 1's winner
    (the winner's group counted as an alternation for it): with the two decoders' order swapped, that frame is no longer published
    as it was (found by another decoder, elsewhere, or not at all)."""
    found, total, only = Counter(), Counter(), Counter()
    for name in ("ab", "x"):
        streams, _ = stimulus(CASES[name][0])
        for s, recs in enumerate(checked(name)):
            by_item = {}
            for r in recs:
                it = item_of(streams, s, r)
                if it is not None and it.family == "replay":
                    by_item.setdefault(id(it), []).append(r)
            for tr in streams[s]:
                for it in tr.items:
                    if it.family != "replay":
                        continue
                    pair = by_item.get(id(it), [])
                    total[it.k] += 1
                    if len(pair) != 2:
                        continue
                    found[it.k] += 1
                    order = counter_order(pair[0].pub, pair[1].pub)
                    if order is not None:
                        other = {r.rkey() for r in runs(name, "port", order)[s]}
                        if pair[1].rkey() not in other:
                            only[(pair[0].pub < 5, pair[1].channel)] += 1
    assert all(found[k] == 0 for k in total if k <= 2) and all(found[k] >= 0.9 * total[k] for k in total if k >= 3), (found, total)
    # Only f4 after a coherent winner can do it (measured A 8, B 9, X 8): the FM branch runs a bit ahead of the coherent one, so at
    # a coherent winner's group an FM sibling sees the flag's last 0, an alternation.  After an FM winner the coherent siblings are
    # still in its closing 1s, where the group's bit is no alternation whoever steps first.
    low = {ch: only[(True, ch)] for ch in "ABX" if only[(True, ch)] < 4}
    assert not low, "second frames found only by a decoder stepping after the first frame's winner: %r" % dict(only)


def test_ppm_block(built):
    """Every winner carries the ppm of the CGF block that delivered its closing sample: an FM winner its own sample's, a coherent one
    its group's fifth sample's.  Enough FM winners have a closing group across two blocks whose estimates differ.  (A/B mode: the
    single-channel harness keeps ModelChallenger's CGF untapped.)"""
    n = Counter()
    for name in ("ab",):
        x_mode, flags, _ = CASES[name]
        _, xs = stimulus(x_mode)
        for s, lengths in enumerate(schedules(name)):
            m = make("port", x_mode, flags, taps=True)
            pos, recs, ppm = 0, [], {"A": [], "B": []}
            for L in lengths:
                m.push(xs[s][pos:pos + L])
                pos += L
                pubs, msgs = m.publishers(), m.messages()
                recs += [Rec(q, p) for q, p in zip(msgs, pubs)]
                ppm["A"] += m.tap_ppm(O.TAP_CGF_A).tolist()
                ppm["B"] += m.tap_ppm(O.TAP_CGF_B).tolist()
                for t in range(9):
                    m.tap_c(t)
                for t in range(14):
                    m.tap_f(t)
            m.close()
            assert [r.full() for r in recs] == [r.full() for r in checked(name)[s]]
            for r in recs:
                blocks = np.array(ppm[r.channel], np.float32).view(np.uint32)
                own, fifth = r.end // CA.BLOCK, (r.end // 5 * 5 + 4) // CA.BLOCK
                assert r.ppm == int(blocks[own if r.pub >= 5 else fifth]), (name, s, r.full())
                if r.pub >= 5 and own != fifth and blocks[own] != blocks[fifth]:
                    n[r.channel] += 1
    assert all(n[ch] >= MIN for ch in "AB"), dict(n)


def test_level_carry_from_channel_a(built):
    """Channel B's FM decoders f0..f3 read, at the first group of a submit's CGF output, the level channel A's chain has just left
    in the shared tag.  Count the B winners among f0..f3 whose frame contains such a read (phase j reads it at group E // 5 when
    E % 5 <= j, E the first sample of a submit's output)."""
    n = Counter()
    for name in ("ab", "ab_split"):
        for recs, lengths in zip(checked(name), schedules(name)):
            edges = CA.submit_edges(lengths, FS_AB)
            for r in recs:
                if r.channel == "B" and 5 <= r.pub <= 8 and any(r.start <= E <= r.end and E % 5 <= r.pub - 5 for E in edges):
                    n[name] += 1
    assert n["ab"] >= MIN and n["ab_split"] >= MIN, dict(n)


def test_split_closing_groups(built):
    """The split schedules put a submit boundary inside closing groups at every position the 512-sample CGF block allows (the
    block boundary 1..4 samples into the group), for FM and coherent winners."""
    for name in ("ab_split", "x_split"):
        fs = FS_X if CASES[name][0] else FS_AB
        n = Counter()
        for recs, lengths in zip(checked(name), schedules(name)):
            edges = set(CA.submit_edges(lengths, fs))
            for r in recs:
                for B, pos in CA.closing_splits([r.end]).items():
                    if B in edges:
                        n[(pos, r.pub >= 5)] += 1
        low = {(p, fm): n[(p, fm)] for p in range(1, 5) for fm in (False, True) if n[(p, fm)] < MIN // 4}
        assert not low, "%s: split positions (position, FM winner) reached too rarely: %r of %r" % (name, low, dict(n))


ORDER_MIN = {"f4_before_coherent": 12, "coherent_before_fm": 20, "fm_reversed": 800}  # records that differ, per case (see below)


@pytest.mark.parametrize("alt", sorted(ORDERS))
def test_order_decides(built, alt):
    """Each mis-ordering of the ten decoders changes which frames are published, where and by whom -- compared without level and
    ppm, which the order also decides (the group's level is written just before the first coherent decoder steps, and a delayed FM
    step can see the next CGF block's ppm).  Measured records that differ (AB / X): f4_before_coherent 34 / 16, coherent_before_fm
    68 / 44, fm_reversed 3248 / 1636."""
    for name in ("ab", "x"):
        moved = 0
        for g, w in zip(runs(name, "port", ORDERS[alt]), checked(name)):
            a, b = Counter(r.rkey() for r in g), Counter(r.rkey() for r in w)
            moved += sum(((a - b) + (b - a)).values())
        assert moved >= ORDER_MIN[alt], "%s: the order %s moves %d frames" % (name, alt, moved)


if __name__ == "__main__":  # regenerate the stored digests from the reference (needs oracle/_ref)
    assert O.have_ref() and OX.have_refx(), "oracle/_ref not built"
    out = {}
    for name in sorted(CASES):
        recs = runs(name, "ref")
        out[name] = {"sha256": digest(recs, schedules(name)), "frames": sum(len(r) for r in recs)}
    with open(GOLDEN, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
