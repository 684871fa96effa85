"""The frame decoders' length rules on the CPU: frames cut at every abort position of cannotBeValid and at MaxBits (the tie, where
the closing flag completes on the abort position, and the neighbours one bit either side), frames aborted in mid-frame with a
stuffing zero next to the abort position, each at 32 one-symbol start offsets (tests/decoder_limits.py).  The plain restatement of
the reference's decoder says which frames are published; the compiled reference (oracle/_ref, models 0, 1, 2, 4 and 11) and the C
restatement the GPU tests fall back to (oracle/ais_oracle.c, models 0, 1 and 2) must publish exactly those, in order, per channel.

At positions 30 and 62 the tie (7 and 39 payload bits) is too short for Message::validate whatever its fields, so it is never
published; there the frames show only the untriggered 40-bit neighbour at 62 and nothing at 30 (type 0, which fires at 30, never
validates either, so its aborts are invisible in the frames).  Those positions are still checked on the predicted decoder events."""
from collections import Counter

import numpy as np
import pytest

import decoder_limits as DL
import oracle as O

FS, CHUNK, B = 96000, 4096, 8


@pytest.fixture(scope="module")
def stim():
    st = DL.Stimulus(DL.designs(), B)
    return st, st.render_ab(FS)


def by_kind(st, kind, P=None):
    return [d for d in st.designs if d.kind == kind and (P is None or d.P == P)]


def test_designs_reach_every_boundary(stim):
    st, _ = stim
    for P in DL.ABORT_POSITIONS:
        tie = {(d.L - P, d.trig): d for d in by_kind(st, "tie", P)}
        assert sorted(tie) == [(dl, t) for dl in (-24, -23, -22) for t in (False, True)], P
        for trig in (False, True):
            # the tie closes on the abort position itself, the shorter frame one bit before it
            assert tie[(-23, trig)].closed_at() == [("frame", P)], (P, trig)
            assert tie[(-24, trig)].closed_at() == [("frame", P - 1)], (P, trig)
        # one bit longer: the triggered frame is reset on P, one bit before its flag completes; the other one closes on P + 1
        assert tie[(-22, True)].closed_at() == [("abort", P)], P
        assert tie[(-22, False)].closed_at() == [("frame", P + 1)], P
        assert DL.published(tie[(-22, True)].outcome) == [], P
        short = P in (30, 62)  # 7 and 39 bits: below every type's minimum length
        for trig in (False, True):
            assert bool(DL.published(tie[(-23, trig)].outcome)) == (not short), (P, trig)
        # the untriggered neighbour: published at 62 (type 13, 40 bits) and from 96 on
        assert bool(DL.published(tie[(-22, False)].outcome)) == (P != 30), P
        for d in by_kind(st, "abort", P):  # aborted on P in mid-frame, whatever side of P the stuffing zero falls on
            assert d.closed_at()[0] == ("abort", P) and DL.published(d.outcome) == [], d
            # without the abort these frames would be published (type 0 at 30 never is)
            buf = bytearray(d.frame()[1])
            assert DL.validate(buf, d.L) == (P != 30), d
        assert sorted(d.stuff - P for d in by_kind(st, "abort", P)) == [-2, -1, 0, 1, 2], P
    mb = {d.L: d for d in by_kind(st, "maxbits")}
    assert mb[1063].closed_at() == [("frame", 1086)] and mb[1064].closed_at() == [("frame", DL.MAX_BITS)]
    assert DL.published(mb[1064].outcome) == [mb[1064].frame()] and DL.published(mb[1063].outcome) == [mb[1063].frame()]
    assert mb[1065].closed_at()[0] == ("abort", DL.MAX_BITS) and mb[1100].closed_at()[0] == ("abort", DL.MAX_BITS)
    for d in by_kind(st, "abort", DL.MAX_BITS):
        assert d.closed_at()[0] == ("abort", DL.MAX_BITS), d
    for d in by_kind(st, "tie_stuff"):  # a stuffing zero among the last data bits does not move the tie
        want = [("frame", d.P)] if d.L == d.P - 23 else [("abort", d.P)]
        assert d.closed_at()[:1] == want, d
        assert d.onair[d.stuff - 6] == 0 and d.onair[d.stuff - 5:d.stuff].all(), d
    # every published design publishes its own frame, bit for bit, trailing partial byte with FCS bits included
    for d in st.designs:
        for f in DL.published(d.outcome):
            assert f == d.frame(), d


def test_predicted_payload_ends_in_fcs_bits(stim):
    st, _ = stim
    d = next(d for d in by_kind(st, "tie", 448) if d.L == 425 and d.trig)  # type 5, 425 bits: 53 bytes + 1 bit
    nbits, payload = DL.published(d.outcome)[0]
    crc = DL.S.crc16_x25(d.onair)
    assert nbits == 425 and len(payload) == 54
    assert payload[53] == ((int(d.onair[424]) | ((crc & 0x7F) << 1)) & 0xFF)


def check_model(make, st, x, model):
    """Runs every stream through its own checker instance; returns the problems and the frames per design it published."""
    problems = []
    seen = Counter()
    for s in range(st.n_streams):
        m = make(model=model, sample_rate=FS)
        m.run(x[s], CHUNK)
        msgs = m.messages()
        m.close()
        for ch in "AB":
            got = [(q.nbits, q.payload) for q in msgs if q.channel == ch]
            want = st.expected(s, ch)
            seen.update(got)
            if got != want:
                problems.append((s, ch, len(got), len(want), [g for g in got if g not in want][:2], [w for w in want if w not in got][:2]))
    return problems, seen


@pytest.mark.parametrize("model", [O.MODEL_STANDARD, O.MODEL_BASE, O.MODEL_DEFAULT, O.MODEL_CHALLENGER, O.MODEL_V2])
def test_reference_publishes_predicted(built, stim, model):
    if not O.have_ref():
        pytest.skip("oracle/_ref not built (the reference sources were not present at build time)")
    st, x = stim
    problems, seen = check_model(O.RefModel, st, x, model)
    assert not problems, "reference model %d differs from the predicted frames (stream, channel, got, want, ...): %r" % (model, problems[:4])
    DL.assert_boundaries(st.designs, seen, "reference model %d" % model)


@pytest.mark.parametrize("model", [O.MODEL_STANDARD, O.MODEL_BASE, O.MODEL_DEFAULT])
def test_port_publishes_predicted(built, stim, model):
    st, x = stim
    problems, seen = check_model(O.PortModel, st, x, model)
    assert not problems, "ais_oracle.c model %d differs from the predicted frames (stream, channel, got, want, ...): %r" % (model, problems[:4])
    DL.assert_boundaries(st.designs, seen, "ais_oracle.c model %d" % model)
