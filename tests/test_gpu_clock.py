"""-m gpu: a receive time per frame (aisgpu_set_clock).  Expected stamps are computed here, with Python integers, from the submit
lengths each test used: stamp(s, c) = start_us[s] + S_c * 10^6 // fs, S_c the samples per stream submitted through submit c.
  1. Recording clock, every format: models 2 and 0, AB at 1536 kS/s and at 288 kS/s (the /3 filter), streams with distinct starts
     (one with a microsecond fraction, one that crosses a new year during the run, one in the year 9999), submit lengths that change
     from call to call.  aisgpu_stamp is the formula, the whole aisgpu_poll_lines output is aisgpu_msg_format of every frame with
     its stamp from a zeroed state, and a sample of records is the reference's own record of that stamp.
  2. Live clock: the system clock read before and after each submit call brackets every stamp of that submit; all streams share it.
  3. Unchanged: frames, counters and taps are the same with and without a clock; without one the records carry the tag's time.
  4. Receivers: per-stream tag modes with bit 1 on and off; JSON_FULL and FULL print the stamp only where it is on, NMEA_TAG always.
  5. Feeders: aisgpu_feed_files over recordings of different lengths, stamped block by block, the zero-padded tail included.
  6. Groups: the leader's clock stamps a member's records, whether the member was attached before or after it was set.
  7. Rules on a live handle: after the first submit, a second time, on a group member, and aisgpu_stamp without a clock or out of
     range, are refused and leave the handle as it was."""
import ctypes as C
import re
import time

import numpy as np
import pytest

import aisgpu
import aissynth as S
import oracle_fmt
import parity_util as U

pytestmark = pytest.mark.gpu

B = 6
# distinct starts: whole seconds, a microsecond fraction, 0.2 s before 2026-01-01, the epoch, a year-2000 eve, the year 9999
STARTS = [1700000000000000, 1700000000654321, 1767225599800000, 0, 946684799999999, 253402300000000000]
TAG = dict(version=81, driver=3, hardware="clock-rx", mode=3, status=0, ipv4=0, rxtime_us=1234567890123456, toa_us=0, station=7,
           include_ssl=False, uuid=None, suffix=None)


def lengths(fs):
    """submit lengths (multiples of the granule, 64 at both rates) that change from call to call: about 0.4 s in all"""
    g = 64
    base = fs // 8 // g * g
    return [base, base // 2 // g * g + 3 * g, base + 11 * g, base * 3 // 4 // g * g]


def streams(fs, total, seed):
    return [S.random_stream(fs, total, seed + s, bursts_per_sec=(15, 25), multi_sentence=True)[0] for s in range(B)]


def block(xs, a, n):
    return np.ascontiguousarray(np.stack([x[a:a + n] for x in xs]))


def expected_stamp(starts, lens, fs, s, c):
    return starts[s] + sum(lens[:c + 1]) * 10 ** 6 // fs


def drive(e, xs, lens, fmt=None):
    """(frames, record bytes, record count) of the submits of lens, polled by ticket"""
    frames, text, nrec, a = [], [], 0, 0
    for c, n in enumerate(lens):
        e.submit(block(xs, a, n), n)
        a += n
        frames += e.poll_upto(c)
        if fmt is not None:
            b, k = e.poll_lines(c)
            text.append(b)
            nrec += k
    frames += e.poll()
    if fmt is not None:
        b, k = e.poll_lines()
        text.append(b)
        nrec += k
    assert e.overflows == 0
    return frames, b"".join(text), nrec


def records(frames, stamp, tag_of=lambda s: TAG, fmt=aisgpu.MSGFORMAT_JSON_FULL):
    """aisgpu_msg_format of every frame with its stream's tag and its stamp, from a zeroed state"""
    st = aisgpu.FormatState(0, 0)
    return [aisgpu.msg_format(m, aisgpu.make_tag(**dict(tag_of(m.stream), rxtime_us=stamp(m.stream, m.chunk))), fmt, st) for m in frames]


def ref_records(frames, stamp, fmt):
    oracle_fmt.hub(0)
    oracle_fmt.group_seed(0)
    t = TAG
    return [oracle_fmt.ref_record(fmt, m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value, C.c_float(m.ppm).value, t["version"],
                                  t["driver"], t["hardware"], t["mode"], stamp(m.stream, m.chunk), t["toa_us"], t["station"],
                                  t["include_ssl"], m.start_idx, m.end_idx, "", t["status"], t["ipv4"], t["suffix"]) for m in frames]


CASES = [(2, 1536000), (0, 1536000), (2, 288000), (0, 288000)]


@pytest.mark.parametrize("model,fs", CASES, ids=["M%d_%d" % c for c in CASES])
def test_recording_clock_every_format(model, fs):
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4100)
    stamp = lambda s, c: expected_stamp(STARTS, lens, fs, s, c)
    assert stamp(2, 0) < 1767225600000000 <= stamp(2, len(lens) - 1)  # stream 2 crosses into 2026
    for fmt in range(1, 10):
        e = aisgpu.Engine(model=model, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)
        if fmt % 2:
            e.set_clock(STARTS)
        e.lines_enable(fmt, aisgpu.make_tag(**TAG), 1 << 24)
        if not fmt % 2:  # the clock may come before or after the format
            e.set_clock(STARTS)
        frames, text, nrec = drive(e, xs, lens, fmt)
        for s in range(B):
            for c in range(len(lens)):
                assert e.stamp(s, c) == stamp(s, c)
        e.close()
        assert nrec == len(frames) > 3 * B
        assert len({m.chunk for m in frames}) > 1
        want = records(frames, stamp, fmt=fmt)
        assert text == b"".join(want), fmt
        if oracle_fmt.have_ref():
            pick = frames[::max(1, len(frames) // 24)]
            assert records(pick, stamp, fmt=fmt) == ref_records(pick, stamp, fmt), fmt


def test_live_clock_brackets_each_submit():
    fs = 1536000
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4200)
    e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)
    e.set_clock()
    e.lines_enable(aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.make_tag(**TAG), 1 << 24)
    frames, text, a, brackets = [], [], 0, []
    for c, n in enumerate(lens):
        x = block(xs, a, n)
        a += n
        t0 = time.time_ns() // 1000
        if c % 2:
            e.submit(x, n)
        else:
            e.submit_v(list(x), n)
        t1 = time.time_ns() // 1000
        brackets.append((t0, t1))
        frames += e.poll_upto(c)
        text.append(e.poll_lines(c)[0])
    stamps = {c: e.stamp(0, c) for c in range(len(lens))}
    for c, (t0, t1) in enumerate(brackets):
        assert t0 <= stamps[c] <= t1
        assert all(e.stamp(s, c) == stamps[c] for s in range(B))
    e.close()
    assert len(frames) > 3 * B
    assert b"".join(text) == b"".join(records(frames, lambda s, c: stamps[c], fmt=aisgpu.MSGFORMAT_NMEA_TAG))


def test_frames_counters_and_taps_unchanged():
    fs = 1536000
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4300)
    out = {}
    for clock in (False, True):
        e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14, taps=True)
        if clock:
            e.set_clock(STARTS)
        e.lines_enable(aisgpu.MSGFORMAT_JSON_FULL, aisgpu.make_tag(**TAG), 1 << 24)
        frames, text, nrec = drive(e, xs, lens, aisgpu.MSGFORMAT_JSON_FULL)
        taps = [e.tap(aisgpu.TAP_C, s, ch) for s in range(B) for ch in (0, 1)]
        out[clock] = (frames, text, e.counters(), taps)
        e.close()
    (f0, t0, c0, p0), (f1, t1, c1, p1) = out[False], out[True]
    per = lambda fr: [[m for m in fr if m.stream == s] for s in range(B)]
    assert not U.compare_frames(per(f1), per(f0))
    assert [m.chunk for m in f1] == [m.chunk for m in f0]
    assert c1 == c0
    assert all(U.bits_equal(a, b) for a, b in zip(p1, p0))
    assert t0 == b"".join(records(f0, lambda s, c: TAG["rxtime_us"]))  # without a clock: the tag's time
    assert t1 != t0 and t1 == b"".join(records(f1, lambda s, c: expected_stamp(STARTS, lens, fs, s, c)))


def test_receivers_decide_where_the_time_is_printed():
    fs = 1536000
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4400)
    rx = [dict(channels="AB", station=40 + s, tag_mode=[3, 1, 2, 0, 7, 5][s], driver=s, hardware="site-%d" % s) for s in range(B)]
    tag_of = lambda s: dict(TAG, station=rx[s]["station"], driver=rx[s]["driver"], hardware=rx[s]["hardware"], mode=rx[s]["tag_mode"])
    stamp = lambda s, c: expected_stamp(STARTS, lens, fs, s, c)
    for fmt in (aisgpu.MSGFORMAT_JSON_FULL, aisgpu.MSGFORMAT_FULL, aisgpu.MSGFORMAT_NMEA_TAG):
        e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)
        e.set_clock(STARTS)
        e.set_receivers(rx)
        e.lines_enable(fmt, aisgpu.make_tag(**TAG), 1 << 24)
        frames, text, nrec = drive(e, xs, lens, fmt)
        e.close()
        want = records(frames, stamp, tag_of, fmt)
        assert nrec == len(frames) > 3 * B and text == b"".join(want)
        for m, r in zip(frames, want):
            t = stamp(m.stream, m.chunk)
            if fmt == aisgpu.MSGFORMAT_NMEA_TAG:
                shown = [float(v) for v in re.findall(rb",c:([0-9.]+)", r)]
                assert len(shown) == len(m.nmea) and all(abs(v - t / 1e6) < 1e-3 for v in shown), (m.stream, r)
            else:
                shown = b'"rxtime":"' in r if fmt == aisgpu.MSGFORMAT_JSON_FULL else b", timestamp: " in r
                assert shown == bool(rx[m.stream]["tag_mode"] & 2), (fmt, m.stream, r)


def test_feed_files_stamped_by_block(tmp_path):
    fs, n = 1536000, 65536
    sizes = [n * 3 + 5000, n * 2, n * 5 + 64, n, n * 4 - 640, n * 3]  # the longest ends inside block 5
    xs = streams(fs, max(sizes), 4500)
    paths = []
    for s in range(B):
        p = tmp_path / ("rec%d.cf32" % s)
        np.asarray(xs[s][:sizes[s]], dtype=np.complex64).tofile(p)
        paths.append(str(p))
    e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=n, max_frames=1 << 14)
    e.set_clock(STARTS)
    e.lines_enable(aisgpu.MSGFORMAT_JSON_NMEA, aisgpu.make_tag(**TAG), 1 << 24)
    frames, blocks = e.feed_files(paths, n)
    text, nrec = e.poll_lines()
    assert blocks == 6 == -(-max(sizes) // n)
    stamp = lambda s, c: STARTS[s] + (c + 1) * n * 10 ** 6 // fs
    assert [e.stamp(s, c) for s in range(B) for c in range(blocks)] == [stamp(s, c) for s in range(B) for c in range(blocks)]
    with pytest.raises(aisgpu.AisGpuError):
        e.stamp(0, blocks)
    e.close()
    assert nrec == len(frames) > B
    assert text == b"".join(records(frames, stamp, fmt=aisgpu.MSGFORMAT_JSON_NMEA))


def test_group_members_take_the_leaders_clock():
    fs = 1536000
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4600)
    stamp = lambda s, c: expected_stamp(STARTS, lens, fs, s, c)
    lead = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)
    before = lead.attach(model=aisgpu.MODEL_STANDARD)
    with pytest.raises(aisgpu.AisGpuError, match="member of a group"):
        before.set_clock(STARTS)
    before.lines_enable(aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.make_tag(**TAG), 1 << 24)
    lead.set_clock(STARTS)
    after = lead.attach(model=aisgpu.MODEL_CHALLENGER)
    after.lines_enable(aisgpu.MSGFORMAT_JSON_FULL, aisgpu.make_tag(**TAG), 1 << 24)
    with pytest.raises(aisgpu.AisGpuError, match="member of a group"):
        after.set_clock(None)
    got = {"before": ([], []), "after": ([], [])}
    a = 0
    for c, n in enumerate(lens):
        lead.submit(block(xs, a, n), n)
        a += n
        for k, m in (("before", before), ("after", after)):
            got[k][0].extend(m.poll_upto(c))
            got[k][1].append(m.poll_lines(c)[0])
    for m in (before, after):
        assert [m.stamp(s, c) for s in range(B) for c in range(len(lens))] == \
            [stamp(s, c) for s in range(B) for c in range(len(lens))]
    after.close()
    before.close()
    lead.close()
    for k, fmt in (("before", aisgpu.MSGFORMAT_NMEA_TAG), ("after", aisgpu.MSGFORMAT_JSON_FULL)):
        frames, text = got[k]
        assert len(frames) > 3 * B
        assert b"".join(text) == b"".join(records(frames, stamp, fmt=fmt))


def test_rules_on_a_live_handle():
    fs = 1536000
    lens = lengths(fs)
    xs = streams(fs, sum(lens), 4700)
    mk = lambda: aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)

    def refused(f, *args):
        with pytest.raises(aisgpu.AisGpuError):
            f(*args)

    # without a clock: no stamps; a clock after the first submit is refused and the engine keeps none
    e = mk()
    refused(e.stamp, 0, 0)
    e.submit(block(xs, 0, lens[0]), lens[0])
    refused(e.set_clock, STARTS)
    refused(e.set_clock, None)
    refused(e.stamp, 0, 0)
    e.close()
    # refused tables leave the handle without a clock
    e = mk()
    refused(e.set_clock, STARTS[:-1])
    refused(e.set_clock, STARTS[:-1] + [-1])
    refused(e.set_clock, STARTS[:-1] + [253402300800000000])
    refused(e.stamp, 0, 0)
    # a second clock is refused and the first one stays
    e.set_clock(STARTS)
    refused(e.set_clock, [1] * B)
    refused(e.set_clock, None)
    e.submit(block(xs, 0, lens[0]), lens[0])
    assert [e.stamp(s, 0) for s in range(B)] == [expected_stamp(STARTS, lens, fs, s, 0) for s in range(B)]
    # out of range: streams and submits that do not exist
    for s, c in ((-1, 0), (B, 0), (0, -1), (0, 1), (0, 1 << 40)):
        refused(e.stamp, s, c)
    e.close()
