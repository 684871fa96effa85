"""-m gpu: a receiver per stream (aisgpu_set_receivers).  One batch mixes AB, CD and other designations, distinct stations, tag modes
0-7, and own MMSIs that occur in the streams' own traffic.
  - Frames: stream s of the table engine equals stream s of a plain engine created with s's receiver, bit for bit (NMEA, sequence
    ids, level, ppm, start / end index), for models 0, 2, 4 and 11 in AB mode, 0 and 2 in X mode, and model 3.
  - Records: in every format, the records equal aisgpu_msg_format of the polled frames with each stream's tag, in frame order from a
    zeroed state, and a sample of them the reference's record for that receiver; the table may come before or after the format.
  - Groups: a leader and a member with tables of their own each equal standalone engines of their tables.
  - Feeder: aisgpu_feed_files over per-stream recordings gives NMEA_TAG records whose s: is each file's station.
  - Rules on a live handle: refused after a submit, a second time, and with n != n_streams, and the handle is unchanged."""
import ctypes as C

import numpy as np
import pytest

import aisgpu
import aissynth as S
import disc_util as D
import mode_x_util as X
import oracle_fmt
import parity_util as U

pytestmark = pytest.mark.gpu

B = 40
NSUB = 3
KINDS = 8  # distinct receivers: stream s has receiver s % KINDS
LETTERS = ["AB", "CD", "12", "?X", "CD", "AB", "9Z", "?D"]
OUTPUT = dict(version=81, status=0, rxtime_us=1700000000654321, toa_us=0, include_ssl=False, uuid=None, suffix=None)


def inputs(kind):
    """(rate, chunk, per-stream flat arrays, values per sample) of the batch"""
    if kind == "AB":
        fs, n = 1536000, 65536
        xs = [S.random_stream(fs, n * NSUB, 3000 + s, bursts_per_sec=(10, 20), multi_sentence=True)[0] for s in range(B)]
        return fs, n, xs, 1
    if kind == "X":
        fs, n = 48000, 8192
        return fs, n, [X.stream_input(fs, n * NSUB, 3100 + s, aisgpu.FMT_CF32)[0] for s in range(B)], 1
    fs, n = 48000, 8192
    raws = [D.stream_input(fs, n * NSUB, 3200 + s, aisgpu.FMT_CF32, True) for s in range(B)]
    return fs, n, [r for r, _ in raws], raws[0][1]


def chunk(xs, per, n, c):
    return np.ascontiguousarray(np.stack([x[c * n * per:(c + 1) * n * per] for x in xs]))


def engine_kw(model, kind, fs):
    kw = dict(model=model, sample_rate=fs, n_streams=B)
    if kind == "X":
        kw.update(channel_mode=aisgpu.MODE_X, channels="XX")
    return kw


def run(kw, xs, per, n, receivers=None, fmt=None, before=True):
    """(frames, record bytes, record count, counters) of NSUB submits polled by ticket"""
    e = aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw)
    if receivers is not None and before:
        e.set_receivers(receivers)
    if fmt is not None:
        e.lines_enable(fmt, aisgpu.make_tag(**OUTPUT), 1 << 26)
    if receivers is not None and not before:
        e.set_receivers(receivers)
    frames, text, nrec = [], [], 0
    for c in range(NSUB):
        e.submit(chunk(xs, per, n, c), n)
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
    counters = e.counters()
    assert e.overflows == 0
    e.close()
    return frames, b"".join(text), nrec, counters


def mmsi(m):
    return int.from_bytes(bytes(m.data[1:5]), "big") >> 2 & 0x3FFFFFFF


def table(frames0):
    """KINDS receivers; the odd ones own an MMSI of their first stream's traffic (so !AIVDO comes out)"""
    rx = []
    for k in range(KINDS):
        own = next((mmsi(m) for m in frames0 if m.stream == k and m.nbits >= 38), -1) if k % 2 else -1
        rx.append(dict(channels=LETTERS[k], station=100 + k if k != 3 else 0, own_mmsi=own, tag_mode=k, driver=k * 3,
                       hardware=["", "RTL-SDR", 'rx "n"\\1', "H100"][k % 4], ipv4=0 if k % 3 else 0x0A000001 + k))
    return rx


def tag_fields(rx):
    t = dict(OUTPUT)
    t.update(station=rx["station"], driver=rx["driver"], hardware=rx["hardware"], mode=rx["tag_mode"], ipv4=rx["ipv4"])
    return t


def per_stream(frames):
    out = [[] for _ in range(B)]
    for m in frames:
        out[m.stream].append(m)
    return out


def plain_kw(kw, rx):
    return dict(kw, channels=rx["channels"], own_mmsi=rx["own_mmsi"], tag_mode=rx["tag_mode"])


def check_against_plain(kw, xs, per, n, rxs, frames):
    """stream s of frames equals stream s of a plain engine of its receiver"""
    got = per_stream(frames)
    for k, rx in enumerate(rxs):
        want = per_stream(run(plain_kw(kw, rx), xs, per, n)[0])
        streams = list(range(k, B, KINDS))
        problems = U.compare_frames([got[s] for s in streams], [want[s] for s in streams])
        assert not problems, (k, rx, problems[:2])
        assert all(len(got[s]) for s in streams)


CASES = [("M0_AB", 0, "AB"), ("M2_AB", 2, "AB"), ("M4_AB", 4, "AB"), ("M11_AB", 11, "AB"), ("M0_X", 0, "X"), ("M2_X", 2, "X"),
         ("M3", 3, "DISC")]


@pytest.mark.parametrize("name,model,kind", CASES, ids=[c[0] for c in CASES])
def test_frames_equal_plain_engines_of_each_receiver(name, model, kind):
    fs, n, xs, per = inputs(kind)
    kw = engine_kw(model, kind, fs)
    frames0 = run(kw, xs, per, n)[0]
    rxs = table(frames0)
    frames, _, _, counters = run(kw, xs, per, n, receivers=[rxs[s % KINDS] for s in range(B)])
    assert any(s.startswith("!AIVDO") for m in frames for s in m.nmea)
    assert {m.channel for m in frames} >= {rx["channels"][0] for rx in rxs}
    # the counters of the first / second channel do not depend on the letters (none of LETTERS repeats its first letter)
    first = sum(1 for m in frames if m.channel == rxs[m.stream % KINDS]["channels"][0])
    assert counters[5] == (len(frames) if kind == "X" else first)
    assert counters[5] + counters[6] == counters[1] == len(frames)
    check_against_plain(kw, xs, per, n, rxs, frames)


def expected_records(frames, rxs, fmt):
    st = aisgpu.FormatState(0, 0)
    return [aisgpu.msg_format(m, aisgpu.make_tag(**tag_fields(rxs[m.stream % KINDS])), fmt, st) for m in frames]


def ref_records(frames, rxs, fmt):
    oracle_fmt.hub(0)
    oracle_fmt.group_seed(0)
    out = []
    for m in frames:
        t = tag_fields(rxs[m.stream % KINDS])
        out.append(oracle_fmt.ref_record(fmt, m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value, C.c_float(m.ppm).value,
                                         t["version"], t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"],
                                         t["station"], t["include_ssl"], m.start_idx, m.end_idx, t["uuid"] or "", t["status"],
                                         t["ipv4"], t["suffix"]))
    return out


@pytest.mark.parametrize("fmt", range(1, 10))
def test_records_are_each_streams_own(fmt):
    fs, n, xs, per = inputs("AB")
    kw = engine_kw(2, "AB", fs)
    rxs = table(run(kw, xs, per, n)[0])
    table_rx = [rxs[s % KINDS] for s in range(B)]
    frames, text, nrec, _ = run(kw, xs, per, n, receivers=table_rx, fmt=fmt, before=fmt % 2 == 1)
    assert nrec == len(frames) > 0
    want = expected_records(frames, rxs, fmt)
    assert text == b"".join(want)
    if fmt == aisgpu.MSGFORMAT_NMEA_TAG:
        for m, r in zip(frames, want):
            assert r.startswith(b"\\s:s%d," % rxs[m.stream % KINDS]["station"])
    if oracle_fmt.have_ref():  # a prefix of the run: the reference's counters start from a fresh output as the engine's do
        assert want[:300] == ref_records(frames[:300], rxs, fmt)


def test_group_leader_and_member_have_their_own_tables():
    fs, n, xs, per = inputs("AB")
    kw = engine_kw(2, "AB", fs)
    rxs = table(run(kw, xs, per, n)[0])
    t_lead = [rxs[s % KINDS] for s in range(B)]
    t_mem = [dict(rxs[(s + 3) % KINDS], station=500 + s) for s in range(B)]
    lead = aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw)
    mem = lead.attach(model=aisgpu.MODEL_STANDARD)
    lead.set_receivers(t_lead)
    mem.lines_enable(aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.make_tag(**OUTPUT), 1 << 26)
    mem.set_receivers(t_mem)
    got_l, got_m = [], []
    for c in range(NSUB):
        lead.submit(chunk(xs, per, n, c), n)
        got_l += lead.poll_upto(c)
        got_m += mem.poll_upto(c)
    got_l += lead.poll()
    got_m += mem.poll()
    text, nrec = mem.poll_lines()
    mem.close()
    lead.close()
    for got, tab, model in ((got_l, t_lead, 2), (got_m, t_mem, 0)):
        want = run(dict(kw, model=model), xs, per, n, receivers=tab)[0]
        assert not U.compare_frames(per_stream(got), per_stream(want))
    st = aisgpu.FormatState(0, 0)
    assert nrec == len(got_m)
    assert text == b"".join(aisgpu.msg_format(m, aisgpu.make_tag(**dict(OUTPUT, station=t_mem[m.stream]["station"],
                                                                          driver=t_mem[m.stream]["driver"],
                                                                          hardware=t_mem[m.stream]["hardware"],
                                                                          mode=t_mem[m.stream]["tag_mode"],
                                                                          ipv4=t_mem[m.stream]["ipv4"])),
                                              aisgpu.MSGFORMAT_NMEA_TAG, st) for m in got_m)


def test_feed_files_attributes_each_station(tmp_path):
    fs, n, xs, per = inputs("AB")
    paths = []
    for s, x in enumerate(xs):
        p = tmp_path / ("station%03d.cf32" % s)
        np.asarray(x, dtype=np.complex64).tofile(p)
        paths.append(str(p))
    rx = [dict(channels="AB" if s % 2 else "CD", station=1000 + s, tag_mode=3, hardware="site-%d" % s) for s in range(B)]
    e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=n, max_frames=1 << 16)
    e.set_receivers(rx)
    e.lines_enable(aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.make_tag(**OUTPUT), 1 << 26)
    frames, blocks = e.feed_files(paths, n)
    text, nrec = e.poll_lines()
    e.close()
    assert blocks == NSUB and nrec == len(frames) > 0
    st = aisgpu.FormatState(0, 0)
    recs = [aisgpu.msg_format(m, aisgpu.make_tag(**dict(OUTPUT, station=1000 + m.stream, hardware="site-%d" % m.stream)),
                              aisgpu.MSGFORMAT_NMEA_TAG, st) for m in frames]
    assert text == b"".join(recs)
    for m, r in zip(frames, recs):
        assert all(line.startswith(b"\\s:s%d," % (1000 + m.stream)) for line in r.split(b"\r\n") if line)
        assert m.channel in ("AB" if m.stream % 2 else "CD")
    assert len({m.stream for m in frames}) > B // 2


def test_rules_on_a_live_handle():
    fs, n, xs, per = inputs("AB")
    kw = engine_kw(2, "AB", fs)
    rxs = table(run(kw, xs, per, n)[0])
    tab = [rxs[s % KINDS] for s in range(B)]
    other = [dict(r, channels="??", tag_mode=0) for r in tab]

    def refused(e, rx):
        with pytest.raises(aisgpu.AisGpuError):
            e.set_receivers(rx)

    def drive(e):
        out = []
        for c in range(NSUB):
            e.submit(chunk(xs, per, n, c), n)
            out += e.poll_upto(c)
        return out + e.poll()

    plain = drive_close(aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw), drive)
    with_tab = run(kw, xs, per, n, receivers=tab)[0]
    # n != n_streams: refused, and the engine stays plain
    e = aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw)
    refused(e, tab[:-1])
    refused(e, tab + tab[:1])
    refused(e, [dict(tab[0], channels="A,")] + tab[1:])
    assert not U.compare_frames(per_stream(drive_close(e, drive)), per_stream(plain))
    # a second table: refused, the first one stays
    e = aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw)
    e.set_receivers(tab)
    refused(e, other)
    assert not U.compare_frames(per_stream(drive_close(e, drive)), per_stream(with_tab))
    # after a submit: refused, the engine stays plain
    e = aisgpu.Engine(max_chunk=n, max_frames=1 << 16, **kw)
    got = []
    e.submit(chunk(xs, per, n, 0), n)
    refused(e, tab)
    got += e.poll_upto(0)
    for c in range(1, NSUB):
        e.submit(chunk(xs, per, n, c), n)
        got += e.poll_upto(c)
    got += e.poll()
    e.close()
    assert not U.compare_frames(per_stream(got), per_stream(plain))


def drive_close(e, drive):
    out = drive(e)
    e.close()
    return out
