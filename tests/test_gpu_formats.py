"""-m gpu: the output records formatted on the device (aisgpu_lines_enable / aisgpu_poll_lines), every message format.  The records
an engine returns must equal aisgpu_msg_format of the same polled frames, in order, from a fresh counter state (the host build of
the same formatter) and, when the harness is built, the reference's OutputMessage records for them; record i belongs to frame i.
Frames, sentences and counters must not change with a format on.  Also checked: the counters carried across 4096-frame decode
batches and poll tickets, the byte budget, a small cap, the queue bound, JSON_FULL against aisgpu_json_enable, and groups whose
members use different formats."""
import ctypes as C

import numpy as np
import pytest

import aisgpu
import aissynth as S
import oracle_fmt
from test_gpu_json_full import inputs

pytestmark = pytest.mark.gpu

B = 4
NSUB = 4
TAG = dict(version=77, driver=2, hardware="H100", mode=7, rxtime_us=1700000000123456, toa_us=0, station=12, status=0, ipv4=0,
           include_ssl=False, uuid=None, suffix=None)
FORMATS = list(range(1, 10))


def tag(**kw):
    t = dict(TAG)
    t.update(kw)
    return aisgpu.make_tag(**t)


def host_records(frames, fmt, tg):
    st = aisgpu.FormatState(0, 0)
    return [aisgpu.msg_format(m, tg, fmt, st) for m in frames]


def ref_records(frames, fmt, t):
    oracle_fmt.hub(0)
    oracle_fmt.group_seed(0)
    return [oracle_fmt.ref_record(fmt, m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value, C.c_float(m.ppm).value,
                                  t["version"], t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"], t["station"],
                                  t["include_ssl"], m.start_idx, m.end_idx, t["uuid"] or "", t["status"], t["ipv4"], t["suffix"])
            for m in frames]


def run(kw, xs, n, fmt=None, tg=None, cap=1 << 24):
    """(frames, record bytes, record count, counters, overflows) of NSUB submits of n samples per stream, polled by ticket."""
    e = aisgpu.Engine(n_streams=B, max_chunk=n, **kw)
    if fmt is not None:
        e.lines_enable(fmt, tg if tg is not None else tag(), cap)
    frames, text, nrec = [], [], 0
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
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
    counters, ov = e.counters(), e.overflows
    e.close()
    return frames, b"".join(text), nrec, counters, ov


def check(frames, text, nrec, fmt, t, with_ref=True):
    want = host_records(frames, fmt, aisgpu.make_tag(**t))
    assert nrec == len(frames)
    assert text == b"".join(want)
    if with_ref and oracle_fmt.have_ref():
        assert want == ref_records(frames, fmt, t)


CASES = [
    ("M2_1536k_CF32", dict(model=aisgpu.MODEL_DEFAULT, sample_rate=1536000), 1536000, aisgpu.MODE_AB),
    ("M0_1536k_CF32", dict(model=aisgpu.MODEL_STANDARD, sample_rate=1536000), 1536000, aisgpu.MODE_AB),
    ("M2_X48k_CF32", dict(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX"), 48000,
     aisgpu.MODE_X),
    ("M0_X48k_CF32", dict(model=aisgpu.MODEL_STANDARD, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX"), 48000,
     aisgpu.MODE_X),
]


@pytest.mark.parametrize("name,kw,fs,mode", CASES, ids=[c[0] for c in CASES])
def test_every_format_matches_host_and_reference(name, kw, fs, mode):
    n = 131072 if fs > 100000 else 8192
    xs = inputs(fs, n * NSUB, 1500, mode, fuzz=mode == aisgpu.MODE_AB)
    f0, _, _, _, _ = run(kw, xs, n)
    if mode == aisgpu.MODE_AB:
        # own MMSI: a multi-sentence frame's MMSI becomes the receiver's, so its sentences are !AIVDO
        own = next(int.from_bytes(bytes(m.data[1:5]), "big") >> 2 & 0x3FFFFFFF for m in f0 if len(m.nmea) > 1)
        kw = dict(kw, own_mmsi=own)
    f0, _, _, c0, _ = run(kw, xs, n)
    assert f0
    if mode == aisgpu.MODE_AB:
        assert any(len(m.nmea) > 1 for m in f0) and any(s.startswith("!AIVDO") for m in f0 for s in m.nmea)
    for fmt in FORMATS:
        t = dict(TAG, mode=[7, 1, 2, 0, 3, 5, 6, 7, 4][fmt - 1], include_ssl=fmt % 2 == 0, uuid="u-%d" % fmt if fmt == 6 else None,
                 suffix="\n" if fmt in (1, 7) else None, status=3 if fmt == 3 else 0)
        frames, text, nrec, counters, ov = run(kw, xs, n, fmt, aisgpu.make_tag(**t))
        assert ov == 0
        assert [m.key() for m in frames] == [m.key() for m in f0]
        assert [(m.stream, m.chunk, m.start_idx, m.end_idx, m.level, m.ppm) for m in f0] == \
            [(m.stream, m.chunk, m.start_idx, m.end_idx, m.level, m.ppm) for m in frames]
        assert counters == c0
        check(frames, text, nrec, fmt, t)


def test_counters_carry_across_decode_batches_and_tickets():
    """More than 4096 frames in one drain: the NMEA_TAG group id and the COMMUNITY_HUB ordinal continue across decode batches and
    across polls by ticket."""
    fs, n, b, nsub = 1536000, 65536, 384, 8
    xs = [S.random_stream(fs, n * nsub, 1300 + s, bursts_per_sec=(30, 30), multi_sentence=True)[0] for s in range(8)]
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    for fmt in (aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.MSGFORMAT_COMMUNITY_HUB):
        for split in (False, True):
            e = aisgpu.Engine(n_streams=b, max_chunk=n, **kw)
            e.lines_enable(fmt, tag(), 1 << 30)
            frames, text, nrec = [], [], 0
            for c in range(nsub):
                e.submit(np.ascontiguousarray(np.stack([xs[s % 8][c * n:(c + 1) * n] for s in range(b)])), n)
                if split and c in (2, 5):
                    x, k = e.poll_lines(c)
                    text.append(x)
                    nrec += k
                    frames += e.poll_upto(c)
            x, k = e.poll_lines()
            text.append(x)
            nrec += k
            frames += e.poll()
            e.close()
            assert len(frames) > 4096 and sum(len(m.nmea) > 1 for m in frames) > 100
            check(frames, b"".join(text), nrec, fmt, TAG, with_ref=False)


def test_budget_cap_and_queue_bound():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 700)
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    fmt = aisgpu.MSGFORMAT_JSON_SPARSE
    frames, text, nrec, _, _ = run(kw, xs, n, fmt)
    recs = host_records(frames, fmt, tag())
    per = {}
    for m, r in zip(frames, recs):
        per.setdefault(m.chunk, []).append(r)
    # the byte budget keeps a prefix of each submit's records
    cap = max(sum(len(r) for r in v) for v in per.values()) // 2
    _, cut, k, _, ov = run(kw, xs, n, fmt, cap=cap)
    want = []
    for c in sorted(per):
        used = 0
        for r in per[c]:
            used += len(r)
            if used > cap:
                break
            want.append(r)
    assert ov >= 1 and k == len(want) and cut == b"".join(want)
    # a cap smaller than the next record; poll_json on an engine of another format
    lib = aisgpu.load()
    e = aisgpu.Engine(n_streams=B, max_chunk=n, **kw)
    e.lines_enable(fmt, tag())
    e.submit(np.ascontiguousarray(np.stack([x[:n] for x in xs])), n)
    nb, nr = C.c_size_t(0), C.c_int(0)
    buf = C.create_string_buffer(8)
    assert lib.aisgpu_poll_lines(e.h, -1, buf, 8, C.byref(nb), C.byref(nr)) == aisgpu.EINVAL
    assert lib.aisgpu_poll_json(e.h, -1, buf, 8, C.byref(nb), C.byref(nr)) == aisgpu.EINVAL
    e.close()
    # a caller that reads only records: all arrive, the unread frames are cut to max_frames
    cap_frames = max(len(v) for v in per.values())
    assert sum(len(v) for v in per.values()) > cap_frames
    e = aisgpu.Engine(n_streams=B, max_chunk=n, max_frames=cap_frames, **kw)
    e.lines_enable(fmt, tag())
    got, k = [], 0
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        x, kk = e.poll_lines(c)
        got.append(x)
        k += kk
    assert b"".join(got) == text and k == nrec and e.overflows == 0
    assert len(e.poll()) == cap_frames and e.overflows == 1
    e.close()


def test_enable_rules():
    lib = aisgpu.load()
    e = aisgpu.Engine(n_streams=1, max_chunk=65536)
    nb, nr = C.c_size_t(0), C.c_int(0)
    assert lib.aisgpu_poll_lines(e.h, -1, None, 0, C.byref(nb), C.byref(nr)) == aisgpu.EINVAL  # not enabled
    for fmt in (0, 10):
        assert lib.aisgpu_lines_enable(e.h, fmt, C.byref(tag()), 4096) == aisgpu.EINVAL
    assert lib.aisgpu_lines_enable(e.h, 2, C.byref(tag()), 4096) == 0
    assert lib.aisgpu_lines_enable(e.h, 3, C.byref(tag()), 4096) == aisgpu.EINVAL  # one format per engine
    assert lib.aisgpu_json_enable(e.h, C.byref(tag()), 4096) == aisgpu.EINVAL
    e.close()


def test_json_full_through_lines_equals_json_enable():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 800)
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    _, text, nrec, _, _ = run(kw, xs, n, aisgpu.MSGFORMAT_JSON_FULL, tag(suffix="\n"))
    e = aisgpu.Engine(n_streams=B, max_chunk=n, **kw)
    e.json_enable(tag())
    lines = []
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        lines += e.poll_json(c)
    lines += e.poll_json()
    e.close()
    assert nrec == len(lines) > 0 and text == "".join(l + "\n" for l in lines).encode("utf-8", "surrogateescape")


def test_group_members_format_their_own_frames():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 600)
    cfg = [(aisgpu.MODEL_DEFAULT, aisgpu.MSGFORMAT_NMEA_TAG), (aisgpu.MODEL_STANDARD, aisgpu.MSGFORMAT_JSON_ANNOTATED),
           (aisgpu.MODEL_V2, aisgpu.MSGFORMAT_FULL)]
    want = [run(dict(model=md, sample_rate=fs), xs, n, fmt)[1:3] for md, fmt in cfg]
    lead = aisgpu.Engine(n_streams=B, max_chunk=n, model=cfg[0][0], sample_rate=fs)
    engines = [lead] + [lead.attach(model=md) for md, _ in cfg[1:]]
    for e, (_, fmt) in zip(engines, cfg):
        e.lines_enable(fmt, tag())
    text, nrec = [[] for _ in engines], [0] * len(engines)
    for c in range(NSUB):
        lead.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        for i, e in enumerate(engines):
            b, k = e.poll_lines(c)
            text[i].append(b)
            nrec[i] += k
    for i, e in enumerate(engines):
        b, k = e.poll_lines()
        text[i].append(b)
        nrec[i] += k
        assert (b"".join(text[i]), nrec[i]) == want[i] and nrec[i] > 0
    for e in engines[1:] + [lead]:
        e.close()
