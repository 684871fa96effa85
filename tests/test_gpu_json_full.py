"""-m gpu: the full AIS JSON decoded on the device (aisgpu_json_enable / aisgpu_poll_json).  Every line the engine returns must equal
aisgpu_msg_json_full of the same polled frame (the host build of the same interpreter) and, when the harness is built, the
reference's JSONAIS line for it; line i belongs to frame i.  Frames, sentences and counters must not change with JSON on.  Also
checked: random payloads carried by synthetic bursts (every type, random lengths), text overflow, poll tickets, and groups."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import aisgpu
import aissynth as S
import json_cases
import mode_x_util as X
import oracle_json

pytestmark = pytest.mark.gpu

B = 4
NSUB = 4
TAG = dict(version=77, driver=2, hardware="H100", mode=7, rxtime_us=1700000000123456, toa_us=0, station=12)


def tag(**kw):
    t = dict(TAG)
    t.update(kw)
    return aisgpu.make_tag(**t)


def ref_line(m, t):
    return oracle_json.ref_line(m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value, C.c_float(m.ppm).value, t["version"],
                                t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"], t["station"])


def fuzz_stream(fs, n, seed):
    """A stream whose bursts carry random payloads: every message type, random contents, from the type's published minimum to
    600 bits, and the (DAC, FI) pairs of the application messages."""
    rng = np.random.default_rng(seed)
    prng = random.Random(seed)
    bursts, t = [], 0
    for ch in "AB":
        t = int(rng.integers(0, 2000))
        while True:
            typ = prng.randint(1, 28)
            ml = (json_cases.MIN_BITS[typ - 1] + 7) // 8 * 8  # whole bytes, at least the length the type is published with
            nbits = prng.choice([ml, max(ml, 168), prng.randrange(ml, max(ml, 600) + 8, 8)])
            d = json_cases.msg(prng, typ)
            if typ in (6, 8) and prng.random() < 0.6:
                dac, fid = prng.choice(json_cases.ASM6 if typ == 6 else json_cases.ASM8)
                json_cases.setu(d, 72 if typ == 6 else 40, 10, dac)
                json_cases.setu(d, 82 if typ == 6 else 50, 6, fid)
            bits = np.array([(d[i >> 3] >> (7 - (i & 7))) & 1 for i in range(nbits)], dtype=np.uint8)
            ln = S.burst_len_samples(nbits, fs)
            start = t + int(rng.integers(ln // 8, ln // 2 + 1))
            if start + ln >= n:
                break
            bursts.append(S.Burst(start, ch, bits, amp=rng.uniform(0.1, 0.5), foffs=rng.uniform(-400, 400), timing=rng.uniform(0, 1)))
            t = start + ln
    return S.render_stream(fs, n, bursts, seed=seed)


def inputs(fs, n, seed, mode=aisgpu.MODE_AB, fuzz=False):
    if mode == aisgpu.MODE_X:
        return [X.stream_input(fs, n, seed + s, aisgpu.FMT_CF32)[0] for s in range(B)]
    if fuzz:
        return [fuzz_stream(fs, n, seed + s) for s in range(B)]
    return [S.random_stream(fs, n, seed + s, bursts_per_sec=(10, 20), multi_sentence=True)[0] for s in range(B)]


def run(kw, xs, n, json_tag=None, cap=1 << 24, per_ticket=True):
    """(frames, lines, counters, overflows) of NSUB submits of n samples per stream."""
    e = aisgpu.Engine(n_streams=B, max_chunk=n, **kw)
    if json_tag is not None:
        e.json_enable(json_tag, cap)
    frames, lines = [], []
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        if per_ticket:
            frames += e.poll_upto(c)
            if json_tag is not None:
                lines += e.poll_json(c)
    frames += e.poll()
    if json_tag is not None:
        lines += e.poll_json()
    counters = e.counters()
    ov = e.overflows
    e.close()
    return frames, lines, counters, ov


def check_lines(frames, lines, t, with_ref=True):
    assert len(lines) == len(frames)
    tg = aisgpu.make_tag(**t)
    use_ref = with_ref and oracle_json.have_ref()
    for m, line in zip(frames, lines):
        got = line.encode("utf-8", "surrogateescape")
        host = aisgpu.msg_json_full(m, tg)
        assert got == host, "device %r\nhost   %r" % (got, host)
        if use_ref:
            assert got == ref_line(m, t)


CASES = [
    ("M2_1536k_CF32", dict(model=aisgpu.MODEL_DEFAULT, sample_rate=1536000), 1536000, aisgpu.MODE_AB),
    ("M0_1536k_CF32", dict(model=aisgpu.MODEL_STANDARD, sample_rate=1536000), 1536000, aisgpu.MODE_AB),
    ("M11_1536k_CF32", dict(model=aisgpu.MODEL_V2, sample_rate=1536000), 1536000, aisgpu.MODE_AB),
    ("M2_X48k_CF32", dict(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX"), 48000,
     aisgpu.MODE_X),
]


@pytest.mark.parametrize("name,kw,fs,mode", CASES, ids=[c[0] for c in CASES])
def test_lines_match_host_and_reference(name, kw, fs, mode):
    n = 65536 if fs > 100000 else 8192
    xs = inputs(fs, n * NSUB, 500, mode)
    frames, lines, counters, ov = run(kw, xs, n, tag(), per_ticket=True)
    assert frames and ov == 0
    check_lines(frames, lines, TAG)
    # frames, sentences and counters are the same without JSON
    f0, _, c0, _ = run(kw, xs, n, None)
    assert [m.key() for m in f0] == [m.key() for m in frames]
    assert [(m.stream, m.chunk, m.start_idx, m.end_idx, m.level, m.ppm) for m in f0] == \
        [(m.stream, m.chunk, m.start_idx, m.end_idx, m.level, m.ppm) for m in frames]
    assert c0 == counters


@pytest.mark.parametrize("model", [aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD])
def test_fuzzed_payloads(model):
    fs, n = 1536000, 131072
    xs = inputs(fs, n * NSUB, 900 + model, fuzz=True)
    for mode in (0, 5, 7):
        t = dict(TAG, mode=mode, station=0 if mode == 5 else 3)
        frames, lines, _, ov = run(dict(model=model, sample_rate=fs), xs, n, aisgpu.make_tag(**t))
        types = {m.data[0] >> 2 for m in frames}
        assert len(types) >= 12 and ov == 0, types
        check_lines(frames, lines, t)


def test_text_overflow_keeps_a_prefix_of_each_submit():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 700)
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    frames, full, _, _ = run(kw, xs, n, tag())
    per = {}
    for m, l in zip(frames, full):
        per.setdefault(m.chunk, []).append(l)
    cap = max(sum(len(l.encode("utf-8", "surrogateescape")) + 1 for l in v) for v in per.values()) // 2
    frames2, cut, _, ov = run(kw, xs, n, tag(), cap=cap)
    assert ov >= 1 and len(cut) < len(full)
    want = []
    for c in sorted(per):
        used = 0
        for l in per[c]:
            used += len(l.encode("utf-8", "surrogateescape")) + 1
            if used > cap:
                break
            want.append(l)
    assert cut == want
    assert [m.key() for m in frames2] == [m.key() for m in frames]


def test_tickets_and_poll_order():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 800)
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    frames, lines, _, _ = run(kw, xs, n, tag(), per_ticket=False)
    e = aisgpu.Engine(n_streams=B, max_chunk=n, **kw)
    e.json_enable(tag())
    got = []
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
    for c in range(NSUB):  # JSON first, frames never polled: the lines still come in frame order
        got += e.poll_json(c)
    e.close()
    assert got == lines
    check_lines(frames, lines, TAG, with_ref=False)


def test_group_members_decode_their_own_frames():
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 600)
    models = [aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD, aisgpu.MODEL_V2]
    want = [run(dict(model=md, sample_rate=fs), xs, n, tag()) for md in models]
    lead = aisgpu.Engine(n_streams=B, max_chunk=n, model=models[0], sample_rate=fs)
    mem = [lead.attach(model=md) for md in models[1:]]
    engines = [lead] + mem
    for e in engines:
        e.json_enable(tag())
    lines = [[] for _ in engines]
    for c in range(NSUB):
        lead.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        for i, e in enumerate(engines):
            lines[i] += e.poll_json(c)
    for i, e in enumerate(engines):
        lines[i] += e.poll_json()
        assert lines[i] == want[i][1] and lines[i]
    for e in mem + [lead]:
        e.close()


def test_enable_rules():
    e = aisgpu.Engine(n_streams=1, max_chunk=65536)
    lib = aisgpu.load()
    nb, nl = C.c_size_t(0), C.c_int(0)
    assert lib.aisgpu_poll_json(e.h, -1, None, 0, C.byref(nb), C.byref(nl)) == aisgpu.EINVAL  # not enabled
    assert lib.aisgpu_json_enable(e.h, C.byref(tag()), 0) == aisgpu.EINVAL
    assert lib.aisgpu_json_enable(e.h, C.byref(tag()), 4096) == 0
    assert lib.aisgpu_json_enable(e.h, C.byref(tag()), 4096) == aisgpu.EINVAL  # once
    e.close()
    e = aisgpu.Engine(n_streams=1, max_chunk=65536)
    e.submit(np.zeros((1, 65536), np.complex64), 65536)
    assert lib.aisgpu_json_enable(e.h, C.byref(tag()), 4096) == aisgpu.EINVAL  # after the first submit
    e.close()


def test_queues_are_bounded_when_one_is_not_read():
    """Frames and lines are queued side by side; a caller that reads only one of them keeps at most max_frames of the other."""
    fs, n = 1536000, 65536
    xs = inputs(fs, n * NSUB, 1100)
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)
    frames, lines, _, _ = run(kw, xs, n, tag())
    per = {}
    for m in frames:
        per[m.chunk] = per.get(m.chunk, 0) + 1
    cap_frames = max(per.values())  # every submit fits the ring, all of them do not
    assert sum(per.values()) > cap_frames
    # only lines: every line arrives; the frames left unread are cut to the newest max_frames
    e = aisgpu.Engine(n_streams=B, max_chunk=n, max_frames=cap_frames, **kw)
    e.json_enable(tag())
    got = []
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        got += e.poll_json(c)
    assert got == lines and e.overflows == 0
    left = e.poll()
    assert e.overflows == 1 and [m.key() for m in left] == [m.key() for m in frames[-cap_frames:]]
    e.close()
    # only frames: every frame arrives; the lines left unread are cut to the newest max_frames
    e = aisgpu.Engine(n_streams=B, max_chunk=n, max_frames=cap_frames, **kw)
    e.json_enable(tag())
    got = []
    for c in range(NSUB):
        e.submit(np.ascontiguousarray(np.stack([x[c * n:(c + 1) * n] for x in xs])), n)
        got += e.poll_upto(c)
    assert [m.key() for m in got] == [m.key() for m in frames] and e.overflows == 0
    assert e.poll_json() == lines[-cap_frames:] and e.overflows == 1
    e.close()


def test_submits_larger_than_a_decode_batch():
    """A drain of more than one 4096-frame decode batch: the lines of a submit split over two batches share its byte budget."""
    fs, n, b, nsub = 1536000, 65536, 256, 8
    xs = [S.random_stream(fs, n * nsub, 1200 + s, bursts_per_sec=(30, 30))[0] for s in range(8)]
    kw = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=fs)

    def go(cap):
        e = aisgpu.Engine(n_streams=b, max_chunk=n, **kw)
        e.json_enable(tag(), cap)
        for c in range(nsub):  # polled once at the end: one drain of every submit
            e.submit(np.ascontiguousarray(np.stack([xs[s % 8][c * n:(c + 1) * n] for s in range(b)])), n)
        fr, ln, ov = e.poll(), e.poll_json(), e.overflows
        e.close()
        return fr, ln, ov

    frames, lines, ov = go(1 << 30)
    assert ov == 0 and len(frames) > 4096 and len(lines) == len(frames)
    check_lines(frames, lines, TAG, with_ref=False)
    per = {}
    for m, l in zip(frames, lines):
        per.setdefault(m.chunk, []).append(len(l.encode("utf-8", "surrogateescape")) + 1)
    cap = max(sum(v) for v in per.values()) * 3 // 4
    _, cut, ov = go(cap)
    want = []
    for c in sorted(per):
        used = 0
        for l, m in zip(lines, frames):
            if m.chunk != c:
                continue
            used += len(l.encode("utf-8", "surrogateescape")) + 1
            if used > cap:
                break
            want.append(l)
    assert ov >= 1 and cut == want
