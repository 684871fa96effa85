"""Several tunings of one input on the GPU (aisgpu_set_tunings, per_input = T), bit for bit (tolerance 0) against the compiled reference.

The engine decodes n_streams streams from R = n_streams / T input rows; stream s reads row s / T with its own offset.  Stream s must
yield exactly what the reference yields on aisgpu_tune_restate(format, fs, offset[s], 0, input row s / T) as CF32, fed in the same
blocks: the frames (payload, NMEA, channel, start / end counters, level and ppm bit patterns) and, at rates without a resampler, every
tap of each submit.  Each input carries traffic at each of its T offsets, so every tuning of it has something to decode.
  1. Four channels, one engine: a 12.288 MS/s CS16 capture with A/B at +2.6 MHz and C/D at -2.6 MHz, T = 2, receivers AB / CD; it
     also equals the two-engine arrangement (one engine per pair) on the same recordings.
  2. Every input format at 1536 kS/s with T = 2 and T = 3, offsets of 0 among them.   3. Single-channel mode, two channels per input.
  4. The pre-stage paths: a resampled rate, a DownsampleKFilter rate, a resampler that the tune feeds directly (D0).
  5. Every input entry point: host, per-row pointers, async + poll_upto, device batches at a padded stride and offset base, changing
     lengths, aisgpu_feed_files and aisgpu_feed_wav_files over R files of different lengths.
  6. A fan leader with members.   7. The channel dump.   8. Receivers and a recording clock: records and stamps per stream.
  9. T = 1 is aisgpu_set_tuning; refused calls leave the handle untouched; Python refuses n_streams rows on a fan engine."""
import numpy as np
import pytest

import afc_signals as A
import aisgpu
import dc16h_util as DC
import fs4_util as F4
import oracle as O
import oracle_x as OX
import parity_util as U
import wav_util as W

pytestmark = pytest.mark.gpu

AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS8, CS16, FS4, DC16H = (aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16, aisgpu.FMT_F32_FS4,
                                    aisgpu.FMT_DC16H)
M0, M2, M4, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2
PER = {CF32: 1, CU8: 2, CS8: 2, CS16: 2, FS4: 1, DC16H: 3}  # raw array elements per sample
WIDE = 2600000  # 162.000 MHz (A/B) and 156.800 MHz (C/D) either side of a capture centred at 159.4 MHz


def need_ref(mode):
    if not (OX.have_refx() if mode == MX else O.have_ref()):
        pytest.skip("the tune is checked against the compiled reference only")


def placed(fs, n, f, seed, mode):
    """Traffic centred on f Hz: the pair at f -+ 25 kHz (AB), or one channel at f (X), with small carrier errors of its own."""
    x = A.row(fs, n, float((seed * 37) % 600 - 300), seed, kind=A.X_ if mode == MX else A.AB).astype(np.complex128)
    return (x * np.exp(2j * np.pi * f * np.arange(n, dtype=np.float64) / fs)).astype(np.complex64)


def fan_input(fs, n, offsets, seed, mode):
    """One input row with traffic at each of its tunings' offsets"""
    x = sum(placed(fs, n, f, seed + 11 * t, mode).astype(np.complex128) for t, f in enumerate(offsets))
    return (x / len(offsets)).astype(np.complex64)


def to_raw(x, fmt, seed=0):
    if fmt == FS4:
        return F4.real_stream(x)
    if fmt == DC16H:
        return DC.from_complex(x, seed)[0]
    return A.to_raw(x, fmt)[0]


def inputs(fmt, fs, n, offsets, T, mode, seed=40):
    R = len(offsets) // T
    return [to_raw(fan_input(fs, n, offsets[r * T:(r + 1) * T], seed + r, mode), fmt, r) for r in range(R)]


def reference(model, fs, mode, dsk=False):
    flags = O.DEFAULT_FLAGS | (O.FLAG_DSK if dsk else 0)
    if mode == MX:
        return OX.RefModelX(model=model, sample_rate=fs, fmt=CF32, flags=flags, taps=True)
    return O.RefModel(model=model, sample_rate=fs, fmt=CF32, flags=flags, taps=True)


def resampled(fs, mode, dsk):
    if mode == MX:
        return fs not in (48000, 96000, 192000)
    buckets = (96000, 192000, 288000, 384000, 576000, 768000, 1152000, 1536000, 2304000, 3072000, 6144000, 12288000) if dsk else \
        (96000, 192000, 384000, 768000, 1536000, 3072000, 6144000, 12288000)
    return fs not in buckets or fs in (288000, 576000, 1152000, 2304000)


def lengths_of(n, schedule):
    out, i = [], 0
    while sum(out) + schedule[i % len(schedule)] <= n:
        out.append(schedule[i % len(schedule)])
        i += 1
    return out


def submit(eng, blk, n, how, keep):
    """One submit of the R rows blk through entry point `how`; returns the frames it published (polled by ticket for "async")."""
    import torch
    batch = np.ascontiguousarray(np.stack(blk))
    if how == "host":
        eng.submit(batch, n)
        return eng.poll()
    if how == "v":
        eng.submit_v(list(blk), n)
        return eng.poll()
    if how == "async":
        keep.append(batch)  # untouched until poll_upto(ticket) returned
        t = eng.submit_async_ptr(batch.ctypes.data, n)
        return eng.poll_upto(t)
    # a device batch at a padded stride and an offset base: rows `stride` samples apart, from 4 samples into the allocation
    per_bytes = batch.nbytes // (len(blk) * n)
    stride, lead = n + 4 * (1 + len(keep) % 3), 4
    dev = torch.zeros((lead + len(blk) * stride) * per_bytes, dtype=torch.uint8, device="cuda")
    rows = torch.from_numpy(batch.view(np.uint8).reshape(len(blk), -1)).cuda()
    view = dev[lead * per_bytes:].view(-1)[:len(blk) * stride * per_bytes].view(len(blk), stride * per_bytes)
    view[:, :n * per_bytes] = rows
    torch.cuda.synchronize()
    keep.append(dev)
    eng.submit_device(dev.data_ptr() + lead * per_bytes, stride, n, rows=len(blk))
    return eng.poll()


def strip(m, letters):
    """frame_key with the channel as its position in the stream's letters, so that a C/D stream compares with the reference's A/B"""
    return (m.nbits, m.payload, m.start_idx, m.end_idx, int(np.float32(m.level).view(np.uint32)),
            int(np.float32(m.ppm).view(np.uint32)), letters.index(m.channel))


def run(model, mode, fmt, fs, offsets, T, n, schedule, how=("host",), dsk=False, members=(), max_chunk=None, letters=None, raws=None):
    """A fan engine (and members attached to it) against one reference per stream and unit on each stream's restated input.
    letters: per-stream receiver letters (a receiver table).  Returns (raws, frames per unit and stream, reference frame count)."""
    need_ref(mode)
    B = len(offsets)
    raws = raws if raws is not None else inputs(fmt, fs, n, offsets, T, mode)
    lengths = lengths_of(n, schedule)
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=max_chunk or max(lengths), taps=True, dsk=dsk,
                        channel_mode=mode, channels="XX" if mode == MX else "AB")
    if letters:
        eng.set_receivers([dict(channels=c) for c in letters])
    eng.set_tuning(offsets, per_input=T)
    assert eng.inputs == B // T == len(raws)
    units = [(eng, model, [reference(model, fs, mode, dsk) for _ in range(B)])]
    for m in members:
        units.append((eng.attach(model=m), m, [reference(m, fs, mode, dsk) for _ in range(B)]))
    taps = not resampled(fs, mode, dsk)
    chans = (0,) if mode == MX else (0, 1)
    per = PER[fmt]
    problems, keep, pos = [], [], 0
    got = [[[] for _ in range(B)] for _ in units]
    want = [[[] for _ in range(B)] for _ in units]
    for c, k in enumerate(lengths):
        blk = [r[pos * per:(pos + k) * per] for r in raws]
        for q in submit(eng, blk, k, how[c % len(how)], keep):
            got[0][q.stream].append(q)
        eng.sync()
        for u, (e, m, refs) in enumerate(units):
            for s in range(B):
                refs[s].push(aisgpu.tune_restate(fmt, fs, offsets[s], pos, blk[s // T]))
                if taps:
                    problems += U.compare_taps(e, s, refs[s], m, "submit %d" % c, chans)
            for s in range(B):
                want[u][s] += refs[s].messages()
            if u:
                for q in e.poll():
                    got[u][q.stream].append(q)
        pos += k
    for u in range(len(units)):
        for s in range(B):
            lt = letters[s] if letters else ("XX" if mode == MX else "AB")
            g, w = [strip(q, lt) for q in got[u][s]], [strip(q, "XX" if mode == MX else "AB") for q in want[u][s]]
            if g != w:
                problems.append(("unit %d" % u, "stream %d" % s, len(g), len(w)))
            if not letters:
                problems += [("unit %d" % u,) + p for p in U.compare_frames([got[u][s]], [want[u][s]])]
    for e, _, _ in units[:0:-1]:
        e.close()
    eng.close()
    assert not problems, "parity problems (first 10): %r" % (problems[:10],)
    return raws, got, sum(len(w) for wu in want for w in wu)


def test_four_channels_one_engine(built):
    """Three 12.288 MS/s recordings, each with the A/B pair at +2.6 MHz and the C/D pair at -2.6 MHz: one engine, T = 2, receivers
    AB on the even streams and CD on the odd ones.  Each stream is the reference on its restated input, and the frames are those of
    the two-engine arrangement (an AB engine tuned to +2.6 MHz, a CD engine tuned to -2.6 MHz) on the same recordings."""
    fs, N, n = 12288000, 262144, 12288000 // 4
    offsets, letters = [WIDE, -WIDE] * 3, ["AB", "CD"] * 3
    raws, got, nframes = run(M2, AB, CS16, fs, offsets, 2, n, [N], letters=letters)
    assert nframes > 0
    for r in range(3):
        assert not np.array_equal(raws[r], raws[(r + 1) % 3])
    pair = {}
    for f, lt in ((WIDE, "AB"), (-WIDE, "CD")):
        e = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CS16, n_streams=3, max_chunk=N)
        e.set_receivers([dict(channels=lt)] * 3)
        e.set_tuning([f] * 3)
        frames = [[] for _ in range(3)]
        for c in range(n // N):
            e.submit(np.ascontiguousarray(np.stack([x[c * N * 2:(c + 1) * N * 2] for x in raws])), N)
            for q in e.poll():
                frames[q.stream].append(q)
        e.close()
        pair[lt] = frames
    for s in range(6):
        want = pair[letters[s]][s // 2]
        assert [U.frame_key(q) for q in got[0][s]] == [U.frame_key(q) for q in want], "stream %d" % s
        assert len(want) > 0, "stream %d" % s
    channels = {q.channel for s in range(1, 6, 2) for q in got[0][s]}
    assert channels == {"C", "D"}
    assert {q.channel for s in range(0, 6, 2) for q in got[0][s]} <= {"A", "B"}


@pytest.mark.parametrize("model,fmt,T,offsets", [
    (M2, CF32, 2, [0, 301234, -517001, 742500]),
    (M0, CU8, 3, [250000, -400000, 0, 123457, -700001, 555555]),
    (M4, CS8, 2, [-333333, 333333, 600000, -10]),
    (M11, CS16, 3, [0, 450000, -450000, 77777, -222222, 666666]),
    (M2, FS4, 2, [180000, -300000, 0, 512345]),
    (M0, DC16H, 3, [-600000, 0, 600000, 1, -1, 300001]),
], ids=["M2-CF32-T2", "M0-CU8-T3", "M4-CS8-T2", "M11-CS16-T3", "M2-FS4-T2", "M0-DC16H-T3"])
def test_every_format_at_a_bucket_rate(built, model, fmt, T, offsets):
    _, _, nframes = run(model, AB, fmt, 1536000, offsets, T, 1536000 * 3 // 10, [65536])
    assert nframes > 0


@pytest.mark.parametrize("fs,fmt", [(96000, CU8), (192000, CS16)])
def test_single_channel_mode_two_channels_per_input(built, fs, fmt):
    """X mode: each capture centred between two channels 50 kHz apart, one stream per channel"""
    _, _, nframes = run(M2, MX, fmt, fs, [25000, -25000] * 2, 2, fs * 4 // 10, [4096])
    assert nframes > 0


@pytest.mark.parametrize("model,fmt,fs,dsk", [
    (M2, CF32, 1000000, False),   # Upsample behind two CIC stages: the tune feeds the CIC stage
    (M2, CU8, 288000, False),     # a DownsampleKFilter bucket: the tune feeds it directly
    (M11, DC16H, 2304000, True),  # a DSK bucket behind three CIC stages (-go DSK on)
    (M0, CS16, 250000, False),    # Upsample behind no CIC stage: the tune writes the resampler's input (D0)
], ids=["resampled", "dsk-bucket", "dsk-cic", "into-d0"])
def test_prestage_paths(built, model, fmt, fs, dsk):
    h = fs // 2
    offsets = [-(h // 2), h - 30000, 0, 7777]
    n = fs * 3 // 10
    _, _, nframes = run(model, AB, fmt, fs, offsets, 2, n // 16384 * 16384, [32768], dsk=dsk)
    assert nframes > 0


def test_every_host_and_device_entry_point(built):
    run(M0, AB, CF32, 1536000, [0, 123457, -700001, 400000], 2, 1536000 * 3 // 10, [16384, 65536, 4096, 98304, 32768, 8192],
        how=("host", "device", "v", "async", "device", "host"), max_chunk=98304)
    run(M2, MX, DC16H, 96000, [-31000, 0, 40000, 31000, -20000, 9000], 3, 96000 * 4 // 10, [1024, 4096, 64, 2048],
        how=("device", "async", "v", "host"), max_chunk=4096)


@pytest.mark.parametrize("feeder", ["feed_files", "feed_wav_files"])
def test_feeders_read_one_file_per_input(built, tmp_path, feeder):
    need_ref(AB)
    fs, N, T, fmt = 1536000, 32768, 2, CS16
    offsets = [210000, 0, -640000, 350000, 500000, -123456]
    R = len(offsets) // T
    lengths = [N * 9, N * 5 + 777, N * 7 - 3]
    paths, raws = [], []
    for r in range(R):
        raw = to_raw(fan_input(fs, lengths[r], offsets[r * T:(r + 1) * T], 70 + r, AB), fmt)
        p = tmp_path / ("rec%d.%s" % (r, "wav" if feeder == "feed_wav_files" else "raw"))
        if feeder == "feed_wav_files":
            W.write_wav(str(p), raw.tobytes(), fmt, fs)
        else:
            raw.tofile(p)
        paths.append(str(p))
        raws.append(raw)
    eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=fmt, n_streams=len(offsets), max_chunk=N)
    eng.set_tuning(offsets, per_input=T)
    with pytest.raises(ValueError):
        getattr(eng, feeder)(paths + paths, N)  # one path per stream: refused before anything is read
    got, nblocks = getattr(eng, feeder)(paths, N)
    eng.close()
    assert nblocks == 9
    total = 0
    for s, f in enumerate(offsets):
        padded = np.zeros(nblocks * N * 2, np.int16)  # the feeders zero-fill the tail of a file's last block
        padded[:len(raws[s // T])] = raws[s // T]
        ref = reference(M2, fs, AB)
        for c in range(nblocks):
            ref.push(aisgpu.tune_restate(fmt, fs, f, c * N, padded[c * N * 2:(c + 1) * N * 2]))
        want = ref.messages()
        assert [U.frame_key(q) for q in got if q.stream == s] == [U.frame_key(q) for q in want], "stream %d" % s
        total += len(want)
    assert total > 0


def test_group_leader_fans_its_members(built):
    run(M2, AB, CU8, 1536000, [0, 400000, -350000, 150000], 2, 1536000 * 3 // 10, [65536], members=(M0, M11))


def test_channel_dump(built, tmp_path):
    """Stream s's two dump files equal those of a plain CF32 engine fed stream s's restated input"""
    fs, N, nsub, T, fmt = 1536000, 65536, 5, 2, CU8
    offsets = [300000, -300000, 0, 555555]
    B, R = len(offsets), len(offsets) // T
    raws = inputs(fmt, fs, N * nsub, offsets, T, AB, seed=90)
    fan = aisgpu.Engine(model=M2, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N)
    fan.set_tuning(offsets, per_input=T)
    fan.dump_open([str(tmp_path / ("fan%d" % s)) for s in range(B)])
    plain = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CF32, n_streams=B, max_chunk=N)
    plain.dump_open([str(tmp_path / ("plain%d" % s)) for s in range(B)])
    a, b = [], []
    for c in range(nsub):
        blk = [r[c * N * 2:(c + 1) * N * 2] for r in raws]
        fan.submit(np.ascontiguousarray(np.stack(blk)), N)
        plain.submit(np.stack([aisgpu.tune_restate(fmt, fs, offsets[s], c * N, blk[s // T]) for s in range(B)]), N)
        a += fan.poll()
        b += plain.poll()
    fan.dump_close()
    plain.dump_close()
    fan.close()
    plain.close()
    assert R == 2 and len(b) > 0
    assert [U.frame_key(q) for q in a] == [U.frame_key(q) for q in b]
    for s in range(B):
        for ch in "AB":
            x = (tmp_path / ("fan%d_%s.wav" % (s, ch))).read_bytes()
            y = (tmp_path / ("plain%d_%s.wav" % (s, ch))).read_bytes()
            assert len(y) > 44 and x == y, (s, ch)


OUTPUT = dict(version=81, status=0, rxtime_us=0, toa_us=0, include_ssl=False, uuid=None, suffix=None)


def test_records_and_stamps_per_stream(built):
    """A receiver table and a recording clock on a fan engine: every NMEA_TAG record is aisgpu_msg_format of its frame with its
    stream's tag and stamp, and the streams of one input with equal starts have equal stamps."""
    fs, T, fmt = 1536000, 2, CU8
    lens = [65536, 32768 + 64 * 3, 65536 + 64 * 11, 49152]
    offsets = [WIDE // 8, -WIDE // 8] * 3
    B = len(offsets)
    raws = inputs(fmt, fs, sum(lens), offsets, T, AB, seed=120)
    rx = [dict(channels="AB" if s % 2 == 0 else "CD", station=500 + s, tag_mode=3, driver=s, hardware="site-%d" % (s // T),
               ipv4=0x0A000001 + s) for s in range(B)]
    starts = [1700000000000000 + (s // T) * 3600000000 for s in range(B)]  # both tunings of one input share its start
    e = aisgpu.Engine(model=M2, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=max(lens), max_frames=1 << 14)
    e.set_receivers(rx)
    e.set_clock(starts)
    e.set_tuning(offsets, per_input=T)
    e.lines_enable(aisgpu.MSGFORMAT_NMEA_TAG, aisgpu.make_tag(**OUTPUT), 1 << 24)
    frames, text, nrec, a = [], [], 0, 0
    for c, n in enumerate(lens):
        e.submit(np.ascontiguousarray(np.stack([r[a * 2:(a + n) * 2] for r in raws])), n)
        a += n
        frames += e.poll_upto(c)
        b, k = e.poll_lines(c)
        text.append(b)
        nrec += k
    stamp = lambda s, c: starts[s] + sum(lens[:c + 1]) * 10 ** 6 // fs
    stamps = [[e.stamp(s, c) for c in range(len(lens))] for s in range(B)]
    e.close()
    assert stamps == [[stamp(s, c) for c in range(len(lens))] for s in range(B)]
    for s in range(0, B, T):
        assert stamps[s] == stamps[s + 1]
    assert nrec == len(frames) > 0
    assert {m.channel for m in frames if m.stream % 2} <= {"C", "D"} and {m.stream for m in frames} == set(range(B))
    st = aisgpu.FormatState(0, 0)
    want = [aisgpu.msg_format(m, aisgpu.make_tag(**dict(OUTPUT, station=rx[m.stream]["station"], driver=rx[m.stream]["driver"],
                                                       hardware=rx[m.stream]["hardware"], mode=3, ipv4=rx[m.stream]["ipv4"],
                                                       rxtime_us=stamp(m.stream, m.chunk))), aisgpu.MSGFORMAT_NMEA_TAG, st)
            for m in frames]
    assert b"".join(text) == b"".join(want)


def test_one_tuning_per_input_is_set_tuning(built):
    fs, N, nsub = 1536000, 65536, 5
    offsets = [0, 222222, -444444]
    raws = inputs(CU8, fs, N * nsub, offsets, 1, AB, seed=150)
    out = []
    for per_input in (None, 1):
        e = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=3, max_chunk=N)
        if per_input is None:
            e._chk(e.lib.aisgpu_set_tuning(e.h, aisgpu._offsets(offsets), 3))
        else:
            e.set_tuning(offsets, per_input=per_input)
        frames = []
        for c in range(nsub):
            e.submit(np.ascontiguousarray(np.stack([r[c * N * 2:(c + 1) * N * 2] for r in raws])), N)
            frames += e.poll()
        e.close()
        out.append([(q.stream,) + U.frame_key(q) for q in frames])
    assert out[0] == out[1] and len(out[0]) > 0


def test_refused_calls_leave_the_handle_untouched(built):
    need_ref(AB)
    fs, N, nsub = 1536000, 65536, 4
    offsets = [0, 333333, -250000, 100000]
    raws = inputs(CU8, fs, N * nsub, offsets, 2, AB, seed=160)
    flat = [r for r in raws for _ in range(2)]  # the same recordings, one copy per stream, for the untuned comparisons

    def frames_of(e, rows):
        out = []
        for c in range(nsub):
            e.submit(np.ascontiguousarray(np.stack([r[c * N * 2:(c + 1) * N * 2] for r in rows])), N)
            out += [(q.stream,) + U.frame_key(q) for q in e.poll()]
        return out

    plain = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=4, max_chunk=N)
    want = frames_of(plain, flat)
    plain.close()
    assert len(want) > 0
    # every refusal on a fresh engine, then it runs as an untouched one (one row per stream)
    e = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=4, max_chunk=N)
    member = e.attach(model=M0)
    for bad, per_input, text in (([0] * 4, 3, "per_input 3 must be at least 1 and divide n_streams 4"),
                                 ([0] * 4, 0, "per_input 0 must be at least 1"), ([0] * 3, 2, "3 offsets for 4 streams"),
                                 ([0, 0, 768000, 0], 2, "stream 2: offset 768000 Hz")):
        with pytest.raises(aisgpu.AisGpuError, match=text):
            e.set_tuning(bad, per_input=per_input)
        assert e.inputs == 4
    with pytest.raises(aisgpu.AisGpuError, match="member of a group"):
        member.set_tuning(offsets, per_input=2)
    member.close()
    assert frames_of(e, flat) == want
    with pytest.raises(aisgpu.AisGpuError, match="submitted to"):
        e.set_tuning(offsets, per_input=2)
    e.close()
    # a fan engine refuses a second table, and Python refuses n_streams rows before anything is submitted
    e = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=4, max_chunk=N)
    e.set_tuning(offsets, per_input=2)
    with pytest.raises(aisgpu.AisGpuError, match="already installed"):
        e.set_tuning(offsets, per_input=2)
    blk4 = np.ascontiguousarray(np.stack([r[:N * 2] for r in flat]))
    with pytest.raises(ValueError):
        e.submit(blk4, N)
    with pytest.raises(ValueError):
        e.submit_v(list(blk4), N)
    with pytest.raises(ValueError):
        e.submit_device(0, N, N, rows=4)
    with pytest.raises(ValueError):
        e.submit(blk4[:1], N)
    assert e.counters()[3] == 0
    refs = [reference(M2, fs, AB) for _ in offsets]
    got = frames_of(e, raws)
    e.close()
    for c in range(nsub):
        for s in range(4):
            refs[s].push(aisgpu.tune_restate(CU8, fs, offsets[s], c * N, raws[s // 2][c * N * 2:(c + 1) * N * 2]))
    want = [(s,) + U.frame_key(q) for s in range(4) for q in refs[s].messages()]
    assert sorted(got) == sorted(want) and len(want) > 0
