"""The per-stream digital tune on the GPU (aisgpu_set_tuning), bit for bit (tolerance 0) against the compiled reference (oracle/_ref).

Every stream carries AIS traffic (tests/afc_signals.py) placed at its own offset from the capture's centre.  A tuned engine's stream
must yield exactly what the reference yields on aisgpu_tune_restate of that stream's input as CF32, fed in the same blocks: the frames
(payload, NMEA, channel, start / end counters, level and ppm bit patterns) and, at rates without a resampler, every tap of each
submit (C, and the back-end taps of the model).  Streams with offset 0 must equal a plain engine on the raw input."""
import numpy as np
import pytest

import afc_signals as A
import aisgpu
import dc16h_util as DC
import fs4_util as F4
import oracle as O
import oracle_x as OX
import parity_util as U

pytestmark = pytest.mark.gpu

AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS8, CS16, FS4, DC16H = (aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16, aisgpu.FMT_F32_FS4,
                                    aisgpu.FMT_DC16H)
M0, M1, M2, M4, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2
PER = {CF32: 1, CU8: 2, CS8: 2, CS16: 2, FS4: 1, DC16H: 3}  # raw array elements per sample


def need_ref(mode):
    if not (OX.have_refx() if mode == MX else O.have_ref()):
        pytest.skip("the tune is checked against the compiled reference only")


def placed(fs, n, f, seed, mode):
    """Traffic centred on f Hz: the pair at f -+ 25 kHz (AB), or one channel at f (X), with small carrier errors of its own."""
    x = A.row(fs, n, float((seed * 37) % 600 - 300), seed, kind=A.X_ if mode == MX else A.AB).astype(np.complex128)
    return (x * np.exp(2j * np.pi * f * np.arange(n, dtype=np.float64) / fs)).astype(np.complex64)


def to_raw(x, fmt, seed=0):
    if fmt == FS4:
        return F4.real_stream(x)
    if fmt == DC16H:
        return DC.from_complex(x, seed)[0]
    return A.to_raw(x, fmt)[0]


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
    import torch
    batch = np.ascontiguousarray(np.stack(blk))
    if how == "host":
        eng.submit(batch, n)
        return
    # a device batch at a padded stride and an offset base: rows `stride` samples apart, from 4 samples into the allocation
    per_bytes = batch.nbytes // (len(blk) * n)
    stride, lead = n + 4 * (1 + len(keep) % 3), 4
    dev = torch.zeros((lead + len(blk) * stride) * per_bytes, dtype=torch.uint8, device="cuda")
    rows = torch.from_numpy(batch.view(np.uint8).reshape(len(blk), -1)).cuda()
    view = dev[lead * per_bytes:].view(-1)[:len(blk) * stride * per_bytes].view(len(blk), stride * per_bytes)
    view[:, :n * per_bytes] = rows
    torch.cuda.synchronize()
    keep.append(dev)
    eng.submit_device(dev.data_ptr() + lead * per_bytes, stride, n)


def run(model, mode, fmt, fs, offsets, n, schedule, how=("host",), dsk=False, members=(), max_chunk=None):
    """A tuned engine (and members attached to it) against one reference per stream and unit on the restated input."""
    need_ref(mode)
    B = len(offsets)
    xs = [placed(fs, n, f, 40 + s, mode) for s, f in enumerate(offsets)]
    raws = [to_raw(x, fmt, s) for s, x in enumerate(xs)]
    lengths = lengths_of(n, schedule)
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=max_chunk or max(lengths), taps=True, dsk=dsk,
                        channel_mode=mode, channels="XX" if mode == MX else "AB")
    eng.set_tuning(offsets)
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
        submit(eng, blk, k, how[c % len(how)], keep)
        eng.sync()
        for u, (e, m, refs) in enumerate(units):
            for s in range(B):
                refs[s].push(aisgpu.tune_restate(fmt, fs, offsets[s], pos, blk[s]))
                if taps:
                    problems += U.compare_taps(e, s, refs[s], m, "submit %d" % c, chans)
            for s in range(B):
                want[u][s] += refs[s].messages()
            for q in e.poll():
                got[u][q.stream].append(q)
        pos += k
    for u in range(len(units)):
        problems += [("unit %d" % u,) + p for p in U.compare_frames(got[u], want[u])]
    for e, _, _ in units[:0:-1]:
        e.close()
    eng.close()
    assert not problems, "parity problems (first 10): %r" % (problems[:10],)
    return raws, got, sum(len(w) for wu in want for w in wu)


@pytest.mark.parametrize("model,fmt", [(M2, CF32), (M0, CU8), (M1, CS16), (M4, DC16H), (M11, FS4), (M2, CS8)])
def test_ab_bucket_rate(built, model, fmt):
    offsets = [0, 301234, -517001, 742500]
    _, _, nframes = run(model, AB, fmt, 1536000, offsets, 1536000 * 3 // 10, [65536])
    assert nframes > 0


@pytest.mark.parametrize("model,fmt,fs", [(M2, CF32, 96000), (M0, CU8, 48000), (M11, CS16, 192000), (M4, DC16H, 96000),
                                          (M2, FS4, 192000)])
def test_x_bucket_rate(built, model, fmt, fs):
    h = fs // 2
    offsets = [0, h // 3, -(h - 13000), 1]
    _, _, nframes = run(model, MX, fmt, fs, offsets, fs * 4 // 10, [4096])
    assert nframes > 0


@pytest.mark.parametrize("mode,model,fmt,fs,dsk", [
    (AB, M2, CF32, 1000000, False),   # Upsample behind two CIC stages: the tune feeds the CIC stage
    (AB, M0, CS16, 250000, False),    # Upsample behind no CIC stage, then DownsampleKFilter: the tune writes the resampler's input
    (AB, M2, CU8, 288000, False),     # a DownsampleKFilter bucket: the tune feeds it directly
    (AB, M11, DC16H, 2304000, True),  # a DSK bucket behind three CIC stages (-go DSK on)
    (MX, M2, CU8, 60000, False),      # single-channel mode, Upsample straight behind the tune
])
def test_resampled_and_dsk_rates(built, mode, model, fmt, fs, dsk):
    h = fs // 2
    offsets = [0, -(h // 2), h - 30000, 7777] if mode == AB else [0, -(h // 2), h - 10000, 7777]
    n = fs * 3 // 10
    q = 4096 if mode == MX else 16384
    _, _, nframes = run(model, mode, fmt, fs, offsets, n // q * q, [q * 2], dsk=dsk)
    assert nframes > 0


def test_wideband_offsets_of_several_mhz(built):
    run(M2, AB, CS16, 12288000, [3000000, -4500125, 0, 6100000], 12288000 // 4, [262144])


def test_zero_offset_streams_equal_a_plain_engine(built):
    fs, N = 1536000, 65536
    offsets = [0, 250000, 0, -600000, 0]
    raws, got, _ = run(M2, AB, CU8, fs, offsets, N * 6, [N])
    plain = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=len(raws), max_chunk=N)
    want = [[] for _ in raws]
    for c in range(6):
        plain.submit(np.ascontiguousarray(np.stack([r[c * N * 2:(c + 1) * N * 2] for r in raws])), N)
        for q in plain.poll():
            want[q.stream].append(q)
    plain.close()
    for s, f in enumerate(offsets):
        if f == 0:
            assert [U.frame_key(q) for q in got[0][s]] == [U.frame_key(q) for q in want[s]], "stream %d" % s
            assert len(want[s]) > 0


def test_changing_submit_lengths_and_device_batches(built):
    run(M0, AB, CF32, 1536000, [0, 123457, -700001], 1536000 * 3 // 10, [16384, 65536, 4096, 98304, 32768],
        how=("host", "device", "device", "host"), max_chunk=98304)
    run(M2, MX, DC16H, 96000, [-31000, 0, 40000], 96000 * 4 // 10, [1024, 4096, 64, 2048], how=("device", "host"), max_chunk=4096)


def test_group_leader_tunes_its_members(built):
    run(M2, AB, CU8, 1536000, [0, 400000, -350000], 1536000 * 3 // 10, [65536], members=(M0, M11))


def test_feed_files_on_a_tuned_engine(built, tmp_path):
    need_ref(AB)
    fs, N = 1536000, 32768
    offsets = [210000, 0, -640000]
    lengths = [N * 9, N * 5 + 777, N * 7 - 3]
    paths, raws = [], []
    for s, f in enumerate(offsets):
        raw = to_raw(placed(fs, lengths[s], f, 70 + s, AB), CU8)
        p = tmp_path / ("rec%d.raw" % s)
        raw.tofile(p)
        paths.append(str(p))
        raws.append(raw)
    eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=3, max_chunk=N)
    eng.set_tuning(offsets)
    got, nblocks = eng.feed_files(paths, N)
    eng.close()
    assert nblocks == 9
    total = 0
    for s, f in enumerate(offsets):
        padded = np.zeros(nblocks * N * 2, np.uint8)  # RAWFile zero-fills the tail of its last block
        padded[:len(raws[s])] = raws[s]
        ref = reference(M2, fs, AB)
        for c in range(nblocks):
            ref.push(aisgpu.tune_restate(CU8, fs, f, c * N, padded[c * N * 2:(c + 1) * N * 2]))
        want = ref.messages()
        assert [U.frame_key(q) for q in got if q.stream == s] == [U.frame_key(q) for q in want], "stream %d" % s
        total += len(want)
    assert total > 0


def test_four_channels_from_one_recording(built):
    """A 12.288 MS/s capture centred at 159.4 MHz: the A/B pair (162.000 MHz) 2.6 MHz above it, the C/D pair (156.800 MHz) 2.6 MHz
    below.  An AB engine tuned to +2.6 MHz and a CD engine (receiver letters C / D) tuned to -2.6 MHz give the reference's frames
    on the two restated signals; the CD engine's carry the letters C / D, and equal an untuned CD engine on the restated signal."""
    need_ref(AB)
    fs, N, n = 12288000, 262144, 12288000 // 4
    x = (placed(fs, n, 2600000, 90, AB).astype(np.complex128) + placed(fs, n, -2600000, 91, AB)).astype(np.complex64) * 0.5
    raw = to_raw(x, CS16)
    frames = {}
    for name, f, letters in (("AB", 2600000, "AB"), ("CD", -2600000, "CD")):
        eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CS16, n_streams=1, max_chunk=N)
        eng.set_receivers([dict(channels=letters)])
        eng.set_tuning([f])
        plain = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CF32, n_streams=1, max_chunk=N, channels=letters)
        ref = reference(M2, fs, AB)
        got, plain_got = [], []
        for c in range(n // N):
            blk = raw[c * N * 2:(c + 1) * N * 2]
            eng.submit(blk[None, :], N)
            restated = aisgpu.tune_restate(CS16, fs, f, c * N, blk)
            plain.submit(restated[None, :], N)
            ref.push(restated)
            got += eng.poll()
            plain_got += plain.poll()
        eng.close()
        plain.close()
        want = ref.messages()
        assert len(want) > 0
        assert [U.frame_key(q) for q in got] == [U.frame_key(q) for q in plain_got], name
        strip = lambda q: (q.nbits, q.payload, q.start_idx, q.end_idx, int(np.float32(q.level).view(np.uint32)),
                           int(np.float32(q.ppm).view(np.uint32)), "AB".index(q.channel) if name == "AB" else "CD".index(q.channel))
        strip_ref = lambda q: (q.nbits, q.payload, q.start_idx, q.end_idx, int(np.float32(q.level).view(np.uint32)),
                               int(np.float32(q.ppm).view(np.uint32)), "AB".index(q.channel))
        assert [strip(q) for q in got] == [strip_ref(q) for q in want], name
        frames[name] = got
    assert {q.channel for q in frames["AB"]} <= {"A", "B"} and {q.channel for q in frames["CD"]} <= {"C", "D"}
    assert {q.channel for q in frames["CD"]} == {"C", "D"}


def test_refused_calls_leave_the_handle_unchanged(built):
    need_ref(AB)
    fs, N = 1536000, 65536
    offsets = [0, 333333]
    raws = [to_raw(placed(fs, N * 5, f, 60 + s, AB), CU8) for s, f in enumerate(offsets)]
    eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=2, max_chunk=N)
    member = eng.attach(model=M0)
    for bad in ([0], [0, 0, 0], [0, 768000], [-768000, 0]):
        with pytest.raises(aisgpu.AisGpuError):
            eng.set_tuning(bad)
    with pytest.raises(aisgpu.AisGpuError, match="member of a group"):
        member.set_tuning(offsets)
    eng.set_tuning(offsets)
    with pytest.raises(aisgpu.AisGpuError, match="already installed"):
        eng.set_tuning(offsets)
    refs = [reference(M2, fs, AB) for _ in offsets]
    got = [[] for _ in offsets]
    for c in range(5):
        blk = [r[c * N * 2:(c + 1) * N * 2] for r in raws]
        eng.submit(np.ascontiguousarray(np.stack(blk)), N)
        for s in range(2):
            refs[s].push(aisgpu.tune_restate(CU8, fs, offsets[s], c * N, blk[s]))
        for q in eng.poll():
            got[q.stream].append(q)
    assert not U.compare_frames(got, [r.messages() for r in refs])
    assert sum(len(g) for g in got) > 0
    member.close()
    eng.close()
    # an engine whose every call was refused runs as an untuned one
    eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=2, max_chunk=N)
    plain = aisgpu.Engine(model=M2, sample_rate=fs, fmt=CU8, n_streams=2, max_chunk=N)
    with pytest.raises(aisgpu.AisGpuError):
        eng.set_tuning([0, 900000])
    a, b = [], []
    for c in range(5):
        batch = np.ascontiguousarray(np.stack([r[c * N * 2:(c + 1) * N * 2] for r in raws]))
        eng.submit(batch, N)
        plain.submit(batch, N)
        if c == 0:
            with pytest.raises(aisgpu.AisGpuError, match="submitted to"):
                eng.set_tuning([0, 100000])
        a += eng.poll()
        b += plain.poll()
    assert [U.frame_key(q) for q in a] == [U.frame_key(q) for q in b]
    eng.close()
    plain.close()
