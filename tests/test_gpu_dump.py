"""-m gpu: the 48 kHz channel dump (aisgpu_dump_open, -go DUMP) byte for byte against the files the unmodified reference writes
(oracle/_ref/libaisref_dump.so: SetKey(KEY_SETTING_DUMP) before buildModel) from the same blocks.

A  front-end families: streaming CF32 / CU8 / CS8 at 1536K, FP_DS, tiled CS16 at 96K / 192K / 384K, the 288K, 6000K, 240K and
   1152K-DSK pre-stages and 12288K, each at an odd batch with some streams not dumped (they must get no file), models 0, 2 and 11,
   CD letters once and droop off once.
B  submit shapes: a length that changes from call to call, pre-stage submits that complete no block, all four submit entry points
   (aisgpu_submit_device at a padded stride and an offset base), ten asynchronous submits before the first poll.
C  the archive path: aisgpu_feed_files on recordings of different lengths.
D  nothing else changes: frames, order, counters, level/ppm bits and AISGPU_TAP_C with the dump on and off; launch counts against
   torch.profiler; a group leader's dump equals a standalone engine's and its members' frames are unchanged.
E  refusals, file errors, aisgpu_destroy without aisgpu_dump_close, and the ModelGPU adapter against the reference's own model."""
import os
import subprocess

import numpy as np
import pytest
import torch

import aisgpu
import aissynth as S
import mode_x_util as X
import oracle as O
import oracle_dump as OD
import parity_util as U

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not OD.have_refdump(), reason="reference dump harness not built")]

CF32, CU8, CS8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16
M0, M2, M3, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR, aisgpu.MODEL_V2
BPS = {CF32: 8, CU8: 2, CS8: 2, CS16: 4}
B = 33


class Fam:
    def __init__(self, name, model, fs, fmt=CF32, dsk=False, fp_ds=False, droop=True, channels="AB", fixed=False):
        self.name, self.model, self.fs, self.fmt, self.dsk, self.fp_ds = name, model, fs, fmt, dsk, fp_ds
        self.droop, self.channels, self.fixed = droop, channels, fixed  # fixed: an Upsample rate (one submit length)

    def __repr__(self):
        return self.name

    def kw(self, **extra):
        return dict(dict(model=self.model, sample_rate=self.fs, fmt=self.fmt, dsk=self.dsk, fp_ds=self.fp_ds, droop=self.droop,
                         channels=self.channels), **extra)

    def flags(self):
        return (O.FLAG_PS_EMA | O.FLAG_AFC_WIDE | (O.FLAG_DROOP if self.droop else 0) | (O.FLAG_DSK if self.dsk else 0) |
                (O.FLAG_FP_DS if self.fp_ds else 0))

    def granule(self):
        return aisgpu.chunk_granule(self.fs, self.model, self.dsk, self.fp_ds, self.fmt)


def stimulus(fam, total, seed=0):
    """Per stream: (raw array, elements per sample)."""
    out = []
    for s in range(B):
        x, _ = S.random_stream(fam.fs, total, 100 * seed + s)
        out.append(X.to_raw(x, fam.fmt))
    return out


def block(raws, s, pos, n):
    raw, per = raws[s]
    return np.ascontiguousarray(raw[pos * per:(pos + n) * per])


def submit(eng, fam, raws, pos, n, entry, keep):
    """One submit of samples [pos, pos + n) of every stream through one of the four entry points."""
    rows = [block(raws, s, pos, n) for s in range(B)]
    if entry == "v":
        eng.submit_v(rows, n)
    elif entry == "async":
        batch = np.ascontiguousarray(np.stack(rows))
        keep.append(batch)
        return eng.submit_async_ptr(batch.ctypes.data, n)
    elif entry == "device":  # a padded stride and a base 8 samples into the allocation (16-byte rows for every format)
        per = raws[0][1]
        stride, off = n + 16, 8
        flat = np.zeros((B * stride + off) * per, dtype=rows[0].dtype)
        for s in range(B):
            flat[(off + s * stride) * per:(off + s * stride + n) * per] = rows[s]
        t = torch.from_numpy(flat.view(np.uint8)).cuda()
        keep.append(t)
        eng.submit_device(t.data_ptr() + off * BPS[fam.fmt], stride, n)
    else:
        eng.submit(np.ascontiguousarray(np.stack(rows)), n)
    return None


def prefixes(d, tag, dumped):
    return [str(d / ("%s%d" % (tag, s))) if s in dumped else None for s in range(B)]


def reference_files(d, fam, raws, schedule, dumped, tag="ref"):
    """The reference's files of every dumped stream, fed the blocks of `schedule` (the engine's submit lengths)."""
    for s in dumped:
        ref = OD.RefModelDump(str(d / ("%s%d" % (tag, s))), model=fam.model, sample_rate=fam.fs, fmt=fam.fmt, flags=fam.flags(),
                              channels=fam.channels)
        pos = 0
        for n in schedule:
            ref.push(block(raws, s, pos, n))
            pos += n
        ref.close()


def assert_same_files(d, dumped, got="gpu", want="ref"):
    for s in range(B):
        for ch in "AB":
            g, w = d / ("%s%d_%s.wav" % (got, s, ch)), d / ("%s%d_%s.wav" % (want, s, ch))
            if s not in dumped:
                assert not g.exists(), "stream %d is not dumped but has %s" % (s, g.name)
                continue
            assert g.exists() == w.exists(), "stream %d %s: engine file %s, reference file %s" % (s, ch, g.exists(), w.exists())
            if not w.exists():
                continue
            gb, wb = g.read_bytes(), w.read_bytes()
            if gb != wb:
                n = min(len(gb), len(wb))
                diff = next((i for i in range(n) if gb[i] != wb[i]), n)
                raise AssertionError("stream %d %s: %d bytes, reference %d, first difference at byte %d" % (s, ch, len(gb), len(wb), diff))


def run_engine(d, fam, raws, schedule, entries, dumped, tag="gpu", dump=True, poll_every=1, **kw):
    eng = aisgpu.Engine(n_streams=B, max_chunk=max(schedule), **fam.kw(**kw))
    if dump:
        eng.dump_open(prefixes(d, tag, dumped))
    keep, frames, pos = [], [], 0
    for i, n in enumerate(schedule):
        submit(eng, fam, raws, pos, n, entries[i % len(entries)], keep)
        pos += n
        if (i + 1) % poll_every == 0:
            frames += eng.poll()
    frames += eng.poll()
    counters = eng.counters()
    if dump:
        eng.dump_close()
    eng.close()
    return frames, counters


DUMPED = [s for s in range(B) if s % 4 != 1]  # streams 1, 5, 9, ... get no file

FAMILIES = [
    Fam("cf32_1536k_m2", M2, 1536000),
    Fam("cu8_1536k_m0", M0, 1536000, CU8),
    Fam("cs8_1536k_m11", M11, 1536000, CS8),
    Fam("cu8_1536k_fpds", M2, 1536000, CU8, fp_ds=True),
    Fam("cs16_96k_m2_cd", M2, 96000, CS16, channels="CD"),
    Fam("cs16_192k_m0", M0, 192000, CS16),
    Fam("cs16_384k_m2_nodroop", M2, 384000, CS16, droop=False),
    Fam("dsk_288k_m2", M2, 288000),
    Fam("us_6000k_m0", M0, 6000000, fixed=True),
    Fam("us_dsk_240k_m2", M2, 240000, fixed=True),
    Fam("dsk_1152k_m2", M2, 1152000, dsk=True),
    Fam("cf32_12288k_m2", M2, 12288000),
]


def schedule_for(fam, seconds=0.1):
    g = fam.granule()
    base = max(g, int(seconds * fam.fs / 4) // g * g)
    if fam.fixed:
        return [base] * 4
    return [base, base // 2 // g * g or g, base + 3 * g, g * max(1, 64 // g), base]  # changes from call to call, one short submit


@pytest.mark.parametrize("fam", FAMILIES, ids=[f.name for f in FAMILIES])
def test_family(built, tmp_path, fam):
    sched = schedule_for(fam, 0.03 if fam.fs > 6144000 else (0.3 if fam.fixed else 0.1))
    raws = stimulus(fam, sum(sched), 1)
    run_engine(tmp_path, fam, raws, sched, ["sync"], DUMPED)
    reference_files(tmp_path, fam, raws, sched, DUMPED)
    assert (tmp_path / "ref0_A.wav").stat().st_size > 44  # the run yields 48 kHz samples
    assert_same_files(tmp_path, DUMPED)


def test_all_entry_points(built, tmp_path):
    fam = Fam("cf32_1536k_m2", M2, 1536000)
    sched = [16384, 8192, 24576, 4096, 16384, 8192, 65536, 64]
    raws = stimulus(fam, sum(sched), 2)
    run_engine(tmp_path, fam, raws, sched, ["sync", "v", "async", "device"], DUMPED, poll_every=3)
    reference_files(tmp_path, fam, raws, sched, DUMPED)
    assert_same_files(tmp_path, DUMPED)


def test_prestage_submits_without_a_block(built, tmp_path):
    # 288K: DownsampleKFilter fills 8192-sample blocks at 96K; 240K: Upsample -> DownsampleKFilter with a short fixed length
    for fam, sched in ((Fam("dsk_288k_m0", M0, 288000), [192, 576, 64, 24576, 1920, 30720, 64]),
                       (Fam("us_dsk_240k_m11", M11, 240000, fixed=True), [2048] * 14)):
        d = tmp_path / fam.name
        d.mkdir()
        raws = stimulus(fam, sum(sched), 3)
        run_engine(d, fam, raws, sched, ["sync", "async", "device"], DUMPED)
        reference_files(d, fam, raws, sched, DUMPED)
        assert_same_files(d, DUMPED)


def test_ten_async_submits_before_the_first_poll(built, tmp_path):
    # three slots: submits 3..9 reuse slots whose rows are still in flight and have to be written out by the submit that needs them
    fam = Fam("cf32_1536k_m2", M2, 1536000)
    sched = [8192, 16384, 8192, 4096, 8192, 16384, 8192, 8192, 4096, 8192]
    raws = stimulus(fam, sum(sched), 4)
    eng = aisgpu.Engine(n_streams=B, max_chunk=max(sched), **fam.kw())
    eng.dump_open(prefixes(tmp_path, "gpu", DUMPED))
    keep, tickets, pos = [], [], 0
    for n in sched:
        tickets.append(submit(eng, fam, raws, pos, n, "async", keep))
        pos += n
    eng.poll_upto(tickets[4])
    eng.poll()
    eng.dump_close()
    eng.close()
    reference_files(tmp_path, fam, raws, sched, DUMPED)
    assert_same_files(tmp_path, DUMPED)


def test_feed_files_ragged(built, tmp_path):
    fam = Fam("cu8_1536k_m2", M2, 1536000, CU8)
    n = 16384
    lengths = [n * 3 + 640 * (s % 5) - 64 * (s % 3) for s in range(B)]  # ragged: whole and partial blocks, the longest sets the run
    paths, padded = [], []
    nblk = (max(lengths) + n - 1) // n
    for s in range(B):
        x, _ = S.random_stream(fam.fs, lengths[s], 500 + s)
        raw = S.to_cu8(x)
        p = tmp_path / ("in%d.cu8" % s)
        raw.tofile(p)
        paths.append(str(p))
        padded.append((np.concatenate([raw, np.zeros(2 * nblk * n - len(raw), np.uint8)]), 2))  # RAWFile's zero-padded blocks
    eng = aisgpu.Engine(n_streams=B, max_chunk=n, **fam.kw())
    eng.dump_open(prefixes(tmp_path, "gpu", DUMPED))
    _, blocks = eng.feed_files(paths, n)
    eng.dump_close()
    eng.close()
    assert blocks == nblk
    reference_files(tmp_path, fam, padded, [n] * nblk, DUMPED)
    assert_same_files(tmp_path, DUMPED)


def frames_key(frames):
    return [(m.stream, m.chunk) + U.frame_key(m) for m in frames]


@pytest.mark.parametrize("fam", [Fam("cf32_1536k_m2", M2, 1536000), Fam("us_6000k_m0", M0, 6000000, fixed=True)], ids=repr)
def test_dump_changes_nothing_else(built, tmp_path, fam):
    sched = schedule_for(fam, 0.2)
    raws = stimulus(fam, sum(sched), 5)
    # pipelined back end: frames, order, counters
    on = run_engine(tmp_path, fam, raws, sched, ["sync", "async"], DUMPED)
    off = run_engine(tmp_path, fam, raws, sched, ["sync", "async"], DUMPED, dump=False)
    assert frames_key(on[0]) == frames_key(off[0]) and len(on[0]) > 0
    assert list(on[1]) == list(off[1])
    # taps on: AISGPU_TAP_C after every submit
    engs = [aisgpu.Engine(n_streams=B, max_chunk=max(sched), taps=True, **fam.kw()) for _ in range(2)]
    engs[0].dump_open(prefixes(tmp_path, "tap", DUMPED))
    pos = 0
    for n in sched:
        for e in engs:
            submit(e, fam, raws, pos, n, "sync", [])
            e.sync()
        pos += n
        for s in range(0, B, 4):
            for ch in (0, 1):
                a, b = (e.tap(aisgpu.TAP_C, s, ch) for e in engs)
                assert U.bits_equal(a, b)
    assert frames_key(engs[0].poll()) == frames_key(engs[1].poll())
    for e in engs:
        e.close()


# One dumped submit under torch.profiler, in a process of its own: a profiler session leaves CUPTI state behind in the process that
# ran it, and the other profiler tests of the suite (tests/test_gpu_prestage_launches.py) count kernels in this one.
PROFILE_CHILD = r"""
import json, sys
sys.path[:0] = sys.argv[1].split("|")
import numpy as np, torch, aisgpu, aissynth as S
fs, N, d = int(sys.argv[2]), int(sys.argv[3]), sys.argv[4]
nsub, b = 4, 3
x = np.stack([S.random_stream(fs, N * nsub, 40 + s)[0] for s in range(b)])
eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=b, max_chunk=N)
eng.dump_open([d + "/l%d" % s for s in range(b)])
for i in range(nsub - 1):
    eng.submit(np.ascontiguousarray(x[:, i * N:(i + 1) * N]), N)
eng.join()
torch.cuda.synchronize()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    eng.submit(np.ascontiguousarray(x[:, (nsub - 1) * N:]), N)
    eng.join()
    torch.cuda.synchronize()
prof.export_chrome_trace(d + "/trace.json")
kernels = [e["name"] for e in json.load(open(d + "/trace.json"))["traceEvents"] if e.get("cat") == "kernel"]
print(json.dumps(dict(launches=eng.last_launches(), kernels=kernels)))
eng.close()
"""


@pytest.mark.parametrize("fs,N", [(1536000, 65536), (6000000, 65536)], ids=["plain_1536k", "resampled_6000k"])
def test_launch_count_with_dump(built, tmp_path, fs, N):
    import json
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    paths = "|".join([os.path.join(os.path.dirname(here), "ais-catcher_b200"), here])
    p = subprocess.run([sys.executable, "-s", "-c", PROFILE_CHILD, paths, str(fs), str(N), str(tmp_path)], capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-2000:]
    r = json.loads(p.stdout.strip().splitlines()[-1])
    kernels = r["kernels"]
    assert r["launches"] == len(kernels), "last_launches() = %d, profiler: %d kernels %r" % (r["launches"], len(kernels), kernels)
    assert sum("k_c_fanout" in k for k in kernels) >= 1  # the export


def test_group_leader(built, tmp_path):
    fam = Fam("cf32_1536k_m2", M2, 1536000)
    sched = [16384, 8192, 16384, 32768]
    raws = stimulus(fam, sum(sched), 6)

    def group(dump):
        lead = aisgpu.Engine(n_streams=B, max_chunk=max(sched), **fam.kw())
        mem = [lead.attach(model=M0), lead.attach(model=M11)]
        if dump:
            with pytest.raises(aisgpu.AisGpuError, match="rc=-1"):  # a member has no front end
                mem[0].dump_open(prefixes(tmp_path, "mem", DUMPED))
            lead.dump_open(prefixes(tmp_path, "grp", DUMPED))
        pos, out = 0, [[] for _ in mem]
        for n in sched:
            submit(lead, fam, raws, pos, n, "sync", [])
            pos += n
            for i, m in enumerate(mem):
                out[i] += m.poll()
            lead.poll()
        for m in mem:
            m.close()
        lead.close()  # closes the dump
        return out

    with_dump, without = group(True), group(False)
    for a, b in zip(with_dump, without):
        assert frames_key(a) == frames_key(b)
    run_engine(tmp_path, fam, raws, sched, ["sync"], DUMPED, tag="solo")
    assert_same_files(tmp_path, DUMPED, got="grp", want="solo")


def test_refusals(built, tmp_path):
    fam = Fam("cf32_1536k_m2", M2, 1536000)
    sched = [16384, 16384, 8192]
    raws = stimulus(fam, sum(sched), 7)
    p = prefixes(tmp_path, "r", DUMPED)
    import ctypes as C

    def refused(eng, *args, match):
        with pytest.raises(aisgpu.AisGpuError, match=match):
            eng.dump_open(*args)

    for kw, why in ((dict(channel_mode=aisgpu.MODE_X, sample_rate=48000), "single-channel"),
                    (dict(model=M3, sample_rate=48000), "FM-discriminator")):
        e = aisgpu.Engine(n_streams=B, max_chunk=16384, **dict(fam.kw(), **kw))
        refused(e, p, match=why)
        e.close()
    eng = aisgpu.Engine(n_streams=B, max_chunk=max(sched), **fam.kw())
    assert eng.lib.aisgpu_dump_open(eng.h, None) == aisgpu.EINVAL
    eng.dump_open(p)
    refused(eng, p, match="already open")
    eng.dump_close()
    frames, pos = [], 0
    for i, n in enumerate(sched):
        submit(eng, fam, raws, pos, n, "sync", [])
        pos += n
        if i == 0:
            refused(eng, p, match="already been submitted")
        frames += eng.poll()
    eng.close()
    assert not any(tmp_path.iterdir())
    twin = run_engine(tmp_path, fam, raws, sched, ["sync"], DUMPED, dump=False)[0]
    assert frames_key(frames) == frames_key(twin)


def test_file_error(built, tmp_path):
    fam = Fam("cf32_1536k_m2", M2, 1536000)
    sched = [16384, 16384, 16384, 16384]
    raws = stimulus(fam, sum(sched), 8)
    bad = [str(tmp_path / "missing" / ("x%d" % s)) if s == 2 else None for s in range(B)]
    eng = aisgpu.Engine(n_streams=B, max_chunk=max(sched), **fam.kw())
    eng.dump_open(bad)
    frames = []
    submit(eng, fam, raws, 0, sched[0], "sync", [])
    frames += eng.poll()  # writes submit 0: the create fails, the poll does not
    want = 'WAV out: Cannot open WAV file for writing: "%s_A.wav"' % bad[2]
    with pytest.raises(aisgpu.AisGpuError) as ei:
        submit(eng, fam, raws, sched[0], sched[1], "sync", [])
    assert "rc=-6" in str(ei.value) and want in str(ei.value)
    with pytest.raises(aisgpu.AisGpuError) as ei:
        submit(eng, fam, raws, sched[0], sched[1], "async", [])
    assert "rc=-6" in str(ei.value)
    with pytest.raises(aisgpu.AisGpuError) as ei:
        eng.dump_close()
    assert "rc=-6" in str(ei.value) and want in str(ei.value)
    # submits run again; the refused ones were never enqueued
    pos = sched[0]
    for n in sched[1:]:
        submit(eng, fam, raws, pos, n, "sync", [])
        pos += n
        frames += eng.poll()
    eng.close()
    twin = run_engine(tmp_path, fam, raws, sched, ["sync"], DUMPED, dump=False)[0]
    assert frames_key(frames) == frames_key(twin)


def test_destroy_without_close(built, tmp_path):
    fam = Fam("cs16_384k_m0", M0, 384000, CS16)
    sched = [8192, 4096, 8192]
    raws = stimulus(fam, sum(sched), 9)
    eng = aisgpu.Engine(n_streams=B, max_chunk=max(sched), **fam.kw())
    eng.dump_open(prefixes(tmp_path, "gpu", DUMPED))
    pos, keep = 0, []
    for n in sched:
        submit(eng, fam, raws, pos, n, "async", keep)
        pos += n
    eng.close()  # no poll, no dump_close
    reference_files(tmp_path, fam, raws, sched, DUMPED)
    assert_same_files(tmp_path, DUMPED)


ADAPTER = OD.adapter_dump_path()


@pytest.mark.skipif(not os.path.exists(ADAPTER), reason="adapter_dump_test not built")
@pytest.mark.parametrize("mode,model,fs,fmt", [("AB", 2, 1536000, "CF32"), ("CD", 0, 288000, "CS16"), ("X", 2, 48000, "CF32")])
def test_adapter(built, tmp_path, mode, model, fs, fmt):
    n, block = int(0.3 * fs) // 64 * 64, 8192 if fs < 1000000 else 65536
    x = X.x_stream(fs, n, 11)[0] if mode == "X" else S.random_stream(fs, n, 11)[0]
    raw, _ = X.to_raw(x, O.FMT_CS16 if fmt == "CS16" else O.FMT_CF32)
    f = tmp_path / "in.raw"
    raw.tofile(f)
    out = {}
    for side in ("gpu", "cpu"):
        d = tmp_path / side
        d.mkdir()
        args = [ADAPTER, str(f), fmt, str(fs), str(block), str(model), mode, str(d / "ch")] + (["cpu"] if side == "cpu" else [])
        p = subprocess.run(args, capture_output=True)
        assert p.returncode == 0, p.stderr.decode("latin-1")
        out[side] = (p.stdout, {q.name: q.read_bytes() for q in d.iterdir()})
    assert out["gpu"][0] == out["cpu"][0]  # message count
    assert out["gpu"][1] == out["cpu"][1]
    assert sorted(out["gpu"][1]) == ([] if mode == "X" else ["ch_A.wav", "ch_B.wav"])
