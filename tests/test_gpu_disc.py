"""-m gpu: the FM-discriminator input model (-m 3) through the C ABI, bit for bit (tolerance 0) against the reference's
ModelDiscriminator (oracle/_ref/libaisrefd.so, when it travelled) and always against tests/golden/disc.json.  Levels and ppm are
compared as bit patterns.  Below 48 kHz the engine's per-submit taps hold the last Upsample block of the submit, so they are checked
against the tail of what the reference emitted in that submit; the Upsample output itself is checked as one stream."""
import os
import subprocess

import numpy as np
import pytest

import aisgpu
import disc_util as D
import oracle_disc as OD

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTER = os.path.join(ROOT, "oracle", "_ref", "adapter_disc_test")
M3 = aisgpu.MODEL_DISCRIMINATOR


def gpu_taps():
    """(name, aisgpu tap, channel argument) per channel ch; names as in disc_util.FTAPS."""
    return lambda ch: [("C", aisgpu.TAP_C, ch), ("FR", aisgpu.TAP_FIR, ch)] + [("DEC%d" % ph, aisgpu.TAP_DEC, ch + 2 * ph) for ph in range(5)]


def run_disc(fs, N, nchunks, fmt, letters, seeds, submit="submit", taps=True, type5=False, mode=aisgpu.MODE_AB):
    """len(seeds) streams through one -m 3 engine.  Returns (raw inputs, per stream: messages per chunk, per stream: tap -> per-chunk
    arrays)."""
    B = len(seeds)
    raws = [D.stream_input(fs, N * nchunks, sd, fmt, type5) for sd in seeds]
    per = raws[0][1]
    eng = aisgpu.Engine(model=M3, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N, taps=taps, channel_mode=mode, channels=letters)
    msgs = [[[] for _ in range(nchunks)] for _ in range(B)]
    tapv = [{} for _ in range(B)]
    for c in range(nchunks):
        batch = np.stack([r[c * N * per:(c + 1) * N * per] for r, _ in raws])
        if submit == "submit":
            eng.submit(batch, N)
        else:
            eng.submit_v(list(batch), N)
        if taps:
            for s in range(B):
                for ch in (0, 1):
                    for name, t, arg in gpu_taps()(ch):
                        tapv[s].setdefault("%s_%d" % (name, ch), []).append(eng.tap(t, s, arg, dtype=np.float32))
                if fs != 48000:
                    tapv[s].setdefault("US", []).append(eng.tap(aisgpu.TAP_PRE, s, 0))
        for m in eng.poll():
            msgs[m.stream][c].append(D.msg_rec(m))
    cnt = eng.counters()
    eng.close()
    assert cnt[5] + cnt[6] == cnt[1]
    return raws, msgs, tapv


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def compare_ref(fs, N, nchunks, fmt, letters, raws, msgs, tapv, streams=None):
    """Every stream (or the given ones) against its own reference instance; returns a list of problems."""
    problems = []
    for s in (range(len(raws)) if streams is None else streams):
        raw, per = raws[s]
        chunks, want = D.ref_run(fs, N, nchunks, fmt, letters, raw, per)
        if msgs[s] != chunks:
            problems.append(("MSG", s, [len(c) for c in msgs[s]], [len(c) for c in chunks]))
        for name, got in tapv[s].items():
            if name == "US":  # the reference holds a partial block back: compare the common prefix
                g, w = np.concatenate(got), np.concatenate(want["US"])
                n = min(len(g), len(w))
                if n == 0 or not bits_equal(g[:n], w[:n]):
                    problems.append(("US", s, len(g), len(w)))
                continue
            for c in range(nchunks):
                g, w = got[c], want[name][c]
                if fs != 48000:
                    if len(w) == 0:
                        continue
                    w = w[-len(g):] if len(g) <= len(w) else None
                    if w is None:
                        problems.append((name, s, c, "longer than the reference's", len(g)))
                        continue
                if not bits_equal(g, w):
                    problems.append((name, s, c, len(g), len(w)))
    return problems


def compare_golden(case, msgs0, tap0):
    problems = []
    if msgs0 != case["messages"]:
        problems.append(("golden MSG", [len(c) for c in msgs0], [len(c) for c in case["messages"]]))
    for name, got in tap0.items():
        n, h = case["taps"][name]
        g = np.concatenate(got)
        if name == "US":
            g = g[:n]
        elif case["fs"] != 48000:
            continue  # per-submit taps hold the last block only: checked against the reference
        if len(g) != n or D.sha(g) != h:
            problems.append(("golden tap", name, len(g), n))
    return problems


@pytest.mark.parametrize("name", [c[0] for c in D.CASES])
def test_golden_cases(built, name):
    case = D.load()[name]
    t5 = name.startswith("type5")
    seeds = [case["seed"], case["seed"] + 1000, case["seed"] + 2000]
    raws, msgs, tapv = run_disc(case["fs"], case["N"], case["nchunks"], case["fmt"], case["letters"], seeds, type5=t5)
    assert D.sha(raws[0][0]) == case["input_sha256"]
    problems = compare_golden(case, msgs[0], tapv[0])
    if OD.have_refd():
        problems += compare_ref(case["fs"], case["N"], case["nchunks"], case["fmt"], case["letters"], raws, msgs, tapv)
    assert not problems, problems[:12]
    assert sum(map(len, msgs[0])) > 0


@pytest.mark.skipif(not OD.have_refd(), reason="checked against the compiled reference")
@pytest.mark.parametrize("fmt", [aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16])
@pytest.mark.parametrize("mode,letters", [(aisgpu.MODE_AB, "AB"), (aisgpu.MODE_X, "XX")])
def test_formats_48k(built, fmt, mode, letters):
    raws, msgs, tapv = run_disc(48000, 2048, 6, fmt, letters, [40 + fmt, 50 + fmt], mode=mode)
    assert not compare_ref(48000, 2048, 6, fmt, letters, raws, msgs, tapv)


@pytest.mark.skipif(not OD.have_refd(), reason="checked against the compiled reference")
@pytest.mark.parametrize("fs,N", [(44100, 4416), (32000, 2048), (22050, 1024), (12000, 1024), (12000, 4096)])
@pytest.mark.parametrize("fmt", [aisgpu.FMT_CS16, aisgpu.FMT_CF32])
def test_interpolated_rates(built, fs, N, fmt):
    # each submit is re-blocked by Upsample into several blocks of N (up to 4 at 12 kS/s): the frames of one submit interleave
    # A, B, A, B block by block, as the reference's two sinks of US do
    nch = max(4, 40000 // N)
    raws, msgs, tapv = run_disc(fs, N, nch, fmt, "AB", [60, 61], submit="submit_v")
    assert not compare_ref(fs, N, nch, fmt, "AB", raws, msgs, tapv)
    assert sum(len(c) for s in msgs for c in s) > 0


@pytest.mark.parametrize("B", [1, 3, 33])
@pytest.mark.parametrize("name", ["cs16_48k", "cs16_44k1", "cf32_12k"])
def test_odd_batches(built, B, name):
    case = D.load()[name]
    seeds = [case["seed"]] + [case["seed"] + 1000 * s for s in range(1, B)]
    raws, msgs, tapv = run_disc(case["fs"], case["N"], case["nchunks"], case["fmt"], case["letters"], seeds, taps=B < 33)
    problems = compare_golden(case, msgs[0], tapv[0]) if B < 33 else ([] if msgs[0] == case["messages"] else ["golden MSG"])
    if OD.have_refd():
        problems += compare_ref(case["fs"], case["N"], case["nchunks"], case["fmt"], case["letters"], raws, msgs, tapv,
                                streams=range(B) if B < 33 else (0, 16, 31, 32))
    assert not problems, problems[:12]


def test_taps_rejected(built):
    N = 4096
    eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=2, max_chunk=N, taps=True)
    eng.submit(np.zeros((2, 2 * N), np.int16), N)
    for tap in (aisgpu.TAP_ROT, aisgpu.TAP_CGF, aisgpu.TAP_PRE2, aisgpu.TAP_FM):
        with pytest.raises(aisgpu.AisGpuError):
            eng.tap(tap, 0, 0)
    c = eng.tap(aisgpu.TAP_C, 1, 1, dtype=np.float32)  # 4-byte elements: the real row
    assert len(c) == N
    with pytest.raises(aisgpu.AisGpuError, match="multiple of 64"):
        eng.submit(np.zeros((2, 2 * N), np.int16), 4000)
    eng.close()
    for fs, msg in ((48001, "Internal error: sample rate not supported in FM discriminator model."), (11999, "between 12k and 48k")):
        with pytest.raises(aisgpu.AisGpuError, match=msg):
            aisgpu.Engine(model=M3, sample_rate=fs)


def test_back_to_back_entry_points(built):
    """Ten submits without a sync through each of the four submit entry points give the same frames as one submit + poll each."""
    import torch
    N, nchunks, B = 2048, 10, 3
    raws = [D.stream_input(48000, N * nchunks, 80 + s, aisgpu.FMT_CS16)[0] for s in range(B)]
    x = np.stack(raws)  # [B][2 * N * nchunks] int16

    def run(kind):
        eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=B, max_chunk=N, max_frames=4096)
        out, keep, tickets = [], [], []
        dev = torch.from_numpy(x).cuda() if kind == "device" else None
        for c in range(nchunks):
            blk = np.ascontiguousarray(x[:, c * 2 * N:(c + 1) * 2 * N])
            if kind == "submit":
                eng.submit(blk, N)
            elif kind == "v":
                eng.submit_v(list(blk), N)
            elif kind == "async":
                keep.append(blk)
                tickets.append(eng.submit_async_ptr(blk.ctypes.data, N))
            else:
                eng.submit_device(dev.data_ptr() + c * N * 4, N * nchunks, N)
            if kind == "async" and c == 4:
                out += eng.poll_upto(tickets[2])  # the frames of submits 0..2 only
        out += eng.poll()
        eng.close()
        return [(m.stream, m.chunk, m.key(), m.start_idx, D.fbits(m.level)) for m in out]

    want = []
    eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=B, max_chunk=N)
    for c in range(nchunks):
        eng.submit(np.ascontiguousarray(x[:, c * 2 * N:(c + 1) * 2 * N]), N)
        want += [(m.stream, m.chunk, m.key(), m.start_idx, D.fbits(m.level)) for m in eng.poll()]
    eng.close()
    assert len(want) > 0 and {k[2][0] for k in want} == {"A", "B"}
    for kind in ("submit", "v", "async", "device"):
        assert run(kind) == want, kind


def test_ring_overflow_reported(built):
    case = D.load()["cs16_48k"]
    N, nchunks = case["N"], case["nchunks"]
    raw = D.case_input(case)[0]
    eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=4, max_chunk=N * nchunks, max_frames=2)
    eng.submit(np.stack([raw] * 4), N * nchunks)
    got = eng.poll()
    c = eng.counters()
    eng.close()
    assert eng.overflows >= 1 and c[4] > 0 and len(got) <= 2


def test_feed_files_ragged(built, tmp_path):
    # stereo CS16 recordings of different lengths, read in blocks, the tails zero-padded: the same frames as submitting the padded blocks
    N = 2048
    lens = [N * 5, N * 3 + 700, N * 7 - 64]
    xs = [D.stream_input(48000, n, 70 + s, aisgpu.FMT_CS16)[0] for s, n in enumerate(lens)]
    paths = []
    for s, x in enumerate(xs):
        p = os.path.join(tmp_path, "x%d.cs16" % s)
        x.tofile(p)
        paths.append(p)
    eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=3, max_chunk=N)
    got, nb = eng.feed_files(paths, N)
    eng.close()
    nblk = max((n + N - 1) // N for n in lens)
    assert nb == nblk
    pad = np.zeros((3, nblk * N * 2), np.int16)  # zero bytes, as the feeder pads (FileRAW.cpp:91-94)
    for s, x in enumerate(xs):
        pad[s, :len(x)] = x
    eng = aisgpu.Engine(model=M3, sample_rate=48000, fmt=aisgpu.FMT_CS16, n_streams=3, max_chunk=N)
    want = []
    for c in range(nblk):
        eng.submit(np.ascontiguousarray(pad[:, c * 2 * N:(c + 1) * 2 * N]), N)
        want += eng.poll()
    eng.close()
    key = lambda ms: [(m.stream, m.key(), m.start_idx, m.end_idx) for m in ms]
    assert len(want) > 0 and key(got) == key(want)


@pytest.mark.skipif(not os.path.exists(ADAPTER), reason="adapter_disc_test not built (needs the reference tree at build time)")
@pytest.mark.parametrize("mode,fs,fmt", [("AB", 48000, "CS16"), ("X", 48000, "CS16"), ("X", 44100, "CS16"), ("AB", 32000, "CF32"),
                                         ("AB", 48000, "CU8")])
def test_adapter(built, tmp_path, mode, fs, fmt):
    """AIS::ModelGPU(AISGPU_MODEL_DISCRIMINATOR) prints exactly what the reference's ModelDiscriminator prints in the same binary."""
    f = {"CS16": aisgpu.FMT_CS16, "CF32": aisgpu.FMT_CF32, "CU8": aisgpu.FMT_CU8}[fmt]
    x = D.stream_input(fs, fs * 2, 90, f)[0]
    path = os.path.join(tmp_path, "in.raw")
    x.tofile(path)
    outs = [subprocess.run([ADAPTER, mode, path, fmt, str(fs), "4096", side], capture_output=True, text=True, timeout=300)
            for side in ("gpu", "cpu")]
    assert outs[0].returncode == 0 and outs[1].returncode == 0, (outs[0].stderr, outs[1].stderr)
    assert outs[0].stdout == outs[1].stdout
    assert outs[1].stdout.count("\n") > 0
    assert "class FM" in outs[0].stderr and "class FM" in outs[1].stderr
    letters = ("X",) if mode == "X" else ("A", "B")
    assert {l[0] for l in outs[1].stdout.splitlines()} == set(letters)
