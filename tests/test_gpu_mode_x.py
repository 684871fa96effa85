"""-m gpu: single-channel mode (-c X) through the C ABI, bit for bit (tolerance 0) against the compiled reference in mode X
(oracle/_ref, when it travelled) and always against tests/golden/mode_x.json.  Levels and ppm are compared as bit patterns with
tag_mode = 3.  At interpolated rates the engine's per-submit taps hold the last reference block of the submit, so they are
checked against the tail of what the reference emitted in that submit; the Upsample output itself is checked as one stream."""
import os
import subprocess

import numpy as np
import pytest

import aisgpu
import mode_x_util as X
import oracle as O
import oracle_x as OX

pytestmark = pytest.mark.gpu

BUCKETS = (48000, 96000, 192000)


def interpolated(fs):
    return fs not in BUCKETS


def gpu_taps(model):
    """(name, aisgpu tap, channel argument, dtype) of the taps one model exposes; names as in mode_x_util.CTAPS / FTAPS."""
    t = [("C", aisgpu.TAP_C, 0, np.complex64)]
    if model == aisgpu.MODEL_DEFAULT:
        t += [("CGF", aisgpu.TAP_CGF, 0, np.complex64), ("FC", aisgpu.TAP_FIR, 0, np.complex64)]
        t += [("DEC%d" % ph, aisgpu.TAP_DEC, 2 * ph, np.float32) for ph in range(5)]
    elif model in (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE):
        t += [("FM", aisgpu.TAP_FM, 0, np.float32), ("FR", aisgpu.TAP_FIR, 0, np.float32)]
        t += [("DEC%d" % ph, aisgpu.TAP_DEC, 2 * ph, np.float32) for ph in range(5 if model == aisgpu.MODEL_STANDARD else 1)]
    return t


def msg_rec(m):
    return {"ch": m.channel, "nbits": m.nbits, "payload": m.payload.hex(), "nmea": list(m.nmea), "start": m.start_idx, "end": m.end_idx,
            "level": X.fbits(m.level), "ppm": X.fbits(m.ppm)}


def run_x(model, fs, N, nchunks, fmt, flags, seeds, submit="submit", taps=True):
    """Runs len(seeds) streams through one X engine.  Returns (raw inputs, per stream: messages per chunk, per stream: tap name ->
    list of per-chunk arrays)."""
    B = len(seeds)
    raws = [X.stream_input(fs, N * nchunks, sd, fmt) for sd in seeds]
    per = raws[0][1]
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N, ps_ema=bool(flags & O.FLAG_PS_EMA),
                        afc_wide=bool(flags & O.FLAG_AFC_WIDE), droop=bool(flags & O.FLAG_DROOP), taps=taps, channel_mode=aisgpu.MODE_X,
                        channels="XX")
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
                for name, t, ch, dt in gpu_taps(model):
                    tapv[s].setdefault(name, []).append(eng.tap(t, s, ch, dtype=dt))
                if interpolated(fs):
                    tapv[s].setdefault("US", []).append(eng.tap(aisgpu.TAP_PRE, s, 0))
        for m in eng.poll():
            msgs[m.stream][c].append(msg_rec(m))
    cnt = eng.counters()
    eng.close()
    assert cnt[6] == 0 and cnt[5] == cnt[1], "single-channel frames count as channel A only: %r" % (cnt,)
    return raws, msgs, tapv


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def compare_ref(model, fs, N, nchunks, fmt, flags, raws, msgs, tapv, streams=None):
    """Every stream (or the given ones) against its own reference instance; returns a list of problems."""
    problems = []
    for s in (range(len(raws)) if streams is None else streams):
        raw, per = raws[s]
        chunks, want = X.ref_run(model, fs, N, nchunks, fmt, flags, raw, per)
        if msgs[s] != chunks:
            problems.append(("MSG", s, sum(map(len, msgs[s])), sum(map(len, chunks)), [m for c in msgs[s] for m in c if m not in [q for cc in chunks for q in cc]][:1]))
        for name, got in tapv[s].items():
            if name == "US":  # the reference holds a partial block back: compare the common prefix
                g, w = np.concatenate(got), np.concatenate(want["US"])
                n = min(len(g), len(w))
                if n == 0 or not bits_equal(g[:n], w[:n]):
                    problems.append(("US", s, len(g), len(w)))
                continue
            for c in range(nchunks):
                g, w = got[c], want[name][c]
                if interpolated(fs):
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
        problems.append(("golden MSG", sum(map(len, msgs0)), sum(map(len, case["messages"]))))
    for name, got in tap0.items():
        n, h = case["taps"][name]
        g = np.concatenate(got)
        if name == "US":
            g = g[:n]
        elif interpolated(case["fs"]):
            continue  # per-submit taps hold the last block only: checked against the reference
        if len(g) != n or X.sha(g) != h:
            problems.append(("golden tap", name, len(g), n))
    return problems


@pytest.mark.parametrize("name", [c[0] for c in X.CASES])
def test_golden_cases(built, name):
    case = X.load()[name]
    seeds = [case["seed"], case["seed"] + 1000, case["seed"] + 2000]
    raws, msgs, tapv = run_x(case["model"], case["fs"], case["N"], case["nchunks"], case["fmt"], case["flags"], seeds)
    assert X.sha(raws[0][0]) == case["input_sha256"]
    problems = compare_golden(case, msgs[0], tapv[0])
    if OX.have_refx():
        problems += compare_ref(case["model"], case["fs"], case["N"], case["nchunks"], case["fmt"], case["flags"], raws, msgs, tapv)
    assert not problems, problems[:12]
    if case["fs"] > 24000:  # 12-24 kS/s is undersampled and may decode nothing; the taps must still match
        assert sum(map(len, msgs[0])) > 0


@pytest.mark.skipif(not OX.have_refx(), reason="the model x bucket x format matrix is checked against the compiled reference")
@pytest.mark.parametrize("fmt", [aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16])
@pytest.mark.parametrize("fs", BUCKETS)
@pytest.mark.parametrize("model", [aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2])
def test_matrix(built, model, fs, fmt):
    N = fs // 48000 * 2048
    raws, msgs, tapv = run_x(model, fs, N, 5, fmt, O.DEFAULT_FLAGS, [40 + model, 50 + fmt])
    assert not compare_ref(model, fs, N, 5, fmt, O.DEFAULT_FLAGS, raws, msgs, tapv)


@pytest.mark.skipif(not OX.have_refx(), reason="checked against the compiled reference")
@pytest.mark.parametrize("fs,N", [(12000, 1024), (24000, 1024), (50000, 2048), (100000, 4096), (150000, 6400)])
@pytest.mark.parametrize("flags", [O.DEFAULT_FLAGS, X.NODROOP, X.NOEMA])
def test_interpolated_rates(built, fs, N, flags):
    raws, msgs, tapv = run_x(aisgpu.MODEL_DEFAULT, fs, N, 8, aisgpu.FMT_CF32, flags, [60, 61], submit="submit_v")
    assert not compare_ref(aisgpu.MODEL_DEFAULT, fs, N, 8, aisgpu.FMT_CF32, flags, raws, msgs, tapv)


@pytest.mark.parametrize("B", [1, 3, 33])
@pytest.mark.parametrize("name", ["default_48k", "challenger_48k", "standard_48k", "v2_48k", "default_192k_cs16"])
def test_odd_batches(built, B, name):
    # the back end has only ever run even row counts in AB mode; in X a row is a stream
    case = X.load()[name]
    seeds = [case["seed"]] + [case["seed"] + 1000 * s for s in range(1, B)]
    raws, msgs, tapv = run_x(case["model"], case["fs"], case["N"], case["nchunks"], case["fmt"], case["flags"], seeds, taps=B < 33)
    problems = compare_golden(case, msgs[0], tapv[0]) if B < 33 else ([] if msgs[0] == case["messages"] else ["golden MSG"])
    if OX.have_refx():
        problems += compare_ref(case["model"], case["fs"], case["N"], case["nchunks"], case["fmt"], case["flags"], raws, msgs, tapv,
                                streams=range(B) if B < 33 else (0, 16, 31, 32))
    assert not problems, problems[:12]


def test_x_taps_rejected(built):
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, n_streams=2, max_chunk=4096, taps=True, channel_mode=aisgpu.MODE_X)
    eng.submit(np.zeros((2, 4096), np.complex64), 4096)
    for tap, ch in ((aisgpu.TAP_ROT, 0), (aisgpu.TAP_C, 1), (aisgpu.TAP_DEC, 3)):
        with pytest.raises(aisgpu.AisGpuError, match="single-channel"):
            eng.tap(tap, 0, ch)
    assert len(eng.tap(aisgpu.TAP_C, 1, 0)) == 4096
    with pytest.raises(aisgpu.AisGpuError, match="granule|multiple of 64"):
        eng.submit(np.zeros((2, 4096), np.complex64)[:, :4032].copy(), 4000)
    eng.close()
    with pytest.raises(aisgpu.AisGpuError, match="between 12k and 192k"):
        aisgpu.Engine(sample_rate=11999, channel_mode=aisgpu.MODE_X)


def test_x_launches(built):
    # one front-end kernel and no Rotate table: one launch fewer than the AB chain at the same bucket
    counts = {}
    for mode in (aisgpu.MODE_AB, aisgpu.MODE_X):
        eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=96000, n_streams=2, max_chunk=8192, channel_mode=mode)
        for _ in range(3):
            eng.submit(np.zeros((2, 8192), np.complex64), 8192)
        eng.sync()
        counts[mode] = eng.last_launches()
        eng.close()
    assert counts[aisgpu.MODE_X] == counts[aisgpu.MODE_AB] - 1


def test_back_to_back_entry_points(built):
    """Ten submits without a sync through each of the four submit entry points give the same frames as one submit + poll each."""
    import torch
    case = X.load()["default_48k"]
    N, nchunks, B = 2048, 10, 3
    raws = [X.stream_input(48000, N * nchunks, case["seed"] + s, aisgpu.FMT_CF32)[0] for s in range(B)]
    x = np.stack(raws)  # [B][N * nchunks]

    def run(kind):
        eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, n_streams=B, max_chunk=N, channel_mode=aisgpu.MODE_X,
                            max_frames=4096)
        out, keep, tickets = [], [], []
        dev = torch.from_numpy(x.view(np.float32)).cuda() if kind == "device" else None
        for c in range(nchunks):
            blk = np.ascontiguousarray(x[:, c * N:(c + 1) * N])
            if kind == "submit":
                eng.submit(blk, N)
            elif kind == "v":
                eng.submit_v(list(blk), N)
            elif kind == "async":
                keep.append(blk)
                tickets.append(eng.submit_async_ptr(blk.ctypes.data, N))
            else:
                eng.submit_device(dev.data_ptr() + c * N * 8, N * nchunks, N)
            if kind == "async" and c == 4:
                out += eng.poll_upto(tickets[2])  # the frames of submits 0..2 only
        out += eng.poll()
        eng.close()
        return [(m.stream, m.chunk, m.key(), m.start_idx, X.fbits(m.level)) for m in out]

    want = []
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, n_streams=B, max_chunk=N, channel_mode=aisgpu.MODE_X)
    for c in range(nchunks):
        eng.submit(np.ascontiguousarray(x[:, c * N:(c + 1) * N]), N)
        want += [(m.stream, m.chunk, m.key(), m.start_idx, X.fbits(m.level)) for m in eng.poll()]
    eng.close()
    assert len(want) > 0
    for kind in ("submit", "v", "async", "device"):
        assert run(kind) == want, kind


def test_ring_overflow_reported(built):
    case = X.load()["default_48k"]
    N, nchunks = case["N"], case["nchunks"]
    raws = [X.stream_input(48000, N * nchunks, case["seed"], aisgpu.FMT_CF32)[0]] * 4
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, n_streams=4, max_chunk=N * nchunks, max_frames=2,
                        channel_mode=aisgpu.MODE_X)
    eng.submit(np.stack(raws), N * nchunks)
    got = eng.poll()
    c = eng.counters()
    eng.close()
    assert eng.overflows >= 1 and c[4] > 0 and len(got) <= 2


def test_feed_files_ragged(built, tmp_path):
    # recordings of different lengths, read in blocks, the tails zero-padded: the same frames as submitting the padded blocks
    N = 2048
    lens = [N * 5, N * 3 + 700, N * 7 - 64]
    xs = [X.stream_input(48000, n, 70 + s, aisgpu.FMT_CU8)[0] for s, n in enumerate(lens)]
    paths = []
    for s, x in enumerate(xs):
        p = os.path.join(tmp_path, "x%d.cu8" % s)
        x.tofile(p)
        paths.append(p)
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, fmt=aisgpu.FMT_CU8, n_streams=3, max_chunk=N, channel_mode=aisgpu.MODE_X)
    got, nb = eng.feed_files(paths, N)
    eng.close()
    nblk = max((n + N - 1) // N for n in lens)
    assert nb == nblk
    pad = np.zeros((3, nblk * N * 2), np.uint8)  # zero bytes, as the feeder pads (FileRAW.cpp:91-94)
    for s, x in enumerate(xs):
        pad[s, :len(x)] = x
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, fmt=aisgpu.FMT_CU8, n_streams=3, max_chunk=N, channel_mode=aisgpu.MODE_X)
    want = []
    for c in range(nblk):
        eng.submit(np.ascontiguousarray(pad[:, c * 2 * N:(c + 1) * 2 * N]), N)
        want += eng.poll()
    eng.close()
    key = lambda ms: [(m.stream, m.key(), m.start_idx, m.end_idx) for m in ms]
    assert len(want) > 0 and key(got) == key(want)


ADAPTER = os.path.join(os.path.dirname(O.HERE), "oracle", "_ref", "adapter_mode_test")


@pytest.mark.skipif(not os.path.exists(ADAPTER), reason="adapter_mode_test not built (needs the reference tree at build time)")
@pytest.mark.parametrize("mode,fs,fmt", [("X", 48000, "CF32"), ("X", 96000, "CU8"), ("X", 50000, "CF32"), ("CD", 96000, "CU8")])
def test_adapter_modes(built, tmp_path, mode, fs, fmt):
    """AIS::ModelGPU with setMode(X / CD) prints exactly what the reference's ModelDefault prints in the same binary."""
    import aissynth as S
    f = aisgpu.FMT_CF32 if fmt == "CF32" else aisgpu.FMT_CU8
    n = fs * 2
    x = X.stream_input(fs, n, 90, f)[0] if mode == "X" else X.to_raw(S.random_stream(fs, n, 90)[0], f)[0]
    path = os.path.join(tmp_path, "in.raw")
    x.tofile(path)
    outs = [subprocess.run([ADAPTER, mode, path, fmt, str(fs), "4096"] + extra, capture_output=True, text=True, timeout=300)
            for extra in ([], ["cpu"])]
    assert outs[0].returncode == 0 and outs[1].returncode == 0, (outs[0].stderr, outs[1].stderr)
    assert outs[0].stdout == outs[1].stdout
    assert outs[1].stdout.count("\n") > 0
    letters = ("X",) if mode == "X" else ("C", "D")
    assert all(l[0] in letters for l in outs[1].stdout.splitlines())
