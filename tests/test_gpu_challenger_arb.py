"""-m gpu: ModelChallenger's ten cross-reset decoders (k_decode10) on the stimulus where their order within a group decides what is
published, frame by frame against the compiled reference.

The stimulus is tests/challenger_arb.py's: threshold sweeps where coherent decoders win, FM-only nulls that hand frames to a0..a4,
back-to-back frames on the alternation threshold (the Reset's replay), closing groups across CGF blocks whose ppm differ, and submit
schedules with a boundary inside closing groups (the FM lanes' partial groups and channel B's first-group level carry).  Frames are
compared through parity_util.compare_frames (payload, NMEA, channel, start / end counters, level and ppm bit patterns), and no frame
may be lost to ring overflow.  Reference runs are shared between the variants of a case."""
import os
import threading

import numpy as np
import pytest

import aisgpu
import aissynth as S
import challenger_arb as CA
import oracle as O
import oracle_x as OX
import parity_util as U

pytestmark = pytest.mark.gpu

M4 = aisgpu.MODEL_CHALLENGER
FS = 96000
B = 16
NARROW = O.FLAG_PS_EMA | O.FLAG_DROOP
SCHEDULE = [4096, 256, 32768, 1000, 7776, 16384, 332, 65536, 12000, 2048]  # test_gpu_decoder_limits' changing submit lengths

_ref = {}  # (kind, rate, flags, submit lengths, input id) -> per-stream reference frames


@pytest.fixture(scope="module")
def ab():
    return CA.render(CA.build(B), FS)


@pytest.fixture(scope="module")
def xx():
    return CA.render(CA.build(B, x_mode=True), 48000)


def lengths_of(total, chunk):
    out, pos, k = [], 0, 0
    while pos < total:
        n = min(chunk if chunk else SCHEDULE[k % len(SCHEDULE)], total - pos)
        out.append(n)
        pos += n
        k += 1
    return out


def run_refs(make, xs, lengths):
    """One reference instance per stream, fed the same submits; host threads in parallel (ctypes releases the GIL)."""
    out = [None] * len(xs)
    nthr = min(len(xs), max(1, len(os.sched_getaffinity(0))))

    def work(ids):
        for s in ids:
            m = make()
            pos = 0
            for n in lengths:
                m.push(xs[s][pos:pos + n])
                pos += n
            out[s] = m.messages()
            m.close()

    ths = [threading.Thread(target=work, args=(list(range(t, len(xs), nthr)),)) for t in range(nthr)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    return out


def ref_frames(kind, fs, flags, xs, lengths):
    key = (kind, fs, flags, tuple(lengths), id(xs))
    if key not in _ref:
        if kind == "x":
            make = lambda: OX.RefModelX(model=M4, sample_rate=fs, flags=flags)
        else:
            make = lambda: O.RefModel(model=M4, sample_rate=fs, flags=flags)
        _ref[key] = run_refs(make, xs, lengths)
    return _ref[key]


def split_lengths(kind, fs, flags, xs):
    """One submit schedule for the batch: a boundary inside the closing group of every frame of every stream (the reference's own
    end_idx, from its run in submits of 4096)."""
    base = ref_frames(kind, fs, flags, xs, lengths_of(xs.shape[1], 4096))
    return CA.split_schedule([m.end_idx for frames in base for m in frames], fs, xs.shape[1], 8192)


def run_engine(xs, lengths, **kw):
    n_streams = len(xs)
    eng = aisgpu.Engine(model=M4, n_streams=n_streams, max_chunk=max(lengths), max_frames=1 << 16, **kw)
    got = [[] for _ in range(n_streams)]
    pos = 0
    for i, n in enumerate(lengths):
        eng.submit(np.ascontiguousarray(xs[:, pos:pos + n]), n)
        pos += n
        if i % 64 == 63:
            for m in eng.poll():
                got[m.stream].append(m)
    for m in eng.poll():
        got[m.stream].append(m)
    cnt = eng.counters()
    eng.close()
    assert eng.overflows == 0 and cnt[4] == 0, "frames dropped by ring overflow: %r" % (cnt,)
    return got


def check(got, want, label):
    assert sum(len(w) for w in want) > 0, label
    problems = U.compare_frames(got, want)
    assert not problems, "%s: frames differ from the reference (kind, stream, got, want, only in engine, only in reference): %r" % (
        label, problems[:3])


@pytest.mark.parametrize("afc_wide", [True, False])
@pytest.mark.parametrize("chunk", [256, 4096, 32768, None, "split"])
def test_ab(built, ab, chunk, afc_wide):
    flags = O.DEFAULT_FLAGS if afc_wide else NARROW
    lengths = split_lengths("ab", FS, flags, ab) if chunk == "split" else lengths_of(ab.shape[1], chunk)
    want = ref_frames("ab", FS, flags, ab, lengths)
    got = run_engine(ab, lengths, sample_rate=FS, afc_wide=afc_wide)
    check(got, want, "AB, submits %s, AFC_WIDE %s" % (chunk or "SCHEDULE", afc_wide))


@pytest.mark.parametrize("rpw", ["1", "3"])
@pytest.mark.parametrize("chunk", [4096, "split"])
def test_ab_rows_per_warp(built, ab, monkeypatch, rpw, chunk):
    # rows of different streams (and channels A / B) share a warp, each with its own winners and replay positions
    monkeypatch.setenv("AISGPU_DEC_RPW", rpw)
    flags = O.DEFAULT_FLAGS
    lengths = split_lengths("ab", FS, flags, ab) if chunk == "split" else lengths_of(ab.shape[1], chunk)
    want = ref_frames("ab", FS, flags, ab, lengths)
    got = run_engine(ab, lengths, sample_rate=FS)
    check(got, want, "AB, AISGPU_DEC_RPW=%s, submits %s" % (rpw, chunk))


@pytest.mark.parametrize("chunk", [4096, "split"])
def test_mode_x(built, xx, chunk):
    # one chain per stream: the level the FM decoders carry into a submit is the row's own (lvl_own)
    fs, flags = 48000, O.DEFAULT_FLAGS
    lengths = split_lengths("x", fs, flags, xx) if chunk == "split" else lengths_of(xx.shape[1], chunk)
    want = ref_frames("x", fs, flags, xx, lengths)
    got = run_engine(xx, lengths, sample_rate=fs, channel_mode=aisgpu.MODE_X, channels="XX")
    check(got, want, "X mode, submits %s" % chunk)


def test_cu8_1536k_device_batch(built):
    """CU8 at 1536 kS/s, a batch of 256 streams (16 unique stimuli, each 16 times) submitted from device memory in submits of
    65536 samples; every stream against its unique stimulus's reference."""
    import torch
    fs, Bn, U16, N = 1536000, 256, 16, 65536
    streams = CA.build(U16, per_family=(8, 5, 10, 20), seed=1)
    uniq = np.stack([S.to_cu8(x) for x in CA.render(streams, fs)])  # [U16][2 n] uint8
    K = uniq.shape[1] // (2 * N)
    uniq = np.ascontiguousarray(uniq[:, :2 * N * K])
    want = run_refs(lambda: O.RefModel(model=M4, sample_rate=fs, fmt=O.FMT_CU8), uniq, [2 * N] * K)
    dev = torch.device("cuda", 0)
    x = torch.from_numpy(uniq).to(dev).repeat(Bn // U16, 1).contiguous()  # stream b = stimulus b % 16
    eng = aisgpu.Engine(model=M4, sample_rate=fs, fmt=aisgpu.FMT_CU8, n_streams=Bn, max_chunk=N, max_frames=1 << 18,
                        host_staging=False)
    got = [[] for _ in range(Bn)]
    for c in range(K):
        eng.submit_device(x.data_ptr() + c * 2 * N, K * N, N)
        if c % 8 == 7:
            for m in eng.poll():
                got[m.stream].append(m)
    for m in eng.poll():
        got[m.stream].append(m)
    cnt = eng.counters()
    eng.close()
    assert eng.overflows == 0 and cnt[4] == 0, cnt
    check(got, [want[b % U16] for b in range(Bn)], "CU8 1536 kS/s, batch 256 from device memory")
