"""-m gpu: every frame decoder at its length limits and abort positions, bit for bit against the compiled reference.

The stimulus is tests/decoder_limits.py's: frames cut so that the closing flag completes exactly on each cannotBeValid position
and on MaxBits (published), one bit longer (dropped one bit before the flag completes) and one bit shorter, frames aborted in
mid-frame with a stuffing zero next to the abort position, each at 32 one-symbol start offsets.  The engine's frames are compared
stream by stream, in emission order, with the reference's (payload including the trailing partial byte, NMEA, channel, start/end
counters, level / ppm bit patterns), no frame may be lost to ring overflow, and the published frames must be exactly the ones the
restated decoder predicts.  The cases reach every restatement of the reference's bit decoder:

* k_decode3 (word-parallel, 1 / 3 / 6 rows per warp) for models 0 and 2 and in X mode, k_decode (bit-serial, AISGPU_DECODER=1),
  k_decode10 (ModelChallenger's ten cross-reset decoders, 1 and 3 rows per warp, and one row per stream in X mode), dec_step in
  ModelBase's kernel and in the V2 engine, and model 3's decoders on a discriminator recording;
* submits of 256 samples (every frame spans many submits), 4096 and 32768, a schedule of changing lengths, 7 streams;
* models 4 and 11 at the launch shape their speeds are quoted for (batch 1024 x 131072 @1536 kS/s, three submits back to back
  from device memory)."""
import os
import threading
from collections import Counter

import numpy as np
import pytest

import aisgpu
import decoder_limits as DL
import oracle as O
import oracle_disc as OD
import oracle_x as OX
import parity_util as U

pytestmark = pytest.mark.gpu

FS = 96000
B = 8
M0, M1, M2, M3, M4, M11 = (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR,
                           aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2)
AB_MODELS = [M0, M1, M2, M4, M11]
SCHEDULE = [4096, 256, 32768, 1000, 7776, 16384, 332, 65536, 12000, 2048]  # samples per submit, repeated (multiples of 4: the reference halves 96 kS/s twice)

_ref = {}  # (kind, model, rate, submit lengths) -> per-stream reference frames; shared by the variants of a case


@pytest.fixture(scope="module")
def stim():
    return DL.Stimulus(DL.designs(), B)


@pytest.fixture(scope="module")
def ab(stim):
    return stim.render_ab(FS)


def lengths_of(total, chunk):
    """Submit lengths covering all `total` samples: a fixed chunk, or the SCHEDULE repeated and cut short at the end."""
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


def ref_frames(kind, model, fs, xs, lengths):
    key = (kind, model, fs, tuple(lengths))
    if key not in _ref:
        if kind == "ab":
            make = lambda: O.RefModel(model=model, sample_rate=fs)
        elif kind == "x":
            make = lambda: OX.RefModelX(model=model, sample_rate=fs)
        else:
            make = lambda: OD.RefModelDisc(sample_rate=fs, fmt=O.FMT_CF32)
        _ref[key] = run_refs(make, xs, lengths)
    return _ref[key]


def run_engine(xs, lengths, **kw):
    """xs[n_streams][n] through one engine in the given submits; returns per-stream frames in emission order."""
    n_streams = len(xs)
    eng = aisgpu.Engine(n_streams=n_streams, max_chunk=max(lengths), max_frames=1 << 16, **kw)
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
    problems = U.compare_frames(got, want)
    assert not problems, "%s: frames differ from the reference (kind, stream, got, want, only in engine, only in reference): %r" % (
        label, problems[:3])


def check_predicted(stim, got, label, channels, track_of):
    """The published frames are the restated decoder's, stream by stream and channel by channel, and every tie / dropped
    neighbour shows as predicted.  track_of(s, ch) = (stream, channel) of the stimulus that engine stream s carries."""
    seen = Counter()
    for s, frames in enumerate(got):
        for ch in channels:
            g = [(m.nbits, m.payload) for m in frames if m.channel == ch]
            assert g == stim.expected(*track_of(s, ch)), "%s: stream %d channel %s is not the predicted frames" % (label, s, ch)
            seen.update(g)
    return seen


def ab_case(stim, ab, model, chunk, n_streams=B, env=None, monkeypatch=None):
    label = "model %d, submits of %s, %d streams%s" % (model, chunk or "SCHEDULE", n_streams, "" if not env else ", %r" % (env,))
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    lengths = lengths_of(ab.shape[1], chunk)
    want = ref_frames("ab", model, FS, ab, lengths)[:n_streams]
    got = run_engine(ab[:n_streams], lengths, model=model, sample_rate=FS)
    check(got, want, label)
    seen = check_predicted(stim, got, label, "AB", lambda s, ch: (s, ch))
    if n_streams == B:
        DL.assert_boundaries(stim.designs, seen, label)


@pytest.mark.parametrize("model", AB_MODELS)
@pytest.mark.parametrize("chunk", [256, 4096, 32768])
def test_ab_chunks(built, stim, ab, model, chunk):
    ab_case(stim, ab, model, chunk)


@pytest.mark.parametrize("model", AB_MODELS)
def test_ab_schedule(built, stim, ab, model):
    ab_case(stim, ab, model, None)


@pytest.mark.parametrize("model", AB_MODELS)
def test_ab_seven_streams(built, stim, ab, model):
    # 7 rows pairs: not a multiple of rows per warp x warps per block for any decoder kernel
    ab_case(stim, ab, model, 4096, n_streams=7)


@pytest.mark.parametrize("model,env", [(M0, {"AISGPU_DECODER": "1"}), (M2, {"AISGPU_DECODER": "1"})] +
                         [(m, {"AISGPU_DEC_RPW": r}) for m in (M0, M2) for r in ("1", "3", "6")] +
                         [(M4, {"AISGPU_DEC_RPW": r}) for r in ("1", "3")])
def test_ab_kernel_variants(built, stim, ab, model, env, monkeypatch):
    ab_case(stim, ab, model, 4096, env=env, monkeypatch=monkeypatch)


@pytest.mark.parametrize("model", [M0, M2, M4, M11])
def test_mode_x(built, stim, model):
    fs = 48000
    xs = stim.render_x(fs)  # 2 B streams: the A tracks, then the B tracks
    lengths = lengths_of(xs.shape[1], 4096)
    want = ref_frames("x", model, fs, xs, lengths)
    label = "X mode, model %d" % model
    got = run_engine(xs, lengths, model=model, sample_rate=fs, channel_mode=aisgpu.MODE_X, channels="XX")
    check(got, want, label)
    seen = check_predicted(stim, got, label, "X", lambda s, ch: (s % B, "AB"[s // B]))
    DL.assert_boundaries(stim.designs, seen, label)


def test_discriminator(built, stim):
    fs = 48000
    xs = stim.render_disc(fs)
    lengths = lengths_of(xs.shape[1], 4096)
    want = ref_frames("disc", M3, fs, xs, lengths)
    label = "model 3"
    got = run_engine(xs, lengths, model=M3, sample_rate=fs, fmt=aisgpu.FMT_CF32)
    check(got, want, label)
    seen = check_predicted(stim, got, label, "AB", lambda s, ch: (s, ch))
    DL.assert_boundaries(stim.designs, seen, label)


@pytest.mark.parametrize("model", [M4, M11])
def test_bench_shape(built, model):
    """batch 1024 x 131072 @1536 kS/s, three submits back to back from device memory: stream b = unique stream b % 16 of the ties
    and their neighbours (two start offsets each) plus its own noise; 32 sampled streams against the reference."""
    import torch
    fs, Bn, N, K, U16, NS = 1536000, 1024, 131072, 3, 16, 32
    st = DL.Stimulus(DL.tie_designs(), U16, offsets=(0, 16))
    uniq = st.render_ab(fs, quantum=K * N)
    assert uniq.shape[1] == K * N
    dev = torch.device("cuda", 0)
    ud = torch.view_as_complex(torch.from_numpy(uniq.view(np.float32)).to(dev).view(U16, K * N, 2))
    x = torch.empty((K, Bn, N), dtype=torch.complex64, device=dev)
    for b0 in range(0, Bn, U16):
        x[:, b0:b0 + U16, :] = ud.view(U16, K, N).permute(1, 0, 2)
    g = torch.Generator(device=dev)
    g.manual_seed(model)
    noise = torch.empty((Bn, N), dtype=torch.complex64, device=dev)
    for c in range(K):
        torch.view_as_real(noise).normal_(0.0, 0.005, generator=g)
        x[c] += noise
    torch.cuda.synchronize()
    eng = aisgpu.Engine(model=model, sample_rate=fs, n_streams=Bn, max_chunk=N, max_frames=1 << 19, host_staging=False)
    for c in range(K):
        eng.submit_device(x[c].data_ptr(), N, N)
    msgs = eng.poll()
    cnt = eng.counters()
    eng.close()
    assert eng.overflows == 0 and cnt[4] == 0, cnt
    ids = sorted(int(s) for s in np.random.default_rng(model).choice(Bn, size=NS, replace=False))
    host = x.index_select(1, torch.tensor(ids, device=dev)).cpu().numpy()  # [K][NS][N]
    del x, ud
    torch.cuda.empty_cache()
    xs = np.stack([np.ascontiguousarray(host[:, j, :]).reshape(-1) for j in range(NS)])
    want = run_refs(lambda: O.RefModel(model=model, sample_rate=fs), xs, [N] * K)
    got = [[m for m in msgs if m.stream == s] for s in ids]
    label = "model %d at batch 1024 x 131072 @1536 kS/s" % model
    check(got, want, label)
    check_predicted(st, got, label, "AB", lambda j, ch: (ids[j] % U16, ch))
    assert len(msgs) == sum(len(st.expected(b % U16, ch)) for b in range(Bn) for ch in "AB")
