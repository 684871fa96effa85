"""-m gpu: aisgpu_feed_wav_files (WAV recordings, read as the reference's Device::WAVFile reads them) at tolerance 0: frames, the
order in which the callback receives them and the counters against the unmodified reference pushed the same bytes in the same
blocks (the last one zero-padded as the feeder pads it), equality with aisgpu_feed_files on the same samples, the channel dump read
back in single-channel mode, and the refusals."""
import numpy as np
import pytest

import aisgpu
import aissynth as S
import disc_util as D
import mode_x_util as X
import oracle as O
import oracle_disc as OD
import oracle_x as OX
import parity_util as U
import wav_util as W

pytestmark = pytest.mark.gpu

CF32, CU8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS16
BPS = {CF32: 8, CU8: 2, CS16: 4}
BEFORE = [(), (W.chunk(b"LIST", b"INFOISFT" + b"\x06\0\0\0" + b"SDR#\0\0"),), (W.chunk(b"JUNK", bytes(27)),)]


def _raw(kind, fs, n, seed, fmt):
    if kind == "x":
        return X.stream_input(fs, n, seed, fmt)[0]
    if kind == "disc":
        return D.stream_input(fs, n, seed, fmt)[0]
    return X.to_raw(S.random_stream(fs, n, seed, bursts_per_sec=(10, 20))[0], fmt)[0]


def _ref(kind, model, fs, fmt):
    if kind == "x":
        if not OX.have_refx():
            pytest.skip("reference harness (mode X) not built")
        return OX.RefModelX(model=model, sample_rate=fs, fmt=fmt)
    if kind == "disc":
        if not OD.have_refd():
            pytest.skip("reference harness (model 3) not built")
        return OD.RefModelDisc(sample_rate=fs, fmt=fmt)
    if not O.have_ref():
        pytest.skip("reference harness not built")
    return O.RefModel(model=model, sample_rate=fs, fmt=fmt)


def _ref_frames(kind, model, fs, fmt, datas, N, nblocks):
    """The reference over each stream's sample bytes in blocks of N samples, zero-padded to nblocks blocks: the frames in the order
    the feeder's callback delivers them (per block, stream-major), with their block."""
    per_stream = []
    for d in datas:
        ref = _ref(kind, model, fs, fmt)
        pad = np.zeros(nblocks * N * BPS[fmt], np.uint8)
        pad[:len(d)] = np.frombuffer(d, np.uint8)
        blocks = []
        for c in range(nblocks):
            ref.push(pad[c * N * BPS[fmt]:(c + 1) * N * BPS[fmt]])
            blocks.append([U.frame_key(m) for m in ref.messages()])
        ref.close()
        per_stream.append(blocks)
    return [(s, c) + k for c in range(nblocks) for s in range(len(datas)) for k in per_stream[s][c]]


def _have(got):
    return [(m.stream, m.chunk) + U.frame_key(m) for m in got]


CASES = [("ab", m, 1536000, f, 65536) for f in (CS16, CU8, CF32) for m in (aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD, aisgpu.MODEL_V2)]
CASES += [("ab", aisgpu.MODEL_DEFAULT, 6000000, CS16, None), ("x", aisgpu.MODEL_DEFAULT, 48000, CU8, 8192),
          ("disc", 3, 48000, CS16, 4096), ("disc", 3, 44100, CS16, 4096), ("disc", 3, 44100, CF32, 4096)]


@pytest.mark.parametrize("kind,model,fs,fmt,N", CASES, ids=lambda v: str(v))
def test_matches_reference(built, tmp_path, kind, model, fs, fmt, N):
    mode = aisgpu.MODE_X if kind == "x" else aisgpu.MODE_AB
    if N is None:  # an interpolated rate: every block has the same length, a multiple of the granule
        N = aisgpu.chunk_granule(fs, model, fmt=fmt) * 1024
    n_blk = 5 if kind == "ab" else 12
    lens = [N * n_blk, N * (n_blk - 2) + 333, N * 2 - 1]  # files of unequal length; tails that do not fill a block
    paths, datas = [], []
    for s, n in enumerate(lens):
        d = np.ascontiguousarray(_raw(kind, fs, N * n_blk, 40 + s, fmt)).tobytes()[:n * BPS[fmt]]
        p = str(tmp_path / ("s%d.wav" % s))
        W.write_wav(p, d, fmt, fs, before=BEFORE[s])
        paths.append(p)
        datas.append(d)
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=3, max_chunk=N, channel_mode=mode,
                        channels="XX" if kind == "x" else "AB")
    got, nb = eng.feed_wav_files(paths, N)
    c = eng.counters()
    eng.close()
    assert nb == n_blk
    want = _ref_frames(kind, model, fs, fmt, datas, N, nb)
    assert len(want) > 0
    assert _have(got) == want
    assert c[1] == len(want) and c[3] == nb and c[2] == nb * N and c[4] == 0
    assert c[5] == sum(w[2][0] == ("X" if kind == "x" else "A") for w in want) and c[5] + c[6] == c[1]


def test_equals_raw_feeder(built, tmp_path):
    fs, N, fmt = 1536000, 32768, CU8
    lens = [N * 6 + 100, N * 4]
    raws, wavs, tails = [], [], []
    for s, n in enumerate(lens):
        d = S.to_cu8(S.random_stream(fs, n, 60 + s, bursts_per_sec=(10, 20))[0]).tobytes()
        r, w, t = tmp_path / ("r%d.cu8" % s), tmp_path / ("w%d.wav" % s), tmp_path / ("t%d.wav" % s)
        r.write_bytes(d)
        W.write_wav(str(w), d, fmt, fs, before=BEFORE[s + 1])
        # a LIST chunk after the data chunk is read as samples, as the reference reads it: the same as a raw file that ends in it
        lst = W.chunk(b"LIST", b"INFOICMT" + bytes([20, 0, 0, 0]) + b"recorded by HDSDR\0\0\0")
        W.write_wav(str(t), d, fmt, fs, after=(lst,))
        (tmp_path / ("rt%d.cu8" % s)).write_bytes(d + lst)
        raws.append(str(r))
        wavs.append(str(w))
        tails.append((str(t), str(tmp_path / ("rt%d.cu8" % s))))

    def run(feed, paths):
        eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=fmt, n_streams=2, max_chunk=N)
        got, nb = getattr(eng, feed)(paths, N)
        c = eng.counters()
        eng.close()
        return _have(got), nb, c

    a, b = run("feed_files", raws), run("feed_wav_files", wavs)
    assert len(a[0]) > 0 and a == b
    assert run("feed_files", [t[1] for t in tails]) == run("feed_wav_files", [t[0] for t in tails])


def test_dump_round_trip(built, tmp_path):
    """The engine's channel dump, decoded again by a mode-X engine at 48 kHz, gives the frames of the reference's ModelDefault in
    mode X on the same WAV files."""
    fs, N = 1536000, 65536
    x = S.random_stream(fs, N * 8, 77, bursts_per_sec=(10, 20))[0]
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=CF32, n_streams=1, max_chunk=N)
    eng.dump_open([str(tmp_path / "d")])
    for c in range(8):
        eng.submit(x[c * N:(c + 1) * N], N)
        eng.poll()
    eng.dump_close()
    eng.close()
    paths = [str(tmp_path / "d_A.wav"), str(tmp_path / "d_B.wav")]
    for p in paths:
        assert aisgpu.wav_probe(p) == (CF32, 48000, 44)
    M = 2048
    ex = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=48000, fmt=CF32, n_streams=2, max_chunk=M, channel_mode=aisgpu.MODE_X,
                       channels="XX")
    got, nb = ex.feed_wav_files(paths, M)
    ex.close()
    datas = [open(p, "rb").read()[44:] for p in paths]
    assert nb == -(-max(len(d) for d in datas) // (8 * M))
    want = _ref_frames("x", aisgpu.MODEL_DEFAULT, 48000, CF32, datas, M, nb)
    assert len(want) > 0 and _have(got) == want


def test_refusals(built, tmp_path):
    fs, N = 1536000, 4096
    good, other_rate, other_fmt = tmp_path / "g.wav", tmp_path / "r.wav", tmp_path / "f.wav"
    W.write_wav(str(good), bytes(4 * N * 3), CS16, fs)
    W.write_wav(str(other_rate), bytes(4 * N * 3), CS16, 1536001)
    W.write_wav(str(other_fmt), bytes(2 * N * 3), CU8, fs)
    mono = tmp_path / "m.wav"
    mono.write_bytes(W.riff(W.fmt_chunk(1, 1, fs, 16), W.chunk(b"data", bytes(64))))
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=CS16, n_streams=2, max_chunk=N)
    for bad, text in [(other_rate, "sample rate 1536001 differs from the engine's 1536000"),
                      (other_fmt, "format CU8 differs from the engine's CS16"),
                      (mono, "WAV-file must have 2 channels (I/Q)."),
                      (tmp_path / "missing.wav", "cannot open WAV file")]:
        with pytest.raises(aisgpu.AisGpuError) as e:
            eng.feed_wav_files([str(good), str(bad)], N)
        assert str(bad) in str(e.value) and text in str(e.value)
    assert eng.counters()[3] == 0  # refused before anything was submitted
    with pytest.raises(aisgpu.AisGpuError, match="bad argument"):
        eng.feed_wav_files([str(good), str(good)], N + 2)
    got, nb = eng.feed_wav_files([str(good), str(good)], N)
    assert nb == 3 and got == []
    eng.close()
    # a WAV never maps to F32_FS4 or CS8
    for fmt in (aisgpu.FMT_F32_FS4, aisgpu.FMT_CS8):
        e2 = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=fmt, n_streams=1, max_chunk=N)
        with pytest.raises(aisgpu.AisGpuError, match="format CS16 differs from the engine's"):
            e2.feed_wav_files([str(good)], N)
        e2.close()
    # an engine group is refused, the leader as well as its member
    lead = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=CS16, n_streams=1, max_chunk=N)
    mem = lead.attach(model=aisgpu.MODEL_STANDARD)
    for e3 in (lead, mem):
        with pytest.raises(aisgpu.AisGpuError, match="not available for an engine group"):
            e3.feed_wav_files([str(good)], N)
    mem.close()
    lead.close()
