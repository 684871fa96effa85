"""-m gpu: the 12-byte input format DC16H (Convert::toFloat, Utilities/Convert.cpp:288-301) through the C ABI, bit for bit
(tolerance 0) against the unmodified reference fed the same words as Format::DC16H (oracle/_ref).

Every front end reads the format: the streaming kernel (768 kS/s and up), the tiled kernel (below, and odd block shapes), the
pre-stage's CIC stage and DownsampleKFilter, single-channel mode and the FM-discriminator split.  A sample is three 32-bit words of
which two half-words are read, so what is checked here beyond the other formats' tests is every place a byte offset is formed from
a sample index (lane starts, chunk thirds, padded rows, carried history), that the unread bits stay unread (tests/dc16h_util.py fills
them with garbage) and the integer negation of Q (Q = 0 gives +0.0, Q = -32768 gives 1.0)."""
import os
import subprocess

import numpy as np
import pytest

import aisgpu
import aissynth as S
import dc16h_util as DC
import disc_util as D
import mode_x_util as X
import oracle as O
import oracle_dc16h as ODC
import parity_util as U
import test_gpu_submit_shapes as SH

pytestmark = pytest.mark.gpu

DC16H, CS16 = DC.DC16H, aisgpu.FMT_CS16
AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
M0, M1, M2, M3, M4, M11 = SH.M0, SH.M1, SH.M2, SH.M3, SH.M4, SH.M11
B = SH.B
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "adapter_dc16h_test")
needs_ref = pytest.mark.skipif(not ODC.have_ref(), reason="DC16H is checked against the compiled reference only")


class Fam(SH.Fam):
    """An engine configuration of test_gpu_submit_shapes.py reading DC16H: the same schedules, placements and comparisons."""

    def __init__(self, name, model, fs, mode=AB, dsk=False, ps_ema=True):
        super().__init__(name, model, fs, DC16H, mode, dsk, False, ps_ema)

    def reference(self):
        kind = "disc" if self.model == M3 else ("x" if self.mode == MX else "ab")
        if not ODC.have_ref(kind):
            pytest.skip("DC16H is checked against the compiled reference only")
        return ODC.RefModelDC16H(model=self.model, sample_rate=self.fs, flags=self.flags(), taps=True, kind=kind)

    def inputs(self, n, seed):
        if self.model == M3:
            zs = [D.stereo(self.fs, n, seed + s) for s in range(B)]
        elif self.mode == MX:
            zs = [X.stream_input(self.fs, n, seed + s, O.FMT_CF32)[0] for s in range(B)]
        else:
            zs = [S.random_stream(self.fs, n, seed + s, bursts_per_sec=(6, 12))[0] for s in range(B)]
        return [DC.from_complex(z, seed + s) for s, z in enumerate(zs)]


@pytest.fixture(autouse=True)
def _dc16h_bytes_per_sample(monkeypatch):
    monkeypatch.setitem(SH.BPS, DC16H, 12)


# ---- every model at 1536 kS/s: every tap of every submit, a changing submit length, the four entry points, polls skipped ----

MODELS = [Fam("st1536_standard", M0, 1536000), Fam("st1536_base", M1, 1536000), Fam("st1536_default", M2, 1536000),
          Fam("st1536_default_noema", M2, 1536000, ps_ema=False), Fam("st1536_challenger", M4, 1536000), Fam("st1536_v2", M11, 1536000)]


@pytest.mark.parametrize("fam", MODELS, ids=lambda f: f.name)
def test_models_1536k(built, fam):
    assert SH.run_schedule(fam, SH.random_schedule(fam, 2000 + len(fam.name)), seed=7) >= 1


SCHEDULES = [(Fam("st1536_default", M2, 1536000), k) for k in SH.ALL if k != "random"] + \
            [(Fam("tiled384_standard", M0, 384000), k) for k in ("tiled_streaming_switch", "granule_x40", "random")] + \
            [(Fam("dsk288_default", M2, 288000), k) for k in ("granule_x40", "random")] + \
            [(Fam("x96_default", M2, 96000, mode=MX), k) for k in ("granule_x40", "random")] + \
            [(Fam("disc48", M3, 48000), k) for k in ("granule_x40", "random")]


@pytest.mark.parametrize("fam,kind", SCHEDULES, ids=["%s-%s" % (f.name, k) for f, k in SCHEDULES])
def test_length_schedule(built, fam, kind):
    sched = SH.random_schedule(fam, 3000 + len(fam.name)) if kind == "random" else SH.fixed_schedules(fam.granule())[kind]
    SH.run_schedule(fam, sched, seed=9)


# ---- the other rate buckets: the streaming kernel's K = 3, 5, 6, 7, an interpolated rate, a DSK bucket behind a CIC stage ----

RATES = [(192000, False, 8192), (768000, False, 32768), (3072000, False, 65536), (6144000, False, 131072), (12288000, False, 262144),
         (1152000, True, 49152), (1000000, False, 32768), (6000000, False, 65536)]


@pytest.mark.parametrize("fs,dsk,N", RATES, ids=["%dk%s" % (r // 1000, "_dsk" if d else "") for r, d, _ in RATES])
def test_rate_buckets(built, fs, dsk, N):
    SH.run_schedule(Fam("r%d" % fs, M2, fs, dsk=dsk), [N] * 5, seed=11)


SINGLE = [Fam("x48_default", M2, 48000, mode=MX), Fam("x192_default", M2, 192000, mode=MX), Fam("x24_default", M2, 24000, mode=MX),
          Fam("disc441", M3, 44100)]


@pytest.mark.parametrize("fam", SINGLE, ids=lambda f: f.name)
def test_mode_x_and_discriminator(built, fam):
    N = {48000: 4096, 192000: 16384, 24000: 2048, 44100: 4416}[fam.fs]
    SH.run_schedule(fam, [N] * 6, seed=13)


# ---- forced lane splits of the streaming front end ----

@pytest.mark.parametrize("lanes", ["1", "3", "7", "18", "33", "100"])
def test_streaming_lane_split(built, monkeypatch, lanes):
    """L lanes per stream, L not dividing the block (uneven q / q + 1 split): every lane's byte offset is a whole number of
    16-byte pieces although a sample is 12 bytes."""
    monkeypatch.setenv("AISGPU_ST_L", lanes)
    SH.run_schedule(Fam("st1536_standard", M0, 1536000), [64 * 1017] * 3, seed=41)


@pytest.mark.parametrize("fs,N", [(768000, 32 * 999), (3072000, 128 * 613)])
def test_streaming_lane_split_rates(built, monkeypatch, fs, N):
    for lanes in ("5", "19"):
        monkeypatch.setenv("AISGPU_ST_L", lanes)
        SH.run_schedule(Fam("st%d" % fs, M2, fs), [N] * 3, seed=43)


# ---- device batches ----

PLACED = [(Fam("st1536_default", M2, 1536000), 16384), (Fam("tiled384_standard", M0, 384000), 4096), (Fam("us6000_default", M2, 6000000), 65536),
          (Fam("dsk288_default", M2, 288000), 12288), (Fam("x96_default", M2, 96000, mode=MX), 8192), (Fam("disc48", M3, 48000), 4096)]


@pytest.mark.parametrize("fam,N", PLACED, ids=[f.name for f, _ in PLACED])
def test_device_batch_placement(built, fam, N):
    """Strides N, N + 4, N + 8, N + 64, 3N and a 16-byte offset base (the rule turns N + 2 and N + 6 into the next multiple of 4)
    against the reference and against a packed aisgpu_submit."""
    plan = SH.placements(fam, N, 1 << 20)
    assert {off for _, off in plan} == {0, 16} and all(st % 4 == 0 for st, _ in plan) and (N + 4, 16) in plan
    SH.test_device_batch_placement(built, fam, N)


@pytest.mark.parametrize("fam,N", PLACED[:2] + PLACED[4:], ids=[f.name for f, _ in PLACED[:2] + PLACED[4:]])
def test_refused_placements_leave_engine_untouched(built, fam, N):
    """A base aligned to 4, 8, 12 or 24 bytes (one and two samples are not enough) and strides N + 2, N + 6 are refused."""
    SH.test_refused_placements_leave_engine_untouched(built, fam, N, [(4, 0), (8, 0), (12, 0), (24, 0), (0, 2), (0, 6), (16, 2)])


# ---- values: Q = 0 (+0.0, not -0.0), Q = -32768 (1.0), I = -32768 (-1.0), silence, beside ordinary traffic; through atan2f ----

@needs_ref
@pytest.mark.parametrize("model", [M0, M2])
def test_special_values_every_tap(built, model):
    fs, N, nb, n_streams = 1536000, 16384, 3, 33
    rows = []
    for s in range(n_streams):
        i, q = DC.iq_of(S.random_stream(fs, N * nb, 600 + s, bursts_per_sec=(6, 12))[0])
        kind = s % 7
        if kind == 0:
            i[:], q[:] = 0, 0                     # digital silence
        elif kind == 1:
            q[:] = 0                              # all-zero Q: the imaginary part is +0.0 everywhere
        elif kind == 2:
            q[N // 2:N + 777] = -32768            # a run of Q = -32768 across a submit boundary: exactly 1.0
        elif kind == 3:
            i[N - 500:2 * N + 64] = -32768        # -1.0
            q[N - 500:2 * N + 64] = 0
        elif kind == 4:
            q[::3] = 0                            # zeros between live samples
            i[1::5] = 0
        elif kind == 5:
            i[:], q[:] = -32768, -32768           # (-1.0, 1.0) throughout
        rows.append(DC.pack_iq(i, q, 900 + s))
    refs = [ODC.RefModelDC16H(model=model, sample_rate=fs, taps=True) for _ in range(n_streams)]
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=DC16H, n_streams=n_streams, max_chunk=N, taps=True)
    problems, got, want = [], [[] for _ in rows], [[] for _ in rows]
    for c in range(nb):
        eng.submit(np.stack([r[c * N * 3:(c + 1) * N * 3] for r in rows]), N)
        for s in range(n_streams):
            refs[s].push(rows[s][c * N * 3:(c + 1) * N * 3])
            problems += U.compare_taps(eng, s, refs[s], model, "submit %d kind %d" % (c, s % 7))
            want[s] += refs[s].messages()
        for m in eng.poll():
            got[m.stream].append(m)
    eng.close()
    problems += U.compare_frames(got, want)
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)


# ---- the same I and Q sent as CS16 with Q negated on the host (needs no reference) ----

@pytest.mark.parametrize("fs,N,mode", [(1536000, 65536, AB), (384000, 16384, AB), (1000000, 32768, AB), (96000, 8192, MX)])
def test_equals_cs16_engine_fed_negated_q(built, fs, N, mode):
    z = S.random_stream(fs, 5 * N, 71, bursts_per_sec=(6, 12))[0] if mode == AB else X.stream_input(fs, 5 * N, 71, O.FMT_CF32)[0]
    w = DC.from_complex(z, 71)[0]
    w2 = DC.from_complex(z[::-1], 72)[0]
    kw = dict(model=M0, sample_rate=fs, n_streams=2, max_chunk=N, taps=True, channel_mode=mode, channels="XX" if mode == MX else "AB")
    a, b = aisgpu.Engine(fmt=DC16H, **kw), aisgpu.Engine(fmt=CS16, **kw)
    fa, fb = [], []
    for c in range(5):
        blk, blk2 = w[c * N * 3:(c + 1) * N * 3], w2[c * N * 3:(c + 1) * N * 3]
        a.submit(np.stack([blk, blk2]), N)
        b.submit(np.stack([DC.to_cs16(blk), DC.to_cs16(blk2)]), N)
        for s in range(2):
            for ch in ((0,) if mode == MX else (0, 1)):
                assert U.bits_equal(a.tap(aisgpu.TAP_C, s, ch), b.tap(aisgpu.TAP_C, s, ch)), (c, s, ch)
        fa += [(m.stream,) + U.frame_key(m) for m in a.poll()]
        fb += [(m.stream,) + U.frame_key(m) for m in b.poll()]
    a.close()
    b.close()
    assert fa == fb and len(fa) >= 1


# ---- feeder, groups ----

@needs_ref
def test_feed_files_ragged(built, tmp_path):
    fs, N, n_streams = 1536000, 32768, 5
    lengths = [N * 7 * 3 + 1000, N * 9 * 3, N * 3 * 3 + 17, 1, N * 9 * 3 - 1]  # words: whole blocks, partial tails, a one-word recording
    paths, raws = [], []
    for s in range(n_streams):
        w = DC.from_complex(S.random_stream(fs, N * 9, 7700 + s)[0], s)[0][:lengths[s]]
        p = tmp_path / ("rec%d.dc16h" % s)
        w.tofile(p)
        paths.append(str(p))
        raws.append(w)
    eng = aisgpu.Engine(model=M2, sample_rate=fs, fmt=DC16H, n_streams=n_streams, max_chunk=N)
    got, nblocks = eng.feed_files(paths, N)
    assert nblocks == 9
    total = 0
    for s in range(n_streams):
        padded = np.zeros(nblocks * N * 3, dtype=np.uint32)  # RAWFile zero-fills the tail of its last block: samples (+0, +0)
        padded[:len(raws[s])] = raws[s]
        ref = ODC.RefModelDC16H(model=M2, sample_rate=fs)
        for c in range(nblocks):
            ref.push(padded[c * N * 3:(c + 1) * N * 3])
        want = [U.frame_key(m) for m in ref.messages()]
        assert [U.frame_key(m) for m in got if m.stream == s] == want, "stream %d" % s
        total += len(want)
    assert total >= 5 and eng.counters()[2] == nblocks * N
    eng.close()


def test_group_on_dc16h_leader(built):
    fs, N, nb = 1536000, 32768, 5
    rows = [DC.from_complex(S.random_stream(fs, N * nb, 800 + s, bursts_per_sec=(6, 12))[0], s)[0] for s in range(B)]
    kinds = [M2, M0]
    kw = dict(sample_rate=fs, fmt=DC16H, n_streams=B, max_chunk=N)
    lead = aisgpu.Engine(model=kinds[0], **kw)
    group = [lead] + [lead.attach(model=k) for k in kinds[1:]]
    alone = [aisgpu.Engine(model=k, **kw) for k in kinds]
    for c in range(nb):
        batch = np.stack([r[c * N * 3:(c + 1) * N * 3] for r in rows])
        lead.submit(batch, N)
        for e in alone:
            e.submit(batch, N)
    for g, e, k in zip(group, alone, kinds):
        have = [(m.stream, m.chunk) + U.frame_key(m) for m in g.poll()]
        want = [(m.stream, m.chunk) + U.frame_key(m) for m in e.poll()]
        assert have == want and len(want) >= 1, "model %d" % k
    for e in group[1:] + [lead] + alone:
        e.close()


# ---- the adapter inside the reference's block graph ----

@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/adapter_dc16h_test not built")
@pytest.mark.parametrize("fs,block,model,odd", [(1536000, 65536, 2, False), (1536000, 65536, 2, True), (384000, 16384, 0, True),
                                                (1000000, 32768, 2, True)])
def test_adapter_equals_reference_model_in_same_binary(built, tmp_path, fs, block, model, odd):
    """AIS::ModelGPU against the reference's own model behind the same device on Format::DC16H buffers; odd: every second buffer
    carries one or two words beyond a whole sample, which ConvertRAW drops."""
    f = str(tmp_path / "x.dc16h")
    DC.from_complex(S.random_stream(fs, block * 8 + 64, 77, bursts_per_sec=(20, 30))[0], 77)[0].tofile(f)
    args = [EXE, f, str(fs), str(block), str(model)] + (["odd"] if odd else [])
    gpu = subprocess.run(args, capture_output=True)
    assert gpu.returncode == 0, gpu.stderr
    cpu = subprocess.run(args + ["cpu"], capture_output=True)
    assert cpu.returncode == 0 and gpu.stdout == cpu.stdout and len(cpu.stdout.splitlines()) >= 1
