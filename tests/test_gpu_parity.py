"""-m gpu parity tests: the CUDA path (through the C ABI) against the oracle, bit for bit.

Oracle = oracle/_ref/libaisref.so (the unmodified reference, strict IEEE flags) when it was built, else the
pinned C restatement oracle/libaisoracle.so.  Integer/byte outputs (frames, NMEA) and -- because every kernel
replays the reference's operation order -- all float taps are required to be BIT-IDENTICAL (tolerance 0);
the north_star tolerance for floats (1e-5 rel) is therefore met with margin.
"""
import numpy as np
import pytest

import aisgpu
import aissynth as S
import oracle as O
import parity_util as U

pytestmark = pytest.mark.gpu


def oracle_model(**kw):
    return (O.RefModel if O.have_ref() else O.PortModel)(**kw)


def bits_equal(a, b):
    a = np.ascontiguousarray(a)
    b = np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def first_diff(a, b):
    n = min(len(a), len(b))
    av = a[:n].view(np.uint32).reshape(n, -1)
    bv = b[:n].view(np.uint32).reshape(n, -1)
    d = np.nonzero((av != bv).any(axis=1))[0]
    return (int(d[0]), int(len(d))) if len(d) else (-1, 0)


def run_case(built, model, fs, N, nchunks, B, ps_ema=True, afc_wide=True, droop=True, fmt=aisgpu.FMT_CF32, check_taps=True, seed0=0, dsk=False,
             fp_ds=False):
    xs = [S.random_stream(fs, N * nchunks, seed0 + s)[0] for s in range(B)]
    if fmt == aisgpu.FMT_CU8:
        raw = [S.to_cu8(x) for x in xs]
        per = 2
    elif fmt == aisgpu.FMT_CS8:
        raw = [(S.to_cu8(x).astype(np.int16) - 128).astype(np.int8) for x in xs]
        per = 2
    elif fmt == aisgpu.FMT_CS16:
        raw = []
        for x in xs:
            v = np.empty(2 * len(x), dtype=np.float32)
            v[0::2], v[1::2] = x.real, x.imag
            raw.append(np.clip(np.round(v * 32767.0), -32768, 32767).astype(np.int16))
        per = 2
    else:
        raw = xs
        per = 1
    flags = (O.FLAG_PS_EMA if ps_ema else 0) | (O.FLAG_AFC_WIDE if afc_wide else 0) | (O.FLAG_DROOP if droop else 0)
    flags |= (O.FLAG_DSK if dsk else 0) | (O.FLAG_FP_DS if fp_ds else 0)
    if (dsk or fp_ds) and not O.have_ref():
        pytest.skip("-go DSK / FP_DS are checked against the compiled reference only")
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N, ps_ema=ps_ema, afc_wide=afc_wide,
                        droop=droop, taps=check_taps, dsk=dsk, fp_ds=fp_ds)
    refs = [oracle_model(model=model, sample_rate=fs, fmt=fmt, flags=flags, taps=True) for _ in range(B)]
    problems = []
    got_msgs = [[] for _ in range(B)]
    want_msgs = [[] for _ in range(B)]
    for c in range(nchunks):
        batch = np.stack([r[c * N * per:(c + 1) * N * per] for r in raw])
        eng.submit(batch, N)
        for s in range(B):
            refs[s].push(raw[s][c * N * per:(c + 1) * N * per])
        if check_taps:
            for s in range(B):
                for ch in range(2):
                    want = refs[s].tap_c(O.TAP_CA + ch)
                    got = eng.tap(aisgpu.TAP_C, s, ch)
                    if not bits_equal(got, want):
                        problems.append(("C", c, s, ch, len(got), len(want)) + first_diff(got, want))
                    if model == aisgpu.MODEL_DEFAULT:
                        want = refs[s].tap_c(O.TAP_CGF_A + ch)
                        got = eng.tap(aisgpu.TAP_CGF, s, ch)
                        if not bits_equal(got, want):
                            problems.append(("CGF", c, s, ch, len(got), len(want)) + first_diff(got, want))
                        want = refs[s].tap_c(O.TAP_FC_A + ch)
                        got = eng.tap(aisgpu.TAP_FIR, s, ch)
                        if not bits_equal(got, want):
                            problems.append(("FIR17", c, s, ch, len(got), len(want)) + first_diff(got, want))
                    else:
                        want = refs[s].tap_f(O.TAP_FM_A + ch)
                        got = eng.tap(aisgpu.TAP_FM, s, ch, dtype=np.float32)
                        if not bits_equal(got, want):
                            problems.append(("FM", c, s, ch, len(got), len(want)) + first_diff(got, want))
                        want = refs[s].tap_f(O.TAP_FR_A + ch)
                        got = eng.tap(aisgpu.TAP_FIR, s, ch, dtype=np.float32)
                        if not bits_equal(got, want):
                            problems.append(("FIR37", c, s, ch, len(got), len(want)) + first_diff(got, want))
                    nph = 1 if model == aisgpu.MODEL_BASE else 5
                    for ph in range(nph):
                        want = refs[s].tap_f(ch * 5 + ph)
                        got = eng.tap(aisgpu.TAP_DEC, s, ch + 2 * ph, dtype=np.float32)
                        if not bits_equal(got, want):
                            problems.append(("DEC", c, s, ch, ph, len(got), len(want)) + first_diff(got, want))
            if c == 0:
                rot_w = None  # the oracle does not expose the phasor; C taps cover it
        for m in eng.poll():
            got_msgs[m.stream].append(m)
        for s in range(B):
            want_msgs[s] += refs[s].messages()
    nmsg = 0
    for s in range(B):
        g = [(m.key(), m.start_idx, m.end_idx) for m in got_msgs[s]]
        w = [(m.key(), m.start_idx, m.end_idx) for m in want_msgs[s]]
        nmsg += len(w)
        if g != w:
            problems.append(("MSG", s, len(g), len(w), [x for x in g if x not in w][:2], [x for x in w if x not in g][:2]))
        else:
            for a, b in zip(got_msgs[s], want_msgs[s]):
                if np.float32(a.level).view(np.uint32) != np.float32(b.level).view(np.uint32) or \
                        np.float32(a.ppm).view(np.uint32) != np.float32(b.ppm).view(np.uint32):
                    problems.append(("TAG", s, a.level, b.level, a.ppm, b.ppm))
    eng.close()
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    return nmsg


def test_default_1536k(built):
    n = run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 65536, 4, 3)
    assert n >= 6


def test_standard_1536k(built):
    n = run_case(built, aisgpu.MODEL_STANDARD, 1536000, 65536, 4, 3)
    assert n >= 6


def test_base_1536k(built):
    run_case(built, aisgpu.MODEL_BASE, 1536000, 65536, 4, 3)


def test_default_small_chunks(built):
    # chunks smaller than a CGF block (48 kHz count 128 < 512): exercises the unconsumed-sample carry
    n = run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 4096, 48, 2, seed0=7)
    assert n >= 1


def test_standard_small_chunks(built):
    run_case(built, aisgpu.MODEL_STANDARD, 1536000, 4096, 48, 2, seed0=7)


def test_default_phasesearch(built):
    n = run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 32768, 8, 2, ps_ema=False, seed0=11)
    assert n >= 4


def test_default_narrow_nodroop(built):
    run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 32768, 8, 2, afc_wide=False, droop=False, seed0=13)


def test_default_cu8(built):
    n = run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 65536, 4, 2, fmt=aisgpu.FMT_CU8, seed0=17)
    assert n >= 4


@pytest.mark.parametrize("fs,N", [(96000, 4096), (192000, 8192), (384000, 16384), (768000, 32768), (3072000, 131072),
                                  (6144000, 262144), (12288000, 524288)])
def test_default_rates(built, fs, N):
    n = run_case(built, aisgpu.MODEL_DEFAULT, fs, N, 4, 2, seed0=23)
    assert n >= 2


@pytest.mark.parametrize("fs,N,model", [(288000, 12288, aisgpu.MODEL_DEFAULT), (288000, 49152, aisgpu.MODEL_STANDARD),
                                        (6000000, 262144, aisgpu.MODEL_DEFAULT), (6000000, 65536, aisgpu.MODEL_STANDARD),
                                        (2000000, 65536, aisgpu.MODEL_DEFAULT), (250000, 16384, aisgpu.MODEL_DEFAULT), (300000, 16384, aisgpu.MODEL_DEFAULT),
                                        (1000000, 32768, aisgpu.MODEL_BASE)])
def test_resampled_rates(built, fs, N, model):
    # DownsampleKFilter (/3, 288 kS/s) and Upsample (non-bucket rates; 6 MSPS is the AirSpy shape of BASELINE configs[2]).
    # The reference re-blocks behind the resampler, so per-submit taps do not line up; frames are compared bit for bit.
    n = run_case(built, model, fs, N, 6, 2, check_taps=False, seed0=29)
    assert n >= 2
    if O.have_ref():
        resampler_taps(fs, N, 6, model)


def resampler_taps(fs, N, nchunks, model, dsk=False):
    """The resampler outputs themselves (DSP::Upsample, DownsampleKFilter) against taps on the reference's US.out / DSK.out:
    the sample streams must be bit-identical (the reference emits whole blocks, so the common prefix is compared)."""
    x = S.random_stream(fs, N * nchunks, 91)[0]
    eng = aisgpu.Engine(model=model, sample_rate=fs, n_streams=1, max_chunk=N, taps=True, dsk=dsk)
    ref = O.RefModel(model=model, sample_rate=fs, flags=O.DEFAULT_FLAGS | (O.FLAG_DSK if dsk else 0), taps=True)
    got = {aisgpu.TAP_PRE: [], aisgpu.TAP_PRE2: []}
    want = {O.TAP_US: [], O.TAP_DSK: []}
    for c in range(nchunks):
        eng.submit(x[None, c * N:(c + 1) * N], N)
        ref.push(x[c * N:(c + 1) * N])
        for t in got:
            try:
                got[t].append(eng.tap(t))
            except aisgpu.AisGpuError:
                pass
        for t in want:
            want[t].append(ref.tap_c(t))
    eng.close()
    us, dsk_ = np.concatenate(want[O.TAP_US]), np.concatenate(want[O.TAP_DSK])
    pre = np.concatenate(got[aisgpu.TAP_PRE]) if got[aisgpu.TAP_PRE] else np.zeros(0, np.complex64)
    pre2 = np.concatenate(got[aisgpu.TAP_PRE2]) if got[aisgpu.TAP_PRE2] else np.zeros(0, np.complex64)
    pairs = []
    if len(us) and len(dsk_):
        pairs = [("US", pre, us), ("DSK", pre2, dsk_)]
    elif len(us):
        pairs = [("US", pre, us)]
    elif len(dsk_):
        pairs = [("DSK", pre, dsk_)]
    assert pairs, "no resampler at this rate"
    for name, g, w in pairs:
        n = min(len(g), len(w))
        assert n > 1000 and bits_equal(g[:n], w[:n]), "%s output differs: %r" % (name, first_diff(g[:n], w[:n]))


def test_resampled_cu8(built):
    n = run_case(built, aisgpu.MODEL_DEFAULT, 6000000, 262144, 3, 2, fmt=aisgpu.FMT_CU8, check_taps=False, seed0=31)
    assert n >= 2


@pytest.mark.parametrize("model", [aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD])
def test_pipelined_backend(built, model):
    # without taps the back-end stages of consecutive submits overlap on two streams (per-stage events, double-buffered
    # hand-off buffers): many short submits, frames only
    n = run_case(built, model, 1536000, 32768, 16, 4, check_taps=False, seed0=41)
    assert n >= 8


def test_pipelined_backend_tiny_chunks(built):
    # chunks below one CGF block: several submits share a 512-block, Ec / Cbuf leftovers hop between the streams
    run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 4096, 64, 2, check_taps=False, seed0=43)


@pytest.mark.parametrize("fmt", [aisgpu.FMT_CS8, aisgpu.FMT_CS16])
@pytest.mark.parametrize("fs,N", [(1536000, 65536), (384000, 16384)])
def test_signed_integer_formats(built, fmt, fs, N):
    # Convert::toFloat(CS8) / (CS16) (reference Utilities/Convert.cpp:266-286) through the streaming (1536k) and the tiled
    # (384k) front end
    n = run_case(built, aisgpu.MODEL_DEFAULT, fs, N, 3, 2, fmt=fmt, seed0=37)
    assert n >= 2


@pytest.mark.parametrize("fs,N,model", [(576000, 24576, aisgpu.MODEL_DEFAULT), (1152000, 49152, aisgpu.MODEL_STANDARD), (2304000, 98304, aisgpu.MODEL_DEFAULT),
                                        (500000, 16384, aisgpu.MODEL_DEFAULT), (1000000, 32768, aisgpu.MODEL_DEFAULT), (2000000, 65536, aisgpu.MODEL_STANDARD),
                                        (288000, 12288, aisgpu.MODEL_DEFAULT), (1536000, 65536, aisgpu.MODEL_DEFAULT)])
def test_dsk_buckets(built, fs, N, model):
    # -go DSK on (reference Model.cpp:130, 208-218, 248-258, 278-288): the 576K / 1152K / 2304K buckets = CIC stages ->
    # DownsampleKFilter /3, exact and interpolated (CIC -> Upsample -> /3); rates outside those buckets keep their chain
    n = run_case(built, model, fs, N, 6, 2, check_taps=False, seed0=51, dsk=True)
    assert n >= 2
    if fs != 1536000:
        resampler_taps(fs, N, 6, model, dsk=True)


def test_dsk_cu8(built):
    n = run_case(built, aisgpu.MODEL_DEFAULT, 1152000, 49152, 4, 2, fmt=aisgpu.FMT_CU8, check_taps=False, seed0=53, dsk=True)
    assert n >= 2


@pytest.mark.parametrize("model", [aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD])
def test_fp_ds_integer_frontend(built, model):
    # -go FP_DS on (Model.cpp:233-236; DSP.cpp:499-665): CU8 @1536K through four packed-uint16 CIC stages; the 48 kHz taps and
    # everything behind them are compared bit for bit
    n = run_case(built, model, 1536000, 65536, 4, 3, fmt=aisgpu.FMT_CU8, seed0=57, fp_ds=True)
    assert n >= 4


def test_fp_ds_small_blocks(built):
    # the shortest block the integer front end takes (32 lane sub-segments of 512 samples)
    run_case(built, aisgpu.MODEL_DEFAULT, 1536000, 16384, 12, 2, fmt=aisgpu.FMT_CU8, seed0=59, fp_ds=True)


def test_fp_ds_needs_cu8(built):
    with pytest.raises(aisgpu.AisGpuError, match="needs CU8"):
        aisgpu.Engine(sample_rate=1536000, fmt=aisgpu.FMT_CF32, fp_ds=True)


def run_v2_case(fs, N, nchunks, B, check_taps, seed0, fmt=aisgpu.FMT_CF32):
    """Model 11 "v2_base" (reference DSP/Decoder/V2/V2Engine.cpp, Model.cpp:440-460) against the compiled reference."""
    if not O.have_ref():
        pytest.skip("the V2 engine is checked against the compiled reference only")
    xs = [S.random_stream(fs, N * nchunks, seed0 + s, bursts_per_sec=(6, 12))[0] for s in range(B)]
    per = 1
    if fmt == aisgpu.FMT_CU8:
        xs = [S.to_cu8(x) for x in xs]
        per = 2
    N_el = N * per  # array elements per chunk
    eng = aisgpu.Engine(model=aisgpu.MODEL_V2, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N, taps=check_taps)
    refs = [O.RefModel(model=O.MODEL_V2, sample_rate=fs, fmt=fmt, taps=check_taps) for _ in range(B)]
    problems = []
    got = [[] for _ in range(B)]
    want = [[] for _ in range(B)]
    for c in range(nchunks):
        eng.submit(np.stack([x[c * N_el:(c + 1) * N_el] for x in xs]), N)
        for s in range(B):
            refs[s].push(xs[s][c * N_el:(c + 1) * N_el])
        if check_taps:
            for s in range(B):
                for ch in range(2):
                    for name, g, w in (("V2.CGF", eng.tap(aisgpu.TAP_CGF, s, ch), refs[s].tap_c(O.TAP_CGF_A + ch)),
                                       ("V2.FIR17", eng.tap(aisgpu.TAP_FIR, s, ch), refs[s].tap_c(O.TAP_FC_A + ch)),
                                       ("V2.FIR37", eng.tap(aisgpu.TAP_FM, s, ch, dtype=np.float32), refs[s].tap_f(O.TAP_FR_A + ch))):
                        if not bits_equal(g, w):
                            problems.append((name, c, s, ch, len(g), len(w)) + first_diff(g, w))
        for m in eng.poll():
            got[m.stream].append(m)
        for s in range(B):
            want[s] += refs[s].messages()
    n = 0
    for s in range(B):
        g = [(m.key(), m.start_idx, m.end_idx) for m in got[s]]
        w = [(m.key(), m.start_idx, m.end_idx) for m in want[s]]
        n += len(w)
        if g != w:
            problems.append(("MSG", s, len(g), len(w), [x for x in g if x not in w][:2], [x for x in w if x not in g][:2]))
        else:
            for a, b in zip(got[s], want[s]):
                if np.float32(a.level).view(np.uint32) != np.float32(b.level).view(np.uint32) or \
                        np.float32(a.ppm).view(np.uint32) != np.float32(b.ppm).view(np.uint32):
                    problems.append(("TAG", s, a.level, b.level, a.ppm, b.ppm))
    eng.close()
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    return n


def test_v2_engine_blockwise_taps(built):
    # one 512-sample block per submit: every block's derotated samples, FIR17 and FIR37 outputs are compared bit for bit
    n = run_v2_case(1536000, 16384, 40, 2, True, 61)
    assert n >= 4


@pytest.mark.parametrize("fs,N", [(1536000, 65536), (1536000, 36864), (384000, 16384), (6144000, 262144)])
def test_v2_engine_messages(built, fs, N):
    # several blocks per submit (and submits that are not whole blocks: 36864 / 32 = 1152 samples at 48 kHz)
    n = run_v2_case(fs, N, 8, 3, False, 67)
    assert n >= 6


def test_v2_engine_cu8(built):
    n = run_v2_case(1536000, 65536, 16, 2, False, 71, fmt=aisgpu.FMT_CU8)
    assert n >= 8


def run_msg_case(model, fs, N, nchunks, B, seed0, fmt=aisgpu.FMT_CF32, bursts=(6, 12)):
    """Frames + tags of a model the oracle has no taps for, against the compiled reference."""
    if not O.have_ref():
        pytest.skip("checked against the compiled reference only")
    xs = [S.random_stream(fs, N * nchunks, seed0 + s, bursts_per_sec=bursts)[0] for s in range(B)]
    eng = aisgpu.Engine(model=model, sample_rate=fs, fmt=fmt, n_streams=B, max_chunk=N)
    refs = [O.RefModel(model=model, sample_rate=fs, fmt=fmt) for _ in range(B)]
    got = [[] for _ in range(B)]
    want = [[] for _ in range(B)]
    for c in range(nchunks):
        eng.submit(np.stack([x[c * N:(c + 1) * N] for x in xs]), N)
        for s in range(B):
            refs[s].push(xs[s][c * N:(c + 1) * N])
        for m in eng.poll():
            got[m.stream].append(m)
        for s in range(B):
            want[s] += refs[s].messages()
    problems, n = [], 0
    for s in range(B):
        g = [(m.key(), m.start_idx, m.end_idx) for m in got[s]]
        w = [(m.key(), m.start_idx, m.end_idx) for m in want[s]]
        n += len(w)
        if g != w:
            problems.append(("MSG", s, len(g), len(w), [x for x in g if x not in w][:2], [x for x in w if x not in g][:2]))
        else:
            for a, b in zip(got[s], want[s]):
                if np.float32(a.level).view(np.uint32) != np.float32(b.level).view(np.uint32) or \
                        np.float32(a.ppm).view(np.uint32) != np.float32(b.ppm).view(np.uint32):
                    problems.append(("TAG", s, a.level, b.level, a.ppm, b.ppm))
    eng.close()
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    return n


@pytest.mark.parametrize("fs,N", [(1536000, 65536), (1536000, 16384), (1536000, 4096), (384000, 16384), (3072000, 131072)])
def test_challenger(built, fs, N):
    # model 4 "v1_high" (Model.cpp:601-678): coherent and FM decoders side by side behind one CGF, ten cross-reset decoders per channel
    n = run_msg_case(aisgpu.MODEL_CHALLENGER, fs, N, 8 if N >= 16384 else 64, 3, 81)
    assert n >= 4


def test_challenger_dense(built):
    # many overlapping / back-to-back bursts: frames complete in both branches close together, the Reset crosses branches
    xs = [S.fuzz_stream(96000, 262144, 300 + s)[0] for s in range(6)]
    eng = aisgpu.Engine(model=aisgpu.MODEL_CHALLENGER, sample_rate=96000, n_streams=6, max_chunk=8192)
    got = [[] for _ in range(6)]
    for c in range(32):
        eng.submit(np.stack([x[c * 8192:(c + 1) * 8192] for x in xs]), 8192)
    for m in eng.poll():
        got[m.stream].append(m)
    want = []
    for s in range(6):
        r = O.RefModel(model=O.MODEL_CHALLENGER, sample_rate=96000)
        r.run(xs[s], 8192)
        want.append(r.messages())
    eng.close()
    # payload, NMEA, channel, start / end counters and the level / ppm bit patterns: weak and colliding bursts are where the
    # coherent decoders win, and the winner decides which level and which CGF block's ppm the frame carries
    problems = U.compare_frames(got, want)
    assert not problems, "frames differ from the reference: %r" % (problems[:3],)


@pytest.mark.parametrize("amp", [0.0, 1e-30, 3e-39])
def test_tiny_and_zero_inputs(built, amp):
    """All-zero, tiny NORMAL and SUBNORMAL inputs through the front end are bit-exact: every CIC scaling and add is its own
    __fmul_rn / __fadd_rn (no FMA contraction, no flush to zero), so a subnormal product rounds exactly as in the reference."""
    fs, N, B = 1536000, 65536, 2
    rng = np.random.default_rng(5)
    xs = [((rng.standard_normal(N * 2) + 1j * rng.standard_normal(N * 2)) * amp).astype(np.complex64) for _ in range(B)]
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=N, taps=True)
    refs = [oracle_model(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, taps=True) for _ in range(B)]
    for c in range(2):
        eng.submit(np.stack([x[c * N:(c + 1) * N] for x in xs]), N)
        for s in range(B):
            refs[s].push(xs[s][c * N:(c + 1) * N])
            for ch in range(2):
                w = refs[s].tap_c(O.TAP_CA + ch)
                g = eng.tap(aisgpu.TAP_C, s, ch)
                assert bits_equal(g, w), (amp, c, s, ch, first_diff(g, w))
    eng.close()


@pytest.mark.parametrize("lanes", ["0", "1", "3", "7", "18", "33", "100"])
def test_streaming_frontend_lane_split(built, monkeypatch, lanes):
    """The streaming front end splits a stream's super-steps over L lanes, L not dividing the block (uneven q / q + 1 split,
    warps spanning streams, spare lanes in the last warp): AISGPU_ST_L forces L, "0" lets the launcher plan it.
    N = 64 * 1017 has no power-of-two lane split at all."""
    monkeypatch.setenv("AISGPU_ST_L", lanes)
    n = run_case(built, aisgpu.MODEL_STANDARD, 1536000, 64 * 1017, 4, 5, seed0=41)
    assert n >= 6


@pytest.mark.parametrize("fmt,fs,N", [(aisgpu.FMT_CU8, 1536000, 64 * 1017), (aisgpu.FMT_CS16, 768000, 32 * 999), (aisgpu.FMT_CF32, 3072000, 128 * 613)])
def test_streaming_frontend_lane_split_formats(built, monkeypatch, fmt, fs, N):
    for lanes in ("5", "19"):
        monkeypatch.setenv("AISGPU_ST_L", lanes)
        run_case(built, aisgpu.MODEL_DEFAULT, fs, N, 3, 3, fmt=fmt, seed0=43)
