"""The edge-case stimuli of tests/edge_signals.py reach the paths they exist for.  Checked on the input itself and, where the
reference was built (oracle/_ref), on the reference's own taps -- without this a passing bit-exact test on them might never have
reached the edge.  CPU only."""
import numpy as np
import pytest

import edge_signals as E
import oracle as O

FS, N, G = 1536000, 65536, 64  # 1536 kS/s CF32: the granule is 64 samples
CF32, CU8, CS8, CS16 = E.CF32, E.CU8, E.CS8, E.CS16

need_ref = pytest.mark.skipif(not O.have_ref(), reason="needs the compiled reference (oracle/_ref)")


def fz_none_ppm():
    """tag.ppm of a CGF block without any maximum: fz stays -1, f = -1 / 2 / 512 (DSP.cpp:418, 451-457)."""
    f = np.float32(np.float32(np.float32(-1.0) / np.float32(2.0)) / np.float32(512.0))
    return np.float32(np.float32(f * np.float32(48000.0)) / np.float32(162.0))


def run_ref(raw, per, model, fmt=CF32, nchunks=None, n=N):
    """The reference over raw in submits of n samples: (ref, {tap name: concatenated array}, messages)."""
    nchunks = nchunks or len(raw) // per // n
    r = O.RefModel(model=model, sample_rate=FS, fmt=fmt, taps=True)
    taps = {}
    for c in range(nchunks):
        r.push(raw[c * n * per:(c + 1) * n * per])
        for k in range(11):
            taps.setdefault("c%d" % k, []).append(r.tap_c(k))
        for k in range(14):
            taps.setdefault("f%d" % k, []).append(r.tap_f(k))
    return r, {k: np.concatenate(v) for k, v in taps.items()}, r.messages()


def test_integer_rails_and_codes():
    n = 4 * N
    for fmt, zero in ((CU8, 128), (CS8, 0), (CS16, 0)):
        raw, per = E.make("silence", FS, n, 1, fmt)
        assert per == 2 and len(raw) == 2 * n and (raw == zero).all()
    raw, _ = E.make("silence", FS, n, 1, CF32)
    assert (raw.view(np.uint32) == 0).all()
    for fmt, lo, hi in ((CU8, 0, 255), (CS8, -128, 127), (CS16, -32768, 32767)):
        raw, _ = E.make("clipped", FS, n, 1, fmt)
        assert (raw == lo).sum() > 100 and (raw == hi).sum() > 100, fmt
    raw, _ = E.make("clipped", FS, n, 1, CF32)
    v = raw.view(np.float32)
    assert (v == 1.0).sum() > 100 and (v == -1.0).sum() > 100 and np.abs(v).max() == 1.0
    raw, _ = E.make("dc", FS, n, 1, CU8)
    assert (raw == 127).all()
    raw, _ = E.make("dc", FS, n, 1, CF32)
    assert (raw.view(np.float32) == np.float32(-1.0 / 128.0)).all()
    # CU8 below one LSB: the noise takes only the codes 127 and 128, the bursts a few LSB more
    raw, _ = E.make("quantised", FS, n, 1, CU8)
    x, _ = E.traffic(FS, n, 1, noise_sigma=0.0)
    quiet = np.repeat(np.abs(x) == 0, 2)
    assert quiet.sum() > n // 4 and set(np.unique(raw[quiet])) == {127, 128}
    assert raw[~quiet].min() <= 122 and raw[~quiet].max() >= 134
    raw, _ = E.make("quantised", 48000, 48000, 1, CS16, E.DISC)
    assert np.abs(raw.astype(np.int32)).max() == 8 and (raw == 0).sum() > 0


def test_float_edges_in_input():
    n = 4 * N
    raw, _ = E.make("signed_zero", FS, n, 1)
    u = raw.view(np.uint32)
    assert ((u & 0x7fffffff) == 0).all() and (u == 0x80000000).sum() > n and (u == 0).sum() > n // 2
    raw, _ = E.make("real_only", FS, n, 1)
    assert (raw.imag.view(np.uint32) == 0).all() and (raw.real != 0).all()
    raw, _ = E.make("subnormal", FS, n, 1)
    a = np.abs(raw.view(np.float32))
    assert a.max() < np.finfo(np.float32).tiny and (a > 0).sum() > n
    for name in ("loud", "loud_max"):
        raw, _ = E.make(name, FS, n, 1)
        assert np.isfinite(raw.view(np.float32)).all()
    # the tone on a bin is exactly periodic in the 512-sample FFT of the 48 kHz channel; the other lies half-way between two bins
    assert (E.TONE_BIN_HZ / (48000 / 512)) % 1 == 0 and (E.TONE_BETWEEN_HZ / (48000 / 512)) % 1 == 0.5


def test_gap_layout():
    n = 12 * N
    x, bursts = E.traffic(FS, n, 3)
    gaps = E.gap_ranges(FS, n, N, G, bursts)
    (a0, b0), (a1, b1), (a2, b2) = gaps
    assert b0 - a0 == G and a0 // N == 0 and a0 % N != 0  # one granule inside submit 0
    assert b1 - a1 == E.cgf_block(FS) and a1 < 2 * N < b1  # one CGF block across a submit boundary
    assert b2 - a2 >= 0.15 * FS and any(s < a2 < s + ln for s, ln in bursts)  # long enough, and it cuts a burst
    raw, _ = E.make("gaps", FS, n, 3, submit=N, granule=G)
    for a, b in gaps:
        assert (raw[a:b].view(np.uint32) == 0).all()


@need_ref
def test_silence_takes_the_no_maximum_path():
    # an all-zero CGF block has no bin above 0: the reference keeps fz = -1 and still derotates (the engine's CGF_IDX_NONE)
    raw, per = E.make("silence", FS, 4 * N, 1)
    r, taps, msgs = run_ref(raw, per, O.MODEL_DEFAULT)
    ppm = r.tap_ppm(O.TAP_CGF_A)
    assert len(ppm) == 4 * N // E.cgf_block(FS) and (ppm.view(np.uint32) == fz_none_ppm().view(np.uint32)).all()
    assert not msgs
    # silence gives exact zeros behind the front end: all of the FIR17 output
    assert len(taps["c7"]) == 4 * N // 32 and (taps["c7"].view(np.uint64) == 0).all()
    # in the gaps of S3 the same happens between blocks with a maximum
    raw, per = E.make("gaps", FS, 12 * N, 3, submit=N, granule=G)
    r, taps, _ = run_ref(raw, per, O.MODEL_DEFAULT)
    ppm = r.tap_ppm(O.TAP_CGF_A)
    none = ppm.view(np.uint32) == fz_none_ppm().view(np.uint32)
    assert 10 <= none.sum() < len(ppm) - 10
    fir = taps["c7"].view(np.uint64)
    run, longest = 0, 0
    for z in fir == 0:  # a run of exact zeros in the FIR17 output
        run = run + 1 if z else 0
        longest = max(longest, run)
    assert longest > 4000


@need_ref
def test_fm_tap_reaches_atan2_rare_paths():
    # FM = atan2f(im, re) / PI: zeros behind the front end give atan2(+-0, +-0), i.e. exact +0, -0 and +1 (atan2(+0, -0) = pi)
    for name in ("gaps", "subnormal"):
        raw, per = E.make(name, FS, 6 * N, 3, submit=N, granule=G)
        _, taps, _ = run_ref(raw, per, O.MODEL_STANDARD)
        u = np.concatenate([taps["f10"], taps["f11"]]).view(np.uint32)
        assert (u == 0x3f800000).sum() > 0 and (u == 0x80000000).sum() > 0 and (u == 0).sum() > 0, name


@need_ref
def test_loud_max_is_the_largest_finite_power():
    x, _ = E.traffic(FS, 4 * N, 3)
    for model in (O.MODEL_STANDARD, O.MODEL_BASE, O.MODEL_DEFAULT):
        raw, per = E.make("loud_max", FS, 4 * N, 3)
        _, taps, _ = run_ref(raw, per, model)
        assert all(np.isfinite(v).all() for v in taps.values()), model
    # one power of two more and the FM taps of ModelStandard overflow
    y = (x.astype(np.complex128) * 2.0 ** (E.LOUD_MAX_EXP + 1)).astype(np.complex64)
    _, taps, _ = run_ref(y, 1, O.MODEL_STANDARD)
    assert not np.isfinite(taps["f10"]).all()


@need_ref
def test_reference_decodes_after_every_gap():
    n = 12 * N
    for model in (O.MODEL_STANDARD, O.MODEL_DEFAULT):
        for fmt in (CF32, CU8):
            x, bursts = E.traffic(FS, n, 3)
            gaps = E.gap_ranges(FS, n, N, G, bursts)
            raw, per = E.make("gaps", FS, n, 3, fmt, submit=N, granule=G)
            _, _, msgs = run_ref(raw, per, model, fmt)
            ends = [b // 32 for _, b in gaps] + [n // 32]  # start_idx counts 48 kHz samples
            for k, (a, b) in enumerate(gaps):
                assert any(b // 32 <= m.start_idx and m.end_idx < gaps[k + 1][0] // 32 if k + 1 < len(gaps) else b // 32 <= m.start_idx
                           for m in msgs), (model, fmt, k, [(m.start_idx, m.end_idx) for m in msgs], ends)


@need_ref
def test_clipped_and_quantised_still_decode():
    # the saturated and the nearly silent receiver are worth checking only where the reference still finds frames in them
    for name, fmt in (("clipped", CU8), ("clipped", CS16), ("clipped", CF32), ("quantised", CU8), ("dc_traffic", CU8)):
        raw, per = E.make(name, FS, 8 * N, 5, fmt)
        _, _, msgs = run_ref(raw, per, O.MODEL_DEFAULT, fmt)
        assert len(msgs) >= 2, (name, fmt)
