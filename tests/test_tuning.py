"""The per-stream digital tune without a GPU: aisgpu_tune_restate (the definition the engine's k_tune computes) against a numpy float32
restatement of the definition written in include/aisgpu.h, bit for bit, in every input format; that it is a real oscillator; and the
rules of aisgpu_check_tuning with their texts."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "ais-catcher_b200"), HERE]

import aisgpu  # noqa: E402

FORMATS = (aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16, aisgpu.FMT_F32_FS4, aisgpu.FMT_DC16H)
F32 = np.float32


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def raw_input(fmt, n, rng):
    """n samples of format fmt with every bit pattern the conversion reads: extremes, zeros, negative zeros for the floats."""
    if fmt == aisgpu.FMT_CF32:
        v = rng.standard_normal(2 * n).astype(F32)
        v[::7] = 0.0
        v[1::11] = -0.0
        return v.view(np.complex64)
    if fmt == aisgpu.FMT_CU8:
        return rng.integers(0, 256, 2 * n, dtype=np.uint8)
    if fmt == aisgpu.FMT_CS8:
        return rng.integers(-128, 128, 2 * n, dtype=np.int8)
    if fmt == aisgpu.FMT_CS16:
        return rng.integers(-32768, 32768, 2 * n, dtype=np.int16)
    if fmt == aisgpu.FMT_F32_FS4:
        v = rng.standard_normal(n).astype(F32)
        v[::5] = 0.0
        return v
    w = rng.integers(0, 1 << 32, 3 * n, dtype=np.uint64).astype(np.uint32)  # DC16H: garbage in the halves it does not read
    w[0:3 * 8:3] = np.array([0, 0x8000, 0x7FFF, 0xFFFF, 0x1234, 0, 0x8000, 1], np.uint32)
    w[1:3 * 8:3] = np.array([0, 0x8000, 0x7FFF, 0xFFFF, 0, 0x8000, 0x10000, 0xFFFF8000], np.uint32)
    return w


def convert(fmt, raw, n):
    """ConvertRAW as float32 (re, im) arrays; n: each sample's index in its stream."""
    if fmt == aisgpu.FMT_CF32:
        v = raw.view(F32)
        return v[0::2].copy(), v[1::2].copy()
    if fmt in (aisgpu.FMT_CU8, aisgpu.FMT_CS8):
        q = raw.astype(np.int32) - (128 if fmt == aisgpu.FMT_CU8 else 0)
        return q[0::2].astype(F32) * F32(0.0078125), q[1::2].astype(F32) * F32(0.0078125)
    if fmt == aisgpu.FMT_CS16:
        return raw[0::2].astype(F32) * F32(2.0 ** -15), raw[1::2].astype(F32) * F32(2.0 ** -15)
    if fmt == aisgpu.FMT_F32_FS4:
        y = np.where(n & 2, -raw, raw).astype(F32)
        zero = np.zeros_like(y)
        return np.where(n & 1, zero, y), np.where(n & 1, y, zero)
    w = raw.reshape(-1, 3)
    i = (w[:, 0] & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.int32)
    q = -(w[:, 1] & 0xFFFF).astype(np.uint16).view(np.int16).astype(np.int32)
    return i.astype(F32) * F32(2.0 ** -15), q.astype(F32) * F32(2.0 ** -15)


def tables(fs):
    lo = (2 * np.pi) * np.arange(4096, dtype=np.float64) / fs
    hi = (2 * np.pi) * (np.arange((fs + 4095) // 4096, dtype=np.int64) * 4096).astype(np.float64) / fs
    return (np.cos(hi).astype(F32), np.sin(hi).astype(F32)), (np.cos(lo).astype(F32), np.sin(lo).astype(F32))


def restate(fmt, fs, f, first, raw):
    """The definition: k = ((n mod fs) f) mod fs, p = T_hi[k >> 12] T_lo[k & 4095], out = v conj(p), each operation in float32."""
    cnt = len(raw.view(np.uint8)) // {0: 8, 1: 2, 2: 2, 3: 4, 4: 4, 7: 12}[fmt]
    n = first + np.arange(cnt, dtype=np.int64)
    vr, vi = convert(fmt, raw, n)
    if f != 0:
        k = (n % fs) * (f % fs) % fs
        (hc, hs), (lc, ls) = tables(fs)
        hr, hi_, lr, li = hc[k >> 12], hs[k >> 12], lc[k & 4095], ls[k & 4095]
        pr = hr * lr - hi_ * li
        pi = hr * li + hi_ * lr
        vr, vi = vr * pr + vi * pi, vi * pr - vr * pi
    out = np.empty((cnt, 2), F32)
    out[:, 0], out[:, 1] = vr, vi
    return out.view(np.complex64).reshape(cnt)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


def offsets(fs, rng):
    h = fs // 2
    return [0, 1, -1, h - 1, -(h - 1)] + [f for f in (25000, -25000) if abs(f) < h] + [int(x) for x in rng.integers(-(h - 1), h, 4)]


@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("fs", [48000, 288000, 1536000, 12288000])
def test_restate_matches_the_definition(lib, fmt, fs):
    rng = np.random.default_rng(fs + 17 * fmt)
    raw = raw_input(fmt, 6000, rng)
    for f in offsets(fs, rng):
        for first in (0, 3, int(rng.integers(0, 1 << 40)), (1 << 40) - 5, 7 * fs - 1):
            got = aisgpu.tune_restate(fmt, fs, f, first, raw)
            want = restate(fmt, fs, f, first, raw)
            assert same_bits(got, want), "fmt %d fs %d offset %d first %d" % (fmt, fs, f, first)


@pytest.mark.parametrize("fmt", FORMATS)
def test_split_buffers_match_one_call(lib, fmt):
    rng = np.random.default_rng(99 + fmt)
    fs, n = 1536000, 20000
    raw = raw_input(fmt, n, rng)
    per = len(raw) // n
    for f in (0, 731234, -767999, 3):
        whole = aisgpu.tune_restate(fmt, fs, f, 12345, raw)
        cuts = sorted(set([0, n] + [int(c) for c in rng.integers(0, n, 7)]))
        parts = [aisgpu.tune_restate(fmt, fs, f, 12345 + a, raw[a * per:b * per]) for a, b in zip(cuts, cuts[1:])]
        assert same_bits(np.concatenate(parts), whole)


def test_zero_offset_is_the_conversion_only(lib):
    # multiplying by 1 + 0j is not an identity on signed zeros: an offset of 0 must not multiply at all
    raw = np.array([0.0, -0.0, -0.0, 0.0, -0.0, -0.0, 1.5, -2.0], F32).view(np.complex64)
    assert same_bits(aisgpu.tune_restate(aisgpu.FMT_CF32, 1536000, 0, 5, raw), raw)


@pytest.mark.parametrize("fs", [1536000, 12288000])
def test_oscillator_is_unit_and_on_phase_over_a_period(lib, fs):
    # v = 1 gives conj(p); offset 1 Hz walks k through every value of a full period
    ones = np.ones(fs, np.complex64)
    p = np.conj(aisgpu.tune_restate(aisgpu.FMT_CF32, fs, 1, 0, ones)).astype(np.complex128)
    mag = np.abs(p)
    assert np.max(np.abs(mag - 1.0)) < 4 * 2.0 ** -24
    err = np.angle(p * np.exp(-2j * np.pi * np.arange(fs, dtype=np.float64) / fs))
    assert np.max(np.abs(err)) < 1e-6


def test_restate_arguments(lib):
    raw = np.zeros(4, np.complex64)
    out = np.zeros(4, np.complex64)
    call = lambda fmt, fs, f, first, n: lib.aisgpu_tune_restate(fmt, fs, f, first, raw.ctypes.data_as(C.c_void_p), n,
                                                                 out.ctypes.data_as(C.c_void_p))
    assert call(0, 1536000, 767999, 0, 4) == aisgpu.OK
    assert call(0, 1536000, -767999, 0, 4) == aisgpu.OK
    for bad in [(0, 1536000, 768000, 0, 4), (0, 1536000, -768000, 0, 4), (5, 1536000, 0, 0, 4), (6, 1536000, 0, 0, 4),
                (0, 0, 0, 0, 4), (0, 1536000, 0, -1, 4), (0, 1536000, 0, 0, -1)]:
        assert call(*bad) == aisgpu.EINVAL, bad
    assert lib.aisgpu_tune_restate(0, 1536000, 0, 0, None, 4, out.ctypes.data_as(C.c_void_p)) == aisgpu.EINVAL


def refused(offsets, **engine):
    with pytest.raises(aisgpu.AisGpuError) as e:
        aisgpu.check_tuning(offsets, **engine)
    return str(e.value).split(": ", 1)[1]


def test_check_tuning_accepts(lib):
    aisgpu.check_tuning([0, 767999, -767999, 12], n_streams=4)
    aisgpu.check_tuning([23999, -23999], n_streams=2, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX")
    aisgpu.check_tuning([6000000, -6143999], n_streams=2, sample_rate=12288000)
    aisgpu.check_tuning([100000], n_streams=1, fmt=aisgpu.FMT_CU8, fp_ds=True, sample_rate=3072000)  # FP_DS is read at 1536K only


def test_check_tuning_rules(lib):
    assert refused([0, 0], n_streams=3) == "aisgpu_set_tuning: 2 offsets for 3 streams"
    assert refused([0] * 4, n_streams=3) == "aisgpu_set_tuning: 4 offsets for 3 streams"
    assert refused([0, 768000], n_streams=2) == \
        "aisgpu_set_tuning: stream 1: offset 768000 Hz must lie strictly between -fs/2 and fs/2 (fs = 1536000)"
    assert refused([-768000], n_streams=1).startswith("aisgpu_set_tuning: stream 0: offset -768000 Hz")
    assert refused([24000], n_streams=1, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX").startswith(
        "aisgpu_set_tuning: stream 0: offset 24000 Hz")
    assert "FM-discriminator input model" in refused([0], n_streams=1, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000)
    assert "FP_DS on" in refused([1000], n_streams=1, fmt=aisgpu.FMT_CU8, fp_ds=True)


def test_check_tuning_null_and_size(lib):
    cfg = aisgpu.make_config(n_streams=1)
    assert lib.aisgpu_check_tuning(C.byref(cfg), None, 1) == aisgpu.EINVAL
    assert lib.aisgpu_last_error(None).decode() == "aisgpu_set_tuning: null offset table"
    assert lib.aisgpu_check_tuning(None, (C.c_int32 * 1)(0), 1) == aisgpu.EINVAL
    cfg.struct_size = 12
    assert lib.aisgpu_check_tuning(C.byref(cfg), (C.c_int32 * 1)(0), 1) == aisgpu.EINVAL


def test_exports(lib):
    for name in ("aisgpu_set_tuning", "aisgpu_check_tuning", "aisgpu_tune_restate"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS
