"""The 12-byte input format DC16H without a GPU: the reference fed DC16H against the reference fed CF32 of the samples converted on
the host (pins this suite's reading of the format, tests/dc16h_util.py: which bits are read, the integer negation of Q), ConvertRAW's
size / 12, and the C ABI's rules: granules, the device-batch placement rule, aisgpu_check_attach, the feeder's block arithmetic."""
import ctypes as C
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
import oracle_disc as OD
import oracle_x as OX
import parity_util as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "oracle", "_ref", "adapter_dc16h_test")
DC16H = DC.DC16H

AB_RATES = [96000, 192000, 288000, 384000, 768000, 1536000, 3072000, 6144000, 12288000, 576000, 1152000, 2304000,
            240000, 250000, 1000000, 2000000, 6000000, 10000000]


def _refs(kind, model, fs):
    """(reference fed DC16H, reference fed CF32, complex taps, float taps) of one front-end family."""
    if kind == "x":
        if not (OX.have_refx() and ODC.have_ref("x")):
            pytest.skip("reference harness (mode X) not built")
        return (ODC.RefModelDC16H(model=model, sample_rate=fs, taps=True, kind="x"),
                OX.RefModelX(model=model, sample_rate=fs, fmt=O.FMT_CF32, taps=True), [O.TAP_CA], [])
    if kind == "disc":
        if not (OD.have_refd() and ODC.have_ref("disc")):
            pytest.skip("reference harness (model 3) not built")
        return (ODC.RefModelDC16H(sample_rate=fs, taps=True, kind="disc"), OD.RefModelDisc(sample_rate=fs, fmt=O.FMT_CF32, taps=True), [],
                [OD.TAP_RP, OD.TAP_IP, O.TAP_FR_A, O.TAP_FR_B])
    if not (O.have_ref() and ODC.have_ref()):
        pytest.skip("reference harness not built")
    ctaps = [O.TAP_ROT_IN, O.TAP_UP, O.TAP_DOWN, O.TAP_CA, O.TAP_CB, O.TAP_US, O.TAP_DSK]
    if model == O.MODEL_DEFAULT:
        ctaps += [O.TAP_CGF_A, O.TAP_CGF_B, O.TAP_FC_A, O.TAP_FC_B]
    return (ODC.RefModelDC16H(model=model, sample_rate=fs, taps=True), O.RefModel(model=model, sample_rate=fs, fmt=O.FMT_CF32, taps=True),
            ctaps, list(range(10)))


def _traffic(kind, fs, n, seed):
    if kind == "x":
        z = X.stream_input(fs, n, seed, O.FMT_CF32)[0]
    elif kind == "disc":
        z = D.stereo(fs, n, seed)
    else:
        z = S.random_stream(fs, n, seed, bursts_per_sec=(6, 12))[0]
    return DC.from_complex(z, seed)[0]


def test_conversion_special_values():
    """Q = 0 -> +0.0 (the integer is negated, not the float), Q = -32768 -> 1.0, I = -32768 -> -1.0; the garbage is not read."""
    i = np.array([0, -32768, 32767, 1, -1, 0], dtype=np.int16)
    q = np.array([0, -32768, 32767, 0, 1, -1], dtype=np.int16)
    bits = DC.unpack(DC.pack_iq(i, q, 1)).view(np.uint32).reshape(-1, 2)
    f = lambda v: int(np.float32(v).view(np.uint32))
    assert bits.tolist() == [[0, 0], [f(-1.0), f(1.0)], [f(32767 / 32768), f(-32767 / 32768)], [f(1 / 32768), 0],
                             [f(-1 / 32768), f(-1 / 32768)], [0, f(1 / 32768)]]
    a, b = DC.pack_iq(i, q, 1).reshape(-1, 3), DC.pack_iq(i, q, 2).reshape(-1, 3)
    assert (a[:, 2] != b[:, 2]).any() and ((a[:, :2] >> 16) != (b[:, :2] >> 16)).any()
    assert U.bits_equal(DC.unpack(a.reshape(-1)), DC.unpack(b.reshape(-1)))
    w = DC.from_complex(np.array([0.25 - 0.5j, -1 + 1j], dtype=np.complex64))[0]
    assert DC.unpack(w).tolist() == [complex(8192 / 32768, -16384 / 32768), complex(-32767 / 32768, 32767 / 32768)]
    assert DC.to_cs16(w).tolist() == [8192, -16384, -32767, 32767]


@pytest.mark.parametrize("kind,model,fs,N", [("ab", O.MODEL_DEFAULT, 1536000, 65536), ("ab", O.MODEL_STANDARD, 384000, 16384),
                                             ("ab", O.MODEL_DEFAULT, 1000000, 32768), ("ab", O.MODEL_DEFAULT, 288000, 12288),
                                             ("x", O.MODEL_DEFAULT, 96000, 8192), ("disc", 3, 48000, 4096)],
                         ids=["streaming1536", "tiled384", "prestage1000", "dsk288", "x96", "disc48"])
def test_reference_dc16h_equals_reference_cf32_of_unpacked(built, kind, model, fs, N):
    nchunks = 6
    w = _traffic(kind, fs, N * nchunks, 3)
    a, b, ctaps, ftaps = _refs(kind, model, fs)
    frames = 0
    for c in range(nchunks):
        blk = w[c * N * 3:(c + 1) * N * 3]
        a.push(blk)
        b.push(DC.unpack(blk))
        for t in ctaps:
            assert U.bits_equal(a.tap_c(t), b.tap_c(t)), ("complex tap", t, c)
        for t in ftaps:
            assert U.bits_equal(a.tap_f(t), b.tap_f(t)), ("float tap", t, c)
        ma, mb = a.messages(), b.messages()
        assert [U.frame_key(m) for m in ma] == [U.frame_key(m) for m in mb]
        frames += len(ma)
    assert frames > 0


@pytest.mark.skipif(not (O.have_ref() and ODC.have_ref()), reason="reference harness not built")
def test_reference_special_values_reach_the_fm_taps(built):
    """ModelStandard (atan2f behind the front end) on runs of Q = 0, Q = -32768 and I = -32768: the reference fed DC16H gives the
    bits of the reference fed the host conversion, so the signed zero and the exact 1.0 of tests/dc16h_util.py are the reference's."""
    fs, N = 1536000, 16384
    i, q = DC.iq_of(S.random_stream(fs, 4 * N, 21, bursts_per_sec=(6, 12))[0])
    q[:N] = 0
    i[N // 2:N] = 0
    q[N + 100:N + 3000] = -32768
    i[2 * N:2 * N + 2000] = -32768
    q[3 * N::2] = 0
    w = DC.pack_iq(i, q, 4)
    a, b, ctaps, ftaps = _refs("ab", O.MODEL_STANDARD, fs)
    for c in range(4):
        blk = w[c * N * 3:(c + 1) * N * 3]
        a.push(blk)
        b.push(DC.unpack(blk))
        for t in ctaps:
            assert U.bits_equal(a.tap_c(t), b.tap_c(t)), ("complex tap", t, c)
        for t in ftaps:
            assert U.bits_equal(a.tap_f(t), b.tap_f(t)), ("float tap", t, c)


@pytest.mark.skipif(not (O.have_ref() and ODC.have_ref()), reason="reference harness not built")
@pytest.mark.parametrize("extra", [1, 2])
def test_reference_drops_trailing_words(built, extra):
    """A buffer of 3 m + extra words: ConvertRAW forwards m samples, and the next buffer starts at a sample of its own."""
    fs, N = 384000, 8192
    w = _traffic("ab", fs, 4 * (N + 2), 5)
    a = ODC.RefModelDC16H(model=O.MODEL_DEFAULT, sample_rate=fs, taps=True)
    b = O.RefModel(model=O.MODEL_DEFAULT, sample_rate=fs, fmt=O.FMT_CF32, taps=True)
    off = 0
    for c in range(4):
        n = 3 * N + (extra if c & 1 else 0)
        a.push(w[off:off + n])
        b.push(DC.unpack(w[off:off + n]))
        off += n
        for t in (O.TAP_CA, O.TAP_CB):
            got, want = a.tap_c(t), b.tap_c(t)
            assert len(want) == N // 8 and U.bits_equal(got, want), (t, c)


@pytest.mark.parametrize("dsk", [False, True])
def test_granules_are_those_of_cs16(built, dsk):
    for fs in AB_RATES:
        for model in (aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD):
            g = aisgpu.chunk_granule(fs, model, dsk=dsk, fmt=DC16H)
            assert g % 4 == 0 and g == aisgpu.chunk_granule(fs, model, dsk=dsk, fmt=aisgpu.FMT_CS16), (fs, g)
            assert (6291456 // 12) % g == 0  # a whole Device::RAWFile block (FileRAW.h) is whole samples and whole granules
    for fs in (12000, 24000, 48000, 50000, 96000, 150000, 192000):
        assert aisgpu.chunk_granule(fs, dsk=dsk, fmt=DC16H, channel_mode=aisgpu.MODE_X) == 64
    for fs in (12000, 22050, 44100, 48000):
        assert aisgpu.chunk_granule(fs, aisgpu.MODEL_DISCRIMINATOR, dsk=dsk, fmt=DC16H) == 64


def test_fp_ds_still_needs_cu8(built):
    with pytest.raises(aisgpu.AisGpuError, match="needs CU8 input"):
        aisgpu.chunk_granule(1536000, fp_ds=True, fmt=DC16H)
    assert aisgpu.chunk_granule(3072000, fp_ds=True, fmt=DC16H) == 128


PLACES = [dict(sample_rate=1536000), dict(sample_rate=384000), dict(sample_rate=96000), dict(sample_rate=6000000),
          dict(sample_rate=288000), dict(sample_rate=1152000, dsk=True), dict(sample_rate=96000, channel_mode=aisgpu.MODE_X),
          dict(sample_rate=48000, model=aisgpu.MODEL_DISCRIMINATOR), dict(sample_rate=44100, model=aisgpu.MODEL_DISCRIMINATOR)]


@pytest.mark.parametrize("kw", PLACES, ids=lambda kw: "-".join(str(v) for v in kw.values()))
def test_placement_rule(built, kw):
    """dev_samples 16-byte aligned and stride_samples a multiple of 4 (rows 48 bytes apart at the least), in every mode and model."""
    base, N = 1 << 20, 16384
    for off, stride in [(0, N), (16, N), (0, N + 4), (32, N + 64), (48, N), (0, 3 * N), (0, 0)]:
        aisgpu.check_device_batch(base + off, stride, fmt=DC16H, **kw)
    for off, stride in [(4, N), (8, N), (12, N), (24, N), (0, N + 2), (0, N + 1), (0, N + 6), (16, N + 2), (0, -4)]:
        with pytest.raises(aisgpu.AisGpuError, match="rc=-1: DC16H: the base of a device batch must be 16-byte aligned"):
            aisgpu.check_device_batch(base + off, stride, fmt=DC16H, **kw)
    # the other formats' rule is what it was: CS16 takes a base aligned to two samples and any even stride
    aisgpu.check_device_batch(base + 8, N + 2, fmt=aisgpu.FMT_CS16, **{k: v for k, v in kw.items() if k != "channel_mode"})


def test_check_attach(built):
    lead = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=1536000, fmt=DC16H, n_streams=2, max_chunk=65536)
    aisgpu.check_attach(lead, dict(lead, model=aisgpu.MODEL_STANDARD))
    for other in (aisgpu.FMT_CF32, aisgpu.FMT_CS16, aisgpu.FMT_F32_FS4):
        with pytest.raises(aisgpu.AisGpuError, match="format differs"):
            aisgpu.check_attach(lead, dict(lead, fmt=other))
        with pytest.raises(aisgpu.AisGpuError, match="format differs"):
            aisgpu.check_attach(dict(lead, fmt=other), lead)


@pytest.mark.parametrize("fmt", [8, 100])
def test_values_beyond_dc16h_are_refused(built, fmt):
    """DC16H is 7, the last format; 5 and 6 below it are no formats either (tests/test_fs4.py)."""
    lib = aisgpu.load()
    cfg = aisgpu.make_config(sample_rate=1536000, fmt=fmt)
    h = C.c_void_p()
    assert lib.aisgpu_create(C.byref(cfg), C.byref(h)) == aisgpu.EINVAL and not h
    assert b"bad format" in lib.aisgpu_last_error(None)
    with pytest.raises(aisgpu.AisGpuError, match="bad format"):
        aisgpu.check_device_batch(1 << 20, 16384, fmt=fmt)


def test_abi_version_and_constant(built):
    assert aisgpu.load().aisgpu_abi_version() == 3 and DC16H == 7 and ODC.FMT_DC16H == 7
    with open(os.path.join(ROOT, "include", "aisgpu.h")) as f:
        text = f.read()
    assert "#define AISGPU_FMT_DC16H 7" in text and "but DC16H" not in text and "DC16H is not supported" not in text


@pytest.mark.skipif(not os.path.exists(EXE), reason="oracle/_ref/adapter_dc16h_test not built")
def test_adapter_without_gpu_stops_the_application(built, tmp_path):
    f = str(tmp_path / "x.dc16h")
    _traffic("ab", 384000, 24 * 8192 + 8, 9).tofile(f)
    p = subprocess.run([EXE, f, "384000", "8192", "2"], capture_output=True, env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    assert p.returncode == 3 and p.stdout == b"" and b"1 stop requests" in p.stderr
    # the same binary with the reference's model reads the format (and drops the odd words) without a GPU
    p = subprocess.run([EXE, f, "384000", "8192", "2", "cpu", "odd"], capture_output=True)
    assert p.returncode == 0 and len(p.stdout.splitlines()) >= 1
