"""FM-discriminator input model (-m 3) without a GPU: granules and rate rejections of the C ABI (both config layouts), the seeded
stimulus, the reference harness against tests/golden/disc.json, and the adapter's -go key and rate errors (where the reference was
built)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import aisgpu
import disc_util as D
import oracle_disc as OD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ADAPTER = os.path.join(ROOT, "oracle", "_ref", "adapter_disc_test")
ABOVE = r"Internal error: sample rate not supported in FM discriminator model\."
BELOW = r"FM discriminator model: sample rate must be between 12k and 48k \(inclusive\)\."


@pytest.mark.parametrize("fs", [48000, 44100, 32000, 22050, 12000])
@pytest.mark.parametrize("fmt", [aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16])
@pytest.mark.parametrize("mode", [aisgpu.MODE_AB, aisgpu.MODE_X])
def test_granule(built, fs, fmt, mode):
    # droop / dsk / fp_ds are ignored, and the channel mode builds the same chain
    assert aisgpu.chunk_granule(fs, model=aisgpu.MODEL_DISCRIMINATOR, fmt=fmt, channel_mode=mode) == 64
    assert aisgpu.chunk_granule(fs, model=aisgpu.MODEL_DISCRIMINATOR, fmt=fmt, dsk=True, fp_ds=True, channel_mode=mode) == 64


@pytest.mark.parametrize("fs,msg", [(48001, ABOVE), (96000, ABOVE), (1536000, ABOVE), (11999, BELOW), (8000, BELOW), (0, BELOW)])
def test_rejects_rate(built, fs, msg):
    for mode in (aisgpu.MODE_AB, aisgpu.MODE_X):
        with pytest.raises(aisgpu.AisGpuError, match=msg):
            aisgpu.chunk_granule(fs, model=aisgpu.MODEL_DISCRIMINATOR, channel_mode=mode)


def test_old_config_size(built):
    lib = aisgpu.load()
    cfg = aisgpu.Config()
    lib.aisgpu_default_config(C.byref(cfg))
    cfg.model = aisgpu.MODEL_DISCRIMINATOR
    cfg.struct_size = aisgpu.Config.channel_mode.offset
    for fs, want in ((44100, 64), (12000, 64), (96000, aisgpu.EINVAL), (11025, aisgpu.EINVAL)):
        cfg.sample_rate = fs
        assert lib.aisgpu_chunk_granule(C.byref(cfg)) == want
    cfg.sample_rate = 96000
    lib.aisgpu_chunk_granule(C.byref(cfg))
    assert lib.aisgpu_last_error(None).decode() == "Internal error: sample rate not supported in FM discriminator model."


def test_other_models_unchanged(built):
    assert aisgpu.chunk_granule(96000, model=aisgpu.MODEL_STANDARD) == 4
    assert aisgpu.chunk_granule(48000, model=aisgpu.MODEL_STANDARD, channel_mode=aisgpu.MODE_X) == 64
    with pytest.raises(aisgpu.AisGpuError, match="between 96K and 12288K"):
        aisgpu.chunk_granule(48000, model=aisgpu.MODEL_STANDARD)


def test_stimulus_pinned():
    for case in D.load().values():
        D.case_input(case)


def test_stimulus_sides_differ():
    # channel A in I and B in Q carry different traffic: an I/Q swap cannot pass
    x = D.stereo(48000, 48000, 1)
    assert not np.array_equal(x.real, x.imag)
    case = D.load()["cs16_48k"]
    chans = [m["ch"] for c in case["messages"] for m in c]
    payloads = {ch: {m["payload"] for c in case["messages"] for m in c if m["ch"] == ch} for ch in "AB"}
    assert "A" in chans and "B" in chans and not payloads["A"] & payloads["B"]


def test_golden_known_answers():
    # the reference decodes its own known-answer sentences and a two-sentence type 5 from the discriminator stimulus
    nmea = [s for m in (m for c in D.load()["type5_48k"]["messages"] for m in c) for s in m["nmea"]]
    assert any("15MgK45P3@G?fl0E`JbR0OwT0@MS" in s for s in nmea)
    assert any("15NPOOPP00o?b=bE`UNv4?w428D;" in s for s in nmea)
    assert any(s.startswith("!AIVDM,2,1,") for s in nmea) and any(s.startswith("!AIVDM,2,2,") for s in nmea)


@pytest.mark.skipif(not OD.have_refd(), reason="reference harness (-m 3) not built")
@pytest.mark.parametrize("name", [c[0] for c in D.CASES])
def test_ref_harness_reproduces_golden(built, name):
    case = D.load()[name]
    raw, per = D.case_input(case)
    got = D.record(*D.ref_run(case["fs"], case["N"], case["nchunks"], case["fmt"], case["letters"], raw, per))
    assert got["messages"] == case["messages"]
    assert got["taps"] == case["taps"]


needs_adapter = pytest.mark.skipif(not os.path.exists(ADAPTER), reason="adapter_disc_test not built (needs the reference tree at build time)")


def run_adapter(tmp_path, *args):
    path = os.path.join(tmp_path, "in.cs16")
    np.zeros(4096 * 2, np.int16).tofile(path)
    p = subprocess.run([ADAPTER, args[0], path] + list(args[1:]), capture_output=True, text=True, timeout=120,
                       env=dict(os.environ, CUDA_VISIBLE_DEVICES=""))
    return p.returncode, p.stderr


@needs_adapter
@pytest.mark.parametrize("key,value", [("DROOP", "off"), ("DSK", "on"), ("FP_DS", "on"), ("PS_EMA", "off"), ("AFC_WIDE", "off")])
def test_adapter_rejects_frontend_keys(built, tmp_path, key, value):
    """-m 3 takes no front-end key: the adapter hands it to Model::SetKey, which words the error as the reference does."""
    got = {}
    for side in ("gpu", "cpu"):
        rc, err = run_adapter(tmp_path, "AB", "CS16", "48000", "4096", side, key, value)
        assert rc == 4, err
        got[side] = err
    assert got["cpu"].startswith("config error: FM discriminator output model: setting \"%s\" not supported" % key.lower())
    assert got["gpu"] == got["cpu"].replace("FM discriminator output model", "AIS engine H100 (FM discriminator input)")


@needs_adapter
@pytest.mark.parametrize("fs", [48001, 96000])
def test_adapter_rate_error_above_48k(built, tmp_path, fs):
    for side in ("gpu", "cpu"):
        rc, err = run_adapter(tmp_path, "X", "CS16", str(fs), "4096", side)
        assert rc == 4 and "Internal error: sample rate not supported in FM discriminator model." in err, err


@needs_adapter
def test_adapter_station_keys_accepted(built, tmp_path):
    rc, err = run_adapter(tmp_path, "AB", "CS16", "48000", "4096", "cpu", "STATION_ID", "7", "OWN_MMSI", "123456789")
    assert rc == 0, err
    rc, err = run_adapter(tmp_path, "AB", "CS16", "44100", "4096", "gpu", "STATION_ID", "7", "OWN_MMSI", "123456789")
    assert rc == 3 and "class FM" in err  # getClass is FM; with no GPU the first block stops the application
