"""Single-channel mode (-c X) without a GPU: the rate table and granules of the C ABI, the reference's rejection wording, the
pre-channel_mode config layout, and (where the reference was built) the reference harness against tests/golden/mode_x.json."""
import ctypes as C

import pytest

import aisgpu
import mode_x_util as X
import oracle_x as OX


@pytest.mark.parametrize("fs", [48000, 96000, 192000, 12000, 24000, 50000, 100000, 150000])
@pytest.mark.parametrize("fmt", [aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16])
def test_x_granule(built, fs, fmt):
    # one rule at every X rate and format; the AB table is untouched (fs = 96000/192000 are AB buckets too)
    assert aisgpu.chunk_granule(fs, fmt=fmt, channel_mode=aisgpu.MODE_X) == 64


def test_ab_granules_unchanged(built):
    assert aisgpu.chunk_granule(96000) == 4
    assert aisgpu.chunk_granule(192000) == 8
    assert aisgpu.chunk_granule(1536000) == 64
    with pytest.raises(aisgpu.AisGpuError, match="between 96K and 12288K"):
        aisgpu.chunk_granule(48000)


@pytest.mark.parametrize("fs", [11999, 192001, 0, 1536000])
def test_x_rejects_rate(built, fs):
    with pytest.raises(aisgpu.AisGpuError, match=r"Model: sample rate must be between 12k and 192k \(inclusive\)\."):
        aisgpu.chunk_granule(fs, channel_mode=aisgpu.MODE_X)


def test_x_ignores_dsk_fp_ds(built):
    assert aisgpu.chunk_granule(48000, dsk=True, fp_ds=True, fmt=aisgpu.FMT_CU8, channel_mode=aisgpu.MODE_X) == 64


def test_unknown_channel_mode(built):
    with pytest.raises(aisgpu.AisGpuError, match="channel_mode"):
        aisgpu.chunk_granule(96000, channel_mode=2)  # ABCD is not built


def test_old_config_size_is_ab(built):
    lib = aisgpu.load()
    cfg = aisgpu.Config()
    lib.aisgpu_default_config(C.byref(cfg))
    assert cfg.channel_mode == aisgpu.MODE_AB
    old = aisgpu.Config.channel_mode.offset
    assert old == C.sizeof(aisgpu.Config) - 4
    cfg.sample_rate = 1536000
    cfg.channel_mode = aisgpu.MODE_X  # beyond the caller's struct: must not be read
    cfg.struct_size = old
    assert lib.aisgpu_chunk_granule(C.byref(cfg)) == 64  # the AB granule of 1536K
    cfg.sample_rate = 48000
    assert lib.aisgpu_chunk_granule(C.byref(cfg)) == aisgpu.EINVAL  # AB: 48K is out of range
    cfg.struct_size = old + 2
    assert lib.aisgpu_chunk_granule(C.byref(cfg)) == aisgpu.EINVAL


def test_x_stimulus_pinned():
    # the X generator (mode_x_util.x_stream) has its own RNG streams
    for case in X.load().values():
        X.case_input(case)


@pytest.mark.skipif(not OX.have_refx(), reason="reference harness (mode X) not built")
@pytest.mark.parametrize("name", [c[0] for c in X.CASES])
def test_ref_harness_reproduces_golden(built, name):
    case = X.load()[name]
    raw, per = X.case_input(case)
    got = X.record(*X.ref_run(case["model"], case["fs"], case["N"], case["nchunks"], case["fmt"], case["flags"], raw, per))
    assert got["messages"] == case["messages"]
    assert got["taps"] == case["taps"]
