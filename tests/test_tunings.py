"""Several tunings of one input without a GPU: the rules of aisgpu_check_tunings with their texts, and that with per_input = 1 it
accepts and refuses exactly what aisgpu_check_tuning does."""
import ctypes as C
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "ais-catcher_b200"), HERE]

import aisgpu  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def offsets_of(a):
    return (C.c_int32 * max(len(a), 1))(*a)


def tunings(lib, offsets, per_input, **engine):
    """(rc, text) of aisgpu_check_tunings"""
    rc = lib.aisgpu_check_tunings(C.byref(aisgpu.make_config(**engine)), offsets_of(offsets), len(offsets), per_input)
    return rc, lib.aisgpu_last_error(None).decode() if rc else ""


def tuning(lib, offsets, **engine):
    """(rc, text) of aisgpu_check_tuning"""
    rc = lib.aisgpu_check_tuning(C.byref(aisgpu.make_config(**engine)), offsets_of(offsets), len(offsets))
    return rc, lib.aisgpu_last_error(None).decode() if rc else ""


def test_accepts(lib):
    aisgpu.check_tuning([2600000, -2600000] * 3, per_input=2, n_streams=6, sample_rate=12288000, fmt=aisgpu.FMT_CS16)
    aisgpu.check_tuning([0, 300000, -300000], per_input=3, n_streams=3)
    aisgpu.check_tuning([0, 1, 2, 3], per_input=4, n_streams=4, fmt=aisgpu.FMT_CU8)
    aisgpu.check_tuning([23999, -23999] * 2, per_input=2, n_streams=4, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX")


def test_per_input_rules(lib):
    for per_input, n_streams in ((0, 4), (-1, 4), (3, 4), (5, 4), (2, 3)):
        rc, text = tunings(lib, [0] * n_streams, per_input, n_streams=n_streams)
        assert rc == aisgpu.EINVAL
        assert text == "aisgpu_set_tunings: per_input %d must be at least 1 and divide n_streams %d" % (per_input, n_streams)
    with pytest.raises(aisgpu.AisGpuError, match="per_input 3 must be at least 1 and divide n_streams 4"):
        aisgpu.check_tuning([0] * 4, per_input=3, n_streams=4)


def test_other_rules_keep_their_texts(lib):
    def refused(offsets, per_input, **engine):
        rc, text = tunings(lib, offsets, per_input, **engine)
        assert rc == aisgpu.EINVAL
        return text
    assert refused([0, 0, 0], 2, n_streams=4) == "aisgpu_set_tuning: 3 offsets for 4 streams"
    assert refused([0, 0, 0, 768000], 2, n_streams=4) == \
        "aisgpu_set_tuning: stream 3: offset 768000 Hz must lie strictly between -fs/2 and fs/2 (fs = 1536000)"
    assert refused([0, -768000], 2, n_streams=2).startswith("aisgpu_set_tuning: stream 1: offset -768000 Hz")
    assert "FM-discriminator input model" in refused([0, 0], 2, n_streams=2, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000)
    assert "FP_DS on" in refused([0, 1000], 2, n_streams=2, fmt=aisgpu.FMT_CU8, fp_ds=True)
    assert lib.aisgpu_check_tunings(C.byref(aisgpu.make_config(n_streams=2)), None, 2, 2) == aisgpu.EINVAL
    assert lib.aisgpu_last_error(None).decode() == "aisgpu_set_tuning: null offset table"
    assert lib.aisgpu_check_tunings(None, offsets_of([0, 0]), 2, 2) == aisgpu.EINVAL


@pytest.mark.parametrize("offsets,engine", [
    ([0, 767999, -767999, 12], dict(n_streams=4)),
    ([0, 0], dict(n_streams=3)),
    ([0] * 4, dict(n_streams=3)),
    ([], dict(n_streams=1)),
    ([0, 768000], dict(n_streams=2)),
    ([-768000], dict(n_streams=1)),
    ([23999, -23999], dict(n_streams=2, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX")),
    ([24000], dict(n_streams=1, sample_rate=48000, channel_mode=aisgpu.MODE_X, channels="XX")),
    ([6000000, -6143999], dict(n_streams=2, sample_rate=12288000)),
    ([0], dict(n_streams=1, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000)),
    ([1000], dict(n_streams=1, fmt=aisgpu.FMT_CU8, fp_ds=True)),
    ([100000], dict(n_streams=1, fmt=aisgpu.FMT_CU8, fp_ds=True, sample_rate=3072000)),
])
def test_per_input_one_is_check_tuning(lib, offsets, engine):
    assert tunings(lib, offsets, 1, **engine) == tuning(lib, offsets, **engine)


def test_exports(lib):
    for name in ("aisgpu_set_tunings", "aisgpu_check_tunings"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS
    header = open(os.path.join(ROOT, "include", "aisgpu.h")).read()
    assert "int aisgpu_set_tunings(aisgpu_handle *h, const int32_t *offset_hz, int n, int per_input);" in header
    assert "int aisgpu_check_tunings(const aisgpu_config *cfg, const int32_t *offset_hz, int n, int per_input);" in header
