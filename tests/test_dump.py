"""The 48 kHz channel dump (-go DUMP <prefix>) without a GPU: the reference facts the engine's WAV writer relies on, read from the
unmodified reference through oracle/_ref/libaisref_dump.so, and the Python argument checks of Engine.dump_open.

At every pre-stage chain and front-end family of AB mode, with push lengths that change from block to block, the reference's
<prefix>_A.wav / _B.wav are the 44-byte header (IEEE float, 2 channels, 32 bits, 48000 S/s, byte rate 384000, alignment 8, both
sizes patched at close) followed by every block of C_a / C_b, concatenated.  In single-channel mode it writes no file."""
import ctypes as C
import struct

import numpy as np
import pytest

import aisgpu
import aissynth as S
import mode_x_util as X
import oracle as O
import oracle_dump as OD

need_refdump = pytest.mark.skipif(not OD.have_refdump(), reason="reference dump harness not built (needs the reference tree at build time)")


def wav_header(n_bytes):
    """WriteWAV's header for a CF32 file of n_bytes of data after ~WriteWAV has patched it (StreamHelpers.cpp:135-229)."""
    return (b"RIFF" + struct.pack("<I", (n_bytes + 36) & 0xFFFFFFFF) + b"WAVE" + b"fmt " +
            struct.pack("<IHHIIHH", 16, 3, 2, 48000, 384000, 8, 32) + b"data" + struct.pack("<I", n_bytes & 0xFFFFFFFF))


def pushes(granule, total, seed):
    """Block lengths (multiples of granule) that change from push to push and add up to at most total samples."""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while True:
        k = int(rng.integers(1, 9)) * max(1, 1024 // granule) * granule
        if n + k > total:
            return out
        out.append(k)
        n += k


# name, model, rate, format, flags beyond the defaults
RATES = [
    ("96k", O.MODEL_DEFAULT, 96000, O.FMT_CF32, 0),
    ("384k_cs16", O.MODEL_STANDARD, 384000, O.FMT_CS16, 0),
    ("1536k_cu8", O.MODEL_DEFAULT, 1536000, O.FMT_CU8, 0),
    ("288k", O.MODEL_DEFAULT, 288000, O.FMT_CF32, 0),
    ("6000k", O.MODEL_BASE, 6000000, O.FMT_CF32, 0),
    ("240k", O.MODEL_DEFAULT, 240000, O.FMT_CF32, 0),
    ("1152k_dsk", O.MODEL_V2, 1152000, O.FMT_CF32, O.FLAG_DSK),
    ("12288k", O.MODEL_DEFAULT, 12288000, O.FMT_CS8, 0),
]


@need_refdump
@pytest.mark.parametrize("model,fs,fmt,extra", [r[1:] for r in RATES], ids=[r[0] for r in RATES])
def test_reference_dump_is_header_plus_channel_taps(built, tmp_path, model, fs, fmt, extra):
    g = aisgpu.chunk_granule(fs, model, bool(extra & O.FLAG_DSK), False, fmt)
    total = int(0.12 * fs) // g * g
    x, _ = S.random_stream(fs, total, 7)
    raw, per = X.to_raw(x, fmt)
    prefix = str(tmp_path / "ch")
    ref = OD.RefModelDump(prefix, model=model, sample_rate=fs, fmt=fmt, flags=O.DEFAULT_FLAGS | extra, taps=True)
    pos = 0
    for n in pushes(g, total, fs):
        ref.push(raw[pos * per:(pos + n) * per])
        pos += n
    ca, cb = ref.tap_c(O.TAP_CA), ref.tap_c(O.TAP_CB)
    ref.close()
    assert len(ca) > 0 and len(ca) == len(cb)
    for suffix, c in (("_A.wav", ca), ("_B.wav", cb)):
        data = open(prefix + suffix, "rb").read()
        want = wav_header(c.nbytes) + c.tobytes()
        assert data[:44] == want[:44], "header"
        assert data == want, "%s: %d bytes, want %d" % (suffix, len(data), len(want))


@need_refdump
def test_reference_dump_letters_in_cd_mode(built, tmp_path):
    # the file names are literally _A and _B whatever the channel letters (Model.cpp:390-396)
    x, _ = S.random_stream(96000, 8192, 3)
    ref = OD.RefModelDump(str(tmp_path / "cd"), sample_rate=96000, channels="CD")
    ref.push(x)
    ref.close()
    assert sorted(p.name for p in tmp_path.iterdir()) == ["cd_A.wav", "cd_B.wav"]


@need_refdump
def test_reference_writes_no_file_in_mode_x(built, tmp_path):
    x, _ = X.x_stream(48000, 16384, 5)
    ref = OD.RefModelDump(str(tmp_path / "x"), sample_rate=48000, channel_mode=aisgpu.MODE_X)
    ref.push(x[:8192])
    ref.push(x[8192:])
    ref.close()
    assert list(tmp_path.iterdir()) == []


@need_refdump
def test_reference_creates_files_at_first_block(built, tmp_path):
    # WriteWAV::Open runs at the first Receive: a model that never received a block leaves no file
    ref = OD.RefModelDump(str(tmp_path / "none"), sample_rate=1536000)
    ref.close()
    assert list(tmp_path.iterdir()) == []


def _bare_engine(n_streams):
    e = aisgpu.Engine.__new__(aisgpu.Engine)
    e.lib, e.h, e.n_streams, e.leader = aisgpu.load(), C.c_void_p(), n_streams, None
    return e


def test_dump_open_argument_checks(built):
    e = _bare_engine(3)
    with pytest.raises(ValueError, match="3 streams"):
        e.dump_open(["a", None])
    with pytest.raises(ValueError, match="3 streams"):
        e.dump_open(["a", None, "b", "c"])
    with pytest.raises(aisgpu.AisGpuError, match="rc=-1"):  # a NULL handle is EINVAL in the C ABI
        e.dump_open(["a", None, "b"])
    with pytest.raises(aisgpu.AisGpuError, match="rc=-1"):
        e.dump_close()


def test_eio_code(built):
    assert aisgpu.EIO == -6
    assert "aisgpu_dump_open" in aisgpu.EXPORTS and "aisgpu_dump_close" in aisgpu.EXPORTS
