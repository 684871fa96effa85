"""WAV input without a GPU: aisgpu_wav_probe against the reference's Device::WAVFile::Open (FileWAV.cpp:49-98) on files built
byte by byte -- every header rule and error text, the data offset -- and what the reference reads as samples: everything from the
data chunk to the end of the file, chunks after it included (FileWAV.cpp:107-120)."""
import struct

import pytest

import aisgpu
import oracle_wav as OW
import wav_util as W

CF32, CU8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS16
SAMPLES = bytes(range(256)) * 4
LIST = W.chunk(b"LIST", b"INFOISFT" + struct.pack("<I", 6) + b"Lavf6\0")
JUNK = W.chunk(b"JUNK", bytes(28))
DATA = W.chunk(b"data", SAMPLES)
FMT16 = W.fmt_chunk(1, 2, 48000, 16)

# name -> (file bytes, (format, rate, data offset) or the reference's error text)
CASES = {
    "cs16": (W.riff(FMT16, DATA), (CS16, 48000, 44)),
    "cu8": (W.riff(W.fmt_chunk(1, 2, 1536000, 8), DATA), (CU8, 1536000, 44)),
    "cf32": (W.riff(W.fmt_chunk(3, 2, 2400000, 32), DATA), (CF32, 2400000, 44)),
    "list_before_fmt": (W.riff(LIST, FMT16, DATA), (CS16, 48000, 44 + len(LIST))),
    "junk_list_before_fmt": (W.riff(JUNK, LIST, FMT16, DATA), (CS16, 48000, 44 + len(JUNK) + len(LIST))),
    "odd_chunk_padded": (W.riff(W.chunk(b"bext", b"abc"), FMT16, DATA), (CS16, 48000, 44 + 12)),
    "odd_chunk_between_fmt_and_data": (W.riff(FMT16, W.chunk(b"fact", b"12345"), DATA), (CS16, 48000, 44 + 14)),
    # an odd chunk without its pad byte: the skip takes the first byte of the next chunk, and the walk loses its way
    "odd_chunk_unpadded": (W.riff(W.chunk(b"bext", b"abc", pad=False), FMT16, DATA), "no data in WAV-file."),
    "fmt18": (W.riff(W.fmt_chunk(1, 2, 44100, 16, extra=b"\0\0"), DATA), (CS16, 44100, 46)),
    "fmt40_pcm": (W.riff(W.fmt_chunk(1, 2, 96000, 16, extra=bytes(24)), DATA), (CS16, 96000, 68)),
    "fmt17_odd": (W.riff(W.fmt_chunk(1, 2, 48000, 16, extra=b"\x07"), DATA), (CS16, 48000, 46)),
    "fmt40_extensible": (W.riff(W.fmt_chunk(0xFFFE, 2, 48000, 16, extra=struct.pack("<HHI", 22, 16, 3) + bytes(16)), DATA),
                         "format not supported"),
    "fmt_twice": (W.riff(W.fmt_chunk(1, 2, 48000, 8), W.fmt_chunk(3, 2, 96000, 32), DATA), (CF32, 96000, 68)),
    "mono": (W.riff(W.fmt_chunk(1, 1, 48000, 16), DATA), "WAV-file must have 2 channels (I/Q)."),
    "four_channels": (W.riff(W.fmt_chunk(1, 4, 48000, 16), DATA), "WAV-file must have 2 channels (I/Q)."),
    "pcm24": (W.riff(W.fmt_chunk(1, 2, 48000, 24), DATA), "format not supported"),
    "float64": (W.riff(W.fmt_chunk(3, 2, 48000, 64), DATA), "format not supported"),
    "float16bits": (W.riff(W.fmt_chunk(3, 2, 48000, 16), DATA), "format not supported"),
    "alaw": (W.riff(W.fmt_chunk(6, 2, 48000, 8), DATA), "format not supported"),
    "fmt_short": (W.riff(W.chunk(b"fmt ", struct.pack("<HHIIH", 1, 2, 48000, 192000, 4)), DATA), "invalid fmt chunk in WAV-file."),
    "fmt_cut": (W.riff()[:12] + b"fmt " + struct.pack("<I", 16) + bytes(10), "cannot read fmt chunk from WAV-file."),
    "no_data": (W.riff(FMT16, LIST), "no data in WAV-file."),
    "no_fmt": (W.riff(LIST, DATA), "no data in WAV-file."),
    "fmt_after_data": (W.riff(DATA, FMT16), "no data in WAV-file."),
    "chunk_past_end": (W.riff(FMT16, b"JUNK" + struct.pack("<I", 1 << 30) + bytes(8), DATA), "no data in WAV-file."),
    "only_riff": (W.riff(), "no data in WAV-file."),
    "rifx": (W.riff(FMT16, DATA, riff_id=b"RIFX"), "not a supported WAV-file."),
    "not_wave": (W.riff(FMT16, DATA, wave=b"AVI "), "not a supported WAV-file."),
    "rate_beyond_int32": (W.riff(W.chunk(b"fmt ", struct.pack("<HHIIHH", 1, 2, 0xFFFFFFF0, 0, 4, 16)), DATA), (CS16, 0xFFFFFFF0, 44)),
    # a data chunk header cut short at the end: the walk ends on "data", and there is nothing left to read
    "data_header_cut": (W.riff(FMT16) + b"data" + b"\x10\x00", (CS16, 48000, 42)),
}


def _write(tmp_path, name, b):
    p = tmp_path / (name + ".wav")
    p.write_bytes(b)
    return str(p)


def _probe(path):
    try:
        return aisgpu.wav_probe(path)
    except aisgpu.AisGpuError as e:
        return str(e)


@pytest.mark.parametrize("name", sorted(CASES))
def test_probe(built, tmp_path, name):
    b, want = CASES[name]
    path = _write(tmp_path, name, b)
    got = _probe(path)
    if isinstance(want, str):
        assert got == "rc=-1: " + want
    else:
        assert got == want


@pytest.mark.skipif(not OW.have_ref(), reason="reference WAVFile harness not built")
@pytest.mark.parametrize("name", sorted(CASES))
def test_probe_equals_reference(built, tmp_path, name):
    b, want = CASES[name]
    path = _write(tmp_path, name, b)
    try:
        ref = OW.ref_open(path)
    except OW.RefWavError as e:
        assert isinstance(want, str) and str(e) == want
        return
    fmt, rate, off = aisgpu.wav_probe(path)
    assert (fmt, rate) == ref[:2]
    assert off == ref[2] or (ref[2] == -1 and off == len(b))  # -1: the stream failed at the end of the file
    # what the reference's device delivers as samples is the file from the data offset to its end
    assert OW.ref_read(path) == b[off:]


@pytest.mark.skipif(not OW.have_ref(), reason="reference WAVFile harness not built")
def test_chunks_after_data_are_read_as_samples(built, tmp_path):
    tail = W.chunk(b"LIST", b"INFOICMT" + struct.pack("<I", 9) + b"comment\0\0") + W.chunk(b"id3 ", bytes(11))
    b = W.riff(JUNK, FMT16, DATA, tail)
    path = _write(tmp_path, "tail", b)
    fmt, rate, off = aisgpu.wav_probe(path)
    assert off == 12 + len(JUNK) + len(FMT16) + 8 and b[off:off + len(SAMPLES)] == SAMPLES
    assert OW.ref_read(path) == SAMPLES + tail


def test_truncated_header_and_missing_file(built, tmp_path):
    for n in (0, 4, 11):
        path = _write(tmp_path, "cut%d" % n, W.riff(FMT16, DATA)[:n])
        assert _probe(path) == 'rc=-1: cannot read header from WAV file: "%s"' % path
        if OW.have_ref():
            with pytest.raises(OW.RefWavError) as e:
                OW.ref_open(path)
            assert str(e.value) == 'cannot read header from WAV file: "%s"' % path
    missing = str(tmp_path / "missing.wav")
    assert _probe(missing) == 'rc=-1: cannot open WAV file: "%s"' % missing
    if OW.have_ref():
        with pytest.raises(OW.RefWavError, match="cannot open WAV file"):
            OW.ref_open(missing)


def test_data_offsets(built, tmp_path):
    """The offset is the byte after the data chunk's header, wherever fmt and the other chunks lie."""
    for k, before in enumerate([(), (JUNK,), (LIST, JUNK), (W.chunk(b"bext", bytes(601)),)]):
        for fmt, rate in ((CS16, 48000), (CU8, 1536000), (CF32, 288000)):
            p = str(tmp_path / ("o%d_%d.wav" % (k, fmt)))
            off = W.write_wav(p, SAMPLES, fmt, rate, before=before)
            assert aisgpu.wav_probe(p) == (fmt, rate, off)
            with open(p, "rb") as f:
                assert f.read()[off:] == SAMPLES


def test_c_abi_null_arguments_and_untouched_outputs(built, tmp_path):
    import ctypes as C
    lib = aisgpu.load()
    fmt, rate, off = C.c_int32(-7), C.c_uint32(7), C.c_int64(-7)
    path = _write(tmp_path, "mono", CASES["mono"][0]).encode()
    assert lib.aisgpu_wav_probe(path, C.byref(fmt), C.byref(rate), C.byref(off)) == aisgpu.EINVAL
    assert (fmt.value, rate.value, off.value) == (-7, 7, -7)
    assert lib.aisgpu_last_error(None) == b"WAV-file must have 2 channels (I/Q)."
    assert lib.aisgpu_wav_probe(None, C.byref(fmt), C.byref(rate), C.byref(off)) == aisgpu.EINVAL
    assert lib.aisgpu_wav_probe(path, None, C.byref(rate), C.byref(off)) == aisgpu.EINVAL
    assert b"null argument" in lib.aisgpu_last_error(None)


def test_python_mirror(built, tmp_path):
    p = tmp_path / "m.wav"
    W.write_wav(str(p), SAMPLES, CU8, 1536000)
    assert aisgpu.wav_probe(p) == (CU8, 1536000, 44)  # os.PathLike as well as str
    with pytest.raises(aisgpu.AisGpuError, match=r"^rc=-1: no data in WAV-file\.$"):
        aisgpu.wav_probe(_write(tmp_path, "nd", CASES["no_data"][0]))
    assert hasattr(aisgpu.Engine, "feed_wav_files")
    assert {"aisgpu_wav_probe", "aisgpu_feed_wav_files"} <= set(aisgpu.EXPORTS)
