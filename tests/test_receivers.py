"""aisgpu_check_receivers (the rules of aisgpu_set_receivers without a device) and the records a stream with a receiver of its own is
printed with: aisgpu_msg_format with the output's tag and the receiver's station, driver, hardware, mode and ipv4 must equal the
reference's OutputMessage record for a message of that receiver (oracle/oracle_fmt.py), in every format, when the harness is built.
The frames of such a receiver carry its letters and read !AIVDO for its own MMSI; the sentences here are built that way."""
import ctypes as C
import os
import random
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "oracle"), HERE]

import aisgpu  # noqa: E402
import json_cases  # noqa: E402
import oracle_fmt  # noqa: E402

need_ref = pytest.mark.skipif(not oracle_fmt.have_ref(), reason="reference output harness not built (make -C oracle -f fmt.mk reffmt)")

# the output's fields: every stream's records share them
OUTPUT = dict(version=81, status=0, rxtime_us=1700000000654321, toa_us=0, include_ssl=False, uuid=None, suffix=None)


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def refused(receivers, **engine):
    with pytest.raises(aisgpu.AisGpuError) as e:
        aisgpu.check_receivers(receivers, **engine)
    return str(e.value).split(": ", 1)[1]


def test_exports(lib):
    for name in ("aisgpu_set_receivers", "aisgpu_check_receivers"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS


def test_letters_accepted(lib):
    rx = [dict(channels=c) for c in ("AB", "CD", "XX", "12", "??", "A?", "90", "zq", "Zz")]
    aisgpu.check_receivers(rx, n_streams=len(rx))
    aisgpu.check_receivers(rx, n_streams=len(rx), channel_mode=aisgpu.MODE_X, channels="XX")


@pytest.mark.parametrize("bad", [" ", "!", "-", ",", "*", "\\", "\x00", "\x7f", "\xe9", "_"])
def test_letters_refused_with_the_reference_text(lib, bad):
    assert refused([dict(channels="AB"), dict(channels=bad + "B")], n_streams=2) == "invalid NMEA channel designation: " + bad.rstrip("\x00")
    assert refused([dict(channels="A" + bad)], n_streams=1) == "invalid NMEA channel designation: " + bad.rstrip("\x00")


def test_second_letter_read_only_where_a_stream_has_two_channels(lib):
    # single-channel mode prints channel_a only; the FM-discriminator input model has two channels in either mode
    aisgpu.check_receivers([dict(channels="X!")], n_streams=1, channel_mode=aisgpu.MODE_X, channels="XX", sample_rate=48000)
    assert refused([dict(channels="!X")], n_streams=1, channel_mode=aisgpu.MODE_X, channels="XX") == \
        "invalid NMEA channel designation: !"
    assert refused([dict(channels="A!")], n_streams=1, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000,
                   channel_mode=aisgpu.MODE_X) == "invalid NMEA channel designation: !"


def test_count_and_null(lib):
    assert "2 receivers for 3 streams" in refused([dict(), dict()], n_streams=3)
    assert "4 receivers for 3 streams" in refused([dict()] * 4, n_streams=3)
    cfg = aisgpu.make_config(n_streams=1)
    assert lib.aisgpu_check_receivers(C.byref(cfg), None, 1) == aisgpu.EINVAL
    assert lib.aisgpu_check_receivers(None, aisgpu.receiver_table([dict()]), 1) == aisgpu.EINVAL
    cfg.struct_size = 12
    assert lib.aisgpu_check_receivers(C.byref(cfg), aisgpu.receiver_table([dict()]), 1) == aisgpu.EINVAL


def test_tag_of_a_receiver_keeps_the_outputs_fields(lib):
    r = dict(station=5, driver=9, hardware="hw", tag_mode=4, ipv4=77)
    t = tag_fields(r, OUTPUT)
    assert (t["version"], t["rxtime_us"], t["status"]) == (OUTPUT["version"], OUTPUT["rxtime_us"], OUTPUT["status"])
    assert (t["station"], t["driver"], t["hardware"], t["mode"], t["ipv4"]) == (5, 9, "hw", 4, 77)


def tag_fields(rx, output):
    """the tag stream s's records are printed with: the output's, with the receiver's station, driver, hardware, mode and ipv4"""
    t = dict(output)
    t.update(station=rx.get("station", 0), driver=rx.get("driver", 0), hardware=rx.get("hardware") or "", mode=rx.get("tag_mode", 3),
             ipv4=rx.get("ipv4", 0))
    return t


def receivers(rng):
    """receivers with unusual fields: letters C / D / 1 / ?, stations, hardware names that need JSON escaping, every tag mode"""
    out = []
    for mode in range(8):
        for ch in ("CD", "1?", "?D", "AB"):
            out.append(dict(channels=ch, station=rng.choice([0, 3, -12, 99999]), own_mmsi=-1, tag_mode=mode,
                            driver=rng.choice([0, 2, 17]), hardware=rng.choice(["", "RTL-SDR v3", 'rx "north"\\\t1']),
                            ipv4=rng.choice([0, 0xC0A80101, 0xFFFFFFFF])))
    return out


def frames_of(rx, rng, n):
    """n messages as rx's engine publishes them: its letters, !AIVDO for its own MMSI, multi-sentence ones among them"""
    out = []
    seq = 0
    for i in range(n):
        typ = rng.choice([1, 3, 5, 18, 8, 24, 21])
        nbits = rng.randrange(max(json_cases.MIN_BITS[typ - 1], 72), 1065 if typ in (5, 8, 21) else 200)
        d = json_cases.msg(rng, typ)
        own = json_cases.getu(d, 8, 30) if i % 3 == 0 else rx.get("own_mmsi", -1)
        ch = rx["channels"][i % 2]
        sent, seq = aisgpu.build_nmea(d[:(nbits + 7) // 8], nbits, ch, own, seq)
        m = aisgpu.make_msg(d, nbits, ch, 100 * i, 100 * i + 2000, level=rng.uniform(-60, 0) if rx["tag_mode"] & 1 else 0.0,
                            ppm=rng.uniform(-9, 9), sentences=sent)
        out.append(m)
    assert any(s.startswith("!AIVDO") for m in out for s in aisgpu.Msg(m).nmea)
    return out


@need_ref
@pytest.mark.parametrize("fmt", range(1, 10))
def test_records_of_receivers_match_the_reference(lib, fmt):
    rng = random.Random(4100 + fmt)
    output = dict(OUTPUT, include_ssl=fmt % 2 == 0, uuid="u-rx" if fmt == 6 else None, suffix="\n" if fmt == 1 else None)
    st = aisgpu.FormatState(0, 0)
    oracle_fmt.hub(0)
    oracle_fmt.group_seed(0)
    n = 0
    for rx in receivers(rng):
        t = tag_fields(rx, output)
        tag = aisgpu.make_tag(**t)
        for m in frames_of(rx, rng, 6):
            got = aisgpu.msg_format(m, tag, fmt, st)
            g = aisgpu.Msg(m)
            want = oracle_fmt.ref_record(fmt, g.data, g.nbits, g.channel, g.nmea, C.c_float(g.level).value, C.c_float(g.ppm).value,
                                         t["version"], t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"],
                                         t["station"], t["include_ssl"], g.start_idx, g.end_idx, t["uuid"] or "", t["status"],
                                         t["ipv4"], t["suffix"])
            assert got == want, "format %d receiver %r\n got  %r\n want %r" % (fmt, rx, got, want)
            n += 1
    assert st.records == n
