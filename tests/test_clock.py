"""The rules of aisgpu_set_clock without a device (aisgpu_check_clock), and the time of a record at the ends of the clock's range:
  - the start times are one per stream (also for the live clock, start_us NULL) and lie in [0, 253402300800000000), so that rxtime
    stays YYYYMMDDHHMMSS; each refusal names its reason;
  - aisgpu_msg_format prints the stamps a clock can give -- the epoch, whole and fractional seconds, a year boundary, the last
    microsecond before year 10000 -- where every format prints a time (NMEA_TAG c:, JSON_NMEA rxuxtime, the full JSON's rxtime /
    rxuxtime, FULL's timestamp, the binary time stamp), byte for byte as the reference's outputs do (oracle/oracle_fmt.py) when that
    is built, and with the rxtime of Python's calendar always."""
import datetime
import os
import re

import pytest

import aisgpu
import json_cases
import oracle_fmt

LIMIT = 253402300800000000  # 10000-01-01T00:00:00Z in microseconds
STAMPS = [0, 1, 999999, 1000000, 1700000000654321, 1767225599999999, 1767225600000000, LIMIT - 1]
need_ref = pytest.mark.skipif(not oracle_fmt.have_ref(), reason="reference output harness not built (make -C oracle -f fmt.mk reffmt)")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def refusal(start_us, n=None, **engine):
    with pytest.raises(aisgpu.AisGpuError) as e:
        aisgpu.check_clock(start_us, n, **engine)
    return str(e.value)


def test_exports(lib):
    for name in ("aisgpu_set_clock", "aisgpu_check_clock", "aisgpu_stamp"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS


def test_check_clock_accepts(lib):
    aisgpu.check_clock(None, n_streams=1)
    aisgpu.check_clock(None, n_streams=7)
    aisgpu.check_clock([0, 1, 1700000000654321, LIMIT - 1], n_streams=4)
    aisgpu.check_clock([5], n_streams=1, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000)
    aisgpu.check_clock([5, 6], n_streams=2, channel_mode=aisgpu.MODE_X, sample_rate=48000, channels="XX")


def test_check_clock_refuses(lib):
    assert "3 start times for 4 streams" in refusal([0, 0, 0], n_streams=4)
    assert "5 start times for 4 streams" in refusal([0] * 5, n_streams=4)
    assert "3 start times for 4 streams" in refusal(None, 3, n_streams=4)  # the live clock is one per stream too
    assert "0 start times for 1 streams" in refusal(None, 0, n_streams=1)
    why = refusal([0, -1], n_streams=2)
    assert "stream 1: start -1 us must lie in [0, %d)" % LIMIT in why
    why = refusal([LIMIT, 0], n_streams=2)
    assert "stream 0: start %d us must lie in [0, %d)" % (LIMIT, LIMIT) in why
    assert "stream 2" in refusal([0, 1, -(1 << 63)], n_streams=3)
    assert "stream 0" in refusal([(1 << 63) - 1], n_streams=1)


def rxtime(us):
    return (datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=us // 10 ** 6)).strftime("%Y%m%d%H%M%S")


def frames():
    """a few frames of the structured case set, one of several sentences among them"""
    cases = json_cases.structured_cases()
    out = [c for c in cases if len(c["sentences"]) == 1][:3] + [c for c in cases if len(c["sentences"]) > 1][:1]
    assert len(out) == 4
    return out


def record(fmt, c, us, mode):
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], level=c["level"], ppm=c["ppm"], sentences=c["sentences"])
    return aisgpu.msg_format(m, aisgpu.make_tag(version=81, hardware="rx", mode=mode, rxtime_us=us, station=5), fmt)


@pytest.mark.parametrize("us", STAMPS)
def test_time_of_a_stamp_in_the_records(lib, us):
    c = frames()[0]
    line = record(aisgpu.MSGFORMAT_JSON_FULL, c, us, 3).decode()
    assert '"rxtime":"%s"' % rxtime(us) in line
    assert re.search(r'"rxuxtime":[0-9.]+,', line)
    assert ", timestamp: %s," % rxtime(us) in record(aisgpu.MSGFORMAT_FULL, c, us, 3).decode()
    for fmt in (aisgpu.MSGFORMAT_JSON_FULL, aisgpu.MSGFORMAT_FULL):  # mode bit 1 off: no time
        assert rxtime(us).encode() not in record(fmt, c, us, 1)
    assert b",c:" in record(aisgpu.MSGFORMAT_NMEA_TAG, c, us, 0)  # printed whatever the mode


@need_ref
@pytest.mark.parametrize("us", STAMPS)
def test_stamps_match_reference(lib, us):
    for fmt in range(1, 10):
        for mode in (1, 2, 3, 7):
            for c in frames():
                for hub in (1, 0):  # COMMUNITY_HUB: the binary record, then the JSON_NMEA one
                    oracle_fmt.hub(hub)
                    oracle_fmt.group_seed(0)
                    st = aisgpu.FormatState(hub, 0)
                    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], level=c["level"], ppm=c["ppm"],
                                        sentences=c["sentences"])
                    got = aisgpu.msg_format(m, aisgpu.make_tag(version=81, hardware="rx", mode=mode, rxtime_us=us, station=5), fmt, st)
                    want = oracle_fmt.ref_record(fmt, m.data, c["nbits"], c["channel"], c["sentences"], m.level, m.ppm, 81, 0, "rx",
                                                 mode, us, 0, 5, False, 0, 0, "", 0, 0, None)
                    assert got == want, (fmt, mode, us, got, want)
