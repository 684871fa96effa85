"""aisgpu_msg_json_full (the full AIS JSON, host build of the interpreter the engine runs on the GPU) byte for byte against the
reference's JSONAIS + Serializer(JSON_DICT_FULL):
  - the structured case set (tests/json_cases.py) against the expected lines in tests/golden/json_full.jsonl.gz (no reference needed);
  - the same set, 100 000 random payloads of random lengths with random tags, and the tag variants against the reference harness
    (oracle/oracle_json.py) when it is built.
Every frame gives a line: every application message (DAC, FI) the reference decodes into fields is decoded, records included."""
import ctypes as C
import gzip
import hashlib
import json
import os
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "oracle"), HERE]

import aisgpu  # noqa: E402
import json_cases  # noqa: E402
import oracle_json  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "json_full.jsonl.gz")
need_ref = pytest.mark.skipif(not oracle_json.have_ref(), reason="reference JSON harness not built (make -C oracle -f json.mk refjson)")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def f32(x):
    return C.c_float(x).value


def product(c):
    t = c["tag"]
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], level=c["level"], ppm=c["ppm"], sentences=c["sentences"])
    tag = aisgpu.make_tag(version=t["version"], driver=t["driver"], hardware=t["hardware"], mode=t["mode"], rxtime_us=t["rxtime_us"],
                          toa_us=t["toa_us"], station=t["station"])
    return aisgpu.msg_json_full(m, tag)


def reference(c):
    t = c["tag"]
    return oracle_json.ref_line(bytes.fromhex(c["data"]), c["nbits"], c["channel"], c["sentences"], f32(c["level"]), f32(c["ppm"]),
                                t["version"], t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"], t["station"])


def check(c, want):
    got = product(c)
    assert got == want, "case %r\n got  %r\n want %r" % (c, got, want)


def case_digest(c):
    return hashlib.sha1(json.dumps(c, sort_keys=True).encode()).hexdigest()[:16]


def test_exports(lib):
    for name in ("aisgpu_msg_json_full", "aisgpu_json_enable", "aisgpu_poll_json"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS


def test_golden_structured_set(lib):
    cases = json_cases.structured_cases()
    with gzip.open(GOLDEN, "rt", encoding="utf-8") as f:
        recs = [json.loads(l) for l in f]
    assert len(recs) == len(cases), "tests/golden/json_full.jsonl.gz is out of date: python tools/gen_json_golden.py"
    for c, r in zip(cases, recs):
        assert r["case"] == case_digest(c), "tests/golden/json_full.jsonl.gz is out of date: python tools/gen_json_golden.py"
        check(c, r["line"].encode("utf-8"))
    # every message type and every (DAC, FI) pair the reference decodes was there
    types = {bytes.fromhex(c["data"])[0] >> 2 for c in cases}
    assert set(range(1, 29)) <= types
    pairs6 = {(json_cases.getu(bytes.fromhex(c["data"]), 72, 10), json_cases.getu(bytes.fromhex(c["data"]), 82, 6)) for c in cases
              if bytes.fromhex(c["data"])[0] >> 2 == 6}
    pairs8 = {(json_cases.getu(bytes.fromhex(c["data"]), 40, 10), json_cases.getu(bytes.fromhex(c["data"]), 50, 6)) for c in cases
              if bytes.fromhex(c["data"])[0] >> 2 == 8}
    assert set(json_cases.ASM6) <= pairs6 and set(json_cases.ASM8) <= pairs8


@need_ref
def test_golden_matches_reference(lib):
    with gzip.open(GOLDEN, "rt", encoding="utf-8") as f:
        recs = [json.loads(l) for l in f]
    for c, r in zip(json_cases.structured_cases(), recs):
        assert reference(c) == r["line"].encode("utf-8")


@need_ref
@pytest.mark.parametrize("seed", range(10))
def test_random_payloads_against_reference(lib, seed):
    for c in json_cases.random_cases(10000, 1000 + seed):  # 100 000 over the ten seeds
        check(c, reference(c))


@need_ref
@pytest.mark.parametrize("mode", range(8))
def test_tag_modes_against_reference(lib, mode):
    rng = __import__("random").Random(mode)
    for station in (0, 1, 4242):
        for rx in (0, 1700000000000000, 1700000000999999, 1):
            for toa in (0, 1700000000250000):
                for typ in (1, 4, 5, 18, 21, 24, 27):
                    d = json_cases.msg(rng, typ, rng.choice([244000000 + rng.randrange(999999), 111232000, 982441234]))
                    c = json_cases.case(d, max(json_cases.MIN_BITS[typ - 1], 168), rng.choice("AB"), mode=mode, station=station,
                                        rxtime_us=rx, toa_us=toa, hardware=rng.choice(["", "rtl"]))
                    check(c, reference(c))


def test_suffix_and_overflow(lib):
    c = json_cases.structured_cases()[200]
    line = product(c)
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], level=c["level"], ppm=c["ppm"], sentences=c["sentences"])
    t = dict(c["tag"])
    tag = aisgpu.make_tag(suffix="\r\n", **t)
    assert aisgpu.msg_json_full(m, tag) == line + b"\r\n"
    buf = C.create_string_buffer(len(line))
    assert aisgpu.load().aisgpu_msg_json_full(C.byref(m), C.byref(aisgpu.make_tag(**t)), buf, len(line)) == len(line)
    assert aisgpu.load().aisgpu_msg_json_full(C.byref(m), C.byref(aisgpu.make_tag(**t)), buf, len(line) - 1) == aisgpu.EOVERFLOW
    assert aisgpu.load().aisgpu_msg_json_full(None, C.byref(aisgpu.make_tag(**t)), buf, len(line)) == aisgpu.EINVAL


def test_lengths_outside_the_message_read_as_empty(lib):
    # Message::setLength ignores a length beyond 1064: the reference then prints no type / repeat / mmsi and no field reads nbits
    c = json_cases.case(bytes([4] + [0x55] * 139), 2000)
    got = product(c)
    assert b'"mmsi"' not in got and b'"status":' in got
