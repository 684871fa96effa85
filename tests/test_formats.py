"""aisgpu_msg_format (the record of a frame in each of the reference's message formats, host build of the formatter the engine runs
on the GPU for aisgpu_poll_lines) byte for byte against the reference's OutputMessage::formatInto / JSONAIS + Serializer
(oracle/oracle_fmt.py) when it is built:
  - every format over the structured case set (tests/json_cases.py), random payloads, multi-sentence frames and tag variants;
  - glibc's %g of FULL at adversarial floats;
  - the engine's counters: NMEA_TAG group ids across the 9999 wrap, COMMUNITY_HUB's JSON record every 100th frame;
  - the generated tables (csrc/fmt_text.h) against a fresh run of tools/gen_fmt_text.py.
The JSON_SPARSE and JSON_ANNOTATED records of the case set are also pinned by tests/golden/json_sparse_annotated.jsonl.gz, so those
two formats are checked where the reference is not built."""
import ctypes as C
import gzip
import json
import os
import random
import struct
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "oracle"), HERE, os.path.join(ROOT, "tools")]

import aisgpu  # noqa: E402
import json_cases  # noqa: E402
import oracle_fmt  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "json_sparse_annotated.jsonl.gz")
FORMATS = range(1, 10)
need_ref = pytest.mark.skipif(not oracle_fmt.have_ref(), reason="reference output harness not built (make -C oracle -f fmt.mk reffmt)")


@pytest.fixture(scope="module")
def lib():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    return aisgpu.load()


def f32(x):
    return C.c_float(x).value


TAG_DEFAULTS = dict(include_ssl=False, start_idx=0, end_idx=0, uuid="", status=0, ipv4=0, suffix=None)


def product(fmt, c, st=None):
    t = dict(TAG_DEFAULTS, **c["tag"])
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], t["start_idx"], t["end_idx"], level=c["level"],
                        ppm=c["ppm"], sentences=c["sentences"])
    tag = aisgpu.make_tag(version=t["version"], driver=t["driver"], hardware=t["hardware"], mode=t["mode"], status=t["status"],
                          ipv4=t["ipv4"], rxtime_us=t["rxtime_us"], toa_us=t["toa_us"], station=t["station"],
                          include_ssl=t["include_ssl"], uuid=t["uuid"] or None, suffix=t["suffix"])
    return aisgpu.msg_format(m, tag, fmt, st)


def reference(fmt, c):
    t = dict(TAG_DEFAULTS, **c["tag"])
    return oracle_fmt.ref_record(fmt, bytes.fromhex(c["data"]), c["nbits"], c["channel"], c["sentences"], f32(c["level"]),
                                 f32(c["ppm"]), t["version"], t["driver"], t["hardware"], t["mode"], t["rxtime_us"], t["toa_us"],
                                 t["station"], t["include_ssl"], t["start_idx"], t["end_idx"], t["uuid"], t["status"], t["ipv4"],
                                 t["suffix"])


def compare(fmt, cases):
    """every case in fmt on both sides, the counters of both starting from a fresh process"""
    st = aisgpu.FormatState(0, 0)
    oracle_fmt.hub(0)
    oracle_fmt.group_seed(0)
    for i, c in enumerate(cases):
        got, want = product(fmt, c, st), reference(fmt, c)
        assert got == want, "format %d, case %d %r\n got  %r\n want %r" % (fmt, i, c, got, want)
    assert st.records == len(cases)


def multi_cases(seed, n=400):
    """2-5 sentence frames (types 5, 6, 8, 19, 21, 24, 26 at long lengths), own MMSI (!AIVDO) among them"""
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        typ = rng.choice([5, 6, 8, 19, 21, 26, 8, 5])
        nbits = rng.randrange(max(json_cases.MIN_BITS[typ - 1], 169), 1065)
        d = json_cases.msg(rng, typ)
        own = json_cases.getu(d, 8, 30) if rng.random() < 0.3 else -1
        sent, _ = aisgpu.build_nmea(d[:(nbits + 7) // 8], nbits, rng.choice("AB"), own, rng.randrange(10))
        out.append(json_cases.case(d, nbits, rng.choice("AB"), sentences=sent, level=rng.uniform(-60, 0), ppm=rng.uniform(-9, 9),
                                   mode=rng.randrange(8), station=rng.choice([0, 7, -3]), rxtime_us=1700000000000000 + rng.randrange(10 ** 9)))
    assert any(len(c["sentences"]) >= 4 for c in out) and any(s.startswith("!AIVDO") for c in out for s in c["sentences"])
    return out


def test_exports(lib):
    for name in ("aisgpu_msg_format", "aisgpu_lines_enable", "aisgpu_poll_lines"):
        assert hasattr(lib, name) and name in aisgpu.EXPORTS
    assert (aisgpu.MSGFORMAT_NMEA, aisgpu.MSGFORMAT_JSON_ANNOTATED) == (1, 9)


def test_bad_arguments(lib):
    c = json_cases.structured_cases()[10]
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], sentences=c["sentences"])
    buf = C.create_string_buffer(64)
    for fmt in (0, 10, -1):
        assert lib.aisgpu_msg_format(C.byref(m), C.byref(aisgpu.make_tag()), fmt, None, buf, 64) == aisgpu.EINVAL
    st = aisgpu.FormatState(5, 2)
    assert lib.aisgpu_msg_format(C.byref(m), C.byref(aisgpu.make_tag()), 8, C.byref(st), buf, 64) == aisgpu.EOVERFLOW
    assert (st.records, st.groups) == (5, 2)  # a record that was not written does not advance the counters


def test_golden_sparse_and_annotated(lib):
    cases = json_cases.structured_cases()
    with gzip.open(GOLDEN, "rt", encoding="utf-8") as f:
        recs = [json.loads(l) for l in f]
    assert len(recs) == len(cases), "tests/golden/json_sparse_annotated.jsonl.gz is out of date: python tools/gen_fmt_golden.py"
    for c, r in zip(cases, recs):
        for fmt, key in ((aisgpu.MSGFORMAT_JSON_SPARSE, "sparse"), (aisgpu.MSGFORMAT_JSON_ANNOTATED, "annotated")):
            got = product(fmt, c)
            assert got == r[key].encode("utf-8"), "case %r\n got  %r\n want %r" % (c, got, r[key])


def test_json_full_is_the_full_line_and_suffix(lib):
    for c in json_cases.structured_cases()[:300]:
        m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], level=c["level"], ppm=c["ppm"], sentences=c["sentences"])
        tag = aisgpu.make_tag(**c["tag"])
        assert product(aisgpu.MSGFORMAT_JSON_FULL, c) == aisgpu.msg_json_full(m, tag) + b"\r\n"
        assert product(aisgpu.MSGFORMAT_JSON_NMEA, c) == aisgpu.msg_json(m, aisgpu.make_tag(suffix="\r\n", **c["tag"]))
        assert product(aisgpu.MSGFORMAT_BINARY_NMEA, c) == aisgpu.msg_binary(m, tag, False)


@need_ref
def test_golden_matches_reference(lib):
    with gzip.open(GOLDEN, "rt", encoding="utf-8") as f:
        recs = [json.loads(l) for l in f]
    for c, r in zip(json_cases.structured_cases(), recs):
        assert reference(aisgpu.MSGFORMAT_JSON_SPARSE, c) == r["sparse"].encode("utf-8")
        assert reference(aisgpu.MSGFORMAT_JSON_ANNOTATED, c) == r["annotated"].encode("utf-8")


@need_ref
@pytest.mark.parametrize("fmt", FORMATS)
def test_structured_set_against_reference(lib, fmt):
    compare(fmt, json_cases.structured_cases())


@need_ref
@pytest.mark.parametrize("fmt", FORMATS)
def test_random_payloads_against_reference(lib, fmt):
    compare(fmt, json_cases.random_cases(20000, 7000 + fmt))


@need_ref
@pytest.mark.parametrize("fmt", FORMATS)
def test_multi_sentence_against_reference(lib, fmt):
    compare(fmt, multi_cases(fmt))


@need_ref
@pytest.mark.parametrize("fmt", FORMATS)
def test_tag_variants_against_reference(lib, fmt):
    rng = random.Random(fmt)
    cases = []
    for mode in range(8):
        for station in (0, 4242, -17):
            for suffix in (None, "\n"):
                for uuid in ("", "8b2c4d5e-0f1a-4b3c-9d8e-7f6a5b4c3d2e"):
                    typ = rng.choice([1, 4, 5, 8, 18, 21, 24, 27])
                    d = json_cases.msg(rng, typ, rng.choice([244000000 + rng.randrange(999999), 111232000, 982441234]))
                    c = json_cases.case(d, max(json_cases.MIN_BITS[typ - 1], 168), rng.choice("AB"), mode=mode, station=station,
                                        rxtime_us=rng.choice([0, 1700000000000000, 1700000000999999]),
                                        toa_us=rng.choice([0, 1700000000250000]), hardware=rng.choice(["", "rtl \"x\""]),
                                        include_ssl=rng.random() < 0.5, start_idx=rng.randrange(10 ** 6), end_idx=rng.randrange(10 ** 6, 10 ** 7),
                                        uuid=uuid, status=rng.choice([0, 3]), ipv4=rng.choice([0, 3232235777]), suffix=suffix,
                                        level=rng.choice([1024.0, -23.25, 0.0]), ppm=rng.choice([1024.0, 0.5, -3.0]))
                    cases.append(c)
    compare(fmt, cases)


def adversarial_floats():
    vals = [1024.0, 0.0, -0.0, 1e-5, 9.999995e-5, 9.9999949e-5, 0.0001, 999999.5, 999999.4, 1e6, 123456.5, 100000.0, 0.5,
            -17.25, 3.4028235e38, -3.4028235e38, 1.17549435e-38, 1.4e-45, -1.4e-45, 1e-40, 1.5, 2.5, 1234565.0, 0.000123456]
    rng = random.Random(3)
    for _ in range(3000):
        vals.append(struct.unpack("<f", struct.pack("<I", rng.getrandbits(32)))[0])
    return [f32(v) for v in vals]


FULL_DATA = json_cases.msg(random.Random(1), 1)


def full_case(level, ppm):
    return json_cases.case(FULL_DATA, 168, mode=1, level=level, ppm=ppm)


def test_g_format_of_full_against_python(lib):
    # Python's %g rounds the exact binary value half to even, as glibc does; NaN's sign is left to the reference test
    for v in adversarial_floats():
        if v != v or v == 1024.0:
            continue
        got = product(aisgpu.MSGFORMAT_FULL, full_case(v, 0.5))
        want = ", signalpower: %s, ppm: 0.5)" % ("%g" % v)
        assert want.encode() in got, (v, got)


@need_ref
def test_g_format_of_full_against_reference(lib):
    vals = adversarial_floats()
    cases = [full_case(a, b) for a, b in zip(vals, vals[1:] + vals[:1])]
    compare(aisgpu.MSGFORMAT_FULL, cases)


@need_ref
def test_tag_groups_across_the_wrap(lib):
    cases = multi_cases(99, 60)
    for seed_groups in (9990, 9998, 9999, 19997):
        st = aisgpu.FormatState(0, seed_groups)
        oracle_fmt.group_seed(seed_groups % 9999)
        for c in cases:
            assert product(aisgpu.MSGFORMAT_NMEA_TAG, c, st) == reference(aisgpu.MSGFORMAT_NMEA_TAG, c)
        assert st.groups == seed_groups + sum(len(c["sentences"]) > 1 for c in cases)


def test_hub_ordinals(lib):
    c = json_cases.structured_cases()[5]
    st = aisgpu.FormatState(0, 0)
    recs = [product(aisgpu.MSGFORMAT_COMMUNITY_HUB, c, st) for _ in range(250)]
    for i, r in enumerate(recs):
        assert r.startswith(b'{"class":"AIS"') == (i % 100 == 0), i
    assert recs[1].startswith(b"\xac\x00")
    assert recs[0] == product(aisgpu.MSGFORMAT_JSON_NMEA, c) and recs[1] == product(aisgpu.MSGFORMAT_BINARY_NMEA, c)
    assert st.records == 250


@need_ref
def test_hub_ordinals_against_reference(lib):
    cases = [json_cases.structured_cases()[i] for i in range(0, 4600, 18)]
    for start in (0, 95, 199):
        st = aisgpu.FormatState(start, 0)
        oracle_fmt.hub(start)
        for c in cases:
            assert product(aisgpu.MSGFORMAT_COMMUNITY_HUB, c, st) == reference(aisgpu.MSGFORMAT_COMMUNITY_HUB, c)


@need_ref
def test_generated_tables_reproduce(lib):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "gen_fmt_text.py"), "--check"], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


def test_sentence_lengths_are_taken_up_to_the_sentence_buffer(lib):
    # aisgpu_msg.nmea holds 100 bytes per sentence: a longer nmea_len is read as 100, in aisgpu_msg_json as in aisgpu_msg_format
    c = json_cases.structured_cases()[3]
    m = aisgpu.make_msg(bytes.fromhex(c["data"]), c["nbits"], c["channel"], sentences=["!AIVDM," + "x" * 93])
    m.nmea_len[0] = 250
    got = aisgpu.msg_json(m, aisgpu.make_tag())
    assert got.endswith(b'"nmea":["!AIVDM,' + b"x" * 93 + b'"]}')
    assert aisgpu.msg_format(m, aisgpu.make_tag(), aisgpu.MSGFORMAT_NMEA) == b"!AIVDM," + b"x" * 93 + b"\r\n"
