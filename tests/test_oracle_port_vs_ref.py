"""CPU (-m "not gpu"): pins the plain-C restatement oracle/ais_oracle.c against the UNMODIFIED reference
(oracle/_ref/libaisref.so, strict IEEE flags) -- every tap and every message bit for bit.
The reference holds no golden vectors for the IQ path (SURVEY.md 4, 8c), so outputs of the reference itself are the
pin: tests/golden/port_vs_ref.json holds, per case, a SHA-256 of every tap of every chunk and every message (float tags
as bit patterns), written from the reference by `python tests/test_oracle_port_vs_ref.py`.  The port is checked against
that file everywhere; where oracle/_ref was built, the reference is re-run and checked against it too.
"""
import hashlib
import json
import os

import numpy as np
import pytest

import aissynth as S
import golden_util as G
import oracle as O
import oracle_x as OX

STORE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "port_vs_ref.json")
CASES = []  # (case id, compare() arguments), filled below by case()


def case(name, model, fs, N, nchunks, **kw):
    CASES.append((name, (model, fs, N, nchunks), kw))
    return name


def digest(Model, model, fs, N, nchunks, fmt=O.FMT_CF32, flags=O.DEFAULT_FLAGS, seed=0, multi=False, schedule=None, x_mode=False):
    """Runs one model over the seeded stimulus; returns the input hash, one hash over every tap of every chunk (in order,
    with lengths) and the per-chunk message records.  schedule: the length of every chunk (instead of nchunks chunks of N).
    x_mode: single-channel mode (the reference's oracle_x.RefModelX) on mode_x_util's stimulus at 0 Hz.  For ModelChallenger
    the records also name the decoder that published each message."""
    lengths = list(schedule) if schedule is not None else [N] * nchunks
    offs = np.cumsum([0] + lengths)
    if x_mode:
        import mode_x_util as MX
        x = MX.x_stream(fs, int(offs[-1]), seed)[0]
        if Model is O.RefModel:
            Model = OX.RefModelX
        else:
            flags |= O.FLAG_MODE_X
    else:
        x = S.random_stream(fs, int(offs[-1]), seed, multi_sentence=multi)[0]
    per = 1
    if fmt == O.FMT_CU8:
        x, per = S.to_cu8(x), 2
    elif fmt == O.FMT_CS8:
        x, per = (S.to_cu8(x).astype(np.int16) - 128).astype(np.int8), 2
    elif fmt == O.FMT_CS16:
        v = np.empty(2 * len(x), dtype=np.float32)
        v[0::2], v[1::2] = x.real, x.imag
        x, per = np.clip(np.round(v * 32767.0), -32768, 32767).astype(np.int16), 2
    m = Model(model=model, sample_rate=fs, fmt=fmt, flags=flags, taps=True)
    h = hashlib.sha256()
    msgs = []
    for c in range(len(lengths)):
        blk = x[offs[c] * per:offs[c + 1] * per]
        m.push(blk)
        taps = [m.tap_c(t) for t in range(9)] + [m.tap_f(t) for t in range(14)] + [m.tap_ppm(t) for t in (O.TAP_CGF_A, O.TAP_CGF_B)]
        for a in taps:
            a = np.ascontiguousarray(a)
            h.update(np.int64(a.size).tobytes())
            h.update(a.tobytes())
        pubs = m.publishers() if model == O.MODEL_CHALLENGER else None
        recs = [G.msg_record(q.channel, q.nbits, q.payload, q.nmea, q.start_idx, q.end_idx, q.level, q.ppm) for q in m.messages()]
        msgs.append(recs if pubs is None else [[r, p] for r, p in zip(recs, pubs)])
    return {"input_sha256": hashlib.sha256(np.ascontiguousarray(x).tobytes()).hexdigest(), "taps_sha256": h.hexdigest(), "messages": msgs}


def load_store():
    with open(STORE) as f:
        return json.load(f)


def compare(name):
    """The port (and the reference, where it was built) against the stored reference outputs; returns the message count."""
    _, args, kw = [c for c in CASES if c[0] == name][0]
    want = load_store()[name]
    got = digest(O.PortModel, *args, **kw)
    assert got["input_sha256"] == want["input_sha256"], "seeded generator no longer reproduces the stored input (numpy RNG change?)"
    for c, (g, w) in enumerate(zip(got["messages"], want["messages"])):
        assert g == w, "messages differ in chunk %d" % c
    assert got == want, "taps differ from the reference's"
    if O.have_ref() and (not kw.get("x_mode") or OX.have_refx()):
        assert digest(O.RefModel, *args, **kw) == want, "the reference no longer reproduces tests/golden/port_vs_ref.json"
    return sum(len(c) for c in want["messages"])


MODELS = {m: case("models_1536k_m%d" % m, m, 1536000, 65536, 4) for m in (O.MODEL_DEFAULT, O.MODEL_STANDARD, O.MODEL_BASE)}
RATES = {(fs, N): case("rates_default_%d_%d" % (fs, N), O.MODEL_DEFAULT, fs, N, 3, seed=23)
         for fs, N in [(96000, 4096), (192000, 8192), (288000, 12288), (384000, 16384), (768000, 32768), (3072000, 131072),
                       (6000000, 262144), (6144000, 262144), (12288000, 524288), (2000000, 65536), (250000, 16384)]}
FORMATS = {f: case("integer_formats_%d" % f, O.MODEL_DEFAULT, 1536000, 65536, 3, fmt=f, seed=17) for f in (O.FMT_CU8, O.FMT_CS8, O.FMT_CS16)}
FLAGS = {f: case("flag_variants_%d" % f, O.MODEL_DEFAULT, 1536000, 32768, 6, flags=f, seed=11)
         for f in (O.FLAG_AFC_WIDE | O.FLAG_DROOP, O.FLAG_PS_EMA, O.FLAG_PS_EMA | O.FLAG_DROOP, 0)}
SMALL = [case("small_chunks_m%d" % m, m, 1536000, 4096, 48, seed=7) for m in (O.MODEL_DEFAULT, O.MODEL_STANDARD)]
MULTI = case("multi_sentence", O.MODEL_DEFAULT, 1536000, 65536, 6, seed=31, multi=True)
# one stream, the chunk length changing from push to push (in granules of the rate: 64 at 1536k): a chunk shorter than the
# front end's history, chunks either side of a 48 kHz CGF block (256 granules), one granule, a long one, no power of two
SCHEDULE = [5, 24, 23, 1024, 1, 257, 255, 1017, 613, 1]
SCHED_RATES = {1536000: 64, 96000: 4, 6144000: 256}
SCHEDULES = {(m, fs, f): case("schedule_m%d_%d_f%d" % (m, fs, f), m, fs, 0, 0, fmt=f, seed=61, schedule=[g * u for u in SCHEDULE])
             for m in (O.MODEL_DEFAULT, O.MODEL_STANDARD, O.MODEL_BASE) for fs, g in SCHED_RATES.items()
             for f in ((O.FMT_CF32, O.FMT_CU8) if fs == 1536000 else (O.FMT_CF32,))}
# ModelChallenger: its ten decoders (with the publisher of every message), its CGF / FIR17 / FM / Filter 37 taps and the coherent
# decoders' inputs; AB at 96 and 1536 kS/s, AFC_WIDE on and off, a changing submit schedule, and single-channel mode at 48 kS/s
CHALLENGER = {"96k": case("challenger_96k", O.MODEL_CHALLENGER, 96000, 4096, 24, seed=41),
              "1536k": case("challenger_1536k", O.MODEL_CHALLENGER, 1536000, 65536, 4, seed=43),
              "96k_afc_narrow": case("challenger_96k_afc_narrow", O.MODEL_CHALLENGER, 96000, 4096, 24, flags=O.FLAG_PS_EMA | O.FLAG_DROOP,
                                     seed=47),
              "schedule_96k": case("challenger_schedule_96k", O.MODEL_CHALLENGER, 96000, 0, 0, seed=61, schedule=[4 * u for u in SCHEDULE]),
              "x_48k": case("challenger_x_48k", O.MODEL_CHALLENGER, 48000, 2048, 24, seed=53, x_mode=True)}


@pytest.mark.parametrize("model", [O.MODEL_DEFAULT, O.MODEL_STANDARD, O.MODEL_BASE])
def test_models_1536k(built, model):
    assert compare(MODELS[model]) >= (1 if model == O.MODEL_BASE else 3)


@pytest.mark.parametrize("fs,N", [(96000, 4096), (192000, 8192), (288000, 12288), (384000, 16384), (768000, 32768),
                                  (3072000, 131072), (6000000, 262144), (6144000, 262144), (12288000, 524288),
                                  (2000000, 65536), (250000, 16384)])
def test_rates_default(built, fs, N):
    # includes the /3 DownsampleKFilter path (288k) and interpolated non-bucket rates (6 MSPS AirSpy shape, 2 M, 250 k)
    assert compare(RATES[(fs, N)]) >= 1


@pytest.mark.parametrize("fmt", [O.FMT_CU8, O.FMT_CS8, O.FMT_CS16])
def test_integer_formats(built, fmt):
    assert compare(FORMATS[fmt]) >= 2


@pytest.mark.parametrize("flags", [O.FLAG_AFC_WIDE | O.FLAG_DROOP, O.FLAG_PS_EMA, O.FLAG_PS_EMA | O.FLAG_DROOP, 0])
def test_flag_variants(built, flags):
    compare(FLAGS[flags])


def test_small_chunks(built):
    # 48 kHz count per chunk (128) below one CGF block (512): re-blocking paths
    assert compare(SMALL[0]) >= 1
    compare(SMALL[1])


def test_multi_sentence(built):
    # 424-bit messages -> two sentences with the sequence id of Message.cpp:28-39
    n = compare(MULTI)
    assert n >= 2


@pytest.mark.parametrize("key", sorted(SCHEDULES), ids=lambda k: "m%d_%d_f%d" % k)
def test_changing_chunk_lengths(built, key):
    # the GPU tests of changing submit lengths fall back on the port where the reference was not built
    assert compare(SCHEDULES[key]) >= 1


@pytest.mark.parametrize("key", sorted(CHALLENGER))
def test_challenger(built, key):
    assert compare(CHALLENGER[key]) >= 2


if __name__ == "__main__":  # regenerate the stored outputs from the reference (needs oracle/_ref): all cases, or those named
    import sys
    assert O.have_ref() and OX.have_refx(), "oracle/_ref not built"
    out = load_store()
    out.update({name: digest(O.RefModel, *args, **kw) for name, args, kw in CASES if len(sys.argv) < 2 or name in sys.argv[1:]})
    with open(STORE, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
        f.write("\n")
