"""CPU: every front-end planning decision visible from the host, replayed against tests/golden/preplan.json.  Over models
0/1/2/3/4/11, AB and X, DSK and FP_DS off and on, all four formats and a rate list of every bucket, a rate between each pair,
the resampler test rates and both sides of every limit, the submit granule (or the refusal) and which device-batch placements
are accepted (or refused, and why) must not change.  tests/golden/make_preplan.py writes the fixture."""
import json
import os

import pytest

import aisgpu

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "preplan.json")) as f:
    PLAN = json.load(f)
MODELS = sorted({int(k.split(",")[0]) for k in PLAN["cases"]})
MODES = sorted({int(k.split(",")[1]) for k in PLAN["cases"]})


def outcome(call, *args, **kw):
    try:
        return call(*args, **kw)
    except aisgpu.AisGpuError as e:
        return str(e)


@pytest.mark.parametrize("mode", MODES, ids=lambda m: "X" if m == aisgpu.MODE_X else "AB")
@pytest.mark.parametrize("model", MODELS)
def test_planner_table(built, model, mode):
    msgs, sets = PLAN["messages"], PLAN["placement_sets"]
    bad, n = [], 0
    for key, entries in PLAN["cases"].items():
        m, cm, dsk, fp_ds, fmt = map(int, key.split(","))
        if (m, cm) != (model, mode):
            continue
        for rate, e in zip(PLAN["sample_rates"], entries, strict=True):
            n += 1
            kw = dict(model=m, dsk=dsk, fp_ds=fp_ds, fmt=fmt, channel_mode=cm)
            g = outcome(aisgpu.chunk_granule, rate, **kw)
            want = msgs[-1 - e[0]] if e[0] < 0 else e[0]
            if g != want:
                bad.append("%s @%d: granule %r, want %r" % (key, rate, g, want))
                continue
            kw = dict(sample_rate=rate, model=m, fmt=fmt, dsk=dsk, fp_ds=fp_ds, channel_mode=cm)
            if e[0] < 0:  # a refused configuration is refused by the placement check with the same message
                got = [outcome(aisgpu.check_device_batch, PLAN["base"], 65536, **kw)]
                want = [g]
            else:
                got = [outcome(aisgpu.check_device_batch, PLAN["base"] + off, stride, **kw) for off, stride in PLAN["placements"]]
                want = [None if i < 0 else msgs[i] for i in sets[e[1]]]
            if got != want:
                bad.append("%s @%d: placements %r, want %r" % (key, rate, got, want))
    assert n > 0
    assert not bad, "%d of %d cases differ:\n%s" % (len(bad), n, "\n".join(bad[:20]))
