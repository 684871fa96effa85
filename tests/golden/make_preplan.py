#!/usr/bin/env python
"""Generates tests/golden/preplan.json: every front-end planning decision the host can see without a GPU, over a grid of
configurations.  For each (model, channel mode, DSK, FP_DS, format, sample rate) it records the submit granule
(aisgpu_chunk_granule) or the refusal, and for accepted configurations which device-batch placements (base offset, stride)
aisgpu_check_device_batch accepts or refuses, with the message.  tests/test_preplan.py replays the grid against the library.

Run against a built library:  python tests/golden/make_preplan.py   (AISGPU_LIB selects another build)"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "ais-catcher_b200"))
import aisgpu  # noqa: E402

PREPLAN = os.path.join(HERE, "preplan.json")

MODELS = [aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2]
MODES = [aisgpu.MODE_AB, aisgpu.MODE_X]
FORMATS = [aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16]
# every bucket of AB (with and without DSK) and of mode X, a rate between each neighbouring pair, the rates the resampler cases are
# tested at, the edges, and one rate either side of each limit (12K and 192K in X, 96K and 12288K in AB, 12K and 48K for -m 3)
BUCKETS = [48000, 96000, 192000, 288000, 384000, 576000, 768000, 1152000, 1536000, 2304000, 3072000, 6144000, 12288000]
BETWEEN = [(a + b) // 2 for a, b in zip(BUCKETS, BUCKETS[1:])]
OTHER = [12000, 24000, 44100, 250000, 1000000, 2000000, 6000000,
         11999, 12001, 47999, 48001, 95999, 96001, 191999, 192001, 12287999, 12288001]
RATES = sorted(set(BUCKETS + BETWEEN + OTHER))
BASE = 1 << 32  # a device address aligned to everything the rule asks for
# (byte offset from BASE, stride in samples): aligned, one and two samples off for every format, 16-byte rows or not, an odd
# stride, and a batch wider than FP_DS's 64 GiB
PLACEMENTS = [(0, 65536), (2, 65536), (4, 65536), (8, 65536), (16, 65536), (0, 65537), (0, 65538), (0, 65540), (0, 1 << 35)]


def grid():
    for model in MODELS:
        for mode in MODES:
            for dsk in (0, 1):
                for fp_ds in (0, 1):
                    for fmt in FORMATS:
                        for rate in RATES:
                            yield model, mode, dsk, fp_ds, fmt, rate


def granule(model, mode, dsk, fp_ds, fmt, rate):
    """The granule, or the refusal as the binding raises it."""
    try:
        return aisgpu.chunk_granule(rate, model=model, dsk=dsk, fp_ds=fp_ds, fmt=fmt, channel_mode=mode)
    except aisgpu.AisGpuError as e:
        return str(e)


def placement(model, mode, dsk, fp_ds, fmt, rate, off, stride):
    """Empty if the batch may lie there, else the refusal."""
    try:
        aisgpu.check_device_batch(BASE + off, stride, sample_rate=rate, model=model, fmt=fmt, dsk=dsk, fp_ds=fp_ds, channel_mode=mode)
        return ""
    except aisgpu.AisGpuError as e:
        return str(e)


def key(model, mode, dsk, fp_ds, fmt):
    return "%d,%d,%d,%d,%d" % (model, mode, dsk, fp_ds, fmt)


def main():
    messages, sets = [], []

    def index(table, item):
        if item not in table:
            table.append(item)
        return table.index(item)

    rows = {}
    for case in grid():
        g = granule(*case)
        if isinstance(g, str):  # refused: [-1 - message]
            entry = [-1 - index(messages, g)]
        else:  # accepted: [granule, placement set], a set holding per PLACEMENTS entry -1 (accepted) or the message
            entry = [g, index(sets, [-1 if not m else index(messages, m) for m in (placement(*case, off, st) for off, st in PLACEMENTS)])]
        rows.setdefault(key(*case[:5]), []).append(entry)
    with open(PREPLAN, "w") as f:
        f.write('{"generator": "tests/golden/make_preplan.py",\n')
        f.write('"rows": "model,channel_mode,dsk,fp_ds,format -> per sample_rate [granule, placement set] or [-1 - message]",\n')
        f.write('"sample_rates": %s,\n"base": %d,\n"placements": %s,\n' % (json.dumps(RATES), BASE, json.dumps(PLACEMENTS)))
        f.write('"messages": [\n%s],\n' % ",\n".join(json.dumps(m) for m in messages))
        f.write('"placement_sets": [\n%s],\n' % ",\n".join(json.dumps(s) for s in sets))
        f.write('"cases": {\n%s}}\n' % ",\n".join('"%s": %s' % (k, json.dumps(v, separators=(",", ":"))) for k, v in rows.items()))
    print("%d rows x %d rates, %d messages, %d placement sets -> %s" % (len(rows), len(RATES), len(messages), len(sets), PREPLAN))


if __name__ == "__main__":
    main()
