"""Shared pieces of the bit-exact GPU tests: bit-pattern comparison of float arrays, the per-submit comparison of one engine
stream's taps with its own reference instance, and the frame comparison at the end of a run.  The reference instance must have
been created with taps on; reading a reference tap clears it, so compare_taps reads each one exactly once per submit."""
import numpy as np

import aisgpu
import oracle as O
import oracle_disc as OD


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def first_diff(a, b):
    """(first differing element, number of differing elements) over the common prefix; (-1, 0) when it is identical."""
    n = min(len(a), len(b))
    av = np.ascontiguousarray(a[:n]).view(np.uint32).reshape(n, -1)
    bv = np.ascontiguousarray(b[:n]).view(np.uint32).reshape(n, -1)
    d = np.nonzero((av != bv).any(axis=1))[0]
    return (int(d[0]), int(len(d))) if len(d) else (-1, 0)


def tap_pairs(model, ch, ps_ema=True):
    """(name, engine tap, engine channel argument, dtype, reference reader, reference tap) of one channel's taps.  C is the front
    end's 48 kHz output and exists for every model; the others are the back-end taps the reference harness records for the model."""
    f32, c64 = np.float32, np.complex64
    if model == aisgpu.MODEL_DISCRIMINATOR:  # oracle_disc: the real rows, Filter 37, the per-phase decoder inputs
        return [("C", aisgpu.TAP_C, ch, f32, "f", OD.TAP_RP + ch), ("FIR37", aisgpu.TAP_FIR, ch, f32, "f", O.TAP_FR_A + ch)] + \
            [("DEC%d" % ph, aisgpu.TAP_DEC, ch + 2 * ph, f32, "f", ch * 5 + ph) for ph in range(5)]
    t = [("C", aisgpu.TAP_C, ch, c64, "c", O.TAP_CA + ch)]
    if model == aisgpu.MODEL_DEFAULT:
        t += [("CGF", aisgpu.TAP_CGF, ch, c64, "c", O.TAP_CGF_A + ch), ("FIR17", aisgpu.TAP_FIR, ch, c64, "c", O.TAP_FC_A + ch)]
        t += [("DEC%d" % ph, aisgpu.TAP_DEC, ch + 2 * ph, f32, "f", ch * 5 + ph) for ph in range(5)]
    elif model in (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE):
        t += [("FM", aisgpu.TAP_FM, ch, f32, "f", O.TAP_FM_A + ch), ("FIR37", aisgpu.TAP_FIR, ch, f32, "f", O.TAP_FR_A + ch)]
        t += [("DEC%d" % ph, aisgpu.TAP_DEC, ch + 2 * ph, f32, "f", ch * 5 + ph) for ph in range(1 if model == aisgpu.MODEL_BASE else 5)]
    return t


def compare_taps(eng, s, ref, model, label, channels=(0, 1)):
    """Every tap of stream s of the last submit against what its reference instance recorded in the same block.  Returns a list of
    problems (name, label, stream, channel, engine length, reference length, first differing index, differing elements)."""
    problems = []
    for ch in channels:
        for name, tap, arg, dt, kind, rtap in tap_pairs(model, ch):
            got = eng.tap(tap, s, arg, dtype=dt)
            want = ref.tap_c(rtap) if kind == "c" else ref.tap_f(rtap)
            if not bits_equal(got, want):
                problems.append((name, label, s, ch, len(got), len(want)) + first_diff(got, want))
    return problems


def frame_key(m):
    return (m.key(), m.start_idx, m.end_idx, int(np.float32(m.level).view(np.uint32)), int(np.float32(m.ppm).view(np.uint32)))


def compare_frames(got, want):
    """Per-stream frame lists (aisgpu.Msg / oracle.Msg, in emission order): payload, NMEA, channel, start/end counters and the
    level / ppm bit patterns.  Returns a list of problems."""
    problems = []
    for s, (g, w) in enumerate(zip(got, want)):
        g, w = [frame_key(m) for m in g], [frame_key(m) for m in w]
        if g != w:
            problems.append(("MSG", s, len(g), len(w), [x for x in g if x not in w][:2], [x for x in w if x not in g][:2]))
    return problems
