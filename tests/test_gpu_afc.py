"""-m gpu: frequency correction over its whole range, bit for bit (tolerance 0) against the compiled reference (oracle/_ref), on
the stimuli of tests/afc_signals.py (tests/test_afc.py proves on the reference which branches they reach).

Every case is one engine whose rows are carrier offsets: the sweep (-12 .. +12 kHz, fine grids across the edges of the wide and the
narrow range), the drift row beside part of it, or slot-aligned traffic that locks the V2 engine's slot predictor.  After every
submit every tap the engine exposes is compared with the reference instance of its row: C, the CGF output, FIR17 and the decoder
inputs of ModelDefault, FM / Filter 37 of the FM chains, and the V2 engine's CGF / FIR17 / FIR37 arrays of the last block the
submit decoded (the reference records the last one); at rates with a resampler its output stream (PRE / PRE2).  At the end the
frames, their order, start/end counters and level / ppm bit patterns.
"""
import itertools

import numpy as np
import pytest

import afc_signals as A
import aisgpu
import oracle as O
import oracle_afc as OA
import oracle_x as OX
import parity_util as U

pytestmark = pytest.mark.gpu

AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS16
M0, M1, M2, M4, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2
HOW = ("submit", "submit_v", "submit_async", "submit_device")

# the sweep at fewer rows where the input is large (6 MS/s)
SWEEP_SHORT = [f for f in A.SWEEP if f in A.COARSE[::2] or abs(abs(f) - 9600.0) <= 100.0 or abs(abs(f) - 800.0) <= 50.0]
DRIFT_BESIDE = (-9600.0, -800.0, 0.0, 800.0, 9600.0)


class Case:
    def __init__(self, name, model, fs, fmt, N, rows, n48, mode=AB, afc_wide=True, ps_ema=True, fp_ds=False, weights=None,
                 schedule=None, how=("submit",), members=()):
        self.name, self.model, self.fs, self.fmt, self.N, self.rows, self.n48 = name, model, fs, fmt, N, rows, n48
        self.mode, self.afc_wide, self.ps_ema, self.fp_ds, self.weights = mode, afc_wide, ps_ema, fp_ds, weights
        self.schedule, self.how, self.members = schedule, how, members

    def __repr__(self):
        return self.name

    def kind(self):
        return A.X_ if self.mode == MX else A.AB

    def n(self):
        return self.n48 * self.fs // 48000

    def inputs(self):
        """complex64 rows of n() samples."""
        n, kind = self.n(), self.kind()
        if self.rows == "sweep":
            return A.rows(self.fs, n, A.SWEEP, kind=kind) + [A.edge_tones(self.fs, n, fz, 0, kind) for fz in A.EDGE_TONE_BINS]
        if self.rows == "sweep_short":
            return A.rows(self.fs, n, SWEEP_SHORT, kind=kind)
        if self.rows == "drift":
            return [A.drift(self.fs, n, 0, kind)] + A.rows(self.fs, n, DRIFT_BESIDE, seed=50, kind=kind)
        if self.rows == "slot":
            out = [A.slotted(self.fs, n, ph, k, kind=kind) for k, ph in enumerate(A.SLOT_PHASES[kind])]
            if self.mode == MX:  # a lock that decays in noise
                out.append(A.slotted(self.fs, n, A.SLOT_PHASES[kind][0], 7, kind=kind, misaligned=0))
            return out
        raise ValueError(self.rows)

    def flags(self, model, afc_wide, ps_ema):
        return (O.FLAG_PS_EMA if ps_ema else 0) | (O.FLAG_AFC_WIDE if afc_wide else 0) | O.FLAG_DROOP | (O.FLAG_FP_DS if self.fp_ds else 0)

    def reference(self, model=None, afc_wide=None, weights=None):
        model = self.model if model is None else model
        afc_wide = self.afc_wide if afc_wide is None else afc_wide
        weights = self.weights if weights is None else weights
        flags = self.flags(model, afc_wide, self.ps_ema)
        if weights is not None:
            return OA.RefModelAFC(model=model, sample_rate=self.fs, fmt=self.fmt, flags=flags, taps=True,
                                  mode="x" if self.mode == MX else "ab", weights=weights)
        if self.mode == MX:
            return OX.RefModelX(model=model, sample_rate=self.fs, fmt=self.fmt, flags=flags, taps=True)
        return O.RefModel(model=model, sample_rate=self.fs, fmt=self.fmt, flags=flags, taps=True)

    def have_reference(self):
        return (OX.have_refx() if self.mode == MX else O.have_ref()) and OA.have_ref("ab") and OA.have_ref("x")

    def engine(self, n_streams, max_chunk):
        kw = {}
        if self.weights is not None:
            kw = dict(dd_train=self.weights[0], dd_weight=self.weights[1])
        return aisgpu.Engine(model=self.model, sample_rate=self.fs, fmt=self.fmt, n_streams=n_streams, max_chunk=max_chunk,
                             ps_ema=self.ps_ema, afc_wide=self.afc_wide, taps=True, fp_ds=self.fp_ds, channel_mode=self.mode,
                             channels="XX" if self.mode == MX else "AB", **kw)

    def channels(self):
        return (0,) if self.mode == MX else (0, 1)

    def resampler(self):
        if self.mode == MX:
            return self.fs not in (48000, 96000, 192000)
        return self.fs not in (96000, 192000, 384000, 768000, 1536000, 3072000, 6144000, 12288000)

    def lengths(self):
        """Submit lengths in samples: N each, or the schedule cycled, until the run is used up."""
        n, out = self.n(), []
        cyc = itertools.cycle(self.schedule or [self.N])
        while True:
            k = next(cyc)
            if sum(out) + k > n:
                break
            out.append(k)
        return out


def v2_problems(eng, s, ref, label, channels):
    """The V2 engine's arrays of the last block the submit decoded against what the reference recorded for it."""
    out = []
    for ch in channels:
        for name, g, w in (("V2.CGF", eng.tap(aisgpu.TAP_CGF, s, ch), ref.tap_c(O.TAP_CGF_A + ch)),
                           ("V2.FIR17", eng.tap(aisgpu.TAP_FIR, s, ch), ref.tap_c(O.TAP_FC_A + ch)),
                           ("V2.FIR37", eng.tap(aisgpu.TAP_FM, s, ch, dtype=np.float32), ref.tap_f(O.TAP_FR_A + ch))):
            if len(g) % 512 or len(w) not in (0, 512) or (len(g) == 0) != (len(w) == 0) or not U.bits_equal(g[len(g) - len(w):], w):
                out.append((name, label, s, ch, len(g), len(w)) + U.first_diff(g[len(g) - len(w):], w))
    return out


def submit(eng, how, blk, n, per, keep):
    import torch
    batch = np.ascontiguousarray(np.stack(blk))
    if how == "submit":
        eng.submit(batch, n)
    elif how == "submit_v":
        eng.submit_v(blk, n)
    elif how == "submit_async":
        t = torch.from_numpy(batch.view(np.uint8)).pin_memory()
        keep.append(t)
        eng.submit_async_ptr(t.data_ptr(), n)
    else:
        t = torch.from_numpy(batch.view(np.uint8)).cuda()
        torch.cuda.synchronize()
        keep.append(t)
        eng.submit_device(t.data_ptr(), n, n)
    eng.sync()


def run(case):
    if not case.have_reference():
        pytest.skip("frequency correction is checked against the compiled reference only")
    xs = case.inputs()
    rows = [A.to_raw(x, case.fmt) for x in xs]
    B, per = len(rows), rows[0][1]
    lengths = case.lengths()
    eng = case.engine(B, max(lengths))
    # (engine, model, reference instances) of the leader and of each group member
    units = [(eng, case.model, [case.reference() for _ in range(B)])]
    for m in case.members:
        units.append((eng.attach(**m), m["model"], [case.reference(m["model"], m.get("afc_wide", True)) for _ in range(B)]))
    rs = case.resampler()
    problems = []
    got = [[[] for _ in range(B)] for _ in units]
    want = [[[] for _ in range(B)] for _ in units]
    pre_got, pre_want = [[] for _ in range(B)], [[] for _ in range(B)]
    keep, pos = [], 0
    for c, n in enumerate(lengths):
        blk = [r[pos * per:(pos + n) * per] for r, _ in rows]
        pos += n
        submit(eng, case.how[c % len(case.how)], blk, n, per, keep)
        label = "submit %d" % c
        for u, (e, model, refs) in enumerate(units):
            for s in range(B):
                refs[s].push(blk[s])
                if rs:
                    if u == 0:
                        pre_got[s].append(e.tap(aisgpu.TAP_PRE, s, 0))
                        pre_want[s].append(refs[s].tap_c(O.TAP_DSK if case.fs == 288000 else O.TAP_US))
                    continue
                problems += U.compare_taps(e, s, refs[s], model, label, case.channels())
                if model == M11:
                    problems += v2_problems(e, s, refs[s], label, case.channels())
        for u, (e, model, refs) in enumerate(units):
            for s in range(B):
                want[u][s] += refs[s].messages()
            for m in e.poll():
                got[u][m.stream].append(m)
        if len(problems) > 50:
            break
    for e, _, _ in units[:0:-1]:
        e.close()
    eng.close()
    if rs:
        for s in range(B):
            a, b = np.concatenate(pre_got[s]), np.concatenate(pre_want[s])
            k = min(len(a), len(b))
            if k < 1000 or not U.bits_equal(a[:k], b[:k]):
                problems.append(("PRE", "stream %d" % s, len(a), len(b)) + U.first_diff(a[:k], b[:k]))
    for u in range(len(units)):
        problems += [("unit %d" % u,) + p for p in U.compare_frames(got[u], want[u])]
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    nframes = sum(len(w) for wu in want for w in wu)
    assert nframes > 0
    return nframes


N48 = A.SWEEP_N48
V2_SCHEDULE = [16384, 40960, 8192 + 64 * 3, 16384 * 3 - 64, 64 * 5, 16384 + 8192]  # blocks of 512 end anywhere in a submit
CASES = [
    # the sweep: models 2 (wide / narrow, PS_EMA on / off), 4, 11, 0, 1 on the streaming CF32 front end at 1536 kS/s
    Case("sweep_m2_wide", M2, 1536000, CF32, 65536, "sweep", N48),
    Case("sweep_m2_narrow", M2, 1536000, CF32, 65536, "sweep", N48, afc_wide=False),
    Case("sweep_m2_noema", M2, 1536000, CF32, 65536, "sweep", N48, ps_ema=False),
    Case("sweep_m2_narrow_noema", M2, 1536000, CF32, 65536, "sweep", N48, afc_wide=False, ps_ema=False),
    Case("sweep_m4", M4, 1536000, CF32, 65536, "sweep", N48),
    Case("sweep_m4_narrow", M4, 1536000, CF32, 65536, "sweep", N48, afc_wide=False),
    Case("sweep_m11", M11, 1536000, CF32, 16384, "sweep", N48),
    Case("sweep_m0", M0, 1536000, CF32, 65536, "sweep", N48),
    Case("sweep_m1", M1, 1536000, CF32, 65536, "sweep", N48),
    # other front ends
    Case("sweep_cu8_fpds_m2", M2, 1536000, CU8, 65536, "sweep", N48, fp_ds=True),
    Case("sweep_tiled384_cs16_m2", M2, 384000, CS16, 16384, "sweep", N48),
    Case("sweep_us240_m2", M2, 240000, CF32, 20480, "sweep_short", N48),
    Case("sweep_dsk288_m2", M2, 288000, CF32, 12288, "sweep_short", N48),
    Case("sweep_x48_m2", M2, 48000, CF32, 4096, "sweep", N48, mode=MX),
    Case("sweep_x48_m11", M11, 48000, CF32, 512, "sweep", N48, mode=MX),
    Case("sweep_x96_m4", M4, 96000, CF32, 8192, "sweep", N48, mode=MX),
    Case("sweep_x96_m0", M0, 96000, CF32, 8192, "sweep", N48, mode=MX),
    # the drift row, submit lengths that change from call to call through all four submit paths
    Case("drift_m2", M2, 1536000, CF32, None, "drift", A.DRIFT_N48 // 4, schedule=[65536, 16384 * 5 + 64 * 3, 64 * 9, 131072 - 64],
         how=HOW),
    Case("drift_m11", M11, 1536000, CF32, None, "drift", A.DRIFT_N48 // 4, schedule=V2_SCHEDULE, how=HOW),
    # slot-aligned traffic in model 11: one block per submit, then submit lengths that end on any block of the slot cycle
    Case("slot_m11", M11, 1536000, CF32, 16384, "slot", A.SLOT_N48),
    Case("slot_m11_sched", M11, 1536000, CF32, None, "slot", A.SLOT_N48, schedule=V2_SCHEDULE),
    Case("slot_m11_weights", M11, 1536000, CF32, 16384, "slot", A.SLOT_N48, weights=(0.5, 0.95)),
    Case("slot_x48_m11", M11, 48000, CF32, 512, "slot", A.SILENT_N48, mode=MX),
    # a group on the sweep's front end: every member equals its standalone reference
    Case("sweep_group", M2, 1536000, CF32, 16384, "sweep", N48,
         members=(dict(model=M2, afc_wide=False), dict(model=M4), dict(model=M11))),
]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_afc(built, case):
    run(case)
