"""-m gpu: the edge-case stimuli of tests/edge_signals.py through every front-end kernel family and every back end, bit for bit
(tolerance 0) against the compiled reference (oracle/_ref).

Every case is one engine over an odd batch: the edge stimuli on the even rows, ordinary traffic (aissynth.random_stream,
mode_x_util.x_stream, disc_util.stereo) on the odd rows between them, so a silent row sits beside loud ones in every warp that spans
rows.  After every submit every tap the engine exposes is compared with the reference instance of its row (the V2 engine's
per-block CGF / FIR17 / FIR37 arrays too; at rates with a resampler its output stream, PRE / PRE2); at the end the frames, their
order, start/end counters and level / ppm bit patterns.  Every 48 kHz block has 37 samples or more (the Filter 37 short-block
divergence is pinned in tests/test_gpu_submit_shapes.py).
"""
import numpy as np
import pytest

import aisgpu
import aissynth as S
import disc_util as D
import edge_signals as E
import mode_x_util as X
import oracle as O
import oracle_disc as OD
import oracle_x as OX
import parity_util as U

pytestmark = pytest.mark.gpu

AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16
M0, M1, M2, M3, M4, M11 = (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR,
                           aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2)
BASIC = ["silence", "gaps", "clipped"]


class Case:
    def __init__(self, name, model, fs, fmt, N, nchunks, kinds, mode=AB, ps_ema=True, dsk=False, fp_ds=False):
        self.name, self.model, self.fs, self.fmt, self.N, self.nchunks, self.kinds = name, model, fs, fmt, N, nchunks, kinds
        self.mode, self.ps_ema, self.dsk, self.fp_ds = mode, ps_ema, dsk, fp_ds

    def __repr__(self):
        return self.name

    def kind(self):
        return E.DISC if self.model == M3 else (E.X_ if self.mode == MX else E.AB)

    def resampler(self):
        """The reference's tap of the resampler output (None where the per-submit taps line up)."""
        if self.model == M3:
            return None if self.fs == 48000 else O.TAP_US
        if self.mode == MX:
            return None if self.fs in (48000, 96000, 192000) else O.TAP_US
        if self.fs == 288000 or (self.dsk and self.fs in (576000, 1152000, 2304000)):
            return O.TAP_DSK
        return None if self.fs in (96000, 192000, 384000, 768000, 1536000, 3072000, 6144000, 12288000) else O.TAP_US

    def flags(self):
        return ((O.FLAG_PS_EMA if self.ps_ema else 0) | O.FLAG_AFC_WIDE | O.FLAG_DROOP | (O.FLAG_DSK if self.dsk else 0)
                | (O.FLAG_FP_DS if self.fp_ds else 0))

    def reference(self):
        if self.model == M3:
            return OD.RefModelDisc(sample_rate=self.fs, fmt=self.fmt, taps=True)
        if self.mode == MX:
            return OX.RefModelX(model=self.model, sample_rate=self.fs, fmt=self.fmt, flags=self.flags(), taps=True)
        return O.RefModel(model=self.model, sample_rate=self.fs, fmt=self.fmt, flags=self.flags(), taps=True)

    def have_reference(self):
        return OD.have_refd() if self.model == M3 else (OX.have_refx() if self.mode == MX else O.have_ref())

    def engine(self, n_streams):
        return aisgpu.Engine(model=self.model, sample_rate=self.fs, fmt=self.fmt, n_streams=n_streams, max_chunk=self.N,
                             ps_ema=self.ps_ema, taps=True, dsk=self.dsk, fp_ds=self.fp_ds, channel_mode=self.mode,
                             channels="XX" if self.mode == MX and self.model != M3 else "AB")

    def channels(self):
        return (0,) if self.mode == MX and self.model != M3 else (0, 1)

    def inputs(self):
        """Per row (raw array, elements per sample): the edge stimuli on the even rows, ordinary traffic on the odd ones."""
        n, kind, g = self.N * self.nchunks, self.kind(), self.granule()
        rows = []
        for i, k in enumerate(self.kinds):
            rows.append(E.make(k, self.fs, n, 100 + i, self.fmt, kind, submit=self.N, granule=g))
            if i + 1 < len(self.kinds):
                seed = 200 + i
                if kind == E.DISC:
                    rows.append(D.stream_input(self.fs, n, seed, self.fmt))
                elif kind == E.X_:
                    rows.append(X.stream_input(self.fs, n, seed, self.fmt))
                else:
                    rows.append(X.to_raw(S.random_stream(self.fs, n, seed, bursts_per_sec=(6, 12))[0], self.fmt))
        return rows

    def granule(self):
        return aisgpu.chunk_granule(self.fs, self.model, self.dsk, self.fp_ds, self.fmt, self.mode)


def v2_problems(eng, s, ref, label):
    """The V2 engine's per-block arrays of the submit: derotated samples, FIR17 and FIR37 outputs."""
    out = []
    for ch in (0, 1):
        for name, g, w in (("V2.CGF", eng.tap(aisgpu.TAP_CGF, s, ch), ref.tap_c(O.TAP_CGF_A + ch)),
                           ("V2.FIR17", eng.tap(aisgpu.TAP_FIR, s, ch), ref.tap_c(O.TAP_FC_A + ch)),
                           ("V2.FIR37", eng.tap(aisgpu.TAP_FM, s, ch, dtype=np.float32), ref.tap_f(O.TAP_FR_A + ch))):
            if not U.bits_equal(g, w):
                out.append((name, label, s, ch, len(g), len(w)) + U.first_diff(g, w))
    return out


def run(case):
    if not case.have_reference():
        pytest.skip("the edge stimuli are checked against the compiled reference only")
    rows = case.inputs()
    B, N, per = len(rows), case.N, rows[0][1]
    assert B % 2 == 1 and all(len(r) == N * case.nchunks * per for r, _ in rows)
    refs = [case.reference() for _ in range(B)]
    eng = case.engine(B)
    rs = case.resampler()
    problems = []
    got, want = [[] for _ in range(B)], [[] for _ in range(B)]
    pre_got = {t: [[] for _ in range(B)] for t in (aisgpu.TAP_PRE, aisgpu.TAP_PRE2)}
    pre_want = {t: [[] for _ in range(B)] for t in (O.TAP_US, O.TAP_DSK)}
    for c in range(case.nchunks):
        blk = [r[c * N * per:(c + 1) * N * per] for r, _ in rows]
        eng.submit(np.stack(blk), N)
        label = "submit %d" % c
        for s in range(B):
            refs[s].push(blk[s])
            if rs is None:
                problems += U.compare_taps(eng, s, refs[s], case.model, label, case.channels())
                if case.model == M11:
                    problems += v2_problems(eng, s, refs[s], label)
            else:
                for t in pre_got:
                    try:
                        pre_got[t][s].append(eng.tap(t, s, 0))
                    except aisgpu.AisGpuError:  # no second pre-stage at this rate
                        pass
                for t in pre_want:
                    if t == O.TAP_US or (case.model != M3 and case.mode == AB):  # the DSK tap exists in the AB harness only
                        pre_want[t][s].append(refs[s].tap_c(t))
        for s in range(B):
            want[s] += refs[s].messages()
        for m in eng.poll():
            got[m.stream].append(m)
    eng.close()
    if rs is not None:
        for s in range(B):
            g = {t: np.concatenate(v[s]) if v[s] else np.zeros(0, np.complex64) for t, v in pre_got.items()}
            w = {t: np.concatenate(v[s]) if v[s] else np.zeros(0, np.complex64) for t, v in pre_want.items()}
            # the engine's PRE is the first pre-stage: Upsample, or DownsampleKFilter where there is no Upsample; PRE2 the DSK behind it
            pairs = [("PRE", g[aisgpu.TAP_PRE], w[O.TAP_US] if len(w[O.TAP_US]) else w[O.TAP_DSK])]
            if len(w[O.TAP_US]) and len(w[O.TAP_DSK]):
                pairs.append(("PRE2", g[aisgpu.TAP_PRE2], w[O.TAP_DSK]))
            for name, a, b in pairs:
                n = min(len(a), len(b))
                if n < 1000 or not U.bits_equal(a[:n], b[:n]):
                    problems.append((name, "stream %d" % s, len(a), len(b)) + U.first_diff(a[:n], b[:n]))
    problems += U.compare_frames(got, want)
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    return sum(map(len, want))


CASES = [
    # streaming CF32 @1536K: every AB back end
    Case("st1536_cf32_m2", M2, 1536000, CF32, 65536, 12, BASIC + ["dc", "carrier_bin", "subnormal"]),
    Case("st1536_cf32_m2_more", M2, 1536000, CF32, 65536, 8, ["signed_zero", "loud", "carrier_between_traffic", "real_only",
                                                              "dc_traffic"]),
    Case("st1536_cf32_m2_noema", M2, 1536000, CF32, 65536, 12, BASIC + ["carrier_bin_traffic", "subnormal"], ps_ema=False),
    Case("st1536_cf32_m0", M0, 1536000, CF32, 65536, 12, BASIC + ["signed_zero", "subnormal", "loud_max"]),
    Case("st1536_cf32_m1", M1, 1536000, CF32, 65536, 12, BASIC + ["dc", "subnormal"]),
    Case("st1536_cf32_m4", M4, 1536000, CF32, 65536, 12, BASIC + ["carrier_bin", "loud"]),
    # one 512-sample block per submit: the reference records the arrays of the last block of each submit
    Case("st1536_cf32_m11", M11, 1536000, CF32, 16384, 48, BASIC + ["signed_zero", "subnormal", "carrier_between"]),
    # streaming integer front end
    Case("st1536_cu8_m0", M0, 1536000, CU8, 65536, 12, BASIC + ["quantised", "dc_traffic"]),
    Case("st1536_cu8_m2", M2, 1536000, CU8, 65536, 12, BASIC + ["quantised", "dc"]),
    Case("st1536_cs8_m0", M0, 1536000, CS8, 65536, 12, BASIC + ["dc"]),
    Case("st1536_cs8_m2", M2, 1536000, CS8, 65536, 12, BASIC + ["dc_traffic"]),
    # FP_DS: the packed-uint16 CIC stages at full scale
    Case("fpds_cu8_m0", M0, 1536000, CU8, 65536, 12, BASIC + ["quantised", "dc"], fp_ds=True),
    Case("fpds_cu8_m2", M2, 1536000, CU8, 65536, 12, BASIC + ["quantised", "dc_traffic"], fp_ds=True),
    # tiled front end
    Case("tiled384_cs16_m2", M2, 384000, CS16, 16384, 12, BASIC + ["dc_traffic", "carrier_bin"]),
    # pre-stages: DownsampleKFilter on the raw input, Upsample, DSK behind two CIC stages
    Case("dsk288_m2", M2, 288000, CF32, 12288, 12, BASIC),
    Case("us6000_m2", M2, 6000000, CF32, 262144, 12, BASIC),
    Case("dsk1152_cu8_m2", M2, 1152000, CU8, 49152, 12, BASIC, dsk=True),
    # single-channel mode
    Case("x48_m0", M0, 48000, CF32, 4096, 12, BASIC + ["real_only", "carrier_bin"], mode=MX),
    Case("x48_m2", M2, 48000, CF32, 4096, 12, BASIC + ["real_only", "carrier_between"], mode=MX),
    Case("x96_m0", M0, 96000, CF32, 8192, 12, BASIC + ["real_only"], mode=MX),
    Case("x96_m2", M2, 96000, CF32, 8192, 12, BASIC + ["real_only", "signed_zero"], mode=MX),
    Case("x24_m0", M0, 24000, CF32, 2048, 12, BASIC + ["real_only"], mode=MX),
    Case("x24_m2", M2, 24000, CF32, 2048, 12, BASIC + ["real_only"], mode=MX),
    # the FM-discriminator input
    Case("disc48_cs16", M3, 48000, CS16, 4096, 12, BASIC + ["quantised"]),
    Case("disc48_cu8", M3, 48000, CU8, 4096, 12, BASIC + ["dc"]),
    Case("disc441_cf32", M3, 44100, CF32, 4416, 12, BASIC + ["signed_zero"]),
]


@pytest.mark.parametrize("case", CASES, ids=[c.name for c in CASES])
def test_edge_signals(built, case):
    run(case)


@pytest.mark.xfail(strict=True, reason="known divergence: where the squared 48 kHz samples overflow binary32 (CF32 input x 2^64), "
                                       "the reference's SquareFreqOffsetCorrection spectrum differs from the engine's (DESIGN.md section 2)")
def test_cgf_overflow(built):
    # ModelStandard at the same scale is bit-exact (st1536_cf32_m0 above): only the CGF estimate of ModelDefault diverges
    run(Case("st1536_cf32_m2_overflow", M2, 1536000, CF32, 65536, 4, ["loud_max"]))
