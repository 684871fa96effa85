"""-m gpu: one engine fed submits of changing length, and device batches at changing strides and base offsets, bit for bit
(tolerance 0) against the unmodified reference (oracle/_ref; the pinned C port for models 0 / 1 / 2 in AB mode where the reference
was not built).

The C ABI lets n_samples change from call to call at every rate without a resampler, and lets a device batch lie at any place its
placement rule accepts (include/aisgpu.h, aisgpu_submit_device).  Both reach state that a fixed-length, packed run never moves:
the Rotate phasor table built ahead for a submit of the same length, the lane planner and the switch between the streaming and the
tiled front end, the warm-up tail when a submit is shorter than the history, the CGF 512-block carry, the 5-phase deinterleaver's
absolute alignment, the V2 block carry, the DownsampleKFilter phase, and the front-end kernels chosen by alignment.

A  length schedules: every tap of every submit against the reference fed the same blocks; then the same schedule without taps
   (pipelined back end) through all four submit entry points, with polls skipped between some submits; frames, NMEA, start/end
   counters and level/ppm bit patterns at the end.  At rates with a resampler a changed length is EINVAL and the engine goes on.
B  device-batch placement: strides N .. 3N and the smallest allowed base offset, changing between the submits of one engine,
   against the reference and against a packed aisgpu_submit engine fed the same data.
C  rejection: a batch the placement rule refuses is EINVAL with a reason, the handle is untouched and the next submit bit-exact.
   Gated on aisgpu_check_device_batch, so a library without the rule is never handed a misaligned batch.
"""
import numpy as np
import pytest

import aisgpu
import aissynth as S
import disc_util as D
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
BPS = {CF32: 8, CU8: 2, CS8: 2, CS16: 4}
B = 3  # streams: the rows >= 1 are where a wrong row stride shows


class Fam:
    """One engine configuration: model, rate, format, channel mode, -go DSK / FP_DS / PS_EMA."""

    def __init__(self, name, model, fs, fmt=CF32, mode=AB, dsk=False, fp_ds=False, ps_ema=True):
        self.name, self.model, self.fs, self.fmt, self.mode = name, model, fs, fmt, mode
        self.dsk, self.fp_ds, self.ps_ema = dsk, fp_ds, ps_ema

    def __repr__(self):
        return self.name

    def granule(self):
        return aisgpu.chunk_granule(self.fs, self.model, self.dsk, self.fp_ds, self.fmt, self.mode)

    def resampler(self):
        """The reference's tap of the resampler output this rate has (None: no resampler; the per-submit taps line up)."""
        if self.model == M3:
            return None if self.fs == 48000 else O.TAP_US
        if self.mode == MX:
            return None if self.fs in (48000, 96000, 192000) else O.TAP_US
        buckets = (96000, 192000, 384000, 768000, 1536000, 3072000, 6144000, 12288000)
        if self.fs in (288000,) or (self.dsk and self.fs in (576000, 1152000, 2304000)):
            return O.TAP_DSK
        return None if self.fs in buckets else O.TAP_US

    def history(self):
        """Warm-up history of the front end in input samples (aisgpu.cu plan_frontend) at the exact AB buckets, else 4 granules."""
        g = self.granule()
        if self.mode != AB or self.model == M3 or self.resampler() is not None or self.fp_ds:
            return 4 * g
        k, hk = int(np.log2(self.fs // 96000)), 17
        for _ in range(k):
            hk = 2 * hk + 5
        q = 1 << (k + 2)
        return (hk + q - 1) // q * q

    def flags(self):
        return ((O.FLAG_PS_EMA if self.ps_ema else 0) | O.FLAG_AFC_WIDE | O.FLAG_DROOP | (O.FLAG_DSK if self.dsk else 0)
                | (O.FLAG_FP_DS if self.fp_ds else 0))

    def reference(self):
        if self.model == M3:
            if not OD.have_refd():
                pytest.skip("the FM-discriminator input model is checked against the compiled reference only")
            return OD.RefModelDisc(sample_rate=self.fs, fmt=self.fmt, taps=True)
        if self.mode == MX:
            if not OX.have_refx():
                pytest.skip("single-channel mode is checked against the compiled reference only")
            return OX.RefModelX(model=self.model, sample_rate=self.fs, fmt=self.fmt, flags=self.flags(), taps=True)
        if O.have_ref():
            return O.RefModel(model=self.model, sample_rate=self.fs, fmt=self.fmt, flags=self.flags(), taps=True)
        if self.model in (M0, M1, M2) and not (self.dsk or self.fp_ds):
            return O.PortModel(model=self.model, sample_rate=self.fs, fmt=self.fmt, flags=self.flags(), taps=True)
        pytest.skip("checked against the compiled reference only")

    def engine(self, n_streams, max_chunk, taps):
        return aisgpu.Engine(model=self.model, sample_rate=self.fs, fmt=self.fmt, n_streams=n_streams, max_chunk=max_chunk,
                             ps_ema=self.ps_ema, taps=taps, dsk=self.dsk, fp_ds=self.fp_ds, channel_mode=self.mode,
                             channels="XX" if self.mode == MX and self.model != M3 else "AB")

    def channels(self):
        return (0,) if self.mode == MX and self.model != M3 else (0, 1)

    def inputs(self, n, seed):
        """Per stream (raw array, array elements per sample) of n samples."""
        if self.model == M3:
            return [D.stream_input(self.fs, n, seed + s, self.fmt) for s in range(B)]
        if self.mode == MX:
            return [X.stream_input(self.fs, n, seed + s, self.fmt) for s in range(B)]
        return [X.to_raw(S.random_stream(self.fs, n, seed + s, bursts_per_sec=(6, 12))[0], self.fmt) for s in range(B)]


def ref_messages(refs, out):
    for s, r in enumerate(refs):
        out[s] += r.messages()


def resampler_problems(f, got, want, label):
    """The resampler's output stream against the reference's (it holds a partial block back: the common prefix)."""
    g = np.concatenate(got) if got else np.zeros(0, np.complex64)
    w = np.concatenate(want) if want else np.zeros(0, np.complex64)
    n = min(len(g), len(w))
    if len(w) > len(g) or not U.bits_equal(g[:n], w[:n]):  # DownsampleKFilter sends whole blocks of 8192: w may be empty
        return [("PRE", label, len(g), len(w)) + U.first_diff(g[:n], w[:n])]
    return []


def fm_floor(f):
    """Shortest submit whose 48 kHz block has >= 37 samples where the model runs the reference's Filter 37 on it (models 0, 1, 3).
    Filter::Receive takes a block shorter than its taps sample by sample in a 37-sample window that is not the history the block
    after it reads (DSP.cpp:247-280); the engine does not reproduce that (test_fm_filter_short_blocks below)."""
    g = f.granule()
    if f.model not in (M0, M1, M3) or f.resampler() is not None:
        return g
    n = -(-37 * f.fs // 48000)
    return -(-n // g) * g


# ---- A: length schedules ------------------------------------------------------------------------------------------------

def fixed_schedules(g):
    """Adversarial schedules in granules (at 1536 kS/s, g = 64: one CGF block is 256 g, the history 6 g)."""
    return {
        "long_short_long": [1024 * g, g, 1024 * g],
        "granule_x40": [g] * 40,
        "tiled_streaming_switch": [5 * g, 24 * g, 23 * g, 2048 * g],  # a tiled chunk 0, then across the switch both ways
        "straddle_cgf_block": [257 * g, 255 * g, 257 * g, 255 * g, 3 * g],
        "no_pow2_lane_split": [1017 * g, 613 * g],
    }


def random_schedule(f, seed, n=10):
    """Seeded draws from: one granule, shorter than the history, one to four histories, not a whole number of 48 kHz CGF blocks,
    max_chunk."""
    g, P = f.granule(), f.history()
    M = 1024 * g
    cgf = 512 * max(1, f.fs // 48000) if f.mode == AB else 512
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        kind = int(rng.integers(5))
        if kind == 0:
            v = g
        elif kind == 1:
            v = g * int(rng.integers(1, max(2, P // g)))
        elif kind == 2:
            v = g * int(rng.integers(max(1, P // g), max(2, 4 * P // g + 1)))
        elif kind == 3:
            v = g * int(rng.integers(1, M // g))
            if v % cgf == 0:
                v += g
        else:
            v = M
        out.append(min(v, M))
    return out


def run_schedule(f, schedule, seed, floor=True):
    """Pass 1: taps on, aisgpu_submit, every tap of every submit.  Pass 2: taps off (pipelined back end), the four entry points in
    turn, polls skipped between some submits.  Frames of both passes against the reference's.  floor: lengths below fm_floor()
    are raised to it."""
    import torch
    if floor:
        schedule = [max(v, fm_floor(f)) for v in schedule]
    total = sum(schedule)
    raws = f.inputs(total, seed)
    per = raws[0][1]
    offs = np.cumsum([0] + list(schedule))
    blocks = [[r[offs[c] * per:offs[c + 1] * per] for r, _ in raws] for c in range(len(schedule))]
    refs = [f.reference() for _ in range(B)]
    rs = f.resampler()
    problems, want = [], [[] for _ in range(B)]
    eng = f.engine(B, max(schedule), taps=True)
    got = [[] for _ in range(B)]
    pre_got, pre_want = [[] for _ in range(B)], [[] for _ in range(B)]
    for c, n in enumerate(schedule):
        eng.submit(np.stack(blocks[c]), n)
        for s in range(B):
            refs[s].push(blocks[c][s])
            if rs is None:
                problems += U.compare_taps(eng, s, refs[s], f.model, "submit %d (n=%d)" % (c, n), f.channels())
            else:
                pre_got[s].append(eng.tap(aisgpu.TAP_PRE, s, 0))
                pre_want[s].append(refs[s].tap_c(rs))
        ref_messages(refs, want)
        for m in eng.poll():
            got[m.stream].append(m)
    cnt = eng.counters()
    eng.close()
    assert cnt[2] == total and cnt[3] == len(schedule), cnt
    if rs is not None:
        for s in range(B):
            problems += resampler_problems(f, pre_got[s], pre_want[s], "stream %d" % s)
    problems += U.compare_frames(got, want)

    eng = f.engine(B, max(schedule), taps=False)
    got = [[] for _ in range(B)]
    keep = []  # host buffers of submit_async and device batches stay untouched until the engine has read them
    for c, n in enumerate(schedule):
        batch = np.ascontiguousarray(np.stack(blocks[c]))
        how = c % 4
        if how == 0:
            eng.submit(batch, n)
        elif how == 1:
            eng.submit_v([np.ascontiguousarray(b) for b in blocks[c]], n)
        elif how == 2:
            t = torch.from_numpy(batch).pin_memory()
            keep.append(t)
            eng.submit_async_ptr(t.data_ptr(), n)
        else:
            t = torch.from_numpy(batch).cuda()
            torch.cuda.synchronize()
            keep.append(t)
            eng.submit_device(t.data_ptr(), n, n)
        if c % 3 == 2:
            for m in eng.poll():
                got[m.stream].append(m)
    for m in eng.poll():
        got[m.stream].append(m)
    cnt2 = eng.counters()
    eng.close()
    del keep
    assert cnt2[:4] == cnt[:4], (cnt2, cnt)
    problems += [("no taps",) + p for p in U.compare_frames(got, want)]
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
    return sum(map(len, want))


ALL = ["long_short_long", "granule_x40", "tiled_streaming_switch", "straddle_cgf_block", "no_pow2_lane_split", "random"]
SOME = ["tiled_streaming_switch", "random"]
FAMILIES = [
    # streaming front end at 1536 kS/s (tiled for blocks below four warm-ups), every format and model
    (Fam("st1536_cf32_default", M2, 1536000), ALL),
    (Fam("st1536_cu8_standard", M0, 1536000, CU8), ALL),
    (Fam("st1536_cs8_base", M1, 1536000, CS8), SOME),
    (Fam("st1536_cs16_default_noema", M2, 1536000, CS16, ps_ema=False), SOME),
    (Fam("st1536_challenger", M4, 1536000), SOME),
    (Fam("st1536_v2", M11, 1536000), ["straddle_cgf_block", "random"]),
    (Fam("st6144_default", M2, 6144000), SOME),
    (Fam("st12288_standard", M0, 12288000), ["long_short_long", "tiled_streaming_switch", "random"]),
    # tiled front end
    (Fam("tiled96_default", M2, 96000), ALL),
    (Fam("tiled192_standard", M0, 192000), SOME),
    (Fam("tiled384_base", M1, 384000), SOME),
    (Fam("tiled384_default_noema", M2, 384000, CU8, ps_ema=False), SOME),
    (Fam("tiled384_challenger", M4, 384000), SOME),
    (Fam("tiled384_v2", M11, 384000), ["straddle_cgf_block", "random"]),
    # DownsampleKFilter at the exact buckets: on the raw input (288k), behind one / two CIC stages (576k, 1152k)
    (Fam("dsk288_default", M2, 288000, CS16), SOME + ["granule_x40"]),
    (Fam("dsk576_standard", M0, 576000, dsk=True), SOME),
    (Fam("dsk1152_default", M2, 1152000, CU8, dsk=True), SOME + ["straddle_cgf_block", "long_short_long"]),  # 64: a block DSK drops
    # single-channel mode and the FM-discriminator input
    (Fam("x48_default", M2, 48000, mode=MX), SOME + ["granule_x40"]),
    (Fam("x96_standard", M0, 96000, CU8, mode=MX), SOME),
    (Fam("x192_default", M2, 192000, CS16, mode=MX), SOME),
    (Fam("disc48_cs16", M3, 48000, CS16), SOME + ["granule_x40"]),
]
SCHEDULE_CASES = [(f, k) for f, ks in FAMILIES for k in ks]


@pytest.mark.parametrize("fam,kind", SCHEDULE_CASES, ids=["%s-%s" % (f.name, k) for f, k in SCHEDULE_CASES])
def test_length_schedule(built, fam, kind):
    sched = random_schedule(fam, 1000 + len(fam.name)) if kind == "random" else fixed_schedules(fam.granule())[kind]
    run_schedule(fam, sched, seed=7)


def test_fp_ds_length_schedule(built):
    # the integer front end takes multiples of 16384 (32 lane sub-segments of 512 samples)
    f = Fam("fpds", M2, 1536000, CU8, fp_ds=True)
    g = f.granule()
    assert g == 16384
    run_schedule(f, [g, 4 * g, g, 3 * g, 2 * g, g], seed=11)


@pytest.mark.xfail(strict=True, reason="known divergence: blocks of fewer than 37 samples at 48 kHz through the reference's Filter 37 "
                                       "(DSP.cpp:247-280) are not reproduced; FIR37 differs in the 36 outputs after the short block")
@pytest.mark.parametrize("model", [M0, M1])
def test_fm_filter_short_blocks(built, model):
    f = Fam("st1536_fm_short", model, 1536000)
    run_schedule(f, [65536, 64, 65536], seed=13, floor=False)


def test_random_schedules_1536k(built):
    # more seeds on the flagship configuration: every tap of every submit
    f = Fam("st1536_cf32_default", M2, 1536000)
    for seed in (1, 2, 3):
        run_schedule(f, random_schedule(f, seed, n=12), seed=20 + seed)


@pytest.mark.parametrize("fam,N", [(Fam("us6000_default", M2, 6000000), 65536), (Fam("us6000_standard_cu8", M0, 6000000, CU8), 65536),
                                   (Fam("dsk2000_default", M2, 2000000, dsk=True), 32768), (Fam("us250_default", M2, 250000), 8192),
                                   (Fam("x150_default", M2, 150000, mode=MX), 6400), (Fam("disc441_cs16", M3, 44100, CS16), 4416),
                                   (Fam("st1536_standard", M0, 1536000), 16384)], ids=lambda v: getattr(v, "name", str(v)))
def test_rejected_lengths_leave_engine_untouched(built, fam, N):
    """At a rate with a resampler a submit of another length is EINVAL (the reference re-blocks by the first length); at every rate
    so are n_samples > max_chunk and a length that is not a whole number of granules.  Afterwards the engine carries on bit for bit
    with a reference that never saw the refused blocks."""
    g = fam.granule()
    good = 7
    raws = fam.inputs(N * good, 31)
    per = raws[0][1]
    refs = [fam.reference() for _ in range(B)]
    eng = fam.engine(B, 2 * N, taps=True)
    rs = fam.resampler()
    got, want = [[] for _ in range(B)], [[] for _ in range(B)]
    pre_got, pre_want = [[] for _ in range(B)], [[] for _ in range(B)]
    problems = []
    junk = np.zeros((B, (2 * N + g) * per), dtype=raws[0][0].dtype)
    for c in range(good):
        blk = [r[c * N * per:(c + 1) * N * per] for r, _ in raws]
        eng.submit(np.stack(blk), N)
        for s in range(B):
            refs[s].push(blk[s])
            if rs is None:
                problems += U.compare_taps(eng, s, refs[s], fam.model, "submit %d" % c, fam.channels())
            else:
                pre_got[s].append(eng.tap(aisgpu.TAP_PRE, s, 0))
                pre_want[s].append(refs[s].tap_c(rs))
        ref_messages(refs, want)
        if c in (1, 4):
            before = eng.counters()
            bad = [2 * N + g, N + 1]  # longer than max_chunk; not a whole number of granules (g >= 4 everywhere)
            if rs is not None:
                bad.append(N + g)
            for n in bad:
                with pytest.raises(aisgpu.AisGpuError, match="rc=-1"):
                    eng.submit(junk[:, :n * per].copy(), n)
                assert eng.lib.aisgpu_last_error(eng.h).decode()
            assert eng.counters() == before
        for m in eng.poll():
            got[m.stream].append(m)
    eng.close()
    if rs is not None:
        for s in range(B):
            problems += resampler_problems(fam, pre_got[s], pre_want[s], "stream %d" % s)
    problems += U.compare_frames(got, want)
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)


# ---- B: device-batch placement --------------------------------------------------------------------------------------

def allowed(f, base, stride):
    try:
        aisgpu.check_device_batch(base, stride, sample_rate=f.fs, model=f.model, fmt=f.fmt, dsk=f.dsk, fp_ds=f.fp_ds, channel_mode=f.mode)
    except aisgpu.AisGpuError:
        return False
    return True


def placements(f, N, base):
    """(stride, base offset in bytes) per submit: strides N, N+2 .. N+8, N+64, 3N, alternating the packed base with the smallest
    offset the placement rule accepts; placements the rule refuses (16-byte rows of mode X / FP_DS) fall back to the next allowed."""
    bps = BPS[f.fmt]
    offs = [o for o in (bps, 2 * bps, 16) if allowed(f, base + o, N)]
    lo = offs[0]
    out = []
    for i, stride in enumerate([N, N + 2, N + 4, N + 6, N + 8, N + 64, 3 * N, N + 2, N + 6]):
        off = lo if i % 2 else 0
        while not allowed(f, base + off, stride):
            stride += 2
        out.append((stride, off))
    return out


def device_batch(blocks, stride, off, bps):
    """A cuda uint8 buffer holding the rows of `blocks` stride samples apart from byte `off` on; returns (tensor, pointer)."""
    import torch
    n_bytes = len(blocks[0].view(np.uint8))
    host = np.zeros(off + (len(blocks) - 1) * stride * bps + n_bytes + 64, np.uint8)
    for s, b in enumerate(blocks):
        o = off + s * stride * bps
        host[o:o + n_bytes] = np.ascontiguousarray(b).view(np.uint8)
    t = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    return t, t.data_ptr() + off


PLACEMENT_FAMILIES = [
    (Fam("st1536_cf32_default", M2, 1536000), 16384),
    (Fam("st1536_cu8_standard", M0, 1536000, CU8), 16384),
    (Fam("st1536_cs8_default", M2, 1536000, CS8), 16384),
    (Fam("st1536_cs16_base", M1, 1536000, CS16), 16384),
    (Fam("tiled384_cu8_default", M2, 384000, CU8), 4096),
    (Fam("tiled384_cf32_standard", M0, 384000), 4096),
    (Fam("us6000_cf32_default", M2, 6000000), 65536),
    (Fam("us6000_cu8_standard", M0, 6000000, CU8), 65536),
    (Fam("dsk288_cs16_default", M2, 288000, CS16), 12288),
    (Fam("dsk1152_cu8_default", M2, 1152000, CU8, dsk=True), 49152),
    (Fam("fpds_cu8_default", M2, 1536000, CU8, fp_ds=True), 16384),
    (Fam("x96_cu8_default", M2, 96000, CU8, mode=MX), 8192),
    (Fam("x48_cf32_standard", M0, 48000, mode=MX), 4096),
    (Fam("disc48_cf32", M3, 48000), 4096),
    (Fam("disc48_cu8", M3, 48000, CU8), 4096),
    (Fam("disc441_cs16", M3, 44100, CS16), 4416),
]


@pytest.mark.parametrize("fam,N", PLACEMENT_FAMILIES, ids=[f.name for f, _ in PLACEMENT_FAMILIES])
def test_device_batch_placement(built, fam, N):
    """Every placement the rule accepts gives the reference's taps and frames, and the same bits as a packed aisgpu_submit."""
    if not hasattr(aisgpu.load(), "aisgpu_check_device_batch"):
        pytest.skip("the library has no placement rule")
    bps = BPS[fam.fmt]
    plan = placements(fam, N, 1 << 20)
    raws = fam.inputs(N * len(plan), 41)
    per = raws[0][1]
    refs = [fam.reference() for _ in range(B)]
    rs = fam.resampler()
    dev = fam.engine(B, N, taps=True)
    packed = fam.engine(B, N, taps=True)
    problems = []
    got, pgot, want = [[] for _ in range(B)], [[] for _ in range(B)], [[] for _ in range(B)]
    pre_got, pre_want = [[] for _ in range(B)], [[] for _ in range(B)]
    for c, (stride, off) in enumerate(plan):
        blk = [r[c * N * per:(c + 1) * N * per] for r, _ in raws]
        t, ptr = device_batch(blk, stride, off, bps)
        assert allowed(fam, ptr, stride)
        dev.submit_device(ptr, stride, N)
        packed.submit(np.stack(blk), N)
        dev.sync()
        del t
        label = "submit %d stride N%+d offset %d" % (c, stride - N, off)
        for s in range(B):
            refs[s].push(blk[s])
            if rs is None:
                for ch in fam.channels():
                    for name, tap, arg, dt, _, _ in U.tap_pairs(fam.model, ch):
                        a, b = dev.tap(tap, s, arg, dtype=dt), packed.tap(tap, s, arg, dtype=dt)
                        if not U.bits_equal(a, b):
                            problems.append(("packed " + name, label, s, ch) + U.first_diff(a, b))
                problems += U.compare_taps(dev, s, refs[s], fam.model, label, fam.channels())
            else:
                a, b = dev.tap(aisgpu.TAP_PRE, s, 0), packed.tap(aisgpu.TAP_PRE, s, 0)
                if not U.bits_equal(a, b):
                    problems.append(("packed PRE", label, s) + U.first_diff(a, b))
                pre_got[s].append(a)
                pre_want[s].append(refs[s].tap_c(rs))
        ref_messages(refs, want)
        for m in dev.poll():
            got[m.stream].append(m)
        for m in packed.poll():
            pgot[m.stream].append(m)
    dev.close()
    packed.close()
    if rs is not None:
        for s in range(B):
            problems += resampler_problems(fam, pre_got[s], pre_want[s], "stream %d" % s)
    problems += U.compare_frames(got, want)
    problems += [("packed",) + p for p in U.compare_frames(got, pgot)]
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)


@pytest.mark.parametrize("fmt", [CU8, CS8])
def test_byte_format_padded_stride_tail(built, fmt):
    """CU8 / CS8 rows N + 2 and N + 6 samples apart (4 mod 8 bytes) from a packed base: the warm-up history each stream carries into
    the next submit must come from its own row.  Only even strides and an aligned base: runs against any build of the library."""
    f = Fam("st1536_%d" % fmt, M0, 1536000, fmt)
    N = 16384
    raws = f.inputs(N * 6, 43)
    refs = [f.reference() for _ in range(B)]
    eng = f.engine(B, N, taps=True)
    problems = []
    for c, stride in enumerate([N + 2, N + 6, N + 2, N + 6, N + 2, N + 6]):
        blk = [r[c * N * 2:(c + 1) * N * 2] for r, _ in raws]
        t, ptr = device_batch(blk, stride, 0, 2)
        eng.submit_device(ptr, stride, N)
        eng.sync()
        del t
        for s in range(B):
            refs[s].push(blk[s])
            problems += U.compare_taps(eng, s, refs[s], f.model, "submit %d stride N%+d" % (c, stride - N))
    eng.close()
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)


# ---- C: rejection -----------------------------------------------------------------------------------------------------

REJECT_FAMILIES = [
    (Fam("st1536_cf32", M2, 1536000), 16384, [(8, 0), (4, 0), (0, 1), (0, -2)]),
    (Fam("st1536_cu8", M0, 1536000, CU8), 16384, [(2, 0), (1, 0), (0, 1), (0, -2)]),
    (Fam("st1536_cs16", M2, 1536000, CS16), 16384, [(4, 0), (2, 0), (0, 3)]),
    (Fam("tiled384_cs8", M2, 384000, CS8), 4096, [(2, 0), (3, 2)]),
    (Fam("us6000_cf32", M2, 6000000), 65536, [(8, 0), (0, 1)]),
    (Fam("dsk288_cu8", M2, 288000, CU8), 12288, [(2, 0)]),
    (Fam("fpds", M2, 1536000, CU8, fp_ds=True), 16384, [(4, 0), (8, 0), (0, 2), (0, 4), (0, 6)]),
    (Fam("x96_cf32", M2, 96000, mode=MX), 8192, [(8, 0), (0, 1)]),
    (Fam("x48_cu8", M0, 48000, CU8, mode=MX), 4096, [(4, 0), (0, 2), (0, 6)]),
    (Fam("disc48_cf32", M3, 48000), 4096, [(4, 0), (0, 1)]),
    (Fam("disc441_cu8", M3, 44100, CU8), 4416, [(2, 0), (1, 0)]),
]


@pytest.mark.parametrize("fam,N,bad", REJECT_FAMILIES, ids=[f.name for f, _, _ in REJECT_FAMILIES])
def test_refused_placements_leave_engine_untouched(built, fam, N, bad):
    """(base offset in bytes, stride - N) pairs the rule refuses, and a stride shorter than the block: EINVAL with a reason, counters
    unchanged, handle usable, and the next submits bit-exact.  The buffer is large enough for every refused placement."""
    lib = aisgpu.load()
    if not hasattr(lib, "aisgpu_check_device_batch"):
        pytest.skip("the library has no placement rule: a misaligned batch is never handed to it")
    import torch
    bps = BPS[fam.fmt]
    nchunks = 5
    raws = fam.inputs(N * nchunks, 47)
    per = raws[0][1]
    refs = [fam.reference() for _ in range(B)]
    rs = fam.resampler()
    eng = fam.engine(B, N, taps=True)
    scratch = torch.zeros((B + 1) * (3 * N) * bps + 64, dtype=torch.uint8, device="cuda")
    base = scratch.data_ptr()
    got, want = [[] for _ in range(B)], [[] for _ in range(B)]
    pre_got, pre_want = [[] for _ in range(B)], [[] for _ in range(B)]
    problems = []
    for c in range(nchunks):
        blk = [r[c * N * per:(c + 1) * N * per] for r, _ in raws]
        if c in (1, 3):
            before = eng.counters()
            for off, dstride in bad + [(0, -8)]:  # the last: rows shorter than the block
                stride = N + dstride
                if stride >= N:  # refused by the rule itself: checked on the host before the engine ever sees the pointer
                    assert not allowed(fam, base + off, stride), (off, dstride)
                with pytest.raises(aisgpu.AisGpuError, match="rc=-1"):
                    eng.submit_device(base + off, stride, N)
                assert len(eng.lib.aisgpu_last_error(eng.h).decode()) > 10
                assert eng.counters() == before
        t, ptr = device_batch(blk, N, 0, bps)
        eng.submit_device(ptr, N, N)
        eng.sync()
        del t
        for s in range(B):
            refs[s].push(blk[s])
            if rs is None:
                problems += U.compare_taps(eng, s, refs[s], fam.model, "submit %d" % c, fam.channels())
            else:
                pre_got[s].append(eng.tap(aisgpu.TAP_PRE, s, 0))
                pre_want[s].append(refs[s].tap_c(rs))
        ref_messages(refs, want)
        for m in eng.poll():
            got[m.stream].append(m)
    cnt = eng.counters()
    eng.close()
    assert cnt[3] == nchunks and cnt[2] == nchunks * N
    if rs is not None:
        for s in range(B):
            problems += resampler_problems(fam, pre_got[s], pre_want[s], "stream %d" % s)
    problems += U.compare_frames(got, want)
    assert not problems, "parity problems (first 12): %r" % (problems[:12],)
