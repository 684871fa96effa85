"""-m gpu: engine groups (aisgpu_attach).  Every member of a group must be bit-identical to a standalone engine of its own config fed
the same submits: frames (payload, NMEA, emission order, msg.chunk, start/end counters, level/ppm bit patterns), counters, and the
taps C and FIR of every stream in the last submit.  At 1536 kS/s and at a resampled rate the members with reference settings are
also checked against the unmodified reference (oracle/_ref) per model.

Each case runs twice: taps off (the pipelined back end over two streams) and taps on (one back-end stream, every tap kept)."""
import ctypes as C

import numpy as np
import pytest

import aisgpu
import aissynth as S
import mode_x_util as X
import oracle as O
import parity_util as U

pytestmark = pytest.mark.gpu

AB, MX = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16
M0, M1, M2, M4, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2
B = 3       # streams: rows >= 1 are where a wrong row offset shows
NSUB = 6    # submits per run


class Case:
    """A group: the front end (rate, format, channel mode, DSK / FP_DS) and the members' back ends, the leader first."""

    def __init__(self, name, fs, fmt, mode, members, dsk=False, fp_ds=False, ref=False):
        self.name, self.fs, self.fmt, self.mode, self.members = name, fs, fmt, mode, members
        self.dsk, self.fp_ds, self.ref = dsk, fp_ds, ref

    def __repr__(self):
        return self.name

    def granule(self):
        return aisgpu.chunk_granule(self.fs, self.members[0]["model"], self.dsk, self.fp_ds, self.fmt, self.mode)

    def n(self):
        g = self.granule()
        return max(g, (self.fs // 10) // g * g)  # about 0.1 s per submit

    def front(self, max_chunk):
        return dict(sample_rate=self.fs, fmt=self.fmt, n_streams=B, max_chunk=max_chunk, dsk=self.dsk, fp_ds=self.fp_ds,
                    channel_mode=self.mode, channels="XX" if self.mode == MX else "AB")

    def inputs(self, n, seed):
        if self.mode == MX:
            return [X.stream_input(self.fs, n, seed + s, self.fmt) for s in range(B)]
        return [X.to_raw(S.random_stream(self.fs, n, seed + s, bursts_per_sec=(6, 12))[0], self.fmt) for s in range(B)]


CASES = [
    Case("AB1536k_CF32", 1536000, CF32, AB, [dict(model=M2), dict(model=M0), dict(model=M11)], ref=True),
    Case("AB96k_CU8", 96000, CU8, AB, [dict(model=M4), dict(model=M1)]),
    Case("AB6144k_CS16", 6144000, CS16, AB, [dict(model=M2), dict(model=M2, ps_ema=False, afc_wide=False)]),
    Case("AB250k_CF32_upsample", 250000, CF32, AB, [dict(model=M11, dd_train=0.5), dict(model=M0)], ref=True),
    Case("AB576k_DSK_CS8", 576000, CS8, AB, [dict(model=M0), dict(model=M2)], dsk=True),
    Case("AB1536k_FPDS_CU8", 1536000, CU8, AB, [dict(model=M2), dict(model=M0)], fp_ds=True),
    Case("X48k_CF32", 48000, CF32, MX, [dict(model=M0), dict(model=M2), dict(model=M11)]),
    Case("X50k_CU8_upsample", 50000, CU8, MX, [dict(model=M0), dict(model=M2)]),
]


def blocks_of(case, schedule, seed):
    raws = case.inputs(sum(schedule), seed)
    per = raws[0][1]
    offs = np.cumsum([0] + list(schedule))
    return [np.stack([r[offs[c] * per:offs[c + 1] * per] for r, _ in raws]) for c in range(len(schedule))]


def fir_dtype(model):
    return np.complex64 if model in (M2, M11) else np.float32


def last_taps(eng, case, model):
    """TAP_C and TAP_FIR of every stream and channel after the last submit."""
    out = {}
    for s in range(B):
        for ch in ((0,) if case.mode == MX else (0, 1)):
            out[("C", s, ch)] = eng.tap(aisgpu.TAP_C, s, ch)
            out[("FIR", s, ch)] = eng.tap(aisgpu.TAP_FIR, s, ch, dtype=fir_dtype(model))
    return out


def seq(msgs):
    """The whole emission order of one engine, every field the comparison covers."""
    return [(m.stream, m.chunk) + U.frame_key(m) for m in msgs]


def per_stream(msgs):
    return [[m for m in msgs if m.stream == s] for s in range(B)]


def run_standalone(case, member, blocks, taps):
    eng = aisgpu.Engine(**dict(case.front(max(b.shape[1] for b in blocks) // (1 if case.fmt == CF32 else 2)), taps=taps, **member))
    msgs = []
    for b in blocks:
        eng.submit(b, b.shape[1] // (1 if case.fmt == CF32 else 2))
        msgs += eng.poll()
    res = (msgs, eng.counters(), last_taps(eng, case, member["model"]) if taps else None, eng.overflows)
    eng.close()
    return res


def make_group(case, max_chunk, taps, members=None):
    members = members or case.members
    lead = aisgpu.Engine(**dict(case.front(max_chunk), taps=taps, **members[0]))
    return [lead] + [lead.attach(taps=taps, **m) for m in members[1:]]


def close_group(group):
    for e in group[::-1]:
        e.close()


def run_group(case, blocks, taps):
    n = [b.shape[1] // (1 if case.fmt == CF32 else 2) for b in blocks]
    group = make_group(case, max(n), taps)
    msgs = [[] for _ in group]
    for c, b in enumerate(blocks):
        group[0].submit(b, n[c])
        order = range(len(group)) if c % 2 == 0 else range(len(group) - 1, -1, -1)  # members polled in both orders
        for i in order:
            msgs[i] += group[i].poll()
    res = [(msgs[i], e.counters(), last_taps(e, case, case.members[i]["model"]) if taps else None, e.overflows) for i, e in enumerate(group)]
    close_group(group)
    return res


def compare(label, got, want):
    """One member (msgs, counters, taps, overflows) against its standalone engine."""
    problems = []
    if seq(got[0]) != seq(want[0]):
        problems.append((label, "frames", len(got[0]), len(want[0])) + tuple(U.compare_frames(per_stream(got[0]), per_stream(want[0]))[:1]))
    if got[1] != want[1]:
        problems.append((label, "counters", got[1], want[1]))
    if got[3] != want[3]:
        problems.append((label, "overflows", got[3], want[3]))
    if want[2] is not None:
        for k, w in want[2].items():
            if not U.bits_equal(got[2][k], w):
                problems.append((label, "tap", k, len(got[2][k]), len(w)) + U.first_diff(got[2][k], w))
    return problems


@pytest.mark.parametrize("taps", [False, True], ids=["pipelined", "taps"])
@pytest.mark.parametrize("case", CASES, ids=repr)
def test_group_matches_standalone(built, case, taps):
    blocks = blocks_of(case, [case.n()] * NSUB, 4100)
    group = run_group(case, blocks, taps)
    problems, total = [], 0
    for i, m in enumerate(case.members):
        want = run_standalone(case, m, blocks, taps)
        total += len(want[0])
        problems += compare("member %d %r" % (i, m), group[i], want)
    assert not problems, problems[:6]
    assert total > 0, "the stimulus produced no frames"
    lead_c = group[0][1]
    for g in group[1:]:
        assert g[1][2:4] == lead_c[2:4]


@pytest.mark.parametrize("case", [c for c in CASES if c.ref], ids=repr)
def test_group_matches_reference(built, case):
    if not O.have_ref():
        pytest.skip("checked against the compiled reference only")
    blocks = blocks_of(case, [case.n()] * NSUB, 4200)
    group = run_group(case, blocks, False)
    checked = 0
    for i, m in enumerate(case.members):
        if set(m) != {"model"}:
            continue  # the reference harness has no DD_TRAIN / DD_WEIGHT settings
        flags = O.FLAG_PS_EMA | O.FLAG_AFC_WIDE | O.FLAG_DROOP
        want = []
        for s in range(B):
            r = O.RefModel(model=m["model"], sample_rate=case.fs, fmt=case.fmt, flags=flags)
            for b in blocks:
                r.push(b[s])
            want.append(r.messages())
            r.close()
        checked += sum(len(w) for w in want)
        problems = U.compare_frames(per_stream(group[i][0]), want)
        assert not problems, ("member %d" % i, problems[:3])
    assert checked > 0


# ---- submit forms ------------------------------------------------------------------------------------------------------------

FORMS_CASE = Case("AB1536k_CF32_forms", 1536000, CF32, AB, [dict(model=M2), dict(model=M0), dict(model=M11)])


def standalone_all(case, blocks, members=None):
    return [run_standalone(case, m, blocks, False) for m in (members or case.members)]


@pytest.mark.parametrize("form", ["submit_v", "async_poll_upto", "device_padded_offset", "changing_lengths", "ten_before_poll"])
def test_group_submit_forms(built, form):
    import torch
    case = FORMS_CASE
    g = case.granule()
    if form == "changing_lengths":
        schedule = [1024 * g, 5 * g, 257 * g, 2048 * g, 64 * g, 613 * g, 2048 * g]
    else:
        schedule = [2048 * g] * (10 if form == "ten_before_poll" else NSUB)
    blocks = blocks_of(case, schedule, 4300)
    group = make_group(case, max(schedule), False)
    msgs = [[] for _ in group]
    keep = []
    dev = None
    for c, (b, n) in enumerate(zip(blocks, schedule)):
        if form == "submit_v":
            group[0].submit_v([b[s] for s in range(B)], n)
        elif form == "async_poll_upto":
            a = np.ascontiguousarray(b)
            keep.append(a)
            t = group[0].submit_async_ptr(a.ctypes.data, n)
            assert t == c
            if c > 0:  # the frames of the submit before, with the leader's ticket, members in changing order
                for i in ((1, 0, 2) if c % 2 else (2, 1, 0)):
                    msgs[i] += group[i].poll_upto(t - 1)
        elif form == "device_padded_offset":
            stride = n + 6 + 2 * c
            off = 2 * (c % 3)  # samples: 16-byte multiples for CF32
            dev = torch.zeros(off + B * stride, dtype=torch.complex64, device="cuda")
            for s in range(B):
                dev[off + s * stride: off + s * stride + n] = torch.from_numpy(b[s]).cuda()
            torch.cuda.synchronize()
            group[0].submit_device(dev.data_ptr() + off * 8, stride, n)
            group[0].sync()
        else:
            group[0].submit(b, n)
        if form in ("submit_v", "device_padded_offset", "changing_lengths"):
            for i in (range(len(group)) if c % 2 else (1, 2, 0)):
                msgs[i] += group[i].poll()
    for i in ((2, 0, 1) if form == "ten_before_poll" else range(len(group))):
        msgs[i] += group[i].poll()
    got = [(msgs[i], e.counters(), None, e.overflows) for i, e in enumerate(group)]
    close_group(group)
    want = standalone_all(case, blocks)
    problems = []
    for i in range(len(group)):
        problems += compare("member %d" % i, got[i], want[i])
    assert not problems, problems[:6]
    assert sum(len(w[0]) for w in want) > 0


# ---- isolation -------------------------------------------------------------------------------------------------------------

ISO_CASE = Case("AB1536k_CF32_iso", 1536000, CF32, AB, [dict(model=M2)])


def test_group_overflow_is_per_member(built):
    case = ISO_CASE
    members = [dict(model=M2), dict(model=M0, max_frames=2), dict(model=M2, channels="CD")]
    blocks = blocks_of(case, [case.n()] * NSUB, 4400)
    n = case.n()
    group = make_group(case, n, False, members)
    msgs = [[] for _ in group]
    for b in blocks:
        group[0].submit(b, n)
        for i, e in enumerate(group):
            msgs[i] += e.poll()
    got = [(msgs[i], e.counters(), None, e.overflows) for i, e in enumerate(group)]
    close_group(group)
    want = standalone_all(case, blocks, members)
    assert got[1][3] > 0 and got[1][1][4] > 0, "the tiny ring should have overflowed"
    assert got[0][3] == 0 and got[2][3] == 0
    problems = []
    for i in range(len(members)):
        problems += compare("member %d" % i, got[i], want[i])
    assert not problems, problems[:6]


def test_group_letters_and_own_mmsi(built):
    case = ISO_CASE
    blocks = blocks_of(case, [case.n()] * NSUB, 4500)
    base = run_standalone(case, dict(model=M2), blocks, False)
    assert base[0]
    p = base[0][0].payload
    mmsi = (p[1] << 22) | (p[2] << 14) | (p[3] << 6) | (p[4] >> 2)
    members = [dict(model=M2), dict(model=M2, channels="CD"), dict(model=M2, own_mmsi=mmsi)]
    n = case.n()
    group = make_group(case, n, False, members)
    msgs = [[] for _ in group]
    for b in blocks:
        group[0].submit(b, n)
        for i, e in enumerate(group):
            msgs[i] += e.poll()
    close_group(group)
    want = standalone_all(case, blocks, members)
    for i in range(3):
        assert seq(msgs[i]) == seq(want[i][0]), "member %d" % i
    # against the leader: CD differs in the letters (and so the NMEA checksums) only, own_mmsi in the talker of that vessel's sentences
    lead, cd, own = msgs
    assert len(lead) == len(cd) == len(own)
    swap = {"A": "C", "B": "D"}
    same = lambda m: (m.stream, m.chunk, m.nbits, m.payload, m.start_idx, m.end_idx) + U.frame_key(m)[3:]
    n_own = 0
    for a, c, o in zip(lead, cd, own):
        assert c.channel == swap[a.channel] and same(c) == same(a) and same(o) == same(a)
        mine = ((a.payload[1] << 22) | (a.payload[2] << 14) | (a.payload[3] << 6) | (a.payload[4] >> 2)) == mmsi
        n_own += mine
        assert [t.startswith("!AIVDO") for t in o.nmea] == [mine] * len(o.nmea)
        body = lambda t: t[6:t.rindex("*")]  # without the talker and the checksum over it
        assert [body(t) for t in o.nmea] == [body(t) for t in a.nmea]
        assert mine or o.nmea == a.nmea
    assert n_own > 0


def test_group_destroy_member_mid_run(built):
    case = ISO_CASE
    members = [dict(model=M2), dict(model=M0), dict(model=M11)]
    blocks = blocks_of(case, [case.n()] * NSUB, 4600)
    n = case.n()
    group = make_group(case, n, False, members)
    msgs = [[] for _ in group]
    for c, b in enumerate(blocks):
        group[0].submit(b, n)
        if c == 2:
            group[1].close()  # mid-run, frames not yet polled
        for i in (0, 2):
            msgs[i] += group[i].poll()
    got_c = [group[0].counters(), group[2].counters()]
    close_group([group[0], group[2]])
    want = standalone_all(case, blocks, members)
    assert seq(msgs[0]) == seq(want[0][0]) and got_c[0] == want[0][1]
    assert seq(msgs[2]) == seq(want[2][0]) and got_c[1] == want[2][1]


# ---- refusals on the GPU ----------------------------------------------------------------------------------------------------

def test_group_refusals(built, tmp_path):
    case = ISO_CASE
    lib = aisgpu.load()
    n = case.n()
    blocks = blocks_of(case, [n] * 3, 4700)
    members = [dict(model=M2), dict(model=M0)]
    group = make_group(case, n, False, members)
    lead, mem = group
    # a front-end field that differs
    bad = aisgpu.make_config(**dict(case.front(n), model=M0, sample_rate=768000))
    out = C.c_void_p()
    assert lib.aisgpu_attach(lead.h, C.byref(bad), C.byref(out)) == aisgpu.EINVAL and not out.value
    assert b"sample_rate differs" in lib.aisgpu_last_error(None)
    # a member cannot lead
    ok = aisgpu.make_config(**dict(case.front(n), model=M0))
    assert lib.aisgpu_attach(mem.h, C.byref(ok), C.byref(out)) == aisgpu.EINVAL
    # submits on a member
    b0 = np.ascontiguousarray(blocks[0])
    ptrs = (C.c_void_p * B)(*[b0[s].ctypes.data for s in range(B)])
    t = C.c_int64(-1)
    assert lib.aisgpu_submit(mem.h, b0.ctypes.data, n) == aisgpu.EINVAL
    assert lib.aisgpu_submit_v(mem.h, ptrs, n) == aisgpu.EINVAL
    assert lib.aisgpu_submit_async(mem.h, b0.ctypes.data, n, C.byref(t)) == aisgpu.EINVAL
    assert lib.aisgpu_submit_device(mem.h, b0.ctypes.data, n, n) == aisgpu.EINVAL
    assert b"member of a group" in lib.aisgpu_last_error(mem.h)
    assert mem.counters() == [0] * 8
    # file feeding: not for groups
    paths = []
    for s in range(B):
        p = tmp_path / ("s%d.raw" % s)
        blocks[0][s].tofile(p)
        paths.append(str(p))
    arr = (C.c_char_p * B)(*[p.encode() for p in paths])
    nb = C.c_uint64(0)
    for e in (lead, mem):
        assert lib.aisgpu_feed_files(e.h, arr, n, aisgpu.MSG_FN(0), None, C.byref(nb)) == aisgpu.EINVAL
    assert lead.counters() == [0] * 8
    # front-end queries on a member
    for tap in (aisgpu.TAP_ROT, aisgpu.TAP_PRE, aisgpu.TAP_PRE2):
        with pytest.raises(aisgpu.AisGpuError, match="no front end"):
            mem.tap(tap)
    # the group runs on, then attach after the first submit is refused
    msgs = [[], []]
    for c, b in enumerate(blocks):
        lead.submit(b, n)
        if c == 0:
            assert lib.aisgpu_attach(lead.h, C.byref(ok), C.byref(out)) == aisgpu.EINVAL
            assert b"already been submitted" in lib.aisgpu_last_error(None)
        msgs[0] += lead.poll()
        msgs[1] += mem.poll()
    assert mem.last_frontend_ms() < 0 and mem.frontend_times() == []
    assert lead.last_frontend_ms() >= 0
    got = [mem.counters(), lead.counters()]
    close_group(group)
    want = standalone_all(case, blocks, members)
    assert seq(msgs[0]) == seq(want[0][0]) and seq(msgs[1]) == seq(want[1][0])
    assert got == [want[1][1], want[0][1]]


def test_group_size_limit_and_leader_destroyed_first(built):
    case = ISO_CASE
    n = 4096
    lead = aisgpu.Engine(**dict(case.front(n), model=M2))
    mems = [lead.attach(model=(M0, M1, M2, M4, M11)[i % 5]) for i in range(7)]
    with pytest.raises(aisgpu.AisGpuError, match="at most 8"):
        lead.attach(model=M0)
    mems[3].close()
    mems[3] = lead.attach(model=M0)  # a detached member frees its place
    x = blocks_of(case, [n], 4800)[0]
    lead.submit(x, n)
    lead.sync()
    lead.join()
    lead.close()  # members first is the documented order; a leader destroyed first poisons them
    for m in mems:
        with pytest.raises(aisgpu.AisGpuError, match="leader was destroyed"):
            m.poll()
        m.close()
