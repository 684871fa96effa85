"""The frequency-correction stimuli of tests/afc_signals.py reach the branches they exist for, proven on the compiled reference
(oracle/_ref) -- without this a passing bit-exact test on them (tests/test_gpu_afc.py) might never have left the centre of the
estimators' range.  Counts, not just "reached":

  ModelDefault, AFC wide    the peak fz at both ends of [-205, 208]; peaks where the search's index wraps; pinned past the edge
  ModelDefault, AFC narrow  blocks pinned at fz = -17 and at fz = 18
  ModelEngineV2             fz = 0 and fz >= 409 (no sub-bin step); frac clamped to +-0.5; the tone gate; midWins
  V2 slot lock (AB and X)   locked blocks at every targeted split; frames tagged ppm_prev; a lock that is lost again
  frames                    decoded at carriers of +-9 kHz and more by models 2, 4 and 11

The fz of a ModelDefault block is read off the ppm tag it carries (f = fz / 1024, ppm = f * 48000 / 162); that of a V2 block from
the magnitudes the reference's estimate left behind (afc_signals.v2_estimate), checked against the reference's own last_f.  CPU only.
"""
import numpy as np
import pytest

import afc_signals as A
import oracle as O
import oracle_afc as OA

FS = 1536000
AB, X_ = A.AB, A.X_

pytestmark = pytest.mark.skipif(not (OA.have_ref("ab") and OA.have_ref("x")), reason="needs the compiled reference probe (oracle/_ref)")

_cache = {}


def sweep_input(fs=FS, kind=AB):
    key = ("sweep", fs, kind)
    if key not in _cache:
        _cache[key] = A.rows(fs, A.SWEEP_N48 * fs // 48000, A.SWEEP, kind=kind)
    return _cache[key]


def cgf_fz(ppm):
    """fz of each block from its ppm tag (exact: fz is an integer below 2^8)."""
    return np.rint(ppm.astype(np.float64) * 162.0 / 48000.0 * 1024.0).astype(int)


def run_cgf(x, flags, fs=FS, chunk=65536, model=O.MODEL_DEFAULT):
    """ModelDefault over one stream: (fz per CGF block of channel A, of channel B, messages)."""
    r = O.RefModel(model=model, sample_rate=fs, flags=flags, taps=model == O.MODEL_DEFAULT)
    r.run(x, chunk)
    if model != O.MODEL_DEFAULT:
        return None, None, r.messages()
    return cgf_fz(r.tap_ppm(O.TAP_CGF_A)), cgf_fz(r.tap_ppm(O.TAP_CGF_B)), r.messages()


def v2_blocks(x, fs=FS, mode=AB, weights=None, ch=(0, 1)):
    """ModelEngineV2 over one stream, one 512-block per push: per channel a list of per-block dicts, and the messages."""
    blk = 512 * fs // 48000
    r = OA.RefModelAFC(model=O.MODEL_V2, sample_rate=fs, mode=mode, taps=True, weights=weights)
    prev = {c: None for c in ch}
    cprev = {c: np.zeros(512, np.complex64) for c in ch}
    out = {c: [] for c in ch}
    for b in range(len(x) // blk):
        r.push(x[b * blk:(b + 1) * blk])
        cc = {c: r.tap_c(O.TAP_CA + c) for c in ch}
        for c in ch:
            s = r.v2_state(c)
            p = prev[c]
            d = {"s": s, "b": b}
            # what this block's CGF saw: the decayed slot_ema, the split, busy from the decoders the previous block left behind
            ema = np.complex64(complex(np.float32(p.slot_ema.real) * np.float32(0.9999), np.float32(p.slot_ema.imag) * np.float32(0.9999))) \
                if p is not None else np.complex64(0)
            n2 = np.float32(np.float32(ema.real * ema.real) + np.float32(ema.imag * ema.imag))
            ph = 0 if p is None else p.slot_phase
            e = ((ph - b * 512) % A.SLOT + A.SLOT) % A.SLOT
            d["locked"] = bool(n2 >= np.float32(0.64)) and e < 512
            d["e"] = e
            d["busy"] = False if p is None else p.busy
            d["last_f_prev"] = np.float32(0) if p is None else p.last_f
            u, v = cprev[c][:256], cc[c][:256]
            head = np.cumsum((u.real * u.real + u.imag * u.imag).astype(np.float32), dtype=np.float32)[-1]
            tail = np.cumsum((v.real * v.real + v.imag * v.imag).astype(np.float32), dtype=np.float32)[-1]
            d["mid"] = (not d["locked"]) and (not d["busy"]) and bool(tail > head)
            d["est"] = A.v2_estimate(s.mag)
            d["gated"] = (not d["locked"]) and d["busy"] and s.prominence < np.float32(5.5)
            out[c].append(d)
            prev[c] = s
            cprev[c] = cc[c]
    return out, r.messages()


@pytest.fixture(scope="module")
def cgf_wide():
    return [run_cgf(x, O.DEFAULT_FLAGS) for x in sweep_input()]


def test_afc_wide_reaches_both_ends_and_the_wrap(cgf_wide):
    fz = np.concatenate([np.concatenate([a, b]) for a, b, _ in cgf_wide])
    assert fz.min() <= -203 and fz.max() >= 206, (fz.min(), fz.max())
    # the search runs over i in [wi + 187, wi + 223) of the fftshift-ordered spectrum, fz = 205 - i: its index wraps when
    # i < 0 (fz >= 206) or i + 102 > 511 (fz = -205)
    wrap = (fz >= 206) | (fz == -205)
    assert wrap.sum() >= 5, wrap.sum()
    # far from the centre: more than a hundred blocks beyond +-150 bins on each side
    assert (fz <= -150).sum() >= 100 and (fz >= 150).sum() >= 100
    # past the edge (|offset| > 10 kHz) the estimate is pinned to the outermost bins in a good share of the blocks
    past = np.concatenate([np.concatenate([a, b]) for off, (a, b, _) in zip(A.SWEEP, cgf_wide) if abs(off) >= 10500])
    assert len(past) >= 200 and (np.abs(past) >= 190).mean() >= 0.3, (len(past), (np.abs(past) >= 190).mean())


def test_afc_narrow_pins_at_the_window_edges():
    fz = np.concatenate([np.concatenate(run_cgf(x, O.DEFAULT_FLAGS & ~O.FLAG_AFC_WIDE)[:2]) for x in sweep_input()])
    assert fz.min() == -17 and fz.max() == 18
    assert (fz == -17).sum() >= 100 and (fz == 18).sum() >= 100, ((fz == -17).sum(), (fz == 18).sum())


def test_frames_at_wide_offsets_in_models_2_and_4(cgf_wide):
    # ModelChallenger's FM branch decodes at +-9 kHz; the coherent chains of models 2 and 11 lose the bursts beyond about +-6 kHz,
    # where the front end's channel filter takes too much of them
    for model, res, edge in ((O.MODEL_DEFAULT, cgf_wide, 4000), (O.MODEL_CHALLENGER, None, 9000)):
        lo = hi = 0
        for off, x, k in zip(A.SWEEP, sweep_input(), range(len(A.SWEEP))):
            if abs(off) < edge:
                continue
            msgs = res[k][2] if res else run_cgf(x, O.DEFAULT_FLAGS, model=model)[2]
            # channel A sits at +off, channel B at -off
            lo += sum(1 for m in msgs if (m.channel == "A") == (off < 0))
            hi += sum(1 for m in msgs if (m.channel == "A") == (off > 0))
        assert lo >= 5 and hi >= 5, (model, lo, hi)


@pytest.fixture(scope="module")
def v2_sweep():
    return [v2_blocks(x) for x in sweep_input()]


def test_v2_estimator_window_ends():
    # the tone pairs put the peak on fz = 0 and fz = 409, in AB at 1536 kS/s and in mode X at 48 kS/s
    for fs, kind, ch in ((FS, AB, (0, 1)), (48000, X_, (0,))):
        for fz in A.EDGE_TONE_BINS:
            out, _ = v2_blocks(A.edge_tones(fs, A.SWEEP_N48 * fs // 48000, fz, 0, kind), fs, kind, ch=ch)
            got = [d["est"][1] for c in out for d in out[c][1:]]
            assert all(d["est"][4] == d["s"].last_f for c in out for d in out[c])
            assert got.count(fz) >= 10 * len(ch), (fs, fz, got)


def test_v2_estimator_edges(v2_sweep):
    blocks = [d for out, _ in v2_sweep for c in out for d in out[c]]
    ungated = [d for d in blocks if not d["gated"]]
    # the restatement of the search agrees with the reference's own frequency wherever the tone gate did not hold it
    assert all(d["est"][4].view(np.uint32) == np.float32(d["s"].last_f).view(np.uint32) for d in ungated)
    fz = np.array([d["est"][1] for d in ungated])
    assert fz.min() <= 3 and fz.max() >= 405, (fz.min(), fz.max())
    wi = np.array([d["est"][0] for d in ungated])
    assert wi.min() == 0 and wi.max() == 512 - 133, (wi.min(), wi.max())
    clamped = [d for d in ungated if d["est"][2] is not None and abs(d["est"][2]) > 0.5]
    assert len(clamped) >= 5, len(clamped)
    gated = [d for d in blocks if d["gated"]]
    assert len(gated) >= 20 and all(d["s"].last_f == d["last_f_prev"] for d in gated), len(gated)
    assert sum(d["mid"] for d in blocks) >= 50


def test_v2_frames_at_wide_offsets(v2_sweep):
    lo = hi = 0
    for off, (_, msgs) in zip(A.SWEEP, v2_sweep):
        if abs(off) >= 4000:
            lo += sum(1 for m in msgs if (m.channel == "A") == (off < 0))
            hi += sum(1 for m in msgs if (m.channel == "A") == (off > 0))
    assert lo >= 5 and hi >= 5, (lo, hi)


def slot_runs(mode):
    fs = FS if mode == AB else 48000
    res = []
    for k, ph in enumerate(A.SLOT_PHASES[mode]):
        x = A.slotted(fs, A.SLOT_N48 * fs // 48000, ph, k, kind=mode)
        res.append(v2_blocks(x, fs, mode, ch=(0, 1) if mode == AB else (0,)))
    return res


@pytest.mark.parametrize("mode", [AB, X_])
def test_v2_slot_lock(mode):
    splits, prev_tagged, lost = set(), 0, 0
    for out, msgs in slot_runs(mode):
        for c, blocks in out.items():
            was = False
            for d in blocks:
                if d["locked"]:
                    assert d["s"].ppm_split == d["e"]
                    splits.add(d["e"])
                    was = True
                elif was and d["s"].norm2 < np.float32(0.64):
                    lost += 1
                    was = False
            by_block = {d["b"]: d["s"] for d in blocks}
            letter = "AB"[c] if mode == AB else "X"
            for m in msgs:
                s = by_block.get(m.end_idx // 512)
                if m.channel == letter and s and s.ppm != s.ppm_prev and np.float32(m.ppm) == s.ppm_prev:
                    prev_tagged += 1
    assert {0, 1, 255, 256, 511} <= splits, sorted(splits)
    assert prev_tagged >= 2 and lost >= 3, (prev_tagged, lost)


def test_v2_lock_decays_in_silence():
    # mode X at 48 kS/s: a lock, then no decode for ~24 s; 0.9999 per block takes it below 0.64
    x = A.slotted(48000, A.SILENT_N48, A.SLOT_PHASES[X_][0], 7, kind=X_, misaligned=0)
    out, msgs = v2_blocks(x, 48000, X_, ch=(0,))
    locked = [d["b"] for d in out[0] if d["locked"]]
    last_msg = max(m.end_idx for m in msgs) // 512
    assert locked and last_msg < locked[-1] - 1000, (len(locked), last_msg)
    assert out[0][-1]["s"].norm2 < np.float32(0.64)


def test_v2_weights_change_the_decode():
    # a non-default DD_TRAIN / DD_WEIGHT pair reaches the phase trackers: the reference decodes differently
    x = A.slotted(FS, A.SLOT_N48 * 32, A.SLOT_PHASES[AB][0], 3)
    a = [(m.start_idx, m.end_idx, m.level) for m in v2_blocks(x)[1]]
    b = [(m.start_idx, m.end_idx, m.level) for m in v2_blocks(x, weights=(0.5, 0.95))[1]]
    assert a and b and a != b
