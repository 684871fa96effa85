"""CPU (-m "not gpu"): the compatibility rule of engine groups (aisgpu_check_attach / aisgpu_attach) and the Python mirror's
argument checks.  A member may differ from its leader in every back-end field, never in a field the shared front end reads."""
import ctypes as C

import pytest

import aisgpu

LEADER = dict(model=aisgpu.MODEL_DEFAULT, sample_rate=1536000, fmt=aisgpu.FMT_CF32, n_streams=4, max_chunk=65536)

BACKEND_DIFFS = [dict(model=m) for m in (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2)] + [
    dict(ps_ema=False), dict(afc_wide=False), dict(dd_train=0.5), dict(dd_weight=0.5), dict(channels="CD"), dict(own_mmsi=123456789),
    dict(taps=True), dict(max_frames=16), dict(tag_mode=0), dict(host_staging=False),
    dict(model=aisgpu.MODEL_V2, ps_ema=False, afc_wide=False, dd_train=0.1, dd_weight=0.2, channels="CD", own_mmsi=1, taps=True,
         max_frames=7, tag_mode=2)]

# (field named in the error, Engine keyword argument, a different value)
FRONTEND_DIFFS = [("sample_rate", "sample_rate", 768000), ("format", "fmt", aisgpu.FMT_CU8), ("n_streams", "n_streams", 5),
                  ("max_chunk_samples", "max_chunk", 32768), ("channel_mode", "channel_mode", aisgpu.MODE_X), ("droop", "droop", False),
                  ("dsk", "dsk", True), ("fp_ds", "fp_ds", True), ("device", "device", 1)]


@pytest.mark.parametrize("diff", BACKEND_DIFFS, ids=lambda d: ",".join("%s=%s" % kv for kv in d.items()))
def test_check_attach_accepts_backend_differences(built, diff):
    aisgpu.check_attach(LEADER, dict(LEADER, **diff))
    aisgpu.check_attach(dict(LEADER, **diff), LEADER)


@pytest.mark.parametrize("field,kw,value", FRONTEND_DIFFS, ids=[f[0] for f in FRONTEND_DIFFS])
def test_check_attach_rejects_frontend_difference(built, field, kw, value):
    with pytest.raises(aisgpu.AisGpuError, match=r"rc=-1: aisgpu_attach: %s differs" % field):
        aisgpu.check_attach(LEADER, dict(LEADER, **{kw: value}))


def test_check_attach_names_first_difference(built):
    with pytest.raises(aisgpu.AisGpuError, match="format differs"):
        aisgpu.check_attach(LEADER, dict(LEADER, fmt=aisgpu.FMT_CS16, droop=False, device=2))


@pytest.mark.parametrize("side", ["leader", "member"])
def test_check_attach_rejects_discriminator(built, side):
    disc = dict(LEADER, model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=48000)
    other = dict(LEADER, sample_rate=48000)
    pair = (disc, other) if side == "leader" else (other, disc)
    with pytest.raises(aisgpu.AisGpuError, match="FM discriminator model cannot be in a group \\(as the %s\\)" % side):
        aisgpu.check_attach(*pair)
    with pytest.raises(aisgpu.AisGpuError, match="as the leader"):
        aisgpu.check_attach(disc, disc)


def test_check_attach_older_struct_size(built):
    lib = aisgpu.load()
    old = aisgpu.Config.channel_mode.offset
    leader, member = aisgpu.make_config(**LEADER), aisgpu.make_config(**dict(LEADER, model=aisgpu.MODEL_V2))
    member.struct_size = old
    assert lib.aisgpu_check_attach(C.byref(leader), C.byref(member)) == 0
    leader.struct_size = old
    assert lib.aisgpu_check_attach(C.byref(leader), C.byref(member)) == 0
    # the older layout means AB: a mode-X partner differs in channel_mode
    x = aisgpu.make_config(**dict(LEADER, sample_rate=96000, channel_mode=aisgpu.MODE_X))
    member = aisgpu.make_config(**dict(LEADER, sample_rate=96000))
    member.struct_size = old
    member.channel_mode = aisgpu.MODE_X  # past the old struct_size: not read
    assert lib.aisgpu_check_attach(C.byref(x), C.byref(member)) == aisgpu.EINVAL
    assert b"channel_mode differs" in lib.aisgpu_last_error(None)
    member.struct_size = 12
    assert lib.aisgpu_check_attach(C.byref(leader), C.byref(member)) == aisgpu.EINVAL
    assert b"struct_size" in lib.aisgpu_last_error(None)


def test_check_attach_null_arguments(built):
    lib = aisgpu.load()
    cfg = aisgpu.make_config(**LEADER)
    assert lib.aisgpu_check_attach(None, C.byref(cfg)) == aisgpu.EINVAL
    assert lib.aisgpu_check_attach(C.byref(cfg), None) == aisgpu.EINVAL


def test_attach_null_leader(built):
    lib = aisgpu.load()
    cfg = aisgpu.make_config(**LEADER)
    out = C.c_void_p(12345)
    assert lib.aisgpu_attach(None, C.byref(cfg), C.byref(out)) == aisgpu.EINVAL
    assert b"aisgpu_attach" in lib.aisgpu_last_error(None)
    assert lib.aisgpu_attach(None, None, None) == aisgpu.EINVAL


class _Stub(aisgpu.Engine):
    """An Engine without a handle: only the argument checks of attach() that come before the library call run."""

    def __init__(self):  # noqa: D401 -- no aisgpu_create
        self.lib = aisgpu.load()
        self.kwargs = dict(LEADER)
        self.h = C.c_void_p()
        self.leader = None


def test_python_attach_argument_checks(built):
    e = _Stub()
    with pytest.raises(TypeError, match="sample_rate"):
        e.attach(sample_rate=768000)
    with pytest.raises(TypeError, match="fmt, n_streams"):
        e.attach(model=0, n_streams=3, fmt=1)
    with pytest.raises(ValueError, match="two letters"):
        e.attach(channels="ABC")
    with pytest.raises(aisgpu.AisGpuError, match="aisgpu_attach rc=-1"):  # a null leader handle reaches the library and is refused
        e.attach(model=aisgpu.MODEL_STANDARD)
    assert set(aisgpu.MEMBER_KEYS) == {"model", "ps_ema", "afc_wide", "dd_train", "dd_weight", "channels", "own_mmsi", "taps", "max_frames",
                                       "tag_mode"}


def test_python_check_attach_argument_checks(built):
    with pytest.raises(TypeError):
        aisgpu.check_attach(dict(LEADER, bogus=1), LEADER)
    aisgpu.check_attach(dict(LEADER, dd_train=0.5, dd_weight=0.9), LEADER)


def test_make_config_carries_dd_fields(built):
    cfg = aisgpu.make_config(dd_train=0.5, dd_weight=0.25)
    assert (cfg.dd_train, cfg.dd_weight) == (0.5, 0.25)
    d = aisgpu.make_config()
    assert abs(d.dd_train - 0.75) < 1e-7 and abs(d.dd_weight - 0.86) < 1e-7
