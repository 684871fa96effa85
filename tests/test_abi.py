"""CPU (-m "not gpu"): the C-ABI library loads, exports every function include/aisgpu.h declares, agrees with the
ctypes mirror on struct layouts, rejects bad configurations with the reference's wording, fails LOUDLY without a GPU
(no CPU fallback), and its host-only per-frame tail (validate + NMEA armouring, reference Message.cpp:398-413,569-686)
reproduces the reference's own known-answer sentences (python/tests/test_decode.py:12-23)."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import aisgpu
import aissynth as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "aisgpu.h")


def declared_functions():
    txt = open(HEADER).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(aisgpu_[a-z_0-9]+)\s*\(", txt)))


def test_exports_match_header(built):
    lib = aisgpu.load()
    names = declared_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), "libaisgpu.so does not export %s" % n
    assert sorted(aisgpu.EXPORTS) == names, "aisgpu.py EXPORTS out of sync with include/aisgpu.h"
    assert lib.aisgpu_abi_version() == 3


def test_struct_layout_matches_ctypes(built, tmp_path):
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "aisgpu.h"\nint main(void){'
                   'printf("%zu %zu %zu %zu %zu %zu %zu\\n", sizeof(aisgpu_config), sizeof(aisgpu_msg), offsetof(aisgpu_config, station),'
                   'offsetof(aisgpu_msg, data), offsetof(aisgpu_msg, nmea), offsetof(aisgpu_msg, nmea_len), offsetof(aisgpu_msg, start_idx));return 0;}\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = list(map(int, subprocess.check_output([str(exe)]).split()))
    want = [C.sizeof(aisgpu.Config), C.sizeof(aisgpu.MsgStruct), aisgpu.Config.station.offset, aisgpu.MsgStruct.data.offset,
            aisgpu.MsgStruct.nmea.offset, aisgpu.MsgStruct.nmea_len.offset, aisgpu.MsgStruct.start_idx.offset]
    assert got == want


def test_default_config_is_reference_default(built):
    lib = aisgpu.load()
    cfg = aisgpu.Config()
    lib.aisgpu_default_config(C.byref(cfg))
    # Model.h:218-222 (PS_EMA on, nDelay 3), Model.h:138-143 (droop on), Common.h:242 (mode 3), FileRAW.h:52 (1536000)
    assert (cfg.model, cfg.sample_rate, cfg.ps_ema, cfg.afc_wide, cfg.droop, cfg.tag_mode) == (2, 1536000, 1, 1, 1, 3)
    assert (cfg.channel_a, cfg.channel_b) == (b"A", b"B")
    assert cfg.struct_size == C.sizeof(aisgpu.Config)


def test_bad_config_rejected_with_reference_wording(built):
    # Model.cpp:109-110 throws "Model: sample rate must be between 96K and 12288K (inclusive)."
    with pytest.raises(aisgpu.AisGpuError, match="between 96K and 12288K"):
        aisgpu.Engine(sample_rate=48000)
    with pytest.raises(aisgpu.AisGpuError, match="unknown model"):
        aisgpu.Engine(model=7)
    lib = aisgpu.load()
    cfg = aisgpu.Config()
    lib.aisgpu_default_config(C.byref(cfg))
    cfg.struct_size = 12
    h = C.c_void_p()
    assert lib.aisgpu_create(C.byref(cfg), C.byref(h)) == -1 and not h


def test_no_gpu_fails_loudly(built):
    """Runs in a child with CUDA hidden: aisgpu_create must return AISGPU_ENODEV, never fall back to a CPU path."""
    code = ("import sys; sys.path.insert(0, %r); import aisgpu\n"
            "try:\n    aisgpu.Engine()\nexcept aisgpu.AisGpuError as e:\n    print('ERR', e)\nelse:\n    print('CREATED')\n"
            % os.path.join(ROOT, "ais-catcher_b200"))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    out = subprocess.check_output([sys.executable, "-c", code], env=env).decode()
    assert out.startswith("ERR") and "rc=-2" in out and "no CPU fallback" in out, out


def test_product_never_touches_the_oracle():
    """The package may not import, link or dlopen anything under oracle/ (the checker is never the product)."""
    forbidden = ["import oracle", "from oracle", "libaisoracle", "libaisref", "aisorc_", "aisref_", "ais_oracle"]
    for dirpath, _, files in os.walk(os.path.join(ROOT, "ais-catcher_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                txt = open(os.path.join(dirpath, f)).read()
                for w in forbidden:
                    assert w not in txt, "%s references %s" % (f, w)
    if os.path.exists(aisgpu.LIB_PATH):
        blob = open(aisgpu.LIB_PATH, "rb").read()
        assert b"aisorc_" not in blob and b"aisref_" not in blob


# ---- placement rule of a device batch (aisgpu_check_device_batch, host-only) -------------------------------------------

BASE = 0x7F0000000000  # a device-looking address, 4 KiB aligned; the rule only looks at the number
AB, X = aisgpu.MODE_AB, aisgpu.MODE_X
CF32, CU8, CS8, CS16 = aisgpu.FMT_CF32, aisgpu.FMT_CU8, aisgpu.FMT_CS8, aisgpu.FMT_CS16
M0, M2, M3, M4, M11 = aisgpu.MODEL_STANDARD, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR, aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2

# (model, rate, format, channel mode, dsk, fp_ds) -> [(base offset in bytes, stride in samples, accepted)]
N = 65536
PLACEMENT = [
    # AB, exact buckets: the base aligned to two samples, any even stride (streaming kernel for 16-byte rows, tiled otherwise)
    ((M2, 1536000, CF32, AB, 0, 0), [(0, N, 1), (16, N + 2, 1), (8, N, 0), (4, N, 0), (0, N + 1, 0), (0, -2, 0), (32, 3 * N, 1)]),
    ((M0, 1536000, CU8, AB, 0, 0), [(0, N, 1), (4, N + 2, 1), (4, N + 6, 1), (2, N, 0), (1, N, 0), (0, N + 1, 0)]),
    ((M4, 1536000, CS8, AB, 0, 0), [(4, N + 2, 1), (8, N + 64, 1), (2, N + 2, 0), (3, N, 0)]),
    ((M11, 1536000, CS16, AB, 0, 0), [(8, N + 2, 1), (16, N + 4, 1), (4, N, 0), (2, N, 0)]),
    ((M2, 384000, CF32, AB, 0, 0), [(16, N + 2, 1), (8, N + 2, 0)]),
    ((M2, 12288000, CU8, AB, 0, 0), [(4, N + 2, 1), (2, N + 2, 0)]),
    # pre-stages: Upsample (6 MS/s: 4 CIC stages in front of it), DownsampleKFilter (288k on the raw input, 1152k behind CIC stages)
    ((M2, 6000000, CF32, AB, 0, 0), [(16, N + 2, 1), (8, N, 0)]),
    ((M0, 6000000, CU8, AB, 0, 0), [(4, N + 6, 1), (2, N, 0)]),
    ((M2, 288000, CS16, AB, 0, 0), [(8, N + 2, 1), (4, N, 0)]),
    ((M2, 288000, CU8, AB, 1, 0), [(4, N + 2, 1), (2, N, 0)]),
    ((M0, 1152000, CF32, AB, 1, 0), [(16, N + 2, 1), (8, N + 2, 0)]),
    # FP_DS: the integer front end only exists as the streaming kernel: 16-byte base and rows (CU8: strides of 8 samples)
    ((M2, 1536000, CU8, AB, 0, 1), [(0, N, 1), (16, N + 8, 1), (4, N, 0), (8, N, 0), (0, N + 2, 0), (0, N + 6, 0), (0, N + 4, 0)]),
    # single-channel mode: 16-byte base and rows at every rate, the interpolated ones included
    ((M2, 96000, CF32, X, 0, 0), [(0, N, 1), (16, N + 2, 1), (8, N, 0)]),
    ((M0, 192000, CU8, X, 0, 0), [(16, N + 8, 1), (0, N + 2, 0), (4, N, 0)]),
    ((M4, 48000, CS16, X, 0, 0), [(16, N + 4, 1), (0, N + 2, 0), (8, N, 0)]),
    ((M2, 44100, CF32, X, 0, 0), [(16, N + 2, 1), (8, N + 2, 0)]),
    # FM-discriminator input: any sample-aligned base at 48 kHz (the split loads single samples there), two samples behind Upsample
    ((M3, 48000, CF32, AB, 0, 0), [(8, N + 2, 1), (16, N, 1), (4, N, 0), (8, N + 1, 0)]),
    ((M3, 48000, CU8, AB, 0, 0), [(2, N + 2, 1), (1, N, 0)]),
    ((M3, 48000, CS16, X, 0, 0), [(4, N + 6, 1), (2, N, 0)]),
    ((M3, 44100, CU8, AB, 0, 0), [(4, N + 2, 1), (2, N, 0)]),
    ((M3, 12000, CF32, AB, 0, 0), [(16, N + 2, 1), (8, N, 0)]),
]


def placement_ok(cfg, off, stride):
    model, fs, fmt, mode, dsk, fp_ds = cfg
    try:
        aisgpu.check_device_batch(BASE + off, stride, sample_rate=fs, model=model, fmt=fmt, dsk=dsk, fp_ds=fp_ds, channel_mode=mode)
    except aisgpu.AisGpuError as e:
        assert "rc=-1" in str(e) and len(str(e)) > 12, e  # EINVAL with the reason
        return 0
    return 1


@pytest.mark.parametrize("cfg,cases", PLACEMENT, ids=["m%d_%d_f%d_mode%d_dsk%d_fpds%d" % c for c, _ in PLACEMENT])
def test_device_batch_placement_rule(built, cfg, cases):
    got = [(off, stride, placement_ok(cfg, off, stride)) for off, stride, _ in cases]
    assert got == cases


def test_device_batch_placement_rule_refusals(built):
    lib = aisgpu.load()
    # the engine's own configuration errors, with the same wording as aisgpu_create
    with pytest.raises(aisgpu.AisGpuError, match="between 96K and 12288K"):
        aisgpu.check_device_batch(BASE, N, sample_rate=48000)
    with pytest.raises(aisgpu.AisGpuError, match="needs CU8"):
        aisgpu.check_device_batch(BASE, N, fmt=CF32, fp_ds=True)
    with pytest.raises(aisgpu.AisGpuError, match="16-byte"):
        aisgpu.check_device_batch(BASE + 8, N, fmt=CU8, fp_ds=True)
    with pytest.raises(aisgpu.AisGpuError, match="two samples"):
        aisgpu.check_device_batch(BASE + 2, N, fmt=CU8)
    # FP_DS lane offsets are 32-bit counts of 16-byte units: the whole batch must span less than 64 GiB
    aisgpu.check_device_batch(BASE, 1 << 24, fmt=CU8, fp_ds=True, n_streams=1024)
    with pytest.raises(aisgpu.AisGpuError, match="64 GiB"):
        aisgpu.check_device_batch(BASE, 1 << 25, fmt=CU8, fp_ds=True, n_streams=1024)
    cfg = aisgpu.Config()
    lib.aisgpu_default_config(C.byref(cfg))
    assert lib.aisgpu_check_device_batch(C.byref(cfg), None, N) == aisgpu.EINVAL
    assert lib.aisgpu_check_device_batch(None, C.c_void_p(BASE), N) == aisgpu.EINVAL
    cfg.format = 9
    assert lib.aisgpu_check_device_batch(C.byref(cfg), C.c_void_p(BASE), N) == aisgpu.EINVAL
    # a caller built before channel_mode existed gets AB
    lib.aisgpu_default_config(C.byref(cfg))
    cfg.struct_size = aisgpu.Config.channel_mode.offset
    assert lib.aisgpu_check_device_batch(C.byref(cfg), C.c_void_p(BASE + 16), N + 2) == 0


# ---- host-only per-frame tail -------------------------------------------------------------------------------------

def pack(bits):
    b = np.zeros((len(bits) + 7) // 8 * 8, dtype=np.uint8)
    b[:len(bits)] = bits
    return bytes(np.packbits(b))


REF_TYPE5 = ["55O0W7`00001L@gCWGA2uItLth@DqtL5@F22220j1h742t0Ht0000000", "000000000000000"]
REF_TYPE26 = ["J1mg=5AEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEEE", "E" * 56, "E" * 56, "EEEEE@4SA@"]


def test_nmea_known_answers(built):
    # reference python/tests/test_decode.py:12-13
    bits = S.payload_to_bits(S.SAMPLE_A)
    assert aisgpu.build_nmea(pack(bits), len(bits), "A")[0] == ["!AIVDM,1,1,,A,15MgK45P3@G?fl0E`JbR0OwT0@MS,0*4E"]
    bits = S.payload_to_bits("177KQJ5000G?tO`K>RA1wUbN0TKH")
    assert aisgpu.build_nmea(pack(bits), len(bits), "B")[0] == ["!AIVDM,1,1,,B,177KQJ5000G?tO`K>RA1wUbN0TKH,0*5C"]
    # :14-17, two sentences, sequence id 4 in the reference's vector
    bits = np.concatenate([S.payload_to_bits(REF_TYPE5[0]), S.payload_to_bits(REF_TYPE5[1], fill=2)])
    s, nxt = aisgpu.build_nmea(pack(bits), len(bits), "A", seq=4)
    assert s == ["!AIVDM,2,1,4,A,55O0W7`00001L@gCWGA2uItLth@DqtL5@F22220j1h742t0Ht0000000,0*08", "!AIVDM,2,2,4,A,000000000000000,2*20"]
    assert nxt == 5
    assert aisgpu.build_nmea(pack(bits), len(bits), "A", seq=9)[1] == 0
    # :18-23, the 1064-bit maximum: 4 sentences.  The reference's encoder writes a NUL as the last letter here
    # (Message::getLetter, Message.cpp:646-647: the 178th letter crosses bit 1064) -- reproduced, not fixed.
    bits = np.concatenate([S.payload_to_bits(q) for q in REF_TYPE26[:3]] + [S.payload_to_bits(REF_TYPE26[3], fill=4)])
    assert len(bits) == 1064
    s, _ = aisgpu.build_nmea(pack(bits), 1064, "A", seq=7)
    assert s[:3] == ["!AIVDM,4,1,7,A," + REF_TYPE26[0] + ",0*69", "!AIVDM,4,2,7,A," + REF_TYPE26[1] + ",0*17", "!AIVDM,4,3,7,A," + REF_TYPE26[2] + ",0*16"]
    assert s[3].startswith("!AIVDM,4,4,7,A,EEEEE@4SA\x00,4*")


def test_nmea_own_mmsi_and_independent_builder(built):
    rng = np.random.default_rng(5)
    for _ in range(200):
        n = int(rng.choice([168, 168, 72, 312, 424, 1008]))
        bits = S.random_message_bits(rng, nbits=n)
        want, nxt = S.nmea_sentences(bits, "B", seq_start=3)
        got, gnxt = aisgpu.build_nmea(pack(bits), n, "B", seq=3)
        assert got == want and gnxt == nxt
    bits = S.payload_to_bits(S.SAMPLE_A)
    assert aisgpu.build_nmea(pack(bits), len(bits), "A", own_mmsi=366730000)[0][0].startswith("!AIVDO,")


def test_validate_min_lengths(built):
    lib = aisgpu.load()
    ml = [149, 149, 149, 168, 418, 88, 72, 56, 168, 70, 168, 72, 40, 40, 88, 92, 80, 168, 312, 70, 271, 145, 154, 160, 72, 60, 96, 168]
    for t in range(0, 32):
        d = bytes([t << 2]) + bytes(139)
        for n in (0, 39, 40, 148, 149, 168, 417, 418, 1064, 1065):
            want = 1 if n == 0 else (0 if n > 1064 or t < 1 or t > 28 else int(n >= ml[t - 1]))
            assert lib.aisgpu_validate(d, n) == want, (t, n)


def test_nmea_armouring_against_reference_sentences(built):
    """aisgpu_build_nmea (host-only) against the sentences the oracle printed for the same frames: every length 40..1064,
    multi-sentence messages with their sequence ids, fill bits -- over the decoder-fuzz stimulus (hundreds of frames)."""
    import oracle as O
    Model = O.RefModel if O.have_ref() else O.PortModel
    n, multi = 0, 0
    for seed in range(6):
        x, _ = S.fuzz_stream(96000, 262144, seed)
        m = Model(model=O.MODEL_STANDARD, sample_rate=96000)
        m.run(x, 8192)
        seq = 0
        for q in m.messages():
            pay = q.payload + bytes(140 - len(q.payload))
            got, seq = aisgpu.build_nmea(pay, q.nbits, channel=q.channel, seq=seq)
            assert got == q.nmea, (seed, q.nbits, got, q.nmea)
            n += 1
            multi += len(q.nmea) > 1
    assert n > 100 and multi > 20
