"""Messages for the full AIS JSON tests (tests/test_json_full.py, tests/test_gpu_json_full.py, tools/gen_json_golden.py).

A case is a dict: data (140 bytes, hex), nbits, channel, sentences, level, ppm and tag (the aisgpu_tag fields the line prints).
``structured_cases()`` walks every message type 1-28 at short, minimal and long lengths, every value of every enumeration, the
"not available" sentinels and their neighbours, the radio states, type 22 / 24 / 25 / 26 variants, text edge cases, the MID rules
of the country lookup, and every (DAC, FI) pair the reference decodes for types 6 and 8; ``random_cases(n, seed)`` draws random
payloads of random lengths with random tags.
"""
import random

# Message::validate's minimum lengths (types 1..28)
MIN_BITS = [149, 149, 149, 168, 418, 88, 72, 56, 168, 70, 168, 72, 40, 40, 88, 92, 80, 168, 312, 70, 271, 145, 154, 160, 72, 60, 96, 168]

# (DAC, FI) pairs the reference decodes into fields: type 6 (addressed) and type 8 (broadcast)
ASM6 = [(0, 0), (1, 0), (1, 2), (1, 3), (1, 4), (1, 16), (1, 40), (1, 20), (1, 23), (1, 25), (1, 28), (1, 32), (1, 30), (210, 0),
        (248, 0), (353, 0), (200, 21), (200, 22), (200, 55), (235, 10), (250, 10), (366, 10), (235, 20), (316, 1), (366, 1),
        (316, 2), (366, 2), (316, 32), (366, 32)]
ASM8 = [(1, 0), (1, 16), (1, 20), (1, 22), (1, 23), (1, 24), (1, 25), (210, 0), (248, 0), (353, 0), (200, 10), (200, 23),
        (200, 24), (200, 40), (200, 55), (1, 31), (200, 25), (1, 21), (1, 29), (1, 27), (1, 19), (1, 17), (1, 26), (1, 11),
        (235, 10), (250, 10), (366, 10), (316, 1), (366, 1), (316, 2), (366, 2), (316, 32), (366, 32), (367, 33), (265, 1)]
def setu(buf, start, n, v):
    """Writes the n-bit unsigned v at bit start (MSB first)."""
    for i in range(n):
        b = start + i
        bit = (v >> (n - 1 - i)) & 1
        buf[b >> 3] = (buf[b >> 3] & ~(0x80 >> (b & 7)) & 0xFF) | (bit << (7 - (b & 7)))


def getu(buf, start, n):
    v = 0
    for i in range(n):
        b = start + i
        v = (v << 1) | ((buf[b >> 3] >> (7 - (b & 7))) & 1)
    return v


DEFAULT_TAG = dict(version=14, driver=3, hardware="H100", mode=3, rxtime_us=0, toa_us=0, station=0)


def case(data, nbits, channel="A", sentences=("!AIVDM,1,1,,A,13u?etPv2;0n:dDPwUM1U1Cb069D,0*23",), level=-17.25, ppm=0.5, **tag):
    t = dict(DEFAULT_TAG)
    t.update(tag)
    return dict(data=bytes(data).hex(), nbits=nbits, channel=channel, sentences=list(sentences), level=level, ppm=ppm, tag=t)


def msg(rng, typ, mmsi=None):
    d = bytearray(rng.getrandbits(8) for _ in range(140))
    setu(d, 0, 6, typ)
    if mmsi is not None:
        setu(d, 8, 30, mmsi)
    return d


def structured_cases(seed=2024):
    rng = random.Random(seed)
    out = []
    # every type at short, minimal, long and maximal lengths, random content
    for typ in range(0, 32):
        ml = MIN_BITS[typ - 1] if 1 <= typ <= 28 else 168
        for nbits in sorted({1, 6, 37, 38, 39, ml - 7, ml - 1, ml, ml + 1, ml + 6, ml + 20, 424, 1000, 1063, 1064}):
            if nbits > 0:
                out.append(case(msg(rng, typ), nbits))
    # every value of every enumeration, and the fields around each sentinel
    for v in range(16):
        d = msg(rng, 1); setu(d, 38, 4, v); out.append(case(d, 168))
        d = msg(rng, 4); setu(d, 134, 4, v); out.append(case(d, 168))
        d = msg(rng, 5); setu(d, 270, 4, v); out.append(case(d, 424))
        d = msg(rng, 27); setu(d, 40, 4, v); out.append(case(d, 96))
        d = msg(rng, 23); setu(d, 110, 4, v); setu(d, 146, 4, v); out.append(case(d, 160))
    for v in range(4):
        d = msg(rng, 3); setu(d, 143, 2, v); out.append(case(d, 168))
    for v in range(256):
        d = msg(rng, 5); setu(d, 232, 8, v); out.append(case(d, 424))
        d = msg(rng, 24); setu(d, 38, 2, 1); setu(d, 40, 8, v); out.append(case(d, 168))
    for v in range(32):
        d = msg(rng, 21); setu(d, 38, 5, v); out.append(case(d, 272))
    for v in range(128):
        d = msg(rng, 28); setu(d, 104, 7, v); setu(d, 101, 3, v & 7); out.append(case(d, 168))
    sentinels = {1: [(50, 10, 1023), (61, 28, 108600000), (89, 27, 54600000), (116, 12, 3600), (128, 9, 511), (137, 6, 60)],
                 4: [(38, 14, 0), (52, 4, 0), (56, 5, 0), (61, 5, 24), (66, 6, 60), (72, 6, 60), (79, 28, 108600000), (107, 27, 54600000)],
                 5: [(40, 30, 0), (274, 4, 0), (278, 5, 0), (283, 5, 24), (288, 6, 60), (294, 8, 0)],
                 9: [(38, 12, 4095), (50, 10, 1023), (61, 28, 108600000), (89, 27, 54600000), (116, 12, 3600), (128, 6, 60)],
                 17: [(40, 18, 108600), (58, 17, 54600)],
                 18: [(46, 10, 1023), (57, 28, 108600000), (85, 27, 54600000), (112, 12, 3600), (124, 9, 511), (133, 6, 60)],
                 19: [(46, 10, 1023), (57, 28, 108600000), (85, 27, 54600000), (112, 12, 3600), (124, 9, 511), (133, 6, 60)],
                 21: [(164, 28, 108600000), (192, 27, 54600000), (253, 6, 60)],
                 27: [(44, 18, 108600), (62, 17, 54600), (79, 6, 63), (85, 9, 511)],
                 28: [(38, 6, 60), (44, 28, 108600000), (72, 27, 54600000)]}
    for typ, fl in sentinels.items():
        ml = max(MIN_BITS[typ - 1], 168)
        for start, n, s in fl:
            for v in {s - 1, s, s + 1, 0, (1 << n) - 1, 1 << (n - 1), (1 << n) - s if s else 1}:
                d = msg(rng, typ)
                setu(d, start, n, v & ((1 << n) - 1))
                out.append(case(d, ml))
    # rate of turn, every value
    for v in range(256):
        d = msg(rng, 1); setu(d, 42, 8, v); out.append(case(d, 168))
    # radio state: every slot timeout, UTC valid and not, radio 0, short radio fields
    for to in range(8):
        for sub in (0, 1, (23 << 9) | (59 << 2), (24 << 9) | (10 << 2), (5 << 9) | (60 << 2), 0x3FFF):
            d = msg(rng, 1); setu(d, 149, 19, (rng.getrandbits(2) << 17) | (to << 14) | sub); out.append(case(d, 168))
            d = msg(rng, 26); setu(d, 38, 2, rng.getrandbits(2)); setu(d, 150, 19, (to << 14) | sub); out.append(case(d, 170))
    d = msg(rng, 4); setu(d, 149, 19, 0); out.append(case(d, 168))
    for nbits in (149, 150, 160, 167):
        out.append(case(msg(rng, 1), nbits))
    # type 22: addressed / broadcast; type 24: part A, part B with dimensions or mothership, with and without EPFD / VDES
    for addressed in (0, 1):
        d = msg(rng, 22); setu(d, 139, 1, addressed); out.append(case(d, 168))
        d = msg(rng, 22); setu(d, 139, 1, addressed); setu(d, 69, 18, 0x3FFFF); setu(d, 87, 17, 0x1FFFF); out.append(case(d, 168))
    for part in range(4):
        for mmsi in (244123456, 980123456, 981234567, 970123456):
            for nbits in (160, 162, 167, 168):
                d = msg(rng, 24, mmsi); setu(d, 38, 2, part); out.append(case(d, nbits))
    # types 25 / 26: every addressed / structured combination, lengths around the comm state
    for typ in (25, 26):
        for flags in range(4):
            for nbits in (40, 59, 60, 72, 88, 100, 168, 1064):
                d = msg(rng, typ); setu(d, 38, 2, flags); out.append(case(d, nbits))
    # text: '@' terminators, trailing and leading spaces, '"' and '\\', a field reaching bit 1064
    for fill in ([0] * 20, [32] * 20, [1, 32, 32, 0, 5], [2, 34, 60, 28, 32], [32, 1, 32], [34] * 20, [28] * 20):
        for typ, start, nbits in ((5, 112, 424), (14, 40, 1064), (12, 72, 200), (21, 43, 272), (24, 40, 160), (19, 143, 312)):
            d = msg(rng, typ)
            for i in range(20):
                setu(d, start + 6 * i, 6, fill[i % len(fill)])
            if typ == 24:
                setu(d, 38, 2, 0)
            out.append(case(d, nbits))
    for nbits in (40, 41, 45, 46, 47, 1063, 1064):
        out.append(case(msg(rng, 14), nbits))
    # country: every MID (as 111MID000 and as MMSI MID000000), and the 98 / 99 / 111 prefixes; tag mode 4 prints it
    for mid in range(0, 1000):
        out.append(case(msg(rng, 1, 111000000 + mid * 1000), 168, mode=7))
    for mid in range(100, 1000, 7):
        out.append(case(msg(rng, 1, mid * 1000000 + rng.randrange(1000000)), 168, mode=5))
    for mmsi in (980000000, 989999999, 990000000, 992351234, 999999999, 982440001, 8, 1000, 1001, 1000000, 1110000000 - 1, 111232000):
        out.append(case(msg(rng, 1, mmsi & 0x3FFFFFFF), 168, mode=4))
    # every (DAC, FI) the reference decodes, a few unknown ones, at several lengths
    for typ, pairs, dpos in ((6, ASM6, 72), (8, ASM8, 40)):
        for dac, fid in pairs + [(0, 1), (1, 1), (999, 63), (1023, 0)]:
            for nbits in sorted({MIN_BITS[typ - 1], dpos + 16, 96, 120, 168, 200, 260, 300, 400, 600, 1000, 1064}):
                d = msg(rng, typ); setu(d, dpos, 10, dac); setu(d, dpos + 10, 6, fid); out.append(case(d, nbits))
    for typ in (25, 26):
        for addressed, pairs in ((1, ASM6), (0, ASM8)):
            for dac, fid in pairs:
                d = msg(rng, typ); setu(d, 38, 1, addressed); setu(d, 39, 1, 1)
                dpos = 72 if addressed else 40
                setu(d, dpos, 10, dac); setu(d, dpos + 10, 6, fid)
                out.append(case(d, rng.choice([120, 168, 300, 600])))
    # the application layouts with records, loops and formatted strings, around their length rules and special values
    def app8(dac, fid, nbits, fields=()):
        d = msg(rng, 8); setu(d, 40, 10, dac); setu(d, 50, 6, fid)
        for st, n, v in fields:
            setu(d, 56 + st, n, v & ((1 << n) - 1))
        out.append(case(d, nbits))

    def app6(dac, fid, nbits, fields=()):
        d = msg(rng, 6); setu(d, 72, 10, dac); setu(d, 82, 6, fid)
        for st, n, v in fields:
            setu(d, 88 + st, n, v & ((1 << n) - 1))
        out.append(case(d, nbits))

    for nwp in (0, 1, 2, 5, 16, 17, 31):  # route: waypoint count, room for fewer, tiny and negative coordinates
        for nbits in (100, 117, 172, 227, 500, 1000, 1064):
            app8(1, 27, nbits, [(56, 5, nwp), (61, 28, -1), (89, 27, 1), (116, 28, -600000), (144, 27, 3)])
            app6(1, 28, min(nbits + 32, 1064), [(56, 5, nwp), (61, 28, 0), (89, 27, -3)])
    for nbits in (100, 111, 112, 175, 176, 183, 184, 247, 248, 500, 600, 700, 1000):  # Swedish route: legs and the last leg
        app8(265, 1, nbits, [(1, 28, -5), (29, 27, 2), (76, 22, 5), (98, 22, -2), (57, 10, 0)])
        app8(265, 1, nbits, [(1, 28, 108000000), (29, 27, -54000000)])
    for lo, la, dr, sp in ((0, 0, 360, 255), (-1, 1, 12, 7), (10800000, -5400000, 359, 254), (10800001, 0, 0, 0), (5, -5400001, 1, 1)):
        for nbits in (120, 300, 350, 400):  # tidal window: valid and off-the-globe points, -1 for "not available"
            app6(1, 32, nbits, [(9, 25, lo), (34, 24, la), (80, 9, dr), (89, 8, sp), (97, 25, -lo), (122, 24, la), (157, 9, dr),
                                (166, 8, sp), (174, 25, lo), (199, 24, -la), (245, 9, dr), (254, 8, sp)])
    for nbits in (100, 175, 176, 295, 296, 415, 416, 535, 536, 1064):  # VTS targets: 1-4 records, ids with '@', ' ' and '"'
        app8(1, 17, nbits, [(2, 6, 0), (8, 6, 34), (14, 6, 32), (38, 6, 0), (48, 24, -1), (72, 25, 1)])
    for idt in range(4):  # VTS target (1,16): text id, numeric id below and above 2^31, short frame
        for hi in (0, 1, 1023):
            for nbits in (175, 176, 200):
                app8(1, 16, nbits, [(0, 2, idt), (2, 10, hi), (12, 32, 12345678)])
    for mid in (0, 1, 2, 3, 4, 5, 6, 7, 63):  # SLS meteo: every report id, at and below its length
        for nbits in (120, 263, 264, 271, 272, 400):
            app8(366, 1, nbits, [(2, 6, mid)])
            app6(316, 1, nbits + 32, [(2, 6, mid)])
    for rt in (0, 1, 2, 3, 4, 15):  # environmental sensor report: every body, headers only, short frames
        for nbits in (70, 82, 83, 167, 168, 300):
            app8(367, 33, nbits, [(0, 4, rt), (91, 12, -4096), (91, 12, 5)])
        app8(1, 26, 82 + rt, [(0, 4, rt)])
    for variant in (0, 1):  # weather observation: both variants
        app8(1, 21, 360, [(0, 1, variant), (121, 25, 10860000), (146, 24, -5460000)])
    for y, mo, d, hh, mm, mag in ((0, 1, 1, 23, 59, 255), (26, 12, 31, 24, 0, 0), (255, 15, 31, 0, 60, 254), (1, 0, 5, 12, 30, 7)):
        app8(200, 23, 256, [(0, 8, y), (8, 4, mo), (12, 5, d), (17, 8, y), (25, 4, mo), (29, 5, d), (34, 5, hh), (39, 6, mm),
                            (45, 5, hh), (50, 6, mm), (170, 1, 1), (171, 8, mag), (179, 1, 0), (180, 8, mag)])
    for ids in ((0, 0, 0, 0), (1, 0, 2047, 5), (7, 8, 9, 10)):  # water level: gauges of id 0 are left out
        app8(200, 24, 168, [(12 + 25 * i, 11, g) for i, g in enumerate(ids)] + [(23, 1, 0), (48, 1, 1)])
    for sal in (0, 509, 510, 511):  # meteo-hydro: salinity below and at its "not available" values, water level offset
        app8(1, 31, 360, [(283, 9, sal), (145, 12, 4001 if sal == 511 else sal)])
    # tags: every mode, station on and off, rx time and toa on and off, hardware with characters to escape
    for mode in range(8):
        for station in (0, 17):
            for rx in (0, 1700000000123456, 1700000000000000, -5):
                for toa in (0, 1700000000654321):
                    out.append(case(msg(rng, rng.choice([1, 5, 18, 24])), 424, mode=mode, station=station, rxtime_us=rx, toa_us=toa,
                                    hardware=rng.choice(["", "H100", 'a"b\\c\td'])))
    # level / ppm: undefined, negative zero, rounding
    for level, ppm in ((1024.0, 1024.0), (1024.0, 0.1), (-0.0, -0.0), (-3.0000005, 2.5e-7), (-123.4567891, 12.3456785)):
        out.append(case(msg(rng, 1), 168, level=level, ppm=ppm, mode=1))
    # sentences: none, four, one with a NUL letter (the last letter of a 1064-bit message)
    out.append(case(msg(rng, 1), 168, sentences=()))
    out.append(case(msg(rng, 8), 1064, sentences=("!AIVDM,4,%d,3,B,%s,0*00" % (i + 1, "w" * 60) for i in range(4))))
    out.append(case(msg(rng, 8), 1064, sentences=("!AIVDM,1,1,,A,ab\0,0*00",)))
    return out


def random_cases(n, seed):
    rng = random.Random(seed)
    out = []
    for _ in range(n):
        typ = rng.randint(0, 63) if rng.random() < 0.05 else rng.randint(1, 28)
        nbits = rng.choice([rng.randint(1, 1064), rng.randint(1, 300), MIN_BITS[(typ - 1) % 28] + rng.randint(-8, 40)])
        nbits = min(max(nbits, 1), 1064)
        d = msg(rng, typ)
        if typ in (6, 8, 25, 26) and rng.random() < 0.5:
            dac, fid = rng.choice(ASM6 + ASM8)
            pos = 72 if typ == 6 or (typ in (25, 26) and getu(d, 38, 1)) else 40
            setu(d, pos, 10, dac)
            setu(d, pos + 10, 6, fid)
        sents = ["!AIVDM,1,1,,%s,%s,0*%02X" % (rng.choice("AB"), "".join(rng.choice("0123456789:;<=>?@ABCDEFGHIJKLMNOPQRSTUVW`abcdefghijklmnopqrstuvw")
                                                                      for _ in range(rng.randint(1, 60))), rng.randrange(256))
                 for _ in range(rng.randint(0, 4))]
        out.append(case(d, nbits, rng.choice("AB12"), sents, rng.choice([1024.0, rng.uniform(-80, 0)]), rng.choice([1024.0, rng.uniform(-10, 10)]),
                        mode=rng.randint(0, 7), station=rng.choice([0, rng.randint(1, 1 << 20)]),
                        rxtime_us=rng.choice([0, rng.randint(0, 1 << 52)]), toa_us=rng.choice([0, rng.randint(1, 1 << 52)]),
                        version=rng.randint(0, 200), driver=rng.randint(0, 30), hardware=rng.choice(["", "RTL-SDR", "H100 80GB"])))
    return out
