"""CPU: the streaming front end's lane planner (st_plan, ais-catcher_b200/csrc/fe_stream.cuh) through its test hook in the library.
Every stream's super-steps are split over L lanes, the first L - r take q, the last r take q + 1."""
import ctypes as C
import os
import random

import pytest

import aisgpu


@pytest.fixture(scope="module")
def plan():
    if not os.path.exists(aisgpu.LIB_PATH):
        pytest.skip("libaisgpu.so not built")
    lib = C.CDLL(aisgpu.LIB_PATH)
    f = lib.aisgpu_dbg_plan_lanes
    f.restype = C.c_int
    f.argtypes = [C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]

    def call(B, nss, warm, wpc, slots, min_ratio=4, forced=0):
        L, q, r = C.c_int(), C.c_int(), C.c_int()
        ok = f(B, nss, warm, wpc, slots, min_ratio, forced, C.byref(L), C.byref(q), C.byref(r))
        return (L.value, q.value, r.value) if ok else None
    return call


def cost(B, nss, warm, wpc, slots, L):
    ctas = -(-(-(-B * L // 32)) // wpc)
    waves = -(-ctas // slots)
    return waves * (-(-nss // L) + warm)


def test_bench_shape_is_one_balanced_wave(plan):
    # 1024 streams x 131072 samples @1536k: 2048 super-steps of 64 samples, 6 warm-up super-steps, four-warp CTAs, one per SM
    L, q, r = plan(1024, 2048, 6, 4, 132)
    assert (L, q, r) == (16, 128, 0)
    assert -(-1024 * L // 32) // 4 == 128  # CTAs: all resident at once on the 132 SMs of an H100


def test_invariants_random(plan):
    rnd = random.Random(5)
    for _ in range(3000):
        B = rnd.choice([1, 2, 3, 5, 64, 512, 1024, 4096, 8192, 65536])
        warm = rnd.choice([1, 2, 3, 6])
        nss = rnd.randint(1, 20000)
        wpc = rnd.choice([1, 4])
        slots = 132 * rnd.choice([1, 2, 8, 12])
        ratio = rnd.choice([1, 4])
        forced = rnd.choice([0, 0, 0, 1, 7, 32, 100, 100000])
        got = plan(B, nss, warm, wpc, slots, ratio, forced)
        if nss < warm * ratio:
            assert got is None  # the block does not cover `ratio` warm-ups: the tiled kernel takes it
            continue
        L, q, r = got
        assert L >= 1 and q * L + r == nss and 0 <= r < L
        assert q >= warm * ratio  # no lane shorter than `ratio` warm-ups: a lane's warm-up never reaches beyond its left neighbour
        if forced:
            assert L == min(forced, nss // (warm * ratio))
        else:  # nothing beats the chosen split by more than the 3 % margin that prefers fewer lanes (less warm-up traffic)
            best = min(cost(B, nss, warm, wpc, slots, l) for l in range(1, nss // (warm * ratio) + 1))
            assert cost(B, nss, warm, wpc, slots, L) <= best / 0.97 + 1e-9
