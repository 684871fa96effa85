"""-m gpu: the device restatements of the C library functions the reference calls, bit for bit against the host C library.

tests/host/exact_math_check.cu evaluates fd_atan2f_common and fd_atan2f (csrc/exact.cuh) against atan2f, habs against hypotf, and
v2_sincosf (csrc/v2_math.cuh) against sincosf / sinf / cosf on the GPU, compiled with the library's own nvcc flags.  The parity tests
reach only a sliver of these domains -- no sample of ordinary input is ever zero, subnormal or saturated -- so this is where the rare
branches of the restatements are checked:
* atan2: every pair of a special set (signed zeros, subnormals, FLT_MIN, 1 and its neighbours, FLT_MAX, infinities, NaN), every
  (exponent, exponent) pair with four sign combinations and 16 mantissa pairs, and 1e8 random bit patterns; NaN compared as a class;
* habs: 5e7 finite pairs (random, subnormal, near FLT_MAX); on the special set the one documented difference is pinned:
  habs(inf, NaN) is NaN where hypotf gives inf (the engine never sees non-finite input, DESIGN.md section 2);
* v2_sincosf: every float of [-8, 8], the engine's domain [-1.27, 2 pi) with a margin;
* v2_atan2_fast(+-0, +-0) == +0.
"""
import os
import subprocess

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exact_math_against_libm(built, tmp_path):
    exe = str(tmp_path / "exact_math_check")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.check_call([nvcc] + built.NVCC_FLAGS + ["-I", os.path.join(ROOT, "ais-catcher_b200", "csrc"), "-o", exe,
                                                       os.path.join(ROOT, "tests", "host", "exact_math_check.cu")])
    out = subprocess.run([exe, "100000000", "50000000", "1"], capture_output=True, text=True, timeout=1200)
    print(out.stdout)
    res = {}
    for line in out.stdout.splitlines():
        w = line.split()
        if len(w) >= 5 and w[1] == "checked" and w[3] == "mismatches":
            res[w[0]] = (int(w[2]), int(w[4]), int(w[6]) if len(w) > 6 and w[5] == "rare" else 0)
    assert out.returncode == 0, (out.returncode, out.stdout[-2000:], out.stderr[-2000:])
    assert {k: v[1] for k, v in res.items()} == {"atan2_special": 0, "atan2_exponents": 0, "atan2_random": 0, "habs_special": 0,
                                                  "habs_random": 0, "sincos": 0, "v2_atan2_zero": 0}, res
    # the arguments were checked and the rare branch was reached
    assert res["atan2_special"][0] == 20 * 20 and res["atan2_special"][2] == 362
    assert res["atan2_exponents"][0] == 256 * 256 * 64 and res["atan2_exponents"][2] > 1000000
    assert res["atan2_random"][0] == 100000000 and res["atan2_random"][2] > 10000000
    assert res["habs_random"][0] == 50000000
    assert res["sincos"][0] == 2 * (0x41000000 + 1)
