"""GPU: aisgpu_last_launches counts every kernel a submit enqueues at each resampler pre-stage.  One submit runs under
torch.profiler with CUDA activity, and the kernels it records must equal the engine's count."""
import json

import numpy as np
import pytest
import torch

import aisgpu
import aissynth as S

pytestmark = pytest.mark.gpu

# name, rate, DSK, submit length: the four pre-stage chains
CASES = [
    ("cic_us_6000k", 6000000, False, 65536),     # 4 x Downsample2CIC5 -> Upsample
    ("dsk_288k", 288000, False, 16384),          # DownsampleKFilter of the caller's input
    ("cic_us_dsk_250k", 250000, False, 16384),   # conversion -> Upsample -> DownsampleKFilter of every Upsample block
    ("cic_dsk_1152k", 1152000, True, 16384),     # 2 x Downsample2CIC5 -> DownsampleKFilter
]


@pytest.mark.parametrize("fs,dsk,N", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_launch_count_matches_profiler(built, tmp_path, fs, dsk, N):
    B, nsub = 2, 4
    x = np.stack([S.random_stream(fs, N * nsub, 40 + s)[0] for s in range(B)])
    eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, n_streams=B, max_chunk=N, dsk=dsk)
    for i in range(nsub - 1):  # module loading, and the Rotate table the next submit finds built
        eng.submit(np.ascontiguousarray(x[:, i * N:(i + 1) * N]), N)
    eng.join()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.submit(np.ascontiguousarray(x[:, (nsub - 1) * N:]), N)
        eng.join()
        torch.cuda.synchronize()
    trace = tmp_path / "trace.json"
    prof.export_chrome_trace(str(trace))
    with open(trace) as f:
        kernels = [e["name"] for e in json.load(f)["traceEvents"] if e.get("cat") == "kernel"]
    launches = eng.last_launches()
    eng.close()
    assert launches == len(kernels), "last_launches() = %d, profiler: %d kernels %r" % (launches, len(kernels), kernels)
