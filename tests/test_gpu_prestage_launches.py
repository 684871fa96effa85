"""GPU: aisgpu_last_launches counts every kernel a submit enqueues, at each resampler pre-stage and in each back-end chain.  One
submit runs under torch.profiler with CUDA activity, and the kernels it records must equal the engine's count (for a group: the
leader's plus its members')."""
import json

import numpy as np
import pytest
import torch

import aisgpu
import aissynth as S

pytestmark = pytest.mark.gpu

M0, M1, M2, M3, M4, M11 = (aisgpu.MODEL_STANDARD, aisgpu.MODEL_BASE, aisgpu.MODEL_DEFAULT, aisgpu.MODEL_DISCRIMINATOR,
                           aisgpu.MODEL_CHALLENGER, aisgpu.MODEL_V2)
AB, X = aisgpu.MODE_AB, aisgpu.MODE_X

# name, models (the engine, then the members attached to it), rate, DSK, channel mode, PS_EMA, submit length
CASES = [
    # the four pre-stage chains
    ("cic_us_6000k", (M2,), 6000000, False, AB, True, 65536),     # 4 x Downsample2CIC5 -> Upsample
    ("dsk_288k", (M2,), 288000, False, AB, True, 16384),          # DownsampleKFilter of the caller's input
    ("cic_us_dsk_250k", (M2,), 250000, False, AB, True, 16384),   # conversion -> Upsample -> DownsampleKFilter of every Upsample block
    ("cic_dsk_1152k", (M2,), 1152000, True, AB, True, 16384),     # 2 x Downsample2CIC5 -> DownsampleKFilter
    # the back-end chains: FM (models 0, 1, 3), coherent (2, 4) and V2 (11)
    ("m0_1536k", (M0,), 1536000, False, AB, True, 65536),
    ("m0_1536k_ps", (M0,), 1536000, False, AB, False, 65536),
    ("m1_1536k", (M1,), 1536000, False, AB, True, 65536),
    ("m1_1536k_ps", (M1,), 1536000, False, AB, False, 65536),
    ("m2_1536k", (M2,), 1536000, False, AB, True, 65536),
    ("m2_1536k_ps", (M2,), 1536000, False, AB, False, 65536),     # PhaseSearch instead of PhaseSearchEMA
    ("m4_1536k", (M4,), 1536000, False, AB, True, 65536),
    ("m11_1536k", (M11,), 1536000, False, AB, True, 65536),
    ("m0_x48k", (M0,), 48000, False, X, True, 16384),
    ("m2_x48k", (M2,), 48000, False, X, True, 16384),
    ("m3_48k", (M3,), 48000, False, AB, True, 16384),
    ("group_m2_m0_m11", (M2, M0, M11), 1536000, False, AB, True, 65536),  # fan-out + three back ends
]


@pytest.mark.parametrize("models,fs,dsk,mode,ps_ema,N", [c[1:] for c in CASES], ids=[c[0] for c in CASES])
def test_launch_count_matches_profiler(built, tmp_path, models, fs, dsk, mode, ps_ema, N):
    B, nsub = 2, 4
    x = np.stack([S.random_stream(fs, N * nsub, 40 + s)[0] for s in range(B)])
    eng = aisgpu.Engine(model=models[0], sample_rate=fs, n_streams=B, max_chunk=N, dsk=dsk, channel_mode=mode, ps_ema=ps_ema)
    members = [eng.attach(model=m) for m in models[1:]]
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
    launches = eng.last_launches() + sum(m.last_launches() for m in members)
    for m in members:
        m.close()
    eng.close()
    assert launches == len(kernels), "last_launches() = %d, profiler: %d kernels %r" % (launches, len(kernels), kernels)
