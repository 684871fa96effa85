#!/usr/bin/env python
"""GPU: step throughput for the other BASELINE.json configs (rate sweep, 6 MSPS AirSpy shape, PhaseSearch variants).
usage: rate_sweep.py fs:B:N:model:ps_ema ...   (synthetic bursts + noise, device-resident input, R=3 chunks cycled)"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "ais-catcher_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import aisgpu
import aissynth

dev = torch.device("cuda", 0)
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0  # H100 SXM data sheet, not measured
for spec in sys.argv[1:]:
    fs, B, N, model, ps_ema = [int(v) for v in spec.split(":")]
    R, U = 3, 8
    uniq = np.stack([aissynth.random_stream(fs, N * R, 2000 + u)[0] for u in range(U)])
    ud = torch.from_numpy(uniq.view(np.float32)).to(dev).view(U, N * R, 2)
    x = torch.empty((R, B, N, 2), dtype=torch.float32, device=dev)
    for b0 in range(0, B, U):
        nb = min(U, B - b0)
        x[:, b0:b0 + nb] = ud[:nb].view(nb, R, N, 2).permute(1, 0, 2, 3)
    torch.manual_seed(3)
    for r in range(R):
        x[r] += torch.randn_like(x[r]) * 0.005
    torch.cuda.synchronize()
    eng = aisgpu.Engine(model=model, sample_rate=fs, n_streams=B, max_chunk=N, ps_ema=bool(ps_ema), max_frames=1 << 21)
    for i in range(3):
        eng.submit_device(x[i % R].data_ptr(), N, N)
    eng.sync()
    eng.poll()
    est = torch.cuda.ExternalStream(eng.cuda_stream(), device=dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    K = 12
    e0.record(est)
    for i in range(K):
        eng.submit_device(x[i % R].data_ptr(), N, N)
    eng.join()
    e1.record(est)
    e1.synchronize()
    ms = e0.elapsed_time(e1) / K
    nm = len(eng.poll())
    iso = []
    for i in range(4):
        eng.submit_device(x[i % R].data_ptr(), N, N)
        eng.sync()
        iso.append(eng.last_frontend_ms())
    eng.poll()
    gbs = B * N * 8 / ms / 1e6
    print(json.dumps({"fs": fs, "B": B, "N": N, "model": model, "ps_ema": ps_ema, "ms_per_step": round(ms, 4), "GSps": round(B * N / ms / 1e6, 1),
                      "input_GBps": round(gbs, 1), "frac_of_hbm_peak": round(gbs / peak, 3), "last_frontend_launch_ms": round(min(iso), 4),
                      "msgs_per_step": nm // K}), flush=True)
    eng.close()
    del x, ud
    torch.cuda.empty_cache()
