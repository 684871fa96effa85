#!/usr/bin/env python
"""bench_tune.py -- what a per-stream digital tune (aisgpu_set_tuning) costs: `python tools/bench_tune.py` prints ONE JSON line.

Batch 1024 streams at 1536 kS/s, N = 131072 samples per stream and submit, inputs resident in HBM, synthetic bursts at --density
messages per second per stream.  The plain engine reads the traffic at baseband; the tuned engine reads the same traffic placed at
an offset of its own per stream (up to +-700 kHz) and mixes it back, so both decode the same frames.  For CF32 and CU8 input and
for ModelStandard (FM chain) and ModelDefault (coherent chain), in one process, alternated round by round:
  step_ms_plain / _tuned : one aisgpu_submit_device plus the poll that publishes its frames, wall clock, median over --blocks rounds;
  tune_kernel_ms         : device time of k_tune per step (torch.profiler, CUDA activity, a run of its own);
  tune_bytes / share_of_hbm_peak : input bytes + 8 B per sample, over that time, as a share of the 3.35 TB/s of the H100 SXM data
                           sheet;
  parity_mismatches      : sampled streams whose frames differ from a plain CF32 engine fed aisgpu_tune_restate of their input;
plus the card's name and power limit read in the same run.  Needs a GPU (no fallback); writes nothing into the tree."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, _p)
import bench as B_  # noqa: E402  (one JSON line on stdout, median)

FS, N, UNIQUE, RESIDENT = 1536000, 131072, 32, 2
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
SAMPLED = (0, 1, 17, 513, 1023)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def offset_of(u):
    return int((u * 45677) % 1400001) - 700000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--density", type=float, default=50.0, help="messages per second per stream")
    args = ap.parse_args()
    import numpy as np
    import torch
    import aisgpu
    import aissynth as S
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("bench_tune.py needs a CUDA device: there is no CPU path to time")
    dev = torch.device("cuda", 0)
    B, R = args.batch, RESIDENT
    per_ch = max(1, int(round(args.density / 2)))
    base = np.stack([S.random_stream(FS, N * R, 9100 + u, bursts_per_sec=(per_ch, per_ch))[0] for u in range(UNIQUE)])
    t = np.arange(N * R, dtype=np.float64)
    moved = np.stack([(base[u] * np.exp(2j * np.pi * offset_of(u) * t / FS)).astype(np.complex64) for u in range(UNIQUE)])
    offsets = [offset_of(s % UNIQUE) for s in range(B)]

    def resident(rows, fmt):
        raw = rows if fmt == aisgpu.FMT_CF32 else np.stack([S.to_cu8(x) for x in rows])
        ud = torch.from_numpy(np.ascontiguousarray(raw).view(np.uint8)).to(dev).view(UNIQUE, R, -1)
        z = torch.empty((R, B, ud.shape[2]), dtype=torch.uint8, device=dev)
        for b0 in range(0, B, UNIQUE):
            nb = min(UNIQUE, B - b0)
            z[:, b0:b0 + nb, :] = ud[:nb].permute(1, 0, 2)
        torch.cuda.synchronize()
        return raw, z

    out = {"step": {}, "tune_kernel": {}, "parity": {}}
    for fmt, fname in ((aisgpu.FMT_CF32, "CF32"), (aisgpu.FMT_CU8, "CU8")):
        _, zp = resident(base, fmt)
        moved_raw, zt = resident(moved, fmt)
        bps = 8 if fmt == aisgpu.FMT_CF32 else 2
        epp = 1 if fmt == aisgpu.FMT_CF32 else 2  # raw array elements per sample
        for model, chain in ((aisgpu.MODEL_STANDARD, "fm"), (aisgpu.MODEL_DEFAULT, "coherent")):
            engs, inp, cnt = {}, {"plain": zp, "tuned": zt}, {"plain": 0, "tuned": 0}
            for k in ("plain", "tuned"):
                engs[k] = aisgpu.Engine(model=model, sample_rate=FS, fmt=fmt, n_streams=B, max_chunk=N, host_staging=False,
                                        max_frames=1 << 20)
                if k == "tuned":
                    engs[k].set_tuning(offsets)
            got = {s: [] for s in SAMPLED}

            def step(k, keep=False):
                e = engs[k]
                e.submit_device(inp[k][cnt[k] % R].data_ptr(), N, N)
                t_ = cnt[k]
                cnt[k] += 1
                if keep:
                    for m in e.poll_upto(t_):
                        if m.stream in got:
                            got[m.stream].append(m)
                    return 0
                return e.poll_upto_count(t_)[0]

            for _ in range(R):  # the first R steps of the tuned engine: kept for the parity check
                step("tuned", keep=True)
                step("plain")
            for k in engs:
                for _ in range(args.warmup):
                    step(k)
            blocks = max(1, min(args.blocks, args.steps))
            per = max(1, args.steps // blocks)
            ms = {k: [] for k in engs}
            frames = {k: 0 for k in engs}
            for _ in range(blocks):
                for k in engs:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(per):
                        frames[k] += step(k)
                    torch.cuda.synchronize()
                    ms[k].append((time.perf_counter() - t0) * 1e3 / per)
            kern = []
            for _ in range(max(1, args.blocks // 2)):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(4):
                        step("tuned")
                    torch.cuda.synchronize()
                kern.append(sum(e.device_time_total for e in prof.key_averages() if "k_tune" in e.key) / 1e3 / 4)
            for e in engs.values():
                e.close()
            key = "%s_%s" % (fname, chain)
            out["step"][key] = {"step_ms_plain": B_.median(ms["plain"]), "step_ms_tuned": B_.median(ms["tuned"]),
                                "spread_plain": [min(ms["plain"]), max(ms["plain"])], "spread_tuned": [min(ms["tuned"]), max(ms["tuned"])],
                                "frames_per_step_plain": frames["plain"] / (blocks * per),
                                "frames_per_step_tuned": frames["tuned"] / (blocks * per)}
            kms = B_.median(kern)
            nbytes = B * N * (bps + 8)
            out["tune_kernel"][key] = {"tune_kernel_ms": kms, "spread": [min(kern), max(kern)], "tune_bytes": nbytes,
                                       "achieved_GBps": nbytes / (kms * 1e-3) / 1e9 if kms > 0 else None,
                                       "share_of_hbm_peak": nbytes / (kms * 1e-3) / HBM_PEAK if kms > 0 else None}
            # parity: the sampled streams' frames of the tuned engine's first R steps against a plain CF32 engine on the restated input
            ref = aisgpu.Engine(model=model, sample_rate=FS, fmt=aisgpu.FMT_CF32, n_streams=len(SAMPLED), max_chunk=N)
            want = {s: [] for s in SAMPLED}
            for c in range(R):
                rows = [aisgpu.tune_restate(fmt, FS, offsets[s], c * N, moved_raw[s % UNIQUE][c * N * epp:(c + 1) * N * epp])
                        for s in SAMPLED]
                ref.submit(np.ascontiguousarray(np.stack(rows)), N)
                for m in ref.poll():
                    want[SAMPLED[m.stream]].append(m)
            ref.close()
            mism = [s for s in SAMPLED if [(m.key(), m.start_idx, m.end_idx) for m in got[s]] != [(m.key(), m.start_idx, m.end_idx) for m in want[s]]]
            out["parity"][key] = {"sampled_streams": list(SAMPLED), "parity_mismatches": len(mism),
                                  "frames_checked": sum(len(v) for v in want.values())}
    s = out["step"]["CF32_coherent"]
    B_.emit({"metric": "step time with a tuning table over without (CF32, coherent chain)", "value": s["step_ms_tuned"] / s["step_ms_plain"],
             "unit": "ratio", "higher_is_better": False, "n_gpus": 1, "steps": args.steps,
             "config": {"workload": "batch=%d streams @%d S/s, chunk %d samples, %.0f msg/s per stream" % (B, FS, N, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "results": out})


if __name__ == "__main__":
    main()
