#!/usr/bin/env python
"""bench_receivers.py -- what a receiver per stream (aisgpu_set_receivers) costs: `python tools/bench_receivers.py` prints ONE JSON line.

Batch 1024 streams of CF32 at 1536 kS/s, N = 131072 samples per stream and submit, inputs resident in HBM, synthetic bursts at
--density messages per second per stream.  The table gives every stream its own letters (AB / CD / 12 / ?X), station, hardware name,
driver and ipv4, with tag mode 3 as the config's, so both engines do the same work and differ only in where each row's level switch
and each record's context come from.  In one process, alternated round by round:
  step_ms_plain / _table      : one aisgpu_submit_device plus the poll that publishes its frames, wall clock, median over --blocks
                                rounds, for ModelStandard (FM chain) and ModelDefault (coherent chain);
  fmt_kernels_ms_plain / _table : device time of the four format kernels per step (torch.profiler, CUDA activity), coherent chain,
                                for NMEA_TAG and JSON_FULL;
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
TAG = dict(version=1, driver=0, hardware="bench", mode=3, rxtime_us=1700000000000000, toa_us=0, station=0)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def receivers(n):
    return [dict(channels=["AB", "CD", "12", "?X"][s % 4], station=s + 1, own_mmsi=-1, tag_mode=3, driver=s % 7,
                 hardware="station-%04d" % s, ipv4=0x0A000000 + s) for s in range(n)]


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
    if not torch.cuda.is_available():
        raise SystemExit("bench_receivers.py needs a CUDA device: there is no CPU path to time")
    dev = torch.device("cuda", 0)
    B, R = args.batch, RESIDENT
    per_ch = max(1, int(round(args.density / 2)))
    uniq = np.stack([S.random_stream(FS, N * R, 9000 + u, bursts_per_sec=(per_ch, per_ch), multi_sentence=True)[0] for u in range(UNIQUE)])
    ud = torch.from_numpy(uniq).to(dev)
    z = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
    for b0 in range(0, B, UNIQUE):
        nb = min(UNIQUE, B - b0)
        z[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
    del ud
    torch.cuda.synchronize()
    rx = receivers(B)

    def engines(model, fmt=None):
        out = {}
        for k in ("plain", "table"):
            e = aisgpu.Engine(model=model, sample_rate=FS, n_streams=B, max_chunk=N, host_staging=False, max_frames=1 << 20)
            if k == "table":
                e.set_receivers(rx)
            if fmt is not None:
                e.lines_enable(fmt, aisgpu.make_tag(**TAG), 256 << 20)
            out[k] = e
        return out

    def stepper(engs, fmt):
        cnt = {k: 0 for k in engs}

        def step(k):
            e = engs[k]
            e.submit_device(z[cnt[k] % R].data_ptr(), N, N)
            t = cnt[k]
            cnt[k] += 1
            fr, _ = e.poll_upto_count(t)
            if fmt is not None:
                e.poll_lines(t, cap=64 << 20)
            return fr
        return step

    out = {"step": {}, "format_kernels": {}}
    for model, chain in ((aisgpu.MODEL_STANDARD, "fm"), (aisgpu.MODEL_DEFAULT, "coherent")):
        engs = engines(model)
        step = stepper(engs, None)
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
        out["step"][chain] = {"step_ms_plain": B_.median(ms["plain"]), "step_ms_table": B_.median(ms["table"]),
                              "spread_plain": [min(ms["plain"]), max(ms["plain"])], "spread_table": [min(ms["table"]), max(ms["table"])],
                              "frames_per_step_plain": frames["plain"] / (blocks * per),
                              "frames_per_step_table": frames["table"] / (blocks * per)}
        for e in engs.values():
            e.close()
    from torch.profiler import ProfilerActivity, profile
    for fmt, name in ((aisgpu.MSGFORMAT_NMEA_TAG, "NMEA_TAG"), (aisgpu.MSGFORMAT_JSON_FULL, "JSON_FULL")):
        engs = engines(aisgpu.MODEL_DEFAULT, fmt)
        step = stepper(engs, fmt)
        for k in engs:
            for _ in range(args.warmup):
                step(k)
        kern = {k: [] for k in engs}
        for _ in range(max(1, args.blocks // 2)):
            for k in engs:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(4):
                        step(k)
                    torch.cuda.synchronize()
                kern[k].append(sum(e.device_time_total for e in prof.key_averages() if "k_fmt" in e.key) / 1e3 / 4)
        out["format_kernels"][name] = {"fmt_kernels_ms_plain": B_.median(kern["plain"]), "fmt_kernels_ms_table": B_.median(kern["table"]),
                                       "spread_plain": [min(kern["plain"]), max(kern["plain"])],
                                       "spread_table": [min(kern["table"]), max(kern["table"])]}
        for e in engs.values():
            e.close()
    s = out["step"]["coherent"]
    B_.emit({"metric": "step time with a receiver table over without (coherent chain)", "value": s["step_ms_table"] / s["step_ms_plain"],
             "unit": "ratio", "higher_is_better": False, "n_gpus": 1, "steps": args.steps,
             "config": {"workload": "batch=%d CF32 streams @%d S/s, chunk %d samples, %.0f msg/s per stream" % (B, FS, N, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "results": out})


if __name__ == "__main__":
    main()
