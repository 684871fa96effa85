#!/usr/bin/env python
"""bench_clock.py -- what a receive time per frame (aisgpu_set_clock) costs: `python tools/bench_clock.py` prints ONE JSON line.

Batch 1024 streams of CF32 at 1536 kS/s, N = 131072 samples per stream and submit, inputs resident in HBM, synthetic bursts at
--density messages per second per stream, ModelDefault (coherent chain).  For NMEA_TAG and JSON_FULL, an engine without a clock
(every record prints the tag's time) and one with a recording clock (every record prints its frame's stamp: 8 bytes uploaded per
frame beside its aisgpu_msg), in one process, alternated round by round:
  step_ms_plain / _clock          : one aisgpu_submit_device plus the polls that publish its frames and their records, wall clock,
                                    median over --blocks rounds;
  fmt_kernels_ms_plain / _clock   : device time of the four format kernels per step (torch.profiler, CUDA activity);
plus the card's name and power limit read in the same run.  Needs a GPU (no fallback); writes nothing into the tree."""
import argparse
import ctypes as C
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
        raise SystemExit("bench_clock.py needs a CUDA device: there is no CPU path to time")
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
    starts = [1700000000000000 + 1000 * s for s in range(B)]

    def engines(fmt):
        out = {}
        for k in ("plain", "clock"):
            e = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=FS, n_streams=B, max_chunk=N, host_staging=False, max_frames=1 << 20)
            if k == "clock":
                e.set_clock(starts)
            e.lines_enable(fmt, aisgpu.make_tag(**TAG), 256 << 20)
            out[k] = e
        return out

    # the records are read into one buffer, as a caller that forwards them would, and not turned into Python objects
    lib, cap = aisgpu.load(), 16 << 20
    jbuf = C.create_string_buffer(cap)
    nb_, nr_ = C.c_size_t(0), C.c_int(0)

    def stepper(engs, text):
        cnt = {k: 0 for k in engs}

        def step(k):
            e = engs[k]
            e.submit_device(z[cnt[k] % R].data_ptr(), N, N)
            t = cnt[k]
            cnt[k] += 1
            fr, _ = e.poll_upto_count(t)
            while True:
                rc = lib.aisgpu_poll_lines(e.h, t, jbuf, cap, C.byref(nb_), C.byref(nr_))
                if rc != 0:
                    raise SystemExit("aisgpu_poll_lines rc=%d" % rc)
                if nr_.value == 0:
                    break
                text[k] += nb_.value
            return fr
        return step

    from torch.profiler import ProfilerActivity, profile
    out = {}
    for fmt, name in ((aisgpu.MSGFORMAT_NMEA_TAG, "NMEA_TAG"), (aisgpu.MSGFORMAT_JSON_FULL, "JSON_FULL")):
        engs = engines(fmt)
        text = {k: 0 for k in engs}
        step = stepper(engs, text)
        for k in engs:
            for _ in range(args.warmup):
                step(k)
        blocks = max(1, min(args.blocks, args.steps))
        per = max(1, args.steps // blocks)
        ms = {k: [] for k in engs}
        frames = {k: 0 for k in engs}
        text.update({k: 0 for k in engs})
        for _ in range(blocks):
            for k in engs:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(per):
                    frames[k] += step(k)
                torch.cuda.synchronize()
                ms[k].append((time.perf_counter() - t0) * 1e3 / per)
        timed_text = dict(text)
        kern = {k: [] for k in engs}
        for _ in range(max(1, args.blocks // 2)):
            for k in engs:
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(4):
                        step(k)
                    torch.cuda.synchronize()
                kern[k].append(sum(e.device_time_total for e in prof.key_averages() if "k_fmt" in e.key) / 1e3 / 4)
        out[name] = {"step_ms_plain": B_.median(ms["plain"]), "step_ms_clock": B_.median(ms["clock"]),
                     "step_spread_plain": [min(ms["plain"]), max(ms["plain"])], "step_spread_clock": [min(ms["clock"]), max(ms["clock"])],
                     "fmt_kernels_ms_plain": B_.median(kern["plain"]), "fmt_kernels_ms_clock": B_.median(kern["clock"]),
                     "fmt_spread_plain": [min(kern["plain"]), max(kern["plain"])],
                     "fmt_spread_clock": [min(kern["clock"]), max(kern["clock"])],
                     "frames_per_step_plain": frames["plain"] / (blocks * per),
                     "frames_per_step_clock": frames["clock"] / (blocks * per),
                     "record_bytes_per_step_plain": timed_text["plain"] / (blocks * per),
                     "record_bytes_per_step_clock": timed_text["clock"] / (blocks * per)}
        for e in engs.values():
            e.close()
    s = out["JSON_FULL"]
    B_.emit({"metric": "step time with a recording clock over without (JSON_FULL records)", "value": s["step_ms_clock"] / s["step_ms_plain"],
             "unit": "ratio", "higher_is_better": False, "n_gpus": 1, "steps": args.steps,
             "config": {"workload": "batch=%d CF32 streams @%d S/s, chunk %d samples, %.0f msg/s per stream, ModelDefault" % (B, FS, N, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "results": out})


if __name__ == "__main__":
    main()
