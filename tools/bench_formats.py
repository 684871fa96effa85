#!/usr/bin/env python
"""bench_formats.py -- the output records of every message format on the GPU: `python tools/bench_formats.py` prints ONE JSON line.

Batch 1024 streams of CF32 at 1536 kS/s, N = 131072 samples per stream and submit (85 ms of signal), inputs resident in HBM, bursts
at --density messages per second per stream (half per channel; 50 is a busy shore station).  For ModelStandard (FM chain) and
ModelDefault (coherent chain) and each format (--formats, default all nine) an engine with aisgpu_lines_enable is timed in
alternation with one without; a step is one aisgpu_submit_device plus the poll that publishes its frames (and aisgpu_poll_lines of
its records), wall clock, median over --blocks rounds.  Reported per chain and format:
  ms_per_step_off / _on, frames_per_step, records_polled
  format_kernels_ms_per_step : device time of the four format kernels per step (torch.profiler, CUDA activity)
  device_records_per_s       : records per second of those kernels
  parity                     : one step's records against aisgpu_msg_format from the engine's counters, and sampled ones against
                               the reference's OutputMessage records (oracle/_ref)
plus the card's name and power limit read in the same run.  Needs a GPU (no fallback); writes nothing into the tree."""
import argparse
import ctypes as C
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, _p)
import bench as B_  # noqa: E402  (one JSON line on stdout, median)

FS, N, UNIQUE, RESIDENT = 1536000, 131072, 32, 2
TAG = dict(version=1, driver=0, hardware="bench", mode=7, rxtime_us=1700000000000000, toa_us=0, station=0)


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
    ap.add_argument("--blocks", type=int, default=4)
    ap.add_argument("--density", type=float, default=50.0, help="messages per second per stream")
    ap.add_argument("--parity-lines", type=int, default=1000)
    ap.add_argument("--formats", default="1,2,3,4,5,6,7,8,9")
    args = ap.parse_args()
    import numpy as np
    import torch
    import aisgpu
    import aissynth as S
    import oracle_fmt
    if not torch.cuda.is_available():
        raise SystemExit("bench_formats.py needs a CUDA device: there is no CPU path to time")
    dev = torch.device("cuda", 0)
    B, R = args.batch, RESIDENT
    per_ch = max(1, int(round(args.density / 2)))
    uniq = np.stack([S.random_stream(FS, N * R, 7000 + u, bursts_per_sec=(per_ch, per_ch), multi_sentence=True)[0] for u in range(UNIQUE)])
    ud = torch.from_numpy(uniq).to(dev)
    z = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
    for b0 in range(0, B, UNIQUE):
        nb = min(UNIQUE, B - b0)
        z[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
    del ud
    torch.cuda.synchronize()
    lib = aisgpu.load()
    cap = 64 << 20
    jbuf = C.create_string_buffer(cap)
    nb_, nl_ = C.c_size_t(0), C.c_int(0)
    out = {}
    for model, chain in ((aisgpu.MODEL_STANDARD, "fm"), (aisgpu.MODEL_DEFAULT, "coherent")):
        out[chain] = {}
        for fmt in [int(f) for f in args.formats.split(",")]:
            engs = {k: aisgpu.Engine(model=model, sample_rate=FS, n_streams=B, max_chunk=N, host_staging=False, max_frames=1 << 20)
                    for k in ("off", "on")}
            engs["on"].lines_enable(fmt, aisgpu.make_tag(**TAG), 256 << 20)
            cnt = {"off": 0, "on": 0}
            seen = {"frames": [], "records": 0, "bytes": 0}

            def step(k):
                e = engs[k]
                e.submit_device(z[cnt[k] % R].data_ptr(), N, N)
                t = cnt[k]
                cnt[k] += 1
                fr, _ = e.poll_upto_count(t)
                if k == "on":
                    while True:
                        rc = lib.aisgpu_poll_lines(e.h, t, jbuf, cap, C.byref(nb_), C.byref(nl_))
                        if rc not in (0, aisgpu.EOVERFLOW) or nl_.value == 0:
                            break
                        seen["records"] += nl_.value
                        seen["bytes"] += nb_.value
                return fr

            for k in engs:
                for _ in range(args.warmup):
                    step(k)
            blocks = max(1, min(args.blocks, args.steps))
            per = max(1, args.steps // blocks)
            ms = {"off": [], "on": []}
            frames = 0
            for _ in range(blocks):
                for k in ("off", "on"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(per):
                        f = step(k)
                        if k == "on":
                            frames += f
                    torch.cuda.synchronize()
                    ms[k].append((time.perf_counter() - t0) * 1e3 / per)
            nsteps = blocks * per
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(4):
                    step("on")
                torch.cuda.synchronize()
            kern = sum(e.device_time_total for e in prof.key_averages() if "k_fmt" in e.key) / 1e3 / 4  # ms per step
            fr_per_step = frames / nsteps
            # parity on a fresh engine of the same format: every frame of two steps formatted on the host from a zeroed state
            e = aisgpu.Engine(model=model, sample_rate=FS, n_streams=B, max_chunk=N, host_staging=False, max_frames=1 << 20)
            e.lines_enable(fmt, aisgpu.make_tag(**TAG), 256 << 20)
            msgs, text = [], []
            for t in range(2):
                e.submit_device(z[t % R].data_ptr(), N, N)
                msgs += e.poll_upto(t, batch=8192)
                text.append(e.poll_lines(t, cap=cap)[0])
            e.close()
            tag = aisgpu.make_tag(**TAG)
            st = aisgpu.FormatState(0, 0)
            host = [aisgpu.msg_format(m, tag, fmt, st) for m in msgs]
            mism_ref = None
            checked = min(len(msgs), args.parity_lines)
            if oracle_fmt.have_ref():
                oracle_fmt.hub(0)
                oracle_fmt.group_seed(0)
                mism_ref = 0
                for m, h in list(zip(msgs, host))[:checked]:
                    want = oracle_fmt.ref_record(fmt, m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value,
                                                 C.c_float(m.ppm).value, TAG["version"], TAG["driver"], TAG["hardware"], TAG["mode"],
                                                 TAG["rxtime_us"], TAG["toa_us"], TAG["station"], False, m.start_idx, m.end_idx)
                    mism_ref += h != want
            out[chain][str(fmt)] = {
                "ms_per_step_off": B_.median(ms["off"]), "ms_per_step_on": B_.median(ms["on"]),
                "spread_off": [min(ms["off"]), max(ms["off"])], "spread_on": [min(ms["on"]), max(ms["on"])],
                "frames_per_step": fr_per_step, "records_polled": seen["records"], "bytes_polled": seen["bytes"],
                "format_kernels_ms_per_step": kern, "device_records_per_s": fr_per_step / (kern * 1e-3) if kern > 0 else None,
                "parity": {"records": len(msgs), "device_equals_host": b"".join(text) == b"".join(host),
                           "checked_vs_reference": checked if mism_ref is not None else 0, "mismatches_vs_reference": mism_ref}}
            for x in engs.values():
                x.close()
    first = sorted(out["coherent"])[0]
    B_.emit({"metric": "output records per second formatted on the GPU (coherent chain, format %s)" % first,
             "value": out["coherent"][first]["device_records_per_s"], "unit": "records/s", "higher_is_better": True, "n_gpus": 1, "steps": args.steps,
             "config": {"workload": "batch=%d CF32 streams @%d S/s, chunk %d samples, %.0f msg/s per stream" % (B, FS, N, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "chains": out})


if __name__ == "__main__":
    main()
