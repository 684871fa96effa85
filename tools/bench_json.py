#!/usr/bin/env python
"""bench_json.py -- the full AIS JSON on the GPU: `python tools/bench_json.py` prints ONE JSON line.

Batch 1024 streams of CF32 at 1536 kS/s, N = 131072 samples per stream and submit (85 ms of signal), inputs resident in HBM, bursts
at --density messages per second per stream (half per channel; 50 is a busy shore station).  For ModelStandard (FM chain) and
ModelDefault (coherent chain) two engines are timed in alternation, one with aisgpu_json_enable and one without; a step is one
aisgpu_submit_device plus the poll that publishes its frames (and, with JSON, aisgpu_poll_json of its lines), wall clock, median
over --blocks rounds.  Reported per chain:
  ms_per_step_json_off / _on, frames_per_step
  decode_kernels_ms_per_step : device time of the three JSON kernels per step (torch.profiler, CUDA activity)
  device_lines_per_s          : lines per second of those kernels
  host_lines_per_s_one_thread : aisgpu_msg_json_full over the same frames on one host thread (called through ctypes, so this
                                counts the call overhead too)
  parity                      : sampled lines against aisgpu_msg_json_full and the reference's JSONAIS line (oracle/_ref)
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
    ap.add_argument("--parity-lines", type=int, default=3000)
    args = ap.parse_args()
    import numpy as np
    import torch
    import aisgpu
    import aissynth as S
    import oracle_json
    if not torch.cuda.is_available():
        raise SystemExit("bench_json.py needs a CUDA device: there is no CPU path to time")
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
        engs = {k: aisgpu.Engine(model=model, sample_rate=FS, n_streams=B, max_chunk=N, host_staging=False, max_frames=1 << 20)
                for k in ("off", "on")}
        engs["on"].json_enable(aisgpu.make_tag(**TAG), 256 << 20)
        cnt = {"off": 0, "on": 0}
        lines = {"n": 0, "bytes": 0}

        def step(k):
            e = engs[k]
            e.submit_device(z[cnt[k] % R].data_ptr(), N, N)
            t = cnt[k]
            cnt[k] += 1
            fr, _ = e.poll_upto_count(t)
            if k == "on":
                while True:
                    rc = lib.aisgpu_poll_json(e.h, t, jbuf, cap, C.byref(nb_), C.byref(nl_))
                    if rc not in (0, aisgpu.EOVERFLOW) or nl_.value == 0:
                        break
                    lines["n"] += nl_.value
                    lines["bytes"] += nb_.value
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
        # device time of the JSON kernels
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(4):
                step("on")
            torch.cuda.synchronize()
        kern = sum(e.device_time_total for e in prof.key_averages() if "k_json" in e.key) / 1e3 / 4  # ms per step
        fr_per_step = frames / nsteps
        # frames for the host comparison and parity: one more step, polled as structs
        e = engs["on"]
        e.submit_device(z[cnt["on"] % R].data_ptr(), N, N)
        t = cnt["on"]
        cnt["on"] += 1
        msgs = e.poll_upto(t, batch=8192)
        dl = e.poll_json(t, cap=cap)
        structs = [aisgpu.msg_struct(m) for m in msgs]
        tag = aisgpu.make_tag(**TAG)
        hb = C.create_string_buffer(1 << 16)
        f = lib.aisgpu_msg_json_full
        t0 = time.perf_counter()
        for s in structs:
            f(C.byref(s), C.byref(tag), hb, 1 << 16)
        host_lps = len(structs) / (time.perf_counter() - t0)
        mism_host = mism_ref = checked = 0
        have_ref = oracle_json.have_ref()
        for m, line in list(zip(msgs, dl))[:args.parity_lines]:
            got = line.encode("utf-8", "surrogateescape")
            h = aisgpu.msg_json_full(m, tag)
            checked += 1
            if got != h:
                mism_host += 1
            if have_ref:
                want = oracle_json.ref_line(m.data, m.nbits, m.channel, m.nmea, C.c_float(m.level).value, C.c_float(m.ppm).value,
                                            TAG["version"], TAG["driver"], TAG["hardware"], TAG["mode"], TAG["rxtime_us"], TAG["toa_us"],
                                            TAG["station"])
                mism_ref += got != want
        out[chain] = {"ms_per_step_json_off": B_.median(ms["off"]), "ms_per_step_json_on": B_.median(ms["on"]),
                      "spread_off": [min(ms["off"]), max(ms["off"])], "spread_on": [min(ms["on"]), max(ms["on"])],
                      "frames_per_step": fr_per_step, "lines_polled": lines["n"], "json_bytes_polled": lines["bytes"],
                      "decode_kernels_ms_per_step": kern, "device_lines_per_s": fr_per_step / (kern * 1e-3) if kern > 0 else None,
                      "host_lines_per_s_one_thread": host_lps,
                      "parity": {"lines_checked": checked, "mismatches_vs_host": mism_host,
                                 "mismatches_vs_reference": mism_ref if have_ref else None}}
        for e in engs.values():
            e.close()
    B_.emit({"metric": "full AIS JSON lines per second decoded on the GPU (coherent chain)", "value": out["coherent"]["device_lines_per_s"],
             "unit": "lines/s", "higher_is_better": True, "n_gpus": 1, "steps": args.steps,
             "config": {"workload": "batch=%d CF32 streams @%d S/s, chunk %d samples, %.0f msg/s per stream" % (B, FS, N, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "chains": out})


if __name__ == "__main__":
    main()
