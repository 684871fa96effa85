#!/usr/bin/env python
"""bench_dump.py -- what the 48 kHz channel dump (aisgpu_dump_open, -go DUMP) costs.  Prints ONE JSON line per measurement.

Workload: batch 1024 CF32 @1536 kS/s, 131072 samples per stream and step (bench.py's default shape), ModelStandard.  Every stream is
dumped, so one step writes 2048 rows x 4096 samples x 8 B = 67 MB of WAV data into a directory this script creates and deletes.

  device    the batch is resident on the GPU (aisgpu_submit_device).  Blocks of --steps submits that end in aisgpu_sync (which also
            writes the last slots), timed with the host clock; an engine without a dump and one with a dump alternate, --reps times.
  e2e       the same from two pinned host buffers: aisgpu_submit_async(c) + aisgpu_poll_upto(c - 1), off and on alternated.
  profile   a separate run of a few dumped steps under torch.profiler: the export kernel's (k_c_fanout) time and achieved bandwidth
            (it reads and writes the rows once: 2 x 67 MB per step) and the duration of the device-to-host copy of each slot.

The card's name and power limit are read in the same run.  One file descriptor per file stays open while a dump is open (2048
here): the script raises its own soft RLIMIT_NOFILE to the hard limit.  Writes nothing into the tree.
"""
import argparse
import json
import os
import resource
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200")):
    sys.path.insert(0, _p)


def card():
    """(name, power limit in W) of GPU 0, read now."""
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True)
        name, watts = [t.strip() for t in out.strip().split(",")]
        return name, float(watts)
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e, None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--n", type=int, default=131072)
    ap.add_argument("--steps", type=int, default=13, help="timed steps per block")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--e2e-steps", type=int, default=8)
    ap.add_argument("--profile-steps", type=int, default=4)
    ap.add_argument("--model", type=int, default=0)
    ap.add_argument("--dir", default=None, help="where the temporary directory of the files is made (default: the system's temp dir)")
    a = ap.parse_args()

    import torch
    import aisgpu

    name, watts = card()
    B, N, fs = a.batch, a.n, 1536000
    soft, hard = resource.getrlimit(resource.RLIMIT_NOFILE)
    need = 2 * B + 256
    if soft < need:
        resource.setrlimit(resource.RLIMIT_NOFILE, (min(need, hard) if hard != resource.RLIM_INFINITY else need, hard))
    rows, n48 = 2 * B, N // 32
    bytes_step = rows * n48 * 8
    base = dict(card=name, power_limit_w=watts, batch=B, n=N, rate=fs, model=a.model, dump_bytes_per_step=bytes_step,
                dir=a.dir or tempfile.gettempdir())
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (torch.randn(B, N, 2, device="cuda", generator=g) * 0.05).contiguous()  # noise: the cost does not depend on the content
    work = tempfile.mkdtemp(prefix="aisgpu_dump_", dir=a.dir)
    try:
        def engine(dump, tag):
            e = aisgpu.Engine(model=a.model, sample_rate=fs, n_streams=B, max_chunk=N)
            if dump:
                d = os.path.join(work, tag)
                os.makedirs(d)
                e.dump_open([os.path.join(d, "s%d" % s) for s in range(B)])
            return e

        # ---- device-resident ----
        engs = {"off": engine(False, "dev_off"), "on": engine(True, "dev_on")}
        for e in engs.values():  # warm-up: module loading, the slots' first use
            for _ in range(4):
                e.submit_device(x.data_ptr(), N, N)
            e.sync()
        times = {"off": [], "on": []}
        for _ in range(a.reps):
            for k in ("off", "on"):
                e = engs[k]
                t0 = time.perf_counter()
                for _ in range(a.steps):
                    e.submit_device(x.data_ptr(), N, N)
                e.sync()
                times[k].append((time.perf_counter() - t0) * 1e3 / a.steps)
        for e in engs.values():
            e.close()
        med = {k: statistics.median(v) for k, v in times.items()}
        print(json.dumps(dict(base, what="device", ms_per_step_off=round(med["off"], 4), ms_per_step_on=round(med["on"], 4),
                              blocks_off=[round(t, 4) for t in times["off"]], blocks_on=[round(t, 4) for t in times["on"]],
                              dump_gb_per_s=round(bytes_step / (med["on"] * 1e-3) / 1e9, 3),
                              timed_dump_steps=a.reps * a.steps)), flush=True)
        shutil.rmtree(os.path.join(work, "dev_on"), ignore_errors=True)

        # ---- end to end: pinned host buffers, submit_async + poll_upto ----
        pin = [torch.empty(B, N, 2, dtype=torch.float32, pin_memory=True) for _ in range(2)]
        for p in pin:
            p.copy_(x.cpu())
        e2e = {}
        engs = {"off": engine(False, "e2e_off"), "on": engine(True, "e2e_on")}
        for k, e in engs.items():
            for c in range(2):
                e.submit_async_ptr(pin[c].data_ptr(), N)
            e.poll_count()
        res = {"off": [], "on": []}
        for _ in range(a.reps):
            for k in ("off", "on"):
                e = engs[k]
                t0 = time.perf_counter()
                prev = None
                for c in range(a.e2e_steps):
                    t = e.submit_async_ptr(pin[c & 1].data_ptr(), N)
                    if prev is not None:
                        e.poll_upto_count(prev)
                    prev = t
                e.poll_count()
                res[k].append((time.perf_counter() - t0) * 1e3 / a.e2e_steps)
        for e in engs.values():
            e.close()
        e2e = {k: statistics.median(v) for k, v in res.items()}
        print(json.dumps(dict(base, what="e2e", ms_per_step_off=round(e2e["off"], 3), ms_per_step_on=round(e2e["on"], 3),
                              blocks_off=[round(t, 3) for t in res["off"]], blocks_on=[round(t, 3) for t in res["on"]])), flush=True)
        shutil.rmtree(os.path.join(work, "e2e_on"), ignore_errors=True)

        # ---- profile: the export kernel and the slot copy ----
        e = engine(True, "prof")
        for _ in range(3):
            e.submit_device(x.data_ptr(), N, N)
        e.sync()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.profile_steps):
                e.submit_device(x.data_ptr(), N, N)
            e.sync()
            torch.cuda.synchronize()
        e.close()
        trace = os.path.join(work, "trace.json")
        prof.export_chrome_trace(trace)
        with open(trace) as f:
            ev = json.load(f)["traceEvents"]
        kern = [x_["dur"] for x_ in ev if x_.get("cat") == "kernel" and "k_c_fanout" in x_.get("name", "")]
        d2h = [x_["dur"] for x_ in ev if x_.get("cat") == "gpu_memcpy" and "DtoH" in x_.get("name", "") and
               x_.get("args", {}).get("bytes", 0) == bytes_step]
        kmed = statistics.median(kern) if kern else None
        cmed = statistics.median(d2h) if d2h else None
        print(json.dumps(dict(base, what="profile", export_launches=len(kern), export_us=kmed,
                              export_tb_per_s=round(2 * bytes_step / (kmed * 1e-6) / 1e12, 3) if kmed else None,
                              d2h_copies=len(d2h), d2h_us=cmed, d2h_gb_per_s=round(bytes_step / (cmed * 1e-6) / 1e9, 2) if cmed else None)),
              flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
