#!/usr/bin/env python
"""bench_tunings.py -- four AIS channels from one wideband input: one engine with two tunings per input (aisgpu_set_tunings,
per_input = 2) against two engines with one tuning each.  `python tools/bench_tunings.py` prints ONE JSON line.

R = 512 recordings at 6.144 MS/s, N = 524288 samples per recording and submit, synthetic bursts at --density messages per second
per pair: the A/B pair at +2.6 MHz and the C/D pair at -2.6 MHz of the capture's centre (a few unique recordings reused, as
bench_tune.py does).  For CU8 and CF32 input and each --models chain, in one process, the two arrangements alternated round by round:
  (a) fan : one engine of 1024 streams, stream 2r tuned to +2.6 MHz and stream 2r + 1 to -2.6 MHz of input r;
  (b) pair: an engine of 512 streams tuned to +2.6 MHz and one tuned to -2.6 MHz, both fed the same 512 inputs.
Reported per arrangement:
  step_ms       : device-resident: aisgpu_submit_device of the inputs plus the polls that publish its frames, wall clock, median
                  and [min, max] over --blocks rounds;
  e2e_GSps      : input samples per second end to end from pinned host memory (aisgpu_submit_async, polling the previous ticket);
  h2d_bytes     : bytes copied host to device per step on that path;
  tune_kernel_ms: device time of every k_tune launch of one step (torch.profiler, CUDA activity, a run of its own), its bytes (input
                  once per launch + 8 B per tuned sample) and their share of the 3.35 TB/s of the H100 SXM data sheet;
  parity        : sampled streams of (a) against (b), and against a plain CF32 engine fed aisgpu_tune_restate of their input;
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

FS, N, UNIQUE, RESIDENT, WIDE = 6144000, 524288, 8, 2, 2600000
HBM_PEAK = 3.35e12  # bytes/s, H100 SXM data sheet
SAMPLED_INPUTS = (0, 1, 9, 255, 511)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:
        return "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", type=int, default=512)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--blocks", type=int, default=5)
    ap.add_argument("--density", type=float, default=50.0, help="messages per second per channel pair")
    ap.add_argument("--models", default="default", help="comma-separated: default (ModelDefault), standard (ModelStandard)")
    args = ap.parse_args()
    import numpy as np
    import torch
    import aisgpu
    import aissynth as S
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("bench_tunings.py needs a CUDA device: there is no CPU path to time")
    dev = torch.device("cuda", 0)
    R, RES = args.inputs, RESIDENT
    per_ch = max(1, int(round(args.density / 2)))
    t = np.arange(N * RES, dtype=np.float64)
    rot = {f: np.exp(2j * np.pi * f * t / FS) for f in (WIDE, -WIDE)}
    wide = np.stack([(0.5 * (S.random_stream(FS, N * RES, 9300 + u, bursts_per_sec=(per_ch, per_ch))[0] * rot[WIDE] +
                             S.random_stream(FS, N * RES, 9400 + u, bursts_per_sec=(per_ch, per_ch))[0] * rot[-WIDE])).astype(np.complex64)
                     for u in range(UNIQUE)])
    models = {"default": (aisgpu.MODEL_DEFAULT, "coherent"), "standard": (aisgpu.MODEL_STANDARD, "fm")}

    out = {"step": {}, "e2e": {}, "tune_kernel": {}, "parity": {}}
    for fmt, fname in ((aisgpu.FMT_CU8, "CU8"), (aisgpu.FMT_CF32, "CF32")):
        raw = wide if fmt == aisgpu.FMT_CF32 else np.stack([S.to_cu8(x) for x in wide])
        bps = 8 if fmt == aisgpu.FMT_CF32 else 2
        epp = 1 if fmt == aisgpu.FMT_CF32 else 2  # raw array elements per sample
        rb = N * bps  # bytes of one input row of one step
        ud = torch.from_numpy(np.ascontiguousarray(raw).view(np.uint8)).view(UNIQUE, RES, -1)
        host = torch.empty((RES, R, rb), dtype=torch.uint8, pin_memory=True)
        for r0 in range(0, R, UNIQUE):
            nr = min(UNIQUE, R - r0)
            host[:, r0:r0 + nr, :] = ud[:nr].permute(1, 0, 2)
        z = host.to(dev)
        torch.cuda.synchronize()
        for mname in args.models.split(","):
            model, chain = models[mname]
            kw = dict(model=model, sample_rate=FS, fmt=fmt, max_chunk=N, max_frames=1 << 20)
            fan = aisgpu.Engine(n_streams=2 * R, **kw)
            fan.set_tuning([WIDE, -WIDE] * R, per_input=2)
            pair = [aisgpu.Engine(n_streams=R, **kw) for _ in range(2)]
            pair[0].set_tuning([WIDE] * R)
            pair[1].set_tuning([-WIDE] * R)
            arr = {"fan": [fan], "pair": pair}
            cnt = {"fan": 0, "pair": 0}
            got = {"fan": {}, "pair": {}}

            def step(k, keep=False):
                """one device-resident step of arrangement k: submit, then the polls that publish its frames"""
                c = cnt[k]
                cnt[k] += 1
                for e in arr[k]:
                    e.submit_device(z[c % RES].data_ptr(), N, N)
                frames = 0
                for i, e in enumerate(arr[k]):
                    if keep:
                        for m in e.poll_upto(c):
                            s = m.stream if k == "fan" else 2 * m.stream + i  # the fan's stream numbering
                            if s // 2 in SAMPLED_INPUTS:
                                got[k].setdefault(s, []).append(m)
                    else:
                        frames += e.poll_upto_count(c)[0]
                return frames

            for _ in range(RES):  # the first RES steps: kept for the parity checks
                for k in arr:
                    step(k, keep=True)
            for k in arr:
                for _ in range(args.warmup):
                    step(k)
            blocks = max(1, min(args.blocks, args.steps))
            per = max(1, args.steps // blocks)
            ms = {k: [] for k in arr}
            frames = {k: 0 for k in arr}
            for _ in range(blocks):
                for k in arr:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(per):
                        frames[k] += step(k)
                    torch.cuda.synchronize()
                    ms[k].append((time.perf_counter() - t0) * 1e3 / per)
            key = "%s_%s" % (fname, chain)
            out["step"][key] = {k: {"step_ms": B_.median(ms[k]), "spread": [min(ms[k]), max(ms[k])],
                                    "frames_per_step": frames[k] / (blocks * per)} for k in arr}

            # end to end from pinned host memory: submit_async of step c, then the frames of step c - 1 (every engine's tickets are
            # its submit ordinals, which cnt counts)
            def e2e_step(k, first):
                c = cnt[k]
                cnt[k] += 1
                for e in arr[k]:
                    assert e.submit_async_ptr(host[c % RES].data_ptr(), N) == c
                if not first:
                    for e in arr[k]:
                        e.poll_upto_count(c - 1)

            e2e = {k: [] for k in arr}
            for k in arr:
                for i in range(args.warmup):
                    e2e_step(k, i == 0)
                for e in arr[k]:
                    e.poll_upto_count(-1)
            for _ in range(blocks):
                for k in arr:
                    t0 = time.perf_counter()
                    for i in range(per):
                        e2e_step(k, i == 0)
                    for e in arr[k]:
                        e.poll_upto_count(-1)
                    e2e[k].append(R * N * per / (time.perf_counter() - t0) / 1e9)
            out["e2e"][key] = {k: {"e2e_GSps": B_.median(e2e[k]), "spread": [min(e2e[k]), max(e2e[k])],
                                   "h2d_bytes": len(arr[k]) * R * rb} for k in arr}

            kern = {k: [] for k in arr}
            for _ in range(max(1, blocks // 2)):
                for k in arr:
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(4):
                            step(k)
                        torch.cuda.synchronize()
                    kern[k].append(sum(e.device_time_total for e in prof.key_averages() if "k_tune" in e.key) / 1e3 / 4)
            res = {}
            for k in arr:
                kms = B_.median(kern[k])
                nbytes = len(arr[k]) * R * rb + 2 * R * N * 8  # each launch reads the inputs once; every stream's row is written
                res[k] = {"tune_kernel_ms": kms, "spread": [min(kern[k]), max(kern[k])], "tune_bytes": nbytes,
                          "achieved_GBps": nbytes / (kms * 1e-3) / 1e9 if kms > 0 else None,
                          "share_of_hbm_peak": nbytes / (kms * 1e-3) / HBM_PEAK if kms > 0 else None}
            out["tune_kernel"][key] = res
            for e in [fan] + pair:
                e.close()

            # parity: (a) against (b), and both tunings of each sampled input against a plain CF32 engine on the restated input
            sampled = [2 * r + t_ for r in SAMPLED_INPUTS for t_ in (0, 1)]
            ref = aisgpu.Engine(model=model, sample_rate=FS, fmt=aisgpu.FMT_CF32, n_streams=len(sampled), max_chunk=N)
            want = {s: [] for s in sampled}
            for c in range(RES):
                rows = [aisgpu.tune_restate(fmt, FS, WIDE if s % 2 == 0 else -WIDE, c * N,
                                            raw[(s // 2) % UNIQUE][c * N * epp:(c + 1) * N * epp]) for s in sampled]
                ref.submit(np.ascontiguousarray(np.stack(rows)), N)
                for m in ref.poll():
                    want[sampled[m.stream]].append(m)
            ref.close()
            fk = lambda ms_: [(m.key(), m.start_idx, m.end_idx, m.level, m.ppm) for m in ms_]
            out["parity"][key] = {
                "sampled_streams": sampled,
                "fan_vs_pair_mismatches": sum(fk(got["fan"].get(s, [])) != fk(got["pair"].get(s, [])) for s in sampled),
                "fan_vs_restated_mismatches": sum(fk(got["fan"].get(s, [])) != fk(want[s]) for s in sampled),
                "frames_checked": sum(len(v) for v in want.values())}
        del z, host
        torch.cuda.empty_cache()
    first = sorted(out["e2e"])[0]
    e = out["e2e"][first]
    B_.emit({"metric": "end-to-end input rate, one engine with two tunings per input over two engines (%s)" % first,
             "value": e["fan"]["e2e_GSps"] / e["pair"]["e2e_GSps"], "unit": "ratio", "higher_is_better": True, "n_gpus": 1,
             "steps": args.steps,
             "config": {"workload": "%d inputs @%d S/s, chunk %d samples, A/B at +%d Hz and C/D at -%d Hz, %.0f msg/s per pair" %
                                    (R, FS, N, WIDE, WIDE, args.density),
                        "card": card(), "device": torch.cuda.get_device_name(dev)}, "results": out})


if __name__ == "__main__":
    main()
