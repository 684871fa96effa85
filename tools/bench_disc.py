#!/usr/bin/env python
"""bench_disc.py -- the FM-discriminator input workload (-m 3): `python tools/bench_disc.py --fmt cs16` prints ONE JSON line.

Batch 8192 stereo discriminator recordings at 48 kHz (tests/disc_util.stereo: channel A in I, channel B in Q; 32 unique
recordings, each stream its own added noise), 0.5 s per step (N = 24000), inputs resident in HBM, timed like bench.py's default
workload and tools/bench_x.py: exactly --steps submits between CUDA events on the engine's stream (median over --blocks).  Also reports
  e2e       : the same through aisgpu_submit_async / aisgpu_poll_upto with two pinned host buffers
  roofline  : the front-end kernel (k_frontend_disc) in algorithmic bytes -- input plus the two real 48 kHz Cbuf rows written per
              stream -- over its CUDA-event time, against the H100 SXM data sheet's 3.35 TB/s
  kernels   : mean device time per launch of the FIR37 kernel (k_fm_fir5) and the decoder (k_decode*), from a separate
              torch.profiler pass over --profile-steps submits (CUPTI kernel records), after the timed region
  parity    : sampled streams of the timed region re-run through the reference's ModelDiscriminator (oracle/_ref/libaisrefd.so)
              with the same chunking; NMEA sentences, their order and start/end counters must be identical
Writes nothing into the tree.  Single GPU.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, _p)
import bench as B_  # noqa: E402  (its helpers: one JSON line on stdout, median, frame polling)

FS = 48000
D_BATCH = 8192
D_UNIQUE = 32
D_RESIDENT = 4


def kernel_times(eng, x, R, N, steps):
    """Mean device ms per launch of the FIR37 and decoder kernels over `steps` submits (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    eng.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for j in range(steps):
            eng.submit_device(x[j % R].data_ptr(), N, N)
        eng.sync()
        torch.cuda.synchronize()
    acc = {}
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        k = "fir37" if "k_fm_fir5" in e.name else ("decoder" if "k_decode" in e.name else ("frontend" if "k_frontend_disc" in e.name else None))
        if k:
            t, n = acc.get(k, (0.0, 0))
            acc[k] = (t + e.device_time / 1e3, n + 1)  # device_time is in us
    return {k: {"ms_per_launch": t / n, "launches": n} for k, (t, n) in acc.items()}


def run_disc_workload(args):
    import numpy as np
    import torch
    import aisgpu
    import disc_util as D
    import oracle as O
    import oracle_disc as OD

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    B, N, R, U = args.batch, FS // 2, D_RESIDENT, D_UNIQUE
    fmt = {"cf32": O.FMT_CF32, "cs16": O.FMT_CS16}[args.fmt]
    bps = 8 if fmt == O.FMT_CF32 else 4
    uniq = np.stack([D.stream_input(FS, N * R, 1000 + u, fmt)[0] for u in range(U)])  # [U][N * R * per]
    if fmt == O.FMT_CF32:
        ud = torch.from_numpy(uniq.view(np.float32)).to(dev).view(U, R, N * 2)
        x = torch.empty((R, B, N * 2), dtype=torch.float32, device=dev)
    else:
        ud = torch.from_numpy(uniq).to(dev).view(U, R, N * 2)
        x = torch.empty((R, B, N * 2), dtype=torch.int16, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(4321)
    for b0 in range(0, B, U):
        nb = min(U, B - b0)
        x[:, b0:b0 + nb, :] = ud[:nb].permute(1, 0, 2)
    for r in range(R):  # each stream its own noise
        if fmt == O.FMT_CF32:
            x[r] += torch.empty((B, N * 2), device=dev).normal_(0.0, 0.005, generator=g)
        else:
            nz = torch.randint(-160, 161, (B, N * 2), device=dev, generator=g, dtype=torch.int32)
            x[r] = (x[r].to(torch.int32) + nz).clamp_(-32768, 32767).to(torch.int16)
    del ud
    torch.cuda.synchronize()
    # the frames of the whole timed region wait in the ring until the poll after it: room for 8 per stream and step (the stimulus has
    # at most 7 bursts per 0.5 s over both channels)
    eng = aisgpu.Engine(model=aisgpu.MODEL_DISCRIMINATOR, sample_rate=FS, fmt=fmt, n_streams=B, max_chunk=N,
                        max_frames=max(1 << 20, 8 * B * (args.steps + args.warmup)), host_staging=False)
    rng = np.random.default_rng(99)
    sample_streams = sorted(int(s) for s in rng.choice(B, size=min(args.parity_streams, B), replace=False))
    got = {s: [] for s in sample_streams}
    i = 0
    for _ in range(args.warmup):
        eng.submit_device(x[i % R].data_ptr(), N, N)
        i += 1
    eng.sync()
    B_.poll_streams(eng, set(sample_streams), got)
    est = torch.cuda.ExternalStream(eng.cuda_stream(), device=dev)
    sizes = [args.steps // args.blocks + (1 if b < args.steps % args.blocks else 0) for b in range(args.blocks)]
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(args.blocks + 1)]
    eng.join()
    evs[0].record(est)
    for b in range(args.blocks):
        for _ in range(sizes[b]):
            eng.submit_device(x[i % R].data_ptr(), N, N)
            i += 1
        eng.join()
        evs[b + 1].record(est)
    evs[-1].synchronize()
    blk_ms = [evs[b].elapsed_time(evs[b + 1]) / sizes[b] for b in range(args.blocks)]
    step_ms = B_.median(blk_ms)
    fe = eng.frontend_times(min(128, args.steps))
    launches = eng.last_launches()
    B_.poll_streams(eng, set(sample_streams), got)
    c1 = eng.counters()
    parity = None
    if not args.no_parity and OD.have_refd():
        idx = torch.tensor(sample_streams, device=dev)
        blocks = [x[r].index_select(0, idx).cpu().numpy() for r in range(R)]
        mism, nmsg, first = 0, 0, None
        for j, s in enumerate(sample_streams):
            m = OD.RefModelDisc(sample_rate=FS, fmt=fmt)
            for c in range(i):
                blk = blocks[c % R][j]
                m.push(blk.view(np.complex64) if fmt == O.FMT_CF32 else blk)
            want = [(q.key(), q.start_idx, q.end_idx) for q in m.messages()]
            m.close()
            nmsg += len(want)
            if want != got[s]:
                mism += 1
                first = first or {"stream": s, "got": len(got[s]), "want": len(want)}
        parity = {"streams_checked": len(sample_streams), "msgs_checked": nmsg, "mismatches": mism, "first_mismatch": first, "chunks": i,
                  "frames_dropped": int(c1[4]), "oracle": "libaisrefd.so (unmodified reference ModelDiscriminator, strict IEEE flags)"}
    kt = None
    if args.profile_steps > 0:
        try:
            kt = kernel_times(eng, x, R, N, args.profile_steps)
        except Exception as e:  # the profiler is optional: the timed numbers above do not depend on it
            kt = {"error": repr(e)}
    B_.poll_streams(eng, set(), {})
    host = [x[j].cpu().pin_memory() for j in range(2)]
    prev = eng.submit_async_ptr(host[0].data_ptr(), N)
    eng.poll_upto_count(prev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for j in range(args.e2e_steps):
        tk = eng.submit_async_ptr(host[j & 1].data_ptr(), N)
        eng.poll_upto_count(prev)
        prev = tk
    eng.poll_upto_count(prev)
    torch.cuda.synchronize()
    e2e_dt = time.perf_counter() - t0
    eng.close()
    del host
    fe_ms = sum(fe) / max(1, len(fe))
    algo_bytes = B * N * bps + B * 2 * N * 4  # input + the two real 48 kHz Cbuf rows written per stream
    B_.emit({"metric": "stereo MSamples/s through the FM-discriminator input (-m 3) demod chain", "value": B * N / (step_ms * 1e-3) / 1e6,
             "unit": "MSamples/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms,
             "higher_is_better": True, "scaling": "weak", "dtype": "f32", "data": "synthetic",
             "config": {"workload": "batch=%d synthetic %s stereo discriminator recordings @%d S/s, model 3, chunk %d samples/stream/launch" % (
                 B, args.fmt.upper(), FS, N), "model": 3, "format": args.fmt, "sample_rate": FS, "batch_per_gpu": B, "chunk_samples": N,
                 "resident_chunks": R, "bytes_per_step_per_gpu": B * N * bps, "device": torch.cuda.get_device_name(dev)},
             "spread": {"min_ms_per_step": min(blk_ms), "max_ms_per_step": max(blk_ms), "blocks": args.blocks},
             "parity": parity,
             "e2e": {"value": B * N * args.e2e_steps / e2e_dt / 1e6, "unit": "MSamples/s", "h2d_bytes_per_step": B * N * bps,
                     "steps": args.e2e_steps, "api": "aisgpu_submit_async + aisgpu_poll_upto, two caller-owned pinned buffers"},
             "gpu_launches": launches * args.steps, "launches_per_submit": launches,
             "frames": int(c1[0]),
             "kernels": kt,
             "roofline": {"bound": "hbm", "kernel": "k_frontend_disc", "frontend_ms_per_launch": fe_ms, "algorithmic_bytes": algo_bytes,
                          "achieved": algo_bytes / (fe_ms * 1e-3) / 1e9, "peak": 3350.0, "unit": "GB/s",
                          "frac": algo_bytes / (fe_ms * 1e-3) / 1e9 / 3350.0, "peak_source": "H100 SXM data sheet (700 W)",
                          "frontend_share_of_step": fe_ms / step_ms}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fmt", choices=("cf32", "cs16"), default="cs16")
    ap.add_argument("--batch", type=int, default=D_BATCH)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=1)
    ap.add_argument("--e2e-steps", type=int, default=12)
    ap.add_argument("--profile-steps", type=int, default=20)
    ap.add_argument("--parity-streams", type=int, default=32)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    args.blocks = max(1, min(args.blocks, args.steps))
    run_disc_workload(args)


if __name__ == "__main__":
    main()
