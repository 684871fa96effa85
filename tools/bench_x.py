#!/usr/bin/env python
"""bench_x.py -- the single-channel (-c X) workload: `python tools/bench_x.py --rate R` prints ONE JSON line.

Batch 8192 synthetic CF32 streams already centred on one AIS channel (tests/mode_x_util.x_stream, each stream its own noise),
about 0.5 s of signal per step (N = rate / 2 rounded to the X granule, 64), inputs resident in HBM, timed like bench.py's
default workload: exactly --steps submits between CUDA events on the engine's stream (median over --blocks).  Also reports
  e2e       : the same through aisgpu_submit_async / aisgpu_poll_upto with two pinned host buffers
  roofline  : the front-end kernel (k_frontend_x) in algorithmic bytes -- input plus the 48 kHz Cbuf row written per stream --
              over its CUDA-event time, against the H100 SXM data sheet's 3.35 TB/s
  parity    : sampled streams of the timed region re-run through the reference in mode X (oracle/_ref/libaisrefx.so) with the
              same chunking; NMEA sentences, their order and start/end counters must be identical
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

X_BATCH = 8192
X_UNIQUE = 32
X_RESIDENT = 4


def run_x_workload(args, rank, world, local_rank):
    """Single-channel mode (AISGPU_MODE_X): batch of CF32 streams already centred on one AIS channel, ~0.5 s per step."""
    import numpy as np
    import torch
    import aisgpu
    import mode_x_util
    import oracle as O
    import oracle_x as OX

    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    fs = args.rate
    B = args.batch
    N = max(64, (fs // 2) // 64 * 64)  # about 0.5 s of signal, a multiple of the X granule (64)
    R, U = X_RESIDENT, X_UNIQUE
    K = {48000: 0, 96000: 1, 192000: 2}[next(b for b in (48000, 96000, 192000) if b >= fs)]
    uniq = np.stack([mode_x_util.x_stream(fs, N * R, 1000 * rank + u)[0] for u in range(U)])
    ud = torch.view_as_complex(torch.from_numpy(uniq.view(np.float32)).to(dev).view(U, N * R, 2))
    x = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(4321 + rank)
    for b0 in range(0, B, U):
        nb = min(U, B - b0)
        x[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
    noise = torch.empty((B, N), dtype=torch.complex64, device=dev)
    for r in range(R):
        torch.view_as_real(noise).normal_(0.0, 0.005, generator=g)
        x[r] += noise
    del noise, ud
    torch.cuda.synchronize()
    # the frames of the whole timed region wait in the ring until the poll after it: room for 6 per stream and step (the stimulus
    # has at most 5 bursts per 0.5 s)
    eng = aisgpu.Engine(model=args.model, sample_rate=fs, n_streams=B, max_chunk=N, device=local_rank,
                        max_frames=max(1 << 20, 6 * B * (args.steps + args.warmup)), host_staging=False, channel_mode=aisgpu.MODE_X, channels="XX")
    rng = np.random.default_rng(99 + rank)
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
    # parity: the sampled streams through the reference in mode X, same inputs, same chunking
    parity = None
    if not args.no_parity and OX.have_refx():
        flags = O.FLAG_PS_EMA | O.FLAG_AFC_WIDE | O.FLAG_DROOP
        idx = torch.tensor(sample_streams, device=dev)
        blocks = [x[r].index_select(0, idx).cpu().numpy() for r in range(R)]
        mism, nmsg, first = 0, 0, None
        for j, s in enumerate(sample_streams):
            m = OX.RefModelX(model=args.model, sample_rate=fs, flags=flags)
            for c in range(i):
                m.push(blocks[c % R][j])
            want = [(q.key(), q.start_idx, q.end_idx) for q in m.messages()]
            m.close()
            nmsg += len(want)
            if want != got[s]:
                mism += 1
                first = first or {"stream": s, "got": len(got[s]), "want": len(want)}
        parity = {"streams_checked": len(sample_streams), "msgs_checked": nmsg, "mismatches": mism, "first_mismatch": first, "chunks": i,
                  "frames_dropped": int(c1[4]), "oracle": "libaisrefx.so (unmodified reference, strict IEEE flags, mode X)"}
    # end to end: pinned host buffers through aisgpu_submit_async / aisgpu_poll_upto
    host = [torch.view_as_real(x[j]).cpu().pin_memory() for j in range(2)]
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
    algo_bytes = B * N * 8 + B * (N >> K) * 8  # CF32 input + the 48 kHz Cbuf row written per stream
    if rank == 0:
        name = torch.cuda.get_device_name(dev)
        B_.emit({"metric": "IQ MSamples/s through the single-channel (-c X) demod chain", "value": world * B * N / (step_ms * 1e-3) / 1e6,
              "unit": "MSamples/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms,
              "higher_is_better": True, "scaling": "weak", "dtype": "f32", "data": "synthetic",
              "config": {"workload": "batch=%d synthetic CF32 single-channel IQ streams @%d S/s, model %d, chunk %d samples/stream/launch (X mode)" % (
                  B, fs, args.model, N), "channel_mode": "X", "model": args.model, "sample_rate": fs, "batch_per_gpu": B, "chunk_samples": N,
                  "resident_chunks": R, "bytes_per_step_per_gpu": B * N * 8, "device": name},
              "spread": {"min_ms_per_step": min(blk_ms), "max_ms_per_step": max(blk_ms), "blocks": args.blocks},
              "parity": parity,
              "e2e": {"value": world * B * N * args.e2e_steps / e2e_dt / 1e6, "unit": "MSamples/s", "h2d_bytes_per_step": B * N * 8,
                      "steps": args.e2e_steps, "api": "aisgpu_submit_async + aisgpu_poll_upto, two caller-owned pinned buffers"},
              "gpu_launches": launches * args.steps, "launches_per_submit": launches,
              "frames": int(c1[0]),
              "roofline": {"bound": "hbm", "kernel": "k_frontend_x", "frontend_ms_per_launch": fe_ms, "algorithmic_bytes": algo_bytes,
                           "achieved": algo_bytes / (fe_ms * 1e-3) / 1e9, "peak": 3350.0, "unit": "GB/s",
                           "frac": algo_bytes / (fe_ms * 1e-3) / 1e9 / 3350.0, "peak_source": "H100 SXM data sheet (700 W)",
                           "frontend_share_of_step": fe_ms / step_ms}})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rate", type=int, default=48000, help="sample rate, 12000..192000")
    ap.add_argument("--model", type=int, default=0, help="0 ModelStandard, 1 ModelBase, 2 ModelDefault, 4 ModelChallenger, 11 V2")
    ap.add_argument("--batch", type=int, default=X_BATCH)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=1)
    ap.add_argument("--e2e-steps", type=int, default=12)
    ap.add_argument("--parity-streams", type=int, default=32)
    ap.add_argument("--no-parity", action="store_true")
    args = ap.parse_args()
    args.blocks = max(1, min(args.blocks, args.steps))
    run_x_workload(args, 0, 1, 0)


if __name__ == "__main__":
    main()
