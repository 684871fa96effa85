#!/usr/bin/env python
"""bench_dc16h.py -- the 12-byte input format DC16H beside CS16 and CF32: `python tools/bench_dc16h.py` prints ONE JSON line.

bench.py's default workload shape -- batch 1024 streams at 1536 kS/s, N = 131072 samples per stream and submit, ModelStandard,
inputs resident in HBM -- in three input formats: DC16H (12 B per sample, of which 4 are read), CS16 (4 B) and CF32 (8 B).  The three
engines live in one process and are timed in alternation: --steps submits per format between CUDA events on the engine's stream,
in --blocks rounds that visit every format in turn (median over the rounds, min / max as the spread).  Per format it reports
  step      : ms per submit and GS/s, device resident
  e2e       : the same through aisgpu_submit_async / aisgpu_poll_upto with two pinned host buffers (host-to-device bytes per step)
  frontend  : the streaming front-end kernel's CUDA-event time per launch and its algorithmic bytes (input + 0.5 B of 48 kHz
              output per input sample) over that time, against the H100 SXM data sheet's 3.35 TB/s
and for DC16H the parity of sampled streams of the timed region against the reference fed the same words (oracle/_ref), plus
the card's name and power limit read in the same run.  Needs a GPU (no fallback); writes nothing into the tree."""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, _p)
import bench as B_  # noqa: E402  (its helpers: one JSON line on stdout, median, frame polling)

FS, N, UNIQUE, RESIDENT = 1536000, 131072, 32, 2
OUT_BYTES_PER_SAMPLE = 0.5  # two channels x 8 B per 48 kHz sample, one per 32 input samples


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # the numbers stay, without what they were measured on
        return "unknown (%s)" % e


def reference_check(streams, held, n_chunks, got, model):
    """The sampled streams through the reference as Format::DC16H (oracle/_ref/libaisref_dc16h.so) with the engine's chunking, one
    thread per host CPU; message lists incl. order and start / end counters.  held[c % len(held)][j] = chunk c of streams[j]."""
    import threading
    import oracle as O
    import oracle_dc16h as OF
    if not OF.have_ref():
        raise SystemExit("bench_dc16h.py: oracle/_ref/libaisref_dc16h.so is not built (build() makes it where the reference sources lie)")
    refs = [OF.RefModelDC16H(model=model, sample_rate=FS, flags=O.DEFAULT_FLAGS) for _ in streams]

    def run(js):
        for j in js:
            for c in range(n_chunks):
                refs[j].push(held[c % len(held)][j])

    T = max(1, min(len(B_.host_cpus()), len(streams)))
    ths = [threading.Thread(target=run, args=(range(t, len(streams), T),)) for t in range(T)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    mism, nmsg, first = 0, 0, None
    for j, s in enumerate(streams):
        want = [(m.key(), m.start_idx, m.end_idx) for m in refs[j].messages()]
        nmsg += len(want)
        if want != got[s]:
            mism += 1
            first = first or {"stream": int(s), "got": len(got[s]), "want": len(want)}
    return {"streams_checked": len(streams), "msgs_checked": nmsg, "mismatches": mism, "first_mismatch": first,
            "oracle": "libaisref_dc16h.so (unmodified reference fed Format::DC16H, strict IEEE flags)"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--model", type=int, default=0)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--e2e-steps", type=int, default=12)
    ap.add_argument("--parity-streams", type=int, default=32)
    args = ap.parse_args()
    import numpy as np
    import torch
    import aisgpu
    if not torch.cuda.is_available():
        raise SystemExit("bench_dc16h.py needs a CUDA device: there is no CPU path to time")
    dev = torch.device("cuda", 0)
    B, R = args.batch, RESIDENT
    uniq = B_.make_unique_streams(UNIQUE, N * R, seed0=5000)
    ud = torch.view_as_complex(torch.from_numpy(uniq.view(np.float32)).to(dev).view(UNIQUE, N * R, 2))
    z = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
    g = torch.Generator(device=dev)
    g.manual_seed(1234)
    for b0 in range(0, B, UNIQUE):
        nb = min(UNIQUE, B - b0)
        z[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
    noise = torch.empty((B, N), dtype=torch.complex64, device=dev)
    for r in range(R):
        torch.view_as_real(noise).normal_(0.0, 0.005, generator=g)
        z[r] += noise
    del noise, ud
    zr = torch.view_as_real(z)  # [R][B][N][2]
    # CS16: z quantised; DC16H: the same I and Q (Q stored negated) in the low halves of words 0 and 1, seeded garbage in the
    # high halves and in word 2 (tests/dc16h_util.pack_iq)
    cs16 = torch.clamp(torch.round(zr * 32767.0), -32767, 32767).to(torch.int16)
    dc16h = torch.empty((R, B, N, 3), dtype=torch.int32, device=dev)
    for r in range(R):
        dc16h[r].random_(-(1 << 31), (1 << 31) - 1, generator=g)
    dc16h[..., 0] = (dc16h[..., 0] & -65536) | (cs16[..., 0].to(torch.int32) & 0xFFFF)
    dc16h[..., 1] = (dc16h[..., 1] & -65536) | ((-cs16[..., 1].to(torch.int32)) & 0xFFFF)
    torch.cuda.synchronize()
    inputs = {"DC16H": (aisgpu.FMT_DC16H, dc16h, 12), "CS16": (aisgpu.FMT_CS16, cs16, 4), "CF32": (aisgpu.FMT_CF32, z, 8)}
    total = args.steps + args.warmup
    engines = {k: aisgpu.Engine(model=args.model, sample_rate=FS, fmt=v[0], n_streams=B, max_chunk=N, host_staging=False,
                                max_frames=max(1 << 20, 4 * B * total)) for k, v in inputs.items()}
    rng = np.random.default_rng(99)
    sample_streams = sorted(int(s) for s in rng.choice(B, size=min(args.parity_streams, B), replace=False))
    got = {s: [] for s in sample_streams}
    count = {k: 0 for k in inputs}

    def submit(k):
        engines[k].submit_device(inputs[k][1][count[k] % R].data_ptr(), N, N)
        count[k] += 1

    for k in inputs:
        for _ in range(args.warmup):
            submit(k)
        engines[k].sync()
    blocks = max(1, min(args.blocks, args.steps))
    sizes = [args.steps // blocks + (1 if b < args.steps % blocks else 0) for b in range(blocks)]
    blk_ms = {k: [] for k in inputs}
    fe_ms = {k: [] for k in inputs}
    for b in range(blocks):  # every round visits the three formats in turn
        for k, eng in engines.items():
            est = torch.cuda.ExternalStream(eng.cuda_stream(), device=dev)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            eng.join()
            e0.record(est)
            for _ in range(sizes[b]):
                submit(k)
            eng.join()
            e1.record(est)
            e1.synchronize()
            blk_ms[k].append(e0.elapsed_time(e1) / sizes[b])
            fe_ms[k] += eng.frontend_times(min(128, sizes[b]))
            if k == "DC16H":
                B_.poll_streams(eng, set(sample_streams), got)
            else:
                eng.poll_count()
    # parity of the DC16H run: the sampled streams through the reference as Format::DC16H, same words, same chunking
    idx = torch.tensor(sample_streams, device=dev)
    held = [dc16h[r].index_select(0, idx).cpu().numpy().view(np.uint32).reshape(len(sample_streams), 3 * N) for r in range(R)]
    parity = reference_check(sample_streams, held, count["DC16H"], got, args.model)
    parity["chunks"] = count["DC16H"]
    parity["frames_dropped"] = int(engines["DC16H"].counters()[4])
    res = {}
    for k, (fmt, x, bps) in inputs.items():
        eng = engines[k]
        host = [x[j].cpu().contiguous().view(torch.uint8).pin_memory() for j in range(2)]
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
        dt = time.perf_counter() - t0
        del host
        step = B_.median(blk_ms[k])
        fe = sum(fe_ms[k]) / max(1, len(fe_ms[k]))
        algo = B * N * (bps + OUT_BYTES_PER_SAMPLE)
        res[k] = {"bytes_per_sample": bps, "ms_per_step": step, "gsamples_per_s": B * N / (step * 1e-3) / 1e9,
                  "min_ms_per_step": min(blk_ms[k]), "max_ms_per_step": max(blk_ms[k]),
                  "e2e_gsamples_per_s": B * N * args.e2e_steps / dt / 1e9, "e2e_h2d_bytes_per_step": B * N * bps,
                  "frontend_ms_per_launch": fe, "frontend_algorithmic_gb_per_s": algo / (fe * 1e-3) / 1e9,
                  "frontend_frac_of_3350_gb_per_s": algo / (fe * 1e-3) / 1e9 / 3350.0, "frontend_share_of_step": fe / step,
                  "launches_per_submit": eng.last_launches()}
        eng.close()
    B_.emit({"metric": "IQ GSamples/s through the AB demod chain from DC16H input (device resident)", "value": res["DC16H"]["gsamples_per_s"],
             "unit": "GSamples/s", "higher_is_better": True, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "blocks": blocks,
             "config": {"workload": "batch=%d synthetic streams @%d S/s, model %d, chunk %d samples/stream/launch; formats alternated per block" % (
                 B, FS, args.model, N), "card": card(), "device": torch.cuda.get_device_name(dev), "peak": "H100 SXM data sheet 3.35 TB/s (700 W), not measured"},
             "formats": res, "parity": parity})


if __name__ == "__main__":
    main()
