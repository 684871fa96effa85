#!/usr/bin/env python
"""bench_group.py -- several models on one front end (engine groups, aisgpu_attach).  Prints ONE JSON line per workload.

  default    batch 1024 CF32 @1536 kS/s, 131072 samples per stream and step (bench.py's default shape), device-resident; the group
             {ModelDefault (leader), ModelStandard, V2} against the three standalone engines of the same configs
  lowdec     single-channel mode @48 kS/s, batch 8192, 0.5 s per step; the group {ModelStandard (leader), ModelDefault}.  Here the
             48 kHz rows are as large as the input, so a group saves little or nothing: the workload shows by how much.

Timing: host clock around whole blocks of --steps submits that end in a device synchronise (every engine's streams), so group and
standalone are timed the same way.  The blocks alternate in one process -- group, standalone 1, standalone 2, ... -- --reps times;
the medians are reported, with the spread.  A standalone engine's ms/step is its own block's; "standalone_sum" adds them.  GS/s
counts the input once per group step.

Parity in the same run: every frame of every member (all streams, every field of aisgpu_msg) against its standalone engine, which
received the same submits; and sampled streams of every member against the unmodified reference per model (oracle/_ref).
The card's name and power limit are read in the same run.  Writes nothing into the tree.
"""
import argparse
import ctypes
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, _p)
import bench as B_  # noqa: E402  (one JSON line on stdout, median)


def card():
    """(name, power limit in W) of GPU 0, read now."""
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"], text=True)
        name, watts = [t.strip() for t in out.strip().split(",")]
        return name, float(watts)
    except Exception as e:  # pragma: no cover
        return "unknown (%s)" % e, None


def drain(eng, sample, raw, kept):
    """Every frame of the engine's queue: the raw aisgpu_msg bytes into `raw`, aisgpu.Msg of the sampled streams into kept[s]."""
    import numpy as np
    import aisgpu
    batch = 8192
    buf = (aisgpu.MsgStruct * batch)()
    n = ctypes.c_int(0)
    size = ctypes.sizeof(aisgpu.MsgStruct)
    while True:
        eng._chk(eng.lib.aisgpu_poll(eng.h, buf, batch, ctypes.byref(n)))
        if n.value == 0:
            return
        b = bytes(memoryview(buf).cast("B")[:n.value * size])
        raw.append(b)
        streams = np.frombuffer(b, dtype=np.uint8).reshape(n.value, size)[:, :4].copy().view(np.int32)[:, 0]
        for i in np.nonzero(np.isin(streams, sample))[0]:
            m = aisgpu.Msg(buf[int(i)])
            kept[m.stream].append((m.key(), m.start_idx, m.end_idx))


def run(args, name, fs, B, N, R, mode, models, make_inputs, ref_factory):
    import numpy as np
    import torch
    import aisgpu

    dev = torch.device("cuda", 0)
    x = make_inputs(dev)  # [R][B][N] complex64, device-resident
    # the frames of a whole block wait in the ring until the drain after it: room for 8 per stream and step (the stimuli have fewer).
    # An overflowing ring drops frames in the order the decoders reach it, which is not deterministic, so parity needs none dropped.
    ring = max(1 << 20, 8 * B * max(args.steps, args.warmup))
    common = dict(sample_rate=fs, fmt=aisgpu.FMT_CF32, n_streams=B, max_chunk=N, host_staging=False, channel_mode=mode,
                  channels="XX" if mode == aisgpu.MODE_X else "AB", max_frames=ring)
    lead = aisgpu.Engine(model=models[0], **common)
    group = [lead] + [lead.attach(model=m, max_frames=ring) for m in models[1:]]
    alone = [aisgpu.Engine(model=m, **common) for m in models]
    rng = np.random.default_rng(7)
    sample = sorted(int(s) for s in rng.choice(B, size=min(args.parity_streams, B), replace=False))
    graw, araw = [[] for _ in models], [[] for _ in models]
    gkept = [{s: [] for s in sample} for _ in models]
    akept = [{s: [] for s in sample} for _ in models]
    steps = {"group": 0, **{j: 0 for j in range(len(models))}}

    def block(who, n_steps):
        engs = [lead] if who == "group" else [alone[who]]
        for _ in range(n_steps):
            i = steps[who]
            for e in engs:
                e.submit_device(x[i % R].data_ptr(), N, N)
            steps[who] = i + 1
        for e in (group if who == "group" else engs):
            e.sync()

    def drain_all():
        for j in range(len(models)):
            drain(group[j], sample, graw[j], gkept[j])
            drain(alone[j], sample, araw[j], akept[j])

    for who in ["group"] + list(range(len(models))):
        block(who, args.warmup)
    drain_all()
    times = {who: [] for who in steps}
    for _ in range(args.reps):
        for who in ["group"] + list(range(len(models))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            block(who, args.steps)
            times[who].append((time.perf_counter() - t0) * 1e3 / args.steps)
            drain_all()
    gms = B_.median(times["group"])
    sms = [B_.median(times[j]) for j in range(len(models))]
    # parity: member vs its standalone engine, every frame of every stream, byte for byte
    mism = [int(b"".join(graw[j]) != b"".join(araw[j])) for j in range(len(models))]
    nframes = [sum(len(b) for b in graw[j]) // ctypes.sizeof(aisgpu.MsgStruct) for j in range(len(models))]
    counters = [(group[j].counters(), alone[j].counters()) for j in range(len(models))]
    # parity: sampled streams of every member against the reference, same inputs, same chunking
    ref = None
    if not args.no_parity and ref_factory is not None:
        idx = torch.tensor(sample, device=dev)
        blocks = [x[r].index_select(0, idx).cpu().numpy() for r in range(R)]
        rm, nmsg, first = 0, 0, None
        for j, m in enumerate(models):
            for k, s in enumerate(sample):
                r = ref_factory(m)
                for c in range(steps["group"]):
                    r.push(blocks[c % R][k])
                want = [(q.key(), q.start_idx, q.end_idx) for q in r.messages()]
                r.close()
                nmsg += len(want)
                if want != gkept[j][s]:
                    rm += 1
                    first = first or {"model": m, "stream": s, "got": len(gkept[j][s]), "want": len(want)}
        ref = {"streams_checked": len(sample), "models": list(models), "msgs_checked": nmsg, "mismatches": rm, "first_mismatch": first,
               "chunks": steps["group"], "oracle": "unmodified reference (oracle/_ref), strict IEEE flags"}
    for e in group[::-1] + alone:
        e.close()
    del x
    torch.cuda.empty_cache()
    name_, watts = card()
    in_bytes = B * N * 8
    k48 = 2 * (N // 32) * 8 * B if mode == aisgpu.MODE_AB else N * 8 * B  # the 48 kHz rows of one step
    B_.emit({"metric": "engine group vs standalone engines (%s)" % name, "workload": name, "value": B * N / (gms * 1e-3) / 1e9,
             "unit": "GS/s (input counted once per group step)", "group_ms_per_step": gms, "standalone_ms_per_step": sms,
             "standalone_sum_ms_per_step": sum(sms), "speedup": sum(sms) / gms, "models": list(models),
             "config": {"batch": B, "sample_rate": fs, "chunk_samples": N, "format": "CF32", "channel_mode": "X" if mode == aisgpu.MODE_X else "AB",
                        "resident_chunks": R, "input_bytes_per_step": in_bytes, "rows48_bytes_per_step": k48},
             "spread": {w if w == "group" else "standalone_%d" % w: [min(v), max(v)] for w, v in times.items()},
             "steps_per_block": args.steps, "reps": args.reps, "warmup": args.warmup,
             "parity_vs_standalone": {"mismatches": sum(mism), "per_member": mism, "frames": nframes,
                                      "counters_equal": [a == b for a, b in counters],
                                      "frames_dropped": [int(a[4]) + int(b[4]) for a, b in counters]},
             "parity_vs_reference": ref, "device": name_, "power_limit_w": watts,
             "timing": "host clock around blocks of submits ending in a synchronise of every engine of the block"})


def default_inputs(B, N, R):
    def make(dev):
        import torch
        uniq = B_.make_unique_streams(8, N * R)
        ud = torch.from_numpy(uniq).to(dev)
        x = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
        g = torch.Generator(device=dev)
        g.manual_seed(1234)
        for b0 in range(0, B, 8):
            nb = min(8, B - b0)
            x[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
        noise = torch.empty((B, N), dtype=torch.complex64, device=dev)
        for r in range(R):
            torch.view_as_real(noise).normal_(0.0, 0.005, generator=g)
            x[r] += noise
        torch.cuda.synchronize()
        return x
    return make


def x_inputs(fs, B, N, R):
    def make(dev):
        import numpy as np
        import torch
        import mode_x_util
        U = 32
        uniq = np.stack([mode_x_util.x_stream(fs, N * R, u)[0] for u in range(U)])
        ud = torch.from_numpy(uniq).to(dev)
        x = torch.empty((R, B, N), dtype=torch.complex64, device=dev)
        g = torch.Generator(device=dev)
        g.manual_seed(4321)
        for b0 in range(0, B, U):
            nb = min(U, B - b0)
            x[:, b0:b0 + nb, :] = ud[:nb].view(nb, R, N).permute(1, 0, 2)
        noise = torch.empty((B, N), dtype=torch.complex64, device=dev)
        for r in range(R):
            torch.view_as_real(noise).normal_(0.0, 0.005, generator=g)
            x[r] += noise
        torch.cuda.synchronize()
        return x
    return make


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["default", "lowdec", "all"], default="all")
    ap.add_argument("--steps", type=int, default=40, help="submits per timed block")
    ap.add_argument("--reps", type=int, default=5, help="rounds of alternating blocks")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parity-streams", type=int, default=4)
    ap.add_argument("--no-parity", action="store_true")
    ap.add_argument("--batch", type=int, default=0, help="override the batch of the selected workloads (0: theirs)")
    args = ap.parse_args()
    import aisgpu
    import oracle as O
    import oracle_x as OX
    flags = O.FLAG_PS_EMA | O.FLAG_AFC_WIDE | O.FLAG_DROOP
    if args.workload in ("default", "all"):
        B, N, R = args.batch or B_.BATCH, B_.N_CHUNK, 4
        ref = (lambda m: O.RefModel(model=m, sample_rate=1536000, flags=flags)) if O.have_ref() else None
        run(args, "default", 1536000, B, N, R, aisgpu.MODE_AB, (aisgpu.MODEL_DEFAULT, aisgpu.MODEL_STANDARD, aisgpu.MODEL_V2),
            default_inputs(B, N, R), ref)
    if args.workload in ("lowdec", "all"):
        B, N, R = args.batch or 8192, 24000, 4
        ref = (lambda m: OX.RefModelX(model=m, sample_rate=48000, flags=flags)) if OX.have_refx() else None
        run(args, "lowdec", 48000, B, N, R, aisgpu.MODE_X, (aisgpu.MODEL_STANDARD, aisgpu.MODEL_DEFAULT), x_inputs(48000, B, N, R), ref)


if __name__ == "__main__":
    main()
