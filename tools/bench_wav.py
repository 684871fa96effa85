#!/usr/bin/env python
"""bench_wav.py -- aisgpu_feed_wav_files against aisgpu_feed_files on the same samples.  Prints ONE JSON line.

Workload: --batch CU8 recordings @1536 kS/s of --seconds each, ModelDefault, blocks of 131072 samples.  Every stream is written
twice into a temporary directory this script creates and deletes: as a raw file and as a WAV file with the same samples.  The two
feeders alternate, --reps times each, on one engine per run; the time is the host clock around the whole call (it ends when the
frames of the last block have been delivered).  The card's name and power limit are read in the same run.  Writes nothing into
the tree.
"""
import argparse
import json
import os
import shutil
import statistics
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "tests")):
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
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--n", type=int, default=131072)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--dir", default=None, help="where the temporary directory of the files is made (default: the system's temp dir)")
    a = ap.parse_args()

    import aisgpu
    import aissynth as S

    name, watts = card()
    B, N, fs = a.batch, a.n, 1536000
    n = int(fs * a.seconds)
    d = tempfile.mkdtemp(prefix="bench_wav_", dir=a.dir)
    try:
        raws, wavs = [], []
        for s in range(B):
            x = S.to_cu8(S.random_stream(fs, n, 900 + s)[0]).tobytes()
            r, w = os.path.join(d, "r%d.cu8" % s), os.path.join(d, "w%d.wav" % s)
            with open(r, "wb") as f:
                f.write(x)
            fmt = struct.pack("<HHIIHH", 1, 2, fs, fs * 2, 2, 8)
            with open(w, "wb") as f:
                f.write(b"RIFF" + struct.pack("<I", 4 + 24 + 8 + len(x)) + b"WAVE" + b"fmt " + struct.pack("<I", 16) + fmt +
                        b"data" + struct.pack("<I", len(x)) + x)
            raws.append(r)
            wavs.append(w)
        times = {"feed_files": [], "feed_wav_files": []}
        frames = {}
        for rep in range(a.reps + 1):  # the first round warms the page cache and the modules; it is not kept
            for feed, paths in (("feed_files", raws), ("feed_wav_files", wavs)):
                eng = aisgpu.Engine(model=aisgpu.MODEL_DEFAULT, sample_rate=fs, fmt=aisgpu.FMT_CU8, n_streams=B, max_chunk=N, max_frames=1 << 16)
                t0 = time.perf_counter()
                got, nb = getattr(eng, feed)(paths, N)
                dt = time.perf_counter() - t0
                eng.close()
                frames[feed] = sorted((m.stream, m.chunk, m.key(), m.start_idx) for m in got)
                if rep:
                    times[feed].append(dt)
        out = {"workload": "feed_wav_files vs feed_files, batch %d CU8 @1536 kS/s, %.2f s per stream, blocks of %d, ModelDefault" % (B, a.seconds, N),
               "gpu": name, "power_limit_w": watts, "blocks": nb, "frames": len(frames["feed_files"]),
               "same_frames": frames["feed_files"] == frames["feed_wav_files"]}
        for k, v in times.items():
            out[k + "_s"] = [round(t, 4) for t in v]
            out[k + "_median_s"] = round(statistics.median(v), 4)
            out[k + "_msamples_per_s"] = round(B * n / statistics.median(v) / 1e6, 1)
        print(json.dumps(out))
    finally:
        shutil.rmtree(d, ignore_errors=True)


if __name__ == "__main__":
    main()
