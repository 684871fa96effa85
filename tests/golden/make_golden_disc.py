#!/usr/bin/env python
"""Generates tests/golden/disc.json from the UNMODIFIED reference's FM-discriminator input model (-m 3, ModelDiscriminator):
oracle/_ref/libaisrefd.so (oracle/ref_harness_disc.cpp, built by oracle/disc.mk).  Run where /root/reference exists:
python tests/golden/make_golden_disc.py.  Same record format as mode_x.json (messages per chunk with level/ppm bit patterns, tap
counts and sha256); taps are named per channel ("C_0" is channel A's real row, "FR_1" channel B's Filter 37 output, "US" the
Upsample output)."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import disc_util as D  # noqa: E402
import oracle_disc as OD  # noqa: E402


def main():
    if not OD.have_refd():
        sys.exit("oracle/_ref/libaisrefd.so missing: run `make -C oracle ref && make -C oracle -f disc.mk refd` where the reference tree exists")
    out = {"generator": "tests/golden/make_golden_disc.py", "source": "oracle/_ref/libaisrefd.so (unmodified reference, strict IEEE flags, -m 3)",
           "cases": {}}
    for name, fs, N, nchunks, fmt, letters, seed in D.CASES:
        raw, per = D.stream_input(fs, N * nchunks, seed, fmt, name.startswith("type5"))
        r = D.record(*D.ref_run(fs, N, nchunks, fmt, letters, raw, per))
        r.update({"name": name, "fs": fs, "N": N, "nchunks": nchunks, "fmt": fmt, "letters": letters, "seed": seed, "input_sha256": D.sha(raw)})
        out["cases"][name] = r
        print(name, sum(len(c) for c in r["messages"]), "messages")
    with open(D.GOLDEN_DISC, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
