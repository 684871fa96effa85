#!/usr/bin/env python
"""Generates tests/golden/mode_x.json from the UNMODIFIED reference in single-channel mode (-c X): oracle/_ref/libaisrefx.so
(oracle/ref_harness_x.cpp, built by oracle/mode_x.mk).  Run where /root/reference exists:  python tests/golden/make_golden_x.py
Same record format as golden.json (messages per chunk with level/ppm bit patterns, tap counts and sha256).  The plain-C port has
no X mode, so these cases live apart from golden.json."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (os.path.join(ROOT, "ais-catcher_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import mode_x_util as X  # noqa: E402
import oracle_x as OX  # noqa: E402


def main():
    if not OX.have_refx():
        sys.exit("oracle/_ref/libaisrefx.so missing: run `make -C oracle ref && make -C oracle -f mode_x.mk refx` where the reference tree exists")
    out = {"generator": "tests/golden/make_golden_x.py", "source": "oracle/_ref/libaisrefx.so (unmodified reference, strict IEEE flags, mode X)",
           "cases": {}}
    for name, model, fs, N, nchunks, fmt, flags, seed in X.CASES:
        raw, per = X.stream_input(fs, N * nchunks, seed, fmt)
        r = X.record(*X.ref_run(model, fs, N, nchunks, fmt, flags, raw, per))
        r.update({"model": model, "fs": fs, "N": N, "nchunks": nchunks, "fmt": fmt, "flags": flags, "seed": seed, "input_sha256": X.sha(raw)})
        out["cases"][name] = r
        print(name, sum(len(c) for c in r["messages"]), "messages")
    with open(X.GOLDEN_X, "w") as f:
        json.dump(out, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
