"""Writes tests/golden/hrpt_pins.json from the reference's own HRPT deframers (oracle/_ref/libsatref_hrpt.so, built by oracle/Makefile): for
every stream of tests/hrpt_cases.NOAA and METEOR the records, a digest of the output and the stats after every push, pushed whole and in
the ragged pieces of piece_cuts (stats as a digest there: one entry per piece), and the same for the large pushes of LARGE; for the IQ streams of CHAIN (reference pm_demod + deframer)
the output size and a digest of the frames after the lock. Run from the
repository root: python tests/golden/make_hrpt_pins.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import hrpt as O  # noqa: E402
from tests.hrpt_cases import (CHAIN, LARGE, METEOR, NOAA, PINS, after_lock, boundary_cuts, chain_reference, digest, frames_of,  # noqa: E402
                              large_stream, params, piece_cuts, stats_rows, stream)


def pin(soft, cuts, meteor, thr):
    r = O.run_pieces(soft, cuts, meteor, thr)
    rows = stats_rows(r["stats"])
    return {"out": digest(r["out"]), "units": int(r["out"].shape[0]), "recs": r["recs"].tolist(), "stats": rows if len(rows) <= 8 else digest(rows)}


def main():
    assert O.available(), "build oracle/_ref/libsatref_hrpt.so first (make -C oracle ref)"
    out = {"cases": {}, "pieces": {}, "large": {}, "chain": {}}
    for name in [*NOAA, *METEOR]:
        soft, cuts = stream(name)
        out["cases"][name] = pin(soft, cuts, *params(name))
        out["pieces"][name] = pin(soft, piece_cuts(soft.size, extra=boundary_cuts(name)), *params(name))
        print(name, out["cases"][name]["units"], flush=True)
    for name in LARGE:
        soft, cuts, meteor, thr = large_stream(name)
        out["large"][name] = pin(soft, cuts, meteor, thr)
        print(name, out["large"][name]["units"], flush=True)
    for name in CHAIN:
        o, clear, meteor = chain_reference(name)
        tail = after_lock(frames_of(o, meteor), clear)
        out["chain"][name] = {"units": int(o.shape[0]), "ntail": int(tail.shape[0]), "tail": digest(tail)}
        print(name, o.shape[0], tail.shape[0], flush=True)
    with open(PINS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
