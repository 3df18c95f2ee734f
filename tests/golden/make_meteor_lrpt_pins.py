"""Writes tests/golden/meteor_lrpt_pins.json from the reference's own METEOR LRPT decoder parts (oracle/_ref/libsatref_meteor.so, built by
oracle/Makefile): for every stream of tests/meteor_lrpt_cases.CASES the frame records, the stats and a digest of the written CADUs, whole
and in the pieces of piece_cuts for PIECES; for M2X the CADU digest and stats; for the IQ streams of CHAIN (reference demodulator + decoder)
the number of CADUs and a digest of those after the lock. Run from the repository root: python tests/golden/make_meteor_lrpt_pins.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import meteor as O  # noqa: E402
from tests.meteor_lrpt_cases import (CASES, CHAIN, M2X, M2X_PARAMS, PIECES, PINS, after_lock, chain_reference, digest,  # noqa: E402
                                     piece_cuts, stream)


def case_pin(name, pieces=False):
    case = CASES[name]
    soft, _, cuts = stream(case)
    r = O.run_pieces(soft, piece_cuts(soft.size) if pieces else cuts, case.get("diff", False))
    return {"cadu": digest(r["cadu"]), "ncadu": int(r["cadu"].shape[0]), "recs": r["recs"].tolist(), "stats": r["stats"]}


def m2x_pin(name):
    case = M2X[name]
    soft, _, _ = stream(case)
    r = O.MeteorM2x(case.get("diff", False), M2X_PARAMS["viterbi_ber_thresold"], M2X_PARAMS["viterbi_outsync_after"]).run(soft)
    return {"cadu": digest(r["cadu"]), "ncadu": int(r["cadu"].shape[0]), "stats": r["stats"]}


def main():
    assert O.available(), "build oracle/_ref/libsatref_meteor.so first (make -C oracle ref)"
    out = {"cases": {}, "pieces": {}, "m2x": {}, "chain": {}}
    for name in CASES:
        out["cases"][name] = case_pin(name)
        print(name, out["cases"][name]["ncadu"], flush=True)
    for name in PIECES:
        out["pieces"][name] = case_pin(name, pieces=True)
    for name in M2X:
        out["m2x"][name] = m2x_pin(name)
        print(name, out["m2x"][name]["ncadu"], flush=True)
    for name in CHAIN:
        cadu, clear = chain_reference(name)
        tail = after_lock(cadu, clear)
        out["chain"][name] = {"ncadu": int(cadu.shape[0]), "ntail": int(tail.shape[0]), "tail": digest(tail)}
        print(name, cadu.shape[0], tail.shape[0], flush=True)
    with open(PINS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
