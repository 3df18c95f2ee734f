"""Writes tests/golden/turbo_pins.json from the reference's own turbo decoder (oracle/_ref/libsatref_turbo.so, built by oracle/Makefile):
for every stream of tests/turbo_cases.CASES the frame records and a digest of the written CADUs, the interleaver of each base and the
encoder output of each rate and base, and the CADUs of the IQ streams of tests/turbo_cases.CHAIN (reference demodulator + decoder); and
tests/golden/turbo_llr.npz: the a-priori arrays after the last iteration of the frames of tests/turbo_cases.LLR_CASES. Run from the repository root: python tests/golden/make_turbo_pins.py"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import turbo as O  # noqa: E402
from satdump_b200 import synth  # noqa: E402
from tests.turbo_cases import (CASES, CHAIN, LLR, LLR_CASES, PINS, RATE_NAME, chain_reference, digest, encoder_info, llr_frames,  # noqa: E402
                               reference_llr, stream)


def main():
    assert O.available(), "build oracle/_ref/libsatref_turbo.so first (make -C oracle ref)"
    out = {"perm": {}, "encode": {}, "cases": {}}
    for base in synth.TURBO_BASES:
        out["perm"][str(base)] = digest(O.perm(base).astype(np.int32))
        for rate in (2, 3, 4, 6):
            out["encode"][f"{rate}_{base}"] = digest(O.encode(RATE_NAME[rate], base, encoder_info(rate, base)).astype(np.uint8))
    for name, case in CASES.items():
        soft, _, _ = stream(case)
        r = O.Turbo(RATE_NAME[case["rate"]], case["base"], case["iters"]).run(soft)
        out["cases"][name] = {"cadu": digest(r["cadu"]), "ncadu": int(r["cadu"].shape[0]), "recs": r["recs"].tolist()}
        print(name, r["cadu"].shape[0], r["recs"].shape[0], flush=True)
    out["chain"] = {}
    for name in CHAIN:
        cadu = chain_reference(name)
        out["chain"][name] = {"tail": digest(cadu[2:]), "ncadu": int(cadu.shape[0])}
        print(name, cadu.shape[0], flush=True)
    with open(PINS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)
    llr = {}
    for name in LLR_CASES:
        case = CASES[name]
        for k, up, lo in llr_frames(name):
            llr[f"{name}_{k}_0"], llr[f"{name}_{k}_1"] = reference_llr(case["rate"], case["base"], case["iters"], up, lo)
    np.savez_compressed(LLR, **llr)


if __name__ == "__main__":
    main()
