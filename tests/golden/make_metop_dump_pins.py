"""Writes tests/golden/metop_dump_pins.json from the reference's own MetOp dump decoder parts (oracle/_ref/libsatref_dump.so, built by
oracle/Makefile): for every stream of tests/metop_dump_cases.CASES the frame records and a digest of the written CADUs, and for the IQ
streams of tests/metop_dump_cases.CHAIN (reference demodulator + decoder) the number of CADUs and a digest of those after the lock. Run
from the repository root: python tests/golden/make_metop_dump_pins.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import dump as O  # noqa: E402
from tests.metop_dump_cases import CASES, CHAIN, PINS, after_lock, chain_reference, digest, stream  # noqa: E402


def main():
    assert O.available(), "build oracle/_ref/libsatref_dump.so first (make -C oracle ref)"
    out = {"cases": {}, "chain": {}}
    for name, case in CASES.items():
        soft, _, _ = stream(case)
        r = O.Dump().run(soft)
        out["cases"][name] = {"cadu": digest(r["cadu"]), "ncadu": int(r["cadu"].shape[0]), "recs": r["recs"].tolist()}
        print(name, r["cadu"].shape[0], flush=True)
    for name in CHAIN:
        cadu, clear = chain_reference(name)
        tail = after_lock(cadu, clear)
        out["chain"][name] = {"ncadu": int(cadu.shape[0]), "ntail": int(tail.shape[0]), "tail": digest(tail)}
        print(name, cadu.shape[0], tail.shape[0], flush=True)
    with open(PINS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
