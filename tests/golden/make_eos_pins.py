"""Writes tests/golden/eos_pins.json from the reference's own Aqua DB decoder blocks (oracle/_ref/libsatref_eos.so, built by oracle/Makefile):
for every stream of tests/eos_cases.CASES the CADUs' digest and count, every frame's RS results and the stats after every push, pushed in
whole reads and in the ragged pieces of ragged_cuts (the stats of the last piece there); the same for the large push; and for the IQ
streams of CHAIN (reference psk_demod + decoder) and the Terra DB signal (reference terra_db_demod chain + ccsds_conv_concat_decoder) the
CADUs after the lock; and the M&M floor of the Terra configuration (tests/eos_cases.terra_floor) with the CRC of its signal. Run from the repository root: python tests/golden/make_eos_pins.py"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import eos as O  # noqa: E402
from tests.eos_cases import (CASES, CHAIN, PINS, after_lock, chain_reference, digest, large_stream, ragged_cuts, read_cuts,  # noqa: E402
                             stats_rows, stream, terra_chain_reference, terra_floor, terra_signal)


def pin(soft, cuts):
    r = O.run_pieces(soft, cuts)
    rows = stats_rows(r["stats"])
    return {"cadu": digest(r["cadu"]), "frames": int(r["cadu"].shape[0]), "rs": r["rs"].tolist(), "stats": rows if len(rows) <= 64 else rows[-1:]}


def main():
    assert O.available(), "build oracle/_ref/libsatref_eos.so first (make -C oracle ref)"
    out = {"cases": {}, "ragged": {}, "large": {}, "chain": {}}
    for name in CASES:
        soft, _ = stream(name)
        out["cases"][name] = pin(soft, read_cuts(soft.size))
        out["ragged"][name] = pin(soft, ragged_cuts(soft.size, CASES[name]["lead"]))
        print(name, out["cases"][name]["frames"], out["cases"][name]["stats"][-1], flush=True)
    soft, _ = large_stream()
    p = pin(soft, [])
    p["rs"] = digest(p["rs"])
    out["large"] = p
    print("large", soft.size, p["frames"], flush=True)
    for name in CHAIN:
        o, clear = chain_reference(name)
        tail = after_lock(o, clear)
        out["chain"][name] = {"frames": int(o.shape[0]), "ntail": int(tail.shape[0]), "tail": digest(tail)}
        print(name, o.shape[0], tail.shape[0], flush=True)
    o = terra_chain_reference()
    tail = after_lock(o, terra_signal()[1])
    out["terra_chain"] = {"frames": int(o.shape[0]), "ntail": int(tail.shape[0]), "tail": digest(tail)}
    print("terra", o.shape[0], tail.shape[0], flush=True)
    out["terra_floor"] = terra_floor()
    print("terra floor", out["terra_floor"], flush=True)
    with open(PINS, "w") as f:
        json.dump(out, f, indent=0, sort_keys=True)


if __name__ == "__main__":
    main()
