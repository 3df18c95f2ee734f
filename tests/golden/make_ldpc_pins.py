"""Writes tests/golden/ldpc_pins.json: digests of what the reference's own CCSDS LDPC code (oracle/_ref/libsatref_ldpc.so) computes on the
deterministic inputs of tests/test_ldpc_oracle.py, so that the C restatement (oracle/ldpc_port.c) is pinned where oracle/_ref is absent.
Touches no other fixture. Usage: python tests/golden/make_ldpc_pins.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from tests.test_ldpc_oracle import CASES, digest_decode, digest_matrix, digest_stream  # noqa: E402

if __name__ == "__main__":
    pins = {"matrix": digest_matrix("ref")}
    for name in CASES:
        pins[name] = digest_decode(name, "ref") if name.startswith("dec_") else digest_stream(name, "ref")
    with open(os.path.join(HERE, "ldpc_pins.json"), "w") as f:
        json.dump(pins, f, indent=1, sort_keys=True)
        f.write("\n")
