"""Writes tests/golden/fengyun_mpt_pins.json: the reference's result (oracle/_ref/libsatref_fengyun_mpt.so) on every case stream of
tests/fengyun_mpt_cases.py, for runs where the reference is absent. Run from the repository root: python tests/golden/make_fengyun_mpt_pins.py"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import fengyun_mpt  # noqa: E402
from tests import fengyun_mpt_cases as X  # noqa: E402

assert fengyun_mpt.available(), "build oracle/_ref first (oracle/fengyun_mpt.mk)"
pins = {name: X.reference(name) for name in X.CASES + X.LARGE}
with open(X.PINS, "w") as f:
    json.dump(pins, f, indent=1, sort_keys=True)
    f.write("\n")
print(f"wrote {len(pins)} entries to {X.PINS}")
