"""Writes tests/golden/fengyun_pins.json: the reference's result (oracle/_ref/libsatref_fengyun.so) on every case stream of
tests/fengyun_cases.py, for runs where the reference is absent. Run from the repository root: python tests/golden/make_fengyun_pins.py"""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import fengyun  # noqa: E402
from tests import fengyun_cases as X  # noqa: E402

assert fengyun.available(), "build oracle/_ref first (oracle/fengyun.mk)"
pins = {name: X.reference(name) for name in X.CASES + X.LARGE}
with open(X.PINS, "w") as f:
    json.dump(pins, f, indent=1, sort_keys=True)
    f.write("\n")
print(f"wrote {len(pins)} entries to {X.PINS}")
