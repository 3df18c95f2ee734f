"""Writes tests/golden/gac_pins.json: the reference's results on every case stream of tests/gac_cases.py (oracle/_ref/libsatref_gac.so
must be built: python -c "import __graft_entry__ as g; g.build()"), and a digest of the reference's GAC PN table."""
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from oracle import gac as O  # noqa: E402
from tests import gac_cases as G  # noqa: E402


def main():
    assert O.available(), "oracle/_ref/libsatref_gac.so is not built"
    out = dict(pn_table=G.digest(O.pn_table()), cases={name: G.ref_result(name) for name in G.CASES})
    with open(G.PINS, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
