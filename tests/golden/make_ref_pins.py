"""Regenerates tests/golden/ref_pins.json: digests of every reference array the CPU tests compare with (tests/refpin.py: the
C restatement in tests/test_oracle.py, the synthetic transmitter's encoders, the demultiplexer model, the frame stage models). Needs
oracle/_ref; the cases run as tests, so they also check what they compare.

    python tests/golden/make_ref_pins.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
TESTS = ["test_oracle.py", "test_synth.py", "test_demux_model.py", "test_rs_model.py"]


def main():
    import pytest
    from oracle import ref
    from tests import refpin
    assert ref.available(), "needs the compiled reference (oracle/_ref)"
    refpin.RECORD = True
    rc = pytest.main(["-q", "-p", "no:cacheprovider"] + [os.path.join(ROOT, "tests", t) for t in TESTS])
    assert rc == 0, "a test failed: nothing written"
    with open(refpin.PATH, "w") as f:
        json.dump({c: " ".join(d) for c, d in refpin.RECORDED.items()}, f, indent=0, sort_keys=True)
    print(sum(len(v) for v in refpin.RECORDED.values()), "digests of", len(refpin.RECORDED), "cases ->", refpin.PATH)


if __name__ == "__main__":
    main()
