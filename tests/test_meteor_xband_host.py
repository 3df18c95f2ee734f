"""CPU: the host module layer's refusals for meteor_xband_decoder name the option before any device is looked at: a missing or unknown
instrument_type, hard_symbols."""
import os
import subprocess

import pytest

from tests.common import ROOT


def _run(tmp_path, *extra):
    tool = os.path.join(ROOT, "satdump_b200", "host", "b200_pipeline")
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    return subprocess.run([tool, "meteor_mtvza", "baseband", str(inp), str(tmp_path / "out"), "--samplerate", "30720000", *extra],
                          capture_output=True, text=True, timeout=60)


@pytest.mark.parametrize("fused", [False, True])
def test_unknown_instrument_type(built, tmp_path, fused):
    r = _run(tmp_path, "--instrument_type", "kmss_qpsk", *(["--fused"] if fused else []))
    assert r.returncode == 1 and "Invalid METEOR instrument type!" in r.stderr


@pytest.mark.parametrize("fused", [False, True])
def test_hard_symbols(built, tmp_path, fused):
    r = _run(tmp_path, "--hard_symbols", "true", *(["--fused"] if fused else []))
    assert r.returncode == 1 and "hard_symbols" in r.stderr
