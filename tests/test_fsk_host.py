"""CPU: fsk_demod's parameters through the host module layer (b200_pipeline bluewalker3_*). They are validated before any device is
touched, so the messages can be checked without a GPU."""
import os
import subprocess

import pytest

from tests.common import ROOT

TOOL = os.path.join(ROOT, "satdump_b200", "host", "b200_pipeline")


def run(pipe, extra, tmp_path):
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    return subprocess.run([TOOL, pipe, "baseband", str(inp), str(tmp_path / "out"), "--baseband_format", "cs16"] + extra, capture_output=True,
                          text=True, timeout=60)


@pytest.mark.parametrize("pipe,extra,needle", [
    ("bluewalker3_narrow", ["--samplerate", "500000", "--basic_shaping", "true"], "basic_shaping"),
    ("bluewalker3_narrow", ["--samplerate", "500000", "--enable_doppler", "true"], "enable_doppler"),
    ("bluewalker3_wide", ["--samplerate", "400000"], "sampling rate is too low"),                    # module_demod_base.cpp:96-105
    ("bluewalker3_narrow", [], "Samplerate parameter must be present!"),                           # the pipeline names no samplerate
])
def test_unsupported_parameters_are_named(built, tmp_path, pipe, extra, needle):
    r = run(pipe, extra, tmp_path)
    assert r.returncode != 0 and needle in r.stderr, r.stderr


@pytest.mark.parametrize("mode", [[], ["--fused"]], ids=["two_stage", "fused"])
def test_valid_parameters_reach_the_library(built, tmp_path, mode):
    """With BlueWalker3.json's parameters the host layer accepts fsk_demod and hands it to the library (which then needs a device)."""
    r = run("bluewalker3_wide", ["--samplerate", "2000000"] + mode, tmp_path)
    assert "unknown demodulator" not in r.stderr and "not supported" not in r.stderr, r.stderr
