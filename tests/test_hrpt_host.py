"""CPU: the host module layer's handling of noaa_hrpt_decoder and meteor_hrpt_decoder (satdump_b200/host/stream_modules.cpp), through the
b200_pipeline CLI: the decoder's parameters are read and checked before any device is touched, and valid ones reach the device check."""
import os
import subprocess

import pytest

from tests.common import ROOT

TOOL = os.path.join(ROOT, "satdump_b200", "host", "b200_pipeline")


def run(pipe, extra, tmp_path):
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    cmd = [TOOL, pipe, "baseband", str(inp), str(tmp_path / "out"), "--samplerate", "3e6", "--baseband_format", "cs16"] + extra
    return subprocess.run(cmd, capture_output=True, text=True, timeout=60)


@pytest.mark.parametrize("fused", [[], ["--fused"]])
@pytest.mark.parametrize("thr", ["61", "-1"])
def test_threshold_out_of_range_is_refused_by_name(built, tmp_path, fused, thr):
    r = run("noaa_hrpt", ["--deframer_thresold", thr] + fused, tmp_path)
    assert r.returncode == 1 and "deframer_thresold must be 0..60" in r.stderr, r.stderr


@pytest.mark.parametrize("pipe", ["noaa_hrpt", "meteor_hrpt"])
def test_valid_parameters_reach_the_device_check(built, tmp_path, pipe):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = run(pipe, [], tmp_path)
    assert r.returncode == 1 and "no cpu fallback" in r.stderr.lower() and "cuda" in r.stderr.lower(), r.stderr
