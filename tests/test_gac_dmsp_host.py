"""CPU: the host module layer's handling of noaa_gac_decoder and dmsp_rtd_decoder (satdump_b200/host/stream_modules.cpp), through the
b200_pipeline CLI: the parameters are read and checked before any device is touched, and valid ones reach the device check."""
import os
import subprocess

import pytest

from tests.common import ROOT

TOOL = os.path.join(ROOT, "satdump_b200", "host", "b200_pipeline")


def run(pipe, extra, tmp_path):
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    cmd = [TOOL, pipe, "baseband", str(inp), str(tmp_path / "out"), "--samplerate", "6e6", "--baseband_format", "cs16"] + extra
    return subprocess.run(cmd, capture_output=True, text=True, timeout=60)


def test_fused_chain_refuses_dmsp_timestamps_by_name(built, tmp_path):
    r = run("dmsp_rtd", ["--fused", "--start_timestamp", "1700000000"], tmp_path)
    assert r.returncode == 1 and "start_timestamp is not built in the fused chain" in r.stderr, r.stderr


@pytest.mark.parametrize("pipe", ["noaa_gac", "dmsp_rtd"])
@pytest.mark.parametrize("fused", [[], ["--fused"]])
def test_valid_parameters_reach_the_device_check(built, tmp_path, pipe, fused):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = run(pipe, fused, tmp_path)
    assert r.returncode == 1 and "no cpu fallback" in r.stderr.lower() and "cuda" in r.stderr.lower(), r.stderr
