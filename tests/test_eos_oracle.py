"""CPU: the checker of aqua_db_decoder and the host layer's handling of it. The compiled reference blocks (oracle/_ref/libsatref_eos.so)
equal their committed pins on every test stream, the synthesised streams decode to the frames sent, the RS results of the cases are the
ones they were built for, b200_pipeline aqua_db | aura_db | terra_db reads EOS.json's parameters and reaches the device check, the Terra DB signal decodes through
the reference's terra_db_demod chain, the Terra mapping's omega and RRC taps are the reference's, and a working rate below 1.1 samples per
half-symbol is refused by name."""
import os
import subprocess

import numpy as np
import pytest

from oracle import eos as O
from tests.common import reference
from tests.eos_cases import CASES, after_lock, digest, pins, ragged_cuts, read_cuts, stats_rows, stream


def _same(r, pin):
    assert digest(r["cadu"]) == pin["cadu"] and r["cadu"].shape[0] == pin["frames"] and r["rs"].tolist() == pin["rs"]
    rows = stats_rows(r["stats"])
    assert (rows if len(rows) <= 64 else rows[-1:]) == pin["stats"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_reference_equals_pins(name):
    reference(O)
    soft, _ = stream(name)
    _same(O.run_pieces(soft, read_cuts(soft.size)), pins()["cases"][name])
    _same(O.run_pieces(soft, ragged_cuts(soft.size, CASES[name]["lead"])), pins()["ragged"][name])


def test_synthesised_streams_come_out_as_sent():
    """The decoded stream's rails NRZ-M encoded on Q (A) and I (B): the reference writes the sent CADUs; on swapped rails it never syncs"""
    reference(O)
    from satdump_b200 import synth
    bits, sent = synth.aqua_db_frames(16, seed=3)
    soft = synth.aqua_db_soft(bits, sigma=10.0, seed=4)
    soft = np.concatenate([soft, np.zeros((-soft.size) % 65536, np.int8)])
    assert np.array_equal(O.Aqua().run(soft)["cadu"], sent)
    assert O.Aqua().run(synth.aqua_db_soft(np.concatenate([bits.reshape(-1)] * 8), swap_iq=True))["cadu"].shape[0] == 0


def test_iq_signal_decodes_through_the_reference_chain():
    """psk_demod OQPSK at 15 MS/s (EOS.json's parameters) -> the module loop: after the lock every CADU is a sent one"""
    reference(O)
    from tests.eos_cases import chain_reference
    o, clear = chain_reference("cs16")
    tail = after_lock(o, clear)
    assert tail.shape[0] >= 200 and all(any(np.array_equal(row[:896], c[:896]) for c in clear) for row in tail)  # (RS corrects the data only)


TOOL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "satdump_b200", "host", "b200_pipeline")


def _cli(pipe, tmp_path, extra):
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    rate = "45e6" if pipe == "terra_db" else "15e6"
    cmd = [TOOL, pipe, "baseband", str(inp), str(tmp_path / "out"), "--samplerate", rate, "--baseband_format", "cs16"] + extra
    return subprocess.run(cmd, capture_output=True, text=True, timeout=60)


@pytest.mark.parametrize("pipe", ["aqua_db", "aura_db", "terra_db"])
@pytest.mark.parametrize("fused", [[], ["--fused"]])
def test_valid_parameters_reach_the_device_check(built, tmp_path, pipe, fused):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = _cli(pipe, tmp_path, fused)
    assert r.returncode == 1 and "no cpu fallback" in r.stderr.lower() and "cuda" in r.stderr.lower(), r.stderr


@pytest.mark.parametrize("fused", [[], ["--fused"]])
def test_terra_refuses_too_few_samples_per_half_symbol(built, tmp_path, fused):
    """26 MS/s is inside [1.1, 4.0] samples per symbol (no resampler) but 0.99 per half-symbol: refused by name before any device"""
    r = _cli("terra_db", tmp_path, ["--samplerate", "26000000"] + fused)
    assert r.returncode == 1 and "terra_db_demod: samplerate 26000000" in r.stderr and "samples per half-symbol" in r.stderr, r.stderr
    from satdump_b200 import capi
    with pytest.raises(ValueError, match="terra_db_demod: samplerate 26000000"):
        capi.terra_db_demod_kwargs(26e6, 13125000)


def test_terra_omega_and_taps_equal_the_reference():
    """The mapping runs psk_demod's BPSK chain at 2 x symbolrate. Its M&M omega fs / (2 rs) in float is bitwise TerraDBDemodModule's
    ((float)fs / (float)rs) / 2 at every rate of the window (halving is exact), and its RRC is firdes' RRC at the same arguments."""
    reference(O)
    from oracle import ref as R
    from satdump_b200 import capi
    for fs in (15e6, 26.5e6, 30e6, 45e6, 52.5e6):
        rs = 13125000
        ours = np.float32(fs) / np.float32(2 * rs)
        theirs = (np.float32(fs) / np.float32(rs)) / np.float32(2)
        assert ours.view(np.uint32) == theirs.view(np.uint32)
    kw = capi.terra_db_demod_kwargs(45e6, 13125000)
    assert kw["symbolrate"] == 26250000 and kw["final_samplerate"] == 0.0 and kw["clock_omega_limit"] == 1e-4
    assert np.array_equal(R.rrc_design(1, np.float32(45e6), 26250000, 0.5, 31), R.rrc_design(1, np.float32(45e6), 2 * 13125000, 0.5, 31))


def test_terra_signal_decodes_through_the_reference_chain():
    reference(O)
    from tests.eos_cases import terra_chain_reference, terra_signal
    o = terra_chain_reference()
    clear = terra_signal()[1]
    tail = after_lock(o, clear)
    assert tail.shape[0] >= 60 and all(any(np.array_equal(row[:896], c[:896]) for c in clear) for row in tail)
    assert digest(tail) == pins()["terra_chain"]["tail"]
