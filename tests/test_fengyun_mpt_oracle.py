"""CPU: the fengyun_mpt_decoder checker (oracle/_ref, the reference's own blocks wired as the module) against its pins, the synthetic
FengYun-3 MPT transmitter decoded by it to the frames that were sent, the configuration's refusals, and b200_pipeline fengyun_mpt."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests import common
from tests import fengyun_mpt_cases as X

needs_ref = pytest.mark.skipif("not __import__('oracle.fengyun_mpt').fengyun_mpt.available()", reason="oracle/_ref not built (the pins stand in)")
TOOL = os.path.join(common.ROOT, "satdump_b200", "host", "b200_pipeline")


@needs_ref
@pytest.mark.parametrize("name", X.CASES + X.LARGE)
def test_pins(name):
    assert X.reference(name) == common.load_pins(X.PINS)[name]


def _sent_in_order(out, clear):
    return [int(np.nonzero((clear == o).all(1))[0][0]) for o in out if (clear == o).all(1).any()]


@needs_ref
@pytest.mark.parametrize("phase90", [False, True])
def test_transmitter(phase90):
    from oracle import fengyun_mpt
    i_bits, q_bits, clear = synth.fengyun_mpt_frames(40, seed=11)
    soft = synth.fengyun_mpt_soft(i_bits, q_bits, sigma=12.0, seed=5, phase90=phase90)
    # noise in front (zeros would lock both Viterbis at phase 0 until they lose it outsync_after reads later)
    noise = np.random.default_rng(9).integers(-127, 128, 2 * X.READ).astype(np.int8)
    soft = np.concatenate([noise, soft])
    soft = np.concatenate([soft, np.zeros((-soft.size) % X.READ, np.int8)])
    r = fengyun_mpt.RefMpt(X.OUTSYNC, X.BER).run(soft)
    # every sent frame in order from the third on (the Viterbis lock on the first read with signal, and the deframer needs a whole
    # frame to find the ASM), but the last (its tail runs into the zero padding) may be lost
    got = _sent_in_order(r["out"], clear)
    assert got[0] <= 2 and got == list(range(got[0], got[0] + len(got))) and got[-1] >= 38
    assert (r["recs"][-15:-1, 8] == 12).all() and (r["recs"][-15:-1, 2:4] == 4096).all()


@needs_ref
def test_shift_follows_viterbi1_only():
    """the module's shift test names viterbi1 twice: a buried Q branch drops viterbi2 to NOSYNC for many reads without a toggle, a
    buried I branch drops viterbi1 and toggles"""
    from oracle import fengyun_mpt
    q = fengyun_mpt.RefMpt(X.OUTSYNC, X.BER).run(X.stream("q_buried"))["recs"]
    i = fengyun_mpt.RefMpt(X.OUTSYNC, X.BER).run(X.stream("i_buried"))["recs"]
    assert (q[:, 5] == 0).sum() >= 10 + (q[:, 4] == 0).sum() and (np.diff(q[:, 0]) == 0).all()
    assert (i[:, 4] == 0).sum() >= 10 + (i[:, 5] == 0).sum() and (np.diff(i[:, 0]) != 0).any()


def test_transmitter_pairs_invert_the_split():
    """the transmitter's pair order against a restatement of the module's split and its two rotate_soft calls (shift 0)"""
    rng = np.random.default_rng(4)
    i_bits, q_bits = rng.integers(0, 2, 8192).astype(np.uint8), rng.integers(0, 2, 8192).astype(np.uint8)
    soft = synth.fengyun_mpt_soft(i_bits, q_bits)
    buf = soft.reshape(-1, 2)[:, ::-1].reshape(-1)           # rotate_soft(PHASE_0, true) on the read
    i_soft, q_soft = buf[0::2], ~buf[1::2]
    i2 = i_soft.reshape(-1, 2)[:, ::-1].reshape(-1)           # rotate_soft(PHASE_0, true) on each branch
    q2 = q_soft.reshape(-1, 2)[:, ::-1].reshape(-1)
    assert np.array_equal((i2 > 0).astype(np.uint8), i_bits) and np.array_equal((q2 > 0).astype(np.uint8), q_bits)


@pytest.mark.parametrize("missing", ["viterbi_outsync_after", "viterbi_ber_thresold"])
def test_missing_parameter(missing):
    """both are required, refused by name before a device is looked at"""
    kw = dict(viterbi_outsync_after=20, viterbi_ber_thresold=0.3)
    del kw[missing]
    with pytest.raises(ValueError, match=missing):
        capi.fengyun_mpt_cfg(**kw)


def test_invert_second_viterbi_refused(built):
    """the module has no invert_second_viterbi: a nonzero one is refused by name before the device is looked at (so this holds without
    a GPU)"""
    cfg = capi.fengyun_mpt_cfg(20, 0.3, max_soft=1 << 20)
    cfg.invert_second_viterbi = 1
    assert not capi.lib().b200_fec_create(ctypes.byref(cfg))
    assert "invert_second_viterbi" in capi.last_error() and "fengyun_mpt_decoder" in capi.last_error()


def _cli(tmp_path, *extra):
    inp = tmp_path / "in.cs16"
    inp.write_bytes(b"\0" * 4096)
    cmd = [TOOL, "fengyun_mpt", "baseband", str(inp), str(tmp_path / "out"), "--samplerate", "40e6", "--baseband_format", "cs16", *extra]
    return subprocess.run(cmd, capture_output=True, text=True, timeout=60)


def test_cli_lists_fengyun_mpt(built):
    r = subprocess.run([TOOL], capture_output=True, text=True, timeout=60)
    assert r.returncode != 0 and "|fengyun_mpt|" in r.stderr


@pytest.mark.parametrize("fused", [[], ["--fused"]])
def test_cli_valid_parameters_reach_the_device_check(built, tmp_path, fused):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = _cli(tmp_path, *fused)
    assert r.returncode == 1 and "no cpu fallback" in r.stderr.lower() and "cuda" in r.stderr.lower(), r.stderr
