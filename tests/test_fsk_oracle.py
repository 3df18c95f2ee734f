"""CPU: the fsk_demod checker (oracle/fsk.py) and the parameter handling of satdump_b200.capi.fsk_demod_kwargs."""
import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests.common import reference


@pytest.fixture(scope="module")
def O():
    from oracle import fsk
    return reference(fsk)


def test_correctly_rounded_arm_is_within_one_ulp_of_glibc(O):
    rng = np.random.default_rng(5)
    y = (rng.standard_normal(20000) * 10.0 ** rng.uniform(-3, 3, 20000)).astype(np.float32)
    x = (rng.standard_normal(20000) * 10.0 ** rng.uniform(-3, 3, 20000)).astype(np.float32)
    O.atan2_mode(False)
    g = O.atan2f(y, x)
    O.atan2_mode(True)
    c = O.atan2f(y, x)
    assert np.array_equal(c, np.arctan2(y.astype(np.float64), x.astype(np.float64)).astype(np.float32))
    ulps = np.abs(g.view(np.int32).astype(np.int64) - c.view(np.int32).astype(np.int64))
    assert ulps.max() <= 1


@pytest.mark.parametrize("fs,rs,alpha,clock_alpha", [(500_000, 128_000, 0.35, None), (48_000, 9_600, 0.5, 0.8)])
def test_reference_chain_recovers_the_sent_bits(O, fs, rs, alpha, clock_alpha):
    """synth.fsk_signal's deviation sign: bit 1 = positive frequency = positive symbol, a few symbols of delay."""
    cfg = capi.DemodCfg(**{k: v for k, v in zip([f for f, _ in capi.DemodCfg._fields_], [0] * len(capi.DemodCfg._fields_))})
    kw = capi.fsk_demod_kwargs(fs, rs, alpha, clock_alpha=clock_alpha)
    cfg.samplerate, cfg.symbolrate, cfg.rrc_alpha, cfg.rrc_taps, cfg.agc_rate = fs, rs, alpha, 31, 1e-2
    cfg.clock_gain_omega, cfg.clock_gain_mu, cfg.clock_mu, cfg.clock_omega_limit = kw["clock_gain_omega"], kw["clock_gain_mu"], 0.5, 0.005
    x, bits = synth.fsk_signal(1 << 17, fs, rs, h=0.7, seed=1, carrier=fs * 0.004, snr_db=15)
    hd = (O.Fsk(cfg).run(x)["sym"] > 0).astype(np.uint8)
    k = slice(hd.size // 2, hd.size - 50)
    best = max(np.mean(hd[k] == bits[k.start - d:k.stop - d]) for d in range(0, 20))
    assert best == 1.0


def test_kwargs_follow_the_module():
    kw = capi.fsk_demod_kwargs(500_000, 128_000, 0.35)
    assert kw["clock_gain_omega"] == float(np.float32(pow(1.7e-2, 2) / 4.0)) and kw["clock_gain_mu"] == float(np.float32(1.7e-2))
    assert kw["clock_mu"] == 0.5 and kw["clock_omega_limit"] == 0.005 and kw["fsk_demod"] and kw["constellation"] == "bpsk"
    kw = capi.fsk_demod_kwargs(9_600 * 5, 9_600, 0.5, clock_alpha=0.8)
    assert kw["clock_gain_omega"] == float(np.float32(np.float32(0.8) ** 2 / np.float32(4.0))) and kw["clock_gain_mu"] == float(np.float32(0.8))
    kw = capi.fsk_demod_kwargs(9_600 * 5, 9_600, 0.5, clock_alpha=0.8, clock_gain_mu=0.1)  # explicit gains win (module_fsk_demod.cpp:37-44)
    assert kw["clock_gain_mu"] == float(np.float32(0.1))
    with pytest.raises(ValueError, match="RRC Alpha parameter must be present!"):
        capi.fsk_demod_kwargs(500_000, 128_000, None)


def test_reference_chain_recovers_the_sent_frames(O):
    """synth.fsk_frames through the reference's fsk_demod and ccsds_conv_concat_decoder with BlueWalker3.json's bluewalker3_narrow
    parameters (bpsk_90, 2648-bit CADUs, no RS, derandomised): every CADU written is a sent frame, and all but the first few are written."""
    from oracle import ref
    fs, rs = 500_000, 128_000
    cfg = capi.DemodCfg()
    kw = capi.fsk_demod_kwargs(fs, rs, 0.35)
    cfg.samplerate, cfg.symbolrate, cfg.rrc_alpha, cfg.rrc_taps, cfg.agc_rate = fs, rs, 0.35, 31, 1e-2
    cfg.clock_gain_omega, cfg.clock_gain_mu, cfg.clock_mu, cfg.clock_omega_limit = kw["clock_gain_omega"], kw["clock_gain_mu"], 0.5, 0.005
    bits, clear = synth.fsk_frames(60, 2648, seed=2)
    x, _ = synth.fsk_signal(1 << 20, fs, rs, h=0.7, seed=1, bits=bits, carrier=2000.0, snr_db=12)
    soft = O.Fsk(cfg).run(x)["soft"]
    got = ref.Fec(ref.ccsds_cfg("bpsk_90", 2648, 0.3, 20, 0)).run(soft)["cadu"].reshape(-1, 331)
    sent = {r.tobytes() for r in clear}
    assert got.shape[0] >= 45 and all(r.tobytes() in sent for r in got)
