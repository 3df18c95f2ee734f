"""CPU: the decomposition behind the device Viterbi decoder (tests/viterbi_model.py) pinned against the oracle, and the streams that make
its correction paths run. The model decodes the way the device does (speculated start states, block chainback with an edge check, redo
rounds, adaptive windows); its bits and per-chunk BERs must equal the reference's, and each stream builder must make the paths it is meant
for run at the default windows: tests/test_gpu_viterbi_paths.py feeds the same streams to the device and asserts its counters."""
import numpy as np
import pytest

from tests import viterbi_model as M
from tests.common import oracle


def _cfgs(O, kind):
    if kind == "metop":
        return M.Geom("metop"), O.metop_cfg(0.28, 10), {}
    if kind == "bpsk":
        return M.Geom("ccsds", 8192, "bpsk"), O.ccsds_cfg("bpsk", 8192, 0.3, 20, 4), {}
    # jpss-shaped: OQPSK (IQ-swap hypotheses), NRZ-M, 10232-bit CADUs: F = 5116 decoded bits per chunk, not a multiple of 32
    return (M.Geom("ccsds", 10232, "oqpsk", nrzm=True), O.ccsds_cfg("oqpsk", 10232, 0.3, 20, 5, nrzm=True, rs_usecheck=True),
            dict(cadu_size=10232, interleave=5))


def _pin(O, geom, ocfg, soft):
    want = O.Fec(ocfg).run(soft)
    d = M.Decoder(geom, ocfg.ber_thresold, ocfg.outsync_after)
    got = d.run(soft)
    assert np.array_equal(got["bits"], want["bits"])
    assert np.array_equal(got["vit_state"], want["vit_state"])
    # (the BER reported while IDLE is the reference's lock test on its first chunk, which reads never-written scratch bytes)
    sy = want["vit_state"] == 1
    assert sy.any() and np.array_equal(got["vit_ber"][sy], want["vit_ber"][sy])
    return d, want


def test_acs_matches_reference_decoder():
    """The ACS alone, unbiased start, against the reference's CCDecoder on random symbols (wrap-around, ties, flush steps)."""
    O = oracle()
    rng = np.random.default_rng(2)
    F = 1024
    syms = rng.integers(0, 256, 2 * (F + 6) * 3, dtype=np.uint8)
    want = O.cc_decode(syms, F, 3)
    start, got = [-1], []
    for c in range(3):
        X, dec = M.acs(syms[c * 2 * F:c * 2 * F + 2 * (F + 6)].reshape(1, F + 6, 2), M.init_metrics(start))
        bits, nxt, _ = M.serial_chainback(dec, X, F)
        got.append(bits[0])
        start = [int(nxt[0])]
    assert np.array_equal(np.concatenate(got), want)


@pytest.mark.parametrize("kind", ["metop", "bpsk", "jpss"])
def test_model_equals_oracle_on_weak_stretch(kind):
    """Six WEAK chunks inside a good stream: the model's bits, lock states and BERs equal the oracle's, and at the default windows the
    device would mis-speculate start states (more than one redo round), chain blocks back serially, and still end consistent."""
    O = oracle()
    geom, ocfg, kw = _cfgs(O, kind)
    soft, _ = M.weak_stretch(geom, 16, set(range(5, 11)), 7, **kw)
    d, want = _pin(O, geom, ocfg, soft)
    k = d.counters
    assert (want["vit_state"] == 1).all() and want["nframes"] > 0
    assert k["misses"][0] > 0 and k["start_redone"] > k["misses"][0] and max(k["rounds"]) >= 2, k
    assert k["tb_first"][0] > 0 and k["tb_serial"] > 0, k


def test_model_equals_oracle_on_metric_wraparound():
    """The clean +-100 stream wraps the reference's uint8 path metrics (BER ~0.25): the model wraps the same way."""
    from satdump_b200 import synth
    O = oracle()
    rng = np.random.default_rng(8)
    bits = rng.integers(0, 2, 4096 * 10, dtype=np.uint8)
    soft = np.where(synth.conv_encode(bits) > 0, 100, -100).astype(np.int8)[:8192 * 8]
    geom = M.Geom("ccsds", 8192, "qpsk")
    ocfg = O.ccsds_cfg("qpsk", 8192, 0.3, 20, 0)
    want = O.Fec(ocfg).run(soft)
    got = M.Decoder(geom, 0.3, 20).run(soft)
    assert want["bits"].size > 0 and np.array_equal(got["bits"], want["bits"])


def test_model_equals_oracle_noise_lock_unlock():
    """Noise (IDLE, lock search with the chained test decoder), signal (lock), a long weak stretch (unlock after outsync_after + 1 bad
    chunks), signal again (lock from the carried start state)."""
    O = oracle()
    geom, ocfg, _ = _cfgs(O, "bpsk")
    coded = M.coded_stream(geom, 40, 11)
    prof = [(3, 40)] * 3 + [M.GOOD] * 8 + [M.WEAK] * 24 + [M.GOOD] * 5
    soft = M.soft_stream(geom, coded, prof, 11)
    d, want = _pin(O, geom, ocfg, soft)
    vs = want["vit_state"]
    assert vs[0] == 0 and vs[5] == 1 and (vs[11:35] == 0).any() and vs[-1] == 1


def test_adaptive_window_rule():
    w, c = 512, 0
    w, c = M.adapt_window(w, c, 0.03, 512, 4096)
    assert (w, c) == (1024, 0)
    for i in range(31):
        w, c = M.adapt_window(w, c, 0.0, 512, 4096)
    assert (w, c) == (1024, 31)
    w, c = M.adapt_window(w, c, 0.01, 512, 4096)  # neither clean nor bad: the count holds
    assert (w, c) == (1024, 31)
    w, c = M.adapt_window(w, c, 0.0, 512, 4096)
    assert (w, c) == (512, 0)
    for i in range(5):
        w, c = M.adapt_window(w, c, 0.5, 512, 4096)
    assert w == 4096


def test_launch_of_65_chunks_grows_both_windows():
    """The stream of the GPU window test: 65 chunks of which 16 are WEAK make more than 2 % of the launch miss its start state and more
    than 2 % disagree at a block edge, so both windows double (512 -> 1024, 256 -> 512); the lock holds (16 bad chunks < outsync_after)."""
    O = oracle()
    geom, ocfg, _ = _cfgs(O, "bpsk")
    n = 65
    weak = set(range(20, 36))
    soft, _ = M.weak_stretch(geom, n, weak, 21)
    d = M.Decoder(geom, ocfg.ber_thresold, ocfg.outsync_after)
    got = d.run(soft)
    k = d.counters
    assert len(k["misses"]) == 1 and k["misses"][0] / n > 0.02 and k["tb_first"][0] / n > 0.02, k
    assert (d.spec, d.overlap) == (1024, 512)
    assert (got["vit_state"] == 1).all()


def test_forty_weak_chunks_exhaust_six_redo_rounds():
    """The stream of the GPU exhausted-rounds case: after six rounds some start state still disagrees with its predecessor's next start,
    so the device falls back to decoding again from the first inconsistent chunk; redoing until consistent gives the oracle's bits."""
    O = oracle()
    geom, ocfg, _ = _cfgs(O, "bpsk")
    soft, _ = M.weak_stretch(geom, 44, set(range(2, 42)), 7)
    syms = np.stack([geom.symbols(soft[i * geom.chunk:(i + 1) * geom.chunk], (0, 0, 0)) for i in range(44)])
    r = M.decode_range(geom, syms, -1, 0, geom.spec_base, M.TB_OVERLAP, rounds=6)
    assert r.rounds == 6 and not r.consistent
    ocfg.outsync_after = 100
    _pin(O, geom, ocfg, soft)


def test_half_weak_chunk_makes_a_stale_successor_ber():
    """The stream of the GPU successor-BER case: the HALF chunk is redone, its successor is not, and the redo changes the predecessor tail
    the successor's BER check reads - so a decoder that did not recompute that BER would report another one."""
    geom = M.Geom("ccsds", 8192, "bpsk")
    prof = [(40, 8)] * 5 + [M.WEAK] * 3 + [M.HALF] + [M.GOOD] * 5
    soft = M.soft_stream(geom, M.coded_stream(geom, len(prof), 7), prof, 7)
    d = M.Decoder(geom, 0.3, 20)
    d.run(soft)
    r = d.last
    assert 9 in r.succ_stale and 9 not in sum(r.redo_chunks, [])
    stale = M.ber_counts(geom, d.last_syms[9], r.bits[9], r.first_tail[8])
    assert stale != r.ber[9]
