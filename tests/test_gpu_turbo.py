"""GPU: ccsds_turbo_decoder parity. The correlator, the frame walk and the frame bytes fed to the decoder (shift quirk included) are exact;
the BCJR runs in double with the reference's operation order. Given a soft stream, the CUDA path must write the reference's CADUs and
reproduce every frame's (offset, pos, correlator_corr, swapped, crc_ok) record: against oracle/_ref where it was built, else against
tests/golden/turbo_pins.json. Decision margins below 1e-9 (where a last-ulp difference of exp / log could tip a bit) are counted and
reported."""
import numpy as np
import pytest

from tests.common import assert_pin, run_chain, run_cli
from tests.turbo_cases import CASES, RATE_NAME, digest, frame_size, pins, stream

pytestmark = pytest.mark.gpu


def expected(name):
    """The reference's (CADU digest, number of CADUs, records) for a case"""
    from oracle import turbo as O
    case = CASES[name]
    pin = pins()["cases"][name]
    if O.available():
        soft, _, _ = stream(case)
        r = O.Turbo(RATE_NAME[case["rate"]], case["base"], case["iters"]).run(soft)
        assert_pin(pin, "turbo_pins.json", cadu=digest(r["cadu"]), recs=r["recs"].tolist())
    return pin["cadu"], pin["ncadu"], np.array(pin["recs"], np.int64).reshape(-1, 6)


def gpu(case, max_soft):
    from satdump_b200 import capi
    return capi.Fec(capi.turbo_cfg(RATE_NAME[case["rate"]], case["base"], case["iters"], max_soft=max_soft))


def check(name, capsys=None):
    case = CASES[name]
    want_digest, ncadu, want_recs = expected(name)
    soft, clear, cuts = stream(case)
    g = gpu(case, max(1 << 16, soft.size))
    cuts = [0] + list(cuts) + [soft.size]
    frames, recs = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        g.push(soft[a:b])
        frames.append(g.frames())
        recs.append(g.turbo_frames())
    got, grec = np.concatenate(frames), np.concatenate(recs)
    assert np.array_equal(grec, want_recs), (grec, want_recs)
    assert got.shape[0] == ncadu and digest(got) == want_digest
    s = g.stats()
    assert s["crc_ok"] == ncadu and s["crc_fail"] == want_recs.shape[0] - ncadu and s["frames_out"] == ncadu
    if want_recs.shape[0]:
        assert s["correlator_lock"] == want_recs[-1, 5]
        assert np.float32(s["correlator_corr"]).view(np.uint32) == np.uint32(want_recs[-1, 2])
    for row in got:  # every written frame is a transmitted one
        assert any(np.array_equal(row, c) for c in clear)
    print(f"{name}: {want_recs.shape[0]} frames, {ncadu} CADUs, decision margins below 1e-9: {s['turbo_near_ties']}")
    return got, want_recs, s


@pytest.mark.parametrize("rate", [2, 3, 4, 6])
@pytest.mark.parametrize("base", [223, 446, 892, 1115])
def test_every_rate_and_base(built, rate, base):
    """All 16 combinations at 1-2 iterations; the first frame, behind 37 bytes of noise, is read with the shift quirk and fails its CRC."""
    got, recs, _ = check(f"combo_{rate}_{base}")
    assert recs.shape[0] == 2 and recs[0, 1] == 37 and got.shape[0] == 1


@pytest.mark.parametrize("name", ["r2_1115_it1", "r2_1115_it5", "r2_1115_it50", "r4_1115_it2", "r6_1115_it1", "r6_1115_it20", "r2_223_it10"])
def test_shipped_iteration_counts(built, name):
    check(name)


def test_crc_failures(built):
    """A noise level at which some frames fail their CRC: only the others are written."""
    got, recs, s = check("crc_failures")
    assert 0 < got.shape[0] < recs.shape[0] and s["crc_fail"] > 0


def test_swapped_polarity(built):
    got, recs, _ = check("swapped")
    assert recs[:, 3].all() and got.shape[0] >= 3


def test_inserted_and_deleted_soft_bytes(built):
    """Bytes inserted and deleted mid-stream shift the walk's lattice; the shifted frames hold the stale bytes the module's buffer keeps."""
    _, recs, _ = check("inserted_deleted")
    assert (recs[1:, 1] != 0).sum() >= 2


def test_noise_signal_noise(built):
    """Noise -> signal -> noise -> signal, including a shift above F / 2 (where the module's memmove reads past its buffer)."""
    _, recs, _ = check("noise_signal_noise")
    F = frame_size(2, 223)
    assert (recs[:, 1] > F // 2).any() and (recs[:, 5] == 1).sum() >= 3


def test_ragged_pushes(built):
    """Cut points inside the ASM, mid-frame and one byte apart give the records and CADUs of one push."""
    check("ragged")


def test_large_push_matches_transmitted_frames(built):
    """500 frames in one push (one decoding batch): every CADU is the transmitted one."""
    from satdump_b200 import synth
    from satdump_b200 import capi
    tx, clear = synth.turbo_frames(500, 2, 223, seed=99)
    soft = synth.ldpc_soft(tx.reshape(-1), "bpsk", sigma=30.0, seed=5)
    g = capi.Fec(capi.turbo_cfg("1/2", 223, 2, max_soft=soft.size + 65536))
    got = g.push(soft).frames()
    assert got.shape == clear.shape and np.array_equal(got, clear)
    t = g.turbo_timing()
    assert t["push"] > 0 and t["bcjr"] > 0


def chain_expected(name):
    """(CADU digest of the reference's frames from the third on, their number): the reference's demodulator + turbo decoder where it was
    built, else the pins"""
    from oracle import turbo as O
    from tests.turbo_cases import chain_reference
    pin = pins()["chain"][name]
    if O.available():
        want = chain_reference(name)
        assert_pin(pin, "turbo_pins.json", tail=digest(want[2:]), ncadu=want.shape[0])
    return pin["tail"], pin["ncadu"]


def same_after_lock(got, name, clear):
    """The first frames are read while the demodulator's loops still acquire: their soft bytes sit on the float floor of the demodulator
    (DESIGN §5). From the third frame on the CADUs are the reference's; every written CADU passed its CRC and is a transmitted frame."""
    from tests.common import match_frames
    tail, n = chain_expected(name)
    assert got.shape[0] == n and digest(got[2:]) == tail
    assert all(any(np.array_equal(row, c) for c in clear) for row in got)
    assert match_frames(got[2:], clear)[1]


@pytest.mark.parametrize("name", ["turbo_pm", "turbo_bpsk"])
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain_end_to_end(built, name, pipelined):
    """IQ -> pm_demod (Juice-like) / psk_demod BPSK (Psyche-like) -> ccsds_turbo_decoder through the fused chain, synchronous and
    pipelined, in three pushes."""
    from satdump_b200 import capi
    from tests.common import signal
    from tests.turbo_cases import CHAIN, chain_demod_kwargs
    log2n, seed = CHAIN[name]
    cfg, raw, clear = signal(name, log2n, seed=seed)
    n = raw.size // 2
    got, _ = run_chain(capi.demod_cfg(max_batch=n, **chain_demod_kwargs(cfg)), capi.fec_cfg_for(cfg, max_soft=4 * n), raw, cfg.fmt,
                       pipelined)
    same_after_lock(got, name, clear)


@pytest.mark.parametrize("name", ["turbo_pm", "turbo_bpsk"])
@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli_module_layer(built, tmp_path, name, mode):
    """The C++ module layer with module id ccsds_turbo_decoder (parameters parsed as CCSDSTurboDecoderModule's constructor), as the
    b200_pipeline CLI runs it with the Juice / Psyche module parameters: the .cadu file holds the reference's frames."""
    from tests.common import signal
    from tests.turbo_cases import CHAIN
    log2n, seed = CHAIN[name]
    cfg, raw, clear = signal(name, log2n, seed=seed)
    inp = tmp_path / "in.raw"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    # pm_demod's own clock-recovery defaults (0.01) differ from the psk_demod ones the checker's configuration carries: pass those
    extra = ["--clock_gain_omega", repr(float(np.float32(8.7e-3 ** 2 / 4.0))), "--clock_gain_mu", "0.0087"] if name == "turbo_pm" else []
    run_cli(name, inp, hint, "--samplerate", str(int(cfg.samplerate)), "--symbolrate", str(int(cfg.symbolrate)), "--baseband_format", cfg.fmt,
            *extra, fused=mode == "fused")
    got = np.fromfile(hint + ".cadu", np.uint8).reshape(-1, cfg.cadu_bytes)
    same_after_lock(got, name, clear)


@pytest.mark.parametrize("name", ["llr_2_223", "llr_6_223"])
def test_extrinsic_values_match_reference(built, name):
    """The a-priori arrays after the last iteration (turbo_decode's messages) against the reference's convcode_extrinsic
    (tests/golden/turbo_llr.npz): the difference relative to the array's largest magnitude is at most 1e-12. CUDA's double exp / log are
    not glibc's and may differ in the last ulp, so the values are not claimed bitwise; the decisions are (the records and CADUs are
    compared exactly). Each value is a log-sum of terms of the array's scale, so it carries their absolute rounding: where a value
    crosses zero (2.5e-4 in a frame whose values reach 7.7) that rounding is 1e-10 of the value itself, which is why the gate is not
    element by element."""
    from tests.turbo_cases import LLR, llr_frames
    check(name)
    case = CASES[name]
    soft, _, _ = stream(case)
    g = gpu(case, max(1 << 16, soft.size))
    g.push(soft)
    gold = np.load(LLR)
    K = 8 * case["base"]
    worst = worst_elem = 0.0
    for k, _, _ in llr_frames(name):
        got = g.turbo_llr(k, K)
        for u in (0, 1):
            want = gold[f"{name}_{k}_{u}"]
            d = np.abs(got[u] - want)
            rel = float(d.max() / np.abs(want).max())
            worst = max(worst, rel)
            worst_elem = max(worst_elem, float((d / np.maximum(np.abs(want), 1e-300)).max()))
            assert rel <= 1e-12, (k, u, rel, int(d.argmax()))
    print(f"{name}: a-priori arrays: largest difference / largest magnitude {worst:.3g}; element by element {worst_elem:.3g}")
