"""GPU: aqua_db_decoder (EOS Aqua / Aura DB) parity. The decoder has no FEC stage that could hide a difference, so the CUDA path must
reproduce the reference bit for bit: the CADUs, the deframer state and the RS counts after every push of whole reads, against oracle/_ref
where it was built, else against tests/golden/eos_pins.json."""
import numpy as np
import pytest

from tests.common import assert_pin, pieces, run_chain, run_cli
from tests.eos_cases import (CASES, CHAIN, READ, TERRA_FEC, TERRA_RATE, after_lock, aqua_demod_kwargs, chain_reference, chain_signal, digest,
                             large_stream, pins, ragged_cuts, read_cuts, stats_rows, stream, terra_chain_reference, terra_demod_kwargs,
                             terra_floor, terra_reference, terra_signal)

pytestmark = pytest.mark.gpu


def run_gpu(soft, cuts):
    """The decoder over soft pushed in the pieces cut at `cuts`: the CADUs, and [frames, state, corrected, failed] after every push"""
    from satdump_b200 import capi
    g = capi.Fec(capi.aqua_db_cfg(max_soft=max(1 << 17, soft.size)))
    out, rows = [], []
    for a, b in pieces(soft.size, cuts):
        g.push(soft[a:b])
        out.append(g.frames())
        s = g.stats()
        rows.append([s["frames_out"], s["deframer_state"], s["rs_corrected"], s["rs_failed"]])
    return np.concatenate(out), rows


def check(pin, soft, cuts, every_push=True):
    from oracle import eos as O
    if O.available():
        r = O.run_pieces(soft, cuts)
        assert_pin(dict(cadu=pin["cadu"], stats=pin["stats"][-1]), "eos_pins.json", cadu=digest(r["cadu"]), stats=stats_rows(r["stats"])[-1])
    got, rows = run_gpu(soft, cuts)
    assert got.shape[0] == pin["frames"] and digest(got) == pin["cadu"]
    if every_push:
        assert rows == pin["stats"]
    else:  # (the reference decodes whole reads only: after a ragged push it may still hold bytes the GPU has decoded)
        assert rows[-1] == pin["stats"][-1]
    return got, rows


@pytest.mark.parametrize("name", sorted(CASES))
def test_cadus_state_and_rs_after_every_push(built, name):
    soft, _ = stream(name)
    check(pins()["cases"][name], soft, read_cuts(soft.size))


@pytest.mark.parametrize("name", sorted(CASES))
def test_ragged_pushes(built, name):
    """Pieces of 1, 3, 65 535 and 65 537 bytes, with cuts inside a symbol and inside an ASM: the same CADUs and final stats, and the same
    stats after every push that ends where both decoders have consumed the same bytes (a multiple of the reference's 65 536-byte read;
    DESIGN §9: elsewhere the reference still holds the bytes of its unfinished read)"""
    soft, _ = stream(name)
    cuts = ragged_cuts(soft.size, CASES[name]["lead"])
    pin = pins()["ragged"][name]
    _, rows = check(pin, soft, cuts, every_push=False)
    from oracle import eos as O
    if O.available():
        ref = stats_rows(O.run_pieces(soft, cuts)["stats"])
        ends = [*cuts, soft.size]
        same = [k for k, e in enumerate(ends) if e % READ == 0]
        assert same and all(rows[k] == ref[k] for k in same)


def test_clean_stream_is_the_sent_frames(built):
    soft, clear = stream("clean")
    got, rows = run_gpu(soft, read_cuts(soft.size))
    assert np.array_equal(got, clear) and rows[-1][2:] == [0, 0]


def test_thresholds_and_branches(built):
    """The transitions the cases were built for, as the decoder reports them: SYNCED is state 10, swapped rails never sync, t + 1 RS errors
    fail and the frames are written, and the inversion branch writes the frames upright"""
    soft, _ = stream("synced_asm_9_10")
    assert any(row[1] == 10 for row in run_gpu(soft, read_cuts(soft.size))[1])
    soft, _ = stream("iq_swapped")
    assert run_gpu(soft, [])[0].shape[0] == 0
    soft, _ = stream("rs")
    got, rows = run_gpu(soft, [])
    assert rows[-1][3] == 2 and got.shape[0] == CASES["rs"]["frames"] - 1
    for name in ("inverted", "inverted_start"):
        soft, clear = stream(name)
        got, _ = run_gpu(soft, read_cuts(soft.size))
        assert sum(any(np.array_equal(g[:896], c[:896]) for c in clear) for g in got) >= got.shape[0] - 2


def test_large_push(built):
    """At least 2^26 soft bytes in one push"""
    soft, clear = large_stream()
    assert soft.size >= 1 << 26
    pin = pins()["large"]
    got, rows = run_gpu(soft, [])
    assert got.shape[0] == pin["frames"] and digest(got) == pin["cadu"] and rows == pin["stats"]
    assert all(any(np.array_equal(got[k, :896], c[:896]) for c in clear) for k in range(0, got.shape[0], 997))


def _chain_tail_matches(got, name, clear):
    pin = pins()["chain"][name]
    from oracle import eos as O
    if O.available():
        o, _ = chain_reference(name)
        t = after_lock(o, clear)
        assert_pin(pin, "eos_pins.json", ntail=t.shape[0], tail=digest(t))
    tail = after_lock(got, clear)
    # the reference decodes whole reads only, so the GPU, which decodes every byte, may write more frames at the end
    assert tail.shape[0] >= pin["ntail"] >= 100 and digest(tail[:pin["ntail"]]) == pin["tail"]
    assert all(any(np.array_equal(row[:896], c[:896]) for c in clear) for row in tail)  # (RS corrects the data, not the check bytes)


@pytest.mark.parametrize("name", sorted(CHAIN))
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain(built, name, pipelined):
    """IQ at 15 MS/s -> psk_demod OQPSK (EOS.json's parameters) -> aqua_db_decoder through the fused chain, in three pushes"""
    from satdump_b200 import capi
    cfg, raw, clear = chain_signal(name)
    n = raw.size // 2
    got, fs = run_chain(capi.demod_cfg(max_batch=n, **aqua_demod_kwargs(cfg.fmt)), capi.aqua_db_cfg(max_soft=n + READ), raw, cfg.fmt,
                        pipelined)
    _chain_tail_matches(got, name, clear)
    assert fs["deframer_state"] == 10


@pytest.mark.parametrize("pipe", ["aqua_db", "aura_db"])
@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli(built, tmp_path, pipe, mode):
    """b200_pipeline aqua_db | aura_db (EOS.json's psk_demod parameters) writes the reference chain's .cadu after the lock and reports
    deframer_state"""
    cfg, raw, clear = chain_signal("cs16")
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    r = run_cli(pipe, inp, hint, "--samplerate", "15000000", "--baseband_format", "cs16", fused=mode == "fused")
    _chain_tail_matches(np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024), "cs16", clear)
    assert "deframer_state SYNCED" in r.stdout


# ---- Terra DB: terra_db_demod (BPSK loops at twice the symbol rate, 1.714 samples per half-symbol) -> ccsds_conv_concat_decoder ----------
def _terra_demod(n, keep_stages=False):
    from satdump_b200 import capi
    return capi.Demod(capi.demod_cfg(max_batch=max(n, 4096), keep_stages=keep_stages, **terra_demod_kwargs()))


def test_terra_taps_and_omega_bitwise(built):
    """RRC(1, 45 MS/s, 2 x 13.125 Msym/s, 0.5, 31) and the M&M's starting omega ((float)fs / (float)rs) / 2 are the reference's"""
    from tests.common import oracle
    O = oracle()
    g = _terra_demod(4096)
    rrc, bank = g.taps()
    assert np.array_equal(rrc, O.rrc_design(1, np.float32(TERRA_RATE[0]), 2 * TERRA_RATE[1], 0.5, 31)) and np.array_equal(bank, O.mm_taps())
    omega = (np.float32(TERRA_RATE[0]) / np.float32(TERRA_RATE[1])) / np.float32(2)
    assert np.float32(g.stats()["mm_omega"]).view(np.uint32) == omega.view(np.uint32)


def test_terra_strict_sequential_mm_is_the_reference_block(built):
    """At omega 1.714 (advances of one or two samples per half-symbol) the strict sequential M&M is bitwise the reference block"""
    O, oc, o = terra_reference()
    x = o["costas"][:1 << 19]
    want = O.run_stage(oc, "mm", x)
    got = _terra_demod(x.size).run_stage("mm", x, strict=True, sequential=True)
    assert got.size == want.size and np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_terra_segmented_soft_within_gates(built):
    """The production demodulator (segmented loops) on the Terra signal: the same symbol count, symbols and soft bytes within
    max(SURVEY 8c gate, 1.2 x the reference's own floor), and its junction counters"""
    from tests.test_gpu_demod import check_mm
    raw, _ = terra_signal()
    _, _, o = terra_reference()
    g = _terra_demod(raw.size // 2).push(raw)
    check_mm(g.symbols(), o["mm"], g.soft(), o["soft"], floor=terra_floor())
    s = g.stats()
    _, mm_res, L = g.junctions()
    print(f"terra junctions: {mm_res.size} segments of {L} samples, costas_unconverged {s['costas_unconverged']}, "
          f"mm_unconverged {s['mm_unconverged']}, repairs {s['repairs']}")
    assert mm_res.size > 1 and s["costas_unconverged"] == 0 and s["mm_unconverged"] == 0


def _terra_tail_matches(got, clear):
    pin = pins()["terra_chain"]
    from tests.common import oracle
    from oracle import ref
    if oracle() is ref:
        t = after_lock(terra_chain_reference(), clear)
        assert_pin(pin, "eos_pins.json", ntail=t.shape[0], tail=digest(t))
    tail = after_lock(got, clear)
    assert tail.shape[0] >= pin["ntail"] >= 50 and digest(tail[:pin["ntail"]]) == pin["tail"]
    assert all(any(np.array_equal(row[:896], c[:896]) for c in clear) for row in tail)


@pytest.mark.parametrize("pipelined", [False, True])
def test_terra_fused_chain(built, pipelined):
    """IQ at 45 MS/s -> terra_db_demod -> ccsds_conv_concat_decoder (EOS.json's parameters) through the fused chain, in three pushes"""
    from satdump_b200 import capi
    raw, clear = terra_signal()
    n = raw.size // 2
    got, _ = run_chain(capi.demod_cfg(max_batch=n, **terra_demod_kwargs()),
                       capi.ccsds_cfg("bpsk_90", 8192, 0.3, 20, max_soft=2 * n, **TERRA_FEC), raw, "cs16", pipelined)
    _terra_tail_matches(got, clear)


@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_terra_cli(built, tmp_path, mode):
    """b200_pipeline terra_db (terra_db_demod, then EOS.json's decoder parameters) writes the reference chain's .cadu after the lock"""
    raw, clear = terra_signal()
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    hint = str(tmp_path / "out")
    run_cli("terra_db", inp, hint, "--samplerate", "45000000", "--baseband_format", "cs16", fused=mode == "fused", timeout=600)
    _terra_tail_matches(np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024), clear)


def test_library_refuses_too_few_samples_per_half_symbol(built):
    """26 MS/s lies inside [1.1, 4.0] samples per symbol, so nothing resamples it, but it is 0.99 per half-symbol: the library names the
    samples per symbol its loops would run at"""
    from satdump_b200 import capi
    with pytest.raises(capi.B200Error, match="samples per symbol 0.99"):
        capi.Demod(capi.demod_cfg(26e6, 26250000, "bpsk", 0.5, final_samplerate=0.0, max_batch=4096))


def test_library_refuses_an_aqua_push_size_above_2_30(built):
    from satdump_b200 import capi
    with pytest.raises(capi.B200Error, match="max_soft must be <= 2\\^30"):
        capi.Fec(capi.aqua_db_cfg(max_soft=(1 << 30) + 1))


@pytest.mark.parametrize("cuts", [(), (8191, 3 * 8192 + 1, 300001)])
def test_terra_decoder_equals_the_reference(built, cuts):
    """EOS.json's ccsds_conv_concat_decoder ("bpsk_90": every soft pair swapped, then Viterbi at 90 degrees) on the reference
    demodulator's soft bytes, pushed whole and cut inside pairs: the reference's CADUs, deframer state and RS counts"""
    from satdump_b200 import capi
    O, _, o = terra_reference(stages=False)
    soft = o["soft"][:o["soft"].size // 8192 * 8192]
    want = O.Fec(O.ccsds_cfg("bpsk_90", 8192, 0.3, 20, **TERRA_FEC)).run(soft)
    g = capi.Fec(capi.ccsds_cfg("bpsk_90", 8192, 0.3, 20, max_soft=soft.size, **TERRA_FEC))
    got = np.concatenate([g.push(soft[a:b]).frames() for a, b in pieces(soft.size, cuts)])
    assert got.shape[0] >= 60 and np.array_equal(got.reshape(-1), want["cadu"])
    s = g.stats()
    e = want["rs_err"]
    assert s["deframer_state"] == int(want["defr_state"][-1]) and s["rs_corrected"] == int(e[e >= 0].sum()) and s["rs_failed"] == int((e < 0).sum())
