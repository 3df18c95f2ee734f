"""GPU: fengyun_mpt_decoder (B200_FEC_FENGYUN_MPT) against the reference (oracle/_ref, else the pins of
tests/golden/fengyun_mpt_pins.json) on every case stream: the records after every read (shift, invert_branches, v1, v2, both Viterbi
states and BERs, deframer state), the CADUs and the stats, pushed whole, in ragged pieces (1, 3, 16383 and 16385 bytes, so that a partial
read and the search machines cross pushes) and as one push of 2^26 bytes; IQ (cs16, cs8) -> psk_demod QPSK -> the decoder through
b200_chain, synchronous and pipelined, against the reference chain and the sent frames; b200_pipeline fengyun_mpt, two-stage and fused."""
import numpy as np
import pytest

from satdump_b200 import capi, synth
from tests import fengyun_mpt_cases as X
from tests.common import pieces, run_chain, run_cli

pytestmark = pytest.mark.gpu


def _decode(soft, cuts=(), max_soft=1 << 22):
    f = capi.Fec(capi.fengyun_mpt_cfg(X.OUTSYNC, X.BER, max_soft=max_soft))
    out, recs = [], []
    for a, b in pieces(soft.size, cuts):
        f.push(soft[a:b])
        out.append(f.frames())
        recs.append(f.fengyun_reads())
    st = f.stats()
    f.close()
    return np.concatenate(out), np.concatenate(recs), st


def _check(name, out, recs, st):
    pin = X.ref_result(name)
    assert recs.shape[0] == pin["reads"]
    if X.recs_digest(recs) != pin["recs"]:
        from oracle import fengyun_mpt
        if fengyun_mpt.available():  # name the first read that differs
            want = fengyun_mpt.RefMpt(X.OUTSYNC, X.BER).run(X.stream(name))["recs"].astype(np.float32)
            bad = np.nonzero((want != recs.astype(np.float32)).any(1))[0]
            raise AssertionError(f"{name}: read {bad[0]}: reference {want[bad[0]].tolist()} decoder {recs[bad[0]].tolist()}")
        raise AssertionError(f"{name}: per-read records differ")
    assert out.shape[0] == pin["frames"] and X.digest(out) == pin["out"]
    assert st["frames_out"] == pin["frames"] and st["rs_avg"] == pin["rs_avg"]
    assert (st["deframer_state"] == 12) == bool(pin["deframer_lock"])
    if recs.shape[0]:
        last = recs[-1]
        assert (st["viterbi_state"], st["viterbi2_state"], st["deframer_state"]) == (last[4], last[5], last[8])
        assert np.float32(st["viterbi_ber"]) == np.float32(last[6]) and np.float32(st["viterbi2_ber"]) == np.float32(last[7])


@pytest.mark.parametrize("name", X.CASES)
def test_whole_stream(name):
    _check(name, *_decode(X.stream(name)))


def test_shift_quirk():
    """the Q branch buried: viterbi2 in NOSYNC for more than ten reads and shift never toggles; the I branch buried: shift toggles"""
    _, q, _ = _decode(X.stream("q_buried"))
    _, i, _ = _decode(X.stream("i_buried"))
    assert (q[:, 5] == 0).sum() >= 10 + (q[:, 4] == 0).sum() and (np.diff(q[:, 0]) == 0).all()
    assert (np.diff(i[:, 0]) != 0).any()


def _cuts(n, sizes, limit=2000):
    """cuts cycling through `sizes` for the first `limit` pieces, then whole reads"""
    cuts, at, i = [], 0, 0
    while at < n and len(cuts) < limit:
        at += sizes[i % len(sizes)]
        i += 1
        if at < n:
            cuts.append(at)
    nxt = (at // X.READ + 1) * X.READ
    return cuts + list(range(nxt, n, X.READ))


@pytest.mark.parametrize("sizes", [(1, 3, 16383, 16385), (16383,), (16385, 1), (100003,)])
@pytest.mark.parametrize("name", X.CASES)
def test_pieces(name, sizes):
    soft = X.stream(name)
    _check(name, *_decode(soft, _cuts(soft.size, sizes)))


@pytest.mark.parametrize("name", X.LARGE)
def test_one_large_push(name):
    soft = X.stream(name)
    _check(name, *_decode(soft, max_soft=soft.size))


def test_short_last_read_waits():
    """a push that ends inside a read decodes nothing of it: only what was pushed is decoded"""
    soft = X.stream("clean")
    f = capi.Fec(capi.fengyun_mpt_cfg(X.OUTSYNC, X.BER, max_soft=1 << 22))
    f.push(soft[:10 * X.READ + 5000])
    assert f.fengyun_reads().shape[0] == 10 and f.stats()["chunks"] == 10
    f.push(soft[10 * X.READ + 5000:11 * X.READ - 1])
    assert f.fengyun_reads().shape[0] == 0
    f.push(soft[11 * X.READ - 1:11 * X.READ])
    assert f.fengyun_reads().shape[0] == 1
    f.close()


def test_invert_second_viterbi_refused():
    cfg = capi.fengyun_mpt_cfg(X.OUTSYNC, X.BER, max_soft=1 << 20)
    cfg.invert_second_viterbi = 1
    with pytest.raises(capi.B200Error, match="invert_second_viterbi"):
        capi.Fec(cfg)


def _signal(fmt, n=1 << 22):
    cfg = synth.CONFIGS["fengyun_mpt"]
    cfg = synth.SignalCfg(**{**cfg.__dict__, "fmt": fmt})
    raw, clear = synth.make_signal(cfg, n, seed=5)
    return cfg, raw.numpy(), clear


def _chain(cfg, raw, pipelined):
    n = raw.size // 2
    return run_chain(capi.demod_cfg_for(cfg, max_batch=n), capi.fec_cfg_for(cfg, max_soft=n), raw, cfg.fmt, pipelined)


@pytest.mark.parametrize("fmt", ["cs16", "cs8"])
def test_chain(fmt):
    """IQ -> psk_demod QPSK with the pipeline's parameters -> the decoder through b200_chain, in three pushes: synchronous and pipelined
    write the same CADUs, the reference chain writes them too, and after the lock they are the sent frames"""
    cfg, raw, clear = _signal(fmt)
    sync, fs = _chain(cfg, raw, False)
    pipe, fp = _chain(cfg, raw, True)
    assert np.array_equal(sync, pipe) and fs["frames_out"] == fp["frames_out"] == sync.shape[0]
    sent = {bytes(r) for r in np.asarray(clear)}
    good = sum(bytes(r) in sent for r in sync)
    assert sync.shape[0] >= 100 and good >= sync.shape[0] - 8
    try:
        from oracle import ref as orc
        if not orc.available():
            raise ImportError
    except ImportError:
        from oracle import port as orc
    from oracle import fengyun_mpt
    if fengyun_mpt.available():
        soft = orc.Demod(orc.demod_cfg(cfg.samplerate, cfg.symbolrate, cfg.constellation, cfg.rrc_alpha, cfg.pll_bw, cfg.fmt)).run(raw, stages=False)["soft"]
        want = fengyun_mpt.RefMpt(cfg.outsync_after, cfg.ber_thresold).run(soft)["out"]
        assert np.array_equal(sync, want)


def test_cli(built, tmp_path):
    """b200_pipeline fengyun_mpt, two-stage and fused, write the same .cadu, the sent frames after the lock"""
    cfg, raw, clear = _signal("cs16")
    inp = tmp_path / "in.cs16"
    raw.tofile(inp)
    got = {}
    for mode in ("two_stage", "fused"):
        hint = str(tmp_path / mode)
        r = run_cli("fengyun_mpt", inp, hint, "--samplerate", str(int(cfg.samplerate)), "--baseband_format", "cs16", fused=mode == "fused",
                    timeout=600)
        got[mode] = np.fromfile(hint + ".cadu", np.uint8).reshape(-1, 1024)
        assert "deframer_state SYNCED" in r.stdout
    assert np.array_equal(got["two_stage"], got["fused"])
    sent = {bytes(x) for x in np.asarray(clear)}
    assert got["fused"].shape[0] >= 100 and sum(bytes(x) in sent for x in got["fused"]) >= got["fused"].shape[0] - 8
