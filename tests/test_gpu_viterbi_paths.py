"""GPU: the correction paths of the optimistic Viterbi decoder (api_fec.cu decode_range / viterbi_segment / decode_conv), each driven by
its input alone in the configuration that ships: start-state redo, serial chainback of blocks whose edges disagree, the adaptive speculation
and warm-up windows, and the MetOp "deframer stuck in NOSYNC -> viterbi.reset()" rollback. Every case checks that the outputs equal the
oracle's AND that the counter of the path it targets is nonzero: a case whose path did not run tests nothing. The streams come from
tests/viterbi_model.py, whose CPU test (tests/test_viterbi_model.py) predicts the same paths from the same streams."""
import numpy as np
import pytest

from tests import viterbi_model as M
from tests.common import oracle

pytestmark = pytest.mark.gpu


def _cfgs(kind, outsync=None):
    from satdump_b200 import capi
    O = oracle()
    if kind == "metop":
        o = 10 if outsync is None else outsync
        return M.Geom("metop"), O.metop_cfg(0.28, o), lambda n: capi.metop_cfg(0.28, o, max_soft=n), {}
    if kind == "bpsk":
        o = 20 if outsync is None else outsync
        return (M.Geom("ccsds", 8192, "bpsk"), O.ccsds_cfg("bpsk", 8192, 0.3, o, 4),
                lambda n: capi.ccsds_cfg("bpsk", 8192, 0.3, o, 4, max_soft=n), {})
    return (M.Geom("ccsds", 10232, "oqpsk", nrzm=True), O.ccsds_cfg("oqpsk", 10232, 0.3, 20, 5, nrzm=True, rs_usecheck=True),
            lambda n: capi.ccsds_cfg("oqpsk", 10232, 0.3, 20, 5, nrzm=True, rs_usecheck=True, max_soft=n), dict(cadu_size=10232, interleave=5))


def _run(gcfg, soft, cuts, max_push=None, want=None, chunk=None, resets=()):
    """Pushes soft[prev:cut] for every cut; returns (bits, frames, stats) of the whole stream. With `want`: after every push the lock state
    and the BER the decoder reports equal the oracle's at the push's last complete chunk (the oracle records the lock state of a chunk
    before a MetOp reset that follows it: after a push that ends on a reset chunk the decoder is IDLE)."""
    from satdump_b200 import capi
    g = capi.Fec(gcfg(max(65536, max_push or soft.size)))
    bits, frames, prev = [], [], 0
    for c in cuts:
        g.push(soft[prev:c])
        bits.append(g.bits())
        frames.append(g.frames().reshape(-1))
        prev = c
        if want is not None and c >= chunk:
            s, q = g.stats(), c // chunk - 1
            assert s["viterbi_state"] == (0 if q in resets else int(want["vit_state"][q])), (c, q)
            if want["vit_state"][q]:
                assert np.float32(s["viterbi_ber"]) == want["vit_ber"][q], (c, q, s["viterbi_ber"], want["vit_ber"][q])
    return np.concatenate(bits), np.concatenate(frames), g.stats()


def _check(want, bits, frames, s):
    assert np.array_equal(bits, want["bits"])
    assert np.array_equal(frames, want["cadu"])
    assert s["viterbi_state"] == int(want["vit_state"][-1])
    ok = want["rs_err"][want["rs_err"] >= 0]
    assert s["rs_corrected"] == int(ok.sum()) and s["rs_failed"] == int((want["rs_err"] < 0).sum())


@pytest.mark.parametrize("kind", ["metop", "bpsk", "jpss"])
def test_start_redo_and_serial_chainback(built, kind):
    """Six WEAK chunks inside a good stream: start states mis-speculated (redone over several rounds), block edges that disagree (chained
    back serially). One push - where the counters equal what the model predicts - and ragged pushes cut at a mis-speculated chunk, so that
    it starts the second push from the carried state, and just behind it, so that its redo is the last chunk of the first push."""
    geom, ocfg, gcfg, kw = _cfgs(kind)
    n = 16
    soft, _ = M.weak_stretch(geom, n, set(range(5, 11)), 7, **kw)
    want = oracle().Fec(ocfg).run(soft)
    model = M.Decoder(geom, ocfg.ber_thresold, ocfg.outsync_after)
    model.run(soft)
    k = model.counters
    assert (want["vit_state"] == 1).all() and want["nframes"] > 0
    bits, frames, s = _run(gcfg, soft, [soft.size], want=want, chunk=geom.chunk)
    _check(want, bits, frames, s)
    print(kind, "one push:", {x: s[x] for x in ("start_redone", "tb_serial", "replays", "spec_steps", "tb_overlap")}, "model:", k)
    assert s["start_redone"] > 0 and s["tb_serial"] > 0
    assert s["start_redone"] == k["start_redone"] and s["tb_serial"] == k["tb_serial"]
    m = k["redo"][0][0]  # the first chunk whose start state the speculation got wrong
    for cuts in ([m * geom.chunk, soft.size], [(m + 1) * geom.chunk + 3, soft.size]):
        bits, frames, s = _run(gcfg, soft, cuts, want=want, chunk=geom.chunk)
        _check(want, bits, frames, s)
        assert s["start_redone"] > 0 and s["tb_serial"] > 0, cuts


def test_successor_ber_decides_the_lock(built):
    """Three WEAK chunks and a HALF one (weak first half) in a good stream: the HALF chunk is mis-speculated and redone, and the redo
    changes the predecessor tail its (correctly speculated, not redone) successor's BER check reads. The BER threshold sits between that
    successor's BER from the redone bits and its BER from the first-pass bits, and outsync_after = 4 leaves the four bad chunks before it
    one short of unlocking: the lock at the successor is decided by the recomputed BER. Pushes end on the successor, so the lock state and
    the BER the decoder reports there are compared with the oracle's too."""
    from satdump_b200 import capi
    geom = M.Geom("ccsds", 8192, "bpsk")
    prof = [(40, 8)] * 5 + [M.WEAK] * 3 + [M.HALF] + [M.GOOD] * 5  # (chunks 0-4 so clean that their BER is far below the threshold)
    soft = M.soft_stream(geom, M.coded_stream(geom, len(prof), 7), prof, 7)
    probe = M.Decoder(geom, 0.3, 20)
    probe.run(soft)
    r, j = probe.last, 9  # the successor of the HALF chunk (the range starts at chunk 0)
    assert j in r.succ_stale and 8 in r.redo_chunks[0] and j not in sum(r.redo_chunks, [])
    true_ber = M.ber_value(geom, *r.ber[j])
    stale_ber = M.ber_value(geom, *M.ber_counts(geom, probe.last_syms[j], r.bits[j], r.first_tail[j - 1]))
    assert true_ber != stale_ber
    thr = float(np.float32((np.float64(true_ber) + np.float64(stale_ber)) / 2))
    O = oracle()
    want = O.Fec(O.ccsds_cfg("bpsk", 8192, thr, 4, 4)).run(soft)
    model = M.Decoder(geom, thr, 4).run(soft)
    assert np.array_equal(model["vit_state"], want["vit_state"])
    # the successor is the chunk that keeps or loses the lock: all good chunks before the weak ones are locked, and the lock at chunk 9
    # follows the side of the threshold its true BER is on
    assert (want["vit_state"][:j] == 1).all() and want["vit_state"][j] == (1 if true_ber <= thr else 0)
    gcfg = lambda n: capi.ccsds_cfg("bpsk", 8192, thr, 4, 4, max_soft=n)
    for cuts in ([(j + 1) * geom.chunk, soft.size], [soft.size]):
        bits, frames, s = _run(gcfg, soft, cuts, want=want, chunk=geom.chunk)
        _check(want, bits, frames, s)
        assert s["start_redone"] > 0
    print("successor BER: true", true_ber, "first pass", stale_ber, "threshold", thr, "lock at the successor", want["vit_state"][j])


def test_redo_rounds_exhausted(built):
    """40 WEAK chunks (the lock held by outsync_after) chain mis-speculations deeper than six redo rounds settle (the model predicts
    it): the chunks up to the first inconsistent one are accepted and the rest is decoded again from the true state, bit-exact."""
    geom, ocfg, gcfg, kw = _cfgs("bpsk", outsync=100)
    n = 44
    soft, _ = M.weak_stretch(geom, n, set(range(2, 42)), 7)
    want = oracle().Fec(ocfg).run(soft)
    assert (want["vit_state"] == 1).all()
    bits, frames, s = _run(gcfg, soft, [soft.size], want=want, chunk=geom.chunk)
    _check(want, bits, frames, s)
    fallback = s["replays"] - s["start_redone"] - s["tb_serial"]
    print("exhausted:", s["start_redone"], s["tb_serial"], "fallbacks", fallback)
    assert fallback > 0 and s["start_redone"] > 0


PUNC = {"p2/3": "2/3", "p7/8": "7/8"}


def _punc_stream(conv, ncalls, weak, seed):
    """QPSK soft bytes of the punctured code (synth.puncture_dvb) carrying RS I=4 CADUs; the calls in `weak` are WEAK."""
    from satdump_b200 import synth
    rng = np.random.default_rng(seed)
    nfr = ncalls + 2
    tx, _ = synth.build_cadus(rng.integers(0, 256, size=(nfr, 4 * 223), dtype=np.uint8), 4)
    coded = synth.puncture_dvb(synth.conv_encode(np.unpackbits(tx.reshape(-1))), conv)
    out = np.empty(ncalls * 8192, np.int8)
    for c in range(ncalls):
        amp, sigma = M.WEAK if c in weak else M.GOOD
        x = coded[c * 8192:(c + 1) * 8192] * 2.0 - 1
        out[c * 8192:(c + 1) * 8192] = np.clip(np.round(x * amp + rng.normal(0, sigma, x.size)), -127, 127)
    return out


@pytest.mark.parametrize("conv", ["p2/3", "p7/8"])
@pytest.mark.parametrize("nweak", [6, 24])
def test_punctured_start_redo_and_serial_chainback(built, conv, nweak):
    """Viterbi_Depunc's windows go through the same speculation and redo rounds: WEAK calls inside a good stream (24 of them with the lock
    held by outsync_after: mis-speculations chained deeper than six rounds, which the depunctured path settles by redoing until every
    window agrees with its predecessor), one push and ragged pushes, bit-exact with the oracle."""
    from satdump_b200 import capi
    O = oracle()
    n = nweak + 10
    soft = _punc_stream(conv, n, set(range(5, 5 + nweak)), 3)
    outsync = 20 if nweak < 20 else 100
    want = O.Fec(O.ccsds_cfg("qpsk", 8192, 0.3, outsync, 4, conv_rate=PUNC[conv])).run(soft)
    assert (want["vit_state"] == 1).all() and want["nframes"] > 0
    gcfg = lambda m: capi.ccsds_cfg("qpsk", 8192, 0.3, outsync, 4, conv_rate=PUNC[conv], max_soft=m)
    for cuts in ([soft.size], [7 * 8192 + 5, 8 * 8192, soft.size]):
        bits, frames, s = _run(gcfg, soft, cuts, want=want, chunk=8192)
        _check(want, bits, frames, s)
        print(conv, nweak, cuts, {x: s[x] for x in ("start_redone", "tb_serial", "replays")})
        assert s["start_redone"] > 0 and s["tb_serial"] > 0, cuts


def test_two_deframer_replay(built):
    """Plain QPSK (ccsds_simple_psk_decoder, two deframers 90 degrees apart): the first part of the push is rotated so that only the
    second deframer finds frames, the rest so that only the main one does. Both find frames in one push, so the push is redone chunk by
    chunk and the frames come out in the reference's order."""
    from satdump_b200 import capi
    from tests.common import simple_soft_cases
    O = oracle()
    cases, _ = simple_soft_cases()
    a = next(c for c in cases if c[0] == "qpsk_rot0")[2]
    b = next(c for c in cases if c[0] == "qpsk_rot1")[2]
    cut = 8192 * 10
    soft = np.concatenate([a[:cut], b[cut:]])
    soft = soft[:soft.size // 8192 * 8192]
    want = O.Fec(O.simple_cfg("qpsk", 8192, 4)).run(soft)
    # vit_state of the simple decoder = the second deframer's state, defr_state = the main one's (2 = NOSYNC)
    first, second = slice(0, 10), slice(10, None)
    assert (want["vit_state"][first] != 2).any() and (want["defr_state"][first] == 2).all()
    assert (want["defr_state"][second] != 2).any()
    g = capi.Fec(capi.simple_cfg("qpsk", 8192, 4, max_soft=soft.size))
    g.push(soft)
    s = g.stats()
    assert np.array_equal(g.bits(), want["bits"])
    assert np.array_equal(g.frames().reshape(-1), want["cadu"]) and want["nframes"] > 0
    print("two deframers: replays", s["replays"], "frames", want["nframes"])
    assert s["replays"] == 1 and s["deframer_state"] == int(want["defr_state"][-1])


def test_adaptive_windows_grow_and_shrink(built):
    """A launch of 65 chunks with 16 WEAK ones (> 2 % misses, lock held) doubles both windows; 32 clean launches of 65 chunks halve them
    back to their defaults. The bits stay exact throughout."""
    geom, ocfg, gcfg, _ = _cfgs("bpsk")
    n, launches = 65, 33
    coded = M.coded_stream(geom, n * launches, 21)
    soft = M.soft_stream(geom, coded, [M.WEAK if 20 <= c < 36 else M.GOOD for c in range(n * launches)], 21)
    want = oracle().Fec(ocfg).run(soft)
    from satdump_b200 import capi
    g = capi.Fec(gcfg(n * geom.chunk))
    bits, frames = [], []
    for i in range(launches):
        g.push(soft[i * n * geom.chunk:(i + 1) * n * geom.chunk])
        bits.append(g.bits())
        frames.append(g.frames().reshape(-1))
        s = g.stats()
        if i == 0:
            print("after growth:", s["spec_steps"], s["tb_overlap"], s["start_redone"], s["tb_serial"])
            assert (s["spec_steps"], s["tb_overlap"]) == (1024, 512)
            assert s["start_redone"] > 0 and s["tb_serial"] > 0
        elif i < launches - 1:
            assert (s["spec_steps"], s["tb_overlap"]) == (1024, 512), i
    print("after shrinking:", s["spec_steps"], s["tb_overlap"])
    assert (s["spec_steps"], s["tb_overlap"]) == (512, 256)
    _check(want, np.concatenate(bits), np.concatenate(frames), s)


def test_spec_steps_reach_their_cap(built):
    """Launches of 65 WEAK chunks (behind five good ones that lock; a large outsync_after holds the lock) double the speculation window
    up to its cap (F / 32) * 32 and the warm-up up to TB_OVERLAP_MAX; the bits stay exact."""
    geom, ocfg, gcfg, _ = _cfgs("bpsk", outsync=100000)
    n, launches = 65, 4
    soft = M.soft_stream(geom, M.coded_stream(geom, n * launches, 3), [M.GOOD] * 5 + [M.WEAK] * (n * launches - 5), 3)
    want = oracle().Fec(ocfg).run(soft)
    assert (want["vit_state"] == 1).all()
    bits, frames, s = _run(gcfg, soft, [(i + 1) * n * geom.chunk for i in range(launches)], max_push=n * geom.chunk)
    print("cap:", s["spec_steps"], s["tb_overlap"], s["start_redone"], s["tb_serial"])
    assert s["spec_steps"] == (geom.F // 32) * 32 == 4096 and s["tb_overlap"] == M.TB_OVERLAP_MAX
    assert s["start_redone"] > 0 and s["tb_serial"] > 0
    _check(want, bits, frames, s)


def _resets(want):
    """viterbi.reset() calls of the reference (module_metop_ahrpt_decoder.cpp:59-72) from its per-chunk deframer states (2 = NOSYNC): the
    tenth chunk in a row that ends in NOSYNC resets the decoder (every chunk of these streams is decoded)."""
    runs, out = 0, []
    for c, st in enumerate(want["defr_state"]):
        if st == 2:
            runs += 1
            if runs >= 10:
                out.append(c)
                runs = 0
        else:
            runs = 0
    return out


@pytest.mark.parametrize("K,resets,cut", [(9, 0, None), (10, 1, None), (25, 2, None), (10, 1, "last"), (25, 2, "inside")])
def test_metop_viterbi_reset_rollback(built, K, resets, cut):
    """MetOp frames, then K chunks of coded random bits without ASM (the Viterbi stays locked, the deframer falls to NOSYNC), then frames
    again. Ten NOSYNC chunks in a row reset the Viterbi: the device rolls the deframer and the frame counters back to the reset chunk and
    decodes the rest from IDLE. `last`: the push ends on the reset chunk; `inside`: ragged pushes cut inside the NOSYNC run, so that the
    run's count carries over."""
    geom, ocfg, gcfg, _ = _cfgs("metop")
    n = 4 + K + 6
    soft = M.soft_stream(geom, M.coded_stream(geom, n, 5, noframes=range(4, 4 + K)), [M.GOOD] * n, 5)
    want = oracle().Fec(ocfg).run(soft)
    r = _resets(want)
    assert len(r) == resets, r
    if cut == "last":
        cuts = [(r[0] + 1) * geom.chunk, soft.size]
    elif cut == "inside":
        cuts = [(4 + 5) * geom.chunk + 123, (4 + 14) * geom.chunk + 7, soft.size]
    else:
        cuts = [soft.size]
    bits, frames, s = _run(gcfg, soft, cuts, want=want, chunk=geom.chunk, resets=r)
    _check(want, bits, frames, s)
    print("reset", K, cut, "resets at", r, "replays", s["replays"])
    # one rollback per reset and nothing else (these streams are clean: no mis-speculation, no serial chainback); a reset on a push's
    # last chunk has nothing to roll back
    assert s["start_redone"] == 0 and s["tb_serial"] == 0
    assert s["replays"] == (resets - 1 if cut == "last" else resets)
