"""GPU: the decoder half of the benchmark path (Viterbi, NRZ-M, deframer, Reed-Solomon) at the push sizes a `bench.py` step decodes, bit
for bit against the oracle on the same int8 soft bytes. A 2^29-sample step is 25 000 - 52 000 decoder chunks in one push; the other
decoder tests push at most about a hundred. At this size the redo lists, the serial-chainback list, the adaptive windows, the MetOp
rollback, the lock search after a loss and the one-warp deframer walk run over tens of thousands of chunks and frames.

  * designed streams (tests/viterbi_model.py's transmitter) at the chunk count of a 2^29-sample step of each benchmark decoder: a noisy
    GOOD background with a few hundred WEAK stretches, stretches that lose the lock, inserted noise, MetOp runs without frames and frames
    with t + 1 byte errors; each row checks that its correction paths ran at scale, then decodes the same stream in ragged pushes;
  * the benchmark's own c3 workload at 5.5 dB Es/N0 (2^28 samples): the decoder alone, the synchronous chain and the pipelined chain
    run as the benchmark's timed loop runs it;
  * one ASM in four damaged, so that the deframer loses and finds its lock thousands of times in one push.

The oracle decodes run on a thread pool while the GPU works (ctypes releases the GIL)."""
import concurrent.futures
import dataclasses
import os
import time

import numpy as np
import pytest

from satdump_b200 import synth
from tests import rs_model
from tests import viterbi_model as M
from tests.common import oracle, oracle_fec

pytestmark = pytest.mark.gpu

LOG2_STEP = 29  # bench.py --log2-samples default
KINDS = {"metop_ahrpt": dict(geom=lambda: M.Geom("metop")),
         "bpsk_half": dict(geom=lambda: M.Geom("ccsds", 8192, "bpsk")),
         "jpss_hrd": dict(geom=lambda: M.Geom("ccsds", 10232, "oqpsk", nrzm=True))}
NOISE = 40  # sigma of the pure-noise gaps (soft bytes)


def _bench_max_soft(cfg, n):
    """ChainPipe.max_soft of bench.py for an n-sample step: the decoder's max_soft in the benchmark."""
    import bench

    class _NoChain:  # ChainPipe's constructor sizes the chain; nothing is created
        Chain = staticmethod(lambda dcfg, fcfg: None)
        demod_cfg_for = fec_cfg_for = staticmethod(lambda *a, **k: None)

    return bench.ChainPipe(_NoChain, cfg, n, 0).max_soft


def _step_chunks(cfg, geom):
    """Decoder chunks of the soft bytes of one 2^29-sample step: one soft byte per BPSK symbol, two per QPSK / OQPSK symbol."""
    soft = (1 << LOG2_STEP) * (1 if cfg.constellation == "bpsk" else 2) / (cfg.samplerate / cfg.symbolrate)
    return int(soft) // geom.chunk


@pytest.fixture(scope="module")
def pool():
    with concurrent.futures.ThreadPoolExecutor(max_workers=max(8, os.cpu_count() or 8)) as p:
        yield p


def _timed(f, *a):
    t0 = time.perf_counter()
    r = f(*a)
    return r, time.perf_counter() - t0


@pytest.fixture(scope="module")
def designed(pool):
    """The three designed streams, built in parallel; each one's oracle decode starts as soon as it is built."""
    def job(name):
        (soft, info), t = _timed(_design, name)
        info["t_build"] = t
        return soft, info, pool.submit(_timed, oracle_fec(oracle(), info["cfg"]).run, soft)
    return {name: pool.submit(job, name) for name in KINDS}


# ----------------------------------------------------------------------------------------------------------------- stream builders
def _coded(geom, cfg, nch, seed, noframes=(), rs_bad=(), asm_bad=()):
    """tests/viterbi_model.coded_stream at benchmark size, encoded in blocks: CADUs (frames in `rs_bad` with t + 1 = 17 byte errors in
    their first codeword, frames in `asm_bad` with 16 of the 32 ASM bits flipped), random bits without ASM over the chunk ranges in
    `noframes`, NRZ-M, the k=7 encoder, MetOp puncturing. Returns (coded symbols, the transmitted CADUs)."""
    rng = np.random.default_rng(seed)
    I, cadu = cfg.interleave, cfg.cadu_bytes * 8
    nbits = geom.F * (nch + 1)
    nfr = nbits // cadu + 2
    tx, _ = synth.build_cadus(rng.integers(0, 256, size=(nfr, I * 223), dtype=np.uint8), I)
    for f in rs_bad:
        tx[f, 4 + I * np.arange(17)] ^= rng.integers(1, 256, 17, dtype=np.uint8)
    for f in asm_bad:
        tx[f, :2] ^= 0xFF
    bits = np.unpackbits(tx.reshape(-1))[:nbits]
    for a, b in noframes:
        bits[a * geom.F:b * geom.F] = rng.integers(0, 2, (b - a) * geom.F, dtype=np.uint8)
    if geom.nrzm:
        bits = np.bitwise_xor.accumulate(bits)
    blk = 3 << 22  # (a multiple of 3 bits: whole MetOp puncturing periods)
    out, prev = [], np.zeros(6, np.uint8)
    for a in range(0, bits.size, blk):
        b = bits[a:a + blk]
        coded = synth.conv_encode(np.concatenate([prev, b]))[12:]  # the six bits before the block set the encoder's register
        out.append(synth.puncture_34_metop(coded) if geom.rate34 else coded)
        prev = b[-6:]
    return np.concatenate(out), tx


def _soft(geom, coded, amp, sigma, seed):
    """tests/viterbi_model.soft_stream, vectorised over blocks of chunks: chunk c = coded symbols * amp[c] + N(0, sigma[c]), int8."""
    rng = np.random.default_rng(seed + 1)
    nch, C = amp.size, geom.chunk
    out = np.empty(nch * C, np.int8)
    for c0 in range(0, nch, 1024):
        c1 = min(nch, c0 + 1024)
        x = coded[c0 * C:c1 * C].astype(np.float32) * 2 - 1
        x *= np.repeat(amp[c0:c1], C)
        x += rng.standard_normal(x.size, dtype=np.float32) * np.repeat(sigma[c0:c1], C)
        out[c0 * C:c1 * C] = np.clip(np.rint(x), -127, 127)
    return out


def _design(name, seed=11):
    """The designed stress stream of one benchmark decoder at the chunk count of a 2^29-sample step. Returns (soft, info)."""
    cfg = synth.CONFIGS[name]
    geom = KINDS[name]["geom"]()
    nch = _step_chunks(cfg, geom)
    rng = np.random.default_rng(seed)
    o = cfg.outsync_after
    metop = cfg.decoder == "metop"
    events = ([("weak", int(L)) for L in rng.integers(1, 7, 300)]            # mis-speculated start states, settled by the redo rounds
              + [("weak", int(L)) for L in rng.integers(8, o + 1, 10)]     # lock held; redo chains deeper than six rounds
              + [("weak", int(L)) for L in rng.integers(o + 2, 41, 12)]    # lock lost mid-stretch, searched for again
              + [("noise", int(L)) for L in rng.integers(2, 31, 12)]       # pure noise inserted (lock lost when longer than outsync)
              + ([("noframes", int(L)) for L in rng.integers(12, 26, 8)] if metop else []))  # MetOp: Viterbi reset, rollback
    order = rng.permutation(len(events))
    slot = (nch - 32) // len(events)
    assert slot >= 48, slot
    amp, sigma = np.full(nch, M.GOOD[0], np.float32), np.full(nch, M.GOOD[1], np.float32)
    quiet = np.ones(nch + 2, bool)
    noframes, gaps, weak = [], [], []
    for i, k in enumerate(order):
        what, L = events[k]
        c = 16 + i * slot + int(rng.integers(0, slot - L - 4))
        quiet[c - 1:c + L + 1] = False
        if what == "weak":
            amp[c:c + L], sigma[c:c + L] = M.WEAK
            weak.append((c, L))
        elif what == "noframes":
            noframes.append((c, c + L))
        else:  # (positions and lengths are multiples of 4 soft bytes: an odd offset splits the I/Q pairs, see test_gpu_fec.py)
            gaps.append((c * geom.chunk + 4 * int(rng.integers(0, geom.chunk // 4)), 4 * (L * geom.chunk // 4 + int(rng.integers(0, geom.chunk // 4)))))
    cadu = cfg.cadu_bytes * 8
    rs_bad = []
    for f in rng.permutation(geom.F * nch // cadu - 2):
        if quiet[f * cadu // geom.F:((f + 1) * cadu - 1) // geom.F + 1].all():
            rs_bad.append(int(f))
        if len(rs_bad) == 40:
            break
    coded, _ = _coded(geom, cfg, nch, seed, noframes=noframes, rs_bad=rs_bad)
    sig = _soft(geom, coded, amp, sigma, seed)
    del coded
    nrng = np.random.default_rng(seed + 2)
    pieces, prev = [], 0
    for p, L in sorted(gaps):
        pieces += [sig[prev:p], np.clip(np.rint(nrng.normal(0, NOISE, L)), -127, 127).astype(np.int8)]
        prev = p
    pieces.append(sig[prev:])
    soft = np.concatenate(pieces)[:nch * geom.chunk]
    # a cut inside a WEAK stretch (stream coordinates: the inserted noise in front shifts it) and one a byte after a chunk edge
    c, L = next((c, L) for c, L in weak if L >= 4 and c > nch // 4)
    p = (c + L // 2) * geom.chunk + 1001
    cut1 = p + sum(g for q, g in gaps if q <= p)
    cut2 = (2 * nch // 3) * geom.chunk + 1
    assert cut1 < cut2 < soft.size
    return soft, dict(cfg=cfg, geom=geom, nch=nch, cuts=[cut1, cut2, soft.size], nweak=len(weak), gaps=len(gaps), noframes=len(noframes),
                      rs_bad=len(rs_bad))


# ----------------------------------------------------------------------------------------------------------------- checks
def _push(gcfg, soft, cuts):
    """GPU Fec over soft[prev:cut] for every cut: (bits, CADUs, stats, seconds)."""
    from satdump_b200 import capi
    g = capi.Fec(gcfg)
    bits, frames, prev = [], [], 0
    t0 = time.perf_counter()
    for c in cuts:
        g.push(soft[prev:c])
        bits.append(g.bits())
        frames.append(g.frames().reshape(-1))
        prev = c
    dt = time.perf_counter() - t0
    s = g.stats()
    g.close()
    return np.concatenate(bits), np.concatenate(frames), s, dt


def _check(want, bits, frames, s):
    assert bits.size == want["bits"].size and np.array_equal(bits, want["bits"])
    assert frames.size == want["cadu"].size and np.array_equal(frames, want["cadu"])
    assert s["viterbi_state"] == int(want["vit_state"][-1])
    assert s["deframer_state"] == int(want["defr_state"][-1])
    ok = want["rs_err"][want["rs_err"] >= 0]
    assert s["rs_corrected"] == int(ok.sum()) and s["rs_failed"] == int((want["rs_err"] < 0).sum())


def _resets(want):
    """viterbi.reset() calls of metop_ahrpt_decoder (module_metop_ahrpt_decoder.cpp:59-72): the tenth decoded chunk in a row that ends
    with the deframer in NOSYNC (2). A chunk is decoded when the Viterbi is locked on it or was locked on the chunk before (the chunk
    that loses the lock still has its bits); chunks searched for the lock leave the count alone. (A lock search that fails right after
    a reset would count one chunk too many: the count is an upper bound.)"""
    vs, runs, out = want["vit_state"], 0, []
    for c, st in enumerate(want["defr_state"]):
        if not (vs[c] == 1 or (c > 0 and vs[c - 1] == 1)):
            continue
        runs = runs + 1 if st == 2 else 0
        if runs >= 10:
            out.append(c)
            runs = 0
    return out


@pytest.mark.parametrize("name", list(KINDS))
def test_designed_stress_at_bench_chunk_count(built, designed, name):
    """One push of the chunk count of a 2^29-sample step, bit-exact with the oracle, with every correction path run at scale: >= 100
    start states redone, >= 20 chunks chained back serially, at least one redo-round fallback, >= 10 losses and regains of the lock,
    (MetOp) >= 5 Viterbi resets rolled back, RS failures. Then the same stream in three ragged pushes."""
    from satdump_b200 import capi
    soft, info, job = designed[name].result()
    cfg, geom, nch = info["cfg"], info["geom"], info["nch"]
    max_soft = _bench_max_soft(cfg, 1 << LOG2_STEP)
    assert soft.size == nch * geom.chunk <= max_soft
    gcfg = capi.fec_cfg_for(cfg, max_soft)
    g = capi.Fec(gcfg)
    assert g.chunk == geom.chunk
    g.close()
    bits, frames, s, dt = _push(gcfg, soft, [soft.size])
    bits3, frames3, s3, dt3 = _push(gcfg, soft, info["cuts"])
    want, t_oracle = job.result()
    vs = want["vit_state"]
    losses, regains = int(((vs[:-1] == 1) & (vs[1:] == 0)).sum()), int(((vs[:-1] == 0) & (vs[1:] == 1)).sum())
    resets = _resets(want) if cfg.decoder == "metop" else []
    # replays = start states redone + serial chainbacks + redo-round fallbacks + MetOp rollbacks (at most one per reset)
    fallback = s["replays"] - s["start_redone"] - s["tb_serial"] - len(resets)
    print(f"\n{name}: {nch} chunks of {geom.chunk} soft bytes in one push ({info['nweak']} WEAK stretches, {info['gaps']} noise gaps, "
          f"{info['noframes']} runs without frames, {info['rs_bad']} frames with t+1 errors); counters",
          {k: s[k] for k in ("start_redone", "tb_serial", "replays", "spec_steps", "tb_overlap", "rs_corrected", "rs_failed")},
          f"fallbacks >= {fallback}, lock losses {losses}, regains {regains}, MetOp resets {len(resets)}, frames {want['nframes']}; "
          f"build {info['t_build']:.1f} s, GPU one push {dt:.2f} s, three pushes {dt3:.2f} s, oracle {t_oracle:.1f} s")
    _check(want, bits, frames, s)
    assert s["start_redone"] >= 100 and s["tb_serial"] >= 20 and fallback >= 1
    assert losses >= 10 and regains >= 10
    assert s["rs_failed"] >= 1
    if cfg.decoder == "metop":
        assert len(resets) >= 5
    _check(want, bits3, frames3, s3)


def test_bench_workload_at_stress_snr(built, pool):
    """bench.py's c3 workload (MetOp AHRPT, generated on the device the way the benchmark makes it) at 5.5 dB and 2^28 samples: the soft
    bytes of one standalone demodulator push, decoded by one Fec push, equal the oracle's decode; the chain run synchronously, and
    pipelined the way the benchmark's timed loop runs it (reset, push, pull per step, then sync), gives the oracle's CADUs in every step.
    The main Viterbi launches of each synchronous step decode every chunk after the first lock."""
    import ctypes

    import torch
    from satdump_b200 import capi, shard
    cfg = dataclasses.replace(synth.CONFIGS["metop_ahrpt"], esn0_db=5.5)
    raw, _ = synth.make_signal(cfg, 1 << 28, seed=shard.stream_seed(3, 0), device="cuda")
    n = raw.numel() // 2
    torch.cuda.synchronize()
    d = capi.Demod(capi.demod_cfg_for(cfg, n))
    d.push_device(raw.data_ptr(), n)
    soft = d.soft()
    d.close()
    job = pool.submit(oracle_fec(oracle(), cfg).run, soft)
    max_soft = _bench_max_soft(cfg, n)
    gcfg = capi.fec_cfg_for(cfg, max_soft)
    bits, frames, s, _ = _push(gcfg, soft, [soft.size])
    ch = capi.Chain(capi.demod_cfg_for(cfg, n), capi.fec_cfg_for(cfg, max_soft))
    sync_frames, vit = [], []
    for _ in range(2):
        ch.reset()
        ch.push_device(raw.data_ptr(), n)
        sync_frames.append(ch.frames().reshape(-1))
        vit.append(int(ch.timing()["vit_chunks"]))
    steps = 3
    ch.set_pipelined(True)
    out = np.zeros(steps * (frames.size + (1 << 20)), np.uint8)
    got = 0
    for _ in range(steps):
        ch.reset()
        ch.push_device(raw.data_ptr(), n)
        got += ch.pull_into(out.ctypes.data + got, out.size - got)
    ch.sync()
    while True:
        nb = ch.pull_into(out.ctypes.data + got, out.size - got)
        if nb == 0:
            break
        got += nb
    ch.set_pipelined(False)
    ch.close()
    want = job.result()
    nch = soft.size // 16384
    lead = int(np.argmax(want["vit_state"] == 1))
    print(f"\nc3 at 5.5 dB, 2^28 samples: {soft.size} soft bytes = {nch} chunks, {lead} before the first lock (lock search); vit_chunks per "
          f"synchronous step {vit}; frames {want['nframes']}, counters", {k: s[k] for k in ("start_redone", "tb_serial", "replays", "rs_corrected", "rs_failed")})
    _check(want, bits, frames, s)
    assert want["nframes"] > 10000 and s["rs_corrected"] > 0
    for f in sync_frames:
        assert np.array_equal(f, want["cadu"])
    assert got == steps * want["cadu"].size
    assert np.array_equal(out[:got].reshape(steps, -1), np.tile(want["cadu"], (steps, 1)))
    # every chunk after the first lock goes through the main launches; exactly once when the lock holds and every redo settles
    assert vit[0] == vit[1] >= nch - lead
    if (want["vit_state"][lead:] == 1).all() and s["replays"] == s["start_redone"] + s["tb_serial"]:
        assert vit[0] == nch - lead


def _asm_damaged_soft(cfg, geom, nch, seed):
    """All-GOOD coded stream whose frames 3, 7, 11, ... (from frame 16 on) carry 16 flipped ASM bits: the SYNCED test (< 12 differing
    bits) and the SYNCING test (< 6) both fail there, so the deframer falls to NOSYNC, finds the next exact ASM, and needs 11 good ASMs in
    a row to be SYNCED again, which it never reaches."""
    nfr = geom.F * (nch + 1) // (cfg.cadu_bytes * 8) + 2
    bad = [f for f in range(16, nfr) if f % 4 == 3]
    coded, tx = _coded(geom, cfg, nch, seed, asm_bad=bad)
    return _soft(geom, coded, np.full(nch, M.GOOD[0], np.float32), np.full(nch, M.GOOD[1], np.float32), seed), tx


def test_deframer_event_list_at_scale(built, pool):
    """One ASM in four damaged, in a c2-shaped push at the chunk count of a 2^29-sample step (about 6 500 deframer state changes), and in
    a ccsds_simple_psk_decoder BPSK stream of raw soft bits: both equal the oracle. The frame list and the number of state changes come
    also from tests/rs_model.py's bit-serial deframer run over the oracle's bits."""
    from satdump_b200 import capi
    cfg = synth.CONFIGS["bpsk_half"]
    geom = KINDS["bpsk_half"]["geom"]()
    nch = _step_chunks(cfg, geom)
    max_soft = _bench_max_soft(cfg, 1 << LOG2_STEP)
    soft, _ = _asm_damaged_soft(cfg, geom, nch, 5)
    assert soft.size <= max_soft
    job = pool.submit(oracle_fec(oracle(), cfg).run, soft)
    # the simple decoder's input: the same frames and damage as hard bits + noise, one soft byte per bit (chunk = cadu_size bytes)
    rng = np.random.default_rng(6)
    nfr = 16384
    tx, _ = synth.build_cadus(rng.integers(0, 256, size=(nfr, 4 * 223), dtype=np.uint8), 4)
    tx[[f for f in range(16, nfr) if f % 4 == 3], :2] ^= 0xFF
    lead = rng.integers(0, 2, 3001, dtype=np.uint8)
    sbits = np.concatenate([lead, np.unpackbits(tx.reshape(-1))])[:(nfr - 1) * 8192]
    ssoft = np.clip(np.rint((sbits.astype(np.float32) * 2 - 1) * 60 + rng.standard_normal(sbits.size, dtype=np.float32) * 20), -127, 127).astype(np.int8)
    O = oracle()
    sjob = pool.submit(O.Fec(O.simple_cfg("bpsk", 8192, 4)).run, ssoft)
    bits, frames, s, dt = _push(capi.fec_cfg_for(cfg, max_soft), soft, [soft.size])
    sbits_g, sframes, ss, _ = _push(capi.simple_cfg("bpsk", 8192, 4, max_soft=ssoft.size), ssoft, [ssoft.size])
    want, swant = job.result(), sjob.result()
    model = rs_model.deframe(want["bits"], 8192)
    smodel = rs_model.deframe(swant["bits"], 8192)
    print(f"\nASM damage: c2 push of {nch} chunks, {want['nframes']} frames, {len(model['events'])} deframer state changes (GPU {dt:.2f} s); "
          f"simple BPSK {ssoft.size} soft bytes, {swant['nframes']} frames, {len(smodel['events'])} state changes")
    _check(want, bits, frames, s)
    assert np.array_equal(sbits_g, swant["bits"]) and np.array_equal(sframes, swant["cadu"])
    assert ss["deframer_state"] == int(swant["defr_state"][-1])
    for m, w in ((model, want), (smodel, swant)):
        assert len(m["events"]) > 4096 and m["asm_end"].size == w["nframes"]
