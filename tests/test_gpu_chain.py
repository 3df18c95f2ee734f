"""GPU: the fused chain (raw IQ -> CADUs, soft stream kept in HBM) end to end: CADUs bit-exact vs the oracle's end to end run
at oracle-sized inputs, and size-independent properties at BASELINE-sized inputs."""
import numpy as np
import pytest

from tests.common import gpu_chain, match_frames, nsamples, oracle, oracle_demod, oracle_fec, signal

pytestmark = pytest.mark.gpu
DECODED = ["metop_ahrpt", "bpsk_half", "jpss_hrd", "hrpt_bpsk", "metop_oversampled", "bpsk_decim8", "bpsk_simple", "qpsk_simple"]


@pytest.mark.parametrize("name", DECODED)
def test_cadus_bit_exact_vs_oracle(built, name):
    O = oracle()
    cfg, raw, clear = signal(name, 22)
    n = nsamples(raw, cfg)
    soft = oracle_demod(O, cfg).run(raw, stages=False)["soft"]
    want = oracle_fec(O, cfg).run(soft)["cadu"].reshape(-1, cfg.cadu_bytes)
    ch = gpu_chain(cfg, n).push(raw)
    got = ch.frames()
    assert want.shape[0] >= 5
    assert got.shape == want.shape and np.array_equal(got, want)
    ds, fs = ch.stats()
    assert ds["costas_unconverged"] == 0 and ds["mm_unconverged"] == 0 and fs["replays"] == 0
    assert ds["kernel_launches"] > 0 and fs["kernel_launches"] > 0


@pytest.mark.parametrize("name", DECODED)
def test_streaming_batches_bit_exact(built, name):
    O = oracle()
    cfg, raw, _ = signal(name, 22)
    n = nsamples(raw, cfg)
    per = 1 if cfg.fmt == "cf32" else 2
    soft = oracle_demod(O, cfg).run(raw, stages=False)["soft"]
    want = oracle_fec(O, cfg).run(soft)["cadu"].reshape(-1, cfg.cadu_bytes)
    ch = gpu_chain(cfg, n)
    cuts = [0, n // 5 + 3, n // 2 + 1001, n]
    got = np.concatenate([ch.push(raw[a * per:b * per]).frames() for a, b in zip(cuts[:-1], cuts[1:])])
    # batching only moves where the soft stream is cut into decoder chunks relative to symbol production, not its content
    assert got.shape == want.shape and np.array_equal(got, want)


def test_low_snr_end_to_end(built):
    """5.5 dB: RS does real work. The soft bytes differ from the oracle's by +-1 LSB on a fraction of a percent (M&M arm
    choice), so CADU bit-exactness here rests on the Viterbi/RS margin — the survey's 'stress case', reported separately."""
    O = oracle()
    cfg, raw, clear = signal("metop_ahrpt", 22, seed=3, esn0=5.5)
    n = nsamples(raw, cfg)
    soft = oracle_demod(O, cfg).run(raw, stages=False)["soft"]
    want = oracle_fec(O, cfg).run(soft)["cadu"].reshape(-1, 1024)
    got = gpu_chain(cfg, n).push(raw).frames()
    assert got.shape == want.shape
    # message part (bytes 4..895 of each interleaved codeword set) is RS corrected on both sides: must be identical
    same_rows = (got[:, :4 + 223 * 4] == want[:, :4 + 223 * 4]).all(axis=1).mean()
    assert same_rows >= 0.98, same_rows
    first, ok = match_frames(got[:, :4 + 223 * 4], clear[:, :4 + 223 * 4])
    assert first is not None


def test_baseline_size_properties(built):
    """2^26 samples (11 s of MetOp signal): no oracle run at this size; every CADU must be one of the transmitted frames, in
    order, none missing after the first lock (encode -> channel -> decode round trip)."""
    cfg, raw, clear = signal("metop_ahrpt", 26, seed=21)
    n = nsamples(raw, cfg)
    ch = gpu_chain(cfg, n).push(raw)
    got = ch.frames()
    first, ok = match_frames(got, clear)
    assert ok and first is not None and first <= 4
    expected = int(n * 2 * 0.75 / (cfg.samplerate / cfg.symbolrate) / 8192)
    assert got.shape[0] >= expected - 6, (got.shape[0], expected)
    ds, fs = ch.stats()
    assert ds["costas_unconverged"] == 0 and ds["mm_unconverged"] == 0 and fs["rs_failed"] == 0
    t = ch.timing()
    assert t["push_events"] > 0 and t["k_vit_acs"] > 0


def test_reset_starts_a_new_stream(built):
    """One decoder of each kind (MetOp, CCSDS r=1/2, punctured, two deframers, NRZ-M): reset() after an odd-length part of another
    signal, i.e. mid-frame and mid-lock, and the next stream gives exactly the frames of a fresh chain."""
    from satdump_b200 import capi
    from tests.common import demod_kwargs
    for name in ["metop_ahrpt", "bpsk_half", "qpsk_p34", "qpsk_simple", "bpsk_simple"]:
        cfg, raw, _ = signal(name, 21)
        _, other, _ = signal(name, 21, seed=2)
        n = nsamples(raw, cfg)
        per = 1 if cfg.fmt == "cf32" else 2

        def chain():
            return capi.Chain(capi.demod_cfg(max_batch=n, **demod_kwargs(cfg)), capi.fec_cfg_for(cfg, 2 * n))

        want = chain().push(raw).frames()
        ch = chain()
        lead = (n // 2) | 1
        assert ch.push(other[:lead * per]).frames().shape[0] > 0, name
        ch.reset()
        got = ch.push(raw).frames()
        assert want.shape[0] > 0 and got.shape == want.shape and np.array_equal(got, want), name


def test_prefetched_host_batches_equal_plain_pushes(built):
    """b200_chain_prefetch_iq double buffering (H2D of batch i+1 under the kernels of batch i) must not change the stream."""
    import torch
    cfg, raw, _ = signal("metop_ahrpt", 22)
    n = nsamples(raw, cfg)
    want = gpu_chain(cfg, n).push(raw).frames()
    pinned = torch.from_numpy(raw).pin_memory()
    half = (n // 2) // 16 * 16
    p0, p1 = pinned.data_ptr(), pinned.data_ptr() + half * 4
    ch = gpu_chain(cfg, n)
    ch.prefetch_ptr(p0, half)
    ch.prefetch_ptr(p1, n - half)
    a = ch.push_ptr(p0, half).frames()
    b = ch.push_ptr(p1, n - half).frames()
    got = np.concatenate([a, b])
    assert got.shape == want.shape and np.array_equal(got, want)


@pytest.mark.parametrize("name", ["metop_ahrpt", "jpss_hrd"])
def test_pipelined_mode_gives_the_same_frames(built, name):
    """Decoder on its worker thread, one batch behind the demodulator: same CADUs, in order; frames of a push become pullable only
    once that batch is decoded; sync() drains; switching back to the synchronous mode continues the same stream."""
    O = oracle()
    cfg, raw, _ = signal(name, 22)
    n = nsamples(raw, cfg)
    per = 1 if cfg.fmt == "cf32" else 2
    soft = oracle_demod(O, cfg).run(raw, stages=False)["soft"]
    want = oracle_fec(O, cfg).run(soft)["cadu"].reshape(-1, cfg.cadu_bytes)
    ch = gpu_chain(cfg, n).set_pipelined(True)
    cuts = [0, n // 7, n // 3 + 5, n // 2, (3 * n) // 4 + 77, n]
    parts = []
    for k, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        if k == 3:  # mode switches drain the decoder and keep the stream
            ch.set_pipelined(False)
        if k == 4:
            ch.set_pipelined(True)
        ch.push(raw[a * per:b * per])
        parts.append(ch.frames())
    ch.sync()
    parts.append(ch.frames())
    got = np.concatenate(parts)
    assert got.shape == want.shape and np.array_equal(got, want)
    ds, fs = ch.stats()
    assert fs["frames_out"] == want.shape[0] and ds["samples_in"] == n
    ch.close()


def test_pipelined_decoder_errors_surface(built):
    """A decoder-side failure on the worker thread (decoded frames piling up because nobody pulls them: the chain sizes the soft FIFO
    itself now, so that cannot be provoked any more) is reported by a later call, not lost."""
    from satdump_b200 import capi
    cfg, raw, _ = signal("metop_ahrpt", 20)
    n = nsamples(raw, cfg)
    ch = capi.Chain(capi.demod_cfg(cfg.samplerate, cfg.symbolrate, cfg.constellation, cfg.rrc_alpha, cfg.pll_bw, cfg.fmt, max_batch=n),
                    capi.metop_cfg(cfg.ber_thresold, cfg.outsync_after, max_soft=65536)).set_pipelined(True)
    with pytest.raises(capi.B200Error) as e:
        for _ in range(8):  # the frame store holds two batches' worth
            ch.push(raw)
        ch.sync()
    assert e.value.code == -5
    ch.close()
