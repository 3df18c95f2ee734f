"""GPU: ccsds_ldpc_decoder (rate 7/8 C2 code) parity. Correlator scores, the frame walk, the phase fix and the min-sum decoder are all
exact: given a soft stream, the CUDA path must reproduce the reference's CADUs, every frame's (offset, pos, correlator_corr, phase, swap,
ldpc_corr) and the module statistics bit for bit; with internal_stream the inner frames and the deframer state. End to end (IQ ->
psk_demod -> LDPC) through the fused chain and the C++ module layer the CADUs equal the reference's and the transmitted ones."""
import numpy as np
import pytest

from oracle import ldpc as O
from satdump_b200 import synth
from tests.common import match_frames, run_chain, run_cli

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def oracle_built(built):
    if not (O.available("ref") or O.available("port")):
        import __graft_entry__ as g
        g.build()
    return True


def stream(constellation, nframes=12, sigma=20.0, rot=0, q_late=False, seed=3, lead=2000, tail=3000):
    """Soft stream: `lead` random bits, nframes C2 frames, `tail` random bits. Returns (soft, the CADUs of the transmitted frames)."""
    rng = np.random.default_rng(seed + 100)
    tx, _, cadu = synth.ldpc_frames(nframes, seed)
    bits = np.concatenate([rng.integers(0, 2, lead, dtype=np.uint8), tx.reshape(-1), rng.integers(0, 2, tail, dtype=np.uint8)])
    return synth.ldpc_soft(bits, constellation, sigma=sigma, rot=rot, q_late=q_late, seed=seed), cadu


def gpu(constellation, iterations=10, max_soft=1 << 20, derandomize=True):
    from satdump_b200 import capi
    return capi.Fec(capi.ldpc_cfg(constellation, ldpc_iterations=iterations, derandomize=derandomize, max_soft=max_soft))


def check(constellation, soft, iterations=10, cuts=None):
    """GPU (one push, or pushes at `cuts`) against the oracle on the same stream; returns the oracle's result."""
    want = O.Fec(O.ldpc_cfg(constellation, iterations)).run(soft)
    g = gpu(constellation, iterations, max_soft=max(1 << 16, soft.size))
    cuts = [0] + list(cuts or []) + [soft.size]
    frames, recs = [], []
    for a, b in zip(cuts[:-1], cuts[1:]):
        g.push(soft[a:b])
        frames.append(g.frames())
        recs.append(g.ldpc_frames())
    got, grec = np.concatenate(frames), np.concatenate(recs)
    assert got.shape == want["cadu"].shape, (got.shape, want["cadu"].shape)
    assert np.array_equal(grec, want["recs"][:, :7]), (grec[:4], want["recs"][:4])
    assert np.array_equal(got, want["cadu"])
    if want["recs"].shape[0]:
        s, last = g.stats(), want["recs"][-1]
        assert s["correlator_lock"] == last[6] and s["ldpc_corr"] == last[5]
        assert np.float32(s["correlator_corr"]).view(np.uint32) == np.uint32(last[2])
        assert s["ldpc_resyncs"] == int((want["recs"][:, 1] != 0).sum()) and s["frames_out"] == want["recs"].shape[0]
    return want


@pytest.mark.parametrize("constellation", ["bpsk", "qpsk", "oqpsk"])
@pytest.mark.parametrize("sigma", [0.0, 29.0])
def test_decoder_alone_bit_exact(oracle_built, constellation, sigma):
    """Clean input, and a noise level at which some codewords do not converge in 10 iterations."""
    soft, clear = stream(constellation, sigma=sigma, rot=1 if constellation == "oqpsk" else 0)
    want = check(constellation, soft)
    n = want["cadu"].shape[0]
    assert n >= 12
    ok = sum(np.array_equal(want["cadu"][k], clear[k]) for k in range(min(n, 12)))
    if sigma == 0:
        assert ok == 12
    else:
        assert ok < 12, "the noisy case should leave codewords unconverged"


@pytest.mark.parametrize("iterations", [0, 1, 50])
def test_iteration_counts(oracle_built, iterations):
    soft, _ = stream("qpsk", nframes=6, sigma=27.0)
    check("qpsk", soft, iterations=iterations)


@pytest.mark.parametrize("constellation,rot,q_late", [("bpsk", 2, False)] + [("qpsk", r, False) for r in range(1, 4)] +
                         [("oqpsk", r, q) for r in range(4) for q in (False, True)])
def test_every_phase_ambiguity(oracle_built, constellation, rot, q_late):
    """Streams rotated by 90, 180 and 270 degrees, and OQPSK with Q on the wrong symbol. The phase fix is the reference's whatever it
    finds; where the reference's tables resolve the ambiguity (BPSK, QPSK; OQPSK at 90 / 270 degrees with Q on time, and at 0 / 180 degrees
    with Q late) the frames are the transmitted ones."""
    soft, clear = stream(constellation, nframes=6, sigma=15.0, rot=rot, q_late=q_late)
    want = check(constellation, soft)
    resolvable = constellation != "oqpsk" or (rot % 2 == 1) != q_late
    if resolvable:
        assert np.array_equal(want["cadu"][:6], clear), "the reference should resolve this ambiguity"


def test_inserted_and_deleted_soft_bytes(oracle_built):
    """Bytes inserted and deleted mid-stream force pos != 0 on the next frame; the walk continues on the shifted lattice."""
    soft, _ = stream("qpsk", nframes=14, sigma=18.0)
    F = 8192
    s = np.concatenate([soft[:2000 + 3 * F + 100], np.full(314, 5, np.int8), soft[2000 + 3 * F + 100:2000 + 7 * F + 50],
                        soft[2000 + 7 * F + 50 + 1000:]])
    want = check("qpsk", s)
    assert (want["recs"][1:, 1] != 0).sum() >= 2


def test_noise_lead_and_noise_signal_noise(oracle_built):
    """A leading stretch of noise whose length is not a multiple of F, then noise -> signal -> noise: every noise frame shifts."""
    rng = np.random.default_rng(11)
    noise = lambda n: np.clip(np.round(rng.normal(0, 40, n)), -127, 127).astype(np.int8)
    soft, _ = stream("bpsk", nframes=8, sigma=15.0, lead=0, tail=0)
    s = np.concatenate([noise(3 * 8192 + 1234), soft, noise(4 * 8192 + 77), soft[:5 * 8192]])
    want = check("bpsk", s)
    assert (want["recs"][:, 1] != 0).sum() >= 4 and (want["recs"][:, 6] == 1).sum() >= 6


def test_ragged_pushes(oracle_built):
    """Arbitrary cut points (inside the ASM, mid-codeword, a push shorter than a frame) are bit-identical to one push."""
    soft, _ = stream("oqpsk", nframes=10, sigma=20.0, rot=3)
    cuts = [1, 2000 + 8, 2000 + 8192 + 4000, 2000 + 8192 + 4100, 2000 + 3 * 8192 + 17, 2000 + 6 * 8192 - 9]
    check("oqpsk", soft, cuts=cuts)


def test_derandomize_off(oracle_built):
    soft, _ = stream("qpsk", nframes=4, sigma=10.0)
    want = O.Fec(O.ldpc_cfg("qpsk", 10, derandomize=False)).run(soft)
    g = gpu("qpsk", derandomize=False).push(soft)
    assert np.array_equal(g.frames(), want["cadu"]) and want["cadu"].shape[0] == 4


def test_large_push_matches_transmitted_frames(oracle_built):
    """Several hundred codewords in one push (many lattice rounds of the walk and many CTAs of the decoder)."""
    tx, _, clear = synth.ldpc_frames(300, 21)
    soft = synth.ldpc_soft(np.concatenate([np.zeros(6, np.uint8), tx.reshape(-1)]), "qpsk", sigma=18.0, seed=4)
    g = gpu("qpsk", max_soft=soft.size + 65536)
    got = g.push(soft).frames()
    assert np.array_equal(got, clear[:got.shape[0]]) and got.shape[0] >= 299
    t = g.timing()
    assert t["push"] > 0 and t["decode"] > 0


@pytest.mark.parametrize("name,constellation,cadu_size,asm", [("landsat", "oqpsk", 8272, 0x352EF853), ("iris", "oqpsk", 14304, 0x1ACFFC1D),
                                                              ("qpsk_8272", "qpsk", 8272, 0x352EF853)])
def test_internal_stream(oracle_built, name, constellation, cadu_size, asm):
    """internal_stream: the 7136 info bits of every codeword through BPSK_CCSDS_Deframer(internal_cadu_size, internal_asm). Inner frames and
    the deframer state equal the reference's, in one push and in ragged pushes; the frames are the transmitted inner frames."""
    from satdump_b200 import capi
    nfr = 30
    info, inner = synth.ldpc_inner_frames(nfr, cadu_size, asm, 5)
    tx, _, _ = synth.ldpc_frames(nfr, 5, info=info)
    rng = np.random.default_rng(6)
    bits = np.concatenate([rng.integers(0, 2, 1000, dtype=np.uint8), tx.reshape(-1)])
    soft = synth.ldpc_soft(bits, constellation, sigma=15.0, rot=1 if constellation == "oqpsk" else 0, seed=7)
    want = O.Fec(O.ldpc_cfg(constellation, 10, internal_cadu_size=cadu_size, internal_asm=asm)).run(soft)
    assert want["cadu"].shape[0] >= inner.shape[0] - 2
    i0 = next(i for i in range(inner.shape[0]) if np.array_equal(inner[i], want["cadu"][0]))
    assert np.array_equal(want["cadu"], inner[i0:i0 + want["cadu"].shape[0]])
    for cuts in ([], [3000, 3000 + 8192 * 4 + 77, soft.size // 2 + 1]):
        g = capi.Fec(capi.ldpc_cfg(constellation, internal_stream=True, internal_cadu_size=cadu_size, internal_asm=asm, max_soft=1 << 20))
        assert g.cadu_bytes == cadu_size // 8
        parts, prev = [], 0
        for c in cuts + [soft.size]:
            parts.append(g.push(soft[prev:c]).frames())
            prev = c
        got = np.concatenate(parts)
        assert got.shape == want["cadu"].shape and np.array_equal(got, want["cadu"])
        st = g.stats()
        assert st["deframer_state"] == want["recs"][-1, 7] and st["frames_out"] == want["cadu"].shape[0]
        assert (want["recs"][:, 7] == 12).any(), "the deframer should reach SYNCED"
        assert st["correlator_lock"] == want["recs"][-1, 6] and st["ldpc_corr"] == want["recs"][-1, 5]


def _oracle_chain(cfg, raw):
    """the reference: psk_demod's soft symbols -> ccsds_ldpc_decoder"""
    from tests.common import oracle, oracle_demod
    soft = oracle_demod(oracle(), cfg).run(raw, stages=False)["soft"]
    return O.Fec(O.ldpc_cfg(cfg.constellation, 10, internal_cadu_size=cfg.internal_cadu_size, internal_asm=cfg.internal_asm)).run(soft)["cadu"]


@pytest.mark.parametrize("name", ["ldpc_qpsk", "ldpc_landsat"])
@pytest.mark.parametrize("pipelined", [False, True])
def test_fused_chain_end_to_end(oracle_built, name, pipelined):
    """IQ -> psk_demod -> ccsds_ldpc_decoder through the fused chain, synchronous and pipelined, in several pushes: the CADUs (LandSat-like:
    the inner frames) equal the reference's and, once the demodulator has locked, the transmitted ones."""
    from satdump_b200 import capi
    from tests.common import signal
    cfg, raw, clear = signal(name, 20, seed=3)
    want = _oracle_chain(cfg, raw)
    n = raw.size // 2
    got, _ = run_chain(capi.demod_cfg_for(cfg, max_batch=n), capi.fec_cfg_for(cfg, max_soft=4 * n), raw, cfg.fmt, pipelined)
    assert got.shape[0] >= 5 and got.shape == want.shape
    same_after_lock(got, want, clear)


def same_after_lock(got, want, clear):
    """The first LDPC windows are read while the demodulator's loops still acquire: their soft bytes sit on the float floor of the
    demodulator (DESIGN §5), and a codeword that does not converge depends on every one of them. From the third frame on, the frames are
    the reference's and the transmitted ones."""
    assert np.array_equal(got[2:], want[2:])
    i0, ok = match_frames(got[2:], clear)
    assert ok, "the CADUs should be the transmitted frames"


@pytest.mark.parametrize("pipe,name", [("ldpc_qpsk", "ldpc_qpsk"), ("landsat", "ldpc_landsat")])
@pytest.mark.parametrize("mode", ["two_stage", "fused"])
def test_cli_module_layer(oracle_built, tmp_path, pipe, name, mode):
    """The C++ module layer with module id ccsds_ldpc_decoder (parameters parsed as CCSDSLDPCDecoderModule's constructor), as the CLI
    runs it: the .cadu file holds the reference's frames."""
    from tests.common import signal
    cfg, raw, clear = signal(name, 20, seed=4)
    inp = tmp_path / "in.raw"
    raw.tofile(inp)
    want = _oracle_chain(cfg, raw)
    hint = str(tmp_path / "out")
    run_cli(pipe, inp, hint, "--samplerate", str(cfg.samplerate), "--symbolrate", str(int(cfg.symbolrate)), "--baseband_format", cfg.fmt,
            fused=mode == "fused")
    got = np.fromfile(hint + ".cadu", np.uint8).reshape(-1, cfg.cadu_bytes)
    assert got.shape[0] >= 5 and got.shape == want.shape
    same_after_lock(got, want, clear)
