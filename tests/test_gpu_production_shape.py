"""GPU: the demodulator's production kernels, sample by sample, at the geometries large pushes run.

`keep_stages` switches the front end to the dumping instantiation of `k_agc_fir_w`, which runs its general per-chunk body only; the
branch-free body with the raw prefetch one chunk ahead runs only when nothing is dumped. `b200_demod_debug_shape` (capi
`Demod.debug_shape`) lets a push keep that production body's RRC output (`keep_front`) and forces the two geometries that otherwise
depend on the push size:

- R, the tiles per range of `k_agc_fir_w`: max(4, ceil(tiles / resident warps)). The floor of 4 only amortises the walk back that
  proves a range's start gain; any R >= 1 computes the same stream, so R = 1 is tested too.
- L, the segment length of the loop kernels (`choose_L`): clamp(ceil(n / (SMs x 2 x 128)), 4096, 16384), rounded up to 16.

At the benchmark's 2^29 samples a 132-SM H100 SXM runs L = 15 888 and, with 8 resident `k_agc_fir_w` CTAs of 4 warps per SM
(64 registers per thread bound it; 11.5 KB of shared memory per CTA), R = ceil(262 144 / 4 224) = 63 tiles; `test_benchmark_sized_push`
asserts L and R > 4 from the hook and records R. A 114-SM H100 PCIe clamps L to 16 384, which `test_segment_lengths` covers.

Every row asserts the R / L it ran from what the handle reports, so a hook that were ignored fails there rather than passing at
R = 4 / L = 4096. Gates are those of tests/test_gpu_demod.py; the floors of tests/floors.py depend only on the reference and the signal,
so the cached 2^21 floors hold at any forced R or L."""
import numpy as np
import pytest

from tests.common import demod_kwargs, nsamples, oracle, signal
from tests.floors import CONFIGS, GX, SURVEY, cached, gate
from tests.test_gpu_demod import check_costas, check_mm

pytestmark = pytest.mark.gpu
LG = 21
N = 1 << LG


def _capi():
    from satdump_b200 import capi
    return capi


def derive(raw, fmt):
    """The samples of a cs16 fixture in another format: cf32 as the reference converts cs16 (x / 32767), cs8 the top byte."""
    if fmt == "cs16":
        return raw
    if fmt == "cf32":
        v = raw.astype(np.float32) / np.float32(32767)
        return (v[0::2] + 1j * v[1::2]).astype(np.complex64)
    return np.clip(raw.astype(np.int32) >> 8, -128, 127).astype(np.int8)


def per_sample(fmt):
    return 1 if fmt == "cf32" else 2


def gpu(cfg, n, fmt=None, range_tiles=0, seg_len=0, keep_front=True, keep_stages=False, **kw):
    capi = _capi()
    k = demod_kwargs(cfg)
    if fmt:
        k["fmt"] = fmt
    d = capi.Demod(capi.demod_cfg(max_batch=max(n, 4096), keep_stages=keep_stages, **k, **kw))
    if not keep_stages:
        d.debug_shape(range_tiles, seg_len, keep_front)
    elif range_tiles or seg_len:
        d.debug_shape(range_tiles, seg_len, False)
    return d


def reference(cfg, raw, fmt=None, stages=True, **kw):
    """The oracle's stage outputs for raw and its loop state after it."""
    O = oracle()
    k = demod_kwargs(cfg)
    if fmt:
        k["fmt"] = fmt
    od = O.Demod(O.demod_cfg(**k, **kw))
    o = od.run(raw, stages=stages)
    return o, od.state()


def gain_matches(stats, st):
    """The AGC gain after the push, within the bound test_stage_parity uses: the reference's own gain drifts by float rounding."""
    return abs(stats["agc_gain"] - st["gain"]) <= 1e-4 * st["gain"]


# ---------------------------------------------------------------------------------------------------------------- 1. production body
FRONT = [(name, None) for name in CONFIGS] + [("metop_ahrpt", "cf32"), ("metop_ahrpt", "cs8")]


@pytest.mark.parametrize("name,fmt", FRONT, ids=[f"{n}-{f or 'native'}" for n, f in FRONT])
def test_production_front_body(built, name, fmt):
    """The branch-free body of k_agc_fir_w (prefetch one chunk ahead, conversion scale carried in the gain, walk-back seeds with the
    AGC on) within 1e-5 of the reference on every sample, and BITWISE the dumping body's output of the same samples: both start from the
    same seeds and run the same per-sample operations (the scale is a power of two, so every product and sum rounds alike)."""
    cfg, raw, _ = signal(name, LG)
    if fmt:
        assert cfg.fmt == "cs16"
        raw = derive(raw, fmt)
    n = raw.size // per_sample(fmt or cfg.fmt)
    o, st = reference(cfg, raw, fmt)
    g = gpu(cfg, n, fmt).push(raw)
    s = g.stats()
    assert s["last_range_tiles"] == 4 and s["agc_exact_passes"] == 0 and s["agc_clamped"] == 0, s
    fir = g.stage("fir")
    dump = gpu(cfg, n, fmt, keep_stages=True).push(raw)
    d = np.abs(fir - o["fir"])
    same = np.array_equal(fir.view(np.uint32), dump.stage("fir").view(np.uint32))
    # both gates evaluated before either is asserted, so that a failure shows whether the body departs from the reference, from the
    # dumping body, or from both
    assert d.max() <= 1e-5 and same, dict(max=float(d.max()), at=int(np.argmax(d)), bitwise_dump=same)
    assert gain_matches(s, st), (s["agc_gain"], st["gain"])
    assert dump.stats()["agc_gain"] == s["agc_gain"]


def test_hook_refusals(built):
    capi = _capi()
    cfg, raw, _ = signal("metop_ahrpt", 16)
    g = gpu(cfg, 1 << 16, keep_front=False)
    with pytest.raises(capi.B200Error) as e:
        g.stage("fir")  # neither keep_stages nor keep_front
    assert e.value.code == -5
    with pytest.raises(capi.B200Error) as e:
        gpu(cfg, 1 << 16, keep_stages=True).debug_shape(keep_front=True)
    assert e.value.code == -1 and "keep_stages" in str(e.value)
    for L in (4095, 4100, 16400, -16):
        with pytest.raises(capi.B200Error) as e:
            g.debug_shape(seg_len=L)
        assert e.value.code == -1 and "seg_len" in str(e.value)
    with pytest.raises(capi.B200Error):
        g.debug_shape(range_tiles=-1)


# ---------------------------------------------------------------------------------------------------------------- 2. range / batch edges
RANGES = [1, 4, 5, 7, 64, 1 << 20]  # 1 << 20: every tile in one range
K2048, K256 = 37 * 2048, 300 * 256
SIZES = [4096, 4097, K2048 - 1, K2048, K2048 + 1, K256 + 31, K256 + 32, K256 + 33, N - 1]  # K256 + 32: c_fast = (N - 32) / 256 turns


@pytest.fixture(scope="module")
def edge_refs():
    cfg, raw, _ = signal("metop_ahrpt", LG)
    return {n: reference(cfg, raw[:2 * n]) for n in SIZES}


@pytest.mark.parametrize("R", RANGES, ids=["R1", "R4", "R5", "R7", "R64", "Rall"])
def test_range_and_batch_edges(built, edge_refs, R):
    """Range starts and ends, walks back across other ranges' tiles, the branch-free body's last chunk and a range ending mid-tile at the
    batch end: each size one-shot against the reference (1e-5) and the R = 4 run (2e-6), then all of them as one ragged stream."""
    cfg, raw, _ = signal("metop_ahrpt", LG)
    g, g4 = gpu(cfg, N, range_tiles=R), gpu(cfg, N, range_tiles=4)
    for n in SIZES:
        o, st = edge_refs[n]
        g.reset().push(raw[:2 * n])
        g4.reset().push(raw[:2 * n])
        s = g.stats()
        assert s["last_range_tiles"] == R and g4.stats()["last_range_tiles"] == 4 and s["agc_exact_passes"] == 0, (n, s)
        fir = g.stage("fir")
        assert fir.size == n
        d = np.abs(fir - o["fir"])
        assert d.max() <= 1e-5, (n, float(d.max()), int(np.argmax(d)))
        assert np.abs(fir - g4.stage("fir")).max() <= 2e-6, n
        assert gain_matches(s, st), (n, s["agc_gain"], st["gain"])
    # ragged: the sizes back to back (carried FIR tail and gain), the rest of the fixture in one more push
    o, st = reference(cfg, raw)
    g.reset()
    parts, prev = [], 0
    for n in SIZES[:-1] + [N - sum(SIZES[:-1])]:
        g.push(raw[2 * prev:2 * (prev + n)])
        assert g.stats()["last_range_tiles"] == R
        parts.append(g.stage("fir"))
        prev += n
    d = np.abs(np.concatenate(parts) - o["fir"])
    assert d.max() <= 1e-5, (float(d.max()), int(np.argmax(d)))
    assert gain_matches(g.stats(), st)


# ---------------------------------------------------------------------------------------------------------------- 3. walk-back seeding
RATE, MAX_GAIN, WARM_TILES = 1e-2, 65536.0, 24


def walk_lengths(x, R):
    """Chunks each range of R tiles walks back before its start gain is proven (k_agc_fir_w: A * max_gain <= B * 2^-30), None where
    the 24-tile limit is hit and the batch takes the exact pass. Evaluated in double from the same step maps."""
    e = RATE * np.abs(x).astype(np.float64)
    nch = x.size // 256
    lg = np.log1p(-e[:nch * 256]).reshape(nch, 256)
    suf = np.cumsum(lg[:, ::-1], axis=1)[:, ::-1]
    tB = RATE * np.exp(suf - lg).sum(axis=1)  # the chunk's map g -> tA g + tB
    tA = np.exp(suf[:, 0])
    out = []
    for t in range(R, x.size // 2048, R):
        A, B, res = 1.0, 0.0, None
        for w, j in enumerate(range(8 * t - 2, -2, -1)):
            if j < 0:
                res = w
                break
            if w >= WARM_TILES * 8:
                break
            B += A * tB[j]
            A *= tA[j]
            if A * MAX_GAIN <= B * 2.0 ** -30:
                res = w + 1
                break
        out.append(res)
    return out


def stepped(x, R, weak):
    """x with its level stepped in front of every range start: x80 (a seed proven within one chunk), x0.28 for 100 000 samples (20-24
    tiles of walk), 1/16 for 60 000 samples (no proof within 24 tiles) when `weak`, the fixture's level elsewhere."""
    lv = np.ones(x.size, np.float32)
    rl = R * 2048
    for k in range(1, x.size // rl):
        s0 = k * rl
        if k % 3 == 1:
            lv[s0 - 30000:s0 + 10000] = 80.0
        elif k % 3 == 2:
            lv[s0 - 100000:s0 + 30000] = 0.28
        elif weak:
            lv[s0 - 60000:s0 + 10000] = 1 / 16
    return (x * lv).astype(np.complex64)


def test_walk_back_seeding(built):
    """Ranges of 64 tiles whose seeds are proven after one chunk, after 20-24 tiles of walk across the previous range, and (second push)
    not at all, so the batch is redone from the scanned seeds. Both pushes against one reference run of the whole stream; the AGC
    output reaches 80x the usual level at the upward steps, so the error is taken relative to max(1, |reference|).
    The x80 stretches are cf32 input far above full scale: a chunk's composed decay 1 - E there is below the float resolution of E, and
    without the decay carried as a product (AGC_A_SMALL in demod.cuh) the first chunks after an upward step were 1.08e-5 off."""
    cfg, raw, _ = signal("metop_ahrpt", LG)
    x = derive(raw, "cf32")
    a, b = stepped(x, 64, False), stepped(x, 64, True)
    wa, wb = walk_lengths(a, 64), walk_lengths(b, 64)
    assert None not in wa and 1 in wa and any(160 < w <= 192 for w in wa), wa
    assert None in wb, wb
    o, st = reference(cfg, np.concatenate([a, b]), "cf32")
    g = gpu(cfg, N, "cf32", range_tiles=64)
    fir = []
    for part, exact, tol in ((a, 0, 1e-5), (b, 1, 3e-5)):
        g.push(part)
        s = g.stats()
        assert s["last_range_tiles"] == 64 and s["agc_exact_passes"] == exact and s["agc_clamped"] == 0, s
        f = g.stage("fir")
        want = o["fir"][len(fir) * N:(len(fir) + 1) * N]
        d = np.abs(f - want) / np.maximum(1.0, np.abs(want))
        assert d.max() <= tol, (exact, float(d.max()), int(np.argmax(d)))
        fir.append(f)
    assert gain_matches(g.stats(), st)


# ---------------------------------------------------------------------------------------------------------------- 4. segment lengths
SEG_LENS = [4096, 4112, 8192, 15888, 16384]
LOOPS = [("metop_ahrpt", ()), ("jpss_hrd", ()), ("bpsk_half", ()), ("psk8", ()), ("metop_ahrpt", GX), ("pm_bpsk", ())]


def junction_bounds(jpss_or_8psk):
    # test_junction_residuals_are_small's bounds; OQPSK and 8PSK junctions are accepted up to their (doubled) repair tolerances
    return (2e-5, 4e-6) if jpss_or_8psk else (1e-5, 2e-6)


@pytest.mark.parametrize("L", SEG_LENS)
@pytest.mark.parametrize("name,extra", LOOPS, ids=[n + ("-gardner" if e else "") for n, e in LOOPS])
def test_segment_lengths(built, name, extra, L):
    """The Costas loop, the M&M / Gardner clock recovery and pm_demod's carrier PLL at every segment length choose_L can return,
    including 15 888 (2^29 samples on 132 SMs: not a power of two, 4x the slots and checkpoints of 4096) and 16 384."""
    from tests.floors import reference_run
    cfg, raw, oc, o = reference_run(name, LG, extra)
    n = nsamples(raw, cfg)
    kw = dict(extra)
    g = gpu(cfg, n, seg_len=L, keep_front=False, **kw).push(raw)
    cj, mj, got_L = g.junctions()
    assert got_L == L and cj.shape[0] == mj.size == (n + L - 1) // L
    s = g.stats()
    assert s["costas_unconverged"] == 0 and s["mm_unconverged"] == 0 and s["pll_unconverged"] == 0, s
    assert s["symbols_out"] == o["mm"].size
    assert np.median(np.abs(mj[1:])) <= 1e-4 and np.abs(mj[1:]).max() <= 0.01, (float(np.median(np.abs(mj[1:]))), float(np.abs(mj[1:]).max()))
    tp, tf = junction_bounds(cfg.constellation in ("oqpsk", "8psk"))
    assert np.abs(cj[1:, 0]).max() <= tp and np.abs(cj[1:, 1]).max() <= tf, (np.abs(cj[1:, 0]).max(), np.abs(cj[1:, 1]).max())
    if cfg.pm_index:
        from tests.test_gpu_pm import soft_gates
        soft_gates(g.symbols(), g.soft(), o)
        return
    fl = cached("chain", name, LG, extra=extra)
    check_mm(g.symbols(), o["mm"], g.soft(), o["soft"], floor=fl)
    st = gpu(cfg, n, seg_len=L, keep_stages=True, **kw).push(raw)
    assert st.junctions()[2] == L
    check_costas(st.stage("costas"), o["costas"], fl)


# ---------------------------------------------------------------------------------------------------------------- 5. multi-block tile scans
BIG = 1 << 24  # 8192 tiles: k_tile_scan takes 8 turns of 1024


def tiled(raw, n, per):
    reps = -(-n * per // raw.size)
    return np.tile(raw, reps)[:n * per]


def test_dc_block_scan_at_2e24(built):
    cfg, raw, _ = signal("metop_ahrpt", LG)
    raw = tiled(raw, BIG, 2)
    raw[0::2] += 900
    raw[1::2] -= 400
    O = oracle()
    oc = O.demod_cfg(dc_block=True, **demod_kwargs(cfg))
    g = _capi().Demod(_capi().demod_cfg(max_batch=BIG, keep_stages=True, dc_block=True, **demod_kwargs(cfg))).push(raw)
    d = np.abs(g.stage("dc") - O.resample(oc, raw))
    assert d.max() <= 1e-6, (float(d.max()), int(np.argmax(d)))


def test_weak_signal_exact_pass_at_2e24(built):
    cfg, raw, _ = signal("metop_ahrpt", LG)
    raw = (tiled(raw, BIG, 2).astype(np.int32) // 16).astype(np.int16)
    o, st = reference(cfg, raw)
    g = gpu(cfg, BIG).push(raw)
    s = g.stats()
    assert s["agc_exact_passes"] == 1 and s["last_range_tiles"] == 4, s
    d = np.abs(g.stage("fir") - o["fir"])
    assert d.max() <= 3e-5, (float(d.max()), int(np.argmax(d)))
    assert gain_matches(s, st) and s["symbols_out"] == o["mm"].size


def test_fsk_scans_at_2e24(built):
    """fsk_demod's tile-scanned DC blocker and AGC against the one-thread float recurrence (test_scans_follow_the_sequential_recurrence)."""
    from tests.test_gpu_fsk import SIGNALS, _cfg, _signal
    sig = SIGNALS[0]
    raw = tiled(_signal(sig, N), BIG, 2)
    d = _capi().Demod(_cfg(sig, max_batch=BIG, keep_stages=True)).push(raw)
    quad, dc2, agc2 = d.stage("quad"), d.stage("dc2"), d.stage("agc2")
    assert np.abs(dc2 - d.run_stage("dc2", quad, strict=True, sequential=True)).max() <= 1e-5
    assert np.abs(agc2 - d.run_stage("agc2", dc2, strict=True, sequential=True)).max() <= 1e-5


# ---------------------------------------------------------------------------------------------------------------- 6. the benchmark's size
def test_benchmark_sized_push(built, record_property):
    """metop_ahrpt, cs16, 2^29 samples in one push (2 GiB of raw input, 4 GiB per cf32 stage buffer), production R and L, generated on the
    device. The reference runs the same samples in 2^24-sample pieces (its Demod keeps state across run()); every piece's RRC output is
    compared with the matching slice, the symbols piece by piece. Maxima grow with length and no floor exists at this size: they are
    recorded, the rates are gated with the 2^21 floor of the same signal kind."""
    import torch
    from satdump_b200 import synth
    capi = _capi()
    n, piece = 1 << 29, 1 << 24
    if torch.cuda.mem_get_info()[0] < (40 << 30):
        pytest.skip(f"needs 40 GiB of free device memory, {torch.cuda.mem_get_info()[0] >> 30} GiB free")
    cfg = synth.CONFIGS["metop_ahrpt"]
    raw_d, _ = synth.make_signal(cfg, n, seed=29, device="cuda")
    raw_d = raw_d.contiguous()
    assert raw_d.numel() == 2 * n
    torch.cuda.empty_cache()
    g = gpu(cfg, n)
    g.push_device(raw_d.data_ptr(), n)
    raw = raw_d.cpu().numpy()
    del raw_d
    torch.cuda.empty_cache()
    s = g.stats()
    cj, mj, L = g.junctions()
    want_L = -(-n // (torch.cuda.get_device_properties(0).multi_processor_count * 2 * 128))
    want_L = (min(16384, max(4096, want_L)) + 15) // 16 * 16
    assert L == want_L and s["last_range_tiles"] > 4, (L, want_L, s["last_range_tiles"])
    record_property("R", s["last_range_tiles"])
    record_property("L", L)
    assert s["costas_unconverged"] == 0 and s["mm_unconverged"] == 0 and s["agc_exact_passes"] == 0, s
    fir = g.stage("fir")
    syms = np.empty(s["symbols_out"], np.complex64)
    assert g.pull_symbols_into(syms.ctypes.data, syms.size) == syms.size
    soft = g.soft()
    O = oracle()
    od = O.Demod(O.demod_cfg(**demod_kwargs(cfg)))
    fmax, pos, mm_bad, mm_max, sd, sgt1 = 0.0, 0, 0, 0.0, 0, 0
    for k in range(n // piece):
        o = od.run(raw[2 * k * piece:2 * (k + 1) * piece])
        d = np.abs(fir[k * piece:(k + 1) * piece] - o["fir"])
        assert d.max() <= 1e-5, (k, float(d.max()), int(np.argmax(d)))
        fmax = max(fmax, float(d.max()))
        m = o["mm"].size
        assert pos + m <= syms.size, (k, pos + m, syms.size)
        dm = np.abs(syms[pos:pos + m] - o["mm"])
        mm_bad += int((dm > 1e-5).sum())
        mm_max = max(mm_max, float(dm.max()))
        ds = np.abs(soft[2 * pos:2 * (pos + m)].astype(np.int16) - o["soft"].astype(np.int16))
        sd += int((ds > 0).sum())
        sgt1 += int((ds > 1).sum())
        pos += m
    assert pos == syms.size == s["symbols_out"], (pos, syms.size)
    st = od.state()
    fl = cached("chain", "metop_ahrpt", LG)
    rates = dict(mm_frac=mm_bad / pos, soft_diff=sd / (2 * pos), soft_gt1=sgt1 / (2 * pos))
    for k, v in dict(fir_max=fmax, mm_max=mm_max, **rates).items():
        record_property(k, v)
    assert rates["mm_frac"] <= gate(SURVEY["mm_frac"], fl.get("mm_frac", 0.0)), (rates, fl)
    assert rates["soft_diff"] <= gate(SURVEY["soft_diff"], fl.get("soft_diff", 0.0)), (rates, fl)
    assert rates["soft_gt1"] <= gate(SURVEY["soft_gt1"], fl.get("soft_gt1", 0.0)) + 2e-5, (rates, fl)
    assert gain_matches(s, st), (s["agc_gain"], st["gain"])
    assert abs(s["mm_omega"] - st["omega"]) <= 1e-4
