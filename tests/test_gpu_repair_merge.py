"""GPU: a repair of a failed junction stops where it meets the segment's stored run.

The loop kernels store their state every 512 owned samples. A repair (the exact continuation of the predecessor segment) compares its
state with the stored one at those checkpoints and stops at the first that agrees within 1/16 of the junction tolerance: the stored outputs,
symbol slots and end record behind it stand. Checked on two signals whose junctions fail (`jpss_hrd`: OQPSK Costas warm-ups that hang
near the unstable lock point; `pm_bpsk`: nearly every clock-recovery junction at 6 samples per symbol and 4096-sample segments):

  - the output of the whole demodulator stays within the gates against the reference's sequential loops that the unrepaired
    segments are held to (tests/floors.py), with every junction converged;
  - repairs happen, every one is counted once in `repair_merge_hist`, and some stop early;
  - with the hook that gives the comparison a tolerance of 0 no repair stops early: each runs its whole segment, and the output
    passes the same gates with the same symbol count.
"""
import numpy as np
import pytest

from tests.common import gpu_demod, nsamples, oracle, oracle_demod, signal
from tests.floors import cached
from tests.test_gpu_demod import check_costas, check_mm
from tests.test_gpu_pm import soft_gates

pytestmark = pytest.mark.gpu
LG = 21


def run(cfg, raw, merge):
    g = gpu_demod(cfg, nsamples(raw, cfg), keep_stages=True).repair_merge(merge).push(raw)
    s = g.stats()
    assert s["costas_unconverged"] == 0 and s["mm_unconverged"] == 0 and s["pll_unconverged"] == 0, s
    hist = s["repair_merge_hist"]
    assert s["repairs"] > 0 and sum(hist) == s["repairs"], s
    return g, hist


@pytest.mark.parametrize("merge", [True, False])
def test_costas_repairs_on_an_oqpsk_signal(built, merge):
    cfg, raw, _ = signal("jpss_hrd", LG)
    o = oracle_demod(oracle(), cfg).run(raw)
    g, hist = run(cfg, raw, merge)
    fl = cached("chain", "jpss_hrd", LG)
    check_costas(g.stage("costas"), o["costas"], fl)
    check_mm(g.symbols(), o["mm"], g.soft(), o["soft"], floor=fl)
    assert (sum(hist[1:]) > 0) == merge, hist


@pytest.mark.parametrize("merge", [True, False])
def test_repairs_of_a_pm_demod_signal(built, merge):
    cfg, raw, _ = signal("pm_bpsk", LG)
    o = oracle_demod(oracle(), cfg).run(raw)
    g, hist = run(cfg, raw, merge)
    assert np.abs(g.stage("pll") - o["pll"]).max() <= 1e-5
    soft_gates(g.symbols(), g.soft(), o)
    assert (sum(hist[1:]) > 0) == merge, hist


def test_repairs_change_nothing_they_need_not(built):
    """Stopping early keeps the stored tail: the symbol count is that of the whole-segment repairs, and the symbols differ from
    them only at the level at which two converged runs of a loop differ."""
    cfg, raw, _ = signal("jpss_hrd", LG)
    a = run(cfg, raw, True)[0].symbols()
    b = run(cfg, raw, False)[0].symbols()
    assert a.size == b.size
    d = np.abs(a - b)
    fl = cached("chain", "jpss_hrd", LG)
    assert (d > 1e-5).mean() <= max(1e-3, 1.2 * fl.get("mm_frac", 0.0)), (float((d > 1e-5).mean()), float(d.max()), fl)
