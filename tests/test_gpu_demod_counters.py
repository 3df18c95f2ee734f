"""GPU: the demodulator's launch and junction counters for one push, pinned.

The loop stages (Costas, carrier PLL, M&M) each issue a main pass, a junction check and a fixed number of repair rounds, and the
front end issues its AGC, FIR and DC-blocker launches. `kernel_launches` counts all of them, and `repairs`, the unconverged
junctions and `agc_exact_passes` record what the checks found. The values below were recorded on an H100 for these seeded
signals; a change to the launch sequence or to the repair bookkeeping changes one of them.
"""
import pytest

from tests.common import demod_kwargs, nsamples, signal

pytestmark = pytest.mark.gpu

COUNTERS = ("kernel_launches", "repairs", "costas_unconverged", "mm_unconverged", "pll_unconverged", "agc_exact_passes")

# (signal, extra demodulator options): a Costas configuration, one without Costas, pm_demod, psk_demod carrier mode, both DC blockers,
# and an OQPSK signal whose Costas junctions need repair rounds (pm_bpsk repairs carrier-PLL junctions)
CASES = {
    "metop_ahrpt": ("metop_ahrpt", {}),
    "dvbs2_front": ("dvbs2_front", {}),
    "pm_bpsk": ("pm_bpsk", {}),
    "bpsk_carrier": ("bpsk_carrier", {}),
    "metop_ahrpt_dc": ("metop_ahrpt", dict(dc_block=True, post_costas_dc=True)),
    "jpss_hrd": ("jpss_hrd", {}),
}

EXPECTED = {
    "bpsk_carrier": {"agc_exact_passes": 0, "costas_unconverged": 0, "kernel_launches": 67, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 0},
    "dvbs2_front": {"agc_exact_passes": 0, "costas_unconverged": 0, "kernel_launches": 28, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 0},
    "jpss_hrd": {"agc_exact_passes": 0, "costas_unconverged": 0, "kernel_launches": 46, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 10},
    "metop_ahrpt": {"agc_exact_passes": 0, "costas_unconverged": 0, "kernel_launches": 46, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 0},
    "metop_ahrpt_dc": {"agc_exact_passes": 0, "costas_unconverged": 0, "kernel_launches": 52, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 0},
    "pm_bpsk": {"agc_exact_passes": 1, "costas_unconverged": 0, "kernel_launches": 72, "mm_unconverged": 0, "pll_unconverged": 0, "repairs": 510},
}


def counters(case):
    from satdump_b200 import capi
    name, kw = CASES[case]
    cfg, raw, _ = signal(name, 21)
    g = capi.Demod(capi.demod_cfg(max_batch=nsamples(raw, cfg), **kw, **demod_kwargs(cfg)))
    st = g.push(raw).stats()
    return {k: int(st[k]) for k in COUNTERS}


@pytest.mark.parametrize("case", sorted(CASES))
def test_counters_of_one_push(built, case):
    assert counters(case) == EXPECTED[case]


def test_some_junction_is_repaired():
    """The pinned configurations run the repair pass of the loop kernels."""
    assert EXPECTED["pm_bpsk"]["repairs"] > 0 and EXPECTED["jpss_hrd"]["repairs"] > 0
