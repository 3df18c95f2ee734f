"""GPU: the cycle-counting build of the loop kernels (-DB200_LOOP_CYCLES, tools/profile_loops.py --cycles) computes what the
production build computes, and its counters count.

The instrumented library is built into a temporary directory and run in a child process (one library per process); its symbols
must equal the production library's bit for bit, and both main passes must have booked cycles. The production library refuses
the counter call.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from satdump_b200 import capi
from tests.common import gpu_demod, nsamples, signal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LG = 20


def test_instrumented_build_matches_production(built, tmp_path):
    out = tmp_path / "lib"
    subprocess.run(["make", "-s", "-j8", "-C", os.path.join(ROOT, "satdump_b200", "csrc"), "cycles", f"CYCLES_DIR={out}"], check=True,
                   stdout=subprocess.DEVNULL)
    child = (
        "import sys\n"
        "import numpy as np\n"
        "sys.path.insert(0, sys.argv[1])\n"
        "from satdump_b200 import capi\n"
        "capi.LIB_PATH = sys.argv[2]\n"
        "from tests.common import gpu_demod, nsamples, signal\n"
        "cfg, raw, _ = signal('metop_ahrpt', int(sys.argv[4]))\n"
        "capi.loop_cycles()\n"
        "sym = gpu_demod(cfg, nsamples(raw, cfg)).push(raw).symbols()\n"
        "c = capi.loop_cycles()\n"
        "np.save(sys.argv[3] + '/sym.npy', sym)\n"
        "np.save(sys.argv[3] + '/cycles.npy', np.array(c['k_costas'] + c['k_mm'], np.uint64))\n"
    )
    subprocess.run([sys.executable, "-c", child, ROOT, str(out / "libb200dsp.so"), str(tmp_path), str(LG)], check=True, cwd=ROOT)
    cfg, raw, _ = signal("metop_ahrpt", LG)
    want = gpu_demod(cfg, nsamples(raw, cfg)).push(raw).symbols()
    got = np.load(tmp_path / "sym.npy")
    assert got.shape == want.shape and got.tobytes() == want.tobytes()
    cyc = np.load(tmp_path / "cycles.npy")
    costas, mm = cyc[:5], cyc[5:]
    assert costas[4] > 0 and mm[4] > 0, cyc  # warps of each main pass
    assert costas[:4].sum() > 0 and mm[:4].sum() > 0 and mm[2] > 0, cyc  # cycles, the symbol loop's among them
    with pytest.raises(capi.B200Error):
        capi.loop_cycles()
