"""Diagnostic: where the largest M&M symbol deviations of the whole chain sit relative to the segment junctions."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from oracle import ref as O  # noqa: E402
from satdump_b200 import capi  # noqa: E402
from tests.common import demod_kwargs, nsamples, signal  # noqa: E402

lg = int(sys.argv[1]) if len(sys.argv) > 1 else 21
for name in sys.argv[2:] or ["bpsk_half"]:
    cfg, raw, _ = signal(name, lg)
    n = nsamples(raw, cfg)
    o = O.Demod(O.demod_cfg(**demod_kwargs(cfg))).run(raw)
    g = capi.Demod(capi.demod_cfg(max_batch=n, keep_stages=True, **demod_kwargs(cfg))).push(raw)
    cj, mj, L = g.junctions()
    sy = g.symbols()
    d = np.abs(sy - o["mm"])
    sps = n / sy.size
    top = np.argsort(-d)[:2000]
    big = np.sort(top[d[top] > 1.5e-2])
    print(name, "L", L, "symbols >1.5e-2:", big.size, "max %.3e" % d.max())
    # cluster the big deviations into events
    ev = []
    for i in big:
        if not ev or i - ev[-1][1] > 2000:
            ev.append([i, i, d[i]])
        else:
            ev[-1][1] = i
            ev[-1][2] = max(ev[-1][2], d[i])
    for a, b, m in ev[:12]:
        s0 = a * sps
        seg = int(s0 // L)
        print("   event symbols %d..%d max %.3e  sample %.0f = segment %d + %.0f, junction residual of that segment %.2e (next %.2e); costas dev there %.2e" % (
            a, b, m, s0, seg, s0 - seg * L, abs(mj[seg]), abs(mj[min(seg + 1, mj.size - 1)]),
            np.abs(g.stage("costas")[int(s0) - 2000:int(s0) + 100] - o["costas"][int(s0) - 2000:int(s0) + 100]).max() if o["costas"] is not None else 0))
