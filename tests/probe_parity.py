"""Diagnostic (not a test): where the float parity of each demodulator stage stands, stage-isolated and end to end.

For every parity configuration it reports, against the compiled reference (oracle/_ref):
  * FIR fed the oracle's AGC output: strict build bitwise?  production (FMA) max |d|
  * Costas fed the oracle's FIR output: segmented (production) and sequential (one thread) error statistics, junction residuals
  * M&M fed the oracle's clock-recovery input: strict sequential bitwise?  production sequential / segmented statistics
  * the oracle's own floor: its Costas / M&M output after a 1-ulp perturbation of the stage input
  * the whole chain from raw IQ
Usage on a GPU box:  python tests/probe_parity.py [out.json] [log2 samples] [config ...]"""
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref as O  # noqa: E402
from satdump_b200 import capi  # noqa: E402
from tests.common import demod_kwargs, nsamples, signal  # noqa: E402

CONFIGS = ["metop_ahrpt", "bpsk_half", "jpss_hrd", "dvbs2_front", "hrpt_bpsk", "psk8"]


def stat(a, b):
    if a.size != b.size:
        return dict(size=(int(a.size), int(b.size)))
    d = np.abs(a - b)
    return dict(n=int(a.size), bitwise=bool(np.array_equal(a.view(np.uint32), b.view(np.uint32))), max=float(d.max()), mean=float(d.mean()),
                gt1e5=float((d > 1e-5).mean()), gt1e4=float((d > 1e-4).mean()), gt1e3=float((d > 1e-3).mean()))


def ulp_perturb(x, seed):
    rng = np.random.default_rng(seed)
    xf = np.ascontiguousarray(x).view(np.float32).copy()
    step = (rng.integers(0, 3, xf.size) - 1).astype(np.int32)
    step[(xf.view(np.int32) & 0x7FFFFFFF) == 0] = 0  # leave zeros alone (the magnitude bits are what moves)
    return (xf.view(np.int32) + step).view(np.float32).view(np.complex64)


def pct(v):
    v = np.abs(np.asarray(v))
    if v.size == 0:
        return {}
    return {f"p{p}": float(np.percentile(v, p)) for p in (50, 90, 99, 99.9)} | {"max": float(v.max())}


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else "gpurun_out/probe_parity.json"
    lg = int(sys.argv[2]) if len(sys.argv) > 2 else 21
    names = sys.argv[3:] or CONFIGS
    res = {}
    for name in names:
        cfg, raw, _ = signal(name, lg)
        n = nsamples(raw, cfg)
        kw = demod_kwargs(cfg)
        oc = O.demod_cfg(**kw)
        o = O.Demod(oc).run(raw)
        nf = o["agc"].size
        g = capi.Demod(capi.demod_cfg(max_batch=max(n, 4096), keep_stages=True, **kw))
        r = {"samples": n, "front": int(nf)}
        # ---- FIR
        r["fir_strict"] = stat(g.run_stage("fir", o["agc"], strict=True), o["fir"])
        r["fir_prod"] = stat(g.run_stage("fir", o["agc"]), o["fir"])
        mm_in = o["fir"]
        if o["costas"] is not None:
            # ---- Costas
            for mode, seq in (("seg", False), ("seq", True)):
                c = g.run_stage("costas", o["fir"], sequential=seq)
                r[f"costas_{mode}"] = stat(c, o["costas"]) | dict(junction=pct(g.junctions()[0][1:, 0]), L=g.junctions()[2])
            r["costas_floor"] = stat(O.run_stage(oc, "costas", ulp_perturb(o["fir"], 11)), o["costas"])
            mm_in = o["costas"]
        # ---- M&M
        r["mm_strict_seq"] = stat(g.run_stage("mm", mm_in, strict=True, sequential=True), o["mm"])
        r["mm_prod_seq"] = stat(g.run_stage("mm", mm_in, sequential=True), o["mm"])
        r["mm_strict_seg"] = stat(g.run_stage("mm", mm_in, strict=True), o["mm"])
        s = g.run_stage("mm", mm_in)
        r["mm_prod_seg"] = stat(s, o["mm"]) | dict(junction=pct(g.junctions()[1][1:]), L=g.junctions()[2])
        fl = [stat(O.run_stage(oc, "mm", ulp_perturb(mm_in, sd)), o["mm"]) for sd in (21, 22, 23)]
        r["mm_floor"] = dict(gt1e5=[f.get("gt1e5") for f in fl], max=[f.get("max") for f in fl])
        # ---- whole chain
        g.push(raw)
        r["chain_agc"] = stat(g.stage("agc"), o["agc"])
        r["chain_fir"] = stat(g.stage("fir"), o["fir"])
        if o["costas"] is not None:
            r["chain_costas"] = stat(g.stage("costas"), o["costas"])
        r["chain_mm"] = stat(g.symbols(), o["mm"])
        gs, os_ = g.soft(), o["soft"]
        if gs.size == os_.size:
            ds = np.abs(gs.astype(np.int16) - os_.astype(np.int16))
            r["chain_soft"] = dict(diff=float((ds > 0).mean()), gt1=float((ds > 1).mean()), max=int(ds.max()))
        cj, mj, L = g.junctions()
        st = g.stats()
        r["chain_junctions"] = dict(L=L, costas=pct(cj[1:, 0]), costas_f=pct(cj[1:, 1]), mm=pct(mj[1:]), repairs=st["repairs"],
                                    costas_unconv=st["costas_unconverged"], mm_unconv=st["mm_unconverged"])
        res[name] = r
        cj = r["chain_junctions"]
        print(name, "L", cj["L"], "costas seg max %.1e gt %.5f | junc p99.9 %.1e max %.1e | mm seg gt %.5f max %.1e junc p50 %.1e p99.9 %.1e | floor gt %.5f max %.1e | chain costas %.1e mm gt %.5f max %.1e soft %s repairs %d unconv %d %d" % (
            r.get("costas_seg", {}).get("max", 0), r.get("costas_seg", {}).get("gt1e5", 0), cj["costas"].get("p99.9", 0), cj["costas"].get("max", 0),
            r["mm_prod_seg"]["gt1e5"], r["mm_prod_seg"]["max"], r["mm_prod_seg"]["junction"]["p50"], r["mm_prod_seg"]["junction"]["p99.9"],
            max(x or 0 for x in r["mm_floor"]["gt1e5"]), max(x or 0 for x in r["mm_floor"]["max"]),
            r.get("chain_costas", {}).get("max", 0), r["chain_mm"].get("gt1e5", -1), r["chain_mm"].get("max", -1), r.get("chain_soft"),
            cj["repairs"], cj["costas_unconv"], cj["mm_unconv"]), flush=True)
        g.close()
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    with open(out_path, "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
