"""Throughput of noaa_gac_decoder and dmsp_rtd_decoder (the NOAA GAC and DMSP RTD pipelines' decoders behind psk_demod BPSK) on the GPU.

  decoder    the decoder alone on a soft stream pushed from host memory: a locked stream and noise
  chain      IQ (cs16 at the pipelines' rates: GAC 6 MS/s, DMSP 2 MS/s) -> psk_demod BPSK -> the decoder through the fused chain,
             synchronous, one push
  reference  the reference's module loop (oracle/_ref/libsatref_gac.so, 8192-byte reads) on one CPU thread of this host, on the same
             locked streams; null where it was not built

Each timing is a host clock around calls that end in a device synchronise (a push returns after its frames are written), after one
warm-up call of the same shape. Prints one JSON line with the card, its power limit and SM clock read in the same run. Every timed locked
push is checked against the transmitted frames. Real time is 2 661 600 (GAC) and 1 024 000 (DMSP) soft bytes/s.

Usage: python tools/bench_gac_dmsp.py [--soft-mib 64] [--repeats 5] [--chain-log2 24]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

REALTIME = dict(noaa_gac=2661600.0, dmsp_rtd=1024000.0)


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, sm, sm_max = [v.strip() for v in out.splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:  # noqa: BLE001
        return dict(card=f"unknown ({e!r})")


def timed(fn, repeats):
    fn()
    t = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        t.append(time.perf_counter() - t0)
    return float(np.median(t))


def locked_stream(name, nbytes):
    from satdump_b200 import synth
    if name == "noaa_gac":
        bits, sent = synth.gac_frames(nbytes // synth.GAC_BITS + 1, seed=1)
    else:
        bits, sent = synth.dmsp_frames(nbytes // synth.DMSP_BITS + 1, seed=1)
    soft = synth.hrpt_soft(bits.reshape(-1)[:nbytes], sigma=10.0, seed=2)
    return soft, sent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--soft-mib", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chain-log2", type=int, default=24)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU")
    from satdump_b200 import capi, synth
    from oracle import gac as O
    res = dict(card())
    n = a.soft_mib << 20
    for name in ("noaa_gac", "dmsp_rtd"):
        cfg = capi.noaa_gac_cfg(False, max_soft=n) if name == "noaa_gac" else capi.dmsp_rtd_cfg(max_soft=n)
        soft, sent = locked_stream(name, n)
        noise = np.clip(np.round(np.random.default_rng(3).normal(0, 90, n)), -127, 127).astype(np.int8)
        f = capi.Fec(cfg)
        got = f.push(soft).frames()
        assert got.shape[0] >= sent.shape[0] - 2 and np.array_equal(got, sent[:got.shape[0]]), "locked push lost frames"
        t_lock = timed(lambda: f.push(soft).frames(), a.repeats)
        t_noise = timed(lambda: f.push(noise).frames(), a.repeats)
        f.close()
        r = dict(decoder_locked_GBps=n / t_lock / 1e9, decoder_noise_GBps=n / t_noise / 1e9,
                 decoder_locked_x_realtime=n / t_lock / REALTIME[name], decoder_noise_x_realtime=n / t_noise / REALTIME[name])
        sig = synth.CONFIGS[name]
        ns = 1 << a.chain_log2
        raw, _ = synth.make_signal(sig, ns, seed=5)
        raw = raw.numpy()
        ch = capi.Chain(capi.demod_cfg_for(sig, max_batch=ns), capi.fec_cfg_for(sig, max_soft=ns))
        t_chain = timed(lambda: (ch.push(raw), ch.frames()), a.repeats)
        ch.close()
        r.update(chain_MSps=ns / t_chain / 1e6, chain_x_realtime=ns / t_chain / sig.samplerate)
        if O.available():
            m = min(n, 1 << 24)
            ref = O.Ref(name == "dmsp_rtd")
            t0 = time.perf_counter()
            ref.run(soft[:m])
            r.update(reference_1thread_MBps=m / (time.perf_counter() - t0) / 1e6)
        else:
            r.update(reference_1thread_MBps=None)
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
