"""Throughput of noaa_hrpt_decoder and meteor_hrpt_decoder (the NOAA and METEOR HRPT pipelines' decoders behind pm_demod) on the GPU.

  decoder    the decoder alone on a device-resident soft stream: a locked stream (one walk step per frame) and noise (the walk scans the
             candidate bitmap 1024 positions per step; this shows that a noise-only push does not crawl bit by bit)
  chain      IQ (cs16 at the pipelines' 3 MS/s) -> pm_demod -> the decoder through the fused chain, synchronous, one push
  reference  the reference's module loop (oracle/_ref/libsatref_hrpt.so, 8192-byte work() calls) on one CPU thread of this host, on the
             same soft streams; null where it was not built

Each timing is a host clock around calls that end in a device synchronise, after one warm-up call of the same shape. Prints one JSON line
with the card, its power limit and SM clock read in the same run. Every timed locked push is checked against the transmitted frames.
Real time is 665 400 soft bytes/s.

Usage: python tools/bench_hrpt.py [--soft-mib 64] [--repeats 5] [--chain-log2 24]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

REALTIME = 665400.0


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], text=True)
        name, power, sm, sm_max = [v.strip() for v in out.splitlines()[0].split(",")]
        return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
    except Exception as e:  # noqa: BLE001
        return dict(card=f"unknown ({e!r})")


def summary(times, nbytes):
    t = np.array(times)
    return dict(soft_bytes=int(nbytes), s_median=float(np.median(t)), s_min=float(t.min()), s_max=float(t.max()),
                soft_bytes_per_s=float(nbytes / np.median(t)), x_realtime=float(nbytes / np.median(t) / REALTIME))


def cfg_of(meteor, max_soft):
    from satdump_b200 import capi
    return capi.meteor_hrpt_cfg(max_soft=max_soft) if meteor else capi.noaa_hrpt_cfg(10, max_soft=max_soft)


def time_decoder(meteor, soft, repeats, check=None):
    """seconds per push of the whole stream (one fresh decoder per push, device-resident input)"""
    import torch
    from satdump_b200 import capi
    dev = torch.from_numpy(soft).cuda()
    L = capi.lib()
    times = []
    for k in range(repeats + 1):
        f = capi.Fec(cfg_of(meteor, soft.size))
        f._n = soft.size
        torch.cuda.synchronize()
        t = time.perf_counter()
        capi._chk(L.b200_fec_push_soft_device(f.h, dev.data_ptr(), soft.size))  # (returns after the decoder's stream synchronised)
        dt = time.perf_counter() - t
        got = f.frames()
        if check is not None:
            check(got)
        if k:
            times.append(dt)
        f.close()
    return times


def time_chain(name, log2n, repeats):
    import torch
    from satdump_b200 import capi, synth
    from tests.hrpt_cases import demod_kwargs
    cfg = synth.CONFIGS[name]
    raw, _ = synth.make_signal(cfg, 1 << log2n, seed=5, device="cuda")
    n = raw.numel() // 2
    times = []
    for k in range(repeats + 1):
        ch = capi.Chain(capi.demod_cfg(max_batch=n, **demod_kwargs(cfg)), capi.fec_cfg_for(cfg, max_soft=n))
        torch.cuda.synchronize()
        t = time.perf_counter()
        ch.push_device(raw.data_ptr(), n)
        got = ch.frames()
        dt = time.perf_counter() - t
        if k:
            times.append(dt)
        ch.close()
    t = np.array(times)
    return dict(samples=int(n), s_median=float(np.median(t)), msamples_per_s=float(n / np.median(t) / 1e6), units_out=int(got.shape[0]))


def reference_rate(meteor, soft):
    from oracle import hrpt as O
    if not O.available():
        return None
    t = time.perf_counter()
    O.Hrpt(meteor, 10).run(soft, records=False)
    return soft.size / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--soft-mib", type=int, default=64, help="soft bytes per decoder push, MiB")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chain-log2", type=int, default=24, help="log2 of the IQ samples of the chain push")
    ap.add_argument("--ref-mib", type=int, default=8, help="soft bytes the reference runs for its rate, MiB")
    a = ap.parse_args()
    from satdump_b200 import synth
    out = dict(repeats=a.repeats)
    nbytes = a.soft_mib << 20
    for meteor, name in ((False, "noaa_hrpt"), (True, "meteor_hrpt")):
        per = 8192 if meteor else synth.NOAA_WORDS * 10
        nfr = nbytes // per
        bits, sent = (synth.meteor_hrpt_frames if meteor else synth.noaa_hrpt_frames)(nfr, 7)
        locked = synth.hrpt_soft(bits, sigma=10.0, seed=1)

        def check(got, sent=sent, meteor=meteor):
            g = got if meteor else got.reshape(-1).view(np.uint16).reshape(-1, synth.NOAA_WORDS)
            assert np.array_equal(g, sent), "locked stream: output differs from the transmitted frames"

        noise = np.clip(np.round(np.random.default_rng(3).normal(0, 60, nbytes)), -127, 127).astype(np.int8)
        r = dict(locked=summary(time_decoder(meteor, locked, a.repeats, check), locked.size),
                 noise=summary(time_decoder(meteor, noise, a.repeats), noise.size),
                 chain=time_chain(name, a.chain_log2, a.repeats))
        nr = a.ref_mib << 20
        r["reference_single_thread"] = dict(locked_soft_bytes_per_s=reference_rate(meteor, locked[:nr]),
                                            noise_soft_bytes_per_s=reference_rate(meteor, noise[:nr]))
        r["locked"]["frames"] = int(nfr)
        out[name] = r
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
