"""Throughput of aqua_db_decoder (the EOS Aqua / Aura DB pipelines' decoder behind psk_demod OQPSK) on the GPU.

  decoder    the decoder alone on a device-resident soft stream: a locked stream and noise (the deframer's NOSYNC search over every bit)
  chain      IQ (cs16 at the pipelines' 15 MS/s) -> psk_demod OQPSK (EOS.json's parameters) -> the decoder through the fused chain:
             synchronous (one push) and pipelined (four pushes, the decoder one batch behind)
  terra      IQ (cs16 at 45 MS/s) -> terra_db_demod -> ccsds_conv_concat_decoder (EOS.json "terra_db") through the fused chain,
             synchronous, one push; its demodulator's stage split (AGC + RRC, k_costas, k_mm main pass and repairs) from the chain's
             event timing, and the M&M warm-up share nseg * (L + W) / owned samples (W = 240 / gain_mu, the BPSK warm-up rule)
  reference  the reference's module loop (oracle/_ref/libsatref_eos.so, 65 536-byte reads) on one CPU thread of this host, on the same
             soft streams; null where it was not built

Each timing is a host clock around calls that end in a device synchronise, after one warm-up call of the same shape. Prints one JSON line
with the card, its power limit and SM clock read in the same run. Every timed locked push is checked against the transmitted frames.
Real time is 15 MS/s of IQ = 15 000 000 soft bytes/s.

Usage: python tools/bench_eos.py [--soft-mib 64] [--repeats 5] [--chain-log2 24]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_hrpt import card  # noqa: E402

REALTIME = 15e6


def summary(times, nbytes):
    t = np.array(times)
    return dict(soft_bytes=int(nbytes), s_median=float(np.median(t)), s_min=float(t.min()), s_max=float(t.max()),
                soft_bytes_per_s=float(nbytes / np.median(t)), x_realtime=float(nbytes / np.median(t) / REALTIME))


def time_decoder(soft, repeats, check=None):
    """seconds per push of the whole stream (one fresh decoder per push, device-resident input)"""
    import torch
    from satdump_b200 import capi
    dev = torch.from_numpy(soft).cuda()
    L = capi.lib()
    times = []
    for k in range(repeats + 1):
        f = capi.Fec(capi.aqua_db_cfg(max_soft=soft.size))
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


def time_chain(log2n, repeats, pipelined):
    import torch
    from satdump_b200 import capi, synth
    from tests.eos_cases import aqua_demod_kwargs
    cfg = synth.CONFIGS["aqua_db"]
    raw, _ = synth.make_signal(cfg, 1 << log2n, seed=5, device="cuda")
    n = raw.numel() // 2
    parts = 4 if pipelined else 1
    step = n // parts
    times = []
    for k in range(repeats + 1):
        ch = capi.Chain(capi.demod_cfg(max_batch=step, **aqua_demod_kwargs("cs16")), capi.aqua_db_cfg(max_soft=step + 65536))
        if pipelined:
            ch.set_pipelined(True)
        nf = 0
        torch.cuda.synchronize()
        t = time.perf_counter()
        for p in range(parts):
            ch.push_device(raw.data_ptr() + 4 * p * step, step)
            nf += ch.frames(cap=step + (1 << 20)).shape[0]
        if pipelined:
            ch.sync()
            nf += ch.frames(cap=step + (1 << 20)).shape[0]
        dt = time.perf_counter() - t
        if k:
            times.append(dt)
        ch.close()
    t = np.array(times)
    ns = step * parts
    return dict(samples=int(ns), pushes=parts, s_median=float(np.median(t)), msamples_per_s=float(ns / np.median(t) / 1e6),
                x_realtime=float(ns / np.median(t) / REALTIME), cadus_out=int(nf))


def time_terra(log2n, repeats):
    import torch
    from satdump_b200 import capi, synth
    from tests.eos_cases import TERRA_FEC, terra_demod_kwargs
    raw, _ = synth.make_signal(synth.CONFIGS["terra_db"], 1 << log2n, seed=5, device="cuda")
    n = raw.numel() // 2
    times, stages = [], []
    for k in range(repeats + 1):
        ch = capi.Chain(capi.demod_cfg(max_batch=n, **terra_demod_kwargs()), capi.ccsds_cfg("bpsk_90", 8192, 0.3, 20, max_soft=2 * n, **TERRA_FEC))
        torch.cuda.synchronize()
        t = time.perf_counter()
        ch.push_device(raw.data_ptr(), n)
        nf = ch.frames(cap=n + (1 << 20)).shape[0]
        dt = time.perf_counter() - t
        if k:
            times.append(dt)
            stages.append([ch.timing()[k] for k in ("agc_fir", "costas", "mm", "viterbi", "deframe_rs")])
        ds, _ = ch.stats()
        ch.close()
    st = np.median(np.array(stages), axis=0)
    d = capi.Demod(capi.demod_cfg(max_batch=n, **terra_demod_kwargs()))
    d.push_device(raw.data_ptr(), n)
    _, mm, L = d.junctions()
    W = int(np.ceil(240.0 / 0.001 / 16) * 16)
    return dict(samples=int(n), s_median=float(np.median(times)), msamples_per_s=float(n / np.median(times) / 1e6),
                x_realtime=float(n / np.median(times) / 45e6), cadus_out=int(nf),
                stage_ms=dict(agc_fir=float(st[0]), costas=float(st[1]), mm_main_and_repairs=float(st[2]), viterbi=float(st[3]),
                              deframe_rs=float(st[4])),
                demod_repairs=int(ds["repairs"]), mm_segments=int(mm.size), segment_len=int(L), mm_warmup=W,
                warmup_share=float(mm.size * (L + W) / n))


def reference_rate(soft):
    from oracle import eos as O
    if not O.available():
        return None
    t = time.perf_counter()
    O.Aqua().run(soft)
    return soft.size / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--soft-mib", type=int, default=64, help="soft bytes per decoder push, MiB")
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--chain-log2", type=int, default=24, help="log2 of the IQ samples of the chain run")
    ap.add_argument("--ref-mib", type=int, default=8, help="soft bytes the reference runs for its rate, MiB")
    a = ap.parse_args()
    from satdump_b200 import synth
    nbytes = a.soft_mib << 20
    nfr = nbytes // 8192
    bits, sent = synth.aqua_db_frames(64, 7)
    locked = synth.aqua_db_soft(np.tile(bits.reshape(-1), nfr // 64 + 1)[:nbytes], sigma=10.0, seed=1)

    def check(got):
        assert got.shape[0] >= nfr - 2 and all(any(np.array_equal(got[k, :896], c[:896]) for c in sent) for k in range(0, got.shape[0], 101)), \
            "locked stream: output differs from the transmitted frames"

    noise = np.clip(np.round(np.random.default_rng(3).normal(0, 60, nbytes)), -127, 127).astype(np.int8)
    out = dict(repeats=a.repeats, locked=summary(time_decoder(locked, a.repeats, check), locked.size),
               noise=summary(time_decoder(noise, a.repeats), noise.size),
               chain_sync=time_chain(a.chain_log2, a.repeats, False), chain_pipelined=time_chain(a.chain_log2, a.repeats, True),
               terra=time_terra(a.chain_log2, a.repeats))
    nr = a.ref_mib << 20
    out["reference_single_thread"] = dict(locked_soft_bytes_per_s=reference_rate(locked[:nr]), noise_soft_bytes_per_s=reference_rate(noise[:nr]))
    out.update(card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
