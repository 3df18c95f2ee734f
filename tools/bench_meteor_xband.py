"""Throughput of meteor_xband_decoder (the METEOR-M MTVZA dump and KMSS BPSK DB pipelines' decoder behind psk_demod BPSK) on the GPU.

  decoder    the decoder alone on a soft stream pushed from host memory: a locked stream and noise
  chain      IQ (cs16 at two samples per symbol: MTVZA 30.72 MS/s, KMSS 122.88 MS/s) -> psk_demod BPSK -> the decoder through the fused
             chain, synchronous, one push
  reference  the reference's module loop (oracle/_ref/libsatref_xband.so, 8192-byte reads) on one CPU thread of this host, on the same
             locked stream; null where it was not built

Each timing is a host clock around calls that end in a device synchronise (a push returns after its frames are written), after one
warm-up call of the same shape. Prints one JSON line with the card, its power limit and SM clock read in the same run. Every timed locked
push is checked against the transmitted frames (99 % of them). Real time is 15 360 000 (MTVZA) and 61 440 000 (KMSS) soft bytes/s.

Usage: python tools/bench_meteor_xband.py [--soft-mib 64] [--repeats 5] [--chain-log2 24]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

REALTIME = dict(meteor_mtvza=15360000.0, meteor_kmss_bpsk=61440000.0)


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


def locked_stream(kmss, nbytes):
    """a whole number of reads of soft bytes carrying frames (a fresh decoder finds them all), and the frames"""
    from satdump_b200 import synth
    per = synth.KMSS_FRM * 8 * 1536 / 1504 if kmss else synth.MTVZA_FRM * 8 * 384 / 368
    bits, sent = synth.meteor_xband_frames(kmss, int(nbytes / per) + 2, seed=1)
    bits = np.concatenate([[0], bits])[:nbytes]
    rng = np.random.default_rng(2)
    soft = np.clip(np.round((bits.astype(np.float32) * 2 - 1) * 60 + rng.normal(0, 10, bits.size)), -127, 127).astype(np.int8)
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
    from oracle import xband as O
    res = dict(card())
    n = a.soft_mib << 20
    for name in ("meteor_mtvza", "meteor_kmss_bpsk"):
        kmss = name == "meteor_kmss_bpsk"
        cfg = capi.meteor_xband_cfg("kmss_bpsk" if kmss else "mtvza", max_soft=n)
        soft, sent = locked_stream(kmss, n)
        noise = np.clip(np.round(np.random.default_rng(3).normal(0, 90, n)), -127, 127).astype(np.int8)
        f = capi.Fec(cfg)
        got = f.push(soft).frames()
        # (random record bytes may match three of MTVZA's four patterns, and random payload a sync word, by chance: the reference then
        # writes a few frames that were not sent, and so does the decoder)
        sent_set = {bytes(x) for x in sent}
        assert got.shape[0] >= 0.99 * sent.shape[0] - 3 and sum(bytes(x) in sent_set for x in got) >= 0.99 * got.shape[0] - 2, "locked push lost frames"
        t_lock = timed(lambda: f.push(soft).frames(), a.repeats)
        t_noise = timed(lambda: f.push(noise).frames(), a.repeats)
        f.close()
        r = dict(frames_per_push=int(got.shape[0]), decoder_locked_GBps=n / t_lock / 1e9, decoder_noise_GBps=n / t_noise / 1e9,
                 decoder_locked_x_realtime=n / t_lock / REALTIME[name], decoder_noise_x_realtime=n / t_noise / REALTIME[name])
        sig = synth.CONFIGS[name]
        ns = 1 << a.chain_log2
        raw, _ = synth.make_signal(sig, ns, seed=5, device="cuda")
        raw = raw.cpu().numpy()
        ch = capi.Chain(capi.demod_cfg_for(sig, max_batch=ns), capi.fec_cfg_for(sig, max_soft=ns))
        t_chain = timed(lambda: (ch.push(raw), ch.frames()), a.repeats)
        ch.close()
        r.update(chain_MSps=ns / t_chain / 1e6, chain_x_realtime=ns / t_chain / sig.samplerate)
        if O.available():
            m = min(n, 1 << 24)
            ref = O.Ref(int(kmss))
            t0 = time.perf_counter()
            ref.run(soft[:m])
            r.update(reference_1thread_MBps=m / (time.perf_counter() - t0) / 1e6,
                     reference_x_realtime=m / (time.perf_counter() - t0) / REALTIME[name])
        else:
            r.update(reference_1thread_MBps=None)
        res[name] = r
    print(json.dumps(res))


if __name__ == "__main__":
    main()
